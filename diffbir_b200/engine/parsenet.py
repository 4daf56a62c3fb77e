"""ParseNet (facexlib parsenet, the unaligned-face loop's face parser) on the sm_90a kernels.

Every ConvLayer of ParseNet pads by reflection, and some also stride by 2 or read a nearest-2x up-sampled input, so
each convolution is dbir_patch_gather (reflection, stride, up-sampling fused) + a matrix-mode GEMM. Eval-mode
BatchNorm is folded into the weights in fp32; LeakyReLU(0.2) sits in the GEMM epilogue; a residual block's second
conv adds the fp32 shortcut in its epilogue. An up block's shortcut and conv1 read the same gathered patches.
Only out_mask_conv runs (the loop reads only the mask); its 19 logits per pixel become the 0/255 face mask in
dbir_parse_mask.

The faces of one call run in batches of at most MAX_BATCH, which bounds the workspace (about 0.94 GB per face, most
of it the 512^2 x 1152 patch matrix of the last decoder block) whatever the number of faces x samples. BatchNorm is in
eval mode and split-K is off, so every output row is summed in the same order whatever the batch: a batch is
bit-identical to single-face calls.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np
import torch

from .. import arch, lib
from .common import Workspace, f32, pack_linear

SIZE = 512
MAX_BATCH = 4            # faces per forward


def _pack(wt: torch.Tensor, dev, n_pad: int = 0) -> torch.Tensor:
    co = wt.shape[0]
    flat = wt.permute(0, 2, 3, 1).reshape(co, -1)
    flat = torch.nn.functional.pad(flat, (0, (-flat.shape[1]) % 64, 0, max(0, n_pad - co)))
    return pack_linear(flat, dev)


class ParseNetEngine:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: dict = None, device="cuda"):
        self.cfg = dict(arch.PARSENET_CFG if cfg is None else cfg)
        sd = arch.parsenet_state_dict(sd, self.cfg)
        self.dev = torch.device(device)
        self.ws = Workspace(self.dev)
        self.blocks = arch.parsenet_blocks(self.cfg)
        dev, w = self.dev, {}

        def layer(name, bn=False, n_pad=0):
            wt, b = sd[name + "conv2d.weight"], sd.get(name + "conv2d.bias")
            if bn:
                wt, b = arch.fold_bn(wt, sd, name + "norm.norm", b)
            w[name + "w"] = _pack(wt, dev, n_pad)
            w[name + "b"] = f32(torch.nn.functional.pad(b.float(), (0, max(0, n_pad - b.shape[0]))), dev)

        layer("encoder.0.")
        for p, ci, co, scale in self.blocks:
            if scale != "none" or ci != co:
                layer(p + "shortcut_func.")
            layer(p + "conv1.", bn=True)
            layer(p + "conv2.", bn=True)
        self.classes = self.cfg["parsing_ch"]
        self.n_mask = (self.classes + 31) // 32 * 32          # 19 logits in rows of 32 (16-byte GEMM output rows)
        layer("out_mask_conv.", n_pad=self.n_mask)
        self.w = w

    def _conv(self, x, n, h, w, c, name, out, *, stride=1, up2=False, act=False, residual=None, g=None):
        """ConvLayer: reflection-padded 3x3 conv of op16 x [n*h*w, c]; returns (ho, wo, gathered patches)."""
        ho, wo = lib.patch_gather_shape(h, w, 3, stride, up2)
        kp = (9 * c + 63) // 64 * 64
        if g is None:
            g = self.ws.get("g", (n * ho * wo, kp), lib.operand_dtype())
            lib.patch_gather(x, c, n, h, w, c, 3, stride, kp, g, reflect=True, up2=up2)
        W = self.w
        lib.gemm(g, W[name + "w"], out, M=n * ho * wo, N=W[name + "w"].shape[0], K=kp, bias=W[name + "b"],
                 act="lrelu" if act else None, act_param=0.2, residual=residual, split_k=1)
        return ho, wo, g

    def logits(self, x16: torch.Tensor, n: int) -> torch.Tensor:
        """op16 NHWC input [n*512*512, 3] -> fp32 mask logits [n*512*512, 32] (first 19 columns)."""
        ws, dt = self.ws, lib.operand_dtype()
        h = w = SIZE
        c = self.cfg["base_ch"]
        x = ws.get("x0", (n * h * w, c), dt)
        self._conv(x16, n, h, w, 3, "encoder.0.", x)
        x32 = feat = None
        flip = 0
        for p, ci, co, scale in self.blocks:
            if p.startswith("body.") and feat is None:             # the encoder output, kept for the body's skip
                feat = ws.get("feat", (n * h * w, ci), torch.float32)
                lib.axpby_cast(x32, 1.0, None, n * h * w, ci, y=feat)
            if p.startswith("decoder.") and feat is not None:      # x = feat + body(feat)
                lib.axpby_cast(x32, 1.0, feat, n * h * w, ci, y=x32, y16=x, ld16=ci)
                feat = None
            ho, wo = (h // 2, w // 2) if scale == "down" else ((2 * h, 2 * w) if scale == "up" else (h, w))
            Mo = n * ho * wo
            r = ws.get("r", (Mo if scale == "up" else n * h * w, co), dt)
            out32 = ws.get(f"s{flip}", (Mo, co), torch.float32)
            if scale == "up":
                idn = ws.get("idn", (Mo, co), torch.float32)
                _, _, g = self._conv(x, n, h, w, ci, p + "shortcut_func.", idn, up2=True)
                self._conv(x, n, h, w, ci, p + "conv1.", r, up2=True, act=True, g=g)
                self._conv(r, n, ho, wo, co, p + "conv2.", out32, residual=idn)
            elif scale == "down":
                idn = ws.get("idn", (Mo, co), torch.float32)
                self._conv(x, n, h, w, ci, p + "shortcut_func.", idn, stride=2)
                self._conv(x, n, h, w, ci, p + "conv1.", r, act=True)
                self._conv(r, n, h, w, co, p + "conv2.", out32, stride=2, residual=idn)
            else:
                self._conv(x, n, h, w, ci, p + "conv1.", r, act=True)
                self._conv(r, n, h, w, co, p + "conv2.", out32, residual=x32)
            x = ws.get(f"x{flip}", (Mo, co), dt)
            lib.axpby_cast(out32, 1.0, None, Mo, co, y16=x, ld16=co)
            x32, h, w, flip = out32, ho, wo, flip ^ 1
        logits = ws.get("logits", (n * h * w, self.n_mask), torch.float32)
        self._conv(x, n, h, w, x.shape[1], "out_mask_conv.", logits)
        return logits

    def masks(self, faces: Sequence[np.ndarray]) -> List[np.ndarray]:
        """512x512 RGB uint8 faces -> uint8 masks in {0, 255} (img2tensor's BGR swap and (x/255 - 0.5)/0.5 applied)."""
        assert all(f.shape == (SIZE, SIZE, 3) and f.dtype == np.uint8 for f in faces)
        out = []
        for i in range(0, len(faces), MAX_BATCH):
            out += self._masks(faces[i:i + MAX_BATCH])
        return out

    def _masks(self, faces: Sequence[np.ndarray]) -> List[np.ndarray]:
        n = len(faces)
        src = torch.from_numpy(np.stack(faces)).to(self.dev)
        x16 = self.ws.get("in16", (n * SIZE * SIZE, 3), lib.operand_dtype())
        lib.face_input(src, n, SIZE, SIZE, x16, scale=1.0 / 255.0, shift=(0.5, 0.5, 0.5), div=0.5, reverse=True)
        logits = self.logits(x16, n)
        out = torch.empty(n * SIZE * SIZE, dtype=torch.uint8, device=self.dev)
        lib.parse_mask(logits, self.n_mask, n * SIZE * SIZE, self.classes, out)
        return list(out.view(n, SIZE, SIZE).cpu().numpy())
