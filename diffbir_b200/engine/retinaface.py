"""RetinaFace-ResNet50 (facexlib retinaface_resnet50, the unaligned-face loop's detector) on the sm_90a kernels.

- Input: the uint8 HWC image minus (104, 117, 123), cast to 16-bit operands (dbir_face_input; integers up to 255
  are exact in fp16 and bf16).
- ResNet-50 body: eval-mode BatchNorm folded into the convs in fp32. The 7x7 / stride-2 stem, the stride-2 3x3
  convs and the stride-2 1x1 downsample convs are dbir_patch_gather + a matrix-mode GEMM; 1x1 convs are plain GEMMs
  on the NHWC activations and the stride-1 3x3 convs run on dbir_gemm's conv mode. A bottleneck's conv3 adds the
  fp32 identity in its epilogue; dbir_relu_cast then writes the fp32 stream and the next operand.
- FPN: 1x1 output convs with ReLU, the top-down `a + nearest(b, size=a)` of dbir_fpn_add_up, 3x3 merge convs.
- SSH: the three branches write their ReLU'd outputs into column slots of one 256-channel buffer (ldo), which is
  ReLU(concat) since ReLU is per element.
- Heads: per level one 1x1 GEMM with N = 4 + 8 + 20 = 32 (class | box | landmarks) into one fp32 buffer whose rows
  run level by level, so prior p reads row p // 2; dbir_retinaface_decode computes the priors in-kernel and decodes
  scores, boxes and landmarks in input pixels.

Shapes change with every input size and dbir_gemm tunes a plan the first time it sees a signature, so the detector
runs eagerly (no per-size CUDA graph).
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch

from .. import arch, lib
from .common import Workspace, f32, op16, pack_conv3x3, pack_linear

DETECTOR_MEAN = (104.0, 117.0, 123.0)


def _pad64(k: int) -> int:
    return (k + 63) // 64 * 64


class RetinaFaceEngine:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: dict = None, device="cuda"):
        self.cfg = dict(arch.RETINAFACE_CFG if cfg is None else cfg)
        sd = arch.retinaface_state_dict(sd, self.cfg)
        self.dev = torch.device(device)
        self.ws = Workspace(self.dev)
        dev, w = self.dev, {}

        def conv(name, wt, bn, mode):
            wf, bf = arch.fold_bn(wt, sd, bn)
            if mode == "1x1":
                w[name + ".w"] = pack_linear(wf, dev)
            elif mode == "3x3":
                w[name + ".w"] = pack_conv3x3(wf, dev)
            else:                                              # gathered patches: K = taps * C, zero-padded to 64
                co = wf.shape[0]
                flat = wf.permute(0, 2, 3, 1).reshape(co, -1)
                w[name + ".w"] = pack_linear(flat, dev, _pad64(flat.shape[1]))
            w[name + ".b"] = f32(bf, dev)

        conv("stem", sd["body.conv1.weight"], "body.bn1", "gather")
        for li, blocks in enumerate(self.cfg["layers"]):
            for b in range(blocks):
                p = f"body.layer{li + 1}.{b}."
                s2 = b == 0 and li > 0
                conv(p + "conv1", sd[p + "conv1.weight"], p + "bn1", "1x1")
                conv(p + "conv2", sd[p + "conv2.weight"], p + "bn2", "gather" if s2 else "3x3")
                conv(p + "conv3", sd[p + "conv3.weight"], p + "bn3", "1x1")
                if b == 0:
                    conv(p + "down", sd[p + "downsample.0.weight"], p + "downsample.1", "1x1")
        for i in (1, 2, 3):
            conv(f"fpn.output{i}", sd[f"fpn.output{i}.0.weight"], f"fpn.output{i}.1", "1x1")
        for i in (1, 2):
            conv(f"fpn.merge{i}", sd[f"fpn.merge{i}.0.weight"], f"fpn.merge{i}.1", "3x3")
        for i in (1, 2, 3):
            for nm in ("conv3X3", "conv5X5_1", "conv5X5_2", "conv7X7_2", "conv7x7_3"):
                conv(f"ssh{i}.{nm}", sd[f"ssh{i}.{nm}.0.weight"], f"ssh{i}.{nm}.1", "3x3")
            hw = torch.cat([sd[f"{h}.{i - 1}.conv1x1.weight"] for h in ("ClassHead", "BboxHead", "LandmarkHead")])
            hb = torch.cat([sd[f"{h}.{i - 1}.conv1x1.bias"] for h in ("ClassHead", "BboxHead", "LandmarkHead")])
            w[f"head{i}.w"] = pack_linear(hw, dev)
            w[f"head{i}.b"] = f32(hb, dev)
        self.w = w
        self.oc = self.cfg["out_channel"]

    # ------------------------------------------------------------------ layers
    def _gemm(self, a, name, out, M, K, act=True, **kw):
        W = self.w
        lib.gemm(a, W[name + ".w"], out, M=M, N=W[name + ".w"].shape[0], K=K, bias=W[name + ".b"],
                 act="lrelu" if act else None, act_param=0.0, **kw)

    def _gathered(self, x, c, h, w, ksize, stride, name, out, tag, act=True):
        ho, wo = lib.patch_gather_shape(h, w, ksize, stride)
        kp = _pad64(ksize * ksize * c)
        g = self.ws.get(tag, (ho * wo, kp), lib.operand_dtype())
        lib.patch_gather(x, c, 1, h, w, c, ksize, stride, kp, g)
        self._gemm(g, name, out, ho * wo, kp, act=act)
        return ho, wo

    def heads(self, img: np.ndarray) -> torch.Tensor:
        """uint8 HWC image (channels used as given) -> fp32 head rows [sum of level pixels, 32]."""
        assert img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3
        ws, dt, W = self.ws, lib.operand_dtype(), self.w
        H, Wd = img.shape[:2]
        src = torch.from_numpy(np.ascontiguousarray(img)).to(self.dev)
        x = ws.get("in16", (H * Wd, 3), dt)
        lib.face_input(src, 1, H, Wd, x, shift=DETECTOR_MEAN)
        h1, w1 = lib.patch_gather_shape(H, Wd, 7, 2)
        stem = ws.get("stem", (h1 * w1, 64), dt)
        self._gathered(x, 3, H, Wd, 7, 2, "stem", stem, "g_stem")
        h, w = lib.patch_gather_shape(h1, w1, 3, 2)
        x16 = ws.get("pool", (h * w, 64), dt)
        lib.maxpool3s2(stem, 1, h1, w1, 64, x16)
        x32, cin, flip, feats = None, 64, 0, []
        for li, blocks in enumerate(self.cfg["layers"]):
            wd = 64 << li
            for b in range(blocks):
                p = f"body.layer{li + 1}.{b}."
                s2 = b == 0 and li > 0
                M = h * w
                t1 = ws.get("t1", (M, wd), dt)
                self._gemm(x16, p + "conv1", t1, M, cin)
                if s2:
                    ho, wo = lib.patch_gather_shape(h, w, 3, 2)
                    t2 = ws.get("t2", (ho * wo, wd), dt)
                    self._gathered(t1, wd, h, w, 3, 2, p + "conv2", t2, "g_c2")
                else:
                    ho, wo = h, w
                    t2 = ws.get("t2", (M, wd), dt)
                    self._gemm(t1, p + "conv2", t2, M, 9 * wd, conv=(1, h, w, wd, 3))
                Mo = ho * wo
                if b == 0:
                    idn = ws.get("idn", (Mo, 4 * wd), torch.float32)
                    if s2:
                        self._gathered(x16, cin, h, w, 1, 2, p + "down", idn, "g_down", act=False)
                    else:
                        self._gemm(x16, p + "down", idn, M, cin, act=False)
                else:
                    idn = x32
                out32 = ws.get(f"s{flip}", (Mo, 4 * wd), torch.float32)
                self._gemm(t2, p + "conv3", out32, Mo, wd, act=False, residual=idn)
                last = b == blocks - 1 and li > 0
                y16 = ws.get(f"c{li + 1}" if last else f"s16_{flip}", (Mo, 4 * wd), dt)
                lib.relu_cast(out32, Mo * 4 * wd, y16, y=out32)
                x16, x32, cin, h, w, flip = y16, out32, 4 * wd, ho, wo, flip ^ 1
                if last:
                    feats.append((y16, h, w))
        # FPN (facexlib net.py FPN.forward)
        oc = self.oc
        (c2, h2, w2), (c3, h3, w3), (c4, h4, w4) = feats
        o1 = ws.get("o1", (h2 * w2, oc), torch.float32)
        self._gemm(c2, "fpn.output1", o1, h2 * w2, c2.shape[1])
        o2 = ws.get("o2", (h3 * w3, oc), torch.float32)
        self._gemm(c3, "fpn.output2", o2, h3 * w3, c3.shape[1])
        o3 = ws.get("o3", (h4 * w4, oc), dt)
        self._gemm(c4, "fpn.output3", o3, h4 * w4, c4.shape[1])
        sum2 = ws.get("sum2", (h3 * w3, oc), dt)
        lib.fpn_add_up(o2, o3, 1, h3, w3, h4, w4, oc, sum2)
        m2 = ws.get("m2", (h3 * w3, oc), dt)
        self._gemm(sum2, "fpn.merge2", m2, h3 * w3, 9 * oc, conv=(1, h3, w3, oc, 3))
        sum1 = ws.get("sum1", (h2 * w2, oc), dt)
        lib.fpn_add_up(o1, m2, 1, h2, w2, h3, w3, oc, sum1)
        m1 = ws.get("m1", (h2 * w2, oc), dt)
        self._gemm(sum1, "fpn.merge1", m1, h2 * w2, 9 * oc, conv=(1, h2, w2, oc, 3))
        # SSH + heads
        levels = ((m1, h2, w2), (m2, h3, w3), (o3, h4, w4))
        rows = sum(hh * ww for _, hh, ww in levels)
        head = torch.empty(rows, 32, dtype=torch.float32, device=self.dev)
        off = 0
        for i, (f, hh, ww) in enumerate(levels, 1):
            M, q = hh * ww, oc // 4
            cv = dict(conv=(1, hh, ww, oc, 3))
            s = ws.get(f"ssh{i}", (M, oc), dt)
            self._gemm(f, f"ssh{i}.conv3X3", s, M, 9 * oc, ldo=oc, **cv)
            t = ws.get("ssh_t", (M, q), dt)
            self._gemm(f, f"ssh{i}.conv5X5_1", t, M, 9 * oc, **cv)
            cq = dict(conv=(1, hh, ww, q, 3))
            self._gemm(t, f"ssh{i}.conv5X5_2", s[:, oc // 2:], M, 9 * q, ldo=oc, **cq)
            t2 = ws.get("ssh_t2", (M, q), dt)
            self._gemm(t, f"ssh{i}.conv7X7_2", t2, M, 9 * q, **cq)
            self._gemm(t2, f"ssh{i}.conv7x7_3", s[:, oc // 2 + q:], M, 9 * q, ldo=oc, **cq)
            self._gemm(s, f"head{i}", head[off:off + M], M, oc, act=False)
            off += M
        return head

    def decode(self, head: torch.Tensor, h: int, w: int) -> torch.Tensor:
        out = torch.empty(2 * head.shape[0], 15, dtype=torch.float32, device=self.dev)
        lib.retinaface_decode(head, h, w, out)
        return out

    def candidates(self, img: np.ndarray):
        """Every prior of the image -> (boxes [P, 4], scores [P], landmarks [P, 10]) in input pixels, on the device."""
        out = self.decode(self.heads(img), img.shape[0], img.shape[1])
        return out[:, :4], out[:, 4], out[:, 5:]
