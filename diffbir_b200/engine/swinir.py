"""Stage-1 SwinIR forward on the sm_90a kernels.

Replaces SwinIR.forward / forward_features (reference model/swinir.py:856-894, 841-854), RSTB
(:487-488), SwinTransformerBlock.forward (:245-285) and WindowAttention.forward (:120-151)
for configs/inference/swinir.yaml (PixelUnshuffle 8, dim 180, 6 heads x 30, window 8,
mlp ratio 2, 'nearest+conv' x8 tail).

Awkward widths are padded once, in the packed weights: the 180-wide token stream lives in
fp32 rows of stride 192 (pad columns stay zero), every GEMM K is padded 180->192 / 360->384
with zero weights, so all TMA rows are 16-byte multiples and conv channel blocks are 64 wide.
"""
from __future__ import annotations

from typing import Dict

import torch

from .. import arch, lib
from .common import GraphCache, Workspace, f32, op16, pack_conv3x3, pack_linear


def _pad_to(n: int, m: int) -> int:
    return (n + m - 1) // m * m


class SwinIREngine:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: dict = None, device="cuda"):
        self.cfg = dict(arch.SWINIR_CFG if cfg is None else cfg)
        cfg = self.cfg
        self.dev = torch.device(device)
        if "state_dict" in sd:
            sd = sd["state_dict"]
        if next(iter(sd)).startswith("module."):
            sd = {k[len("module."):]: v for k, v in sd.items()}
        shapes = arch.swinir_shapes(cfg)
        for k, shp in shapes.items():
            if k not in sd:
                raise KeyError(f"SwinIR checkpoint is missing {k}")
            if tuple(sd[k].shape) != tuple(shp):
                raise ValueError(f"{k}: {tuple(sd[k].shape)} != {shp}")
        assert cfg["window_size"] == 8 and set(cfg["num_heads"]) == {6} and cfg["embed_dim"] == 180, \
            "window attention kernel is built for window 8, 6 heads x 30"
        self.ws = Workspace(self.dev)
        self.graphs = GraphCache(self.ws)       # ~360 launches per image replayed as one graph per input shape
        self.op_dtype = lib.operand_dtype()
        c = cfg["embed_dim"]
        self.c, self.cp = c, _pad_to(c, 64)                     # 180 -> 192
        self.hid = int(c * cfg["mlp_ratio"])
        self.hidp = _pad_to(self.hid, 64)                       # 360 -> 384
        self.qkv_ld = _pad_to(3 * c, 8)                         # 540 -> 544
        self.in_ch = cfg["in_chans"] * cfg["unshuffle_scale"] ** 2   # 192
        self.in_chp = _pad_to(self.in_ch, 64)
        self.nf = cfg.get("num_feat", 64)
        dev, w = self.dev, {}
        self.w = w
        w["conv_first.w"] = pack_conv3x3(sd["conv_first.1.weight"], dev, self.in_chp)
        w["conv_first.b"] = f32(sd["conv_first.1.bias"], dev)
        for nm in ("patch_embed.norm", "norm"):
            w[nm + ".weight"] = f32(sd[nm + ".weight"], dev)
            w[nm + ".bias"] = f32(sd[nm + ".bias"], dev)
        for li, depth in enumerate(cfg["depths"]):
            for bi in range(depth):
                p = f"layers.{li}.residual_group.blocks.{bi}."
                for nm in ("norm1", "norm2"):
                    w[p + nm + ".weight"] = f32(sd[p + nm + ".weight"], dev)
                    w[p + nm + ".bias"] = f32(sd[p + nm + ".bias"], dev)
                w[p + "qkv.w"] = pack_linear(sd[p + "attn.qkv.weight"], dev, self.cp)
                w[p + "qkv.b"] = f32(sd[p + "attn.qkv.bias"], dev)
                w[p + "proj.w"] = pack_linear(sd[p + "attn.proj.weight"], dev, self.cp)
                w[p + "proj.b"] = f32(sd[p + "attn.proj.bias"], dev)
                w[p + "rpb"] = f32(sd[p + "attn.relative_position_bias_table"], dev)
                w[p + "fc1.w"] = pack_linear(sd[p + "mlp.fc1.weight"], dev, self.cp)
                w[p + "fc1.b"] = f32(sd[p + "mlp.fc1.bias"], dev)
                w[p + "fc2.w"] = pack_linear(sd[p + "mlp.fc2.weight"], dev, self.hidp)
                w[p + "fc2.b"] = f32(sd[p + "mlp.fc2.bias"], dev)
            w[f"layers.{li}.conv.w"] = pack_conv3x3(sd[f"layers.{li}.conv.weight"], dev, self.cp)
            w[f"layers.{li}.conv.b"] = f32(sd[f"layers.{li}.conv.bias"], dev)
        w["conv_after_body.w"] = pack_conv3x3(sd["conv_after_body.weight"], dev, self.cp)
        w["conv_after_body.b"] = f32(sd["conv_after_body.bias"], dev)
        w["conv_before_upsample.w"] = pack_conv3x3(sd["conv_before_upsample.0.weight"], dev, self.cp)
        w["conv_before_upsample.b"] = f32(sd["conv_before_upsample.0.bias"], dev)
        self.n_up = {2: 1, 4: 2, 8: 3}[cfg["sf"]]
        for i in range(1, self.n_up + 1):
            w[f"conv_up{i}.w"] = pack_conv3x3(sd[f"conv_up{i}.weight"], dev)
            w[f"conv_up{i}.b"] = f32(sd[f"conv_up{i}.bias"], dev)
        w["conv_hr.w"] = pack_conv3x3(sd["conv_hr.weight"], dev)
        w["conv_hr.b"] = f32(sd["conv_hr.bias"], dev)
        lw = sd["conv_last.weight"]
        w["conv_last.w"] = f32(lw.permute(0, 2, 3, 1).reshape(lw.shape[0], -1), dev)
        w["conv_last.b"] = f32(sd["conv_last.bias"], dev)
        self.mean = (0.4488, 0.4371, 0.4040)                    # swinir.py:687-689
        r = cfg["img_range"]
        self.post_shift = torch.tensor(self.mean, dtype=torch.float32, device=dev)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x fp32 NCHW [nb, 3, H, W] in [0, 1], H and W multiples of 64 -> same shape (CUDA-graphed)."""
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        return self.graphs.run(tuple(x.shape), self._forward, x)

    def _forward(self, x: torch.Tensor) -> torch.Tensor:
        cfg, ws, W = self.cfg, self.ws, self.w
        nb, _, H, Wd = x.shape
        r = cfg["unshuffle_scale"]
        assert H % (r * 8) == 0 and Wd % (r * 8) == 0, "input must be padded to a multiple of 64"
        h, w = H // r, Wd // r
        M = nb * h * w
        c, cp = self.c, self.cp
        rng = float(cfg["img_range"])
        dt = self.op_dtype
        # stem: normalise + PixelUnshuffle -> op16 NHWC, then conv3x3 192 -> 180 (swinir.py:700-705)
        stem = ws.get("stem16", (M, self.in_chp), dt)
        lib.swin_stem(x, nb, H, Wd, r, self.mean, rng, self.in_chp, stem)
        feat0 = ws.get("feat0", (M, cp), torch.float32, zero=True)
        lib.gemm(stem, W["conv_first.w"], feat0, M=M, N=c, K=9 * self.in_chp, bias=W["conv_first.b"],
                 conv=(nb, h, w, self.in_chp, 3), ldo=cp)
        # tokens: patch_embed LayerNorm (fp32 result is needed as the residual stream)
        t = ws.get("tok", (M, cp), torch.float32, zero=True)
        ln16 = ws.get("ln16", (M, cp), dt)
        lib.layernorm(feat0, cp, M, c, W["patch_embed.norm.weight"], W["patch_embed.norm.bias"], t, cp)
        qkv = ws.get("qkv16", (M, self.qkv_ld), dt, zero=True)
        att = ws.get("att16", (M, cp), dt, zero=True)
        hid = ws.get("hid16", (M, self.hidp), dt, zero=True)
        rstb_in = ws.get("rstb_in", (M, cp), torch.float32, zero=True)
        img16 = ws.get("img16", (M, cp), dt)
        for li, depth in enumerate(cfg["depths"]):
            rstb_in.copy_(t)
            for bi in range(depth):
                p = f"layers.{li}.residual_group.blocks.{bi}."
                shift = 0 if bi % 2 == 0 else 4
                lib.layernorm(t, cp, M, c, W[p + "norm1.weight"], W[p + "norm1.bias"], ln16, cp)
                lib.gemm(ln16, W[p + "qkv.w"], qkv, M=M, N=3 * c, K=cp, bias=W[p + "qkv.b"], ldo=self.qkv_ld)
                lib.swin_window_attention(qkv, self.qkv_ld, nb, h, w, shift, W[p + "rpb"], att, cp)
                lib.gemm(att, W[p + "proj.w"], t, M=M, N=c, K=cp, bias=W[p + "proj.b"], residual=t,
                         ldo=cp, ldr=cp)
                lib.layernorm(t, cp, M, c, W[p + "norm2.weight"], W[p + "norm2.bias"], ln16, cp)
                lib.gemm(ln16, W[p + "fc1.w"], hid, M=M, N=self.hid, K=cp, bias=W[p + "fc1.b"], act="gelu",
                         ldo=self.hidp)
                lib.gemm(hid, W[p + "fc2.w"], t, M=M, N=c, K=self.hidp, bias=W[p + "fc2.b"], residual=t,
                         ldo=cp, ldr=cp)
            # RSTB tail: conv3x3 over the token image + residual (swinir.py:487-488)
            lib.gn_apply(t, None, cp, 0, nb, h, w, None, None, None, img16, norm=False, silu=False)
            lib.gemm(img16, W[f"layers.{li}.conv.w"], t, M=M, N=c, K=9 * cp, bias=W[f"layers.{li}.conv.b"],
                     residual=rstb_in, conv=(nb, h, w, cp, 3), ldo=cp, ldr=cp)
        lib.layernorm(t, cp, M, c, W["norm.weight"], W["norm.bias"], ln16, cp)
        body = ws.get("body", (M, cp), torch.float32, zero=True)
        lib.gemm(ln16, W["conv_after_body.w"], body, M=M, N=c, K=9 * cp, bias=W["conv_after_body.b"],
                 residual=feat0, conv=(nb, h, w, cp, 3), ldo=cp, ldr=cp)
        # reconstruction tail (swinir.py:876-885)
        lib.gn_apply(body, None, cp, 0, nb, h, w, None, None, None, img16, norm=False, silu=False)
        nf = self.nf
        cur = ws.get("tail_a", (M, nf), dt)
        lib.gemm(img16, W["conv_before_upsample.w"], cur, M=M, N=nf, K=9 * cp, bias=W["conv_before_upsample.b"],
                 act="lrelu", act_param=0.01, conv=(nb, h, w, cp, 3))
        ch, cw = h, w
        for i in range(1, self.n_up + 1):
            up = ws.get("tail_up", (nb * 4 * ch * cw, nf), dt)
            lib.upsample2x_op16(cur, nb, ch, cw, nf, up)
            ch, cw = 2 * ch, 2 * cw
            nxt = ws.get(f"tail_{'b' if i % 2 else 'a'}", (nb * ch * cw, nf), dt)
            lib.gemm(up, W[f"conv_up{i}.w"], nxt, M=nb * ch * cw, N=nf, K=9 * nf, bias=W[f"conv_up{i}.b"],
                     act="lrelu", act_param=0.2, conv=(nb, ch, cw, nf, 3))
            cur = nxt
        hr = ws.get("tail_hr", (nb * ch * cw, nf), dt)
        lib.gemm(cur, W["conv_hr.w"], hr, M=nb * ch * cw, N=nf, K=9 * nf, bias=W["conv_hr.b"],
                 act="lrelu", act_param=0.2, conv=(nb, ch, cw, nf, 3))
        out = torch.empty(nb, 3, ch, cw, dtype=torch.float32, device=self.dev)
        lib.conv3x3_small_cout(hr, nb, ch, cw, nf, W["conv_last.w"], W["conv_last.b"], 3, out, nchw=True,
                               post_scale=1.0 / rng, post_shift=self.post_shift)
        return out

