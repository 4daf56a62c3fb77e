"""RRDBNet (BSRNet stage-1 cleaner of the v2 recipe) on the sm_90a kernels.

Replaces RRDBNet.forward (reference model/bsrnet.py:89-104): conv_first, 23 RRDB blocks of three
5-convolution residual dense blocks (:36-73), trunk conv + skip, two nearest-2x + conv + LeakyReLU
stages, HRconv, conv_last. Convolution only, so everything runs on dbir_gemm's implicit-GEMM conv.

Data layout: the dense concatenation cat((x, x1, x2, x3, x4)) of a block (bsrnet.py:51-56) is ONE
16-bit NHWC buffer [pixels, nf + 4 gc] (192 channels): conv k reads its first nf + (k-1) gc channels
through the conv's pixel stride (dbir_gemm lda) and writes its LeakyReLU'd gc channels straight into
the next slot with the output row stride — no concat copies. The implicit GEMM walks K in 64-channel
blocks, so convs 2 and 4 (96 / 160 input channels) read up to the next multiple of 64 with zero
weights for the excess; that excess is the slot they are writing themselves (old or new finite
values times an exact zero weight: the result does not depend on it).
The block outputs x5 * 0.2 + x stay fp32 (residual stream) with a fused epilogue; one small pass
per block casts them into the next block's buffer and applies the RRDB-level `out * 0.2 + x`.
"""
from __future__ import annotations

from typing import Dict

import torch

from .. import arch, lib
from .common import GraphCache, Workspace, check_shapes, f32, pack_conv3x3, round_up


class RRDBNetEngine:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: dict = None, device="cuda"):
        self.cfg = dict(arch.RRDBNET_CFG if cfg is None else cfg)
        self.dev = torch.device(device)
        cfg = self.cfg
        check_shapes(sd, arch.rrdbnet_shapes(cfg), "RRDBNet")
        nf, gc = cfg["nf"], cfg["gc"]
        if nf % 64 or (nf + 4 * gc) % 64 or gc % 8:
            raise NotImplementedError("RRDBNetEngine: nf and nf + 4 gc must be multiples of 64, gc of 8")
        self.ws = Workspace(self.dev)
        self.graphs = GraphCache(self.ws)
        self.op_dtype = lib.operand_dtype()
        self.cat_c = nf + 4 * gc
        w, dev = {}, self.dev
        cw = sd["conv_first.weight"]                               # [nf, in, 3, 3] -> [9*in, nf] fp32 (stem kernel)
        w["conv_first.w"] = f32(cw.permute(2, 3, 1, 0).reshape(-1, cw.shape[0]), dev)
        w["conv_first.b"] = f32(sd["conv_first.bias"], dev)
        for b in range(cfg["nb"]):
            for r in (1, 2, 3):
                p = f"RRDB_trunk.{b}.RDB{r}."
                for k in range(1, 6):
                    cin = nf + (k - 1) * gc
                    w[p + f"conv{k}.w"] = pack_conv3x3(sd[p + f"conv{k}.weight"], dev, cin_pad=round_up(cin))
                    w[p + f"conv{k}.b"] = f32(sd[p + f"conv{k}.bias"], dev)
        for nm in ["trunk_conv", "upconv1"] + (["upconv2"] if cfg["sf"] == 4 else []) + ["HRconv"]:
            w[nm + ".w"] = pack_conv3x3(sd[nm + ".weight"], dev)
            w[nm + ".b"] = f32(sd[nm + ".bias"], dev)
        lw = sd["conv_last.weight"]
        w["conv_last.w"] = f32(lw.permute(0, 2, 3, 1).reshape(lw.shape[0], -1), dev)
        w["conv_last.b"] = f32(sd["conv_last.bias"], dev)
        self.w = w

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x fp32 NCHW [nb, in_nc, H, W] -> fp32 NCHW [nb, out_nc, sf*H, sf*W] (CUDA-graphed per shape)."""
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        return self.graphs.run(tuple(x.shape), self._forward, x)

    def _forward(self, x: torch.Tensor) -> torch.Tensor:
        cfg, ws, W, dt = self.cfg, self.ws, self.w, self.op_dtype
        n, cin, h, wd = x.shape
        nf, gc, C = cfg["nf"], cfg["gc"], self.cat_c
        M = n * h * wd
        fea = ws.get("fea", (M, nf), torch.float32)
        lib.conv3x3_small_cin(x, None, cin, 0, n, h, wd, W["conv_first.w"], W["conv_first.b"], nf, fea)
        cat = ws.get("cat16", (M, C), dt, zero=True)               # [x | x1 | x2 | x3 | x4] of the running block
        cur = [ws.get("rs0", (M, nf), torch.float32), ws.get("rs1", (M, nf), torch.float32)]
        rrdb_in = ws.get("rrdb_in", (M, nf), torch.float32)
        lib.axpby_cast(fea, 1.0, None, M, nf, y=rrdb_in, y16=cat, ld16=C)
        blk_in, flip = rrdb_in, 0
        for b in range(cfg["nb"]):
            for r in (1, 2, 3):
                p = f"RRDB_trunk.{b}.RDB{r}."
                for k in range(1, 5):                              # x_k = lrelu(conv_k(cat[:, :nf+(k-1)gc]))
                    ck = nf + (k - 1) * gc
                    ckp = round_up(ck)
                    lib.gemm(cat, W[p + f"conv{k}.w"], cat[:, ck:], M=M, N=gc, K=9 * ckp, bias=W[p + f"conv{k}.b"],
                             act="lrelu", act_param=0.2, conv=(n, h, wd, ckp, 3), lda=C, ldo=C)
                out = cur[flip]                                    # x5 * 0.2 + x (bsrnet.py:57-58), fp32
                lib.gemm(cat, W[p + "conv5.w"], out, M=M, N=nf, K=9 * C, bias=W[p + "conv5.b"], alpha=0.2,
                         residual=blk_in, conv=(n, h, wd, C, 3), lda=C)
                if r < 3:
                    lib.axpby_cast(out, 1.0, None, M, nf, y16=cat, ld16=C)
                    blk_in, flip = out, flip ^ 1
                else:                                              # RRDB: out * 0.2 + x (bsrnet.py:69-70)
                    lib.axpby_cast(out, 0.2, rrdb_in, M, nf, y=rrdb_in, y16=cat, ld16=C)
                    blk_in = rrdb_in
        a16 = ws.get("a16", (M, nf), dt)
        lib.axpby_cast(rrdb_in, 1.0, None, M, nf, y16=a16, ld16=nf)
        t16 = ws.get("t16", (M, nf), dt)                           # fea + trunk_conv(trunk), as the next operand
        lib.gemm(a16, W["trunk_conv.w"], t16, M=M, N=nf, K=9 * nf, bias=W["trunk_conv.b"], residual=fea,
                 conv=(n, h, wd, nf, 3))
        cur16, ch, cw = t16, h, wd
        for nm in ["upconv1"] + (["upconv2"] if cfg["sf"] == 4 else []):
            up = ws.get("up_" + nm, (n * 4 * ch * cw, nf), dt)
            lib.upsample2x_op16(cur16, n, ch, cw, nf, up)
            ch, cw = 2 * ch, 2 * cw
            nxt = ws.get("o_" + nm, (n * ch * cw, nf), dt)
            lib.gemm(up, W[nm + ".w"], nxt, M=n * ch * cw, N=nf, K=9 * nf, bias=W[nm + ".b"], act="lrelu", act_param=0.2,
                     conv=(n, ch, cw, nf, 3))
            cur16 = nxt
        hr = ws.get("hr16", (n * ch * cw, nf), dt)
        lib.gemm(cur16, W["HRconv.w"], hr, M=n * ch * cw, N=nf, K=9 * nf, bias=W["HRconv.b"], act="lrelu", act_param=0.2,
                 conv=(n, ch, cw, nf, 3))
        out = torch.empty(n, cfg["out_nc"], ch, cw, dtype=torch.float32, device=self.dev)
        lib.conv3x3_small_cout(hr, n, ch, cw, nf, W["conv_last.w"], W["conv_last.b"], cfg["out_nc"], out, nchw=True)
        return out
