"""SCUNet (Swin-Conv-UNet, the v2 blind-denoising stage-1 cleaner) on the sm_90a kernels.

Replaces SCUNet.forward (reference model/scunet.py:221-243): head conv, three down stages, body, three up
stages of ConvTransBlocks (:126-156) joined by 2x2 stride-2 convs / transposed convs, tail conv.

A ConvTransBlock splits conv1_1(x) into a conv half (conv3x3 - ReLU - conv3x3 + skip) and a Swin half
(LN - window MSA 8x8, head_dim 32, alternating plain / shifted windows - LN - MLP), concatenates them and
adds conv1_2(cat) to x. Here both halves WRITE their 16-bit result straight into the two column ranges of one
[pixels, C] operand buffer (the concat never exists as a copy), the fp32 halves of conv1_1's output are read in
place through row strides (GEMM residual `ldr`, LayerNorm `ldx`), and the window attention reuses the SwinIR
kernel (same roll / partition / relative-position bias / region mask structure; -inf instead of -100 for the mask,
scunet.py:77). The 2x2 stride-2 convolutions are GEMMs over a space-to-depth view, the transposed ones a GEMM
followed by depth-to-space. fp32 NHWC residual stream, 16-bit tensor-core operands.
"""
from __future__ import annotations

from typing import Dict

import torch

from .. import arch, lib
from .common import GraphCache, Workspace, check_shapes, f32, pack_conv3x3, pack_linear

HEAD_DIM = 32


class SCUNetEngine:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: dict = None, device="cuda"):
        self.cfg = dict(arch.SCUNET_CFG if cfg is None else cfg)
        self.cfg["config"] = tuple(self.cfg["config"])
        self.dev = torch.device(device)
        cfg = self.cfg
        check_shapes(sd, arch.scunet_shapes(cfg), "SCUNet")
        if cfg["dim"] % 64:
            raise NotImplementedError("SCUNetEngine: dim must be a multiple of 64")
        self.ws = Workspace(self.dev)
        self.graphs = GraphCache(self.ws)
        self.op_dtype = lib.operand_dtype()
        w, dev = {}, self.dev
        hw_ = sd["m_head.0.weight"]
        w["head.w"] = f32(hw_.permute(2, 3, 1, 0).reshape(-1, hw_.shape[0]), dev)      # [9*in, dim] (stem kernel)
        w["head.b"] = torch.zeros(hw_.shape[0], dtype=torch.float32, device=dev)        # bias=False in the reference
        tw = sd["m_tail.0.weight"]
        w["tail.w"] = f32(tw.permute(0, 2, 3, 1).reshape(tw.shape[0], -1), dev)
        w["tail.b"] = torch.zeros(tw.shape[0], dtype=torch.float32, device=dev)
        for name, c, nblk, first in arch.scunet_stages(cfg):
            t = c // 2
            tp = max(t, 64)                                   # conv-branch channels padded to the 64-wide k-block
            if first:                                         # ConvTranspose2d [Cin, Cout, 2, 2] -> rows (ky, kx, co), K = ci
                tw_ = sd[f"{name}.0.weight"]
                w[f"{name}.up.w"] = pack_linear(tw_.permute(2, 3, 1, 0).reshape(-1, tw_.shape[0]), dev)
            for i in range(nblk):
                p = f"{name}.{first + i}."
                q = p + "trans_block."
                w[p + "c11.w"] = pack_linear(sd[p + "conv1_1.weight"], dev)
                w[p + "c11.b"] = f32(sd[p + "conv1_1.bias"], dev)
                w[p + "c11c.w"] = pack_linear(sd[p + "conv1_1.weight"][:t], dev)         # conv half again, as a 16-bit operand
                w[p + "c11c.b"] = f32(sd[p + "conv1_1.bias"][:t], dev)
                w[p + "c12.w"] = pack_linear(sd[p + "conv1_2.weight"], dev)
                w[p + "c12.b"] = f32(sd[p + "conv1_2.bias"], dev)
                w[p + "cb0.w"] = pack_conv3x3(sd[p + "conv_block.0.weight"], dev, cin_pad=tp)
                w[p + "cb2.w"] = pack_conv3x3(sd[p + "conv_block.2.weight"], dev, cin_pad=tp)
                for nm in ("ln1", "ln2"):
                    w[q + nm + ".w"] = f32(sd[q + nm + ".weight"], dev)
                    w[q + nm + ".b"] = f32(sd[q + nm + ".bias"], dev)
                kp = max(t, 64)                               # K of the width-t linears padded to one 64-wide k-block
                w[q + "qkv.w"] = pack_linear(sd[q + "msa.embedding_layer.weight"], dev, kp)
                w[q + "qkv.b"] = f32(sd[q + "msa.embedding_layer.bias"], dev)
                rp = sd[q + "msa.relative_position_params"]                              # [heads, 15, 15] -> [225, heads]
                w[q + "rpb"] = f32(rp.permute(1, 2, 0).reshape(-1, rp.shape[0]), dev)
                w[q + "lin.w"] = pack_linear(sd[q + "msa.linear.weight"], dev, kp)
                w[q + "lin.b"] = f32(sd[q + "msa.linear.bias"], dev)
                w[q + "fc1.w"] = pack_linear(sd[q + "mlp.0.weight"], dev, kp)
                w[q + "fc1.b"] = f32(sd[q + "mlp.0.bias"], dev)
                w[q + "fc2.w"] = pack_linear(sd[q + "mlp.2.weight"], dev)
                w[q + "fc2.b"] = f32(sd[q + "mlp.2.bias"], dev)
            if name.startswith("m_down"):                     # Conv2d [2c, c, 2, 2] -> [2c, (ky, kx, c)]
                dw = sd[f"{name}.{nblk}.weight"]
                w[f"{name}.down.w"] = pack_linear(dw.permute(0, 2, 3, 1).reshape(dw.shape[0], -1), dev)
        self.w = w

    # ------------------------------------------------------------------ one ConvTransBlock (scunet.py:147-156)
    def _block(self, p: str, x: torch.Tensor, x16: torch.Tensor, n: int, h: int, w_: int, c: int, shifted: bool):
        """In place on the fp32 stream x [M, c]; x16 is its 16-bit copy on entry and on exit."""
        ws, W, dt = self.ws, self.w, self.op_dtype
        M, t = n * h * w_, c // 2
        tp = max(t, 64)
        q = p + "trans_block."
        y = ws.get("y", (M, c), torch.float32)                                  # conv1_1(x): [conv half | Swin half]
        lib.gemm(x16, W[p + "c11.w"], y, M=M, N=c, K=c, bias=W[p + "c11.b"])
        # conv half: conv3x3 -> ReLU -> conv3x3, + conv_x  -> cat16[:, :t]
        c16 = ws.get(f"c16_{c}", (M, tp), dt, zero=True)                        # columns t..tp stay zero (zero weights anyway)
        lib.gemm(x16, W[p + "c11c.w"], c16, M=M, N=t, K=c, bias=W[p + "c11c.b"], ldo=tp)
        h16 = ws.get(f"h16_{c}", (M, tp), dt, zero=True)
        lib.gemm(c16, W[p + "cb0.w"], h16, M=M, N=t, K=9 * tp, act="lrelu", act_param=0.0, conv=(n, h, w_, tp, 3), ldo=tp)
        cat = ws.get("cat16", (M, c), dt)
        lib.gemm(h16, W[p + "cb2.w"], cat, M=M, N=t, K=9 * tp, residual=y, ldr=c, conv=(n, h, w_, tp, 3), ldo=c)
        # Swin half (Block.forward, scunet.py:120-123) on y[:, t:]  -> cat16[:, t:]
        yt = y[:, t:]
        kp = max(t, 64)                                                         # zero-padded K (see __init__)
        ln16 = ws.get(f"ln16_{c}", (M, kp), dt)
        lib.layernorm(yt, c, M, t, W[q + "ln1.w"], W[q + "ln1.b"], ln16, kp)    # columns t..kp are zero-filled
        qkv = ws.get("qkv16", (M, 3 * t), dt)
        lib.gemm(ln16, W[q + "qkv.w"], qkv, M=M, N=3 * t, K=kp, bias=W[q + "qkv.b"])
        att = ws.get(f"att16_{c}", (M, kp), dt, zero=True)
        lib.window_attention(qkv, 3 * t, n, h, w_, t // HEAD_DIM, HEAD_DIM, 4 if shifted else 0, W[q + "rpb"],
                             float("-inf"), att, kp)
        t1 = ws.get("t1", (M, t), torch.float32)
        lib.gemm(att, W[q + "lin.w"], t1, M=M, N=t, K=kp, bias=W[q + "lin.b"], residual=yt, ldr=c)
        lib.layernorm(t1, t, M, t, W[q + "ln2.w"], W[q + "ln2.b"], ln16, kp)
        hid = ws.get("hid16", (M, 4 * t), dt)
        lib.gemm(ln16, W[q + "fc1.w"], hid, M=M, N=4 * t, K=kp, bias=W[q + "fc1.b"], act="gelu")
        lib.gemm(hid, W[q + "fc2.w"], cat[:, t:], M=M, N=t, K=4 * t, bias=W[q + "fc2.b"], residual=t1, ldo=c)
        # x += conv1_2(cat)
        lib.gemm(cat, W[p + "c12.w"], x, M=M, N=c, K=c, bias=W[p + "c12.b"], residual=x)
        lib.axpby_cast(x, 1.0, None, M, c, y16=x16, ld16=c)

    def _stage(self, name: str, first: int, nblk: int, x, x16, n, h, w_, c):
        for i in range(nblk):
            self._block(f"{name}.{first + i}.", x, x16, n, h, w_, c, shifted=bool(i % 2))

    # ------------------------------------------------------------------ forward
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x fp32 NCHW [n, in_nc, H, W], H and W multiples of 64 -> same shape (CUDA-graphed per shape)."""
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()
        assert x.shape[2] % 64 == 0 and x.shape[3] % 64 == 0, "SCUNetEngine: pad the input to a multiple of 64"
        return self.graphs.run(tuple(x.shape), self._forward, x)

    def _forward(self, x0: torch.Tensor) -> torch.Tensor:
        cfg, ws, W, dt = self.cfg, self.ws, self.w, self.op_dtype
        n, cin, h, w_ = x0.shape
        stages = arch.scunet_stages(cfg)
        d = cfg["dim"]
        M = n * h * w_
        x = ws.get("s0", (M, d), torch.float32)                                 # x1 = m_head(x0)
        lib.conv3x3_small_cin(x0, None, cin, 0, n, h, w_, W["head.w"], W["head.b"], d, x)
        skips = []
        c = d
        for li, (name, c, nblk, first) in enumerate(stages[:3]):               # m_down1..3
            skips.append(x)
            cur = ws.get(f"cur{li}", (M, c), torch.float32)
            cur.copy_(x)                                                        # the stage works in place; x stays the skip
            x16 = ws.get(f"x16_{li}", (M, c), dt)
            lib.axpby_cast(cur, 1.0, None, M, c, y16=x16, ld16=c)
            self._stage(name, first, nblk, cur, x16, n, h, w_, c)
            # Conv2d(c, 2c, 2, 2): GEMM over the space-to-depth view [M/4, (ky, kx, c)]
            s2d = x16.view(n, h // 2, 2, w_ // 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(M // 4, 4 * c)
            h, w_, M = h // 2, w_ // 2, M // 4
            x = ws.get(f"s{li + 1}", (M, 2 * c), torch.float32)
            lib.gemm(s2d, W[f"{name}.down.w"], x, M=M, N=2 * c, K=4 * c)
        name, c, nblk, first = stages[3]                                        # m_body on x4 (x4 itself is a skip)
        skips.append(x)
        cur = ws.get("cur3", (M, c), torch.float32)
        cur.copy_(x)
        x16 = ws.get("x16_3", (M, c), dt)
        lib.axpby_cast(cur, 1.0, None, M, c, y16=x16, ld16=c)
        self._stage(name, first, nblk, cur, x16, n, h, w_, c)
        for li, (name, c, nblk, first) in enumerate(stages[4:]):               # m_up3, m_up2, m_up1
            skip = skips.pop()
            s16 = ws.get(f"sum16_{li}", (M, 2 * c), dt)
            lib.axpby_cast(cur, 1.0, skip, M, 2 * c, y16=s16, ld16=2 * c)       # (x + skip) as the transposed conv's operand
            up = ws.get(f"upo{li}", (M, 4 * c), torch.float32)                  # [M, (ky, kx, co)]
            lib.gemm(s16, W[f"{name}.up.w"], up, M=M, N=4 * c, K=2 * c)
            cur = up.view(n, h, w_, 2, 2, c).permute(0, 1, 3, 2, 4, 5).reshape(4 * M, c)     # depth-to-space (copy)
            h, w_, M = 2 * h, 2 * w_, 4 * M
            x16 = ws.get(f"x16u_{li}", (M, c), dt)
            lib.axpby_cast(cur, 1.0, None, M, c, y16=x16, ld16=c)
            self._stage(name, first, nblk, cur, x16, n, h, w_, c)
        x1 = skips.pop()
        t16 = ws.get("tail16", (M, d), dt)
        lib.axpby_cast(cur, 1.0, x1, M, d, y16=t16, ld16=d)
        out = torch.empty(n, cin, h, w_, dtype=torch.float32, device=self.dev)
        lib.conv3x3_small_cout(t16, n, h, w_, d, W["tail.w"], W["tail.b"], cin, out, nchw=True)
        return out
