"""AutoencoderKL decode / encode on the sm_90a kernels.

Replaces AutoencoderKL.decode -> Decoder.forward (reference model/vae.py:579-582, 526-559)
and AutoencoderKL.encode -> Encoder.forward (vae.py:573-577, 347-371) for the SD VAE of
configs/inference/cldm.yaml (ch 128, mult 1-2-4-4, single-head mid attention of width 512).

fp32 NHWC residual stream; GroupNorm(eps 1e-6)+SiLU is applied while producing the 16-bit
operand of each implicit-GEMM convolution; the mid attention (head_dim = C = 512, outside the
64-wide flash kernel) runs as S = Q K^T (GEMM) -> row softmax -> P V^T (GEMM), with V^T
produced directly by a transposed GEMM so that every operand stays K-major.
"""
from __future__ import annotations

from typing import Dict

import torch

from .. import arch, lib
from .common import GraphCache, Workspace, f32, op16, pack_conv3x3, pack_linear


class VaeEngine:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: dict = None, device="cuda"):
        self.cfg = dict(arch.VAE_CFG if cfg is None else cfg)
        self.dev = torch.device(device)
        shapes = arch.vae_shapes(self.cfg)
        for k, shp in shapes.items():
            if k not in sd:
                raise KeyError(f"VAE checkpoint is missing {k}")
            if tuple(sd[k].shape) != tuple(shp):
                raise ValueError(f"{k}: {tuple(sd[k].shape)} != {shp}")
        self.ws = Workspace(self.dev)
        self.graphs = GraphCache(self.ws)       # decode / encode replayed as one graph per input shape
        self.op_dtype = lib.operand_dtype()
        self.w: Dict[str, torch.Tensor] = {}
        self._part = {}                          # fp32 activation data_ptr -> (GN partial-sum buffer, slots)
        w, dev = self.w, self.dev
        for k, v in sd.items():
            if k not in shapes:
                continue
            if v.dim() == 1:
                w[k] = f32(v, dev)
            elif k.endswith("conv_in.weight") or k in ("quant_conv.weight", "post_quant_conv.weight"):
                pass
            elif v.shape[-1] == 3 and v.shape[0] > 8 and v.shape[1] % 64 == 0:
                w[k] = pack_conv3x3(v, dev)
            elif v.shape[-1] == 1:
                w[k] = pack_linear(v, dev)
        for side in ("encoder.", "decoder."):
            cw = sd[side + "conv_in.weight"]
            w[side + "conv_in.weight"] = f32(cw.permute(2, 3, 1, 0).reshape(-1, cw.shape[0]), dev)
            ow = sd[side + "conv_out.weight"]
            w[side + "conv_out.weight"] = f32(ow.permute(0, 2, 3, 1).reshape(ow.shape[0], -1), dev)
            # fused q|k projection and the (row-major) v projection of the mid attention
            p = side + "mid.attn_1."
            c = sd[p + "q.weight"].shape[0]
            w[p + "qk.w"] = op16(torch.cat([sd[p + "q.weight"], sd[p + "k.weight"]], 0).reshape(2 * c, c), dev)
            w[p + "qk.b"] = f32(torch.cat([sd[p + "q.bias"], sd[p + "k.bias"]], 0), dev)
        w["quant_conv.weight"] = f32(sd["quant_conv.weight"].reshape(sd["quant_conv.weight"].shape[0], -1), dev)
        w["post_quant_conv.weight"] = f32(sd["post_quant_conv.weight"].reshape(sd["post_quant_conv.weight"].shape[0], -1), dev)

    # ------------------------------------------------------------------ blocks
    def _gn(self, x, c, nb, h, w, gamma, beta, out16, silu, out_raw=None):
        """GroupNorm(eps 1e-6)(+SiLU) -> 16-bit operand. Statistics come from the partial sums the
        producing conv's epilogue emitted (dbir_gemm gn_partials -> dbir_gn_finalize: no second read of
        the fp32 tensor); tensors written by other kernels take the stand-alone statistics pass."""
        ws = self.ws
        stats = ws.get("gn_stats", (nb * 64,), torch.float32)
        part = self._part.get(x.data_ptr())
        if part is not None:
            lib.gn_finalize(part[0], part[1], c, None, 0, 0, nb, h * w, 1e-6, stats)
        else:
            wsp = ws.get("gn_ws", (lib.gn_workspace_floats(nb, h * w, c),), torch.float32, zero=True)
            lib.gn_stats(x, None, c, 0, nb, h * w, 1e-6, stats, wsp)
        lib.gn_apply(x, None, c, 0, nb, h, w, stats, gamma, beta, out16, norm=True, silu=silu, out_raw=out_raw)

    def _stats_kw(self, out: torch.Tensor, nb: int, n_cols: int, h: int, w: int) -> dict:
        """kwargs that make a conv-mode dbir_gemm emit GroupNorm partial sums for its output `out`."""
        slots = lib.gemm_gn_slots(h, w)
        if slots <= 0:
            self._part.pop(out.data_ptr(), None)
            return {}
        buf = self.ws.get(f"part:{out.data_ptr()}", (nb * slots * n_cols * 2,), torch.float32)
        self._part[out.data_ptr()] = (buf, slots)
        return dict(gn_partials=buf)

    def _res(self, p, x, cin, cout, nb, h, w, out):
        """ResnetBlock.forward (temb None) — vae.py:97-117."""
        ws, W, M = self.ws, self.w, nb * h * w
        a16 = ws.get("a16", (M, cin), self.op_dtype)
        raw = ws.get("raw16", (M, cin), self.op_dtype) if cin != cout else None
        self._gn(x, cin, nb, h, w, W[p + "norm1.weight"], W[p + "norm1.bias"], a16, True, raw)
        h1 = ws.get("h1", (M, cout), torch.float32)
        lib.gemm(a16, W[p + "conv1.weight"], h1, M=M, N=cout, K=9 * cin, bias=W[p + "conv1.bias"],
                 conv=(nb, h, w, cin, 3), **self._stats_kw(h1, nb, cout, h, w))
        b16 = ws.get("b16", (M, cout), self.op_dtype)
        self._gn(h1, cout, nb, h, w, W[p + "norm2.weight"], W[p + "norm2.bias"], b16, True)
        if cin != cout:
            sk = ws.get("skip", (M, cout), torch.float32)
            lib.gemm(raw, W[p + "nin_shortcut.weight"], sk, M=M, N=cout, K=cin, bias=W[p + "nin_shortcut.bias"])
            res = sk
        else:
            res = x
        lib.gemm(b16, W[p + "conv2.weight"], out, M=M, N=cout, K=9 * cout, bias=W[p + "conv2.bias"],
                 residual=res, conv=(nb, h, w, cout, 3), **self._stats_kw(out, nb, cout, h, w))

    def release_buffers(self) -> None:
        """Frees the workspace and the captured encode / decode graphs; the next call re-creates them."""
        self.ws.clear()                          # also drops the graphs (GraphCache hooks on_grow)
        self._part.clear()

    @staticmethod
    def attn_rows(hw: int) -> int:
        """Query rows per chunk of the mid attention's materialised S: 8192 up to 65536 tokens (2048^2 images),
        beyond that a multiple of 128 that keeps the fp32 S at or below 2 GiB (3584 rows at 3072^2)."""
        return min(8192, max(128, (2 ** 31 // (4 * hw)) // 128 * 128))

    def _attn(self, p, x, c, nb, h, w):
        """Single-head attention over pixels, in place on x — vae.py:232-282."""
        ws, W, hw = self.ws, self.w, h * w
        M = nb * hw
        a16 = ws.get("a16", (M, c), self.op_dtype)
        self._gn(x, c, nb, h, w, W[p + "norm.weight"], W[p + "norm.bias"], a16, False)
        qk = ws.get("qk16", (M, 2 * c), self.op_dtype)
        lib.gemm(a16, W[p + "qk.w"], qk, M=M, N=2 * c, K=c, bias=W[p + "qk.b"])
        o16 = ws.get("o16", (M, c), self.op_dtype)
        rows = min(hw, self.attn_rows(hw))
        for b in range(nb):
            a_b = a16[b * hw:(b + 1) * hw]
            vt = ws.get("vt16", (c, hw), self.op_dtype)               # V^T [C, hw]
            lib.gemm(W[p + "v.weight"], a_b, vt, M=c, N=hw, K=c, bias=W[p + "v.bias"], bias_per_row=True)
            for r0 in range(0, hw, rows):
                r1 = min(hw, r0 + rows)
                s = ws.get("s32", (r1 - r0, hw), torch.float32)
                qb = qk[b * hw + r0: b * hw + r1]
                kb = qk[b * hw:(b + 1) * hw, c:]
                lib.gemm(qb, kb, s, M=r1 - r0, N=hw, K=c, lda=2 * c, ldb=2 * c)
                p16 = ws.get("p16", (r1 - r0, hw), self.op_dtype)
                lib.softmax_rows(s, hw, r1 - r0, hw, float(c) ** -0.5, p16, hw)
                lib.gemm(p16, vt, o16[b * hw + r0: b * hw + r1], M=r1 - r0, N=c, K=hw)
        lib.gemm(o16, W[p + "proj_out.weight"], x, M=M, N=c, K=c, bias=W[p + "proj_out.bias"], residual=x)
        self._part.pop(x.data_ptr(), None)                       # x changed in place: its partials are stale

    # ------------------------------------------------------------------ decode
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """z fp32 NCHW [nb, 4, h, w] (already divided by the scale factor) -> image fp32 NCHW
        [nb, 3, 8h, 8w] in [-1, 1]."""
        assert z.is_cuda and z.dtype == torch.float32 and z.is_contiguous()
        return self.graphs.run(("dec",) + tuple(z.shape), self._decode, z)

    def _decode(self, z: torch.Tensor) -> torch.Tensor:
        cfg, ws, W = self.cfg, self.ws, self.w
        nb, zc, h, w = z.shape
        ch, mult, nres = cfg["ch"], tuple(cfg["ch_mult"]), cfg["num_res_blocks"]
        # post_quant_conv (1x1, 4->4) on NHWC rows, fp32
        z_nhwc = ws.get("z_nhwc", (nb * h * w, zc), torch.float32)
        lib.nchw_to_nhwc(z, nb, zc, h * w, z_nhwc)
        z2 = ws.get("z2", (nb * h * w, zc), torch.float32)
        lib.linear_f32(z_nhwc, zc, nb * h * w, zc, W["post_quant_conv.weight"], W["post_quant_conv.bias"], zc, z2, zc)
        z2n = ws.get("z2n", (nb, zc, h, w), torch.float32)
        lib.nhwc_to_nchw(z2, nb, zc, h * w, z2n)
        p = "decoder."
        c = ch * mult[-1]
        x = ws.get("x0", (nb * h * w, c), torch.float32)
        lib.conv3x3_small_cin(z2n, None, zc, 0, nb, h, w, W[p + "conv_in.weight"], W[p + "conv_in.bias"], c, x)
        self._part.pop(x.data_ptr(), None)                       # written without GEMM partials
        self._res(p + "mid.block_1.", x, c, c, nb, h, w, x)
        self._attn(p + "mid.attn_1.", x, c, nb, h, w)
        self._res(p + "mid.block_2.", x, c, c, nb, h, w, x)
        cur, flip = x, 0
        for lvl in reversed(range(len(mult))):
            cout = ch * mult[lvl]
            for j in range(nres + 1):
                o = ws.get(f"x{1 + flip}", (nb * h * w, cout), torch.float32)
                self._res(f"{p}up.{lvl}.block.{j}.", cur, c, cout, nb, h, w, o)
                cur, c, flip = o, cout, flip ^ 1
            if lvl != 0:
                up16 = ws.get("a16", (nb * 4 * h * w, c), self.op_dtype)
                lib.gn_apply(cur, None, c, 0, nb, h, w, None, None, None, up16, norm=False, silu=False, upsample=2)
                o = ws.get(f"x{1 + flip}", (nb * 4 * h * w, c), torch.float32)
                lib.gemm(up16, W[f"{p}up.{lvl}.upsample.conv.weight"], o, M=nb * 4 * h * w, N=c, K=9 * c,
                         bias=W[f"{p}up.{lvl}.upsample.conv.bias"], conv=(nb, 2 * h, 2 * w, c, 3),
                         **self._stats_kw(o, nb, c, 2 * h, 2 * w))
                cur, flip, h, w = o, flip ^ 1, 2 * h, 2 * w
        a16 = ws.get("a16", (nb * h * w, c), self.op_dtype)
        self._gn(cur, c, nb, h, w, W[p + "norm_out.weight"], W[p + "norm_out.bias"], a16, True)
        out = torch.empty(nb, cfg["out_ch"], h, w, dtype=torch.float32, device=self.dev)
        lib.conv3x3_small_cout(a16, nb, h, w, c, W[p + "conv_out.weight"], W[p + "conv_out.bias"],
                               cfg["out_ch"], out, nchw=True)
        return out

    # ------------------------------------------------------------------ encode
    def encode_moments(self, img: torch.Tensor) -> torch.Tensor:
        """img fp32 NCHW [nb, 3, H, W] in [-1, 1] -> moments fp32 NCHW [nb, 8, H/8, W/8]."""
        assert img.is_cuda and img.dtype == torch.float32 and img.is_contiguous()
        return self.graphs.run(("enc",) + tuple(img.shape), self._encode_moments, img)

    def _encode_moments(self, img: torch.Tensor) -> torch.Tensor:
        cfg, ws, W = self.cfg, self.ws, self.w
        nb, ic, h, w = img.shape
        ch, mult, nres = cfg["ch"], tuple(cfg["ch_mult"]), cfg["num_res_blocks"]
        p = "encoder."
        c = ch
        cur = ws.get("x0", (nb * h * w, c), torch.float32)
        lib.conv3x3_small_cin(img, None, ic, 0, nb, h, w, W[p + "conv_in.weight"], W[p + "conv_in.bias"], c, cur)
        self._part.pop(cur.data_ptr(), None)                     # written without GEMM partials
        flip = 0
        for lvl in range(len(mult)):
            cout = ch * mult[lvl]
            for j in range(nres):
                o = ws.get(f"x{1 + flip}", (nb * h * w, cout), torch.float32)
                self._res(f"{p}down.{lvl}.block.{j}.", cur, c, cout, nb, h, w, o)
                cur, c, flip = o, cout, flip ^ 1
            if lvl != len(mult) - 1:
                ho, wo = h // 2, w // 2
                col = ws.get("a16", (nb * ho * wo, 9 * c), self.op_dtype)
                lib.im2col_s2(cur, nb, h, w, c, 0, col)
                o = ws.get(f"x{1 + flip}", (nb * ho * wo, c), torch.float32)
                lib.gemm(col, W[f"{p}down.{lvl}.downsample.conv.weight"], o, M=nb * ho * wo, N=c, K=9 * c,
                         bias=W[f"{p}down.{lvl}.downsample.conv.bias"])
                self._part.pop(o.data_ptr(), None)               # plain-mode GEMM: no partials requested
                cur, flip, h, w = o, flip ^ 1, ho, wo
        self._res(p + "mid.block_1.", cur, c, c, nb, h, w, cur)
        self._attn(p + "mid.attn_1.", cur, c, nb, h, w)
        self._res(p + "mid.block_2.", cur, c, c, nb, h, w, cur)
        a16 = ws.get("a16", (nb * h * w, c), self.op_dtype)
        self._gn(cur, c, nb, h, w, W[p + "norm_out.weight"], W[p + "norm_out.bias"], a16, True)
        zc2 = 2 * cfg["z_channels"]
        m_nhwc = ws.get("m_nhwc", (nb * h * w, zc2), torch.float32)
        lib.conv3x3_small_cout(a16, nb, h, w, c, W[p + "conv_out.weight"], W[p + "conv_out.bias"], zc2,
                               m_nhwc, nchw=False)
        q = ws.get("q_nhwc", (nb * h * w, zc2), torch.float32)
        lib.linear_f32(m_nhwc, zc2, nb * h * w, zc2, W["quant_conv.weight"], W["quant_conv.bias"], zc2, q, zc2)
        out = torch.empty(nb, zc2, h, w, dtype=torch.float32, device=self.dev)
        lib.nhwc_to_nchw(q, nb, zc2, h * w, out)
        return out

    def encode_mode(self, img: torch.Tensor, scale_factor: float = 0.18215) -> torch.Tensor:
        """ControlLDM.vae_encode(sample=False) — cldm.py:92-119: posterior mean * scale."""
        m = self.encode_moments(img)
        return (m[:, : m.shape[1] // 2] * scale_factor).contiguous()
