"""AutoencoderKL decode / encode on the sm_90a kernels.

Replaces AutoencoderKL.decode -> Decoder.forward (reference model/vae.py:579-582, 526-559)
and AutoencoderKL.encode -> Encoder.forward (vae.py:573-577, 347-371) for the SD VAE of
configs/inference/cldm.yaml (ch 128, mult 1-2-4-4, single-head mid attention of width 512).

fp32 NHWC residual stream; GroupNorm(eps 1e-6)+SiLU is applied while producing the 16-bit
operand of each implicit-GEMM convolution; the mid attention (head_dim = C = 512, outside the
64-wide flash kernel) runs as S = Q K^T (GEMM) -> row softmax -> P V^T (GEMM), with V^T
produced directly by a transposed GEMM so that every operand stays K-major.

This file states the network once, for all three VAE engines: `VaeWalk` runs a batch through the encoder or
the decoder as a generator that stops at each GroupNorm and asks its driver for the statistics. `VaeEngine`
answers at once with the batch's own statistics, inside one CUDA graph per input shape; `vae_tiled.TiledVae`
merges the statistics of all tiles of an image before any of them goes on; `vae_sharded.ShardedVae` runs a band
of image rows per rank (`vae_sharded.BandWalk`, which overrides the few steps where a band differs from a whole
image) and merges the statistics of all bands.
"""
from __future__ import annotations

import itertools
from typing import Dict

import torch

from .. import arch, lib
from .common import GraphCache, Workspace, check_shapes, f32, op16, pack_conv3x3, pack_linear


class VaeEngine:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: dict = None, device="cuda"):
        self.cfg = dict(arch.VAE_CFG if cfg is None else cfg)
        self.dev = torch.device(device)
        shapes = arch.vae_shapes(self.cfg)
        check_shapes(sd, shapes, "VAE")
        self.ws = Workspace(self.dev)
        self.graphs = GraphCache(self.ws)       # decode / encode replayed as one graph per input shape
        self.op_dtype = lib.operand_dtype()
        self.w: Dict[str, torch.Tensor] = {}
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

    # ------------------------------------------------------------------ un-tiled driver
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """z fp32 NCHW [nb, 4, h, w] (already divided by the scale factor) -> image fp32 NCHW
        [nb, 3, 8h, 8w] in [-1, 1]."""
        assert z.is_cuda and z.dtype == torch.float32 and z.is_contiguous()
        return self.graphs.run(("dec",) + tuple(z.shape), self._decode, z)

    def _decode(self, z: torch.Tensor) -> torch.Tensor:
        return self._drive(VaeWalk.decoder, self.post_quant(z, self._scratch()))

    def encode_moments(self, img: torch.Tensor) -> torch.Tensor:
        """img fp32 NCHW [nb, 3, H, W] in [-1, 1] -> moments fp32 NCHW [nb, 8, H/8, W/8]."""
        assert img.is_cuda and img.dtype == torch.float32 and img.is_contiguous()
        return self.graphs.run(("enc",) + tuple(img.shape), self._encode_moments, img)

    def _encode_moments(self, img: torch.Tensor) -> torch.Tensor:
        return self.quant(self._drive(VaeWalk.encoder, img), self._scratch())

    def encode_mode(self, img: torch.Tensor, scale_factor: float = 0.18215) -> torch.Tensor:
        """ControlLDM.vae_encode(sample=False) — cldm.py:92-119: posterior mean * scale."""
        m = self.encode_moments(img)
        return (m[:, : m.shape[1] // 2] * scale_factor).contiguous()

    def _drive(self, net, x: torch.Tensor) -> torch.Tensor:
        """Runs the batch x through `net` (VaeWalk.encoder / .decoder), answering each GroupNorm at once with the
        batch's own statistics: from the partial sums the producing conv's epilogue emitted (dbir_gemm gn_partials
        -> dbir_gn_finalize: no second read of the fp32 tensor); tensors written by other kernels take the
        stand-alone statistics pass. The activations take the walk's three workspace buffers: these are all the
        full-resolution fp32 memory of the un-tiled VAE, which is what bounds the largest image that runs without
        tiling."""
        ws, nb = self.ws, x.shape[0]
        walk = VaeWalk(self, ws, nb)
        stats = ws.get("gn_stats", (nb * 64,), torch.float32)

        def answer(c, h, w, part, slots):
            if part is not None:
                lib.gn_finalize(part, slots, c, None, 0, 0, nb, h * w, 1e-6, stats)
            else:
                wsp = ws.get("gn_ws", (lib.gn_workspace_floats(nb, h * w, c),), torch.float32, zero=True)
                lib.gn_stats(walk.st["cur"], None, c, 0, nb, h * w, 1e-6, stats, wsp)
            return stats
        return walk.run(net, x, answer)

    def _scratch(self):
        """Allocator for the quant convs inside the graph: each call hands out a workspace buffer of its own."""
        n = itertools.count()
        return lambda *shape: self.ws.get(f"q{next(n)}", shape, torch.float32)

    def release_buffers(self) -> None:
        """Frees the workspace and the captured encode / decode graphs; the next call re-creates them."""
        self.ws.clear()                          # also drops the graphs (GraphCache hooks on_grow)

    # ------------------------------------------------------------------ the ends (un-tiled in both engines)
    def post_quant(self, z: torch.Tensor, new) -> torch.Tensor:
        """post_quant_conv (1x1, 4->4) on NHWC rows, fp32: z NCHW -> the decoder's input, NCHW. new(*shape)
        supplies the fp32 tensors."""
        nb, zc, h, w = z.shape
        z_nhwc = new(nb * h * w, zc)
        lib.nchw_to_nhwc(z, nb, zc, h * w, z_nhwc)
        z2 = new(nb * h * w, zc)
        lib.linear_f32(z_nhwc, zc, nb * h * w, zc, self.w["post_quant_conv.weight"], self.w["post_quant_conv.bias"],
                       zc, z2, zc)
        out = new(nb, zc, h, w)
        lib.nhwc_to_nchw(z2, nb, zc, h * w, out)
        return out

    def quant(self, m: torch.Tensor, new) -> torch.Tensor:
        """quant_conv (1x1, 8->8) on the encoder's output m, fp32 NHWC [nb, h, w, 8] -> moments NCHW."""
        nb, h, w, zc2 = m.shape
        q = new(nb * h * w, zc2)
        lib.linear_f32(m, zc2, nb * h * w, zc2, self.w["quant_conv.weight"], self.w["quant_conv.bias"], zc2, q, zc2)
        out = torch.empty(nb, zc2, h, w, dtype=torch.float32, device=self.dev)
        lib.nhwc_to_nchw(q, nb, zc2, h * w, out)
        return out

    @staticmethod
    def attn_rows(hw: int) -> int:
        """Query rows per chunk of the mid attention's materialised S: 8192 up to 65536 tokens (2048^2 images),
        beyond that a multiple of 128 that keeps the fp32 S at or below 2 GiB (3584 rows at 3072^2)."""
        return min(8192, max(128, (2 ** 31 // (4 * hw)) // 128 * 128))


NO_PARTIALS = (None, 0)


class VaeWalk:
    """One batch of nb images (or tiles) through the encoder or the decoder of `eng`, as generators that stop at
    each GroupNorm: 22 times in the encoder, 30 in the decoder.

    At a GroupNorm the walk yields (c, h, w, partials, slots): st["cur"], fp32 NHWC [nb * h * w, c], is about
    to be normalised, and `partials` are the GroupNorm partial sums (`slots` per image) that the convolution
    which wrote it emitted, or None where another kernel wrote it. The driver sends back the fp32 [nb * 64]
    (mean, rstd) buffer that dbir_gn_apply reads. A convolution's partial sums are read at the next yield and
    nowhere else, so one workspace buffer holds them all.

    The state `st` holds the fp32 activations that live from one GroupNorm to the next: "cur" and, inside a
    ResnetBlock, the pending residual "res". new(*shape) supplies fresh fp32 tensors, and the workspace the 16-bit
    operands and scratch. No fp32 activation is held in a local across a yield, and none is read after it has left
    st and new() was called again: between yields a driver may move the state elsewhere (it passes its own st and
    new), and new() may hand out the memory of a tensor that is no longer in st. Split-K is off in every GEMM, so an
    image's bits do not depend on the batch it runs in.

    The walk runs on whole images. A subclass may run it on other layouts of the rows by overriding the steps where
    they differ: `_halo`, `_down`, `_up` and `_attend`, and `gn_partials`."""

    gn_partials = True          # convolutions emit GroupNorm partial sums where the GEMM can

    def __init__(self, eng: VaeEngine, ws: Workspace, nb: int, st: Dict[str, torch.Tensor] = None, new=None):
        self.w, self.cfg, self.dev, self.op_dtype = eng.w, eng.cfg, eng.dev, eng.op_dtype
        self.ws, self.nb = ws, nb
        self.st = {} if st is None else st
        self._alloc, self._held = new, [None] * 3

    def new(self, *shape) -> torch.Tensor:
        """A fresh fp32 tensor from the driver's `new`, else from three workspace buffers, so that nothing is
        allocated during graph capture. A buffer is handed out again once the tensor it last held has left st. Three
        are enough: the walk allocates only while st holds at most two tensors (a ResnetBlock keeps its input or its
        shortcut, and conv1's output while conv2's is allocated), and it reads a tensor that has left the state only
        in launches issued before its next allocation. (Not a bound method stored on the walk: that cycle would keep
        the walk, and the workspace buffers its tensors view, alive after a call until the garbage collector runs.)"""
        if self._alloc is not None:
            return self._alloc(*shape)
        i = next(i for i, t in enumerate(self._held) if not any(t is v for v in self.st.values()))
        self._held[i] = self.ws.get(f"x{i}", shape, torch.float32)
        return self._held[i]

    def run(self, net, x: torch.Tensor, answer):
        """Runs x through `net` (VaeWalk.encoder / .decoder) and returns its output, answering each GroupNorm stop
        with answer(c, h, w, partials, slots): the (mean, rstd) buffer of st["cur"]."""
        gen, stats = net(self, x), None
        try:
            while True:
                stats = answer(*gen.send(stats))
        except StopIteration as end:
            return end.value

    @staticmethod
    def stops(cfg: dict, decoder: bool) -> int:
        """GroupNorms the encoder / decoder stops at, known without running a walk: two per ResnetBlock (the levels'
        blocks, and the mid block's two), one for the mid attention, one before conv_out. 22 / 30 for the SD VAE."""
        blocks = len(cfg["ch_mult"]) * (cfg["num_res_blocks"] + (1 if decoder else 0)) + 2
        return 2 * blocks + 2

    def _conv(self, a16, key, out, cin, cout, h, w, residual=None, partials=True):
        """3x3 implicit-GEMM convolution into `out`. Returns the (partials, slots) to yield at the GroupNorm of
        `out`: NO_PARTIALS when they are not asked for (`out` feeds a resampling, not a GroupNorm) or the GEMM
        cannot emit them for this image shape."""
        W, nb = self.w, self.nb
        self._halo(a16, h, w, cin)
        slots = lib.gemm_gn_slots(h, w) if partials and self.gn_partials else 0
        part = self.ws.get("part", (nb * slots * cout * 2,), torch.float32) if slots > 0 else None
        lib.gemm(a16, W[key + ".weight"], out, M=nb * h * w, N=cout, K=9 * cin, bias=W[key + ".bias"],
                 residual=residual, conv=(nb, h, w, cin, 3), split_k=1, gn_partials=part)
        return (part, slots) if slots > 0 else NO_PARTIALS

    def _res(self, p, cin, cout, h, w, src, partials=True):
        """ResnetBlock.forward (temb None) — vae.py:97-117 — on st["cur"], whose partial sums are `src`; returns
        those of its output."""
        ws, W, st, nb, M = self.ws, self.w, self.st, self.nb, self.nb * h * w
        stats = yield (cin, h, w) + src
        a16 = ws.get("a16", (M, cin), self.op_dtype)
        raw = ws.get("raw16", (M, cin), self.op_dtype) if cin != cout else None
        lib.gn_apply(st["cur"], None, cin, 0, nb, h, w, stats, W[p + "norm1.weight"], W[p + "norm1.bias"], a16,
                     norm=True, silu=True, out_raw=raw)
        if cin != cout:
            st["res"] = self.new(M, cout)
            lib.gemm(raw, W[p + "nin_shortcut.weight"], st["res"], M=M, N=cout, K=cin, bias=W[p + "nin_shortcut.bias"],
                     split_k=1)
            del st["cur"]
        else:
            st["res"] = st.pop("cur")
        st["cur"] = self.new(M, cout)
        src = self._conv(a16, p + "conv1", st["cur"], cin, cout, h, w)
        stats = yield (cout, h, w) + src
        b16 = ws.get("b16", (M, cout), self.op_dtype)
        lib.gn_apply(st["cur"], None, cout, 0, nb, h, w, stats, W[p + "norm2.weight"], W[p + "norm2.bias"], b16,
                     norm=True, silu=True)
        st["cur"] = self.new(M, cout)
        return self._conv(b16, p + "conv2", st["cur"], cout, cout, h, w, residual=st.pop("res"), partials=partials)

    def _attn(self, p, c, h, w, src):
        """AttnBlock (single head over the pixels of each image) — vae.py:232-282 — in place on st["cur"]."""
        ws, W, nb, M = self.ws, self.w, self.nb, self.nb * h * w
        stats = yield (c, h, w) + src
        x = self.st["cur"]
        a16 = ws.get("a16", (M, c), self.op_dtype)
        lib.gn_apply(x, None, c, 0, nb, h, w, stats, W[p + "norm.weight"], W[p + "norm.bias"], a16, norm=True,
                     silu=False)
        self._attend(p, a16, x, c, h, w)
        return NO_PARTIALS

    def _attend(self, p, a16, x, c, h, w):
        """The attention after its GroupNorm: x += proj_out(attention over a16, the normalised x)."""
        ws, W, M = self.ws, self.w, self.nb * h * w
        qk = ws.get("qk16", (M, 2 * c), self.op_dtype)
        lib.gemm(a16, W[p + "qk.w"], qk, M=M, N=2 * c, K=c, bias=W[p + "qk.b"], split_k=1)
        o16 = ws.get("o16", (M, c), self.op_dtype)
        self._softmax_av(p, qk, a16, o16, c, h * w, 0, h * w)
        lib.gemm(o16, W[p + "proj_out.weight"], x, M=M, N=c, K=c, bias=W[p + "proj_out.bias"], residual=x, split_k=1)

    def _softmax_av(self, p, qk, a16, o16, c, hw, q0, nq):
        """Single-head attention of each image b of hw tokens: queries q0 .. q0 + nq - 1 of qk[b * hw:, :c] over the
        keys qk[b * hw:(b + 1) * hw, c:] and the values v(a16[b * hw:(b + 1) * hw]), into o16[b * nq:(b + 1) * nq]."""
        ws, W = self.ws, self.w
        rows = min(nq, VaeEngine.attn_rows(hw))
        # any token count: the key axis of S, P and V^T is padded to a multiple of 8 (16-byte GEMM rows); the
        # softmax runs over the real keys and the padded columns of P and V^T are zero
        kp = -(-hw // 8) * 8
        vt = ws.get("vt16", (c, kp), self.op_dtype)                    # V^T [C, keys]
        p16 = ws.get("p16", (rows, kp), self.op_dtype)
        vt[:, hw:].zero_()
        p16[:, hw:].zero_()
        for b in range(self.nb):
            lib.gemm(W[p + "v.weight"], a16[b * hw:(b + 1) * hw], vt, M=c, N=hw, K=c, bias=W[p + "v.bias"],
                     bias_per_row=True, ldo=kp, split_k=1)
            q = b * hw + q0
            for r0 in range(0, nq, rows):
                r1 = min(nq, r0 + rows)
                s = ws.get("s32", (r1 - r0, kp), torch.float32)
                lib.gemm(qk[q + r0: q + r1], qk[b * hw:(b + 1) * hw, c:], s, M=r1 - r0, N=hw, K=c,
                         lda=2 * c, ldb=2 * c, ldo=kp, split_k=1)
                lib.softmax_rows(s, kp, r1 - r0, hw, float(c) ** -0.5, p16, kp)
                lib.gemm(p16[:r1 - r0], vt, o16[b * nq + r0: b * nq + r1], M=r1 - r0, N=c, K=kp, split_k=1)

    def _mid(self, p, c, h, w, src):
        src = yield from self._res(p + "mid.block_1.", c, c, h, w, src)
        src = yield from self._attn(p + "mid.attn_1.", c, h, w, src)
        return (yield from self._res(p + "mid.block_2.", c, c, h, w, src))

    def encoder(self, img: torch.Tensor):
        """img fp32 NCHW [nb, 3, h, w] -> the encoder's output before quant_conv, fp32 NHWC [nb, h/8, w/8, 8]."""
        cfg, ws, W, st, nb = self.cfg, self.ws, self.w, self.st, self.nb
        ch, mult, nres = cfg["ch"], tuple(cfg["ch_mult"]), cfg["num_res_blocks"]
        _, ic, h, w = img.shape
        p, c = "encoder.", ch
        st["cur"] = self.new(nb * h * w, c)
        lib.conv3x3_small_cin(img, None, ic, 0, nb, h, w, W[p + "conv_in.weight"], W[p + "conv_in.bias"], c, st["cur"])
        del img
        src = NO_PARTIALS
        for lvl in range(len(mult)):
            cout = ch * mult[lvl]
            down = lvl != len(mult) - 1
            for j in range(nres):
                src = yield from self._res(f"{p}down.{lvl}.block.{j}.", c, cout, h, w, src,
                                           partials=not (down and j == nres - 1))
                c = cout
            if down:
                h, w = self._down(f"{p}down.{lvl}.downsample.conv", c, h, w)
                src = NO_PARTIALS                                 # a plain-mode GEMM emits none
        src = yield from self._mid(p, c, h, w, src)
        stats = yield (c, h, w) + src
        a16 = ws.get("a16", (nb * h * w, c), self.op_dtype)
        lib.gn_apply(st.pop("cur"), None, c, 0, nb, h, w, stats, W[p + "norm_out.weight"], W[p + "norm_out.bias"],
                     a16, norm=True, silu=True)
        self._halo(a16, h, w, c)
        zc2 = 2 * cfg["z_channels"]
        m = self.new(nb, h, w, zc2)
        lib.conv3x3_small_cout(a16, nb, h, w, c, W[p + "conv_out.weight"], W[p + "conv_out.bias"], zc2, m, nchw=False)
        return m

    def decoder(self, z: torch.Tensor):
        """z fp32 NCHW [nb, 4, h, w], after post_quant_conv -> image fp32 NCHW [nb, 3, 8h, 8w], a tensor of its own."""
        cfg, ws, W, st, nb = self.cfg, self.ws, self.w, self.st, self.nb
        ch, mult, nres = cfg["ch"], tuple(cfg["ch_mult"]), cfg["num_res_blocks"]
        _, zc, h, w = z.shape
        p, c = "decoder.", ch * mult[-1]
        st["cur"] = self.new(nb * h * w, c)
        lib.conv3x3_small_cin(z, None, zc, 0, nb, h, w, W[p + "conv_in.weight"], W[p + "conv_in.bias"], c, st["cur"])
        del z
        src = yield from self._mid(p, c, h, w, NO_PARTIALS)
        for lvl in reversed(range(len(mult))):
            cout = ch * mult[lvl]
            for j in range(nres + 1):
                src = yield from self._res(f"{p}up.{lvl}.block.{j}.", c, cout, h, w, src,
                                           partials=not (lvl != 0 and j == nres))
                c = cout
            if lvl != 0:
                up16, h, w = self._up(c, h, w)
                st["cur"] = self.new(nb * h * w, c)
                src = self._conv(up16, f"{p}up.{lvl}.upsample.conv", st["cur"], c, c, h, w)
        stats = yield (c, h, w) + src
        a16 = ws.get("a16", (nb * h * w, c), self.op_dtype)
        lib.gn_apply(st.pop("cur"), None, c, 0, nb, h, w, stats, W[p + "norm_out.weight"], W[p + "norm_out.bias"],
                     a16, norm=True, silu=True)
        self._halo(a16, h, w, c)
        out = torch.empty(nb, cfg["out_ch"], h, w, dtype=torch.float32, device=self.dev)
        lib.conv3x3_small_cout(a16, nb, h, w, c, W[p + "conv_out.weight"], W[p + "conv_out.bias"], cfg["out_ch"], out,
                               nchw=True)
        return out

    # ------------------------------------------------------------------ the steps that depend on the layout
    def _halo(self, a16, h, w, c) -> None:
        """Makes the 16-bit operand a16 [nb * h * w, c] of a 3x3 convolution complete: whole images have nothing
        outside them but the convolution's zero padding."""

    def _down(self, key, c, h, w):
        """Downsample (vae.py:51-55: pad (0, 1, 0, 1), stride-2 valid conv) of st["cur"] into a new st["cur"];
        returns its (h, w)."""
        nb, ho, wo = self.nb, h // 2, w // 2
        col = self.ws.get("a16", (nb * ho * wo, 9 * c), self.op_dtype)
        lib.im2col_s2(self.st["cur"], nb, h, w, c, 0, col)
        self.st["cur"] = self.new(nb * ho * wo, c)
        lib.gemm(col, self.w[key + ".weight"], self.st["cur"], M=nb * ho * wo, N=c, K=9 * c, bias=self.w[key + ".bias"],
                 split_k=1)
        return ho, wo

    def _up(self, c, h, w):
        """The operand of the Upsample's conv: st["cur"] repeated 2x2 (nearest), 16-bit; returns it and its (h, w)."""
        up16 = self.ws.get("a16", (self.nb * 4 * h * w, c), self.op_dtype)
        lib.gn_apply(self.st["cur"], None, c, 0, self.nb, h, w, None, None, None, up16, norm=False, silu=False,
                     upsample=2)
        return up16, 2 * h, 2 * w
