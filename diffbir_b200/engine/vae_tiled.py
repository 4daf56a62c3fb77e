"""Tiled VAE encode / decode: the reference's Tiled-VAE hook (utils/tilevae/tilevae.py, non-fast mode, as
model/cldm.py:92-141 calls it) on the sm_90a kernels, for images whose un-tiled VAE does not fit one GPU.

Semantics (these are the reference's, not the un-tiled VAE's):

* The input is split into overlapping tiles (`plan_vae_tiles`): pad 32 image pixels around each encoder tile,
  11 latent pixels around each decoder tile. Each tile runs through the network as an image of its own: every
  convolution zero-pads at the tile border and the mid attention attends over the tile's own tokens. The tile's
  output is cropped to its output box and written into the result.
* Every GroupNorm is shared by the tiles of an image: each tile's (mean, biased variance) per group, averaged
  with weights pixels_t / sum(pixels) (no between-tile variance term; dbir_gn_moments + dbir_gn_merge).
* quant_conv / post_quant_conv run un-tiled.

Execution: tiles of equal shape form a shape class; a class runs as batched "waves" of whole tiles (all images
of a tile together) through the same kernels as VaeEngine, with split-K off so that a tile's bits do not depend
on its wave. The network is cut at each GroupNorm into segments: every wave runs a segment and emits its moments,
the moments are merged, then the next segment starts. Between segments a wave carries its state (the current
fp32 tensor and the pending residual); beyond `state_budget` bytes the state is staged through pinned host
buffers on a side stream, overlapped with the next wave. Launches are eager (no CUDA graphs).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch

from .. import lib
from .common import Workspace
from .vae import VaeEngine

PAD_ENCODER = 32        # image pixels
PAD_DECODER = 11        # latent pixels


def best_tile_size(lower: int, upper: int) -> int:
    """The smallest multiple of 32 (else 16, 8, 4, 2) at or above `lower` that does not exceed `upper`
    (reference tilevae.py:325-338)."""
    div = 32
    while div >= 2:
        r = lower % div
        if r == 0:
            return lower
        if lower - r + div <= upper:
            return lower - r + div
        div //= 2
    return lower


@dataclass
class TilePlan:
    """Boxes are (x0, x1, y0, y1). `in_boxes` are in input units; `out_boxes` in output units (x8 for the
    decoder, /8 for the encoder); `crops` are (y, x) offsets of each output box inside its tile's output.
    `classes` maps each tile shape (th, tw) to its tile indices, in order of first appearance."""
    in_boxes: List[Tuple[int, int, int, int]]
    out_boxes: List[Tuple[int, int, int, int]]
    crops: List[Tuple[int, int]]
    classes: Dict[Tuple[int, int], List[int]] = field(default_factory=dict)


def plan_vae_tiles(h: int, w: int, tile_size: int, is_decoder: bool) -> TilePlan:
    """Row-major tile split of an h x w input (reference split_tiles, tilevae.py:340-397). tile_size is in
    input units: image pixels for the encoder, latent pixels for the decoder."""
    pad = PAD_DECODER if is_decoder else PAD_ENCODER
    nh = max(1, math.ceil((h - 2 * pad) / tile_size))
    nw = max(1, math.ceil((w - 2 * pad) / tile_size))
    th = best_tile_size(math.ceil((h - 2 * pad) / nh), tile_size)
    tw = best_tile_size(math.ceil((w - 2 * pad) / nw), tile_size)

    def scale(v):
        return v * 8 if is_decoder else v // 8

    plan = TilePlan([], [], [])
    for i in range(nh):
        for j in range(nw):
            core = (pad + j * tw, min(pad + (j + 1) * tw, w), pad + i * th, min(pad + (i + 1) * th, h))
            out = (core[0] if core[0] > pad else 0, core[1] if core[1] < w - pad else w,
                   core[2] if core[2] > pad else 0, core[3] if core[3] < h - pad else h)
            out = tuple(scale(v) for v in out)
            box = (max(0, core[0] - pad), min(w, core[1] + pad), max(0, core[2] - pad), min(h, core[3] + pad))
            # crop of the tile's output (reference crop_valid_region, tilevae.py:218-229)
            cy, cx = out[2] - scale(box[2]), out[0] - scale(box[0])
            bh, bw = box[3] - box[2], box[1] - box[0]
            oh, ow = (bh * 8, bw * 8) if is_decoder else (bh // 8, bw // 8)
            if cy < 0 or cx < 0 or oh + out[3] - scale(box[3]) - cy != out[3] - out[2] \
                    or ow + out[1] - scale(box[1]) - cx != out[1] - out[0]:
                raise ValueError(f"tile {box} of a {h}x{w} input does not cover its output box {out}")
            plan.in_boxes.append(box)
            plan.out_boxes.append(out)
            plan.crops.append((cy, cx))
            plan.classes.setdefault((bh, bw), []).append(len(plan.in_boxes) - 1)
    return plan


def whole_image_plan(h: int, w: int, is_decoder: bool) -> TilePlan:
    """The input as one tile: the un-tiled network (the reference's hook falls back to it for inputs no larger than
    2 * pad + tile, tilevae.py:317-323)."""
    oh, ow = (8 * h, 8 * w) if is_decoder else (h // 8, w // 8)
    return TilePlan([(0, w, 0, h)], [(0, ow, 0, oh)], [(0, 0)], {(h, w): [0]})


class _Wave:
    """Tiles of one shape class that run together; entry j = (tile j // N, image j % N)."""

    def __init__(self, tiles: List[int], n_img: int, shape: Tuple[int, int], dev):
        self.tiles, self.h, self.w = tiles, shape[0], shape[1]
        self.nb = len(tiles) * n_img
        self.entries = torch.tensor([t * n_img + b for t in tiles for b in range(n_img)], dtype=torch.int32,
                                    device=dev)
        self.st: Dict[str, torch.Tensor] = {}           # device state between segments
        self.layout: Dict[str, Tuple[tuple, int]] = {}  # spilled state: name -> (shape, offset in host)
        self.host: Optional[torch.Tensor] = None        # pinned fp32 staging buffer
        self.loaded: Optional[torch.cuda.Event] = None
        self.gen = None


class TiledVae:
    # Bytes of wave state kept on the device between segments; None = half the device memory that is free when
    # a call starts. The other half is left to the waves' working buffers (`wave_pixels`), to the weights and
    # to whatever the caller keeps resident. Not tuned against measurements.
    state_budget: Optional[int] = None
    # Most batch entries x full-resolution tile pixels per wave (at least one tile). 4 Mi pixels keep a wave's
    # working buffers to a few GiB at the full config (128 channels at full resolution).
    wave_pixels: int = 1 << 22

    def __init__(self, base: VaeEngine):
        self.base, self.w, self.cfg, self.dev = base, base.w, base.cfg, base.dev
        self.op_dtype = base.op_dtype
        self.ws = Workspace(self.dev)
        self.last_stats: dict = {}

    # ------------------------------------------------------------------ public entry points
    @torch.no_grad()
    def encode_moments(self, img: torch.Tensor, tile_size: int) -> torch.Tensor:
        """img fp32 NCHW [N, 3, H, W] in [-1, 1], tile_size in image pixels -> moments fp32 [N, 8, H/8, W/8]."""
        assert img.is_cuda and img.dtype == torch.float32 and img.is_contiguous()
        n, _, h, w = img.shape
        if max(h, w) <= 2 * PAD_ENCODER + tile_size:
            if (h // 8) * (w // 8) % 8 == 0:
                return self.base.encode_moments(img)
            plan = whole_image_plan(h, w, False)      # a latent the un-tiled engine's attention cannot take
        else:
            plan = plan_vae_tiles(h, w, tile_size, False)
        zc2 = 2 * self.cfg["z_channels"]
        res = torch.empty(n, h // 8, w // 8, zc2, dtype=torch.float32, device=self.dev)      # NHWC
        self._run(plan, img, res, self._encoder, 1)
        rows = n * (h // 8) * (w // 8)
        q = torch.empty(rows, zc2, dtype=torch.float32, device=self.dev)
        lib.linear_f32(res, zc2, rows, zc2, self.w["quant_conv.weight"], self.w["quant_conv.bias"], zc2, q, zc2)
        out = torch.empty(n, zc2, h // 8, w // 8, dtype=torch.float32, device=self.dev)
        lib.nhwc_to_nchw(q, n, zc2, (h // 8) * (w // 8), out)
        return out

    @torch.no_grad()
    def decode(self, z: torch.Tensor, tile_size: int) -> torch.Tensor:
        """z fp32 NCHW [N, 4, h, w] (already divided by the scale factor), tile_size in latent pixels ->
        image fp32 NCHW [N, 3, 8h, 8w]."""
        assert z.is_cuda and z.dtype == torch.float32 and z.is_contiguous()
        n, zc, h, w = z.shape
        if max(h, w) <= 2 * PAD_DECODER + tile_size:
            if h * w % 8 == 0:
                return self.base.decode(z)
            plan = whole_image_plan(h, w, True)
        else:
            plan = plan_vae_tiles(h, w, tile_size, True)
        z_nhwc = torch.empty(n * h * w, zc, dtype=torch.float32, device=self.dev)
        lib.nchw_to_nhwc(z, n, zc, h * w, z_nhwc)
        z2 = torch.empty_like(z_nhwc)
        lib.linear_f32(z_nhwc, zc, n * h * w, zc, self.w["post_quant_conv.weight"], self.w["post_quant_conv.bias"],
                       zc, z2, zc)
        z2n = torch.empty(n, zc, h, w, dtype=torch.float32, device=self.dev)
        lib.nhwc_to_nchw(z2, n, zc, h * w, z2n)
        del z_nhwc, z2
        res = torch.empty(n, self.cfg["out_ch"], 8 * h, 8 * w, dtype=torch.float32, device=self.dev)
        self._run(plan, z2n, res, self._decoder, 8)
        return res

    def release_buffers(self) -> None:
        self.ws.clear()

    # ------------------------------------------------------------------ waves, merge and state staging
    def _waves(self, plan: TilePlan, n_img: int, up: int) -> List[_Wave]:
        waves = []
        for shape, tiles in plan.classes.items():
            full = n_img * shape[0] * shape[1] * up * up
            per = max(1, self.wave_pixels // full)
            for i in range(0, len(tiles), per):
                waves.append(_Wave(tiles[i:i + per], n_img, shape, self.dev))
        return waves

    def _run(self, plan: TilePlan, src: torch.Tensor, res: torch.Tensor, net, up: int) -> None:
        n_img = src.shape[0]
        waves = self._waves(plan, n_img, up)
        entries = len(plan.in_boxes) * n_img
        self._moments = torch.empty(entries, 32, 2, dtype=torch.float64, device=self.dev)
        stats = torch.empty(entries, 64, dtype=torch.float32, device=self.dev)
        image = (torch.arange(entries, dtype=torch.int32) % n_img).to(self.dev)
        pix_cache: Dict[tuple, torch.Tensor] = {}
        budget = self.state_budget
        if budget is None:
            budget = torch.cuda.mem_get_info(self.dev)[0] // 2
        main = torch.cuda.current_stream(self.dev)
        self._side = torch.cuda.Stream(self.dev)
        for wv in waves:
            wv.gen = net(wv, plan, src, res)
        passes, spills = 0, 0
        try:
            sent: List[Optional[torch.Tensor]] = [None] * len(waves)
            while True:
                pix, done, kept = [], 0, 0
                for i, wv in enumerate(waves):
                    self._load(wv, main)
                    if i + 1 < len(waves):
                        self._prefetch(waves[i + 1])
                    try:
                        pix.append(wv.gen.send(sent[i]) if passes else next(wv.gen))
                    except StopIteration:
                        done += 1
                        continue
                    size = sum(t.numel() * t.element_size() for t in wv.st.values())
                    if kept + size <= budget:
                        kept += size
                    else:
                        self._spill(wv, main)
                        spills += 1
                if done:
                    assert done == len(waves), "waves of one network must reach the same GroupNorms"
                    break
                key = tuple(pix)
                if key not in pix_cache:
                    per_entry = [p for wv, p in zip(waves, pix) for _ in range(wv.nb)]
                    order = torch.cat([wv.entries.cpu() for wv in waves]).long()
                    arr = torch.empty(entries, dtype=torch.int64)
                    arr[order] = torch.tensor(per_entry, dtype=torch.int64)
                    pix_cache[key] = arr.to(self.dev)
                # the reference visits the tiles forwards at even GroupNorms and backwards at odd ones
                lib.gn_merge(self._moments, pix_cache[key], image, entries, n_img, stats, reverse=passes % 2 == 1)
                for i, wv in enumerate(waves):
                    sent[i] = stats.index_select(0, wv.entries.long())
                passes += 1
        finally:
            torch.cuda.current_stream(self.dev).wait_stream(self._side)
            self._side.synchronize()
            for wv in waves:
                wv.gen = None
                wv.st.clear()
                wv.host = None
            self._side = None
            self._moments = None
            if spills:
                torch._C._host_emptyCache()       # the pinned staging buffers live for one call
        self.last_stats = dict(tiles=len(plan.in_boxes), waves=len(waves), groupnorms=passes, spills=spills,
                               budget=budget)

    def _spill(self, wv: _Wave, main) -> None:
        """Copies the wave's state to its pinned host buffer on the side stream and drops the device copy."""
        total = sum(t.numel() for t in wv.st.values())
        if wv.host is None or wv.host.numel() < total:
            self._side.synchronize()                       # the old buffer may still be read by a copy
            wv.host = torch.empty(total, dtype=torch.float32, pin_memory=True)
        ev = torch.cuda.Event()
        ev.record(main)
        self._side.wait_event(ev)
        off = 0
        with torch.cuda.stream(self._side):
            for k, t in wv.st.items():
                assert t.dtype == torch.float32 and t.is_contiguous()
                wv.host[off:off + t.numel()].copy_(t.view(-1), non_blocking=True)
                t.record_stream(self._side)
                wv.layout[k] = (tuple(t.shape), off)
                off += t.numel()
        wv.st.clear()

    def _prefetch(self, wv: _Wave) -> None:
        """Starts the host -> device copy of a spilled wave's state on the side stream."""
        if not wv.layout:
            return
        with torch.cuda.stream(self._side):
            for k, (shape, off) in wv.layout.items():
                t = torch.empty(shape, dtype=torch.float32, device=self.dev)
                t.view(-1).copy_(wv.host[off:off + t.numel()], non_blocking=True)
                wv.st[k] = t
            wv.loaded = torch.cuda.Event()
            wv.loaded.record(self._side)
        wv.layout = {}

    def _load(self, wv: _Wave, main) -> None:
        self._prefetch(wv)
        if wv.loaded is not None:
            main.wait_event(wv.loaded)
            for t in wv.st.values():
                t.record_stream(main)
            wv.loaded = None

    # ------------------------------------------------------------------ blocks (generators: one yield per GroupNorm)
    def _new(self, *shape) -> torch.Tensor:
        return torch.empty(*shape, dtype=torch.float32, device=self.dev)

    def _emit(self, wv: _Wave, x: torch.Tensor, c: int, h: int, w: int, part=None, slots=0) -> None:
        """Moments of the wave's fp32 NHWC tensor x into the call's moment buffer, at its entries' indices."""
        if part is not None:
            lib.gn_moments(c, wv.nb, h * w, self._moments, partials=part, slots=slots, entry=wv.entries)
        else:
            ws = self.ws.get("mom_ws", (lib.gn_moments_workspace_floats(wv.nb, h * w, c),), torch.float32)
            lib.gn_moments(c, wv.nb, h * w, self._moments, x=x, workspace=ws, entry=wv.entries)

    def _conv(self, wv, a16, key, out, cin, cout, h, w, residual=None, emit=True) -> None:
        """3x3 implicit-GEMM convolution of the wave; emits the output's moments from the fused partial sums
        (or, where the GEMM cannot emit them for this tile shape, from the output itself)."""
        W = self.w
        slots = lib.gemm_gn_slots(h, w) if emit else 0
        part = self.ws.get("part", (wv.nb * slots * cout * 2,), torch.float32) if slots > 0 else None
        lib.gemm(a16, W[key + ".weight"], out, M=wv.nb * h * w, N=cout, K=9 * cin, bias=W[key + ".bias"],
                 residual=residual, conv=(wv.nb, h, w, cin, 3), split_k=1, gn_partials=part)
        if emit:
            self._emit(wv, out, cout, h, w, part, slots)

    def _res(self, wv, p, cin, cout, h, w, emit=True):
        """ResnetBlock (vae.py:97-117) on st["cur"]; reads its statistics at two yields. No device tensor is
        held in a local across a yield: the state may be staged to the host in between."""
        ws, W, st, M, nb = self.ws, self.w, wv.st, wv.nb * h * w, wv.nb
        stats = yield h * w
        a16 = ws.get("a16", (M, cin), self.op_dtype)
        raw = ws.get("raw16", (M, cin), self.op_dtype) if cin != cout else None
        lib.gn_apply(st["cur"], None, cin, 0, nb, h, w, stats, W[p + "norm1.weight"], W[p + "norm1.bias"], a16,
                     norm=True, silu=True, out_raw=raw)
        if cin != cout:
            st["res"] = self._new(M, cout)
            lib.gemm(raw, W[p + "nin_shortcut.weight"], st["res"], M=M, N=cout, K=cin, bias=W[p + "nin_shortcut.bias"],
                     split_k=1)
            del st["cur"]
        else:
            st["res"] = st.pop("cur")
        st["cur"] = self._new(M, cout)
        self._conv(wv, a16, p + "conv1", st["cur"], cin, cout, h, w)
        stats = yield h * w
        b16 = ws.get("b16", (M, cout), self.op_dtype)
        lib.gn_apply(st["cur"], None, cout, 0, nb, h, w, stats, W[p + "norm2.weight"], W[p + "norm2.bias"], b16,
                     norm=True, silu=True)
        st["cur"] = self._new(M, cout)
        self._conv(wv, b16, p + "conv2", st["cur"], cout, cout, h, w, residual=st.pop("res"), emit=emit)

    def _attn(self, wv, p, c, h, w):
        """AttnBlock (vae.py:232-282) in place on st["cur"], each entry attending over its own tile's tokens."""
        ws, W, st, nb, hw = self.ws, self.w, wv.st, wv.nb, h * w
        M = nb * hw
        stats = yield hw
        x = st["cur"]
        a16 = ws.get("a16", (M, c), self.op_dtype)
        lib.gn_apply(x, None, c, 0, nb, h, w, stats, W[p + "norm.weight"], W[p + "norm.bias"], a16, norm=True,
                     silu=False)
        qk = ws.get("qk16", (M, 2 * c), self.op_dtype)
        lib.gemm(a16, W[p + "qk.w"], qk, M=M, N=2 * c, K=c, bias=W[p + "qk.b"], split_k=1)
        o16 = ws.get("o16", (M, c), self.op_dtype)
        rows = min(hw, VaeEngine.attn_rows(hw))
        # tiles have any token count: the key axis of S, P and V^T is padded to a multiple of 8 (16-byte GEMM rows);
        # the softmax runs over the real keys and the padded columns of P and V^T are zero
        kp = -(-hw // 8) * 8
        vt = ws.get("vt16", (c, kp), self.op_dtype)
        p16 = ws.get("p16", (rows, kp), self.op_dtype)
        vt[:, hw:].zero_()
        p16[:, hw:].zero_()
        for b in range(nb):
            lib.gemm(W[p + "v.weight"], a16[b * hw:(b + 1) * hw], vt, M=c, N=hw, K=c, bias=W[p + "v.bias"],
                     bias_per_row=True, ldo=kp, split_k=1)
            for r0 in range(0, hw, rows):
                r1 = min(hw, r0 + rows)
                s = ws.get("s32", (r1 - r0, kp), torch.float32)
                lib.gemm(qk[b * hw + r0: b * hw + r1], qk[b * hw:(b + 1) * hw, c:], s, M=r1 - r0, N=hw, K=c,
                         lda=2 * c, ldb=2 * c, ldo=kp, split_k=1)
                lib.softmax_rows(s, kp, r1 - r0, hw, float(c) ** -0.5, p16, kp)
                lib.gemm(p16[:r1 - r0], vt, o16[b * hw + r0: b * hw + r1], M=r1 - r0, N=c, K=kp, split_k=1)
        lib.gemm(o16, W[p + "proj_out.weight"], x, M=M, N=c, K=c, bias=W[p + "proj_out.bias"], residual=x, split_k=1)
        self._emit(wv, x, c, h, w)
        del x

    def _mid(self, wv, p, c, h, w):
        yield from self._res(wv, p + "mid.block_1.", c, c, h, w)
        yield from self._attn(wv, p + "mid.attn_1.", c, h, w)
        yield from self._res(wv, p + "mid.block_2.", c, c, h, w)

    def _gather(self, wv: _Wave, plan: TilePlan, src: torch.Tensor) -> torch.Tensor:
        """The wave's input tiles as one NCHW batch, tile-major (entry = tile * N + image)."""
        parts = []
        for t in wv.tiles:
            x0, x1, y0, y1 = plan.in_boxes[t]
            parts.append(src[:, :, y0:y1, x0:x1])
        return torch.cat(parts, 0).contiguous()

    def _encoder(self, wv: _Wave, plan: TilePlan, img: torch.Tensor, res: torch.Tensor):
        cfg, ws, W, st = self.cfg, self.ws, self.w, wv.st
        ch, mult, nres = cfg["ch"], tuple(cfg["ch_mult"]), cfg["num_res_blocks"]
        nb, h, w, p, c = wv.nb, wv.h, wv.w, "encoder.", cfg["ch"]
        x_in = self._gather(wv, plan, img)
        st["cur"] = self._new(nb * h * w, c)
        lib.conv3x3_small_cin(x_in, None, x_in.shape[1], 0, nb, h, w, W[p + "conv_in.weight"], W[p + "conv_in.bias"],
                              c, st["cur"])
        del x_in
        self._emit(wv, st["cur"], c, h, w)
        for lvl in range(len(mult)):
            cout = ch * mult[lvl]
            down = lvl != len(mult) - 1
            for j in range(nres):
                yield from self._res(wv, f"{p}down.{lvl}.block.{j}.", c, cout, h, w, emit=not (down and j == nres - 1))
                c = cout
            if down:
                ho, wo = h // 2, w // 2
                col = ws.get("a16", (nb * ho * wo, 9 * c), self.op_dtype)
                lib.im2col_s2(st["cur"], nb, h, w, c, 0, col)
                st["cur"] = self._new(nb * ho * wo, c)
                lib.gemm(col, W[f"{p}down.{lvl}.downsample.conv.weight"], st["cur"], M=nb * ho * wo, N=c, K=9 * c,
                         bias=W[f"{p}down.{lvl}.downsample.conv.bias"], split_k=1)
                h, w = ho, wo
                self._emit(wv, st["cur"], c, h, w)
        yield from self._mid(wv, p, c, h, w)
        stats = yield h * w
        a16 = ws.get("a16", (nb * h * w, c), self.op_dtype)
        lib.gn_apply(st.pop("cur"), None, c, 0, nb, h, w, stats, W[p + "norm_out.weight"], W[p + "norm_out.bias"],
                     a16, norm=True, silu=True)
        zc2 = 2 * cfg["z_channels"]
        m = self._new(nb, h, w, zc2)
        lib.conv3x3_small_cout(a16, nb, h, w, c, W[p + "conv_out.weight"], W[p + "conv_out.bias"], zc2, m, nchw=False)
        n_img = res.shape[0]
        for i, t in enumerate(wv.tiles):
            x0, x1, y0, y1 = plan.out_boxes[t]
            cy, cx = plan.crops[t]
            res[:, y0:y1, x0:x1] = m[i * n_img:(i + 1) * n_img, cy:cy + y1 - y0, cx:cx + x1 - x0]

    def _decoder(self, wv: _Wave, plan: TilePlan, z: torch.Tensor, res: torch.Tensor):
        cfg, ws, W, st = self.cfg, self.ws, self.w, wv.st
        ch, mult, nres = cfg["ch"], tuple(cfg["ch_mult"]), cfg["num_res_blocks"]
        nb, h, w, p = wv.nb, wv.h, wv.w, "decoder."
        c = ch * mult[-1]
        z_in = self._gather(wv, plan, z)
        st["cur"] = self._new(nb * h * w, c)
        lib.conv3x3_small_cin(z_in, None, z_in.shape[1], 0, nb, h, w, W[p + "conv_in.weight"], W[p + "conv_in.bias"],
                              c, st["cur"])
        del z_in
        self._emit(wv, st["cur"], c, h, w)
        yield from self._mid(wv, p, c, h, w)
        for lvl in reversed(range(len(mult))):
            cout = ch * mult[lvl]
            for j in range(nres + 1):
                yield from self._res(wv, f"{p}up.{lvl}.block.{j}.", c, cout, h, w, emit=not (lvl != 0 and j == nres))
                c = cout
            if lvl != 0:
                up16 = ws.get("a16", (nb * 4 * h * w, c), self.op_dtype)
                lib.gn_apply(st["cur"], None, c, 0, nb, h, w, None, None, None, up16, norm=False, silu=False, upsample=2)
                h, w = 2 * h, 2 * w
                st["cur"] = self._new(nb * h * w, c)
                self._conv(wv, up16, f"{p}up.{lvl}.upsample.conv", st["cur"], c, c, h, w)
        stats = yield h * w
        a16 = ws.get("a16", (nb * h * w, c), self.op_dtype)
        lib.gn_apply(st.pop("cur"), None, c, 0, nb, h, w, stats, W[p + "norm_out.weight"], W[p + "norm_out.bias"],
                     a16, norm=True, silu=True)
        out = self._new(nb, cfg["out_ch"], h, w)
        lib.conv3x3_small_cout(a16, nb, h, w, c, W[p + "conv_out.weight"], W[p + "conv_out.bias"], cfg["out_ch"], out,
                               nchw=True)
        n_img = res.shape[0]
        for i, t in enumerate(wv.tiles):
            x0, x1, y0, y1 = plan.out_boxes[t]
            cy, cx = plan.crops[t]
            res[:, :, y0:y1, x0:x1] = out[i * n_img:(i + 1) * n_img, :, cy:cy + y1 - y0, cx:cx + x1 - x0]
