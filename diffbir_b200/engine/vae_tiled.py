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
of a tile together). The network itself is stated in vae.py: each wave runs `VaeWalk`, the generator VaeEngine
runs too (same kernels, split-K off so that a tile's bits do not depend on its wave), which stops at each
GroupNorm. This file supplies what is the tiled engine's own: the tile plan, the waves, and the driver (`_run`)
that at each stop takes every wave's moments, merges them and sends the statistics back. Between stops a wave
carries its state (the current fp32 tensor and the pending residual, fresh `torch.empty` tensors in the wave's
`st`); beyond `state_budget` bytes the state is staged through pinned host buffers on a side stream, overlapped
with the next wave. Launches are eager (no CUDA graphs).

Cooperating ranks (`TiledVae(base, rank, world)`, all called with the same input) split the tiles
(`tiles_of_ranks`): each runs its own as above; at every GroupNorm the ranks all-gather their entries' fp64 moments
and pixel counts into the global moment buffer and run the same merge, and after the last one they all-gather the
output boxes. A tile's bits do not depend on its wave, so every rank returns the single-rank result bit for bit.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist

from .. import lib
from .common import Workspace
from .vae import VaeEngine, VaeWalk

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


# ---- tiles sharded over cooperating ranks (host logic, shared with the CPU / gloo tests) ----
def tiles_of_ranks(plan: TilePlan, world: int) -> List[List[int]]:
    """Each rank's tiles, ascending. Greedy by full-resolution pixels (a tile's input box scaled by a constant):
    the largest tile first, ties by tile index, each to the rank with the fewest pixels so far, ties to the lowest
    rank. A pure function of the plan, so every rank computes the same split, and the most loaded rank exceeds the
    least loaded by at most one tile. World 1 owns every tile in plan order; ranks beyond the tile count own none."""
    area = [(x1 - x0) * (y1 - y0) for x0, x1, y0, y1 in plan.in_boxes]
    load, owned = [0] * world, [[] for _ in range(world)]
    for t in sorted(range(len(area)), key=lambda t: (-area[t], t)):
        r = min(range(world), key=lambda r: (load[r], r))
        load[r] += area[t]
        owned[r].append(t)
    return [sorted(o) for o in owned]


def entries_of_ranks(owned: List[List[int]], n_img: int) -> List[List[int]]:
    """The batch entries (entry = tile * n_img + image) of each rank's tiles, in its tile order."""
    return [[t * n_img + b for t in tiles for b in range(n_img)] for tiles in owned]


def moment_rows(entries: List[List[int]], slots: int) -> List[int]:
    """Row of every global entry in the gathered moment payloads viewed as [world * slots, ...]."""
    rows = [0] * sum(map(len, entries))
    for r, ents in enumerate(entries):
        for s, e in enumerate(ents):
            rows[e] = r * slots + s
    return rows


MOMENT_COLS = 65        # one payload row: 32 groups x (mean, biased variance), then the entry's pixel count; fp64


def pack_moments(moments: torch.Tensor, mine: torch.Tensor, pixels: torch.Tensor, slots: int) -> torch.Tensor:
    """A rank's payload at one GroupNorm: row s holds its entry mine[s] (global index) -- the fp64 moments of
    `moments` [entries, 32, 2] and the pixel count pixels[s] -- and rows past its entries are zero."""
    k = mine.numel()
    send = moments.new_zeros(slots, MOMENT_COLS)
    send[:k, :64] = moments.index_select(0, mine).view(k, 64)
    send[:k, 64] = pixels
    return send


def unpack_moments(recv: torch.Tensor, rows: torch.Tensor, moments: torch.Tensor) -> torch.Tensor:
    """Every rank's payload, recv [world, slots, MOMENT_COLS], into the global moments [entries, 32, 2]: every entry
    is rewritten from its owner's row (`moment_rows`). Returns the entries' pixel counts, int64."""
    flat = recv.view(-1, MOMENT_COLS).index_select(0, rows)
    moments.copy_(flat[:, :64].view(moments.shape))
    return flat[:, 64].long()


def _box(res: torch.Tensor, box: Tuple[int, int, int, int], nchw: bool) -> torch.Tensor:
    x0, x1, y0, y1 = box
    return res[:, :, y0:y1, x0:x1] if nchw else res[:, y0:y1, x0:x1]


def box_share(res: torch.Tensor, boxes: List[Tuple[int, int, int, int]], nchw: bool) -> int:
    """Elements of `res` (all images, all channels) inside the output boxes."""
    return sum(_box(res, b, nchw).numel() for b in boxes)


def pack_boxes(res: torch.Tensor, boxes: List[Tuple[int, int, int, int]], size: int, nchw: bool) -> torch.Tensor:
    """The output boxes of a rank's tiles, copied from `res` (NCHW or NHWC) one after the other into a flat buffer of
    `size` elements (the largest rank's share); the padding is not written and never read."""
    send = res.new_empty(size)
    off = 0
    for b in boxes:
        v = _box(res, b, nchw)
        send[off:off + v.numel()].view(v.shape).copy_(v)
        off += v.numel()
    return send


def unpack_boxes(recv: torch.Tensor, res: torch.Tensor, boxes: List[List[Tuple[int, int, int, int]]], nchw: bool,
                 skip: int = -1) -> None:
    """Copies every rank's boxes from the gathered buffers recv [world, size] into `res`, except rank `skip`'s."""
    for r, rb in enumerate(boxes):
        if r == skip:
            continue
        off = 0
        for b in rb:
            v = _box(res, b, nchw)
            v.copy_(recv[r, off:off + v.numel()].view(v.shape))
            off += v.numel()


class ProcessGroupGather:
    """The collective of the sharded tiled VAE: all-gather of equal-size tensors over the torch.distributed default
    group (NCCL between GPUs). t [...] on every rank -> [world, ...], rank r's tensor at r. Gathered flat, the form
    every backend takes."""

    def all_gather(self, t: torch.Tensor) -> torch.Tensor:
        world = dist.get_world_size()
        out = torch.empty(world * t.numel(), dtype=t.dtype, device=t.device)
        dist.all_gather_into_tensor(out, t.contiguous().view(-1))
        return out.view((world,) + tuple(t.shape))


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

    def __init__(self, base: VaeEngine, rank: int = 0, world: int = 1, comm=None):
        """world > 1: this is rank `rank` of cooperating ranks that all call with the same input. Each runs its own
        tiles (`tiles_of_ranks`); `comm.all_gather` (default: `ProcessGroupGather`) exchanges the tiles' GroupNorm
        moments at every stop and their outputs at the end, so every rank returns the full result, with the bits
        of one rank. Inputs that run un-tiled stay replicated."""
        self.base, self.cfg, self.dev = base, base.cfg, base.dev
        self.rank, self.world = rank, world
        self.comm = comm if comm is not None or world == 1 else ProcessGroupGather()
        self.ws = Workspace(self.dev)
        self.last_stats: dict = {}

    # ------------------------------------------------------------------ public entry points
    @torch.no_grad()
    def encode_moments(self, img: torch.Tensor, tile_size: int) -> torch.Tensor:
        """img fp32 NCHW [N, 3, H, W] in [-1, 1], tile_size in image pixels -> moments fp32 [N, 8, H/8, W/8]."""
        assert img.is_cuda and img.dtype == torch.float32 and img.is_contiguous()
        n, _, h, w = img.shape
        tiled = max(h, w) > 2 * PAD_ENCODER + tile_size
        if not tiled:
            if (h // 8) * (w // 8) % 8 == 0:
                return self.base.encode_moments(img)
            plan = whole_image_plan(h, w, False)      # a latent the un-tiled engine's attention cannot take
        else:
            plan = plan_vae_tiles(h, w, tile_size, False)
        zc2 = 2 * self.cfg["z_channels"]
        res = torch.empty(n, h // 8, w // 8, zc2, dtype=torch.float32, device=self.dev)      # NHWC
        self._run(plan, img, res, False, tiled and self.world > 1)
        return self.base.quant(res, self._new)

    @torch.no_grad()
    def decode(self, z: torch.Tensor, tile_size: int) -> torch.Tensor:
        """z fp32 NCHW [N, 4, h, w] (already divided by the scale factor), tile_size in latent pixels ->
        image fp32 NCHW [N, 3, 8h, 8w]."""
        assert z.is_cuda and z.dtype == torch.float32 and z.is_contiguous()
        n, zc, h, w = z.shape
        tiled = max(h, w) > 2 * PAD_DECODER + tile_size
        if not tiled:
            if h * w % 8 == 0:
                return self.base.decode(z)
            plan = whole_image_plan(h, w, True)
        else:
            plan = plan_vae_tiles(h, w, tile_size, True)
        z2n = self.base.post_quant(z, self._new)
        res = torch.empty(n, self.cfg["out_ch"], 8 * h, 8 * w, dtype=torch.float32, device=self.dev)
        self._run(plan, z2n, res, True, tiled and self.world > 1)
        return res

    def release_buffers(self) -> None:
        self.ws.clear()

    # ------------------------------------------------------------------ waves, merge and state staging
    def _waves(self, plan: TilePlan, n_img: int, up: int, mine: List[int]) -> List[_Wave]:
        waves, mine = [], set(mine)
        for shape, tiles in plan.classes.items():
            tiles = [t for t in tiles if t in mine]
            full = n_img * shape[0] * shape[1] * up * up
            per = max(1, self.wave_pixels // full)
            for i in range(0, len(tiles), per):
                waves.append(_Wave(tiles[i:i + per], n_img, shape, self.dev))
        return waves

    def _run(self, plan: TilePlan, src: torch.Tensor, res: torch.Tensor, decoder: bool, shard: bool) -> None:
        """Runs the plan's tiles into `res`. shard: this rank runs its own tiles only; at every stop the ranks
        all-gather their entries' moments and pixel counts into the global moment buffer before the same merge,
        and after the last one their output boxes. Every rank issues the same collectives, tiles or not."""
        n_img = src.shape[0]
        owned = tiles_of_ranks(plan, self.world if shard else 1)
        rank = self.rank if shard else 0
        waves = self._waves(plan, n_img, 8 if decoder else 1, owned[rank])
        entries = len(plan.in_boxes) * n_img
        stops = VaeWalk.stops(self.cfg, decoder)
        if shard:
            ents = entries_of_ranks(owned, n_img)
            share = max(map(len, ents))                  # payload rows per rank
            mine = torch.tensor(ents[rank], dtype=torch.int64).to(self.dev)
            rows = torch.tensor(moment_rows(ents, share), dtype=torch.int64).to(self.dev)
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
            wv.gen = self._tiles(wv, plan, src, res, decoder)
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
                        c, h, w, part, slots = wv.gen.send(sent[i]) if passes else next(wv.gen)
                    except StopIteration:
                        done += 1
                        continue
                    self._emit(wv, c, h, w, part, slots)
                    pix.append(h * w)
                    size = sum(t.numel() * t.element_size() for t in wv.st.values())
                    if kept + size <= budget:
                        kept += size
                    else:
                        self._spill(wv, main)
                        spills += 1
                if passes == stops:
                    assert done == len(waves), "the walk has more GroupNorms than VaeWalk.stops"
                    break
                assert not done, "the walk has fewer GroupNorms than VaeWalk.stops"
                key = tuple(pix)
                if key not in pix_cache:
                    arr = torch.empty(entries, dtype=torch.int64)
                    for wv, p in zip(waves, pix):
                        arr[wv.entries.cpu().long()] = p
                    # sharded: the pixel counts of this rank's entries, in its payload's row order
                    pix_cache[key] = (arr[ents[rank]].double() if shard else arr).to(self.dev)
                pixels = pix_cache[key]
                if shard:
                    # a rank sees only its own shape classes: the counts travel with the moments, so every rank
                    # merges the same global buffer with the same weights
                    pixels = unpack_moments(self.comm.all_gather(pack_moments(self._moments, mine, pixels, share)),
                                            rows, self._moments)
                # the reference visits the tiles forwards at even GroupNorms and backwards at odd ones
                lib.gn_merge(self._moments, pixels, image, entries, n_img, stats, reverse=passes % 2 == 1)
                for i, wv in enumerate(waves):
                    sent[i] = stats.index_select(0, wv.entries.long())
                passes += 1
            if shard:
                # the output boxes partition `res`: copies, so every element keeps its owner's bits
                boxes = [[plan.out_boxes[t] for t in tiles] for tiles in owned]
                size = max(box_share(res, b, decoder) for b in boxes)
                recv = self.comm.all_gather(pack_boxes(res, boxes[rank], size, decoder))
                unpack_boxes(recv, res, boxes, decoder, skip=rank)
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
        self.last_stats = dict(tiles=len(plan.in_boxes), owned=len(owned[rank]), waves=len(waves), groupnorms=passes,
                               exchanges=passes + 1 if shard else 0, spills=spills, budget=budget)

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

    # ------------------------------------------------------------------ one wave through the network
    def _new(self, *shape) -> torch.Tensor:
        return torch.empty(*shape, dtype=torch.float32, device=self.dev)

    def _emit(self, wv: _Wave, c: int, h: int, w: int, part, slots: int) -> None:
        """Moments of the wave's st["cur"] into the call's moment buffer, at its entries' indices: from the partial
        sums of the conv that wrote it, or, where there are none, from the tensor itself."""
        if part is not None:
            lib.gn_moments(c, wv.nb, h * w, self._moments, partials=part, slots=slots, entry=wv.entries)
        else:
            ws = self.ws.get("mom_ws", (lib.gn_moments_workspace_floats(wv.nb, h * w, c),), torch.float32)
            lib.gn_moments(c, wv.nb, h * w, self._moments, x=wv.st["cur"], workspace=ws, entry=wv.entries)

    def _tiles(self, wv: _Wave, plan: TilePlan, src: torch.Tensor, res: torch.Tensor, decoder: bool):
        """The wave's tiles through VaeWalk: gathered as one NCHW batch, tile-major (entry = tile * N + image), and
        each tile's output cropped to its box of `res` (NCHW for the decoder, NHWC for the encoder)."""
        walk = VaeWalk(self.base, self.ws, wv.nb, wv.st, self._new)
        boxes = [plan.in_boxes[t] for t in wv.tiles]
        out = yield from (walk.decoder if decoder else walk.encoder)(
            torch.cat([src[:, :, y0:y1, x0:x1] for x0, x1, y0, y1 in boxes], 0).contiguous())
        n_img = res.shape[0]
        for i, t in enumerate(wv.tiles):
            x0, x1, y0, y1 = plan.out_boxes[t]
            cy, cx = plan.crops[t]
            tile = out[i * n_img:(i + 1) * n_img]
            if decoder:
                res[:, :, y0:y1, x0:x1] = tile[:, :, cy:cy + y1 - y0, cx:cx + x1 - x0]
            else:
                res[:, y0:y1, x0:x1] = tile[:, cy:cy + y1 - y0, cx:cx + x1 - x0]
