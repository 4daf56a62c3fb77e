"""Spaced (DDPM-respaced) and DDIM samplers — counterparts of the reference's
diffbir.sampler.{SpacedSampler, DDIMSampler} (sampler/sampler.py, spaced_sampler.py,
ddim_sampler.py) with the same constructors and `sample(...)` signature.

When `model` is a diffbir_b200 ControlLDM the loop runs on the kernel engine:
  * cond and uncond branches (and, when tiled, all latent tiles) are ONE batched forward,
    captured once in a CUDA graph and replayed every step; tiled runs with more tile-forwards than
    `max_tile_forwards` replay that graph once per chunk of tiles of one branch (bounded memory);
  * text K/V and every time embedding are computed before the loop;
  * CFG mix + x0 + posterior/DDIM update is one fused kernel per step (dbir_sampler_step);
  * tiles are gathered / Gaussian-blended on the device in the reference's accumulation order;
    with torch.distributed initialised the tiles are sharded round-robin over the ranks and
    re-assembled by a single all-gather per step (every rank then blends and updates the same
    full latent with the same RNG stream).
Noise is drawn with torch.randn_like once per step exactly like the reference
(spaced_sampler.py:181, ddim_sampler.py:143): the RNG consumption is the reference's. With a NoiseSource set
(`Sampler.noise_source`), every draw comes per sample from that sample's own generators instead, in the same order. Outputs are
bit-reproducible across runs and processes in tiled mode and with DBIR_DETERMINISTIC=1 (batch-invariant
kernel plans); otherwise the timing-based split-K choice of dbir_gemm may differ between processes
(rounding-level differences).
Any other callable `model(x, t, cond)` takes a plain PyTorch loop with identical arithmetic.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from .. import lib
from ..utils.common import gaussian_weights, sliding_windows


class NoiseSource:
    """The random draws of one batch, per sample: sample k draws from its own CUDA and CPU torch.Generator seeded
    seeds[k], in the order a run of that sample alone draws from the global generators right after
    set_seed(seeds[k]). Each sample's noise is then the same whichever batch it runs in.

    Without a source (None) the pipeline and the samplers draw from the global generators, as the reference does."""

    def __init__(self, seeds, device) -> None:
        self.seeds = [int(s) for s in seeds]
        self.device = torch.device(device)
        self.gpu = [torch.Generator(self.device).manual_seed(s) for s in self.seeds]
        # on a CPU device one generator serves both kinds of draw, as torch's global CPU generator does
        self.cpu = self.gpu if self.device.type == "cpu" else [torch.Generator().manual_seed(s) for s in self.seeds]

    def randn(self, shape) -> torch.Tensor:
        """torch.randn(shape) in fp32 on the source's device, row k from sample k's device generator."""
        if shape[0] != len(self.gpu):
            raise ValueError(f"a batch of {shape[0]} samples drawn from a source of {len(self.gpu)} seeds")
        return torch.cat([torch.randn((1, *shape[1:]), generator=g, device=self.device, dtype=torch.float32)
                          for g in self.gpu])

    def randn_like(self, x: torch.Tensor) -> torch.Tensor:
        return self.randn(tuple(x.shape)).to(x.dtype)

    def randint_seeds(self) -> List[int]:
        """torch.randint(0, 2**63 - 1, []) from each sample's CPU generator (the Brownian tree's seed)."""
        return [int(torch.randint(0, 2 ** 63 - 1, [], generator=g).item()) for g in self.cpu]


def randn_like(x: torch.Tensor, source: Optional[NoiseSource]) -> torch.Tensor:
    return torch.randn_like(x) if source is None else source.randn_like(x)


def randn(shape, device, source: Optional[NoiseSource]) -> torch.Tensor:
    return torch.randn(shape, device=device, dtype=torch.float32) if source is None else source.randn(shape)


def space_timesteps(num_timesteps: int, steps: int) -> np.ndarray:
    """space_timesteps(num_timesteps, str(steps)) — spaced_sampler.py:14-64 (single section)."""
    stride = 1.0 if steps <= 1 else (num_timesteps - 1) / (steps - 1)
    out, cur = [], 0.0
    for _ in range(steps):
        out.append(round(cur))
        cur += stride
    return np.array(sorted(set(out)), dtype=np.int32)


# ---- tile sharding (multi-GPU tiled sampling; host-side logic shared with the CPU/gloo test) ----
def tiles_of_rank(num_tiles: int, rank: int, world: int) -> List[int]:
    """Round-robin ownership: tile t belongs to rank t % world, local slot t // world."""
    return list(range(rank, num_tiles, world))


def tile_slots(num_tiles: int, world: int) -> int:
    return (num_tiles + world - 1) // world


def assemble_units(recv: torch.Tensor, num_units: int) -> torch.Tensor:
    """all_gather output [world, slots, ...] of round-robin owned units -> [num_units, ...] in unit order
    (unit u = slot*world + rank; the tail entries are padding)."""
    world, slots = recv.shape[:2]
    return recv.transpose(0, 1).reshape(slots * world, *recv.shape[2:])[:num_units].contiguous()


def plan_tile_chunks(mine: List[int], num_tiles: int, batch: int,
                     max_tile_forwards: int) -> Tuple[int, List[Tuple[int, int, int]]]:
    """Graph replays of one rank's tile-forward units (`mine`: ascending unit ids, unit u = branch * num_tiles
    + tile, each unit is `batch` batch entries). Returns (units per replay, [(first local slot, units, branch)])
    with the chunks in local slot order, so writing each chunk's eps at its slots keeps the blend in unit order.

    When every unit fits under `max_tile_forwards` batch entries there is ONE chunk holding all of them
    (branch -1: it may mix the CFG branches). Otherwise every chunk holds units of one CFG branch, so a replay
    reads one text context, and each branch's units are spread evenly over the fewest chunks that respect the
    cap. All chunks replay one graph of the largest chunk's size; a shorter chunk's spare entries keep earlier
    tiles and their outputs are ignored (batch-invariant plans: they do not touch the other entries' bits)."""
    if max_tile_forwards < batch:
        raise ValueError(f"max_tile_forwards ({max_tile_forwards}) is below the batch size ({batch}): "
                         "one tile-forward of every image must fit into a replay")
    n = len(mine)
    if n * batch <= max_tile_forwards:
        return n, ([(0, n, -1)] if n else [])
    per = max_tile_forwards // batch
    chunks, o = [], 0
    while o < n:
        br = mine[o] // num_tiles
        nb_ = sum(1 for u in mine[o:] if u // num_tiles == br)     # this branch's units (contiguous: mine ascends)
        size = -(-nb_ // -(-nb_ // per))                            # ceil(n / ceil(n / per)) <= per
        for s in range(o, o + nb_, size):
            chunks.append((s, min(size, o + nb_ - s), br))
        o += nb_
    return max(c for _, c, _ in chunks), chunks


def tiled_run_chunked(num_tiles: int, nbr: int, batch: int, max_tile_forwards: int, shard_tiles: bool = True) -> bool:
    """Whether EngineEval replays this rank's tile-forwards in more than one chunk (same ownership and plan)."""
    import torch.distributed as dist
    sharded = shard_tiles and dist.is_available() and dist.is_initialized()
    world, rank = (dist.get_world_size(), dist.get_rank()) if sharded else (1, 0)
    mine = tiles_of_rank(nbr * num_tiles, rank, world)
    return len(plan_tile_chunks(mine, num_tiles, batch, max_tile_forwards)[1]) > 1


def _sync_from_rank0(t: torch.Tensor, dev) -> torch.Tensor:
    import torch.distributed as dist
    t = t.to(dev).contiguous()
    dist.broadcast(t, src=0)
    return t


def _sync_rng_from_rank0(dev) -> None:
    """All ranks continue with rank 0's generator state (per-step randn_like must agree)."""
    import torch.distributed as dist
    dev = torch.device(dev)
    if dev.type == "cuda":
        st = torch.cuda.get_rng_state(dev).to(dev)
        dist.broadcast(st, src=0)
        torch.cuda.set_rng_state(st.cpu(), dev)
    else:
        st = torch.get_rng_state()
        dist.broadcast(st, src=0)
        torch.set_rng_state(st)


def tiled_callable(model, tile_size: int, tile_stride: int):
    """model(x, t, cond) evaluated on Gaussian-weighted sliding latent tiles, accumulated in row-major tile
    order and normalised — the wrapper every reference sampler puts around model.forward when `tiled`
    (spaced_sampler.py:204-219 with utils/common.py:172-232)."""
    def fwd(xx, tt, cd):
        out = torch.zeros_like(xx)
        cnt = torch.zeros_like(xx)
        w = torch.tensor(gaussian_weights(tile_size, tile_size)[None, None], dtype=xx.dtype, device=xx.device)
        for a, b, c, d in sliding_windows(xx.shape[2], xx.shape[3], tile_size, tile_stride):
            out[..., a:b, c:d] += model(xx[..., a:b, c:d], tt, {"c_txt": cd["c_txt"], "c_img": cd["c_img"][..., a:b, c:d]}) * w
            cnt[..., a:b, c:d] += w
        return out / cnt
    return fwd


class EngineEval:
    """Everything between a sampler loop and the kernel engine (shared by the spaced / DDIM loops here and the
    EDM / DPM-Solver samplers): conditioning set-up, ONE batched forward over (CFG branches x images | tiles)
    captured in a CUDA graph and replayed per evaluation, tile gather / Gaussian blend in the reference's
    accumulation order, and - with torch.distributed initialised - tiles (tiled sampling) or (branch, image)
    units (shard_batch) sharded round-robin over the ranks and re-assembled by one all-gather per evaluation.
    Tiled sampling with more than `max_tile_forwards` batch entries on a rank replays the graph once per chunk
    (plan_tile_chunks); the result has the same bits as one replay of all of them.

        ev = EngineEval(model, x_T, cond, uncond, tiled, tile_size, tile_stride)
        ev.set_timesteps([999, 979, ...])      # every model timestep the loop will ask for (floats allowed)
        e_cond, e_uncond = ev.eps(x, k)        # model output at timesteps[k]; views of internal buffers

    `ev.x0` is x_T on the engine's device (rank 0's copy when sharded: every rank must hold the same latent,
    condition and noise stream, otherwise tiles of diverging latents would be blended silently)."""

    def __init__(self, model, x_T, cond, uncond, tiled=False, tile_size=-1, tile_stride=-1, *, shard_tiles=True,
                 shard_batch=False, time_collective=False, max_tile_forwards=128):
        import torch.distributed as dist
        model._build()
        self.model, self.eng = model, model.engine
        eng = self.eng
        dev = self.dev = eng.dev
        x = x_T.to(dev, torch.float32).contiguous().clone()
        B, C, H, W = x.shape
        self.shape = (B, C, H, W)
        self.use_cfg = uncond is not None
        conds = [cond, uncond] if self.use_cfg else [cond]
        nbr = self.nbr = len(conds)
        self.tiled, self.time_collective = bool(tiled), time_collective
        sharded = (shard_tiles if tiled else shard_batch) and dist.is_available() and dist.is_initialized()
        world, rank = (dist.get_world_size(), dist.get_rank()) if sharded else (1, 0)
        self.world, self.dist = world, dist
        if world > 1:
            x = _sync_from_rank0(x, dev)
            conds = [dict(cd, c_img=_sync_from_rank0(cd["c_img"].to(dev, torch.float32).contiguous(), dev))
                     for cd in conds]
            _sync_rng_from_rank0(dev)
        self.x0 = x
        T = Tl = 0
        self.chunked = False
        if tiled:
            # unit u = branch * T + tile: the nbr * T tile-forwards of one evaluation are owned round-robin
            # (u % world). Sharding (tile, CFG branch) units instead of whole tiles keeps the ranks within one
            # forward of each other: 98 units on 8 ranks = 13 / 12 per rank, where 49 whole tiles gave 14 / 12
            # forwards (SURVEY 8e: 94 % vs 87.5 % ideal efficiency).
            wins = sliding_windows(H, W, tile_size, tile_stride)
            T = self.T = len(wins)
            ts_ = self.ts = tile_size
            self.all_coords = torch.tensor([[a, c] for a, _, c, _ in wins], dtype=torch.int32, device=dev)
            U = nbr * T
            mine = tiles_of_rank(U, rank, world)               # may be empty: U < world
            slots = tile_slots(U, world)
            Ul = self.Ul = len(mine)
            self.branch_tiles = []                             # per branch: (first local unit, count, tile coordinates)
            o = 0
            for jb in range(nbr):
                tj = [u - jb * T for u in mine if u // T == jb]
                self.branch_tiles.append((o, len(tj), self.all_coords[tj].contiguous() if tj else self.all_coords[:0]))
                o += len(tj)
            self.wts = torch.tensor(gaussian_weights(ts_, ts_), dtype=torch.float32, device=dev)
            # The tile-forwards of one evaluation are replayed in chunks of at most max_tile_forwards batch
            # entries, so the engine's activations stay bounded whatever the image size (one chunk up to the cap).
            per_chunk, self.chunks = plan_tile_chunks(mine, T, B, max_tile_forwards)
            self.chunked = len(self.chunks) > 1
            c_img = torch.empty(max(Ul, 1) * B, C, ts_, ts_, device=dev)[:Ul * B]
            ctx_parts = []
            for (o, nj, coords), cd in zip(self.branch_tiles, conds):
                if nj:
                    lib.tile_gather(cd["c_img"].to(dev, torch.float32).contiguous(), B, C, H, W, coords, nj, ts_,
                                    c_img[o * B:(o + nj) * B])
                    if not self.chunked:
                        ctx_parts.append(cd["c_txt"].to(dev, torch.float32).expand(B, -1, -1).repeat(nj, 1, 1))
            if self.chunked:
                # pad the replay to a size the engine runs as grouped twin launches where the cap allows it,
                # so chunked runs take the same forward path as the single replay of a smaller image
                per_chunk = next((n for n in range(per_chunk, max_tile_forwards // B + 1)
                                  if eng.twins_feasible(n * B, ts_, ts_)), per_chunk)
                # branch-pure chunks: one text context per branch, its cross-attention K/V built once per run
                self.unit_coords = self.all_coords[[u % T for u in mine]].contiguous()
                self.ctx_layouts = {jb: conds[jb]["c_txt"].to(dev, torch.float32).expand(B, -1, -1)
                                    .repeat(per_chunk, 1, 1) for jb in sorted({c[2] for c in self.chunks})}
                self.c_img_units = c_img
                nb, ctx = per_chunk * B, None
            else:
                nb = Ul * B
                ctx = torch.cat(ctx_parts, 0) if ctx_parts else None
            gh = gw = ts_
            Tl = Ul                                            # (stats) tile-forwards of this rank
            if world > 1:
                self.send = torch.zeros(slots, B, C, ts_, ts_, device=dev)
                self.recv = torch.empty(world, slots, B, C, ts_, ts_, device=dev)
            if self.chunked:                                   # eps of every local unit, in local slot order
                self.eps_units = self.send[:Ul] if world > 1 else torch.empty(Ul, B, C, ts_, ts_, device=dev)
            self.eps_full = torch.empty(nbr, B, C, H, W, device=dev)
        elif world > 1:
            # batch sharding: unit u = branch * B + image, owned round-robin like tiles (u % world)
            U = nbr * B
            mine = tiles_of_rank(U, rank, world)
            slots, nb = tile_slots(U, world), len(mine)
            all_c_img = torch.cat([cd["c_img"].to(dev, torch.float32) for cd in conds], 0)
            all_ctx = torch.cat([cd["c_txt"].to(dev, torch.float32).expand(B, -1, -1) for cd in conds], 0)
            sel = torch.tensor(mine, dtype=torch.long, device=dev)
            c_img = all_c_img.index_select(0, sel).contiguous()
            ctx = all_ctx.index_select(0, sel).contiguous()
            self.img_of_unit = torch.tensor([u % B for u in mine], dtype=torch.long, device=dev)
            gh, gw = H, W
            self.send = torch.zeros(slots, C, H, W, device=dev)
            self.recv = torch.empty(world, slots, C, H, W, device=dev)
        else:
            nb = nbr * B
            c_img = torch.cat([cd["c_img"].to(dev, torch.float32) for cd in conds], 0).contiguous()
            ctx = torch.cat([cd["c_txt"].to(dev, torch.float32) for cd in conds], 0)
            gh, gw = H, W
        self.nb, self.gh, self.gw = nb, gh, gw
        self._c_img, self._ctx = c_img, ctx
        self.scales = [float(s) for s in model.control_scales]
        # Tiled / sharded sampling pins the batch-invariant kernel plans (no split-K, whole attention tiles
        # per CTA): a sample's eps then has the same bits whatever the per-rank batch is, so the sharded
        # run is bit-identical to the single-rank run (SURVEY §8e).
        eng.batch_invariant = bool(tiled) or world > 1 or eng.deterministic
        self.graph = None
        self.stats = dict(world=world, tiles=T, units_this_rank=Tl, forwards_per_step=nb,
                          batch_sharded=bool(world > 1 and not tiled),
                          chunks=len(self.chunks) if tiled else int(nb > 0))

    def set_timesteps(self, model_ts) -> None:
        """Time embeddings of every timestep the loop will evaluate + the CUDA graph of the forward."""
        eng = self.eng
        self.model_ts = list(model_ts)
        if self.nb > 0:
            B, C, H, W = self.shape
            if self.chunked:
                # K/V of each branch's context, kept aside and copied into the engine's static buffers
                # whenever the next chunk belongs to the other branch
                self.kv_layouts = {}
                for jb, ctx in self.ctx_layouts.items():
                    eng.set_context(ctx)
                    self.kv_layouts[jb] = {k: v.clone() for k, v in eng.kv.items() if k.startswith("g")}
                self.kv_cur = jb
            else:
                eng.set_context(self._ctx)
            eng.set_timesteps(self.model_ts, self.nb)
            self.model._ctx_ref = self.model._t_key = None      # generic-path caches are now stale
            eng.load_step(0)
            self.graph, self.x_in, self.c_img_in, self.out, self.graph_launches = eng.graphed_forward(
                self.nb, C, self.gh, self.gw, self.scales)
            if not self.chunked:
                self.c_img_in.copy_(self._c_img)

    def _fill_inputs(self, x: torch.Tensor) -> None:
        B, C, H, W = self.shape
        nbr = self.nbr
        if self.tiled:
            for o, nj, coords in self.branch_tiles:            # this rank's tiles of each branch, in unit order
                if nj:
                    lib.tile_gather(x, B, C, H, W, coords, nj, self.ts, self.x_in[o * B:(o + nj) * B])
        elif self.world > 1:
            torch.index_select(x, 0, self.img_of_unit, out=self.x_in)
        else:
            v = self.x_in.view(nbr, B, C, H, W)
            for j in range(nbr):
                v[j].copy_(x)

    def _replay_chunks(self, x: torch.Tensor, step_idx: int) -> None:
        """One evaluation as several replays of the chunk graph; each writes its units' eps to their local slots."""
        B, C, H, W = self.shape
        ts = self.ts
        self.eng.load_step(step_idx)
        # chunks of the branch whose K/V is loaded go first: one K/V switch per evaluation
        for s, n, jb in sorted(self.chunks, key=lambda c: c[2] != self.kv_cur):
            if jb != self.kv_cur:
                for k, v in self.kv_layouts[jb].items():
                    self.eng.kv[k].copy_(v)
                self.kv_cur = jb
            lib.tile_gather(x, B, C, H, W, self.unit_coords[s:s + n], n, ts, self.x_in[:n * B])
            self.c_img_in[:n * B].copy_(self.c_img_units[s * B:(s + n) * B])
            self.graph.replay()
            lib.count_launch(self.graph_launches)
            self.eps_units[s:s + n].copy_(self.out[:n * B].view(n, B, C, ts, ts))

    def _all_gather(self) -> None:
        if self.time_collective:
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
        self.dist.all_gather_into_tensor(self.recv, self.send)
        if self.time_collective:
            ev1.record()
            self.stats.setdefault("allgather_events", []).append((ev0, ev1))

    def eps(self, x: torch.Tensor, step_idx: int):
        """(cond, uncond | None) model outputs for the full latent x at model_ts[step_idx], fp32 [B,C,H,W]."""
        B, C, H, W = self.shape
        nbr, world = self.nbr, self.world
        if self.chunked:
            self._replay_chunks(x, step_idx)
        elif self.nb > 0:
            self.eng.load_step(step_idx)
            self._fill_inputs(x)
            self.graph.replay()
            lib.count_launch(self.graph_launches)
        if self.tiled:
            if world > 1:
                if self.Ul and not self.chunked:
                    self.send[:self.Ul].copy_(self.out.view(self.Ul, B, C, self.ts, self.ts))
                self._all_gather()
                tiles = assemble_units(self.recv, nbr * self.T).view(nbr, self.T, B, C, self.ts, self.ts)
            else:
                tiles = (self.eps_units if self.chunked else self.out).view(nbr, self.T, B, C, self.ts, self.ts)
            for j in range(nbr):
                lib.tile_blend(tiles[j], B, C, H, W, self.all_coords, self.T, self.ts, self.wts, self.eps_full[j])
            ev = self.eps_full
        elif world > 1:
            if self.nb:
                self.send[:self.nb].copy_(self.out)
            self._all_gather()
            ev = assemble_units(self.recv, nbr * B).view(nbr, B, C, H, W)
        else:
            ev = self.out.view(nbr, B, C, H, W)
        return ev[0], (ev[1] if self.use_cfg else None)


class Sampler:
    time_collective = False        # record CUDA events around the per-step all-gather (bench.py sets it)

    def __init__(self, betas: np.ndarray, parameterization: str, rescale_cfg: bool):
        self.num_timesteps = len(betas)
        self.training_betas = betas
        self.training_alphas_cumprod = np.cumprod(1.0 - betas, axis=0)
        self.parameterization = parameterization
        self.rescale_cfg = rescale_cfg
        self.shard_tiles = True     # tiled sampling: shard tiles over torch.distributed ranks
        # un-tiled sampling of a batch: shard the (CFG branch, image) forwards over the ranks with one
        # all-gather of eps per step (BASELINE configs[4]: 4 images x 2 branches -> one forward per GPU of
        # an 8-GPU box). Opt-in: ranks that restore DIFFERENT images (independent replicas) must not shard.
        self.shard_batch = False
        # tiled sampling: the most batch entries (tile-forwards x images) one graph replay may hold. More units
        # than that run as several replays per evaluation, so memory stops growing with the image size; the
        # 49-tile (98-forward) 2048^2 restoration still takes one replay.
        self.max_tile_forwards = 128
        self.noise_source: Optional[NoiseSource] = None     # per-sample draws (None: the global generators)
        self.last_stats: dict = {}

    def get_cfg_scale(self, default_cfg_scale: float, model_t: int) -> float:
        """Cosine CFG ramp — sampler/sampler.py:31-38."""
        if self.rescale_cfg and default_cfg_scale > 1:
            return 1 + default_cfg_scale * ((1 - math.cos(math.pi * ((1000 - model_t) / 1000) ** 5.0)) / 2)
        return default_cfg_scale

    # ---- subclass interface -------------------------------------------------------------
    def make_schedule(self, steps: int):
        raise NotImplementedError

    def _step_coefs(self) -> Tuple[np.ndarray, torch.Tensor, int]:
        """(model timesteps ascending, fp32 coefficient rows [S, 8] per table index, kernel mode)"""
        raise NotImplementedError

    # ---- shared driver --------------------------------------------------------------------
    @torch.no_grad()
    def sample(self, model, device, steps: int, x_size: Tuple[int], cond: Dict[str, torch.Tensor],
               uncond: Optional[Dict[str, torch.Tensor]], cfg_scale: float, tiled: bool = False,
               tile_size: int = -1, tile_stride: int = -1, x_T: Optional[torch.Tensor] = None,
               progress: bool = True) -> torch.Tensor:
        self.make_schedule(steps)
        ts, coefs, mode = self._step_coefs()
        if x_T is None:
            x_T = randn(x_size, device, self.noise_source)
        from ..model.cldm import ControlLDM
        if isinstance(model, ControlLDM):
            return self._sample_engine(model, ts, coefs, mode, x_T, cond, uncond, cfg_scale, tiled,
                                       tile_size, tile_stride)
        return self._sample_generic(model, ts, coefs, mode, x_T, cond, uncond, cfg_scale, tiled,
                                    tile_size, tile_stride)

    # ---- kernel-engine path -----------------------------------------------------------------
    def _sample_engine(self, model, ts, coefs, mode, x_T, cond, uncond, cfg_scale, tiled, tile_size,
                       tile_stride):
        use_cfg = not (uncond is None or cfg_scale == 1.0)
        ev = EngineEval(model, x_T, cond, uncond if use_cfg else None, tiled, tile_size, tile_stride,
                        shard_tiles=self.shard_tiles, shard_batch=self.shard_batch, time_collective=self.time_collective,
                        max_tile_forwards=self.max_tile_forwards)
        x = ev.x0
        coefs = coefs.to(ev.dev)
        order = list(range(len(ts)))[::-1]                     # table index of each loop iteration
        model_ts = [int(ts[i]) for i in order]
        ev.set_timesteps(model_ts)
        x_next = torch.empty_like(x)
        self.last_stats = ev.stats
        for it, tab_idx in enumerate(order):
            e_c, e_u = ev.eps(x, it)
            noise = randn_like(x, self.noise_source)
            cur_cfg = self.get_cfg_scale(cfg_scale, model_ts[it])
            if cur_cfg == 1.0:
                e_u = None      # the reference takes the cond-only branch on such steps (spaced_sampler.py:150-152)
            lib.sampler_step(e_c, e_u, cur_cfg, x, noise, coefs[tab_idx], mode, x.numel(), x_next)
            x, x_next = x_next, x
        return x

    # ---- plain PyTorch path for foreign models --------------------------------------------
    def _sample_generic(self, model, ts, coefs, mode, x_T, cond, uncond, cfg_scale, tiled, tile_size,
                        tile_stride):
        x = x_T
        dev = x.device
        coefs = coefs.to(dev)
        fwd = tiled_callable(model, tile_size, tile_stride) if tiled else model
        for tab_idx in list(range(len(ts)))[::-1]:
            step = int(ts[tab_idx])
            model_t = torch.full((x.shape[0],), step, device=dev, dtype=torch.long)
            s = self.get_cfg_scale(cfg_scale, step)
            if uncond is None or s == 1.0:
                e = fwd(x, model_t, cond)
            else:
                ec, eu = fwd(x, model_t, cond), fwd(x, model_t, uncond)
                e = eu + s * (ec - eu)
            c = coefs[tab_idx]
            noise = randn_like(x, self.noise_source)
            if mode in (0, 1):
                x0 = c[0] * x - c[1] * e
                x = (c[2] * x0 + c[3] * x) + c[4] * noise
            else:
                if mode == 3:
                    e = c[5] * e + c[1] * x
                x0 = (x - c[1] * e) / c[0]
                x = c[2] * x0 + c[3] * e + c[4] * noise
        return x


class SpacedSampler(Sampler):
    def make_schedule(self, num_steps: int) -> None:
        """spaced_sampler.py:77-116 — respaced betas and posterior tables in fp64."""
        used = space_timesteps(self.num_timesteps, num_steps)
        betas, last = [], 1.0
        for i in used:
            betas.append(1 - self.training_alphas_cumprod[i] / last)
            last = self.training_alphas_cumprod[i]
        self.timesteps = used
        b = np.array(betas, dtype=np.float64)
        a = 1.0 - b
        ac = np.cumprod(a, axis=0)
        ac_prev = np.append(1.0, ac[:-1])
        with np.errstate(divide="ignore"):
            self.tables = dict(
                sqrt_alphas_cumprod=np.sqrt(ac), sqrt_one_minus_alphas_cumprod=np.sqrt(1 - ac),
                sqrt_recip_alphas_cumprod=np.sqrt(1.0 / ac), sqrt_recipm1_alphas_cumprod=np.sqrt(1.0 / ac - 1),
                posterior_variance=b * (1.0 - ac_prev) / (1.0 - ac),
                posterior_mean_coef1=b * np.sqrt(ac_prev) / (1.0 - ac),
                posterior_mean_coef2=(1.0 - ac_prev) * np.sqrt(a) / (1.0 - ac))

    def _step_coefs(self):
        tb = {k: torch.tensor(v, dtype=torch.float32) for k, v in self.tables.items()}
        S = len(self.timesteps)
        c = torch.zeros(S, 8, dtype=torch.float32)
        if self.parameterization == "eps":
            c[:, 0], c[:, 1], mode = tb["sqrt_recip_alphas_cumprod"], tb["sqrt_recipm1_alphas_cumprod"], 0
        else:
            c[:, 0], c[:, 1], mode = tb["sqrt_alphas_cumprod"], tb["sqrt_one_minus_alphas_cumprod"], 1
        c[:, 2], c[:, 3] = tb["posterior_mean_coef1"], tb["posterior_mean_coef2"]
        nonzero = (torch.arange(S) != 0).float()                  # spaced_sampler.py:182
        c[:, 4] = nonzero * torch.sqrt(tb["posterior_variance"])
        return self.timesteps, c, mode


class DDIMSampler(Sampler):
    def __init__(self, betas, parameterization, rescale_cfg, eta: float):
        super().__init__(betas, parameterization, rescale_cfg)
        self.eta = eta

    def make_schedule(self, ddim_num_steps, ddim_discretize="uniform"):
        """ddim_sampler.py:13-58, 73-96 (uniform stride, +1 offset)."""
        c = self.num_timesteps // ddim_num_steps
        self.ddim_timesteps = np.asarray(list(range(0, self.num_timesteps, c))) + 1
        ac = self.training_alphas_cumprod
        alphas = ac[self.ddim_timesteps]
        alphas_prev = np.asarray([ac[0]] + ac[self.ddim_timesteps[:-1]].tolist())
        sigmas = self.eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))
        self.tables = dict(ddim_sigmas=sigmas, ddim_alphas=alphas, ddim_alphas_prev=alphas_prev,
                           ddim_sqrt_alphas=np.sqrt(alphas), ddim_sqrt_one_minus_alphas=np.sqrt(1.0 - alphas))

    def _step_coefs(self):
        tb = {k: torch.tensor(v, dtype=torch.float32) for k, v in self.tables.items()}
        S = len(self.ddim_timesteps)
        c = torch.zeros(S, 8, dtype=torch.float32)
        c[:, 0] = tb["ddim_alphas"].sqrt()                                       # a_t.sqrt()
        c[:, 1] = tb["ddim_sqrt_one_minus_alphas"]
        c[:, 2] = tb["ddim_alphas_prev"].sqrt()
        c[:, 3] = (1.0 - tb["ddim_alphas_prev"] - tb["ddim_sigmas"] ** 2).sqrt()
        c[:, 4] = tb["ddim_sigmas"]
        c[:, 5] = tb["ddim_sqrt_alphas"]
        return self.ddim_timesteps, c, (2 if self.parameterization == "eps" else 3)
