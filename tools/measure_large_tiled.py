"""Peak device memory and sampler-step time of large tiled restorations on one GPU.

Runs the full-configuration SwinIRPipeline on synthetic weights with tiled SwinIR (512 / 256), tiled sampling
(512 / 256) and the un-tiled VAE, 2 spaced steps, at 2048^2, 2560^2 and 3072^2, then attempts 4096^2. Prints one
JSON line per size: torch.cuda.max_memory_allocated of each phase (cleaner, VAE encode, sampler loop, VAE decode),
the number of graph replays per evaluation (chunks), ms per sampler step, and the outcome.

    python tools/measure_large_tiled.py [--sizes 2048,2560,3072,4096] [--steps 2] [--max-tile-forwards 128]
"""
import argparse
import gc
import json
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from diffbir_b200.sampler import sampler as sampler_mod  # noqa: E402
from diffbir_b200.utils.synth import RUN_DEFAULTS, build_synthetic_pipeline, synthetic_lq  # noqa: E402


class PhaseMemory:
    """Wraps callables so that each records the peak allocated memory while it ran, under a phase name."""

    def __init__(self):
        self.peak_gib = {}

    def wrap(self, name, fn):
        def run(*a, **kw):
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            try:
                return fn(*a, **kw)
            finally:
                self.peak_gib[name] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
        return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="2048,2560,3072,4096")
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--max-tile-forwards", type=int, default=128)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev_name = torch.cuda.get_device_name()
    pipe = build_synthetic_pipeline("cuda", seed=1234, small=False)
    pipe.max_tile_forwards = args.max_tile_forwards
    cl = pipe.cldm
    mem = PhaseMemory()
    pipe.apply_cleaner = mem.wrap("cleaner", pipe.apply_cleaner)
    cl.prepare_condition_pair = mem.wrap("encode", cl.prepare_condition_pair)
    cl.vae_decode = mem.wrap("decode", cl.vae_decode)
    step_events = []
    eps = sampler_mod.EngineEval.eps

    def timed_eps(self, x, k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = eps(self, x, k)
        e1.record()
        step_events.append((e0, e1))
        return out
    sampler_mod.EngineEval.eps = timed_eps
    sample = sampler_mod.SpacedSampler.sample
    sampler_mod.SpacedSampler.sample = mem.wrap("sampler_loop", sample)
    kw = dict(RUN_DEFAULTS, steps=args.steps, cldm_tiled=True, cleaner_tiled=True)
    for size in [int(s) for s in args.sizes.split(",")]:
        mem.peak_gib = {}
        step_events.clear()
        rec = dict(size=size, steps=args.steps, max_tile_forwards=args.max_tile_forwards, device=dev_name)
        lq = synthetic_lq(size, size, seed=8)
        t0 = time.perf_counter()
        try:
            torch.manual_seed(231)
            out = pipe.run(lq, **kw)
            torch.cuda.synchronize()
            st = pipe.last_sampler.last_stats
            rec.update(outcome="ok", seconds=round(time.perf_counter() - t0, 1), tiles=st["tiles"],
                       chunks=st["chunks"], entries_per_replay=st["forwards_per_step"],
                       ms_per_step=round(sum(a.elapsed_time(b) for a, b in step_events) / len(step_events), 1),
                       output_mean=round(float(out.mean()), 2))
        except torch.OutOfMemoryError as e:
            rec.update(outcome="out of memory", seconds=round(time.perf_counter() - t0, 1),
                       error=str(e).splitlines()[0][:200])
        rec["peak_gib"] = dict(mem.peak_gib)
        out = None
        cl.release_engine_buffers()
        gc.collect()
        torch.cuda.empty_cache()
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
