"""Time the device Brownian tree (dbir_brownian_increment) per query at the latents of 512² and 1024² images, and the
share of one `edm_dpm++_sde` step it takes (two queries per step) on the synthetic full-size v2.1 pipeline, with
torchsde hidden so that the sampler uses the device tree. Prints one JSON object with the card's name and power limit
read in the same run.

    python tools/measure_brownian.py [--steps 10] [--reps 200] [--windows 5]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def events_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--windows", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "measure_brownian.py needs a CUDA device"
    sys.modules["torchsde"] = None                  # the sampler takes the device tree, as on a stock install
    from diffbir_b200 import lib
    from diffbir_b200.sampler import edm
    from diffbir_b200.utils.synth import RUN_DEFAULTS, build_synthetic_pipeline, synthetic_lq
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    lib.load()
    pipe = build_synthetic_pipeline("cuda", v_prediction=True)
    sampler = edm.EDMSampler(pipe.diffusion.betas, "v", False, "edm_dpm++_sde", 0, 0, 300, 1, 1, 1)
    sampler.make_schedule(a.steps)
    sig = sampler.sigmas.double()
    lo, hi = float(sig[sig > 0].min()), float(sig.max())
    depth = edm.brownian_depth(lo, hi)
    s_i, s_n = float(sig[a.steps // 2]), float(sig[a.steps // 2 + 1])          # a query of a middle step

    result = {"card": card, "config": f"v2.1 ladder, {a.steps} steps, tree [{lo:.6g}, {hi:.6g}], depth {depth}",
              "query_ms": {}, "step_ms": {}, "share_of_step": {}}
    for size in (512, 1024):
        out = torch.empty(1, 4, size // 8, size // 8, device="cuda")
        q = lambda: lib.brownian_increment(out, 12345, lo, hi, s_n, s_i, depth)   # noqa: E731
        q()
        result["query_ms"][f"{size}^2"] = round(float(np.median([events_ms(q, a.reps) for _ in range(a.windows)])), 4)

        lq = synthetic_lq(size, size, seed=3)
        run = dict(RUN_DEFAULTS, steps=a.steps, sampler_type="edm_dpm++_sde")
        torch.manual_seed(0)
        pipe.run(lq, **run)                                                        # warm-up: graphs, plans
        loops = []
        for w in range(3):
            pipe.marks = []
            torch.manual_seed(w)
            pipe.run(lq, **run)
            torch.cuda.synchronize()
            loops.append(pipe.phases_ms()["sampler_loop"])
        pipe.marks = None
        step = float(np.median(loops)) / a.steps
        result["step_ms"][f"{size}^2"] = round(step, 3)
        result["share_of_step"][f"{size}^2"] = round(2 * result["query_ms"][f"{size}^2"] / step, 6)
    result["note"] = ("query_ms: CUDA events around back-to-back launches (median of windows); step_ms: the "
                      "sampler loop of Pipeline.run over its steps (batch 1, CFG 4.0, un-tiled; the last step is an "
                      "Euler step without noise); share_of_step = 2 queries / step")
    print(json.dumps(result))


if __name__ == "__main__":
    main()
