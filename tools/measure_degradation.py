"""Time RealESRGANBatchTransform (v2.1 settings, queue of two batches) on the engine against the same transform
in stock torch ops (oracle/degradation.py) on the same GPU, in alternating windows after warm-up, with device
events; then each stage on its own, engine op against torch op, on fixed inputs of the sizes a v2.1 call sees.
Prints one JSON object (card name and power limit read in the same run).

    python tools/measure_degradation.py [--batch 16] [--size 512] [--windows 6] [--calls 5]
"""
import argparse
import json
import random
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

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
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--size", type=int, default=512)
    ap.add_argument("--windows", type=int, default=6)
    ap.add_argument("--calls", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "measure_degradation.py needs a CUDA device"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from diffbir_b200 import lib
    from diffbir_b200.dataset import batch_transform as bt
    from diffbir_b200.dataset.degradation import random_add_gaussian_noise_pt, random_add_poisson_noise_pt
    from diffbir_b200.dataset.utils import USMSharp, filter2D
    from oracle import degradation as od
    from tests.test_gpu_degradation import V21, v21_batch
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    lib.load()
    cfg = dict(V21, queue_size=2 * a.batch)
    batches = [v21_batch(a.batch, a.size, i) for i in range(a.calls)]
    eng, ora = bt.RealESRGANBatchTransform(**cfg), od.BatchTransform(**cfg)

    def run(t):
        def go():
            for i, b in enumerate(batches):
                random.seed(i)
                np.random.seed(i)
                torch.manual_seed(i)
                t(b)
        return go

    for t in (eng, ora):                       # warm-up: every mode / branch the seeds take, queue filled
        run(t)()
    whole = {"engine": [], "torch": []}
    for _ in range(a.windows):
        whole["engine"].append(events_ms(run(eng), 1) / a.calls)
        whole["torch"].append(events_ms(run(ora), 1) / a.calls)

    # stages on fixed inputs
    b, s = a.batch, a.size
    x = torch.rand(b, 3, s, s, device="cuda")
    small = torch.rand(b, 3, s // 4, s // 4, device="cuda")
    k21 = batches[0]["kernel1"]
    usm, ukern = USMSharp().cuda(), od.usm_kernel().cuda()
    q = torch.full((b,), 60.0, device="cuda")
    jpeger = eng.jpeger
    stages = {
        "usm_sharpen": (lambda: usm(x), lambda: od.usm(x, ukern)),
        "blur_21x21": (lambda: filter2D(x, k21), lambda: od.filter2d(x, k21)),
        "resize_down_bicubic": (lambda: bt.resize(x, "bicubic", scale=0.6),
                                lambda: F.interpolate(x, scale_factor=0.6, mode="bicubic")),
        "resize_down_area": (lambda: bt.resize(x, "area", scale=0.6),
                             lambda: F.interpolate(x, scale_factor=0.6, mode="area")),
        "resize_up_bilinear": (lambda: bt.resize(small, "bilinear", size=(s, s)),
                               lambda: F.interpolate(small, size=(s, s), mode="bilinear")),
        "gaussian_noise_gray": (lambda: random_add_gaussian_noise_pt(x, (1, 30), gray_prob=1.0),
                                lambda: od.gaussian_noise(x, (1, 30), 1.0)),
        "poisson_noise_gray": (lambda: random_add_poisson_noise_pt(x, (0.05, 3), gray_prob=1.0),
                               lambda: od.poisson_noise(x, (0.05, 3), 1.0)),
        "diffjpeg": (lambda: jpeger(x, q), lambda: od.diffjpeg(x, q.clone())),
    }
    per_stage = {}
    for name, (fe, ft) in stages.items():
        fe(), ft()
        e, t = [], []
        for _ in range(3):
            e.append(events_ms(fe, 10))
            t.append(events_ms(ft, 10))
        per_stage[name] = {"engine_ms": round(min(e), 3), "torch_ms": round(min(t), 3)}
    print(json.dumps({"card": card, "batch": b, "size": s, "config": "v2.1 batch_transform, queue 2 batches",
                      "call_ms": {k: [round(v, 2) for v in vs] for k, vs in whole.items()},
                      "call_ms_median": {k: round(float(np.median(v)), 2) for k, v in whole.items()},
                      "stages": per_stage}))


if __name__ == "__main__":
    main()
