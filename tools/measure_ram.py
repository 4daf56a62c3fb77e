"""Time one 384^2 RAM++ captioning (RamPlusEngine graph replay, batch 1) with device events, warm, over >= 20 runs,
and the device memory the captioner adds (packed weights + workspace + graph pool). Synthetic weights (the timing does
not depend on their values).

    python tools/measure_ram.py [--runs 50]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=50)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "measure_ram.py needs a CUDA device"
    from diffbir_b200 import lib
    from diffbir_b200.engine.ram import RamPlusEngine
    from diffbir_b200.utils.synth import synthetic_ram
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    sd, _, _ = synthetic_ram(1)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    eng = RamPlusEngine(sd, device="cuda")
    x = torch.rand(1, 3, 384, 384, generator=torch.Generator().manual_seed(0)).cuda()
    for _ in range(5):
        eng.forward(x)
    torch.cuda.synchronize()
    times = []
    for _ in range(max(a.runs, 20)):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        eng.forward(x)
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    times.sort()
    res = dict(card=card, operands=str(lib.operand_dtype()), runs=len(times), median_ms=times[len(times) // 2],
               min_ms=times[0], max_ms=times[-1], added_peak_gib=(torch.cuda.max_memory_allocated() - base) / 2 ** 30,
               resident_gib=(torch.cuda.memory_allocated() - base) / 2 ** 30)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
