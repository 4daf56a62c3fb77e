"""Peak memory and time of the tiled VAE (engine.vae_tiled) at the full SD configuration (synthetic weights).

    python tools/measure_tiled_vae.py [--sizes 2048 3072 4096] [--tile 1024] [--no-pipeline]

For each image size: a tiled encode of the image and a tiled decode of its latent, once with the wave state resident
on the device and once staged through pinned host memory (state_budget 0). Each is run once to warm up and then
timed with a device synchronise around it; the peak is torch.cuda.max_memory_allocated over the timed call.
Then the full SwinIRPipeline at the largest size with the VAE, the sampler and the cleaner tiled, 2 steps.
"""
import argparse
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[2048, 3072, 4096])
    ap.add_argument("--tile", type=int, default=1024, help="encoder and decoder tile size in image pixels")
    ap.add_argument("--no-pipeline", action="store_true")
    args = ap.parse_args()

    import subprocess
    import torch
    from diffbir_b200 import arch
    from diffbir_b200.engine.vae import VaeEngine
    from diffbir_b200.engine.vae_tiled import TiledVae
    from diffbir_b200.utils.synth import RUN_DEFAULTS, build_synthetic_pipeline, make_state_dict, synthetic_lq

    assert torch.cuda.is_available(), "measure_tiled_vae needs a CUDA device"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print(f"device: {q}")
    tv = TiledVae(VaeEngine(make_state_dict(arch.vae_shapes(arch.VAE_CFG), 77), arch.VAE_CFG, "cuda"))

    def timed(fn, *a):
        fn(*a)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        out = fn(*a)
        torch.cuda.synchronize()
        return out, time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30

    for s in args.sizes:
        g = torch.Generator().manual_seed(s)
        img = (torch.rand(1, 3, s, s, generator=g) * 2 - 1).cuda()
        z = (torch.randn(1, 4, s // 8, s // 8, generator=g) * 0.8).cuda()
        for mode, budget in (("resident", None), ("spilled", 0)):
            tv.state_budget = budget
            _, te, pe = timed(tv.encode_moments, img, args.tile)
            se = dict(tv.last_stats)
            _, td, pd = timed(tv.decode, z, args.tile // 8)
            sdec = dict(tv.last_stats)
            print(f"{s}^2 {mode:8s}: encode {te * 1e3:8.0f} ms peak {pe:5.1f} GiB ({se['tiles']} tiles, {se['waves']} waves, "
                  f"{se['spills']} spills) | decode {td * 1e3:8.0f} ms peak {pd:5.1f} GiB ({sdec['tiles']} tiles, "
                  f"{sdec['waves']} waves, {sdec['spills']} spills)", flush=True)
        del img, z
    tv.state_budget = None
    del tv
    torch.cuda.empty_cache()

    if not args.no_pipeline:
        s = max(args.sizes)
        pipe = build_synthetic_pipeline("cuda", seed=1234, small=False)
        lq = synthetic_lq(s, s, seed=8)
        kw = dict(RUN_DEFAULTS, steps=2, cldm_tiled=True, cleaner_tiled=True, vae_encoder_tiled=True,
                  vae_encoder_tile_size=args.tile, vae_decoder_tiled=True, vae_decoder_tile_size=args.tile)
        pipe.marks = []
        torch.cuda.reset_peak_memory_stats()
        torch.manual_seed(231)
        t0 = time.perf_counter()
        out = pipe.run(lq, **kw)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        ph = {k: round(v) for k, v in pipe.phases_ms().items()}
        print(f"pipeline {s}^2, 2 steps, everything tiled: {dt:.1f} s, peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} "
              f"GiB, phases ms {ph}, output {tuple(out.shape)} std {out.std():.1f}")


if __name__ == "__main__":
    main()
