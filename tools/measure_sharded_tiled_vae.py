"""Time and peak memory of the tiled VAE sharded over cooperating ranks, full SD configuration (synthetic weights).

    torchrun --nproc-per-node R tools/measure_sharded_tiled_vae.py [--sizes 2048 3072 4096] [--tile 1024]

For each image size: a tiled encode of the image and a tiled decode of its latent, with 1024-pixel tiles by default.
Each call runs once to warm up, then, after the allocator's cache is released, once timed with CUDA events around
it on every rank (the first call of a shape also tunes its GEMMs); the peak is torch.cuda.max_memory_allocated over the
timed call. Rank 0 prints, per rank, the time, the peak, the tiles it owns,
its waves and its spills, and the GPU name and power limit. `--nproc-per-node 1` measures the single-rank tiled VAE
(no exchange) on the same path.
"""
import argparse
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[2048, 3072, 4096])
    ap.add_argument("--tile", type=int, default=1024, help="encoder and decoder tile size in image pixels")
    args = ap.parse_args()

    import torch
    import torch.distributed as dist
    from diffbir_b200 import arch
    from diffbir_b200.engine.vae import VaeEngine
    from diffbir_b200.engine.vae_tiled import TiledVae
    from diffbir_b200.utils.synth import make_state_dict

    assert torch.cuda.is_available(), "measure_sharded_tiled_vae needs a CUDA device"
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dev = f"cuda:{local}"
    dist.init_process_group("nccl", device_id=torch.device(dev))
    q = subprocess.run(["nvidia-smi", "-i", str(local), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    devices = [None] * world
    dist.all_gather_object(devices, q)
    if rank == 0:
        for r, d in enumerate(devices):
            print(f"rank {r} device: {d}", flush=True)
    tv = TiledVae(VaeEngine(make_state_dict(arch.vae_shapes(arch.VAE_CFG), 77), arch.VAE_CFG, dev), rank, world)

    def timed(fn, *a):
        fn(*a)
        torch.cuda.synchronize()
        # the default state budget is half the free device memory: memory the caching allocator still holds from
        # earlier calls would count as used and stage waves a fresh process keeps on the device
        torch.cuda.empty_cache()
        dist.barrier()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(*a)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), torch.cuda.max_memory_allocated() / 2 ** 30, dict(tv.last_stats)

    for s in args.sizes:
        g = torch.Generator().manual_seed(s)
        img = (torch.rand(1, 3, s, s, generator=g) * 2 - 1).to(dev)
        z = (torch.randn(1, 4, s // 8, s // 8, generator=g) * 0.8).to(dev)
        for what, fn, x, t in (("encode", tv.encode_moments, img, args.tile), ("decode", tv.decode, z, args.tile // 8)):
            ms, peak, st = timed(fn, x, t)
            rows = [None] * world
            dist.all_gather_object(rows, (ms, peak, st))
            if rank == 0:
                for r, (ms, peak, st) in enumerate(rows):
                    print(f"{s}^2 {what} on {world} rank(s), rank {r}: {ms:8.0f} ms, peak {peak:5.1f} GiB, "
                          f"{st['owned']} of {st['tiles']} tiles, {st['waves']} waves, {st['spills']} spills, "
                          f"{st['exchanges']} exchanges", flush=True)
        del img, z
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
