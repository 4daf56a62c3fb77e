"""Folder throughput of `inference.py --distribute images` at world size 1 and at the world size this is launched with.

  torchrun --nproc-per-node 8 tools/measure_cli_ranks.py [--images 16] [--steps 50]

Every rank builds the CLI's loop on synthetic weights (full SD-2.1 config, v2.1 recipe, 128^2 inputs x4 = 512^2
outputs), warms up on one image, then times (a) rank 0 restoring the whole folder alone, the way `python
inference.py` does, and (b) all ranks restoring it together, images dealt round-robin, prompt.csv gathered to
rank 0. Times are host clocks around work that ends in a device synchronise and a barrier, PNG writes included.
Rank 0 prints one JSON line: MPix/s at both sizes and the scaling efficiency (b over N x a)."""
import argparse
import json
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
from PIL import Image  # noqa: E402

import inference as cli  # noqa: E402
from diffbir_b200.inference import BSRInferenceLoop  # noqa: E402
from diffbir_b200.inference import ranks as rank_mod  # noqa: E402
from diffbir_b200.utils.synth import synthetic_lq  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--steps", type=int, default=50)
    opt = ap.parse_args()
    env = rank_mod.torchrun_env()
    if env is None:
        raise SystemExit("launch with torchrun (any --nproc-per-node, 1 included)")
    root = Path(tempfile.mkdtemp(prefix="measure_cli_ranks_")) if env[0] == 0 else None
    flags = ["--task", "sr", "--version", "v2.1", "--upscale", "4", "--sampler", "spaced", "--steps", str(opt.steps),
             "--cfg_scale", "4.0", "--captioner", "none", "--synthetic", "--distribute", "images"]
    args = cli.parse_args(flags + ["--input", "-", "--output", "-"])
    ranks = rank_mod.launch(args, cli.set_seed)
    try:
        world, rank = ranks.world, ranks.rank
        box = [str(root) if rank == 0 else None]
        dist.broadcast_object_list(box, src=0)              # one folder on the box, rank 0's
        root = Path(box[0])
        if rank == 0:
            for d in ("in", "warm"):
                (root / d).mkdir()
            for i in range(opt.images):
                Image.fromarray(synthetic_lq(128, 128, seed=i)[0]).save(root / "in" / f"{i:03d}.png")
            for i in range(world):
                Image.fromarray(synthetic_lq(128, 128, seed=1000 + i)[0]).save(root / "warm" / f"{i:03d}.png")
        dist.barrier(group=ranks.host_group)
        cli.set_seed(args.seed)
        loop = BSRInferenceLoop(args, ranks)
        ranks.configure(loop.pipelines())

        def timed(inp, out, ranks_):
            loop.args = cli.parse_args(flags + ["--input", str(root / inp), "--output", str(root / out)])
            loop.ranks = ranks_
            t0 = time.perf_counter()
            loop.run()
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        host = ranks.host_group                              # waits of any length (rank 0's world-1 pass)
        timed("warm", "warm_out", ranks)                     # one image per rank: plans, graphs, allocator
        dist.barrier(group=host)
        t1 = timed("in", "out_1", None) if rank == 0 else 0.0
        dist.barrier(group=host)
        t0 = time.perf_counter()
        timed("in", "out_n", ranks)
        dist.barrier(group=host)
        tn = time.perf_counter() - t0
        if rank == 0:
            mpix = opt.images * 512 * 512 / 1e6
            name = torch.cuda.get_device_name()
            limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                   capture_output=True, text=True).stdout.strip()
            print(json.dumps(dict(gpu=name, power_limit=limit, world=world, images=opt.images, steps=opt.steps,
                                  world1_s=round(t1, 3), world1_mpix_s=round(mpix / t1, 4),
                                  worldN_s=round(tn, 3), worldN_mpix_s=round(mpix / tn, 4),
                                  scaling_efficiency=round(t1 / (world * tn), 4))), flush=True)
        dist.barrier(group=host)
        if rank == 0:
            shutil.rmtree(root)
    finally:
        rank_mod.close()


if __name__ == "__main__":
    main()
