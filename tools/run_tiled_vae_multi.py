"""torchrun target: the tiled VAE sharded over NCCL ranks must be BIT-IDENTICAL to the single-rank tiled VAE on
every rank, and all ranks must hold the same result; a small-config SwinIRPipeline.run with tiled sampling and both
VAE flags must give the same uint8 image with the VAE sharded as with `pipe.shard_vae = False`. Exit code 0 = pass."""
import os
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from diffbir_b200 import arch  # noqa: E402
from diffbir_b200.engine.vae import VaeEngine  # noqa: E402
from diffbir_b200.engine.vae_tiled import TiledVae  # noqa: E402
from diffbir_b200.utils.synth import RUN_DEFAULTS, build_synthetic_pipeline, make_state_dict, synthetic_lq  # noqa: E402


def all_ranks_equal(t: torch.Tensor) -> bool:
    out = torch.empty((dist.get_world_size(),) + tuple(t.shape), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, t.contiguous())
    return all(torch.equal(out[0], o) for o in out)


def main():
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    dev = f"cuda:{local}"
    dist.init_process_group("nccl", device_id=torch.device(dev))
    torch.backends.cuda.matmul.allow_tf32 = False
    ok = True
    # (config, image, encoder tile): small config with ragged tiles and two images; full config at 768 x 1280
    for name, cfg, shape, tile in (("small", dict(arch.VAE_CFG, ch=64), (2, 3, 200, 328), 64),
                                   ("full", arch.VAE_CFG, (1, 3, 768, 1280), 256)):
        base = VaeEngine(make_state_dict(arch.vae_shapes(cfg), 77), cfg, dev)
        single, sharded = TiledVae(base), TiledVae(base, rank, world)
        g = torch.Generator().manual_seed(5)
        img = (torch.rand(shape, generator=g) * 2 - 1).to(dev)
        z = (torch.randn(shape[0], 4, shape[2] // 8, shape[3] // 8, generator=g) * 0.8).to(dev)
        for what, fn_s, fn_1, x, t in (("encode", sharded.encode_moments, single.encode_moments, img, tile),
                                       ("decode", sharded.decode, single.decode, z, tile // 8)):
            a = fn_s(x, t)
            stats = dict(sharded.last_stats)
            b = fn_1(x, t)
            same, same_ranks = torch.equal(a, b) and torch.equal(a.signbit(), b.signbit()), all_ranks_equal(a)
            owned = torch.tensor([stats["owned"]], device=dev)
            dist.all_reduce(owned)
            print(f"rank {rank}: {name} {what} {tuple(x.shape)} tile {t}, {world} ranks: bit-equal to one rank {same}, "
                  f"all ranks identical {same_ranks}; {stats}", flush=True)
            ok = ok and same and same_ranks and int(owned) == stats["tiles"] and stats["exchanges"] > 0
        del base, single, sharded
    # the pipeline: tiled sampling (sharded over the ranks), tiled VAE encode and decode, sharded vs replicated VAE
    pipe = build_synthetic_pipeline(dev, seed=1234, small=True)
    scfg = dict(arch.SWINIR_CFG, depths=(2, 2), num_heads=(6, 6))
    pipe.cleaner.engine_sd = make_state_dict(arch.swinir_shapes(scfg), 1234 + 4)
    lq = synthetic_lq(640, 768, seed=3)
    kw = dict(RUN_DEFAULTS, steps=3, cldm_tiled=True, vae_encoder_tiled=True, vae_encoder_tile_size=256,
              vae_decoder_tiled=True, vae_decoder_tile_size=256)
    outs = []
    for shard in (True, False):
        pipe.shard_vae = shard
        torch.manual_seed(231)
        outs.append(pipe.run(lq, **kw))
        st = dict(pipe.cldm._tvae.last_stats)
        print(f"rank {rank}: pipeline 640x768, shard_vae {shard}: tiled VAE decode {st}", flush=True)
        ok = ok and (st["exchanges"] > 0) == shard
    same = bool((outs[0] == outs[1]).all())
    diff = int((outs[0].astype(int) - outs[1].astype(int)).__abs__().max())
    print(f"rank {rank}: pipeline uint8 output sharded vs replicated VAE: equal {same} (max diff {diff})", flush=True)
    ok = ok and same and all_ranks_equal(torch.from_numpy(outs[0]).to(dev))
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    sys.exit(0 if int(flag) == 1 else 1)


if __name__ == "__main__":
    main()
