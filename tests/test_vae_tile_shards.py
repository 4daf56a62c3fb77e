"""The tiled VAE sharded over cooperating ranks, host side (no GPU): tile ownership over the reference's splits, and
the payloads of the GroupNorm exchange and of the output assembly under spawned gloo ranks."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from diffbir_b200 import arch
from diffbir_b200.engine.vae import VaeWalk
from diffbir_b200.engine.vae_tiled import (ProcessGroupGather, box_share, entries_of_ranks, moment_rows, pack_boxes,
                                           pack_moments, plan_vae_tiles, tiles_of_ranks, unpack_boxes,
                                           unpack_moments)


@pytest.fixture(scope="module")
def plans(golden_dir):
    fx = np.load(golden_dir / "tilevae_small.npz")
    out = []
    for key in (k[:-3] for k in fx.files if k.startswith("plan_") and k.endswith("_in")):
        _, side, h, w, t = key.split("_")
        out.append(plan_vae_tiles(int(h), int(w), int(t), side == "dec"))
    assert len(out) == 140
    # 4096^2 with 1024-pixel tiles, encoder and decoder; a ragged 4096 x 3000 image
    out += [plan_vae_tiles(4096, 4096, 1024, False), plan_vae_tiles(512, 512, 128, True),
            plan_vae_tiles(4096, 3000, 1024, False), plan_vae_tiles(512, 375, 128, True)]
    return out


def test_ownership(plans):
    for plan in plans:
        area = [(x1 - x0) * (y1 - y0) for x0, x1, y0, y1 in plan.in_boxes]
        T = len(area)
        assert tiles_of_ranks(plan, 1) == [list(range(T))]
        for world in range(1, 10):
            owned = tiles_of_ranks(plan, world)
            assert len(owned) == world and owned == tiles_of_ranks(plan, world)
            assert sorted(t for o in owned for t in o) == list(range(T))
            assert all(o == sorted(o) for o in owned)
            load = [sum(area[t] for t in o) for o in owned]
            assert max(load) - min(load) <= max(area)
            if world > T:
                assert sum(1 for o in owned if not o) == world - T


def test_ownership_greedy_order():
    """Largest tile first, ties by tile index, to the least loaded rank, ties to the lowest rank."""
    plan = plan_vae_tiles(4096, 3000, 1024, False)       # ragged: a narrower last column
    area = [(x1 - x0) * (y1 - y0) for x0, x1, y0, y1 in plan.in_boxes]
    assert len(set(area)) > 1
    load, owned = [0, 0, 0], [[], [], []]
    for t in sorted(range(len(area)), key=lambda t: (-area[t], t)):
        r = min(range(3), key=lambda r: (load[r], r))
        load[r] += area[t]
        owned[r].append(t)
    assert tiles_of_ranks(plan, 3) == [sorted(o) for o in owned]
    assert tiles_of_ranks(plan, 3)[0][0] == 0


def test_stop_counts():
    """The GroupNorm counts the sharded driver issues its exchanges by (the GPU tests check them against the walk)."""
    assert VaeWalk.stops(arch.VAE_CFG, False) == 22 and VaeWalk.stops(arch.VAE_CFG, True) == 30


# ---- payloads under gloo, through the default communicator -----------------------------------------------------------
def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    comm, ok = ProcessGroupGather(), []
    n_img = 2
    for plan, nchw, shape in ((plan_vae_tiles(40, 40, 16, True), True, (n_img, 3, 320, 320)),     # 4 tiles
                              (plan_vae_tiles(160, 224, 64, False), False, (n_img, 20, 28, 8))):   # 6 tiles
        owned = tiles_of_ranks(plan, world)
        ents = entries_of_ranks(owned, n_img)
        E = len(plan.in_boxes) * n_img
        g = torch.Generator().manual_seed(E)                    # the same truth on every rank
        truth = torch.randn(E, 32, 2, generator=g, dtype=torch.float64)
        pix = torch.randint(1, 1 << 20, (E,), generator=g)
        # this rank's moments; every other entry holds a stale value the exchange must overwrite
        mom = torch.full((E, 32, 2), float("nan"), dtype=torch.float64)
        mine = torch.tensor(ents[rank], dtype=torch.int64)
        mom[mine] = truth[mine]
        share = max(map(len, ents))
        for _ in range(2):                                      # two stops: the buffer is rewritten each time
            got = unpack_moments(comm.all_gather(pack_moments(mom, mine, pix[mine].double(), share)),
                                 torch.tensor(moment_rows(ents, share)), mom)
            ok.append(torch.equal(mom, truth) and torch.equal(got, pix))
        # output boxes: every element from its owner's copy, signed zeros included
        res_truth = torch.randn(shape, generator=g)
        res_truth[res_truth.abs() < 0.05] = -0.0
        res = torch.full(shape, float("nan"))
        boxes = [[plan.out_boxes[t] for t in tiles] for tiles in owned]
        for x0, x1, y0, y1 in boxes[rank]:
            sl = (slice(None), slice(None), slice(y0, y1), slice(x0, x1)) if nchw else \
                 (slice(None), slice(y0, y1), slice(x0, x1))
            res[sl] = res_truth[sl]
        size = max(box_share(res, b, nchw) for b in boxes)
        unpack_boxes(comm.all_gather(pack_boxes(res, boxes[rank], size, nchw)), res, boxes, nchw, skip=rank)
        ok.append(torch.equal(res, res_truth) and torch.equal(res.signbit(), res_truth.signbit()))
        ok.append(box_share(res, [b for bb in boxes for b in bb], nchw) == res.numel())
    q.put((rank, ok, [len(o) for o in tiles_of_ranks(plan_vae_tiles(40, 40, 16, True), world)]))
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3, 5])
def test_exchange_payloads_under_gloo(world):
    """Through ProcessGroupGather, the GroupNorm payloads reassemble the global moments and pixel counts exactly, and
    the output payloads every box of the result, on every rank; at world 5 one rank owns none of the 4 decoder
    tiles."""
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(all(ok) for _, ok, _ in results), results
    counts = results[0][2]
    assert sum(counts) == 4 and (0 in counts) == (world > 4)
