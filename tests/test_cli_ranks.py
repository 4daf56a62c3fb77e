"""CPU, gloo: inference.py's torchrun modes (diffbir_b200/inference/ranks.py) on stub pipelines and captioners, at
world sizes 1, 2 and 3. `images` deals the sorted inputs round-robin and seeds image k with seed + k; `cooperate`
runs every image on every rank with rank 0's prompt and lets rank 0 alone write. prompt.csv is the single-process
file byte for byte. The tiled cleaner sharded over the ranks is the un-sharded one bit for bit (oracle SwinIR)."""
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from PIL import Image

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import inference as cli  # noqa: E402
from diffbir_b200.inference import ranks as rank_mod  # noqa: E402
from diffbir_b200.inference.bsr_loop import BSRInferenceLoop  # noqa: E402

SEED = 231
SIZES = {"a.png": (6, 8), "b.jpg": (5, 7), "c.png": (4, 4), "d.jpeg": (7, 5), "e.png": (3, 9)}   # sorted: a..e


class DrawPipeline:
    """Returns images filled from torch.rand draws, so the files record the RNG state of each call."""

    def __init__(self):
        self.calls = []

    def run(self, *a):
        lq = a[0]
        draw = torch.rand(lq.shape[0])
        self.calls.append((lq.shape, a[13], draw))
        return np.stack([np.full(lq.shape[1:], int(255 * v), dtype=np.uint8) for v in draw])


class SizeCaptioner:
    """A caption that depends on the image and, to show whose caption is used, on the rank that computes it."""

    def __init__(self, tag):
        self.tag = tag

    def __call__(self, img):
        return f"{self.tag} {img.size[0]}x{img.size[1]}, with \"quotes\""


class RecordingLoop(BSRInferenceLoop):
    def save(self, samples, pos_prompt, neg_prompt):
        self.saved.append(self.loop_ctx["file_stem"])
        super().save(samples, pos_prompt, neg_prompt)


def make_loop(tmp, out, mode=None, rank=0, world=1):
    args = cli.parse_args(["--input", str(tmp / "in"), "--output", str(tmp / out), "--upscale", "1", "--n_samples", "3",
                           "--batch_size", "2", "--pos_prompt", "p", "--neg_prompt", "n, m", "--seed", str(SEED)]
                          + (["--distribute", mode] if mode else []))
    lp = RecordingLoop.__new__(RecordingLoop)           # skip model loading (needs the GPU library)
    lp.args, lp.loop_ctx, lp.pipeline, lp.saved = args, {}, DrawPipeline(), []
    lp.captioner = SizeCaptioner("cap" if mode != "cooperate" or rank == 0 else f"rank{rank}")
    if mode is not None:
        lp.ranks = rank_mod.Ranks(mode, rank, world, SEED, cli.set_seed)
    return lp


def make_inputs(tmp):
    (tmp / "in").mkdir(exist_ok=True)
    for name, (h, w) in SIZES.items():
        Image.fromarray(np.zeros((h, w, 3), np.uint8)).save(tmp / "in" / name)
    (tmp / "in" / "notes.txt").write_text("not an image")


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _tiled_cleaner_check():
    """make_tiled_fn(shard=True) over the group vs the same call un-sharded, on the oracle SwinIR."""
    from diffbir_b200 import arch
    from diffbir_b200.utils.common import make_tiled_fn
    from diffbir_b200.utils.synth import make_state_dict
    from oracle.swinir import swinir_forward
    cfg = dict(arch.SWINIR_CFG, embed_dim=24, depths=(1,), num_heads=(2,))
    sd = make_state_dict(arch.swinir_shapes(cfg), 4)

    def cleaner(x):
        return swinir_forward(sd, x, heads=2)

    x = torch.rand(1, 3, 96, 160, generator=torch.Generator().manual_seed(2))    # 3 x 5 windows of 64, stride 24
    sharded = make_tiled_fn(cleaner, 64, 24, shard=True)(x)
    return bool(torch.equal(sharded, make_tiled_fn(cleaner, 64, 24)(x)))


def _worker(rank, world, port, tmp, q):
    torch.set_num_threads(1)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res = {"rank": rank}
        for mode in ("images", "cooperate"):
            lp = make_loop(tmp, f"{mode}_{world}", mode, rank, world)
            cli.set_seed(SEED)
            lp.run()
            res[mode] = dict(calls=[(shape, prompt, draw.tolist()) for shape, prompt, draw in lp.pipeline.calls],
                             saved=list(lp.saved))
        res["cleaner"] = _tiled_cleaner_check()
        q.put(res)
    finally:
        dist.destroy_process_group()


def _run_world(world, tmp):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, tmp, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = [q.get(timeout=300) for _ in procs]
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    return sorted(results, key=lambda r: r["rank"])


def _files(d):
    return {p.name: p.read_bytes() for p in sorted(Path(d).iterdir())}


@pytest.mark.parametrize("world", [1, 2, 3])
def test_torchrun_modes_match_the_single_process_run(tmp_path, world):
    make_inputs(tmp_path)
    single = make_loop(tmp_path, "single")
    cli.set_seed(SEED)
    single.run()
    ref = _files(tmp_path / "single")
    results = _run_world(world, tmp_path)
    stems = sorted(os.path.splitext(n)[0] for n in SIZES)

    # images: rank r restores images r, r + W, ... once each, and image k is drawn from set_seed(SEED + k)
    for r, res in enumerate(results):
        assert res["images"]["saved"] == stems[r::world]
        want = []
        for k in range(r, len(stems), world):
            cli.set_seed(SEED + k)
            want += [torch.rand(2).tolist(), torch.rand(1).tolist()]          # n_samples 3 in batches of 2 + 1
        assert [c[2] for c in res["images"]["calls"]] == want
    out = _files(tmp_path / f"images_{world}")
    assert sorted(out) == sorted(ref)
    assert out["prompt.csv"] == ref["prompt.csv"]
    assert out["a_0.png"] == ref["a_0.png"]                                   # image 0: seed + 0 = the single run's seed

    # cooperate: every rank runs every image with rank 0's prompt and the single run's RNG; only rank 0 writes
    for r, res in enumerate(results):
        calls = res["cooperate"]["calls"]
        assert [c[1] for c in calls] == [c[1] for c in single.pipeline.calls]
        assert all(c[1].startswith("cap ") for c in calls)                   # rank 0's caption
        assert [c[2] for c in calls] == [c[2].tolist() for c in single.pipeline.calls]
        assert res["cooperate"]["saved"] == (stems if r == 0 else [])
    assert _files(tmp_path / f"cooperate_{world}") == ref

    assert all(res["cleaner"] for res in results)


class CountingCleaner:
    """CPU stand-in for a stage-1 network: a fixed per-pixel map, with a count of the calls."""

    def __init__(self):
        self.calls = 0

    def __call__(self, x):
        self.calls += 1
        return torch.tanh(3 * x - 1) * 0.5 + 0.25 * x.flip(1)


def _stage1_worker(rank, world, port, q):
    torch.set_num_threads(1)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from diffbir_b200.pipeline import SwinIRPipeline
        lq = torch.rand(1, 3, 96, 160, generator=torch.Generator().manual_seed(4))
        res = {"rank": rank}
        for name, tiled in (("untiled", False), ("tiled", True)):
            shared = SwinIRPipeline(CountingCleaner(), None, None, None, "cpu")
            shared.shard_cleaner = True
            alone = SwinIRPipeline(CountingCleaner(), None, None, None, "cpu")      # the single-rank stage 1
            got = shared.shared_cleaner(lq, tiled, 64, 32)
            want = alone.shared_cleaner(lq, tiled, 64, 32)
            res[name] = (bool(torch.equal(got, want)), tuple(got.shape), shared.cleaner.calls, alone.cleaner.calls)
        q.put(res)
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_shared_stage1_matches_one_rank(world):
    """Pipeline.shared_cleaner across ranks: un-tiled, rank 0 alone runs the cleaner and broadcasts it; tiled, the
    2 x 4 windows are split round-robin. Either way every rank holds the single-rank output bit for bit."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_stage1_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        results = sorted([q.get(timeout=300) for _ in procs], key=lambda r: r["rank"])
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    for r, res in enumerate(results):
        same, shape, calls, alone_calls = res["untiled"]
        assert same and shape == (1, 3, 512, 853)             # short edge resized to 512 before the cleaner
        assert (calls, alone_calls) == ((1 if r == 0 else 0), 1)
        same, shape, calls, alone_calls = res["tiled"]
        assert same and shape == (1, 3, 512, 853)
        assert alone_calls == 8 and calls == len(range(r, 8, world))


def test_no_torchrun_variables_no_torch_distributed(tmp_path, monkeypatch):
    """Without WORLD_SIZE / RANK / LOCAL_RANK the CLI opens no process group and the loop makes no collective call."""
    for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK"):
        monkeypatch.delenv(k, raising=False)

    def refuse(*a, **k):
        raise AssertionError("torch.distributed was used")

    for name in ("init_process_group", "destroy_process_group", "is_initialized", "get_rank", "get_world_size",
                 "broadcast", "broadcast_object_list", "all_gather", "all_gather_object"):
        monkeypatch.setattr(dist, name, refuse)
    assert rank_mod.torchrun_env({"RANK": "0", "LOCAL_RANK": "0"}) is None
    assert rank_mod.torchrun_env({"RANK": "1", "LOCAL_RANK": "1", "WORLD_SIZE": "2"}) == (1, 1, 2)
    args = cli.parse_args(["--input", "x", "--output", "y", "--distribute", "cooperate"])
    assert rank_mod.launch(args, cli.set_seed) is None
    make_inputs(tmp_path)
    lp = make_loop(tmp_path, "out")
    assert lp.ranks is None
    lp.run()
    assert sorted(p.name for p in (tmp_path / "out").iterdir())[-1] == "prompt.csv"


def test_distribute_flag_and_refusal(tmp_path, monkeypatch):
    assert cli.parse_args(["--input", "x", "--output", "y"]).distribute == "images"
    with pytest.raises(SystemExit):
        cli.parse_args(["--input", "x", "--output", "y", "--distribute", "tiles"])
    monkeypatch.setenv("WORLD_SIZE", "2")
    monkeypatch.setenv("RANK", "0")
    monkeypatch.setenv("LOCAL_RANK", "0")
    args = cli.parse_args(["--input", "x", "--output", "y", "--task", "unaligned_face", "--distribute", "cooperate"])
    with pytest.raises(NotImplementedError, match="--distribute images"):
        rank_mod.launch(args, cli.set_seed)
