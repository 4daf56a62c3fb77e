"""-m gpu: `torchrun ... inference.py --synthetic` in both --distribute modes (full SD-2.1 config, random-init weights).
On one GPU the files must be bit-identical to direct Pipeline.run calls seeded as the mode defines (images: seed + k
before image k; cooperate: the single-process run, seeded once) with the batch-invariant plans torchrun pins. With
two or more GPUs, world size 2 must write the files of world size 1 in both modes."""
import os
import signal
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

pytestmark = pytest.mark.gpu
PORT = 29547
SIZES = {"a.png": (128, 128), "b.png": (96, 160), "c.png": (144, 128)}        # LQ (h, w); x4 by the v2.1 recipe
TILED = {"t.png": (160, 192)}                                                 # 640 x 768: 6 latent tiles of 64
BASE = ["--task", "sr", "--version", "v2.1", "--upscale", "4", "--sampler", "spaced", "--steps", "2", "--cfg_scale", "4.0",
        "--captioner", "none", "--pos_prompt", "a photo", "--neg_prompt", "low quality, blurry", "--synthetic"]
TILED_FLAGS = ["--cldm_tiled", "--cleaner_tiled", "--cleaner_tile_size", "512", "--cleaner_tile_stride", "256"]


def make_inputs(d: Path, sizes) -> Path:
    from diffbir_b200.utils.synth import synthetic_lq
    d.mkdir(parents=True, exist_ok=True)
    for i, (name, (h, w)) in enumerate(sizes.items()):
        Image.fromarray(synthetic_lq(h, w, seed=10 + i)[0]).save(d / name)
    return d


def torchrun(nproc: int, inp: Path, out: Path, mode: str, extra=()) -> None:
    """One torchrun of inference.py; its whole process group is gone when this returns."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}",
           "--master-addr", "127.0.0.1", "--master-port", str(PORT), str(ROOT / "inference.py"), *BASE, *extra,
           "--distribute", mode, "--input", str(inp), "--output", str(out)]
    p = subprocess.Popen(cmd, cwd=str(ROOT), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                         start_new_session=True)
    try:
        log, _ = p.communicate(timeout=900)
    finally:
        if p.poll() is None:
            os.killpg(p.pid, signal.SIGKILL)
            p.wait()
    print(log[-3000:])
    assert p.returncode == 0, log[-3000:]


def files(d: Path) -> dict:
    return {p.name: p.read_bytes() for p in sorted(d.iterdir())}


@pytest.fixture(scope="module")
def reference_loop():
    """The CLI's loop built in this process with the plans torchrun pins (DBIR_DETERMINISTIC=1)."""
    import inference as cli
    from diffbir_b200.inference import BSRInferenceLoop
    old = os.environ.get("DBIR_DETERMINISTIC")
    os.environ["DBIR_DETERMINISTIC"] = "1"
    try:
        loop = BSRInferenceLoop(cli.parse_args(BASE + ["--input", "-", "--output", "-"]))
        loop.pipeline.cldm._build()
    finally:
        if old is None:
            del os.environ["DBIR_DETERMINISTIC"]
        else:
            os.environ["DBIR_DETERMINISTIC"] = old
    assert loop.pipeline.cldm.engine.deterministic
    return loop


def run_single(loop, inp: Path, out: Path, extra=()) -> None:
    """The plain single-process CLI run (seeded once) on the reference loop."""
    import inference as cli
    loop.args = cli.parse_args(BASE + list(extra) + ["--input", str(inp), "--output", str(out)])
    cli.set_seed(loop.args.seed)
    loop.run()


@pytest.mark.parametrize("tiled", [False, True])
def test_one_rank_images_mode_is_seeded_per_image(tmp_path, reference_loop, tiled):
    """tiled: the tiling flags on every input; t.png (k = 3) samples over 6 latent tiles and cleans over 4 windows."""
    import inference as cli
    sizes = dict(SIZES, **TILED) if tiled else SIZES
    extra = TILED_FLAGS if tiled else []
    inp = make_inputs(tmp_path / "in", sizes)
    torchrun(1, inp, tmp_path / "out", "images", extra)
    a = cli.parse_args(BASE + extra + ["--input", str(inp), "--output", "-"])
    lp = reference_loop
    for k, name in enumerate(sorted(sizes)):
        cli.set_seed(a.seed + k)
        lq = lp.after_load_lq(Image.open(inp / name).convert("RGB"))
        want = lp.pipeline.run(
            lq[None], a.steps, a.strength, a.cleaner_tiled, a.cleaner_tile_size, a.cleaner_tile_stride, a.vae_encoder_tiled,
            a.vae_encoder_tile_size, a.vae_decoder_tiled, a.vae_decoder_tile_size, a.cldm_tiled, a.cldm_tile_size,
            a.cldm_tile_stride, a.pos_prompt, a.neg_prompt, a.cfg_scale, a.start_point_type, a.sampler, a.noise_aug,
            a.rescale_cfg, a.s_churn, a.s_tmin, a.s_tmax, a.s_noise, a.eta, a.order)[0]
        got = np.array(Image.open(tmp_path / "out" / name))
        assert got.shape == want.shape and want.std() > 1.0
        assert np.array_equal(got, want), f"{name}: {(got != want).mean():.2%} of the values differ"
    # prompt.csv: the single-process rows (the prompts do not depend on the seed)
    run_single(lp, inp, tmp_path / "single", extra)
    assert files(tmp_path / "out")["prompt.csv"] == files(tmp_path / "single")["prompt.csv"]


@pytest.mark.parametrize("tiled", [False, True])
def test_one_rank_cooperate_mode_is_the_single_process_run(tmp_path, reference_loop, tiled):
    inp = make_inputs(tmp_path / "in", TILED if tiled else SIZES)
    extra = TILED_FLAGS if tiled else []
    torchrun(1, inp, tmp_path / "out", "cooperate", extra)
    run_single(reference_loop, inp, tmp_path / "single", extra)
    got, want = files(tmp_path / "out"), files(tmp_path / "single")
    assert sorted(got) == sorted(want) and len(want) == len(TILED if tiled else SIZES) + 1     # PNGs + prompt.csv
    assert got == want


@pytest.mark.parametrize("mode", ["images", "cooperate"])
def test_two_ranks_write_the_files_of_one(tmp_path, mode):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    inp = make_inputs(tmp_path / "in", dict(SIZES, **TILED))
    for extra in ([], TILED_FLAGS):
        tag = "tiled" if extra else "plain"
        torchrun(1, inp, tmp_path / f"w1_{tag}", mode, extra)
        torchrun(2, inp, tmp_path / f"w2_{tag}", mode, extra)
        assert files(tmp_path / f"w2_{tag}") == files(tmp_path / f"w1_{tag}")
