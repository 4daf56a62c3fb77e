"""`--batch_images N` on the CPU: grouping of the inputs by shape and order, the refusals, the files and prompt.csv rows
in input order, and the per-sample noise source: every sampler family run on a batch with a NoiseSource draws, for
each sample, what the run of that sample alone draws from the global generators after manual_seed(seed + k)."""
import csv
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import inference as cli  # noqa: E402
from diffbir_b200.inference import loop as loop_mod  # noqa: E402
from diffbir_b200.inference.bsr_loop import BSRInferenceLoop  # noqa: E402
from diffbir_b200.sampler import edm as edm_mod  # noqa: E402
from diffbir_b200.sampler.sampler import NoiseSource  # noqa: E402


def args_for(tmp_path, *extra):
    return cli.parse_args(["--input", str(tmp_path / "in"), "--output", str(tmp_path / "out"), *extra])


# ---------------------------------------------------------------------------------------------- grouping
def test_shape_groups_close_on_size_and_on_a_change_of_shape():
    items = [("a", 1), ("b", 1), ("c", 1), ("d", 2), ("e", 2), ("f", 1), ("g", 1), ("h", 1), ("i", 1), ("j", 1)]
    groups = list(loop_mod.shape_groups(items, 3, lambda it: it[1]))
    assert [[n for n, _ in g] for g in groups] == [["a", "b", "c"], ["d", "e"], ["f", "g", "h"], ["i", "j"]]
    assert [[n for n, _ in g] for g in loop_mod.shape_groups(items, 1, lambda it: it[1])] == [[n] for n, _ in items]
    assert list(loop_mod.shape_groups([], 4, lambda it: it)) == []


# ---------------------------------------------------------------------------------------------- refusals
@pytest.mark.parametrize("extra,msg", [
    (["--n_samples", "2"], "n_samples"),
    (["--distribute", "cooperate"], "cooperate"),
    (["--task", "unaligned_face"], "unaligned_face"),
    (["--cleaner_tiled"], "tile"),
    (["--cldm_tiled"], "tile"),
    (["--vae_encoder_tiled", "--vae_encoder_tile_size", "4096"], "VAE tiling"),
    (["--vae_decoder_tiled", "--vae_decoder_tile_size", "4096"], "VAE tiling")])
def test_batch_images_refusals(tmp_path, extra, msg):
    with pytest.raises(NotImplementedError, match=msg):
        loop_mod.check_supported(args_for(tmp_path, "--batch_images", "4", *extra))
    loop_mod.check_supported(args_for(tmp_path, "--batch_images", "1", *extra))    # N = 1: as before
    loop_mod.check_supported(args_for(tmp_path, "--batch_images", "4"))


def test_batch_images_must_be_positive(tmp_path):
    with pytest.raises(ValueError, match="at least 1"):
        loop_mod.check_supported(args_for(tmp_path, "--batch_images", "0"))
    assert args_for(tmp_path).batch_images == 1


# ---------------------------------------------------------------------------------------------- the loop
class StubPipeline:
    def __init__(self):
        self.calls = []

    def run(self, *a, **kw):
        self.calls.append((a, kw))
        lq = a[0]
        return np.stack([np.full(lq.shape[1:], 10 * len(self.calls) + i, dtype=np.uint8) for i in range(lq.shape[0])])


class StubCaptioner:
    def __init__(self):
        self.lists = []

    def caption_list(self, images):
        self.lists.append([im.size for im in images])
        return [f"cap{im.size[0]}x{im.size[1]}" for im in images]


def make_loop(args):
    lp = BSRInferenceLoop.__new__(BSRInferenceLoop)       # skip model loading (needs the GPU library)
    lp.args, lp.loop_ctx, lp.pipeline, lp.captioner = args, {}, StubPipeline(), StubCaptioner()
    return lp


def test_run_batched_groups_seeds_and_writes_in_input_order(tmp_path):
    (tmp_path / "in").mkdir()
    sizes = {"a.png": (6, 8), "b.png": (6, 8), "c.png": (6, 8), "d.png": (6, 8), "e.png": (6, 8), "f.jpg": (5, 7),
             "g.png": (5, 7), "h.png": (6, 8)}
    for name, (h, w) in sizes.items():
        Image.fromarray(np.zeros((h, w, 3), np.uint8)).save(tmp_path / "in" / name)
    (tmp_path / "in" / "notes.txt").write_text("skip me")
    args = args_for(tmp_path, "--batch_images", "4", "--upscale", "2", "--pos_prompt", "p", "--neg_prompt", "n",
                    "--seed", "100")
    lp = make_loop(args)
    lp.run()
    calls = lp.pipeline.calls
    assert [c[0][0].shape for c in calls] == [(4, 12, 16, 3), (1, 12, 16, 3), (2, 10, 14, 3), (1, 12, 16, 3)]
    assert [c[1]["seeds"] for c in calls] == [[100, 101, 102, 103], [104], [105, 106], [107]]
    assert all(len(c[0]) == 26 for c in calls)
    assert calls[0][0][13] == ["cap8x6, p"] * 4 and calls[2][0][13] == ["cap7x5, p"] * 2    # one prompt per image
    assert calls[0][0][14] == "n"
    assert lp.captioner.lists == [[(8, 6)] * 4, [(8, 6)], [(7, 5)] * 2, [(8, 6)]]    # the loaded input, as captioned alone
    out = sorted(p.name for p in (tmp_path / "out").iterdir())
    assert out == ["a.png", "b.png", "c.png", "d.png", "e.png", "f.png", "g.png", "h.png", "prompt.csv"]
    assert np.array(Image.open(tmp_path / "out" / "c.png"))[0, 0, 0] == 12        # call 1, image 2
    assert np.array(Image.open(tmp_path / "out" / "g.png"))[0, 0, 0] == 31        # call 3, image 1
    rows = list(csv.reader(open(tmp_path / "out" / "prompt.csv")))
    assert rows[0] == ["file_name", "pos_prompt", "neg_prompt"]
    assert [r[0] for r in rows[1:]] == ["a", "b", "c", "d", "e", "f", "g", "h"]
    assert rows[6] == ["f", "cap7x5, p", "n"]


def test_run_batched_under_images_mode_groups_the_rank_s_images(tmp_path):
    from diffbir_b200.inference.ranks import Ranks
    (tmp_path / "in").mkdir()
    for i in range(7):
        Image.fromarray(np.zeros((6, 8, 3), np.uint8)).save(tmp_path / "in" / f"{i}.png")
    args = args_for(tmp_path, "--batch_images", "2", "--upscale", "1", "--seed", "5")
    lp = make_loop(args)
    seeded = []
    lp.ranks = Ranks("images", 1, 3, args.seed, seeded.append)
    lp.ranks.finish = lambda save_dir: None                          # the gather to rank 0 needs a process group
    lp.run()
    assert [c[1]["seeds"] for c in lp.pipeline.calls] == [[6, 9]]      # images 1 and 4 of 7 on rank 1 of 3
    assert sorted(p.name for p in (tmp_path / "out").iterdir()) == ["1.png", "4.png"]
    assert [k for k, _ in lp.ranks.rows] == [1, 4]


# ---------------------------------------------------------------------------------------------- noise source
BETAS = np.linspace(1e-4, 2e-2, 1000)


def toy_model(x, t, cond):
    """Elementwise in the sample (no mixing across the batch), so a sample's output is its own."""
    return 0.3 * x + 0.05 * cond["c_img"] + 1e-4 * t.float().view(-1, 1, 1, 1)


def make_sampler(name):
    from diffbir_b200.sampler import DDIMSampler, DPMSolverSampler, EDMSampler, SpacedSampler
    if name == "spaced":
        return SpacedSampler(BETAS, "eps", False)
    if name == "ddim":
        return DDIMSampler(BETAS, "v", True, eta=0)
    if name.startswith("dpm"):
        return DPMSolverSampler(BETAS, "v", False, name)
    return EDMSampler(BETAS, "eps", False, name, s_churn=0.5, s_tmin=0.0, s_tmax=300.0, s_noise=1.0, eta=1.0, order=2)


SAMPLERS = ["spaced", "ddim", "dpm++_m2", "edm_euler", "edm_euler_a", "edm_heun", "edm_dpm_2", "edm_dpm_2_a", "edm_lms",
            "edm_dpm++_2s_a", "edm_dpm++_sde", "edm_dpm++_2m", "edm_dpm++_2m_sde", "edm_dpm++_3m_sde"]


class CpuTree:
    """DeviceBrownianTree's interface on the CPU: a function of (seed, t0, t1) per sample, one tree per seed when
    given a list. Records every seed it is built with."""
    seeds = []

    def __init__(self, x, lo, hi, seed):
        self.shape = (1, *x.shape[1:])
        self.list = seed if isinstance(seed, list) else [seed] * x.shape[0]
        CpuTree.seeds.append(seed)

    def __call__(self, t0, t1):
        def one(s):
            g = torch.Generator().manual_seed((s ^ int(float(t0) * 1e6) ^ (int(float(t1) * 1e6) << 20)) % 2 ** 62)
            return torch.randn(self.shape, generator=g)
        return torch.cat([one(s) for s in self.list])


class RecordingSource(NoiseSource):
    """NoiseSource that records the order of its draws."""

    def __init__(self, seeds, device):
        super().__init__(seeds, device)
        self.log = []

    def randn(self, shape):
        self.log.append(("randn", tuple(shape)))
        return super().randn(shape)

    def randint_seeds(self):
        self.log.append(("randint",))
        return super().randint_seeds()


def run_sampler(name, cond, uncond, batch, source=None):
    sampler = make_sampler(name)
    sampler.noise_source = source
    return sampler.sample(toy_model, "cpu", 5, (batch, 4, 8, 8), cond, uncond, 3.0)


@pytest.mark.parametrize("name", SAMPLERS)
def test_noise_source_draws_each_sample_s_single_run_stream(name, monkeypatch):
    monkeypatch.setattr(edm_mod, "DeviceBrownianTree", CpuTree)
    CpuTree.seeds = []
    B, seeds = 3, [40, 41, 42]
    g = torch.Generator().manual_seed(0)
    c_img = torch.randn(B, 4, 8, 8, generator=g)
    cond = dict(c_txt=torch.zeros(B, 77, 8), c_img=c_img)
    uncond = dict(c_txt=torch.ones(B, 77, 8), c_img=c_img)
    src = RecordingSource(seeds, "cpu")
    got = run_sampler(name, cond, uncond, B, src)
    batch_tree_seeds = list(CpuTree.seeds)
    single_tree_seeds = []
    for k, s in enumerate(seeds):
        torch.manual_seed(s)
        one = {key: v[k:k + 1] for key, v in cond.items()}
        un = {key: v[k:k + 1] for key, v in uncond.items()}
        CpuTree.seeds = []
        want = run_sampler(name, one, un, 1)
        single_tree_seeds += CpuTree.seeds
        assert torch.equal(got[k:k + 1], want), f"{name}: sample {k}"
    # the draw order the stub recorded: x_T first, then the rule's draws (per step or none), a Brownian seed up front
    assert src.log[0] == ("randn", (B, 4, 8, 8))
    brownian = name == "edm_dpm++_sde" or (name in ("edm_dpm++_2m_sde", "edm_dpm++_3m_sde") and
                                           _has_torchsde())
    assert (("randint",) in src.log) == brownian
    if brownian:
        assert src.log[1] == ("randint",) and batch_tree_seeds == [single_tree_seeds]
    per_step = name in ("spaced", "ddim", "edm_euler", "edm_heun", "edm_dpm_2", "edm_euler_a", "edm_dpm_2_a",
                        "edm_dpm++_2s_a") or (name in ("edm_dpm++_2m_sde", "edm_dpm++_3m_sde") and not brownian)
    assert (len([e for e in src.log if e[0] == "randn"]) > 1) == per_step


def _has_torchsde():
    try:
        import torchsde  # noqa: F401
        return True
    except ImportError:
        return False


def test_noise_source_rows_are_the_global_stream_of_each_seed():
    src = NoiseSource([7, 8], "cpu")
    x = src.randn((2, 3, 4))
    seeds = src.randint_seeds()
    for k, s in enumerate((7, 8)):
        torch.manual_seed(s)
        assert torch.equal(x[k:k + 1], torch.randn(1, 3, 4))
        assert seeds[k] == torch.randint(0, 2 ** 63 - 1, []).item()
    with pytest.raises(ValueError, match="2 seeds"):
        src.randn((3, 4))
