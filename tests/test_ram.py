"""CPU: RAM++ captioner (`--captioner ram`): the fp32 oracle against the reference fixture, the strict checkpoint
loader, the tag-list / threshold files, the CLI's acceptance of `ram`, and the prompt assembly."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import inference as cli  # noqa: E402
from diffbir_b200 import arch  # noqa: E402
from diffbir_b200.inference import loop as loop_mod  # noqa: E402
from diffbir_b200.utils import caption as cap  # noqa: E402
from diffbir_b200.utils.synth import make_state_dict, synthetic_ram  # noqa: E402


def fixture_sd(f):
    """The fixture's weights: seeded synthetic RAM++ with fc rescaled (tests/golden/gen_golden_ram.py)."""
    sd = make_state_dict(arch.ram_shapes(arch.RAM_CFG), int(f["seed"]))
    sd["fc.weight"] = sd["fc.weight"] * float(f["fc_scale"])
    sd["fc.bias"] = torch.full((1,), float(f["fc_bias"]))
    return sd


def fixture_image(f):
    x = torch.rand(1, 3, 384, 384, generator=torch.Generator().manual_seed(int(f["image_seed"])))
    assert abs(float(x.double().sum()) - float(f["x_sum"])) < 1e-6 * float(f["x_sum"])
    return x


@pytest.fixture(scope="module")
def ram_fixture(golden_dir):
    return dict(np.load(golden_dir / "ram_small.npz"))


@torch.no_grad()
def test_oracle_reproduces_reference_fixture(ram_fixture):
    from oracle import ram as oram
    f = ram_fixture
    sd = arch.ram_state_dict(fixture_sd(f))
    stages = []
    emb, logits = oram.ram_forward(sd, oram.normalize(fixture_image(f)), stages)
    step = int(f["stage_row_step"])
    for i, s in enumerate(stages):
        ref = torch.from_numpy(f[f"stage{i}"])
        assert (s[0, ::step] - ref).abs().max() <= 2e-5 * ref.abs().max(), i
    ref_emb, ref_logits = torch.from_numpy(f["image_embeds"]), torch.from_numpy(f["logits"])
    assert (emb[0] - ref_emb).abs().max() <= 2e-5 * ref_emb.abs().max()
    assert (logits[0] - ref_logits).abs().max() <= 2e-5 * ref_logits.abs().max()
    thr = torch.from_numpy(f["thresholds"])
    decisions = torch.sigmoid(logits[0]) > thr
    assert torch.equal(decisions, torch.from_numpy(f["decisions"]))
    assert 5 <= int(decisions.sum()) <= 50 and float(f["min_margin"]) > 0.01
    names = dict(zip(f["fired"].tolist(), f["fired_tags"].tolist()))
    tags = [names.get(i, f"unfired{i}") for i in range(len(thr))]
    assert cap.decide(logits[0], thr, tags) == str(f["caption"])


def test_loader_is_strict():
    sd, _, _ = synthetic_ram(5)
    ckpt = {"model": dict(sd)}
    ckpt["model"]["visual_encoder.layers.0.blocks.0.attn.relative_position_index"] = torch.zeros(144, 144)
    ckpt["model"]["visual_encoder.layers.0.blocks.1.attn_mask"] = torch.zeros(64, 144, 144)
    out = arch.ram_state_dict(ckpt)
    assert set(out) == set(arch.ram_shapes(arch.RAM_CFG))
    missing = dict(sd)
    del missing["tagging_head.encoder.layer.1.output.LayerNorm.bias"]
    with pytest.raises(KeyError, match="output.LayerNorm.bias"):
        arch.ram_state_dict(missing)
    wrong = dict(sd)
    wrong["wordvec_proj.weight"] = torch.zeros(768, 256)
    with pytest.raises(ValueError, match="wordvec_proj.weight"):
        arch.ram_state_dict(wrong)
    small_table = dict(sd)
    small_table["visual_encoder.layers.2.blocks.3.attn.relative_position_bias_table"] = torch.zeros(15 * 15, 24)
    with pytest.raises(ValueError, match="225 rows"):
        arch.ram_state_dict(small_table)


def test_tag_files(tmp_path):
    with pytest.raises(FileNotFoundError) as e:
        cap.read_tag_files(str(tmp_path), 3)
    assert cap.TAG_LIST in str(e.value) and cap.THRESHOLDS in str(e.value)
    (tmp_path / cap.TAG_LIST).write_text("3D CG rendering\nabacus\nzebra", encoding="utf-8")
    with pytest.raises(FileNotFoundError, match=cap.THRESHOLDS):
        cap.read_tag_files(str(tmp_path), 3)
    (tmp_path / cap.THRESHOLDS).write_text("0.65\n0.7\n0.9\n", encoding="utf-8")
    tags, thr = cap.read_tag_files(str(tmp_path), 3)
    assert tags == ["3D CG rendering", "abacus", "zebra"] and thr == [0.65, 0.7, 0.9]
    with pytest.raises(ValueError, match="expected 4"):
        cap.read_tag_files(str(tmp_path), 4)
    logits = torch.tensor([2.0, 0.5, 2.0])              # sigmoid: 0.88, 0.62, 0.88
    assert cap.decide(logits, torch.tensor(thr), tags) == "3D CG rendering"
    assert cap.decide(torch.full((3,), -5.0), torch.tensor(thr), tags) == ""


def test_cli_accepts_ram_and_refuses_llava(tmp_path):
    args = lambda *x: cli.parse_args(["--input", str(tmp_path / "in"), "--output", str(tmp_path / "out"), *x])  # noqa: E731
    loop_mod.check_supported(args("--captioner", "ram"))
    with pytest.raises(NotImplementedError, match="captioner"):
        loop_mod.check_supported(args("--captioner", "llava"))


def test_prompt_assembly():
    assert loop_mod.prompt_with_caption("cat, forest", "Cinematic, 4k") == "cat, forest, Cinematic, 4k"
    assert loop_mod.prompt_with_caption("", "Cinematic, 4k") == "Cinematic, 4k"
    assert loop_mod.prompt_with_caption("cat", "") == "cat"
    assert loop_mod.prompt_with_caption("", "") == ""
    assert cap.EmptyCaptioner("cuda")(None) == ""


def test_preprocess_matches_the_reference_transform():
    from PIL import Image
    rng = np.random.default_rng(0)
    img = Image.fromarray(rng.integers(0, 256, (200, 300, 3), dtype=np.uint8))
    x = cap.preprocess(img)
    ref = np.asarray(img.resize((384, 384), Image.BILINEAR), dtype=np.float32) / 255.0
    assert x.shape == (1, 3, 384, 384) and np.array_equal(x[0].permute(1, 2, 0).numpy(), ref)


def test_reference_names_are_aliased():
    from diffbir.utils.caption import EmptyCaptioner, LLaVACaptioner, RAMCaptioner
    assert RAMCaptioner is cap.RAMCaptioner and EmptyCaptioner is cap.EmptyCaptioner
    with pytest.raises(NotImplementedError):
        LLaVACaptioner("cuda", "4")
