"""CPU: LLaVA captioner (`--captioner llava --llava_bit 16`): the fp32 oracle against the reference fixture, the image
preprocessing, the prompt chunks and the -200 splice, the byte stand-in tokenizer, the registry directories, the
strict loader and its refusals, and the CLI's acceptance of --llava_bit 16 only."""
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import inference as cli  # noqa: E402
from diffbir_b200 import arch  # noqa: E402
from diffbir_b200.inference import loop as loop_mod  # noqa: E402
from diffbir_b200.inference.pretrained_models import resolve  # noqa: E402
from diffbir_b200.utils import caption as cap  # noqa: E402
from diffbir_b200.utils.synth import make_state_dict, synthetic_lq  # noqa: E402


def fixture_cfg(f) -> dict:
    return json.loads(str(f["cfg"]))


def fixture_sd(f):
    """The fixture's weights: seeded synthetic LLaVA with lm_head rescaled (tests/golden/gen_golden_llava.py)."""
    sd = make_state_dict(arch.llava_shapes(fixture_cfg(f)), int(f["seed"]))
    sd["lm_head.weight"] = sd["lm_head.weight"] * float(f["lm_head_scale"])
    return sd


def fixture_image(f) -> Image.Image:
    return Image.fromarray(synthetic_lq(200, 300, seed=int(f["image_seed"]))[0])


def fixture_pixels(f) -> torch.Tensor:
    """preprocess_llava of the fixture image (in [0, 1]); checked against the reference's pixel values."""
    x = cap.preprocess_llava(fixture_image(f))
    pv = cap.clip_normalize(x)
    step = int(f["pixel_row_step"])
    assert (pv[0, :, ::step] - torch.from_numpy(f["pixel_rows"])).abs().max() <= 1e-6
    assert abs(float(pv.double().sum()) - float(f["pixel_sum"])) <= 1e-6 * pv.numel()
    return x


@pytest.fixture(scope="module")
def llava_fixture(golden_dir):
    return dict(np.load(golden_dir / "llava_small.npz"))


def test_preprocessing_matches_the_reference(llava_fixture):
    x = fixture_pixels(llava_fixture)
    assert x.shape == (1, 3, 336, 336) and x.dtype == torch.float32
    # padding: a 300 x 200 image is padded top and bottom with (122, 116, 104)
    img = cap.expand2square(Image.new("RGB", (300, 200), (0, 0, 0)))
    assert img.size == (300, 300) and img.getpixel((0, 0)) == cap.CLIP_BACKGROUND and img.getpixel((0, 50)) == (0, 0, 0)
    assert img.getpixel((0, 249)) == (0, 0, 0) and img.getpixel((0, 250)) == cap.CLIP_BACKGROUND


@torch.no_grad()
def test_oracle_reproduces_reference_fixture(llava_fixture):
    from oracle import llava as olv
    f = llava_fixture
    cfg = fixture_cfg(f)
    sd = arch.llava_state_dict(fixture_sd(f), None, cfg)
    pv = cap.clip_normalize(fixture_pixels(f))
    ids = f["input_ids"].tolist()
    toks, logits, feats = olv.greedy(sd, cfg, pv, ids, len(f["tokens"]))
    ref_feats = torch.from_numpy(f["feature_rows"])
    assert (feats[::int(f["feature_row_step"])] - ref_feats).abs().max() <= 2e-5 * ref_feats.abs().max()
    ref = torch.from_numpy(f["forced_logits"])
    assert (logits - ref).abs().max() <= 2e-5 * ref.abs().max()
    assert toks == f["tokens"].tolist()
    assert torch.equal(logits[0], logits[0]) and (logits[0] - torch.from_numpy(f["prefill_logits"])).abs().max() <= \
        2e-5 * ref.abs().max()


def test_prompt_ids_and_image_splice(llava_fixture):
    """The byte stand-in's prompt ids equal the reference tokenizer_image_token's over the same byte tokenizer."""
    ids = cap.llava_prompt_ids(cap.ByteTokenizer())
    assert ids == llava_fixture["input_ids"].tolist()
    assert ids.count(-200) == 1 and ids[0] == 1 and ids.count(1) == 1
    pre, post = cap.LLAVA_PROMPT.split(cap.IMAGE_TOKEN)
    assert pre.endswith("USER: ") and post.startswith("\n" + cap.LLAVA_QUESTION) and post.endswith(" ASSISTANT:")
    # tokenizer_image_token: BOS kept once, -200 between chunks; no BOS -> nothing dropped
    assert cap.splice_image_token([[1, 5, 6], [1, 7], [1, 8]], 1) == [1, 5, 6, -200, 7, -200, 8]
    assert cap.splice_image_token([[5, 6], [7]], 1) == [5, 6, -200, 7]
    assert cap.splice_image_token([[1], [1, 9]], 1) == [1, -200, 9]


def test_byte_tokenizer_round_trip():
    t = cap.ByteTokenizer()
    text = "A photo of a café, 2 cats\n"
    ids = t.encode(text)
    assert ids[0] == t.bos and all(3 <= i < 259 for i in ids[1:]) and ids[1] == 3 + ord("A")
    assert t.decode(ids + [t.eos]) == text
    assert t.decode([t.bos, 3 + ord("x"), 400, 3 + ord("y"), t.eos]) == "x w400y"


def test_registry_directories(tmp_path):
    with pytest.raises(FileNotFoundError, match="llava-v1.5-7b"):
        resolve("llava_v1.5_7b", str(tmp_path))
    with pytest.raises(FileNotFoundError, match="clip-vit-large-patch14-336"):
        resolve("clip_vit_l14_336", str(tmp_path))
    (tmp_path / "llava-v1.5-7b").write_bytes(b"x")            # a file where the directory should be
    with pytest.raises(FileNotFoundError, match="llava-v1.5-7b"):
        resolve("llava_v1.5_7b", str(tmp_path))
    (tmp_path / "clip-vit-large-patch14-336").mkdir()
    assert resolve("clip_vit_l14_336", str(tmp_path)).endswith("clip-vit-large-patch14-336")
    (tmp_path / "v2.pth").mkdir()                              # file keys still need a file
    with pytest.raises(FileNotFoundError, match="v2.pth"):
        resolve("v2", str(tmp_path))


V15 = dict(vocab_size=32000, hidden_size=4096, intermediate_size=11008, num_attention_heads=32, num_hidden_layers=32,
           num_key_value_heads=32, rms_norm_eps=1e-5, rope_scaling=None, mm_projector_type="mlp2x_gelu",
           image_aspect_ratio="pad", mm_vision_select_layer=-2, mm_vision_select_feature="patch",
           mm_use_im_start_end=False, mm_hidden_size=1024, bos_token_id=1, eos_token_id=2)


def test_config_refuses_other_settings():
    cfg = arch.llava_config(V15)
    assert {k: cfg[k] for k in arch.LLAVA_CFG} == arch.LLAVA_CFG
    for key, value in (("mm_projector_type", "linear"), ("image_aspect_ratio", "anyres"),
                       ("mm_vision_select_layer", -1), ("mm_vision_select_feature", "cls_patch"),
                       ("mm_use_im_start_end", True), ("num_key_value_heads", 8),
                       ("rope_scaling", {"type": "linear", "factor": 2.0})):
        with pytest.raises(NotImplementedError, match=key):
            arch.llava_config(dict(V15, **{key: value}))
    with pytest.raises(NotImplementedError, match="quick_gelu"):
        arch.llava_config(V15, {"vision_config": dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16,
                                                      intermediate_size=4096, hidden_act="gelu")})


def test_loader_is_strict(llava_fixture):
    cfg = fixture_cfg(llava_fixture)
    sd = make_state_dict(arch.llava_shapes(cfg), 3)
    # vision tower from a CLIP checkpoint: its vision_model.* keys, the text tower ignored, buffers dropped
    llm = {k: v for k, v in sd.items() if not k.startswith(arch.VISION_PREFIX)}
    clip = {k[len(arch.VISION_PREFIX):]: v for k, v in sd.items() if k.startswith(arch.VISION_PREFIX)}
    clip["text_model.embeddings.token_embedding.weight"] = torch.zeros(8, 4)
    clip["logit_scale"] = torch.tensor(1.0)
    clip["vision_model.embeddings.position_ids"] = torch.arange(577)[None]
    llm["model.layers.0.self_attn.rotary_emb.inv_freq"] = torch.zeros(64)
    out = arch.llava_state_dict(llm, clip, cfg)
    assert set(out) == set(arch.llava_shapes(cfg))
    assert set(arch.llava_state_dict(sd, None, cfg)) == set(out)
    with pytest.raises(ValueError, match="and a CLIP checkpoint"):
        arch.llava_state_dict(sd, clip, cfg)
    missing = dict(sd)
    del missing["model.layers.1.mlp.up_proj.weight"]
    with pytest.raises(ValueError, match="up_proj"):
        arch.llava_state_dict(missing, None, cfg)
    extra = dict(sd, **{"model.layers.9.mlp.up_proj.weight": torch.zeros(1)})
    with pytest.raises(ValueError, match="unexpected.*layers.9"):
        arch.llava_state_dict(extra, None, cfg)
    wrong = dict(sd, **{"lm_head.weight": torch.zeros(3, 4)})
    with pytest.raises(ValueError, match="lm_head.weight"):
        arch.llava_state_dict(wrong, None, cfg)


def test_cli_accepts_llava_bit_16_only(tmp_path):
    args = lambda *x: cli.parse_args(["--input", str(tmp_path / "in"), "--output", str(tmp_path / "out"), *x])  # noqa: E731
    loop_mod.check_supported(args("--captioner", "llava", "--llava_bit", "16"))
    for bit in ("4", "8"):
        with pytest.raises(NotImplementedError, match="captioner") as e:
            loop_mod.check_supported(args("--captioner", "llava", "--llava_bit", bit))
        assert "--llava_bit 16" in str(e.value)
    with pytest.raises(NotImplementedError, match="captioner"):
        loop_mod.check_supported(args("--captioner", "llava"))            # the default --llava_bit is 4
    assert cli.parse_args(["--input", "i", "--output", "o"]).captioner == "none"
    for bit in ("4", "8"):
        with pytest.raises(NotImplementedError, match="--llava_bit 16"):
            cap.LLaVACaptioner("cuda", bit)
    from diffbir.utils.caption import LLaVACaptioner
    assert LLaVACaptioner is cap.LLaVACaptioner
