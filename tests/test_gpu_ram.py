"""-m gpu: RAM++ captioner (`--captioner ram`): the 12x12 window attention, patch merging, token mean and label
reweighting kernels against fp64 references; RamPlusEngine against the fp32 oracle on the GPU and against the
reference fixture; graph replays; the CLI end to end with the caption in the prompt."""
import csv
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from tests.gpu_util import no_tf32, rel_err, rel_rms

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from diffbir_b200 import lib
    lib.load()
    no_tf32()
    return lib


def tol16(L):
    return 1.5e-3 if L.operand_dtype() == torch.float16 else 1e-2


def window_attention_ref(qkv, b, h, w, heads, shift, table, ws=12, dh=32):
    """fp64 WindowAttention + roll + partition + region mask (swin_transformer.py:116-147, 211-266)."""
    from oracle.swinir import rel_pos_index, shift_mask
    c = heads * dh
    y = qkv[:, :3 * c].double().view(b, h, w, 3 * c)
    if shift:
        y = torch.roll(y, (-shift, -shift), (1, 2))
    win = y.view(b, h // ws, ws, w // ws, ws, 3 * c).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, 3 * c)
    nwin = win.shape[0]
    t = win.view(nwin, ws * ws, 3, heads, dh).permute(2, 0, 3, 1, 4)
    attn = (t[0] * dh ** -0.5) @ t[1].transpose(-1, -2)
    attn = attn + table.double()[rel_pos_index(ws).to(qkv.device).view(-1)].view(ws * ws, ws * ws, heads).permute(2, 0, 1)[None]
    if shift:
        m = shift_mask(h, w, ws, shift, qkv.device).double()
        attn = (attn.view(b, m.shape[0], heads, ws * ws, ws * ws) + m[None, :, None]).view(nwin, heads, ws * ws, ws * ws)
    o = (torch.softmax(attn, -1) @ t[2]).transpose(1, 2).reshape(nwin, ws * ws, c)
    o = o.view(b, h // ws, w // ws, ws, ws, c).permute(0, 1, 3, 2, 4, 5).reshape(b, h, w, c)
    if shift:
        o = torch.roll(o, (shift, shift), (1, 2))
    return o.reshape(b * h * w, c)


@pytest.mark.parametrize("heads,side", [(6, 96), (12, 48), (24, 24), (48, 12)])
@pytest.mark.parametrize("shift", [0, 6])
def test_window12_attention(L, heads, side, shift):
    if shift and side == 12:
        pytest.skip("stage 4 is one un-shifted window (swin_transformer.py:195-198)")
    b, c = 2, heads * 32
    g = torch.Generator(device="cuda").manual_seed(heads + shift)
    dt = L.operand_dtype()
    qkv = (torch.randn(b * side * side, 3 * c, device="cuda", generator=g) * 1.5).to(dt)
    table = torch.randn(23 * 23, heads, device="cuda", generator=g) * 0.5
    out = torch.zeros(b * side * side, c, device="cuda", dtype=dt)
    L.window_attention(qkv, 3 * c, b, side, side, heads, 32, shift, table, -100.0, out, c, window=12)
    ref = window_attention_ref(qkv, b, side, side, heads, shift, table)
    assert rel_err(out, ref) < tol16(L)


def test_patch_merge(L):
    n, h, w, c = 2, 24, 24, 768
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(n * h * w, c + 4, device="cuda", generator=g) * 2 + 0.5      # row stride > c
    gamma = 1 + 0.1 * torch.randn(4 * c, device="cuda", generator=g)
    beta = 0.1 * torch.randn(4 * c, device="cuda", generator=g)
    out = torch.empty(n * h * w // 4, 4 * c, device="cuda", dtype=L.operand_dtype())
    L.swin_patch_merge(x, c + 4, n, h, w, c, gamma, beta, out, 4 * c)
    xx = x[:, :c].double().view(n, h, w, c)
    cat = torch.cat([xx[:, 0::2, 0::2], xx[:, 1::2, 0::2], xx[:, 0::2, 1::2], xx[:, 1::2, 1::2]], -1).reshape(-1, 4 * c)
    ref = torch.nn.functional.layer_norm(cat, (4 * c,), gamma.double(), beta.double(), 1e-5)
    assert rel_err(out, ref) < tol16(L)


def test_token_mean(L):
    n, tokens, c = 2, 144, 1536
    x = torch.randn(n * tokens, c, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4))
    out = torch.empty(n * (tokens + 1), c, device="cuda", dtype=L.operand_dtype())
    L.token_mean(x, c, n, tokens, c, out, c)
    xx = x.double().view(n, tokens, c)
    ref = torch.cat([xx.mean(1, keepdim=True), xx], 1).reshape(-1, c)
    assert rel_err(out, ref) < tol16(L)


def test_label_reweight(L):
    b, classes, per, dim = 2, 300, 51, 512
    g = torch.Generator(device="cuda").manual_seed(5)
    dt = L.operand_dtype()
    label = (torch.rand(classes * per, dim, device="cuda", generator=g) * 2 - 1).mul(dim ** -0.5 * 3).to(dt)
    emb = torch.randn(b, 145, dim, device="cuda", generator=g)
    out = torch.empty(b * classes, dim, device="cuda", dtype=dt)
    scale = 1 / 0.07
    L.label_reweight(emb, 145 * dim, b, label, classes, per, scale, out, dim)
    cls = emb[:, 0].double()
    cls = cls / cls.norm(dim=-1, keepdim=True)
    lab = label.double()
    p = torch.softmax((scale * cls @ lab.t()).view(b, classes, per), -1)
    ref = (p.unsqueeze(-1) * lab.view(classes, per, dim)).sum(2).reshape(b * classes, dim)
    assert rel_err(out, ref) < tol16(L)


# ---------------------------------------------------------------------------------------------- engine
@pytest.fixture(scope="module")
def fixture(golden_dir):
    return dict(np.load(golden_dir / "ram_small.npz"))


@pytest.fixture(scope="module")
def engine_and_sd(L, fixture):
    from diffbir_b200 import arch
    from diffbir_b200.engine.ram import RamPlusEngine
    from tests.test_ram import fixture_sd
    sd = fixture_sd(fixture)
    return RamPlusEngine(sd, device="cuda"), arch.ram_state_dict(sd)


def decision_bar(eng):
    """Decisions must agree wherever the reference logit lies farther than this fraction of the reference logits' std
    from the class's threshold logit. Measured on an H100 against the fixture: flips at most 0.006 std from the
    threshold (fp16 operands) and 0.35 std (bf16): the synthetic weights leave the tagging head's residual stream tiny
    before its post-LNs, which amplify the operand rounding (logit error RMS 2.8% / 26% of the logits' std, while
    image_embeds agree to 8e-4 / 6e-3)."""
    return 0.05 if eng.op_dtype == torch.float16 else 0.5


def test_engine_against_reference_fixture(engine_and_sd, fixture):
    from diffbir_b200.utils.caption import decide
    from tests.test_ram import fixture_image
    eng, _ = engine_and_sd
    logits = eng.forward(fixture_image(fixture).cuda())[0].cpu()
    emb = eng.image_embeds(1)[0].cpu()
    ref_logits = torch.from_numpy(fixture["logits"])
    e = rel_rms(emb, torch.from_numpy(fixture["image_embeds"]))
    thr = torch.from_numpy(fixture["thresholds"])
    ref_dec = torch.from_numpy(fixture["decisions"])
    dec = torch.sigmoid(logits) > thr
    distance = (ref_logits - torch.log(thr / (1 - thr))).abs() / ref_logits.std()
    names = dict(zip(fixture["fired"].tolist(), fixture["fired_tags"].tolist()))
    tags = [names.get(i, f"unfired{i}") for i in range(len(thr))]
    flips = (dec != ref_dec).nonzero().flatten().tolist()
    print(f"RAM++ engine vs reference ({eng.op_dtype}): image_embeds rel-rms {e:.2e}, logits error rms / std "
          f"{(logits - ref_logits).pow(2).mean().sqrt() / ref_logits.std():.2e}, decisions differing {len(flips)} "
          f"(largest threshold distance {max([float(distance[i]) for i in flips], default=0.0):.4f} std), "
          f"stages rel-rms " + ", ".join(f"{rel_rms(eng.stage_output(1, i)[0, ::int(fixture['stage_row_step'])].cpu(), torch.from_numpy(fixture[f'stage{i}'])):.1e}" for i in range(4)))
    print(f"  caption: {decide(logits, thr, tags)!r}\n  fixture: {str(fixture['caption'])!r}")
    assert e <= 1e-2
    sure = distance > decision_bar(eng)
    assert torch.equal(dec[sure], ref_dec[sure])


def test_engine_against_oracle_batch2(engine_and_sd, fixture):
    """Batch 2 (the fixture image and a second one) against the fp32 oracle on the GPU (TF32 off)."""
    from oracle import ram as oram
    eng, sd = engine_and_sd
    x = torch.rand(2, 3, 384, 384, generator=torch.Generator().manual_seed(7)).cuda()
    logits = eng.forward(x)
    emb = eng.image_embeds(2)
    with torch.no_grad():
        ref_emb, ref_logits = oram.ram_forward({k: v.cuda() for k, v in sd.items()}, oram.normalize(x))
    thr = torch.from_numpy(fixture["thresholds"]).cuda()
    sure = (ref_logits - torch.log(thr / (1 - thr))).abs() > decision_bar(eng) * ref_logits.std()
    e = rel_rms(emb, ref_emb)
    print(f"RAM++ engine vs oracle, batch 2: image_embeds rel-rms {e:.2e}, logits rel-rms {rel_rms(logits, ref_logits):.2e}")
    assert e <= 1e-2
    assert torch.equal((torch.sigmoid(logits) > thr)[sure], (torch.sigmoid(ref_logits) > thr)[sure])


def test_graph_replay_is_bit_identical(engine_and_sd):
    eng, _ = engine_and_sd
    x = torch.rand(1, 3, 384, 384, generator=torch.Generator().manual_seed(8)).cuda()
    a = eng.forward(x)
    ea = eng.image_embeds(1)
    b = eng.forward(x)
    assert torch.equal(a, b) and torch.equal(ea, eng.image_embeds(1))


def test_cli_captioner_ram_synthetic(tmp_path):
    import inference as cli
    from diffbir_b200.utils.synth import synthetic_lq
    (tmp_path / "in").mkdir()
    from PIL import Image
    Image.fromarray(synthetic_lq(128, 160, seed=3)[0]).save(tmp_path / "in" / "img.png")
    cli.main(["--task", "sr", "--version", "v2.1", "--upscale", "4", "--sampler", "spaced", "--steps", "2",
              "--captioner", "ram", "--pos_prompt", "Cinematic", "--input", str(tmp_path / "in"), "--output",
              str(tmp_path / "out"), "--synthetic"])
    with open(tmp_path / "out" / "prompt.csv") as f:
        rows = list(csv.reader(f))
    pos = rows[1][1]
    print(f"pos_prompt with the RAM++ caption: {pos[:200]!r}")
    assert pos.endswith(", Cinematic") and pos.startswith("tag") and pos.count("tag") >= 5
