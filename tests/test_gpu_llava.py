"""-m gpu: LLaVA captioner (`--captioner llava --llava_bit 16`): RMSNorm, RoPE / KV write, causal and decode-step
attention, GEMV with each epilogue, argmax, embedding gather and the quick_gelu / SwiGLU GEMM epilogues against fp64
references; LlavaEngine against the reference fixture and the fp32 oracle; graph replay against the eager path; a
second image against a fresh engine; the CLI end to end with the caption in the prompt."""
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
    return 2e-3 if L.operand_dtype() == torch.float16 else 1.2e-2


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def test_rmsnorm(L):
    rows, c, ldx = 3, 4096, 4100
    x = torch.randn(rows, ldx, device="cuda", generator=gen(1)) * 3 + 0.5
    w = 1 + 0.1 * torch.randn(c, device="cuda", generator=gen(2))
    out = torch.zeros(rows, c + 8, device="cuda", dtype=L.operand_dtype())
    L.rmsnorm(x, ldx, rows, c, w, out, c + 8)
    xx = x[:, :c].double()
    ref = w.double() * xx * torch.rsqrt(xx.pow(2).mean(-1, keepdim=True) + 1e-5)
    assert rel_err(out[:, :c], ref) < tol16(L)
    assert not out[:, c:].any()


def rope_ref(x, pos, theta=10000.0):
    """fp64 rotate_half RoPE of x [n, heads, 128] at positions pos [n]."""
    inv = 1.0 / theta ** (torch.arange(0, 128, 2, device=x.device).double() / 128)
    f = pos.double()[:, None] * inv[None]
    emb = torch.cat([f, f], -1)[:, None]
    rot = torch.cat([-x[..., 64:], x[..., :64]], -1)
    return x * emb.cos() + rot * emb.sin()


def test_rope_kv_at_device_offset(L):
    rows, heads, cap, p0 = 5, 4, 1200, 1150
    d = heads * 128
    qkv = torch.randn(rows, 3 * d, device="cuda", generator=gen(3))
    dt = L.operand_dtype()
    q = torch.zeros(rows, d, device="cuda", dtype=dt)
    kc = torch.zeros(cap, heads, 128, device="cuda", dtype=dt)
    vc = torch.zeros_like(kc)
    pos0 = torch.tensor([p0], dtype=torch.int32, device="cuda")
    L.rope_kv(qkv, 3 * d, rows, heads, pos0, q, d, kc, vc)
    pos = torch.arange(p0, p0 + rows, device="cuda")
    x = qkv.double().view(rows, 3, heads, 128)
    assert rel_err(q.view(rows, heads, 128), rope_ref(x[:, 0], pos)) < tol16(L)
    assert rel_err(kc[p0:p0 + rows], rope_ref(x[:, 1], pos)) < tol16(L)
    assert torch.equal(vc[p0:p0 + rows], x[:, 2].to(dt))
    assert not kc[:p0].any() and not kc[p0 + rows:].any() and not vc[:p0].any()


def causal_ref(q, kc, vc, heads, n):
    qq = q.double().view(n, heads, 128).transpose(0, 1)
    k = kc[:n].double().transpose(0, 1)
    v = vc[:n].double().transpose(0, 1)
    s = qq @ k.transpose(1, 2) / 128 ** 0.5
    s = s.masked_fill(torch.ones(n, n, device=q.device, dtype=torch.bool).triu(1), float("-inf"))
    return (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(n, heads * 128)


@pytest.mark.parametrize("n", [1, 63, 64, 577, 630])
def test_attention_causal(L, n):
    heads, dt = 4, L.operand_dtype()
    d = heads * 128
    q = (torch.randn(n, d + 64, device="cuda", generator=gen(n)) * 2).to(dt)          # row stride > heads * 128
    kc = (torch.randn(n + 10, heads, 128, device="cuda", generator=gen(n + 1)) * 2).to(dt)
    vc = torch.randn(n + 10, heads, 128, device="cuda", generator=gen(n + 2)).to(dt)
    out = torch.zeros(n, d, device="cuda", dtype=dt)
    L.attention_causal(q, d + 64, kc, vc, heads, n, out, d)
    assert rel_err(out, causal_ref(q[:, :d], kc, vc, heads, n)) < tol16(L)


def test_attention_decode_lengths(L):
    """Lengths across the 64-key split boundaries up to the capacity; the combine is deterministic."""
    heads, cap, dt = 4, 1200, L.operand_dtype()
    q = (torch.randn(heads * 128, device="cuda", generator=gen(11)) * 2).to(dt)
    kc = (torch.randn(cap, heads, 128, device="cuda", generator=gen(12)) * 2).to(dt)
    vc = torch.randn(cap, heads, 128, device="cuda", generator=gen(13)).to(dt)
    ws = torch.empty(L.attention_decode_ws_bytes(heads, cap), dtype=torch.uint8, device="cuda")
    out = torch.empty(heads * 128, device="cuda", dtype=dt)
    length = torch.zeros(1, dtype=torch.int32, device="cuda")
    qq = q.double().view(heads, 1, 128)
    for n in (1, 2, 63, 64, 65, 127, 128, 129, 577, 640, 1023, 1199, 1200):
        length.fill_(n)
        L.attention_decode(q, kc, vc, heads, cap, length, ws, out)
        s = qq @ kc[:n].double().permute(1, 2, 0) / 128 ** 0.5
        ref = (torch.softmax(s, -1) @ vc[:n].double().transpose(0, 1)).reshape(-1)
        assert rel_err(out, ref) < tol16(L), n
        first = out.clone()
        L.attention_decode(q, kc, vc, heads, cap, length, ws, out)
        assert torch.equal(first, out)


GEMV_CASES = [("qkv", 12288, 4096, "none", torch.float32), ("o_proj", 4096, 4096, "residual", torch.float32),
              ("gate_up", 22016, 4096, "swiglu", None), ("down", 4096, 11008, "residual", torch.float32),
              ("lm_head", 32000, 4096, "none", torch.float32)]


@pytest.mark.parametrize("name,N,K,epi,out_dt", GEMV_CASES, ids=[c[0] for c in GEMV_CASES])
def test_gemv(L, name, N, K, epi, out_dt):
    dt = L.operand_dtype()
    out_dt = out_dt or dt
    w = ((torch.rand(N, K, device="cuda", generator=gen(N)) * 2 - 1) * K ** -0.5).to(dt)
    x = torch.randn(K, device="cuda", generator=gen(K)).to(dt)
    y64 = w.double() @ x.double()
    if epi == "swiglu":
        pack = 256
        t = y64.view(N // pack, 2, pack // 2)
        ref = (t[:, 0] * torch.nn.functional.silu(t[:, 1])).reshape(-1)
        y = torch.empty(N // 2, device="cuda", dtype=out_dt)
        L.gemv(w, x, y, N=N, K=K, epilogue="swiglu", pack=pack)
    elif epi == "residual":
        res = torch.randn(N, device="cuda", generator=gen(5))
        ref = y64 + res.double()
        y = res.clone()                                   # in place, as the decode step's residual stream
        L.gemv(w, x, y, N=N, K=K, epilogue="residual", residual=y)
    else:
        ref = y64
        y = torch.empty(N, device="cuda", dtype=out_dt)
        L.gemv(w, x, y, N=N, K=K)
    tol = 2e-5 if out_dt == torch.float32 else tol16(L)
    assert rel_err(y, ref) < tol, name


def test_argmax_ties_and_advance(L):
    n = 32000
    logits = torch.randn(n, device="cuda", generator=gen(7))
    logits[[5, 17000, 31999]] = 10.0                      # a three-way tie: the first index wins
    tok = torch.zeros(1, dtype=torch.int32, device="cuda")
    state = torch.tensor([620, 621], dtype=torch.int32, device="cuda")
    L.argmax(logits, n, tok, advance=state)
    assert int(tok) == 5 and state.tolist() == [621, 622]
    logits[5] = 9.0
    L.argmax(logits, n, tok)
    assert int(tok) == 17000 and state.tolist() == [621, 622]
    x = torch.randn(n, device="cuda", generator=gen(8))
    L.argmax(x, n, tok)
    assert int(tok) == int(x.argmax())


def test_embed_gather(L):
    dt = L.operand_dtype()
    table = torch.randn(512, 256, device="cuda", generator=gen(9)).to(dt)
    ids = torch.tensor([3, 0, 511, 3], dtype=torch.int32, device="cuda")
    out = torch.zeros(4, 300, device="cuda")
    L.embed_gather(table, 512, ids, 4, 256, out, 300)
    assert torch.equal(out[:, :256], table[ids.long()].float()) and not out[:, 256:].any()


def test_gemm_quick_gelu_and_swiglu_epilogues(L):
    dt = L.operand_dtype()
    M, N, K = 577, 512, 256
    a = torch.randn(M, K, device="cuda", generator=gen(20)).to(dt)
    w = ((torch.rand(N, K, device="cuda", generator=gen(21)) * 2 - 1) * K ** -0.5 * 2).to(dt)
    bias = 0.1 * torch.randn(N, device="cuda", generator=gen(22))
    out = torch.empty(M, N, device="cuda")
    L.gemm(a, w, out, M=M, N=N, K=K, bias=bias, act="quick_gelu")
    y = a.double() @ w.double().t() + bias.double()
    assert rel_err(out, y * torch.sigmoid(1.702 * y)) < 2e-5 * 50
    # SwiGLU: rows packed per 256-row tile as [128 values | 128 gates]; output N/2 = values * silu(gates)
    out2 = torch.empty(M, N // 2, device="cuda", dtype=dt)
    L.gemm(a, w, out2, M=M, N=N, K=K, geglu=2, force_bn=256)
    t = (a.double() @ w.double().t()).view(M, N // 256, 2, 128)
    ref = (t[:, :, 0] * torch.nn.functional.silu(t[:, :, 1])).reshape(M, N // 2)
    assert rel_err(out2, ref) < tol16(L)
    # geglu = 1 keeps GELU(erf) gates
    L.gemm(a, w, out2, M=M, N=N, K=K, geglu=True, force_bn=256)
    ref1 = (t[:, :, 0] * torch.nn.functional.gelu(t[:, :, 1])).reshape(M, N // 2)
    assert rel_err(out2, ref1) < tol16(L)


def test_vision_attention_ragged_577(L):
    """dbir_attention (head_dim 64) at CLIP's 577 tokens, q / k / v column slices of the fused QKV rows."""
    dt, heads, n = L.operand_dtype(), 16, 577
    c = heads * 64
    qkv = torch.randn(n, 3 * c, device="cuda", generator=gen(30)).to(dt)
    out = torch.zeros(n, c, device="cuda", dtype=dt)
    ws = torch.zeros(max(L.attention_ws_bytes(1, heads, n, n), 1), dtype=torch.uint8, device="cuda")
    L.attention(qkv, qkv[:, c:], qkv[:, 2 * c:], out, batch=1, heads=heads, sq=n, skv=n, ldq=3 * c, ldk=3 * c,
                ldv=3 * c, ldo=c, ws=ws)
    t = qkv.double().view(n, 3, heads, 64).permute(1, 2, 0, 3)
    ref = (torch.softmax(t[0] @ t[1].transpose(1, 2) / 8, -1) @ t[2]).transpose(0, 1).reshape(n, c)
    assert rel_err(out, ref) < tol16(L)


# ---------------------------------------------------------------------------------------------- engine
@pytest.fixture(scope="module")
def fixture(golden_dir):
    return dict(np.load(golden_dir / "llava_small.npz"))


def make_engine(f, max_new=16):
    from diffbir_b200.engine.llava import LlavaEngine
    from tests.test_llava import fixture_cfg, fixture_sd
    return LlavaEngine(fixture_sd(f), f["input_ids"].tolist(), fixture_cfg(f), device="cuda", max_new_tokens=max_new)


@pytest.fixture(scope="module")
def engine(L, fixture):
    return make_engine(fixture)


def logit_rms_bound(L):
    """Relative RMS of features and logits against the fp32 reference. fp16 operands round at 2^-11, bf16 at 2^-8;
    measured on an H100 at the fixture size: at most 7.9e-4 (fp16) and 6.5e-3 (bf16)."""
    return 3e-3 if L.operand_dtype() == torch.float16 else 2e-2


def margin_bound(L):
    """A token must equal the reference's wherever the reference's top-1 logit margin exceeds this (the fixture's
    logits have an RMS of 2.2; the bf16 logit error RMS is about 0.015 of it)."""
    return 0.05 if L.operand_dtype() == torch.float16 else 0.25


def test_engine_against_reference_fixture(L, engine, fixture):
    from tests.test_llava import fixture_pixels
    f = fixture
    x = fixture_pixels(f).cuda()
    feats = engine.image_features(x).cpu()
    step = int(f["feature_row_step"])
    e_feat = rel_rms(feats[::step], torch.from_numpy(f["feature_rows"]))
    pre = engine.prefill_logits(x).cpu()
    e_pre = rel_rms(pre, torch.from_numpy(f["prefill_logits"]))
    ref_forced = torch.from_numpy(f["forced_logits"])
    forced = engine.forced_logits(x, f["tokens"].tolist()).cpu()
    e_forced = rel_rms(forced, ref_forced)
    toks = engine.generate(x)
    top2 = ref_forced.topk(2, -1).values
    margins = (top2[:, 0] - top2[:, 1]).tolist()
    sure = next((i for i, m in enumerate(margins) if m < margin_bound(L)), len(margins))
    print(f"LLaVA engine vs reference ({L.operand_dtype()}): image features rel-rms {e_feat:.2e}, prefill logits "
          f"{e_pre:.2e}, teacher-forced logits {e_forced:.2e}; tokens {toks} vs {f['tokens'].tolist()} "
          f"(compared over the first {sure} steps)")
    assert e_feat <= logit_rms_bound(L) and e_pre <= logit_rms_bound(L) and e_forced <= logit_rms_bound(L)
    # greedy: equal up to the first step whose margin is below the bound (a flip there changes every later step)
    assert toks[:sure] == f["tokens"].tolist()[:sure]
    # teacher-forced: every step whose margin clears the bound picks the reference's token
    clear = torch.tensor(margins) > margin_bound(L)
    assert torch.equal(forced.argmax(-1)[clear], torch.from_numpy(f["tokens"])[clear])


def test_engine_against_oracle(L, engine, fixture):
    """A second image against the fp32 oracle on the GPU (TF32 off): features and teacher-forced logits."""
    from oracle import llava as olv
    from diffbir_b200 import arch
    from diffbir_b200.utils.caption import clip_normalize
    from tests.test_llava import fixture_cfg, fixture_sd
    cfg = fixture_cfg(fixture)
    sd = {k: v.cuda() for k, v in arch.llava_state_dict(fixture_sd(fixture), None, cfg).items()}
    x = torch.rand(1, 3, 336, 336, generator=torch.Generator().manual_seed(5)).cuda()
    toks, ref_logits, ref_feats = olv.greedy(sd, cfg, clip_normalize(x.cpu()).cuda(), fixture["input_ids"].tolist(), 8)
    feats = engine.image_features(x)
    logits = engine.forced_logits(x, toks)
    print(f"LLaVA engine vs oracle: features rel-rms {rel_rms(feats, ref_feats):.2e}, logits {rel_rms(logits, ref_logits):.2e}")
    assert rel_rms(feats, ref_feats) <= logit_rms_bound(L) and rel_rms(logits, ref_logits) <= logit_rms_bound(L)


def test_graph_replay_matches_eager_and_second_image_matches_fresh_engine(L, engine, fixture):
    from tests.test_llava import fixture_pixels
    x1 = fixture_pixels(fixture).cuda()
    x2 = torch.rand(1, 3, 336, 336, generator=torch.Generator().manual_seed(9)).cuda()
    toks = fixture["tokens"].tolist()
    eager = engine.forced_logits(x1, toks, use_graphs=False)
    graph = engine.forced_logits(x1, toks, use_graphs=True)
    assert torch.equal(eager, graph)
    assert engine.generate(x1, use_graphs=False) == engine.generate(x1, use_graphs=True)
    engine.generate(x1)
    second = engine.generate(x2)
    second_logits = engine.forced_logits(x2, second, use_graphs=True)
    fresh = make_engine(fixture)
    assert fresh.generate(x2) == second
    assert torch.equal(fresh.forced_logits(x2, second, use_graphs=True), second_logits)


def test_cli_captioner_llava_synthetic(tmp_path, monkeypatch):
    import inference as cli
    from diffbir_b200.utils import caption as cap
    from diffbir_b200.utils.synth import synthetic_lq
    from PIL import Image
    (tmp_path / "in").mkdir()
    Image.fromarray(synthetic_lq(128, 160, seed=3)[0]).save(tmp_path / "in" / "img.png")
    captions = []
    call = cap.LLaVACaptioner.__call__
    monkeypatch.setattr(cap.LLaVACaptioner, "__call__", lambda self, im: captions.append(call(self, im)) or captions[-1])
    cli.main(["--task", "sr", "--version", "v2.1", "--upscale", "4", "--sampler", "spaced", "--steps", "2",
              "--captioner", "llava", "--llava_bit", "16", "--pos_prompt", "Cinematic", "--input",
              str(tmp_path / "in"), "--output", str(tmp_path / "out"), "--synthetic"])
    with open(tmp_path / "out" / "prompt.csv") as f:
        rows = list(csv.reader(f))
    pos = rows[1][1]
    print(f"pos_prompt with the LLaVA caption: {pos[:200]!r}")
    assert (tmp_path / "out" / "img.png").exists()
    assert len(captions) == 1 and captions[0] and pos == f"{captions[0]}, Cinematic"
