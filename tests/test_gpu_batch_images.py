"""-m gpu: `--batch_images N` end to end (`--synthetic` weights, full SD-2.1 config) and the kernels it adds.

A folder of 5 inputs, three of one size and two of another, restored with --batch_images 4 (calls of 3 and 2 images):
every PNG must be bit-identical to Pipeline.run of that image alone after set_seed(seed + k) with the batch-invariant
plans (DBIR_DETERMINISTIC=1), for the sampler families, the `cond` start point with noise augmentation, and both
captioners. Kernels: dbir_gemv_rows in each epilogue, dbir_argmax_rows, dbir_rope_kv_seqs / dbir_attention_decode_seqs,
LlavaEngine's batched decode and dbir_brownian_increment_samples, each against its single-row / single-sequence /
single-seed counterpart with torch.equal."""
import csv
import os
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from PIL import Image

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

pytestmark = pytest.mark.gpu
SIZES = {"a0.png": (128, 128), "a1.png": (128, 128), "a2.png": (128, 128), "b0.png": (128, 160), "b1.png": (128, 160)}
BASE = ["--task", "sr", "--version", "v2.1", "--upscale", "4", "--steps", "4", "--cfg_scale", "4.0", "--captioner", "none",
        "--pos_prompt", "a photo", "--neg_prompt", "low quality, blurry", "--synthetic", "--batch_images", "4"]


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    from diffbir_b200.utils.synth import synthetic_lq
    d = tmp_path_factory.mktemp("batch_in")
    for i, (name, (h, w)) in enumerate(SIZES.items()):
        Image.fromarray(synthetic_lq(h, w, seed=20 + i)[0]).save(d / name)
    return d


@pytest.fixture(scope="module")
def batch_loop(inputs):
    """One loop (--batch_images 4, which pins DBIR_DETERMINISTIC=1); each test changes its sampling flags."""
    import inference as cli
    from diffbir_b200.inference import BSRInferenceLoop
    old = os.environ.get("DBIR_DETERMINISTIC")
    try:
        loop = BSRInferenceLoop(cli.parse_args(BASE + ["--input", str(inputs), "--output", "-"]))
        loop.pipeline.cldm._build()
        assert loop.pipeline.cldm.engine.deterministic
    finally:
        if old is None:
            os.environ.pop("DBIR_DETERMINISTIC", None)
        else:
            os.environ["DBIR_DETERMINISTIC"] = old
    return loop


def run_and_compare(loop, inputs, out: Path, extra=()):
    """--batch_images 4 over the folder, then every image alone after set_seed(seed + k) on the same pipeline."""
    import inference as cli
    a = loop.args = cli.parse_args(BASE + list(extra) + ["--input", str(inputs), "--output", str(out)])
    loop.run()
    with open(out / "prompt.csv") as f:
        rows = list(csv.reader(f))[1:]
    assert [r[0] for r in rows] == [Path(n).stem for n in sorted(SIZES)]
    for k, name in enumerate(sorted(SIZES)):
        pos = rows[k][1]
        # as in a fresh process: the single run encodes its [pos, neg] pair as one text-tower batch of 2
        loop.pipeline.cldm._txt_cache.clear()
        cli.set_seed(a.seed + k)
        lq = loop.after_load_lq(Image.open(inputs / name).convert("RGB"))
        want = loop.pipeline.run(
            lq[None], a.steps, a.strength, a.cleaner_tiled, a.cleaner_tile_size, a.cleaner_tile_stride,
            a.vae_encoder_tiled, a.vae_encoder_tile_size, a.vae_decoder_tiled, a.vae_decoder_tile_size, a.cldm_tiled,
            a.cldm_tile_size, a.cldm_tile_stride, pos, a.neg_prompt, a.cfg_scale, a.start_point_type, a.sampler,
            a.noise_aug, a.rescale_cfg, a.s_churn, a.s_tmin, a.s_tmax, a.s_noise, a.eta, a.order)[0]
        got = np.array(Image.open(out / name))
        assert got.shape == want.shape and want.std() > 1.0
        assert np.array_equal(got, want), f"{name}: {(got != want).mean():.2%} of the values differ"
    return rows


@pytest.mark.parametrize("sampler", ["spaced", "ddim", "dpm++_m2", "edm_euler_a", "edm_dpm++_sde"])
def test_batch_images_bit_identical_to_each_image_alone(tmp_path, batch_loop, inputs, sampler):
    rows = run_and_compare(batch_loop, inputs, tmp_path / "out", ["--sampler", sampler])
    assert all(r[1] == "a photo" for r in rows)


def test_batch_images_cond_start_with_noise_aug(tmp_path, batch_loop, inputs):
    run_and_compare(batch_loop, inputs, tmp_path / "out",
                    ["--sampler", "edm_dpm++_2s_a", "--start_point_type", "cond", "--noise_aug", "200"])


@pytest.mark.parametrize("captioner", ["ram", "llava"])
def test_batch_images_with_captioner(tmp_path, batch_loop, inputs, captioner):
    """The list call captions each image as the single call does; the files match the single restorations."""
    import inference as cli
    loop = batch_loop
    loop.args = cli.parse_args(BASE + ["--captioner", captioner, "--llava_bit", "16", "--input", str(inputs),
                                       "--output", "-"])
    loop.load_captioner()
    try:
        if captioner == "ram":              # the batched forward's logits, row by row, against single-image forwards
            from diffbir_b200.utils.caption import preprocess
            eng = loop.captioner.engine
            x = torch.cat([preprocess(Image.open(inputs / n).convert("RGB"), loop.captioner.size)
                           for n in sorted(SIZES)]).to(eng.dev)
            for b0, b1 in ((0, 3), (3, 5)):                       # the calls' batch sizes, 3 and 2
                full = eng.forward(x[b0:b1]).clone()
                for i in range(b0, b1):
                    assert torch.equal(full[i - b0], eng.forward(x[i:i + 1])[0]), i
        rows = run_and_compare(loop, inputs, tmp_path / "out",
                               ["--captioner", captioner, "--llava_bit", "16", "--sampler", "spaced"])
        singles = [loop.captioner(Image.open(inputs / n).convert("RGB")) for n in sorted(SIZES)]
        assert [r[1] for r in rows] == [f"{c}, a photo" if c else "a photo" for c in singles]
        print(f"{captioner} captions: {[c[:60] for c in singles]}")
    finally:
        from diffbir_b200.utils.caption import EmptyCaptioner
        loop.captioner = EmptyCaptioner("cuda")
        torch.cuda.empty_cache()


def test_prompt_pairs_are_the_single_run_s_text_rows(batch_loop):
    """prepare_condition_pairs: image i's cond / uncond text rows equal those of a single run on an empty cache
    ([pos, neg] as one tower batch), whichever prompts share the call. (The text tower's rows do depend on its batch
    size: "a photo" encoded alone differs from its row beside the negative prompt.)"""
    cldm = batch_loop.pipeline.cldm
    neg = "low quality, blurry"
    prompts = ["tags, of, an, image, a photo", "a photo", "", "a photo"]
    img = torch.rand(len(prompts), 3, 512, 512, device="cuda", generator=gen(3))
    cond, uncond = cldm.prepare_condition_pairs(img, prompts, neg)
    for i, p in enumerate(prompts):
        cldm._txt_cache.clear()
        c1, u1 = cldm.prepare_condition_pair(img[i:i + 1], [p], [neg])
        assert torch.equal(cond["c_txt"][i], c1["c_txt"][0]) and torch.equal(uncond["c_txt"][i], u1["c_txt"][0]), p
    cldm._txt_cache.clear()
    print(f"'a photo' alone vs beside the negative prompt equal: "
          f"{torch.equal(cldm.encode_text(['a photo'])[0], cond['c_txt'][1])}")


# ---------------------------------------------------------------------------------------------- kernels
@pytest.fixture(scope="module")
def L():
    from diffbir_b200 import lib
    lib.load()
    return lib


GEMV_CASES = [("qkv", 12288, 4096, "none", torch.float32), ("o_proj", 4096, 4096, "residual", torch.float32),
              ("gate_up", 22016, 4096, "swiglu", None), ("down", 4096, 11008, "residual", torch.float32),
              ("lm_head", 32000, 4096, "none", torch.float32)]


@pytest.mark.parametrize("M", [2, 5, 8])
@pytest.mark.parametrize("name,N,K,epi,out_dt", GEMV_CASES, ids=[c[0] for c in GEMV_CASES])
def test_gemv_rows_equal_single_row_gemv(L, M, name, N, K, epi, out_dt):
    dt = L.operand_dtype()
    out_dt = out_dt or dt
    w = ((torch.rand(N, K, device="cuda", generator=gen(N)) * 2 - 1) * K ** -0.5).to(dt)
    x = torch.randn(M, K + 8, device="cuda", generator=gen(K)).to(dt)          # row stride > K
    n_out = N // 2 if epi == "swiglu" else N
    res = torch.randn(M, n_out + 4, device="cuda", generator=gen(5))
    pack = 256 if epi == "swiglu" else 0
    y = res.clone() if epi == "residual" else torch.zeros(M, n_out + 4, device="cuda", dtype=out_dt)
    L.gemv_rows(w, x, y, M=M, N=N, K=K, ldx=K + 8, ldy=n_out + 4, epilogue=epi, pack=pack,
                residual=y if epi == "residual" else None, ldr=n_out + 4)
    for r in range(M):
        xr = x[r, :K].contiguous()
        yr = res[r, :n_out].clone() if epi == "residual" else torch.zeros(n_out, device="cuda", dtype=out_dt)
        L.gemv(w, xr, yr, N=N, K=K, epilogue=epi, pack=pack, residual=yr if epi == "residual" else None)
        assert torch.equal(y[r, :n_out], yr), f"{name}: row {r}"
    if epi != "residual":
        assert not y[:, n_out:].any()


def test_argmax_rows_equal_single_row_argmax(L):
    M, n = 6, 32000
    logits = torch.randn(M, n + 16, device="cuda", generator=gen(7))
    logits[2, [5, 17000]] = 10.0                                   # a tie: the first index wins
    toks = torch.zeros(M, dtype=torch.int32, device="cuda")
    state = torch.tensor([620, 621], dtype=torch.int32, device="cuda")
    L.argmax_rows(logits, n + 16, M, n, toks, advance=state)
    assert state.tolist() == [621, 622]                            # advanced once for the batch
    one = torch.zeros(1, dtype=torch.int32, device="cuda")
    for r in range(M):
        L.argmax(logits[r, :n].contiguous(), n, one)
        assert int(toks[r]) == int(one)
    assert int(toks[2]) == 5


def test_rope_kv_and_decode_attention_per_sequence(L):
    B, heads, cap, p0 = 5, 4, 700, 650
    d, dt = heads * 128, L.operand_dtype()
    qkv = torch.randn(B, 3 * d, device="cuda", generator=gen(3))
    kc = (torch.randn(B, cap, heads, 128, device="cuda", generator=gen(4)) * 2).to(dt)
    vc = torch.randn(B, cap, heads, 128, device="cuda", generator=gen(5)).to(dt)
    q = torch.zeros(B, d, device="cuda", dtype=dt)
    pos = torch.tensor([p0], dtype=torch.int32, device="cuda")
    length = torch.tensor([p0 + 1], dtype=torch.int32, device="cuda")
    kc1, vc1 = kc.clone(), vc.clone()
    L.rope_kv_seqs(qkv, 3 * d, B, heads, pos, q, d, kc, vc, cap * heads * 128)
    ws = torch.empty(B * L.attention_decode_ws_bytes(heads, cap), dtype=torch.uint8, device="cuda")
    out = torch.zeros(B, d, device="cuda", dtype=dt)
    L.attention_decode_seqs(q, d, kc, vc, cap * heads * 128, B, heads, cap, length, ws, out, d)
    ws1 = torch.empty(L.attention_decode_ws_bytes(heads, cap), dtype=torch.uint8, device="cuda")
    for b in range(B):
        qb = torch.zeros(1, d, device="cuda", dtype=dt)
        L.rope_kv(qkv[b:b + 1], 3 * d, 1, heads, pos, qb, d, kc1[b], vc1[b])
        assert torch.equal(q[b], qb[0]) and torch.equal(kc[b], kc1[b]) and torch.equal(vc[b], vc1[b])
        ob = torch.zeros(d, device="cuda", dtype=dt)
        L.attention_decode(qb, kc1[b], vc1[b], heads, cap, length, ws1, ob)
        assert torch.equal(out[b], ob), b


@pytest.fixture(scope="module")
def small_engine(L, golden_dir):
    from diffbir_b200.engine.llava import LlavaEngine
    from tests.test_llava import fixture_cfg, fixture_sd
    f = dict(np.load(golden_dir / "llava_small.npz"))
    return LlavaEngine(fixture_sd(f), f["input_ids"].tolist(), fixture_cfg(f), device="cuda", max_new_tokens=16), f


def test_batched_decode_equals_single_image_engine(small_engine):
    eng, f = small_engine
    from tests.test_llava import fixture_pixels
    xs = [fixture_pixels(f).cuda()] + [torch.rand(1, 3, 336, 336, generator=torch.Generator().manual_seed(s)).cuda()
                                       for s in (9, 10)]
    toks = f["tokens"].tolist()[:8]
    batched = eng.forced_logits_seqs(xs, [toks] * 3)
    for b, x in enumerate(xs):
        assert torch.equal(batched[:, b], eng.forced_logits(x, toks)[1:]), b
    singles = [eng.generate(x) for x in xs]
    assert eng.generate_list(xs) == singles
    assert eng.generate_list(xs[::-1], use_graphs=False) == singles[::-1]
    assert eng.generate_list(xs[:2]) == singles[:2]                # a smaller batch on the same buffers
    print(f"batched LLaVA decode: tokens {singles}")


def test_brownian_samples_equal_per_slice_trees(L):
    from diffbir_b200.sampler.edm import brownian_depth
    lo, hi = 0.03, 14.6
    depth = brownian_depth(lo, hi)
    seeds = [3, 2 ** 62 + 11, 0, 123456789]
    out = torch.empty(4, 4, 40, 24, device="cuda")
    L.brownian_increment_samples(out, torch.tensor(seeds, dtype=torch.int64, device="cuda"), lo, hi, 0.5, 7.25, depth)
    for b, s in enumerate(seeds):
        one = torch.empty(1, 4, 40, 24, device="cuda")
        L.brownian_increment(one, s, lo, hi, 0.5, 7.25, depth)
        assert torch.equal(out[b:b + 1], one), b
    assert not torch.equal(out[0], out[1])
