"""-m gpu: the tiled VAE (engine.vae_tiled.TiledVae) against the reference's Tiled-VAE hook (fixture
tests/golden/tilevae_small.npz) and against the oracle (tests/tilevae_oracle.py); its two kernels (dbir_gn_moments,
dbir_gn_merge) against float64 references; bit-identity across state staging and wave grouping; the pipeline with
both VAE tiling flags; a 4096^2 full-config restoration on one GPU."""
import gc

import numpy as np
import pytest
import torch

from diffbir_b200 import arch
from diffbir_b200.utils.synth import RUN_DEFAULTS, build_synthetic_pipeline, make_state_dict, synthetic_lq
from tests import tilevae_oracle as otv
from tests.gpu_util import no_tf32, rel_rms, to_dev
from tests.small_cfg import VAE_SMALL

pytestmark = pytest.mark.gpu
# relative RMS error of one network forward with fp16 operands (test_gpu_engines.py); bf16 operands round 8x coarser
TOL16 = 4e-3


def _tol():
    from diffbir_b200 import lib
    return TOL16 * (1 if lib.operand_dtype() == torch.float16 else 8)


@pytest.fixture(scope="module")
def fx(golden_dir):
    return np.load(golden_dir / "tilevae_small.npz")


@pytest.fixture(scope="module")
def small():
    from diffbir_b200.engine.vae import VaeEngine
    from diffbir_b200.engine.vae_tiled import TiledVae
    no_tf32()
    sd = make_state_dict(arch.vae_shapes(VAE_SMALL), 3)
    base = VaeEngine(sd, VAE_SMALL, "cuda")
    return base, TiledVae(base), sd


# ---- kernels ---------------------------------------------------------------------------------------------------------
def _moments64(x, n, hw, c):
    xv = x.double().view(n, hw, 32, c // 32)
    var, mean = torch.var_mean(xv, dim=(1, 3), unbiased=False)
    return torch.stack([mean, var], -1)                                    # [n, 32, 2]


@pytest.mark.parametrize("h,w,c", [(7, 9, 64), (13, 38, 128), (38, 24, 256), (5, 3, 512)])
def test_gn_moments_contract(h, w, c):
    """Both sources (fp32 tensor; the partial sums of a conv-mode GEMM where gemm_gn_slots allows them), written at
    scattered entry indices, against float64 moments of the same fp32 tensor."""
    from diffbir_b200 import lib
    n, hw = 3, h * w
    g = torch.Generator(device="cuda").manual_seed(h * w + c)
    x = (torch.randn(n * hw, c, device="cuda", generator=g) * 3 + torch.linspace(-2, 5, c, device="cuda"))
    entry = torch.tensor([5, 0, 3], dtype=torch.int32, device="cuda")
    mom = torch.full((6, 32, 2), float("nan"), dtype=torch.float64, device="cuda")
    ws = torch.empty(lib.gn_moments_workspace_floats(n, hw, c), device="cuda")
    lib.gn_moments(c, n, hw, mom, x=x, workspace=ws, entry=entry)
    ref = _moments64(x, n, hw, c)
    got = mom[entry.long()]
    # fp32 slot sums of <= 32 pixels, fp64 beyond: error ~ 32 ulp of the sums of squares
    assert torch.allclose(got, ref, rtol=1e-5, atol=1e-5), (got - ref).abs().max()
    assert torch.isnan(mom[[1, 2, 4]]).all()                              # untouched entries
    # entry0 form
    mom2 = torch.zeros(n + 2, 32, 2, dtype=torch.float64, device="cuda")
    lib.gn_moments(c, n, hw, mom2, x=x, workspace=ws, entry0=2)
    assert torch.equal(mom2[2:], mom[entry.long()])
    # from a conv-mode GEMM's fused partial sums
    slots = lib.gemm_gn_slots(h, w)
    if slots > 0:
        a16 = torch.randn(n * hw, 64, device="cuda", generator=g).to(lib.operand_dtype())
        wt = (torch.randn(c, 9 * 64, device="cuda", generator=g) * 0.05).to(lib.operand_dtype())
        out = torch.empty(n * hw, c, device="cuda")
        part = torch.empty(n * slots * c * 2, device="cuda")
        lib.gemm(a16, wt, out, M=n * hw, N=c, K=9 * 64, conv=(n, h, w, 64, 3), split_k=1, gn_partials=part)
        mom3 = torch.empty(n, 32, 2, dtype=torch.float64, device="cuda")
        lib.gn_moments(c, n, hw, mom3, partials=part, slots=slots)
        ref3 = _moments64(out, n, hw, c)
        assert torch.allclose(mom3, ref3, rtol=1e-5, atol=1e-6), (mom3 - ref3).abs().max()


def test_gn_merge_contract():
    """Pixel-weighted means of the entries' moments per image, no between-tile term, against float64 NumPy; entries
    of two images interleaved; reverse order changes at most the last bits."""
    from diffbir_b200 import lib
    g = torch.Generator().manual_seed(9)
    E, images = 7, 2
    image = torch.tensor([0, 1, 0, 1, 0, 1, 0], dtype=torch.int32)
    pixels = torch.tensor([1444, 1444, 912, 912, 576, 576, 1001], dtype=torch.int64)
    mom = torch.stack([torch.randn(E, 32, generator=g, dtype=torch.float64) * 2,
                       torch.rand(E, 32, generator=g, dtype=torch.float64) * 3], -1)
    stats = torch.full((E, 64), float("nan"), device="cuda")
    outs = []
    for rev in (False, True):
        lib.gn_merge(mom.cuda(), pixels.cuda(), image.cuda(), E, images, stats, reverse=rev, eps=1e-6)
        outs.append(stats.clone())
    for img in range(images):
        sel = (image == img).numpy()
        w = pixels.numpy()[sel] / pixels.numpy()[sel].sum()
        m = (w[:, None] * mom.numpy()[sel, :, 0]).sum(0)
        v = (w[:, None] * mom.numpy()[sel, :, 1]).sum(0)
        for st in outs:
            got = st.cpu().view(E, 32, 2).double().numpy()[sel]
            np.testing.assert_allclose(got[..., 0], np.broadcast_to(m, got[..., 0].shape), rtol=1e-6, atol=1e-7)
            np.testing.assert_allclose(got[..., 1], np.broadcast_to(1 / np.sqrt(v + 1e-6), got[..., 1].shape), rtol=1e-6)
    assert (outs[0] - outs[1]).abs().max().item() <= 1e-6


# ---- the engine against the reference and the oracle -----------------------------------------------------------------
@pytest.mark.parametrize("case", ["enc_a", "enc_b", "dec_a", "dec_b"])
def test_small_vs_reference_hook(fx, small, case):
    _, tv, _ = small
    t = int(fx[case + "_tile"])
    if case.startswith("enc"):
        x = otv.fixture_source(fx, case).cuda()
        # a tile larger than the image: the un-tiled network (VaeEngine, or one tile where its attention cannot
        # take the latent's token count)
        out, untiled, ref = tv.encode_moments(x, t), tv.encode_moments(x, 1 << 20), fx[case + "_moments"]
    else:
        st = int(fx["dec_stride"])
        z = otv.fixture_source(fx, case).cuda()
        out, untiled = tv.decode(z, t)[..., ::st, ::st], tv.decode(z, 1 << 20)[..., ::st, ::st]
        ref = fx[case + "_dec"]
    ref = torch.from_numpy(ref).cuda()
    e, eu = rel_rms(out, ref), rel_rms(untiled, ref)
    print(f"{case}: tiled {e:.2e}, un-tiled engine {eu:.2e} vs reference hook")
    # the fixture tells the semantics apart: un-tiled lands > 10x outside the fp16-operand tolerance
    assert e < _tol() and eu > 10 * TOL16


def test_fallback_is_the_untiled_engine(fx, small):
    """Inputs no larger than 2 * pad + tile run un-tiled: through VaeEngine itself where its attention takes the
    latent (token count a multiple of 8), else as one tile through the tiled path."""
    base, tv, _ = small
    x = otv.fixture_source(fx, "enc_fallback").cuda()          # 96 x 120: a 12 x 15 latent
    out = tv.encode_moments(x, int(fx["enc_fallback_tile"]))
    assert tv.last_stats["tiles"] == 1
    e = rel_rms(out, torch.from_numpy(fx["enc_fallback_moments"]).cuda())
    print(f"fallback, one tile: {e:.2e} vs the reference hook")
    assert e < _tol()
    x = x[..., :96].contiguous()                                         # 96 x 96: a 12 x 12 latent
    assert torch.equal(tv.encode_moments(x, 64), base.encode_moments(x))
    z = torch.randn(1, 4, 30, 20, device="cuda")
    assert torch.equal(tv.decode(z, 8), base.decode(z))                  # 30 <= 2 * 11 + 8


@pytest.mark.parametrize("case", ["enc_a", "dec_a"])
def test_spill_and_wave_grouping_bit_identical(fx, small, case):
    """All state on the device against all state staged through the host; one tile per wave against every tile of
    a shape class in one wave."""
    _, tv, _ = small
    t = int(fx[case + "_tile"])
    x = otv.fixture_source(fx, case).cuda()
    fn = tv.encode_moments if case.startswith("enc") else tv.decode
    outs, stats = [], []
    for budget, wave in ((None, 1 << 30), (0, 1 << 30), (None, 1), (0, 1)):
        tv.state_budget, tv.wave_pixels = budget, wave
        outs.append(fn(x, t))
        stats.append(dict(tv.last_stats))
    tv.state_budget, tv.wave_pixels = None, type(tv).wave_pixels
    print(case, stats)
    assert stats[0]["spills"] == 0 and stats[1]["spills"] > 0 and stats[3]["spills"] > 0
    assert stats[0]["waves"] < stats[2]["waves"] == stats[0]["tiles"]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


def test_full_config_vs_oracle_ragged():
    """Full SD VAE, 768 x 1280 image with 256-pixel encoder tiles, and its 96 x 160 latent with 256-pixel decoder
    tiles, against the fp32 oracle on the same device."""
    from diffbir_b200.engine.vae import VaeEngine
    from diffbir_b200.engine.vae_tiled import TiledVae
    no_tf32()
    sd = make_state_dict(arch.vae_shapes(arch.VAE_CFG), 77)
    tv = TiledVae(VaeEngine(sd, arch.VAE_CFG, "cuda"))
    sdd = to_dev(sd)
    g = torch.Generator().manual_seed(5)
    img = (torch.rand(1, 3, 768, 1280, generator=g) * 2 - 1).cuda()
    z = (torch.randn(1, 4, 96, 160, generator=g) * 0.8).cuda()
    mom = tv.encode_moments(img, 256)
    enc_stats = dict(tv.last_stats)
    dec = tv.decode(z, 256 // 8)
    with torch.no_grad():
        rmom = otv.vae_encode_moments_tiled(sdd, img, 256)
        rdec = otv.vae_decode_tiled(sdd, z, 256 // 8)
    e1, e2 = rel_rms(mom, rmom), rel_rms(dec, rdec)
    print(f"full config tiled vs oracle: encode {e1:.2e} ({enc_stats}), decode {e2:.2e} ({tv.last_stats})")
    assert e1 < _tol() and e2 < _tol()


# ---- pipeline --------------------------------------------------------------------------------------------------------
def _psnr_u8(a, b):
    mse = ((a.astype(np.float64) - b.astype(np.float64)) ** 2).mean()
    return float("inf") if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


def test_small_pipeline_both_vae_flags_vs_oracle():
    from oracle import cldm as ocl
    from oracle import sampling as osm
    from oracle import swinir as osw
    no_tf32()
    pipe = build_synthetic_pipeline("cuda", seed=1234, small=True)
    scfg = dict(arch.SWINIR_CFG, depths=(2, 2), num_heads=(6, 6))
    pipe.cleaner.engine_sd = make_state_dict(arch.swinir_shapes(scfg), 1234 + 4)
    lq = synthetic_lq(640, 768, seed=3)            # multiples of 64: the tiled and un-tiled paddings agree
    kw = dict(RUN_DEFAULTS, steps=4, vae_encoder_tiled=True, vae_encoder_tile_size=256, vae_decoder_tiled=True,
              vae_decoder_tile_size=256)
    pipe.taps = {}
    torch.manual_seed(231)
    out = pipe.run(lq, **kw)
    cl = pipe.cldm
    assert cl._tvae is not None and cl._tvae.last_stats["tiles"] > 1
    usd, csd, vsd, clipsd = (to_dev(d) for d in (cl._unet_sd, cl._cn_sd, cl._vae_sd, cl._clip_sd))
    ssd = to_dev(pipe.cleaner.engine_sd)
    scales = {"s": [1.0] * 13}
    torch.manual_seed(231)
    with torch.no_grad():
        ref = osm.swinir_pipeline_run(
            lq, cleaner=lambda im: osw.swinir_forward(ssd, im),
            encode_img=lambda im: otv.vae_encode_moments_tiled(vsd, im, 256)[:, :4] * cl.scale_factor,
            encode_txt=lambda txt: ocl.clip_text_encode(clipsd, cl.tokenize(txt).to("cuda"),
                                                        heads=cl.clip_cfg["text_cfg"]["heads"]),
            decode=lambda z: otv.vae_decode_tiled(vsd, z / cl.scale_factor, 256 // 8),
            model=lambda x, t, c: ocl.cldm_forward(usd, csd, x, t, c["c_txt"], c["c_img"], scales["s"]),
            betas=pipe.diffusion.betas, parameterization=pipe.diffusion.parameterization, steps=kw["steps"],
            strength=kw["strength"], pos_prompt=kw["pos_prompt"], neg_prompt=kw["neg_prompt"],
            cfg_scale=kw["cfg_scale"], sampler=kw["sampler_type"], cldm_tiled=False, rescale_cfg=False,
            device="cuda", set_strength=lambda s: scales.update(s=[s] * 13))
    p = _psnr_u8(out, ref)
    print(f"small pipeline, tiled VAE encode + decode vs oracle: uint8 PSNR {p:.2f} dB")
    # bf16 operands: the un-tiled full pipeline itself lands near 49.5 dB (test_gpu_pipeline.py)
    assert out.shape == ref.shape == lq.shape and p >= (50.0 if cl.vae.op_dtype == torch.float16 else 40.0)


def test_full_config_4096_tiled_vae():
    """SwinIRPipeline at 4096^2 on one GPU: tiled SwinIR, tiled sampling (2 steps), tiled VAE encode and decode
    with 1024-pixel tiles."""
    no_tf32()
    gc.collect()
    torch.cuda.empty_cache()
    pipe = build_synthetic_pipeline("cuda", seed=1234, small=False)
    lq = synthetic_lq(4096, 4096, seed=8)
    kw = dict(RUN_DEFAULTS, steps=2, cldm_tiled=True, cleaner_tiled=True, vae_encoder_tiled=True,
              vae_encoder_tile_size=1024, vae_decoder_tiled=True, vae_decoder_tile_size=1024)
    torch.cuda.reset_peak_memory_stats()
    torch.manual_seed(231)
    out = pipe.run(lq, **kw)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"4096^2 full config, tiled VAE: peak {peak:.1f} GiB on {torch.cuda.get_device_name()}, "
          f"decode {pipe.cldm._tvae.last_stats}")
    assert out.shape == (1, 4096, 4096, 3) and out.dtype == np.uint8 and 0 < out.std()
    del pipe
    gc.collect()
    torch.cuda.empty_cache()
