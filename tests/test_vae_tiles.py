"""Tiled VAE, host side (no GPU): the tile planner and the oracle (tests/tilevae_oracle.py) against the reference's own Tiled-VAE hook
(tests/golden/tilevae_small.npz, tests/golden/gen_golden_tilevae.py), the GroupNorm merge formula, and the
pipeline's tiling decisions."""
import numpy as np
import pytest
import torch

from diffbir_b200 import arch
from diffbir_b200.engine.vae_tiled import plan_vae_tiles
from diffbir_b200.pipeline import vae_tiling
from diffbir_b200.utils.synth import make_state_dict
from tests import tilevae_oracle as otv
from tests.small_cfg import VAE_SMALL


@pytest.fixture(scope="module")
def fx(golden_dir):
    return np.load(golden_dir / "tilevae_small.npz")


def _rel_rms(x, ref):
    x, ref = torch.as_tensor(x).double(), torch.as_tensor(ref).double()
    return ((x - ref).pow(2).mean().sqrt() / ref.pow(2).mean().sqrt()).item()


def test_planner_matches_the_reference_split(fx):
    cases = [k[:-3] for k in fx.files if k.startswith("plan_") and k.endswith("_in")]
    assert len(cases) >= 100
    for key in cases:
        _, side, h, w, t = key.split("_")
        dec = side == "dec"
        plan = plan_vae_tiles(int(h), int(w), int(t), dec)
        assert plan.in_boxes == [tuple(r) for r in fx[key + "_in"].tolist()], key
        assert plan.out_boxes == [tuple(r) for r in fx[key + "_out"].tolist()], key
        ins, outs = otv.split_tiles(int(h), int(w), int(t), dec)
        assert ins == fx[key + "_in"].tolist() and outs == fx[key + "_out"].tolist(), key
        # shape classes partition the tiles, row-major inside each class
        seen = sorted(i for tiles in plan.classes.values() for i in tiles)
        assert seen == list(range(len(plan.in_boxes)))
        for (th, tw), tiles in plan.classes.items():
            assert tiles == sorted(tiles)
            for i in tiles:
                x0, x1, y0, y1 = plan.in_boxes[i]
                assert (y1 - y0, x1 - x0) == (th, tw)
        # output boxes tile the output exactly once
        s = 8 if dec else 1 / 8
        cover = np.zeros((int(int(h) * s), int(int(w) * s)), np.int32)
        for x0, x1, y0, y1 in plan.out_boxes:
            cover[y0:y1, x0:x1] += 1
        assert (cover == 1).all(), key


def test_fixture_inputs_are_fp16_exact(fx):
    for case in ("enc_a", "enc_b", "enc_fallback", "dec_a", "dec_b"):
        x = otv.fixture_source(fx, case)
        assert torch.equal(x.half().float(), x) and x.unique().numel() > 1000


def test_planner_ragged_classes():
    plan = plan_vae_tiles(200, 328, 64, False)
    assert len(plan.in_boxes) == 15 and len(plan.classes) == 4
    plan = plan_vae_tiles(26, 37, 8, True)
    assert any(tw % 2 == 1 or th % 2 == 1 for th, tw in plan.classes)     # odd latent widths reach the engine


@pytest.mark.parametrize("case", ["enc_a", "enc_b", "enc_fallback", "dec_a", "dec_b"])
def test_oracle_matches_the_reference_hook(fx, case):
    """Both sides in fp64 (the fixture is stored in fp32): what remains is the semantics, not rounding."""
    sd = {k: v.double() for k, v in make_state_dict(arch.vae_shapes(VAE_SMALL), 3).items()}
    t = int(fx[case + "_tile"])
    if case.startswith("enc"):
        out = otv.vae_encode_moments_tiled(sd, otv.fixture_source(fx, case).double(), t)
        ref = fx[case + "_moments"]
    else:
        st = int(fx["dec_stride"])
        out = otv.vae_decode_tiled(sd, otv.fixture_source(fx, case).double(), t)[..., ::st, ::st]
        ref = fx[case + "_dec"]
    assert tuple(out.shape) == ref.shape
    e = _rel_rms(out, ref)
    print(f"{case}: oracle vs reference rel-rms {e:.2e}")
    assert e <= 1e-6


def test_tiled_semantics_differ_from_untiled(fx):
    """The fixture is able to tell the tiled semantics from the un-tiled network."""
    from oracle import cldm as ocl
    sd = make_state_dict(arch.vae_shapes(VAE_SMALL), 3)
    img = otv.fixture_source(fx, "enc_a")
    assert _rel_rms(ocl.vae_encode_moments(sd, img), fx["enc_a_moments"]) > 4e-2
    st = int(fx["dec_stride"])
    z = otv.fixture_source(fx, "dec_a")
    assert _rel_rms(ocl.vae_decode(sd, z)[..., ::st, ::st], fx["dec_a_dec"]) > 4e-2


def merge_np(means, variances, pixels, reverse):
    """float64 NumPy restatement of the tiled GroupNorm statistics (tilevae.py:263-278)."""
    order = list(range(len(pixels)))[::-1] if reverse else list(range(len(pixels)))
    wts = np.asarray(pixels, np.float64) / np.sum(pixels, dtype=np.float64)
    mean = sum(wts[t] * np.asarray(means[t], np.float64) for t in order)
    var = sum(wts[t] * np.asarray(variances[t], np.float64) for t in order)
    return mean, var


def test_merge_formula_has_no_between_tile_term():
    g = torch.Generator().manual_seed(5)
    tiles = [torch.randn(2, 64, hh, ww, generator=g) * (1 + t) + 3 * t for t, (hh, ww) in
             enumerate([(7, 9), (7, 4), (3, 9), (3, 4)])]
    vm = [torch.var_mean(x.reshape(2, 32, -1), dim=2, unbiased=False) for x in tiles]
    pixels = [x.shape[2] * x.shape[3] for x in tiles]
    for reverse in (False, True):
        mean, var = otv.merge([m for _, m in vm], [v for v, _ in vm], pixels, reverse)
        rm, rv = merge_np([m.numpy() for _, m in vm], [v.numpy() for v, _ in vm], pixels, reverse)
        np.testing.assert_allclose(mean.numpy(), rm, rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(var.numpy(), rv, rtol=1e-6, atol=1e-6)
    # the pooled statistics of the whole image: the mean agrees, the variance lacks the spread of the tile means
    flat = torch.cat([x.reshape(2, 32, -1) for x in tiles], 2).double()
    pv, pm = torch.var_mean(flat, dim=2, unbiased=False)
    np.testing.assert_allclose(rm, pm.numpy(), rtol=1e-6, atol=1e-6)
    between = sum(p / sum(pixels) * (m.double().numpy() - pm.numpy()) ** 2 for p, (_, m) in zip(pixels, vm))
    np.testing.assert_allclose(rv + between, pv.numpy(), rtol=1e-6, atol=1e-6)
    assert (between > 0.1).all()


def test_pipeline_tiling_decisions():
    # a tile smaller than the image tiles; an image smaller than a tile does not (pipeline.py:105-111, 219-224)
    assert vae_tiling((1024, 768), True, 512, True, 512) == (True, True)
    assert vae_tiling((1024, 768), True, 1024, True, 1024) == (False, False)
    assert vae_tiling((512, 768), True, 768, True, 519) == (False, True)       # the decoder compares 512 // 8, 519 // 8
    assert vae_tiling((512, 768), True, 768, True, 520) == (False, False)
    assert vae_tiling((512, 768), False, 256, False, 256) == (False, False)
    with pytest.raises(ValueError, match="multiple of 8"):
        vae_tiling((1024, 1024), True, 516, False, 512)
    # a tile size that is not a multiple of 8 is accepted when the image is smaller than the tile (tiling is off)
    assert vae_tiling((512, 512), True, 1020, False, 512) == (False, False)
