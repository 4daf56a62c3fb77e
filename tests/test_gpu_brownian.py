"""-m gpu: the device Brownian tree (dbir_brownian_increment / dbir_brownian_draws) against its NumPy restatement
(tests/brownian_oracle.py), and `inference.py --sampler edm_dpm++_sde` end to end with torchsde hidden."""
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from tests import brownian_oracle as bo

pytestmark = pytest.mark.gpu

SEED = 0x5DEECE66DB7A3C21 & (2 ** 63 - 1)
LO, HI = 0.029167, 9999.99995                  # about the v2.1 ladder's ends at 10 steps
DEPTH = bo.tree_depth(LO, HI)                  # 34


def _lib():
    from diffbir_b200 import lib
    lib.load()
    return lib


def device_words(n, node, leaf=False, t=0.0, seed=SEED):
    lib = _lib()
    w = torch.empty(n, 4, dtype=torch.int32, device="cuda")
    z = torch.empty(n, dtype=torch.float64, device="cuda")
    lib.brownian_draws(n, seed, node, leaf=leaf, t=t, words=w, normals=z)
    torch.cuda.synchronize()
    return w.cpu().numpy().view(np.uint32), z.cpu().numpy()


def device_increment(n, t0, t1, seed=SEED, lo=LO, hi=HI, depth=DEPTH):
    lib = _lib()
    out = torch.empty(n, dtype=torch.float32, device="cuda")
    lib.brownian_increment(out, seed, lo, hi, t0, t1, depth)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("n", [1000, 65536 + 37])
@pytest.mark.parametrize("node,leaf,t", [(0, False, 0.0), (1, False, 0.0), (12345, False, 0.0),
                                         (2 ** 34 + 5, False, 0.0), (2 ** 34 + 5, True, 17.25), (3, True, LO)])
def test_draws_match_the_restatement(n, node, leaf, t):
    w, z = device_words(n, node, leaf, t)
    ref_w = np.stack(bo.draw_words(n, SEED, node, leaf, t), 1)
    assert np.array_equal(w, ref_w)                                   # Philox words bit for bit
    ref_z = bo.normal_from_words(bo.draw_words(n, SEED, node, leaf, t))
    err = np.abs(z - ref_z).max()
    print(f"node {node} leaf {leaf}: max |normal - restatement| = {err:.2e}")
    assert err < 1e-10                                                # fp64 Box-Muller, libm vs CUDA rounding


def _ulp_close(got, ref):
    err = np.abs(got.astype(np.float64) - ref.astype(np.float64))
    bound = 2.0 ** -23 * np.abs(ref.astype(np.float64)) + 1e-9       # one fp32 rounding of the difference
    return err.max(), bool(np.all(err <= bound))


NODE1 = 0.5 * (LO + HI)
QUERIES = [(4.0, 7.5), (7.5, 4.0), (LO, HI), (LO, 0.1), (NODE1, HI), (0.5 * (LO + NODE1), NODE1), (123.4, 123.4 + 3e-6),
           (HI * (1 + 1e-7), 50.0)]


@pytest.mark.parametrize("n", [1000, 65536 + 37])
@pytest.mark.parametrize("t0,t1", QUERIES)
def test_increments_match_the_restatement(n, t0, t1):
    got = device_increment(n, t0, t1)
    ref = bo.increment(n, SEED, LO, HI, t0, t1, DEPTH)
    err, ok = _ulp_close(got, ref)
    print(f"[{t0}, {t1}] n={n}: max |kernel - restatement| = {err:.2e}")
    assert ok


def test_repeated_calls_give_identical_bits():
    a = device_increment(65536, 3.0, 900.0)
    for _ in range(3):
        assert np.array_equal(device_increment(65536, 3.0, 900.0), a)


def test_an_element_does_not_depend_on_the_tensor_size():
    big = device_increment(4 * 128 * 128 * 2, 0.5, 80.0)
    for n in (1, 7, 1000, 4 * 64 * 64):
        assert np.array_equal(device_increment(n, 0.5, 80.0), big[:n])


def test_additivity_on_the_device():
    n = 65536
    ab, bc, ac = (device_increment(n, p, q).astype(np.float64) for p, q in [(0.3, 11.0), (11.0, NODE1), (0.3, NODE1)])
    assert np.all(np.abs(ab + bc - ac) <= 2 * np.finfo(np.float32).eps * (np.abs(ab) + np.abs(bc) + np.abs(ac)))


def test_run_rule_on_the_device_tree_matches_the_restated_tree(monkeypatch):
    """The sampler's whole host path on the GPU (seed draw, [min sigma > 0, max sigma], depth, sign, 1/sqrt|dt|)
    against the same run with the restatement as the tree. Both runs do the rule's arithmetic on the device: the
    query times must have the same bits, since the leaf draw is keyed with t (one fp32 ulp of sigma apart, two runs
    would read points of the path 1e-3 apart)."""
    from diffbir_b200.model.gaussian_diffusion import Diffusion
    from diffbir_b200.sampler import edm
    monkeypatch.setitem(sys.modules, "torchsde", None)
    d = Diffusion(linear_start=0.00085, linear_end=0.0120, parameterization="v", zero_snr=True)
    s = edm.EDMSampler(d.betas, "v", False, "edm_dpm++_sde", 0, 0, 300, 1, 1, 1)
    s.make_schedule(6)
    x = torch.randn(2, 4, 16, 16, generator=torch.Generator().manual_seed(0)) * float(s.sigmas[0])

    def den(x, sigma):
        return x / (1 + sigma[:, None, None, None] ** 2) ** 0.5 * 0.3

    hp = dict(eta=1.0, s_noise=1.0)
    torch.manual_seed(11)
    got = edm.run_rule("dpm++_sde", den, x.cuda(), s.sigmas.cuda(), hp).cpu()
    monkeypatch.setattr(edm, "DeviceBrownianTree", bo.RestatedTree)
    torch.manual_seed(11)
    ref = edm.run_rule("dpm++_sde", den, x.cuda(), s.sigmas.cuda(), hp).cpu()
    err = ((got - ref).abs().max() / ref.abs().max()).item()
    print(f"dpm++_sde on the device tree vs the restated tree: max rel err {err:.2e}")
    assert err < 1e-5


def _cli(tmp_path, name, size, extra=()):
    import inference as cli
    from diffbir_b200.utils.synth import synthetic_lq
    src = tmp_path / "in"
    if not src.exists():
        src.mkdir()
        Image.fromarray(synthetic_lq(size[0], size[1], seed=3)[0]).save(src / "img.png")
    cli.main(["--task", "sr", "--version", "v2.1", "--upscale", "4", "--sampler", "edm_dpm++_sde", "--steps", "4",
              "--cfg_scale", "4.0", "--pos_prompt", "", "--neg_prompt", "low quality, blurry", "--captioner", "none",
              "--input", str(src), "--output", str(tmp_path / name), "--synthetic", *extra])
    return np.array(Image.open(tmp_path / name / "img.png"))


def test_cli_edm_dpmpp_sde_without_torchsde(tmp_path, monkeypatch):
    monkeypatch.setitem(sys.modules, "torchsde", None)
    a = _cli(tmp_path, "out1", (128, 160))
    assert a.shape == (512, 640, 3) and a.dtype == np.uint8
    assert a.std() > 1.0                                             # an image, not a constant
    b = _cli(tmp_path, "out2", (128, 160))
    assert np.array_equal(a, b)                                      # same seed, same PNG


def test_cli_edm_dpmpp_sde_tiled_1024(tmp_path, monkeypatch):
    monkeypatch.setitem(sys.modules, "torchsde", None)
    out = _cli(tmp_path, "out", (256, 256), ["--cldm_tiled"])
    assert out.shape == (1024, 1024, 3) and out.dtype == np.uint8 and out.std() > 1.0
