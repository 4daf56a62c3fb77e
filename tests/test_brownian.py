"""The Brownian tree behind `--sampler edm_dpm++_sde` without torchsde (csrc/brownian.cu), restated in NumPy
(tests/brownian_oracle.py): its Philox stream against Random123's known answers, the statistics of the path it
defines, and the sampler's host logic around it (seed, interval, depth, sign and scaling) with the restatement in
place of the kernel."""
import sys

import numpy as np
import pytest
import torch
from scipy import stats

from tests import brownian_oracle as bo
from diffbir_b200.model.gaussian_diffusion import Diffusion
from diffbir_b200.sampler import edm

N = 100_000


def ladder(version="v2.1", steps=10):
    """EDMSampler's sigma ladder (descending, final 0) for the v2 / v2.1 diffusion settings."""
    d = Diffusion(linear_start=0.00085, linear_end=0.0120, parameterization="v" if version == "v2.1" else "eps",
                  zero_snr=version == "v2.1")
    s = edm.EDMSampler(d.betas, d.parameterization, False, "edm_dpm++_sde", 0, 0, 300, 1, 1, 1)
    s.make_schedule(steps)
    return s.sigmas


def tree_of(sig):
    lo, hi = float(sig[sig > 0].min()), float(sig.max())
    return lo, hi, bo.tree_depth(lo, hi)


@pytest.mark.parametrize("ctr,key,expect", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, expect):
    """Random123's kat_vectors for philox4x32 with 10 rounds."""
    assert tuple(int(w) for w in bo.philox4x32_10(ctr, key)) == expect


@pytest.mark.parametrize("version", ["v2", "v2.1"])
@pytest.mark.parametrize("steps", [4, 10, 50])
def test_depth_for_the_v2_ladders(version, steps):
    """sigma_max is about 1e4 (alpha_bar of the first step forced to 1e-8), so 34 levels bring the leaves under 1e-6."""
    lo, hi, depth = tree_of(ladder(version, steps))
    assert edm.brownian_depth(lo, hi) == depth == 34
    assert (hi - lo) / 2 ** depth <= edm.BROWNIAN_TOL < (hi - lo) / 2 ** (depth - 1)


def test_draws_are_standard_normal():
    z = bo.draw(N, seed=12345, node=7)
    assert stats.kstest(z, "norm").pvalue > 1e-3
    zl = bo.draw(N, seed=12345, node=7, leaf=True, t=0.5)
    assert stats.kstest(zl, "norm").pvalue > 1e-3
    assert abs(np.corrcoef(z, zl)[0, 1]) < 5 / N ** 0.5


def test_increments_are_normal_with_the_interval_as_variance():
    sig = ladder("v2.1", 10)
    lo, hi, depth = tree_of(sig)
    s = sig.double().numpy()
    node1 = 0.5 * (lo + hi)                                       # exactly on a dyadic node
    # (the last interval spans a few 1e-6 leaves: two times inside ONE leaf get independent bridge draws, the
    # tolerance below which the tree, like torchsde's, only approximates a Brownian path)
    for a, b in [(s[5], s[4]), (lo, s[8]), (lo, hi), (node1, hi), (s[1], node1), (s[8], s[8] + 3e-6)]:
        a, b = min(a, b), max(a, b)
        w = bo.increment(N, 99, lo, hi, a, b, depth).astype(np.float64)
        assert stats.kstest(w / np.sqrt(b - a), "norm").pvalue > 1e-3, (a, b)


def test_disjoint_increments_are_uncorrelated():
    sig = ladder("v2.1", 10)
    lo, hi, depth = tree_of(sig)
    s = sig.double().numpy()
    w1 = bo.increment(N, 7, lo, hi, s[4], s[3], depth)
    w2 = bo.increment(N, 7, lo, hi, s[3], s[2], depth)
    w3 = bo.increment(N, 7, lo, hi, s[8], s[7], depth)
    for u, v in [(w1, w2), (w1, w3), (w2, w3)]:
        assert abs(np.corrcoef(u, v)[0, 1]) < 5 / N ** 0.5


@pytest.mark.parametrize("i", [0, 4, 8])
def test_the_two_queries_of_a_dpmpp_sde_step_share_one_path(i):
    """Step i queries [sigma_i, sigma_mid] and [sigma_i, sigma_next] (sigma_mid = sqrt(sigma_i sigma_next)): the
    correlation of the two increments is sqrt(delta_mid / delta_step)."""
    sig = ladder("v2.1", 10)
    lo, hi, depth = tree_of(sig)
    s_i, s_n = sig[i], sig[i + 1]
    s_mid = edm._sig(edm._lam(s_i) + (edm._lam(s_n) - edm._lam(s_i)) / 2)
    s_i, s_n, s_mid = float(s_i), float(s_n), float(s_mid)
    w_mid = bo.increment(N, 31, lo, hi, s_mid, s_i, depth)
    w_step = bo.increment(N, 31, lo, hi, s_n, s_i, depth)
    rho = np.sqrt((s_i - s_mid) / (s_i - s_n))
    se = (1 - rho ** 2) / np.sqrt(N)
    assert abs(np.corrcoef(w_mid, w_step)[0, 1] - rho) < 5 * se + 1e-4
    # and the second draw is the first plus an independent remainder
    rest = w_step.astype(np.float64) - w_mid
    assert abs(np.corrcoef(w_mid, rest)[0, 1]) < 5 / N ** 0.5


def test_additivity_to_fp32_rounding():
    sig = ladder("v2", 10)
    lo, hi, depth = tree_of(sig)
    s = sig.double().numpy()
    n = 20_000
    for a, b, c in [(s[6], s[5], s[4]), (lo, s[5], hi), (s[9], s[9] + 2e-7, s[9] + 5e-7), (lo, 0.5 * (lo + hi), hi)]:
        ab, bc, ac = (bo.increment(n, 5, lo, hi, p, q, depth).astype(np.float64) for p, q in [(a, b), (b, c), (a, c)])
        bound = 2 * np.finfo(np.float32).eps * (np.abs(ab) + np.abs(bc) + np.abs(ac))
        assert np.all(np.abs(ab + bc - ac) <= bound), (a, b, c)


def test_query_semantics():
    lo, hi, depth = 0.03, 1.0e4, 34
    n = 64
    assert np.all(bo.point(n, 3, lo, hi, lo, depth) == 0)
    assert np.array_equal(bo.point(n, 3, lo, hi, hi, depth), np.sqrt(hi - lo) * bo.draw(n, 3, 0))
    mid = 0.5 * (lo + hi)                                           # node 1 of the bisection
    assert np.array_equal(bo.point(n, 3, lo, hi, mid, depth),
                          bo._bridge(lo, hi, 0.0, np.sqrt(hi - lo) * bo.draw(n, 3, 0), mid, bo.draw(n, 3, 1)))
    assert np.array_equal(bo.increment(n, 3, lo, hi, 5.0, 7.0, depth), bo.increment(n, 3, lo, hi, 5.0, 7.0, depth))
    assert np.array_equal(bo.increment(n, 3, lo, hi, 5.0, 7.0, depth), -bo.increment(n, 3, lo, hi, 7.0, 5.0, depth))
    assert np.array_equal(bo.increment(10, 3, lo, hi, 5.0, 7.0, depth), bo.increment(n, 3, lo, hi, 5.0, 7.0, depth)[:10])
    assert np.all(bo.increment(n, 3, lo, hi, 5.0, 5.0, depth) == 0)
    assert not np.array_equal(bo.increment(n, 4, lo, hi, 5.0, 7.0, depth), bo.increment(n, 3, lo, hi, 5.0, 7.0, depth))
    # queries just outside [lo, hi] (sigma_fn(t_fn(sigma)) need not return sigma exactly) read the end values
    assert np.array_equal(bo.point(n, 3, lo, hi, hi * (1 + 1e-7), depth), bo.point(n, 3, lo, hi, hi, depth))


def _stub_denoiser(x, sigma):
    return x / (1 + sigma[:, None, None, None] ** 2) ** 0.5 * 0.3


HP = dict(eta=1.0, s_noise=1.0)


def test_run_rule_dpmpp_sde_on_the_restated_tree(monkeypatch):
    """Without torchsde, run_rule("dpm++_sde") builds its noise from DeviceBrownianTree; with the restatement in its
    place the whole host path runs here: it is deterministic under a fixed seed and follows the seed."""
    monkeypatch.setitem(sys.modules, "torchsde", None)
    made = []

    class Tree(bo.RestatedTree):
        def __init__(self, *a):
            super().__init__(*a)
            made.append(self)

    monkeypatch.setattr(edm, "DeviceBrownianTree", Tree)
    sig = ladder("v2.1", 6)
    x = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(0)) * float(sig[0])

    def run(seed):
        torch.manual_seed(seed)
        return edm.run_rule("dpm++_sde", _stub_denoiser, x.clone(), sig, HP)

    a, b, c = run(1), run(1), run(2)
    assert torch.isfinite(a).all() and a.std() > 0
    assert torch.equal(a, b) and not torch.equal(a, c)
    t = made[0]
    assert (t.lo, t.hi, t.depth) == (float(sig[sig > 0].min()), float(sig.max()), 34)
    torch.manual_seed(1)
    assert t.seed == torch.randint(0, 2 ** 63 - 1, []).item()          # k-diffusion's draw, from the CPU generator


def test_run_rule_dpmpp_sde_noise_matches_the_restatement(monkeypatch):
    """The noise the rule adds is k-diffusion's BrownianTreeNoiseSampler on the tree: sign rule and 1/sqrt|t1 - t0|."""
    monkeypatch.setitem(sys.modules, "torchsde", None)
    monkeypatch.setattr(edm, "DeviceBrownianTree", bo.RestatedTree)
    sig = ladder("v2.1", 4)
    x = torch.zeros(1, 4, 4, 4)
    torch.manual_seed(5)
    sample = edm._brownian_noise(x, sig, "dpm++_sde")
    torch.manual_seed(5)
    seed = torch.randint(0, 2 ** 63 - 1, []).item()
    lo, hi, depth = tree_of(sig)
    s0, s1 = sig[1], sig[2]
    got = sample(s0, s1)
    want = -bo.increment(x.numel(), seed, lo, hi, float(s1), float(s0), depth) / np.sqrt(float(s0 - s1))
    assert np.allclose(got.numpy().ravel(), want, rtol=1e-6, atol=0)
    assert np.allclose(got.std().item(), 1.0, atol=0.5)


def test_disjoint_rules_keep_their_randn_fallback(monkeypatch):
    """dpm++_2m_sde / 3m_sde without torchsde still draw randn_like and take nothing from the CPU generator here."""
    monkeypatch.setitem(sys.modules, "torchsde", None)
    sig = ladder("v2.1", 4)
    torch.manual_seed(3)
    before = torch.get_rng_state()
    for solver in ("dpm++_2m_sde", "dpm++_3m_sde"):
        assert edm._brownian_noise(torch.zeros(1, 4, 4, 4), sig, solver) is None
    assert torch.equal(before, torch.get_rng_state())


def test_device_tree_refuses_a_cpu_latent(monkeypatch):
    monkeypatch.setitem(sys.modules, "torchsde", None)
    with pytest.raises(ValueError, match="CUDA"):
        edm.run_rule("dpm++_sde", _stub_denoiser, torch.zeros(1, 4, 4, 4), ladder("v2.1", 4), HP)
