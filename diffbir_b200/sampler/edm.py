"""EDM-formulation samplers — counterpart of the reference's diffbir.sampler.EDMSampler
(sampler/edm_sampler.py:26-186) and of the Karras-ODE / DPM-Solver++ step rules it drives
(sampler/k_diffusion.py:123-306, 514-707; the public k-diffusion algorithms of Karras et al. 2022 and
Lu et al. 2022, restated here as `STEP_RULES`).

The model is evaluated through a *denoiser* D(x, sigma) = c_skip x + c_out F(c_in x, t(sigma))
(edm_sampler.py:98-139); sigma is mapped to the nearest entry of the schedule's own sigma table, so the
network only ever sees the steps+1 integer timesteps of `make_schedule` — which is what lets the kernel
engine pre-compute every time embedding and replay one CUDA graph per evaluation (EngineEval), exactly as
for the spaced / DDIM loops. A foreign `model(x, t, cond)` callable takes the same arithmetic in plain
PyTorch (bit-identical to the reference on the same device; tests/test_oracle_golden.py pins it to
fixtures the reference produced).

Stochastic "SDE" rules draw their noise from torchsde's Brownian tree in the reference
(k_diffusion.py:70-120). torchsde is not a dependency here: when it is importable the same tree is used,
otherwise `dpm++_2m_sde` / `dpm++_3m_sde` (one query per step, disjoint intervals => independent standard
normals, the same distribution) fall back to torch.randn_like, and `dpm++_sde` (two overlapping intervals per
step, whose increments must come from one path) queries `DeviceBrownianTree`: a Brownian tree the engine generates
on the fly from (seed, node, element) (dbir_brownian_increment), with torchsde's tolerance and k-diffusion's
interface (same seed draw, interval [min sigma > 0, max sigma], sign rule and scaling). It has torchsde's
distribution and query semantics, not its random stream.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .sampler import EngineEval, NoiseSource, Sampler, randn, randn_like, tiled_callable


def _bc(v: torch.Tensor, ndim: int) -> torch.Tensor:
    """[B] -> [B, 1, ..., 1] (append_dims, k_diffusion.py:10-15)."""
    return v[(...,) + (None,) * (ndim - v.ndim)]


def _ancestral(sigma_from, sigma_to, eta):
    """(sigma_down, sigma_up) of an ancestral step — k_diffusion.py:56-63."""
    if not eta:
        return sigma_to, 0.0
    up = min(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    return (sigma_to ** 2 - up ** 2) ** 0.5, up


class _Run:
    """One sampling run: the denoiser, the sigma ladder and the noise source shared by every step rule."""

    def __init__(self, denoise: Callable, x: torch.Tensor, sigmas: torch.Tensor, hp: dict, noise: Optional[Callable],
                 source: Optional[NoiseSource] = None):
        self.D, self.x, self.sig, self.hp, self.source = denoise, x, sigmas, hp, source
        self.ones = x.new_ones([x.shape[0]])
        self.noise = noise if noise is not None else (lambda s0, s1: randn_like(self.x, self.source))
        self.n = len(sigmas) - 1

    def den(self, x, sigma):
        return self.D(x, sigma * self.ones)

    def slope(self, x, sigma, denoised):
        """Karras ODE derivative dx/dsigma (to_d, k_diffusion.py:51-53)."""
        return (x - denoised) / _bc(sigma, x.ndim)

    def churn(self, i):
        """Stochastic churn of Algorithm 2 (Karras et al.): returns sigma_hat; x is perturbed in place of
        the trajectory. The noise draw happens every step, churn or not, like the reference."""
        hp, s = self.hp, self.sig
        gamma = min(hp["s_churn"] / self.n, 2 ** 0.5 - 1) if hp["s_tmin"] <= s[i] <= hp["s_tmax"] else 0.0
        eps = randn_like(self.x, self.source) * hp["s_noise"]
        sigma_hat = s[i] * (gamma + 1)
        if gamma > 0:
            self.x = self.x + eps * (sigma_hat ** 2 - s[i] ** 2) ** 0.5
        return sigma_hat


# ---- step rules: each advances run.x from sigmas[i] to sigmas[i+1] -----------------------------------
def _euler(r: _Run, i: int):
    sh = r.churn(i)
    d = r.slope(r.x, sh, r.den(r.x, sh))
    r.x = r.x + d * (r.sig[i + 1] - sh)


def _euler_a(r: _Run, i: int):
    s = r.sig
    den = r.den(r.x, s[i])
    down, up = _ancestral(s[i], s[i + 1], r.hp["eta"])
    d = r.slope(r.x, s[i], den)
    r.x = r.x + d * (down - s[i])
    if s[i + 1] > 0:
        r.x = r.x + r.noise(s[i], s[i + 1]) * r.hp["s_noise"] * up


def _heun(r: _Run, i: int):
    s = r.sig
    sh = r.churn(i)
    d = r.slope(r.x, sh, r.den(r.x, sh))
    dt = s[i + 1] - sh
    if s[i + 1] == 0:
        r.x = r.x + d * dt
        return
    x2 = r.x + d * dt
    d2 = r.slope(x2, s[i + 1], r.den(x2, s[i + 1]))
    r.x = r.x + ((d + d2) / 2) * dt


def _dpm2(r: _Run, i: int):
    s = r.sig
    sh = r.churn(i)
    d = r.slope(r.x, sh, r.den(r.x, sh))
    if s[i + 1] == 0:
        r.x = r.x + d * (s[i + 1] - sh)
        return
    mid = sh.log().lerp(s[i + 1].log(), 0.5).exp()
    x2 = r.x + d * (mid - sh)
    d2 = r.slope(x2, mid, r.den(x2, mid))
    r.x = r.x + d2 * (s[i + 1] - sh)


def _dpm2_a(r: _Run, i: int):
    s = r.sig
    den = r.den(r.x, s[i])
    down, up = _ancestral(s[i], s[i + 1], r.hp["eta"])
    d = r.slope(r.x, s[i], den)
    if down == 0:
        r.x = r.x + d * (down - s[i])
        return
    mid = s[i].log().lerp(down.log(), 0.5).exp()
    x2 = r.x + d * (mid - s[i])
    d2 = r.slope(x2, mid, r.den(x2, mid))
    r.x = r.x + d2 * (down - s[i])
    r.x = r.x + r.noise(s[i], s[i + 1]) * r.hp["s_noise"] * up


def _lms_weight(order: int, t: np.ndarray, i: int, j: int) -> float:
    """Integral over [t_i, t_{i+1}] of the j-th Lagrange basis through the last `order` nodes
    (linear_multistep_coeff, k_diffusion.py:252-263; same quadrature tolerance)."""
    from scipy import integrate
    if order - 1 > i:
        raise ValueError(f"Order {order} too high for step {i}")

    def basis(tau):
        p = 1.0
        for k in range(order):
            if k != j:
                p *= (tau - t[i - k]) / (t[i - j] - t[i - k])
        return p
    return integrate.quad(basis, t[i], t[i + 1], epsrel=1e-4)[0]


def _lms(r: _Run, i: int):
    s = r.sig
    if i == 0:
        r.hist, r.sig_np = [], s.detach().cpu().numpy()
    d = r.slope(r.x, s[i], r.den(r.x, s[i]))
    r.hist.append(d)
    if len(r.hist) > r.hp["order"]:
        r.hist.pop(0)
    k = min(i + 1, r.hp["order"])
    w = [_lms_weight(k, r.sig_np, i, j) for j in range(k)]
    r.x = r.x + sum(c * dd for c, dd in zip(w, reversed(r.hist)))


def _lam(sigma):          # t = -log sigma ("lambda" of DPM-Solver++ in the sigma parameterisation)
    return sigma.log().neg()


def _sig(t):
    return t.neg().exp()


def _dpmpp_2s_a(r: _Run, i: int):
    s = r.sig
    den = r.den(r.x, s[i])
    down, up = _ancestral(s[i], s[i + 1], r.hp["eta"])
    if down == 0:
        d = r.slope(r.x, s[i], den)
        r.x = r.x + d * (down - s[i])
    else:
        t, t_next = _lam(s[i]), _lam(down)
        rr = 1 / 2
        h = t_next - t
        mid = t + rr * h
        x2 = (_sig(mid) / _sig(t)) * r.x - (-h * rr).expm1() * den
        den2 = r.den(x2, _sig(mid))
        r.x = (_sig(t_next) / _sig(t)) * r.x - (-h).expm1() * den2
    if s[i + 1] > 0:
        r.x = r.x + r.noise(s[i], s[i + 1]) * r.hp["s_noise"] * up


def _dpmpp_sde(r: _Run, i: int, rr: float = 1 / 2):
    s, eta, s_noise = r.sig, r.hp["eta"], r.hp["s_noise"]
    den = r.den(r.x, s[i])
    if s[i + 1] == 0:
        d = r.slope(r.x, s[i], den)
        r.x = r.x + d * (s[i + 1] - s[i])
        return
    t, t_next = _lam(s[i]), _lam(s[i + 1])
    h = t_next - t
    mid = t + h * rr
    fac = 1 / (2 * rr)
    sd, su = _ancestral(_sig(t), _sig(mid), eta)
    m_ = _lam(sd)
    x2 = (_sig(m_) / _sig(t)) * r.x - (t - m_).expm1() * den
    x2 = x2 + r.noise(_sig(t), _sig(mid)) * s_noise * su
    den2 = r.den(x2, _sig(mid))
    sd, su = _ancestral(_sig(t), _sig(t_next), eta)
    n_ = _lam(sd)
    dd = (1 - fac) * den + fac * den2
    r.x = (_sig(n_) / _sig(t)) * r.x - (t - n_).expm1() * dd
    r.x = r.x + r.noise(_sig(t), _sig(t_next)) * s_noise * su


def _dpmpp_2m(r: _Run, i: int):
    s = r.sig
    if i == 0:
        r.prev = None
    den = r.den(r.x, s[i])
    t, t_next = _lam(s[i]), _lam(s[i + 1])
    h = t_next - t
    if r.prev is None or s[i + 1] == 0:
        r.x = (_sig(t_next) / _sig(t)) * r.x - (-h).expm1() * den
    else:
        ratio = (t - _lam(s[i - 1])) / h
        dd = (1 + 1 / (2 * ratio)) * den - (1 / (2 * ratio)) * r.prev
        r.x = (_sig(t_next) / _sig(t)) * r.x - (-h).expm1() * dd
    r.prev = den


def _dpmpp_2m_sde(r: _Run, i: int):
    s, eta = r.sig, r.hp["eta"]
    if i == 0:
        r.prev, r.h_prev = None, None
    den = r.den(r.x, s[i])
    if s[i + 1] == 0:
        r.x = den
        h = None
    else:
        t, u = -s[i].log(), -s[i + 1].log()
        h = u - t
        eh = eta * h
        r.x = s[i + 1] / s[i] * (-eh).exp() * r.x + (-h - eh).expm1().neg() * den
        if r.prev is not None:
            ratio = r.h_prev / h
            r.x = r.x + 0.5 * (-h - eh).expm1().neg() * (1 / ratio) * (den - r.prev)      # 'midpoint' variant
        if eta:
            r.x = r.x + r.noise(s[i], s[i + 1]) * s[i + 1] * (-2 * eh).expm1().neg().sqrt() * r.hp["s_noise"]
    r.prev, r.h_prev = den, h


def _dpmpp_3m_sde(r: _Run, i: int):
    s, eta = r.sig, r.hp["eta"]
    if i == 0:
        r.d1 = r.d2 = r.h1 = r.h2 = None
    den = r.den(r.x, s[i])
    h = None
    if s[i + 1] == 0:
        r.x = den
    else:
        t, u = -s[i].log(), -s[i + 1].log()
        h = u - t
        he = h * (eta + 1)
        r.x = torch.exp(-he) * r.x + (-he).expm1().neg() * den
        if r.h2 is not None:
            r0, r1 = r.h1 / h, r.h2 / h
            a = (den - r.d1) / r0
            b = (r.d1 - r.d2) / r1
            g1 = a + (a - b) * r0 / (r0 + r1)
            g2 = (a - b) / (r0 + r1)
            phi2 = he.neg().expm1() / he + 1
            phi3 = phi2 / he - 0.5
            r.x = r.x + phi2 * g1 - phi3 * g2
        elif r.h1 is not None:
            g = (den - r.d1) / (r.h1 / h)
            phi2 = he.neg().expm1() / he + 1
            r.x = r.x + phi2 * g
        if eta:
            r.x = r.x + r.noise(s[i], s[i + 1]) * s[i + 1] * (-2 * h * eta).expm1().neg().sqrt() * r.hp["s_noise"]
    r.d1, r.d2 = den, r.d1
    r.h1, r.h2 = h, r.h1


# name -> (step rule, hyper-parameters it reads, noise source: None | "randn" | "brownian")
STEP_RULES: Dict[str, Tuple[Callable, Tuple[str, ...], Optional[str]]] = {
    "euler": (_euler, ("s_churn", "s_tmin", "s_tmax", "s_noise"), None),
    "euler_a": (_euler_a, ("eta", "s_noise"), "randn"),
    "heun": (_heun, ("s_churn", "s_tmin", "s_tmax", "s_noise"), None),
    "dpm_2": (_dpm2, ("s_churn", "s_tmin", "s_tmax", "s_noise"), None),
    "dpm_2_a": (_dpm2_a, ("eta", "s_noise"), "randn"),
    "lms": (_lms, ("order",), None),
    "dpm++_2s_a": (_dpmpp_2s_a, ("eta", "s_noise"), "randn"),
    "dpm++_sde": (_dpmpp_sde, ("eta", "s_noise"), "brownian"),
    "dpm++_2m": (_dpmpp_2m, (), None),
    "dpm++_2m_sde": (_dpmpp_2m_sde, ("eta", "s_noise"), "brownian"),
    "dpm++_3m_sde": (_dpmpp_3m_sde, ("eta", "s_noise"), "brownian"),
}
_DISJOINT_QUERIES = {"dpm++_2m_sde", "dpm++_3m_sde"}       # one noise query per step over [sigma_i+1, sigma_i]


BROWNIAN_TOL = 1e-6            # torchsde.BrownianTree's default tolerance: the widest leaf of the tree


def brownian_depth(lo: float, hi: float, tol: float = BROWNIAN_TOL) -> int:
    """Fewest bisections of [lo, hi] that leave leaves no wider than `tol` (34 for the v2 / v2.1 ladders, whose
    sigma_max is about 1e4)."""
    d = 0
    while (hi - lo) / 2.0 ** d > tol:
        d += 1
    return d


class DeviceBrownianTree:
    """torchsde.BrownianTree(lo, zeros_like(x), hi, entropy=seed) as the engine builds it: `tree(t0, t1)` is
    W(t1) - W(t0) for every element of x, computed by one dbir_brownian_increment launch from (seed, node, element)
    alone. No tree is stored: the same query gives the same bits every time, and an element's value does not depend
    on the size of x. With a list of seeds, sample b of x has its own tree, seeded seeds[b]: its slice equals the
    single-seed tree of that slice alone (one dbir_brownian_increment_samples launch)."""

    def __init__(self, x: torch.Tensor, lo, hi, seed: Union[int, Sequence[int]]):
        if not x.is_cuda:
            raise ValueError("the device Brownian tree of edm_dpm++_sde needs a CUDA latent (install torchsde to "
                             "sample on another device)")
        self.shape, self.device = x.shape, x.device
        self.lo, self.hi = float(lo), float(hi)
        if isinstance(seed, int):
            self.seed, self.seeds = seed, None
        else:
            if len(seed) != x.shape[0]:
                raise ValueError(f"{len(seed)} seeds for a batch of {x.shape[0]} samples")
            self.seed, self.seeds = None, torch.tensor([int(s) for s in seed], dtype=torch.int64, device=x.device)
        self.depth = brownian_depth(self.lo, self.hi)

    def __call__(self, t0, t1) -> torch.Tensor:
        from .. import lib
        out = torch.empty(self.shape, dtype=torch.float32, device=self.device)
        if self.seeds is None:
            lib.brownian_increment(out, self.seed, self.lo, self.hi, float(t0), float(t1), self.depth)
        else:
            lib.brownian_increment_samples(out, self.seeds, self.lo, self.hi, float(t0), float(t1), self.depth)
        return out


def _brownian_noise(x: torch.Tensor, sigmas: torch.Tensor, solver: str,
                    source: Optional[NoiseSource] = None) -> Optional[Callable]:
    """BrownianTreeNoiseSampler(x, sigma_min, sigma_max) (k_diffusion.py:97-120) on torchsde's tree when torchsde is
    there, else on DeviceBrownianTree. The seed comes from the CPU generator, as in k-diffusion; ranks that cooperate
    on one image are all seeded alike and make the same CPU draws before this one, so they draw the same seed. With a
    NoiseSource each sample draws its own seed from its own CPU generator and has its own tree."""
    try:
        import torchsde
    except ImportError:
        if solver in _DISJOINT_QUERIES:
            return None                                     # independent N(0, I) draws: same distribution
        torchsde = None
    lo, hi = torch.as_tensor(sigmas[sigmas > 0].min()), torch.as_tensor(sigmas.max())
    seed = torch.randint(0, 2 ** 63 - 1, []).item() if source is None else source.randint_seeds()
    if torchsde is None:
        tree = DeviceBrownianTree(x, lo, hi, seed)
    elif source is None:
        tree = torchsde.BrownianTree(lo, torch.zeros_like(x), hi, entropy=seed)
    else:
        trees = [torchsde.BrownianTree(lo, torch.zeros_like(x[k:k + 1]), hi, entropy=s) for k, s in enumerate(seed)]

        def tree(t0, t1):
            return torch.cat([tr(t0, t1) for tr in trees])

    def sample(s0, s1):
        a, b = torch.as_tensor(s0), torch.as_tensor(s1)
        t0, t1, sign = (a, b, 1) if a < b else (b, a, -1)
        return tree(t0, t1) * sign / (b - a).abs().sqrt()
    return sample


def run_rule(solver: str, denoise: Callable, x: torch.Tensor, sigmas: torch.Tensor, hp: dict,
             noise: Optional[Callable] = None, source: Optional[NoiseSource] = None) -> torch.Tensor:
    """Runs one step rule over the sigma ladder. `noise(sigma, sigma_next)` overrides the rule's noise source
    (the k-diffusion `noise_sampler` argument; tests inject a seeded one). `source` draws every other random number
    per sample (None: the global generators)."""
    rule, names, noise_kind = STEP_RULES[solver]
    if noise is None and noise_kind == "brownian":
        noise = _brownian_noise(x, sigmas, solver, source)
    run = _Run(denoise, x, sigmas, {k: hp[k] for k in names}, noise, source)
    for i in range(run.n):
        rule(run, i)
    return run.x


class EDMSampler(Sampler):
    """diffbir.sampler.EDMSampler (edm_sampler.py:26-186): same constructor and `sample` signature."""

    TYPE_TO_SOLVER = {k: v[:2] for k, v in STEP_RULES.items()}     # reference attribute name

    def __init__(self, betas: np.ndarray, parameterization: str, rescale_cfg: bool, solver_type: str,
                 s_churn: float, s_tmin: float, s_tmax: float, s_noise: float, eta: float, order: int):
        super().__init__(betas, parameterization, rescale_cfg)
        self.solver = solver_type[len("edm_"):]
        if self.solver not in STEP_RULES:
            raise KeyError(solver_type)
        self.hp = dict(s_churn=s_churn, s_tmin=s_tmin, s_tmax=s_tmax, s_noise=s_noise, eta=eta, order=order)

    def make_schedule(self, steps: int) -> None:
        """edm_sampler.py:81-96: `steps` integer timesteps from T-1 down, their sigmas (alpha_bar of the
        first forced to 1e-8), then a final (sigma 0, t 0) pair."""
        ac = self.training_alphas_cumprod
        ts = np.linspace(len(ac) - 1, 0, steps, endpoint=False).astype(int)
        a = ac[ts].copy()
        a[0] = 1e-8
        sig = ((1 - a) / a) ** 0.5
        self.sigmas = torch.tensor(np.append(sig, 0), dtype=torch.float32)
        self.timesteps = torch.tensor(np.append(ts, 0), dtype=torch.long)

    def _scalings(self, sigma: torch.Tensor):
        """(c_skip, c_out, c_in) of edm_sampler.py:99-110."""
        if self.parameterization == "eps":
            return torch.ones_like(sigma), -sigma, 1 / (sigma ** 2 + 1.0) ** 0.5
        return 1.0 / (sigma ** 2 + 1.0), -sigma / (sigma ** 2 + 1.0) ** 0.5, 1.0 / (sigma ** 2 + 1.0) ** 0.5

    def _table_index(self, sigma: torch.Tensor) -> torch.Tensor:
        """Index of the nearest schedule sigma per batch element (edm_sampler.py:112-115)."""
        return (sigma.clone() - self.sigmas[:, None]).abs().argmin(dim=0).view(sigma.shape)

    def convert_to_denoiser(self, model, cond, uncond, cfg_scale) -> Callable:
        """Plain-PyTorch denoiser around any `model(x, t, cond)` — edm_sampler.py:98-139."""
        def denoiser(x: torch.Tensor, sigma: torch.Tensor) -> torch.Tensor:
            c_skip, c_out, c_in = self._scalings(sigma)
            t = self.timesteps[self._table_index(sigma)]
            cur = self.get_cfg_scale(cfg_scale, t[0].item())
            c_in, c_out, c_skip = (_bc(c, x.ndim) for c in (c_in, c_out, c_skip))
            if uncond is None or cfg_scale == 1.0:
                return model(x * c_in, t, cond) * c_out + x * c_skip
            dc = model(x * c_in, t, cond) * c_out + x * c_skip
            du = model(x * c_in, t, uncond) * c_out + x * c_skip
            return du + cur * (dc - du)
        return denoiser

    def _engine_denoiser(self, ev: EngineEval, cfg_scale: float) -> Callable:
        """Same arithmetic with the two branches evaluated by ONE graph replay of the kernel engine."""
        def denoiser(x: torch.Tensor, sigma: torch.Tensor) -> torch.Tensor:
            c_skip, c_out, c_in = self._scalings(sigma)
            idx = int(self._table_index(sigma)[0].item())
            cur = self.get_cfg_scale(cfg_scale, int(self.timesteps[idx].item()))
            c_in, c_out, c_skip = (_bc(c, x.ndim) for c in (c_in, c_out, c_skip))
            e_c, e_u = ev.eps((x * c_in).contiguous(), idx)
            dc = e_c * c_out + x * c_skip
            if e_u is None:
                return dc
            du = e_u * c_out + x * c_skip
            return du + cur * (dc - du)
        return denoiser

    @torch.no_grad()
    def sample(self, model, device, steps: int, x_size, cond, uncond, cfg_scale: float, tiled: bool = False,
               tile_size: int = -1, tile_stride: int = -1, x_T: Optional[torch.Tensor] = None,
               progress: bool = True) -> torch.Tensor:
        self.make_schedule(steps)
        if x_T is None:
            x_T = randn(x_size, device, self.noise_source)
        from ..model.cldm import ControlLDM
        if isinstance(model, ControlLDM):
            use_cfg = not (uncond is None or cfg_scale == 1.0)
            ev = EngineEval(model, x_T, cond, uncond if use_cfg else None, tiled, tile_size, tile_stride,
                            shard_tiles=self.shard_tiles, shard_batch=self.shard_batch,
                            time_collective=self.time_collective,
                            max_tile_forwards=self.max_tile_forwards)
            dev = ev.dev
            ev.set_timesteps([int(t) for t in self.timesteps.tolist()])
            self.last_stats = ev.stats
            x_T, denoiser = ev.x0, self._engine_denoiser(ev, cfg_scale)
        else:
            dev = x_T.device
            fn = tiled_callable(model, tile_size, tile_stride) if tiled else model
            denoiser = self.convert_to_denoiser(fn, cond, uncond, cfg_scale)
        self.sigmas, self.timesteps = self.sigmas.to(dev), self.timesteps.to(dev)
        x = x_T * torch.sqrt(1.0 + self.sigmas[0] ** 2.0)
        return run_rule(self.solver, denoiser, x, self.sigmas, self.hp, source=self.noise_source)
