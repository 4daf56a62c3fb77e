"""DPM-Solver / DPM-Solver++ sampler — counterpart of the reference's diffbir.sampler.DPMSolverSampler
(sampler/dpms_sampler.py:17-101) and of the part of the DPM-Solver library it drives
(sampler/dpm_solver_pytorch.py; Lu et al. 2022): the discrete-time VP noise schedule with piecewise
linear log-alpha (:88-169, 1273-1312), the classifier-free-guidance model wrapper (:273-349) and the
multistep solver of order 1-3 with uniform time steps (:565-610, 814-922, 1180-1230).

The CLI exposes one spec, "dpm++_m2" (inference.py:91-107: DPM-Solver++, multistep, order 2); the
constructor accepts every multistep spec "dpm_m{1,2,3}" / "dpm++_m{1,2,3}". Singlestep specs
("..._s2") are refused at construction: no entry point of the reference selects them.

The network is evaluated at the `steps` fractional model times (t_i - 1/N) * 1000 known up front, so
the kernel-engine path pre-computes their embeddings and replays one CUDA graph per step (EngineEval);
a foreign `model(x, t, cond)` callable takes the reference's arithmetic in plain PyTorch.
"""
from __future__ import annotations

import math
from typing import Callable, List, Optional

import numpy as np
import torch

from .sampler import EngineEval, Sampler, randn, tiled_callable


def _piecewise_linear(x: torch.Tensor, xp: torch.Tensor, yp: torch.Tensor) -> torch.Tensor:
    """y = f(x) through the keypoints (xp, yp), extrapolating with the outermost segments; x [N, 1],
    xp / yp [1, K] -> [N, 1]. The bracket is found by sorting x into the keypoints, as the library does
    (dpm_solver_pytorch.py:1273-1312), so that ties at a keypoint resolve identically."""
    N, K = x.shape[0], xp.shape[1]
    merged = torch.cat([x.unsqueeze(2), xp.unsqueeze(0).repeat((N, 1, 1))], dim=2)
    srt, order = torch.sort(merged, dim=2)
    pos = torch.argmin(order, dim=2)                     # rank of x among the keypoints
    one, km2 = torch.tensor(1, device=x.device), torch.tensor(K - 2, device=x.device)
    lo = torch.where(torch.eq(pos, 0), one, torch.where(torch.eq(pos, K), km2, pos - 1))
    hi = torch.where(torch.eq(lo, pos - 1), lo + 2, lo + 1)
    x0 = torch.gather(srt, dim=2, index=lo.unsqueeze(2)).squeeze(2)
    x1 = torch.gather(srt, dim=2, index=hi.unsqueeze(2)).squeeze(2)
    lo_y = torch.where(torch.eq(pos, 0), torch.tensor(0, device=x.device),
                       torch.where(torch.eq(pos, K), km2, pos - 1))
    ypx = yp.unsqueeze(0).expand(N, -1, -1)
    y0 = torch.gather(ypx, dim=2, index=lo_y.unsqueeze(2)).squeeze(2)
    y1 = torch.gather(ypx, dim=2, index=(lo_y + 1).unsqueeze(2)).squeeze(2)
    return y0 + (x - x0) * (y1 - y0) / (x1 - x0)


class DiscreteVP:
    """NoiseScheduleVP(schedule='discrete', betas=...) — dpm_solver_pytorch.py:88-169. The log-SNR near t = T
    is clipped at -5.1 (:115-126), which shortens a zero-terminal-SNR table: `total_N` may be < len(betas)."""

    def __init__(self, betas: torch.Tensor, dtype=torch.float32):
        log_a = 0.5 * torch.log(1 - betas).cumsum(dim=0)
        log_s = 0.5 * torch.log(1.0 - torch.exp(2.0 * log_a))
        cut = torch.searchsorted(torch.flip(log_a - log_s, [0]), -5.1)
        if cut > 0:
            log_a = log_a[:-cut]
        self.T = 1.0
        self.log_alpha_array = log_a.reshape((1, -1)).to(dtype=dtype)
        self.total_N = self.log_alpha_array.shape[1]
        self.t_array = torch.linspace(0.0, 1.0, self.total_N + 1)[1:].reshape((1, -1)).to(dtype=dtype)

    def log_alpha(self, t):
        return _piecewise_linear(t.reshape((-1, 1)), self.t_array.to(t.device), self.log_alpha_array.to(t.device)).reshape((-1))

    def alpha(self, t):
        return torch.exp(self.log_alpha(t))

    def std(self, t):
        return torch.sqrt(1.0 - torch.exp(2.0 * self.log_alpha(t)))

    def lam(self, t):
        la = self.log_alpha(t)
        return la - 0.5 * torch.log(1.0 - torch.exp(2.0 * la))

    def model_time(self, t):
        """continuous t in [1/N, 1] -> the network's time input in [0, 1000 (N-1)/N] (:273-282)."""
        return (t - 1.0 / self.total_N) * 1000.0


def _bc(v: torch.Tensor, ndim: int) -> torch.Tensor:
    return v[(...,) + (None,) * (ndim - 1)]


class _Multistep:
    """DPM_Solver(model_fn, ns, algorithm_type).sample(method='multistep', skip_type='time_uniform',
    solver_type='dpmsolver', lower_order_final=True) — dpm_solver_pytorch.py:1065-1230."""

    def __init__(self, noise_fn: Callable, ns: DiscreteVP, plus: bool):
        self.noise_fn, self.ns, self.plus = noise_fn, ns, plus

    def f(self, x, t, k):
        """Model value the solver integrates: data prediction for ++ (:451-460), noise otherwise. `k` = index
        of t in the run's time grid (lets an engine-backed noise_fn pick its pre-computed embedding)."""
        noise = self.noise_fn(x, t.expand((x.shape[0])), k)
        if not self.plus:
            return noise
        return (x - self.ns.std(t) * noise) / self.ns.alpha(t)

    def update(self, x, m: List[torch.Tensor], tp: List[torch.Tensor], t, order: int):
        """x(t_prev[-1]) -> x(t) with the last `order` model values (:565-610 order 1, :814-870 order 2,
        :872-922 order 3; 'dpmsolver' variant)."""
        ns, plus = self.ns, self.plus
        lam_t, lam_0 = ns.lam(t), ns.lam(tp[-1])
        la_0, la_t = ns.log_alpha(tp[-1]), ns.log_alpha(t)
        s_0, s_t = ns.std(tp[-1]), ns.std(t)
        a_t = torch.exp(la_t)
        h = lam_t - lam_0
        if order == 1:
            if plus:
                return s_t / s_0 * x - a_t * torch.expm1(-h) * m[-1]
            return torch.exp(la_t - la_0) * x - (s_t * torch.expm1(h)) * m[-1]
        if order == 2:
            h_0 = lam_0 - ns.lam(tp[-2])
            r0 = h_0 / h
            D1 = (1.0 / r0) * (m[-1] - m[-2])
            if plus:
                phi = torch.expm1(-h)
                return (s_t / s_0) * x - (a_t * phi) * m[-1] - 0.5 * (a_t * phi) * D1
            phi = torch.expm1(h)
            return (torch.exp(la_t - la_0)) * x - (s_t * phi) * m[-1] - 0.5 * (s_t * phi) * D1
        lam_1, lam_2 = ns.lam(tp[-2]), ns.lam(tp[-3])
        h_1, h_0 = lam_1 - lam_2, lam_0 - lam_1
        r0, r1 = h_0 / h, h_1 / h
        Da = (1.0 / r0) * (m[-1] - m[-2])
        Db = (1.0 / r1) * (m[-2] - m[-3])
        D1 = Da + (r0 / (r0 + r1)) * (Da - Db)
        D2 = (1.0 / (r0 + r1)) * (Da - Db)
        if plus:
            p1 = torch.expm1(-h)
            p2 = p1 / h + 1.0
            p3 = p2 / h - 0.5
            return (s_t / s_0) * x - (a_t * p1) * m[-1] + (a_t * p2) * D1 - (a_t * p3) * D2
        p1 = torch.expm1(h)
        p2 = p1 / h - 1.0
        p3 = p2 / h - 0.5
        return (torch.exp(la_t - la_0)) * x - (s_t * p1) * m[-1] - (s_t * p2) * D1 - (s_t * p3) * D2

    @staticmethod
    def time_grid(ns: DiscreteVP, steps: int, device) -> torch.Tensor:
        return torch.linspace(ns.T, 1.0 / ns.total_N, steps + 1).to(device)

    def sample(self, x, steps: int, order: int):
        assert steps >= order
        ts = self.time_grid(self.ns, steps, x.device)
        tp, m = [ts[0]], [self.f(x, ts[0], 0)]
        for k in range(1, order):                       # warm-up with the lower orders
            x = self.update(x, m, tp, ts[k], k)
            tp.append(ts[k])
            m.append(self.f(x, ts[k], k))
        for k in range(order, steps + 1):
            o = min(order, steps + 1 - k) if steps < 10 else order      # lower_order_final
            x = self.update(x, m, tp, ts[k], o)
            tp = tp[1:] + [ts[k]]
            if k < steps:                               # the final model value is never needed
                m = m[1:] + [self.f(x, ts[k], k)]
        return x


class DPMSolverSampler(Sampler):
    """diffbir.sampler.DPMSolverSampler (dpms_sampler.py:17-101): same constructor and `sample` signature."""

    def __init__(self, betas: np.ndarray, parameterization: str, rescale_cfg: bool, model_spec: str):
        super().__init__(betas, parameterization, rescale_cfg)
        if parameterization not in ("eps", "v"):
            raise ValueError(parameterization)
        kind, (method, order) = model_spec.split("_")
        self.solver_type = {"dpm": "dpmsolver", "dpm++": "dpmsolver++"}[kind]
        self.method = {"s": "singlestep", "m": "multistep"}[method]
        self.order = {"1": 1, "2": 2, "3": 3}[order]
        if self.method != "multistep":
            raise NotImplementedError(
                f"{model_spec}: singlestep DPM-Solver is not reachable from the reference's entry points "
                "(inference.py:91-107 offers dpm++_m2 only); use a multistep spec, e.g. dpm++_m2")
        self.betas = torch.tensor(betas, dtype=torch.float32)

    def _guided_noise(self, ns: DiscreteVP, cfg_scale: float, eval_branches: Callable) -> Callable:
        """noise(x, t[B], k): v -> eps conversion per branch and classifier-free guidance, the model_wrapper of
        dpm_solver_pytorch.py:284-349. eval_branches(x, t_input[B], k) -> (out_cond, out_uncond | None)."""
        def to_noise(out, x, t):
            if self.parameterization == "eps":
                return out
            return _bc(ns.alpha(t), x.dim()) * out + _bc(ns.std(t), x.dim()) * x

        def noise(x, t, k):
            t_in = ns.model_time(t)
            oc, ou = eval_branches(x, t_in, k)
            nc = to_noise(oc, x, t)
            if ou is None:
                return nc
            nu = to_noise(ou, x, t)
            if not self.rescale_cfg:
                return nu + cfg_scale * (nc - nu)
            s = 1 + cfg_scale * ((1 - math.cos(math.pi * ((1000 - t_in) / 1000) ** 5.0)) / 2)
            return nu + s * (nc - nu)
        return noise

    @torch.no_grad()
    def sample(self, model, device, steps: int, x_size, cond, uncond, cfg_scale: float, tiled: bool = False,
               tile_size: int = -1, tile_stride: int = -1, x_T: Optional[torch.Tensor] = None,
               progress: bool = True) -> torch.Tensor:
        if x_T is None:
            x_T = randn(x_size, device, self.noise_source)
        ns = DiscreteVP(self.betas)
        use_cfg = not (cfg_scale == 1.0 or uncond is None)
        from ..model.cldm import ControlLDM
        if isinstance(model, ControlLDM):
            ev = EngineEval(model, x_T, cond, uncond if use_cfg else None, tiled, tile_size, tile_stride,
                            shard_tiles=self.shard_tiles, shard_batch=self.shard_batch,
                            time_collective=self.time_collective,
                            max_tile_forwards=self.max_tile_forwards)
            grid = _Multistep.time_grid(ns, steps, "cpu")
            ev.set_timesteps([float(v) for v in ns.model_time(grid[:-1]).tolist()])
            self.last_stats = ev.stats
            x_T = ev.x0

            def branches(x, t_in, k):
                return ev.eps(x.contiguous(), k)
        else:
            fn = tiled_callable(model, tile_size, tile_stride) if tiled else model

            def branches(x, t_in, k):
                if not use_cfg:
                    return fn(x, t_in, cond), None
                # one batched forward, unconditional half first (dpm_solver_pytorch.py:329-339)
                c2 = {key: torch.cat([uncond[key], cond[key]]) for key in cond}
                ou, oc = fn(torch.cat([x] * 2), torch.cat([t_in] * 2), c2).chunk(2)
                return oc, ou
        solver = _Multistep(self._guided_noise(ns, cfg_scale, branches), ns, self.solver_type == "dpmsolver++")
        return solver.sample(x_T, steps, self.order)
