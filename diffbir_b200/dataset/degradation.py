"""Blur-kernel generators and batch noise of the Real-ESRGAN degradation (reference dataset/degradation.py).

The kernel generators are numpy code run per sample in dataloader workers; they draw from Python's `random`
and numpy's global generator in the reference's order, so a seeded worker produces the reference's kernels
bit for bit. The batch noise functions run on the engine: their draws are the reference's torch calls, the
arithmetic between them is `dbir_gaussian_noise` / `dbir_noise_levels` / `dbir_poisson_rate` /
`dbir_poisson_noise`.
"""
from __future__ import annotations

import math
import random

import numpy as np
import torch
from scipy import special

from ._device import require_cuda


# ---------------------------------------------------------------- blur kernels (numpy)
def sigma_matrix2(sig_x, sig_y, theta):
    """Covariance diag(sig_x^2, sig_y^2) rotated by theta (radians)."""
    rot = np.array([[np.cos(theta), -np.sin(theta)], [np.sin(theta), np.cos(theta)]])
    diag = np.array([[sig_x ** 2, 0], [0, sig_y ** 2]])
    return np.dot(rot, np.dot(diag, rot.T))


def mesh_grid(kernel_size):
    """(xy [k, k, 2], xx, yy): integer offsets centred on the middle tap."""
    ax = np.arange(-kernel_size // 2 + 1.0, kernel_size // 2 + 1.0)
    xx, yy = np.meshgrid(ax, ax)
    n = kernel_size * kernel_size
    xy = np.hstack((xx.reshape((n, 1)), yy.reshape(n, 1))).reshape(kernel_size, kernel_size, 2)
    return xy, xx, yy


def _quadratic_form(sig_x, sig_y, theta, grid, isotropic):
    """d^T Sigma^-1 d at every grid offset d."""
    if isotropic:
        cov = np.array([[sig_x ** 2, 0], [0, sig_x ** 2]])
    else:
        cov = sigma_matrix2(sig_x, sig_y, theta)
    return np.sum(np.dot(grid, np.linalg.inv(cov)) * grid, 2)


def pdf2(sigma_matrix, grid):
    """Un-normalised bivariate Gaussian density on the grid."""
    return np.exp(-0.5 * np.sum(np.dot(grid, np.linalg.inv(sigma_matrix)) * grid, 2))


def bivariate_Gaussian(kernel_size, sig_x, sig_y, theta, grid=None, isotropic=True):
    if grid is None:
        grid, _, _ = mesh_grid(kernel_size)
    k = np.exp(-0.5 * _quadratic_form(sig_x, sig_y, theta, grid, isotropic))
    return k / np.sum(k)


def bivariate_generalized_Gaussian(kernel_size, sig_x, sig_y, theta, beta, grid=None, isotropic=True):
    if grid is None:
        grid, _, _ = mesh_grid(kernel_size)
    k = np.exp(-0.5 * np.power(_quadratic_form(sig_x, sig_y, theta, grid, isotropic), beta))
    return k / np.sum(k)


def bivariate_plateau(kernel_size, sig_x, sig_y, theta, beta, grid=None, isotropic=True):
    if grid is None:
        grid, _, _ = mesh_grid(kernel_size)
    k = np.reciprocal(np.power(_quadratic_form(sig_x, sig_y, theta, grid, isotropic), beta) + 1)
    return k / np.sum(k)


def _draw_shape(sigma_x_range, sigma_y_range, rotation_range, isotropic):
    assert sigma_x_range[0] < sigma_x_range[1], "Wrong sigma_x_range."
    sig_x = np.random.uniform(sigma_x_range[0], sigma_x_range[1])
    if isotropic is False:
        assert sigma_y_range[0] < sigma_y_range[1], "Wrong sigma_y_range."
        assert rotation_range[0] < rotation_range[1], "Wrong rotation_range."
        return sig_x, np.random.uniform(sigma_y_range[0], sigma_y_range[1]), \
            np.random.uniform(rotation_range[0], rotation_range[1])
    return sig_x, sig_x, 0


def _draw_beta(beta_range):
    # below or above 1 with equal odds (beta_range[0] < 1 < beta_range[1])
    if np.random.uniform() < 0.5:
        return np.random.uniform(beta_range[0], 1)
    return np.random.uniform(1, beta_range[1])


def _kernel_noise(kernel, noise_range):
    if noise_range is not None:
        assert noise_range[0] < noise_range[1], "Wrong noise range."
        kernel = kernel * np.random.uniform(noise_range[0], noise_range[1], size=kernel.shape)
    return kernel / np.sum(kernel)


def random_bivariate_Gaussian(kernel_size, sigma_x_range, sigma_y_range, rotation_range, noise_range=None,
                              isotropic=True):
    assert kernel_size % 2 == 1, "Kernel size must be an odd number."
    sx, sy, th = _draw_shape(sigma_x_range, sigma_y_range, rotation_range, isotropic)
    return _kernel_noise(bivariate_Gaussian(kernel_size, sx, sy, th, isotropic=isotropic), noise_range)


def random_bivariate_generalized_Gaussian(kernel_size, sigma_x_range, sigma_y_range, rotation_range, beta_range,
                                          noise_range=None, isotropic=True):
    assert kernel_size % 2 == 1, "Kernel size must be an odd number."
    sx, sy, th = _draw_shape(sigma_x_range, sigma_y_range, rotation_range, isotropic)
    beta = _draw_beta(beta_range)
    return _kernel_noise(bivariate_generalized_Gaussian(kernel_size, sx, sy, th, beta, isotropic=isotropic),
                         noise_range)


def random_bivariate_plateau(kernel_size, sigma_x_range, sigma_y_range, rotation_range, beta_range, noise_range=None,
                             isotropic=True):
    assert kernel_size % 2 == 1, "Kernel size must be an odd number."
    sx, sy, th = _draw_shape(sigma_x_range, sigma_y_range, rotation_range, isotropic)
    beta = _draw_beta(beta_range)
    return _kernel_noise(bivariate_plateau(kernel_size, sx, sy, th, beta, isotropic=isotropic), noise_range)


def random_mixed_kernels(kernel_list, kernel_prob, kernel_size=21, sigma_x_range=(0.6, 5), sigma_y_range=(0.6, 5),
                         rotation_range=(-math.pi, math.pi), betag_range=(0.5, 8), betap_range=(0.5, 8),
                         noise_range=None):
    """One kernel of a type drawn from kernel_list ('iso', 'aniso', 'generalized_iso', 'generalized_aniso',
    'plateau_iso', 'plateau_aniso') with probabilities kernel_prob. Plateau kernels take no multiplicative noise."""
    kind = random.choices(kernel_list, kernel_prob)[0]
    shape = (kernel_size, sigma_x_range, sigma_y_range, rotation_range)
    iso = not kind.endswith("aniso")
    if kind in ("iso", "aniso"):
        return random_bivariate_Gaussian(*shape, noise_range=noise_range, isotropic=iso)
    if kind.startswith("generalized"):
        return random_bivariate_generalized_Gaussian(*shape, betag_range, noise_range=noise_range, isotropic=iso)
    if kind.startswith("plateau"):
        return random_bivariate_plateau(*shape, betap_range, noise_range=None, isotropic=iso)
    raise ValueError(f"unknown kernel type {kind!r}")


def circular_lowpass_kernel(cutoff, kernel_size, pad_to=0):
    """2-D circularly symmetric sinc (ideal low-pass at `cutoff` radians), normalised, zero-padded to pad_to."""
    assert kernel_size % 2 == 1, "Kernel size must be an odd number."
    c = (kernel_size - 1) / 2

    def taps(x, y):
        r = np.sqrt((x - c) ** 2 + (y - c) ** 2)
        return cutoff * special.j1(cutoff * r) / (2 * np.pi * r)

    with np.errstate(divide="ignore", invalid="ignore"):
        kernel = np.fromfunction(taps, [kernel_size, kernel_size])
    kernel[(kernel_size - 1) // 2, (kernel_size - 1) // 2] = cutoff ** 2 / (4 * np.pi)
    kernel = kernel / np.sum(kernel)
    if pad_to > kernel_size:
        p = (pad_to - kernel_size) // 2
        kernel = np.pad(kernel, ((p, p), (p, p)))
    return kernel


# ---------------------------------------------------------------- batch noise (engine)
def random_add_gaussian_noise_pt(img, sigma_range=(0, 1.0), gray_prob=0, clip=True, rounds=False):
    """img + N(0, sigma/255) per sample, sigma ~ U(sigma_range); with probability gray_prob a sample's noise is one
    gray field shared by the batch. Draws: torch.rand(b) (sigma), torch.rand(b) (gray), torch.randn(h, w) when any
    sample is gray, torch.randn(b, c, h, w)."""
    _noise_args(img, clip, rounds)
    b, c, h, w = img.shape
    u_sigma = torch.rand(b, dtype=img.dtype, device=img.device)
    u_gray = torch.rand(b, dtype=img.dtype, device=img.device)
    gray = any_gray(u_gray, gray_prob)
    noise_gray = torch.randn(h, w, dtype=img.dtype, device=img.device) if gray else None
    noise = torch.randn(b, c, h, w, dtype=img.dtype, device=img.device)
    out = torch.empty_like(img)
    from .. import lib
    lib.gaussian_noise(img, noise, noise_gray, u_sigma, sigma_range[0], sigma_range[1] - sigma_range[0], u_gray,
                       gray_prob, out)
    return out


def random_add_poisson_noise_pt(img, scale_range=(0, 1.0), gray_prob=0, clip=True, rounds=False):
    """img + scale * (Poisson(level * vals) / vals - level) per sample, level = the image rounded to 8 bits and
    vals = 2^ceil(log2(distinct levels)). Draws: torch.rand(b) (scale), torch.rand(b) (gray), torch.poisson of the
    gray image when any sample is gray, torch.poisson of the colour image."""
    _noise_args(img, clip, rounds)
    from .. import lib
    b, c, h, w = img.shape
    u_scale = torch.rand(b, dtype=img.dtype, device=img.device)
    u_gray = torch.rand(b, dtype=img.dtype, device=img.device)
    gray = {}
    if any_gray(u_gray, gray_prob):
        q_g, draw_g, vals_g = _poisson_draw(img, True)
        gray = dict(q_gray=q_g, draw_gray=draw_g, vals_gray=vals_g, u_gray=u_gray, gray_prob=gray_prob)
    q, draw, vals = _poisson_draw(img, False)
    out = torch.empty_like(img)
    lib.poisson_noise(img, q, draw, vals, u_scale, scale_range[0], scale_range[1] - scale_range[0], out, **gray)
    return out


def _poisson_draw(img, gray):
    from .. import lib
    b, c, h, w = img.shape
    q = torch.empty(b, 1 if gray else c, h, w, dtype=img.dtype, device=img.device)
    hist = torch.empty(b, 256, dtype=torch.int32, device=img.device)
    vals = torch.empty(b, dtype=img.dtype, device=img.device)
    rate = torch.empty_like(q)
    lib.noise_levels(img, q, hist, gray=gray)
    lib.poisson_rate(q, hist, vals, rate)
    return q, torch.poisson(rate), vals


def any_gray(u_gray, gray_prob) -> bool:
    """torch.sum((u_gray < gray_prob).float()) > 0: the one host sync, where the reference branches on it."""
    return bool((u_gray.cpu().numpy() < np.float32(gray_prob)).any())


def _noise_args(img, clip, rounds):
    require_cuda(img, "noise")
    if not clip or rounds:
        raise NotImplementedError("the engine's batch noise implements clip=True, rounds=False "
                                  "(the only setting RealESRGANBatchTransform uses)")
    if img.dtype != torch.float32 or not img.is_contiguous() or img.dim() != 4:
        raise ValueError("expected a contiguous float32 [b, c, h, w] tensor")
