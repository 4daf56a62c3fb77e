"""ORACLE of the Tiled-VAE hook (reference utils/tilevae/tilevae.py, non-fast mode, as model/cldm.py:92-141 calls
it): a plain torch restatement (fp32, or fp64 against the fixture), on any device, built on oracle/cldm.py.

Each tile runs through the encoder / decoder as an image of its own; every GroupNorm uses the pixel-weighted
average of the tiles' per-(image, group) means and biased variances, the tiles visited forwards at even and
backwards at odd GroupNorms (tilevae.py:232-278, 514-575). Pinned to the reference by
tests/golden/tilevae_small.npz (tests/test_vae_tiles.py)."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

from oracle import cldm as ocl


def fixture_input(seed: int, shape, lo: float, hi: float) -> torch.Tensor:
    """The inputs of the tests/golden/tilevae_small.npz cases, rebuilt instead of stored: an integer hash of the
    element index picks one of 2048 evenly spaced levels in [lo, hi). With lo = -hi and hi = 1 or 2 every level is
    exact in fp16, so the fp16 / fp32 / fp64 runs all see the same values. fp32 NCHW on the CPU."""
    idx = torch.arange(math.prod(shape), dtype=torch.int64)
    h = (idx * 1540483477 + seed * 40503 + 12345) % 2 ** 32
    h = h ^ (h >> 15)
    h = (h * 1540483477) % 2 ** 32
    h = h ^ (h >> 13)
    return ((h % 2048).to(torch.float64) * ((hi - lo) / 2048) + lo).float().reshape(shape)


def fixture_source(fx, case: str) -> torch.Tensor:
    """A fixture case's input (image or latent), rebuilt from its seed and checked against the stored sum."""
    lo, hi = fx[case + "_range"].tolist()
    x = fixture_input(int(fx[case + "_seed"]), tuple(fx[case + "_shape"].tolist()), lo, hi)
    assert x.double().sum().item() == float(fx[case + "_sum"]), f"{case}: the rebuilt input differs from the fixture's"
    return x


def split_tiles(h: int, w: int, tile: int, is_decoder: bool):
    """(input boxes, output boxes) as [x0, x1, y0, y1] lists, row-major (tilevae.py:325-397)."""
    pad = 11 if is_decoder else 32

    def best(lo, hi):
        d = 32
        while d >= 2:
            if lo % d == 0:
                return lo
            if lo - lo % d + d <= hi:
                return lo - lo % d + d
            d //= 2
        return lo

    nh, nw = max(1, math.ceil((h - 2 * pad) / tile)), max(1, math.ceil((w - 2 * pad) / tile))
    th, tw = best(math.ceil((h - 2 * pad) / nh), tile), best(math.ceil((w - 2 * pad) / nw), tile)
    ins, outs = [], []
    for i in range(nh):
        for j in range(nw):
            b = [pad + j * tw, min(pad + (j + 1) * tw, w), pad + i * th, min(pad + (i + 1) * th, h)]
            o = [b[0] if b[0] > pad else 0, b[1] if b[1] < w - pad else w, b[2] if b[2] > pad else 0,
                 b[3] if b[3] < h - pad else h]
            outs.append([v * 8 if is_decoder else v // 8 for v in o])
            ins.append([max(0, b[0] - pad), min(w, b[1] + pad), max(0, b[2] - pad), min(h, b[3] + pad)])
    return ins, outs


def _norm(x, mv, w, b, silu):
    n, c, hh, ww = x.shape
    mean, var = mv
    y = (x.reshape(n, 32, -1) - mean[..., None]) / torch.sqrt(var[..., None] + 1e-6)
    y = y.reshape(n, c, hh, ww) * w.view(1, -1, 1, 1) + b.view(1, -1, 1, 1)
    return F.silu(y) if silu else y


def _res(sd, p, x):
    h = _norm(x, (yield x), sd[p + "norm1.weight"], sd[p + "norm1.bias"], True)
    h = F.conv2d(h, sd[p + "conv1.weight"], sd[p + "conv1.bias"], padding=1)
    if p + "nin_shortcut.weight" in sd:
        x = F.conv2d(x, sd[p + "nin_shortcut.weight"], sd[p + "nin_shortcut.bias"])
    h = _norm(h, (yield h), sd[p + "norm2.weight"], sd[p + "norm2.bias"], True)
    return x + F.conv2d(h, sd[p + "conv2.weight"], sd[p + "conv2.bias"], padding=1)


def _attn(sd, p, x):
    b, c, hh, ww = x.shape
    y = _norm(x, (yield x), sd[p + "norm.weight"], sd[p + "norm.bias"], False)
    q, k, v = (F.conv2d(y, sd[p + n + ".weight"], sd[p + n + ".bias"]).reshape(b, c, hh * ww).transpose(1, 2)
               for n in ("q", "k", "v"))
    o = ocl.attention(q, k, v, 1).transpose(1, 2).reshape(b, c, hh, ww)
    return x + F.conv2d(o, sd[p + "proj_out.weight"], sd[p + "proj_out.bias"])


def _mid(sd, p, h):
    h = yield from _res(sd, p + "mid.block_1.", h)
    h = yield from _attn(sd, p + "mid.attn_1.", h)
    return (yield from _res(sd, p + "mid.block_2.", h))


def _encoder(sd, x):
    p = "encoder."
    h = F.conv2d(x, sd[p + "conv_in.weight"], sd[p + "conv_in.bias"], padding=1)
    for lvl in ocl._indices(sd, p + "down."):
        for j in ocl._indices(sd, f"{p}down.{lvl}.block."):
            h = yield from _res(sd, f"{p}down.{lvl}.block.{j}.", h)
        if f"{p}down.{lvl}.downsample.conv.weight" in sd:
            h = F.conv2d(F.pad(h, (0, 1, 0, 1)), sd[f"{p}down.{lvl}.downsample.conv.weight"],
                         sd[f"{p}down.{lvl}.downsample.conv.bias"], stride=2)
    h = yield from _mid(sd, p, h)
    h = _norm(h, (yield h), sd[p + "norm_out.weight"], sd[p + "norm_out.bias"], True)
    return F.conv2d(h, sd[p + "conv_out.weight"], sd[p + "conv_out.bias"], padding=1)


def _decoder(sd, z):
    p = "decoder."
    h = F.conv2d(z, sd[p + "conv_in.weight"], sd[p + "conv_in.bias"], padding=1)
    h = yield from _mid(sd, p, h)
    for lvl in reversed(ocl._indices(sd, p + "up.")):
        for j in ocl._indices(sd, f"{p}up.{lvl}.block."):
            h = yield from _res(sd, f"{p}up.{lvl}.block.{j}.", h)
        if f"{p}up.{lvl}.upsample.conv.weight" in sd:
            h = F.conv2d(F.interpolate(h, scale_factor=2.0, mode="nearest"), sd[f"{p}up.{lvl}.upsample.conv.weight"],
                         sd[f"{p}up.{lvl}.upsample.conv.bias"], padding=1)
    h = _norm(h, (yield h), sd[p + "norm_out.weight"], sd[p + "norm_out.bias"], True)
    return F.conv2d(h, sd[p + "conv_out.weight"], sd[p + "conv_out.bias"], padding=1)


def merge(means, variances, pixels, reverse: bool):
    """The shared statistics of one GroupNorm from lists over tiles of [N, 32] tensors, in the reference's fp32
    arithmetic (GroupNormParam.summary, tilevae.py:263-278): weights (pixels / max) / sum, tiles stacked in
    visiting order."""
    order = list(range(len(pixels) - 1, -1, -1)) if reverse else list(range(len(pixels)))
    px = torch.tensor([pixels[t] for t in order], dtype=torch.float32, device=means[0].device) / max(pixels)
    px = (px / px.sum())[:, None, None]
    mean = (torch.stack([means[t] for t in order]) * px).sum(0)
    var = (torch.stack([variances[t] for t in order]) * px).sum(0)
    return mean, var


def tiled_forward(sd, x, tile: int, is_decoder: bool, out_ch: int):
    """The hook on x (in the dtype of x and sd); inputs no larger than 2 * pad + tile run as one tile, which is
    the un-tiled network (tilevae.py:317-323)."""
    n, _, h, w = x.shape
    if max(h, w) <= 2 * (11 if is_decoder else 32) + tile:
        ins, outs = [[0, w, 0, h]], [[0, w * 8, 0, h * 8] if is_decoder else [0, w // 8, 0, h // 8]]
    else:
        ins, outs = split_tiles(h, w, tile, is_decoder)
    net = _decoder if is_decoder else _encoder
    gens = [net(sd, x[:, :, b[2]:b[3], b[0]:b[1]].contiguous()) for b in ins]
    cur = [next(g) for g in gens]
    res = [None] * len(gens)
    k = 0
    while True:
        vm = [torch.var_mean(t.reshape(n, 32, -1), dim=2, unbiased=False) for t in cur]
        mv = merge([m for _, m in vm], [v for v, _ in vm], [t.shape[2] * t.shape[3] for t in cur], k % 2 == 1)
        for i, g in enumerate(gens):
            try:
                cur[i] = g.send(mv)
            except StopIteration as e:
                res[i] = e.value
        if all(r is not None for r in res):
            break
        k += 1
    s = 8 if is_decoder else 1 / 8
    out = x.new_zeros(n, out_ch, int(h * s), int(w * s))
    for b, o, t in zip(ins, outs, res):
        pb = [v * 8 if is_decoder else v // 8 for v in b]
        m = [o[i] - pb[i] for i in range(4)]
        out[:, :, o[2]:o[3], o[0]:o[1]] = t[:, :, m[2]:t.shape[2] + m[3], m[0]:t.shape[3] + m[1]]
    return out


@torch.no_grad()
def vae_encode_moments_tiled(sd, img, tile: int):
    """ControlLDM.vae_encode(tiled=True) up to the posterior: [N, 8, H/8, W/8] (tile in image pixels). Computes
    in the dtype of img and sd (fp32, or fp64 against the fixture)."""
    h = tiled_forward(sd, img, tile, False, sd["encoder.conv_out.weight"].shape[0])
    return F.conv2d(h, sd["quant_conv.weight"], sd["quant_conv.bias"])


@torch.no_grad()
def vae_decode_tiled(sd, z, tile: int):
    """ControlLDM.vae_decode(tiled=True) of z already divided by the scale factor (tile in latent pixels)."""
    z = F.conv2d(z, sd["post_quant_conv.weight"], sd["post_quant_conv.bias"])
    return tiled_forward(sd, z, tile, True, sd["decoder.conv_out.weight"].shape[0])
