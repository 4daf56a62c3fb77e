"""-m gpu: tiled sampling in bounded memory and the full-resolution kernels beyond 2^31 elements.

* Chunked tile-forwards (Sampler.max_tile_forwards) give the same bits as one replay of every tile-forward.
* With a fixed cap the sampler loop's peak memory does not grow with the number of tiles.
* A 3072^2 tiled restoration at the full configuration finishes on one 80 GB H100.
* The VAE's full-resolution kernels address tensors of more than 2^31 elements correctly.
"""
import gc

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from diffbir_b200.utils.synth import RUN_DEFAULTS, build_synthetic_pipeline, synthetic_lq
from tests.gpu_util import no_tf32, rel_err

pytestmark = pytest.mark.gpu

BIG = 2 ** 31


def _tol16(L):
    return 1.5e-3 if L.operand_dtype() == torch.float16 else 1e-2


def _free():
    gc.collect()
    torch.cuda.empty_cache()


def _rows(n, step):
    """Strided subsample of 0..n-1 that always contains the last index (the largest offsets)."""
    return sorted(set(range(0, n, step)) | {n - 1})


# ---------------------------------------------------------------- kernels on > 2^31 elements
@pytest.fixture(scope="module")
def L():
    from diffbir_b200 import lib
    lib.load()
    no_tf32()
    return lib


def _group_stats(x, hw, c):
    """(mean, rstd) per group of a [hw, c] fp32 tensor, accumulated in fp64 over row blocks."""
    s = torch.zeros(32, dtype=torch.float64, device="cuda")
    q = torch.zeros_like(s)
    for r0 in range(0, hw, 1 << 20):
        blk = x[r0:r0 + (1 << 20)].view(-1, 32, c // 32).double()
        s += blk.sum((0, 2))
        q += blk.pow(2).sum((0, 2))
    cnt = hw * (c // 32)
    mean = s / cnt
    return mean, 1 / (q / cnt - mean * mean + 1e-6).sqrt()


def _fill(x, seed):
    """In place: a fresh normal sample with a per-channel offset and scale (x is [..., c])."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x.normal_(generator=g)
    c = x.shape[-1]
    x.mul_(1 + torch.arange(c, device="cuda", dtype=x.dtype) / c).add_(torch.linspace(-1, 1, c, device="cuda", dtype=x.dtype))
    return x


def test_gn_stats_and_apply_beyond_2_31(L):
    """gn_stats over 3072^2 x 256 fp32 (2.4e9 elements) and gn_apply with 2x upsample from 1536^2 x 256 into
    3072^2 x 256 op16."""
    h = w = 3072
    c, hw = 256, h * w
    x = _fill(torch.empty(hw, c, device="cuda"), 1)
    assert x.numel() > BIG
    stats = torch.empty(64, device="cuda")
    ws = torch.zeros(L.gn_workspace_floats(1, hw, c), device="cuda")
    L.gn_stats(x, None, c, 0, 1, hw, 1e-6, stats, ws)
    mean, rstd = _group_stats(x, hw, c)
    st = stats.view(32, 2).double()
    assert (st[:, 0] - mean).abs().max() < 1e-4 * (mean.abs().max() + 1)
    assert ((st[:, 1] - rstd).abs() / rstd).max() < 1e-4
    del x, ws
    _free()

    hs = h // 2
    src = _fill(torch.empty(hs * hs, c, device="cuda"), 2)
    gamma = 1 + 0.1 * torch.randn(c, device="cuda")
    beta = 0.1 * torch.randn(c, device="cuda")
    L.gn_stats(src, None, c, 0, 1, hs * hs, 1e-6, stats, torch.zeros(L.gn_workspace_floats(1, hs * hs, c), device="cuda"))
    out = torch.empty(h, w, c, device="cuda", dtype=L.operand_dtype())
    assert out.numel() > BIG
    L.gn_apply(src, None, c, 0, 1, hs, hs, stats, gamma, beta, out, norm=True, silu=True, upsample=2)
    st = stats.view(32, 2)
    a = gamma * st[:, 1].repeat_interleave(c // 32)
    b = beta - st[:, 0].repeat_interleave(c // 32) * a
    sv = src.view(hs, hs, c)
    for y in _rows(h, 97):
        ref = F.silu(sv[y // 2] * a + b).repeat_interleave(2, 0)
        assert rel_err(out[y], ref) < _tol16(L), y
    del src, out
    _free()


def test_gn_apply_rows_and_plain_gemm_beyond_2_31(L):
    """The decoder's full-resolution 256 -> 128 ResBlock entry: gn_apply without upsampling (normalised operand plus
    the raw copy) over 3072^2 x 256 fp32, then the 1x1 nin_shortcut as a plain GEMM whose A operand has 2.4e9
    elements."""
    h = w = 3072
    c, co, hw = 256, 128, h * w
    dt = L.operand_dtype()
    x = _fill(torch.empty(hw, c, device="cuda"), 6)
    stats = torch.empty(64, device="cuda")
    L.gn_stats(x, None, c, 0, 1, hw, 1e-6, stats, torch.zeros(L.gn_workspace_floats(1, hw, c), device="cuda"))
    gamma = 1 + 0.1 * torch.randn(c, device="cuda")
    beta = 0.1 * torch.randn(c, device="cuda")
    a16 = torch.empty(hw, c, device="cuda", dtype=dt)
    raw = torch.empty(hw, c, device="cuda", dtype=dt)
    assert a16.numel() > BIG
    L.gn_apply(x, None, c, 0, 1, h, w, stats, gamma, beta, a16, norm=True, silu=True, out_raw=raw)
    st = stats.view(32, 2)
    a = gamma * st[:, 1].repeat_interleave(c // 32)
    b = beta - st[:, 0].repeat_interleave(c // 32) * a
    rows = [r * w + xx for r in _rows(h, 89) for xx in (0, w - 1)]
    rows = torch.tensor(rows, device="cuda")
    assert rel_err(a16[rows], F.silu(x[rows] * a + b)) < _tol16(L)
    assert rel_err(raw[rows], x[rows]) < _tol16(L)
    del x, a16
    _free()
    wt = (torch.randn(co, c, device="cuda") * c ** -0.5).to(dt)
    bias = 0.1 * torch.randn(co, device="cuda")
    out = torch.empty(hw, co, device="cuda")
    L.gemm(raw, wt, out, M=hw, N=co, K=c, bias=bias)
    ref = raw[rows].float() @ wt.float().t() + bias
    assert rel_err(out[rows], ref) < 3e-5
    del raw, out
    _free()


def test_gn_stats_workspace_shared_across_batch_sizes(L):
    """One zero-initialised gn_stats workspace serves calls of different batch sizes (the engines size it for the
    largest batch and reuse it): a small batch followed by a larger one gives every image of the larger batch its
    own statistics, call after call."""
    hw, c, n_max = 4096, 64, 80
    x = _fill(torch.empty(n_max, hw, c, device="cuda"), 7)
    ws = torch.zeros(L.gn_workspace_floats(n_max, hw, c), device="cuda")
    g = x.view(n_max, hw, 32, c // 32).permute(0, 2, 1, 3).reshape(n_max, 32, -1).double()
    mean, var = g.mean(-1), g.var(-1, unbiased=False)
    for n in (4, n_max, 12, n_max, n_max):
        stats = torch.empty(n * 64, device="cuda")
        L.gn_stats(x[:n], None, c, 0, n, hw, 1e-6, stats, ws)
        st = stats.view(n, 32, 2).double()
        assert (st[..., 0] - mean[:n]).abs().max() < 1e-4 * (mean.abs().max() + 1), n
        rstd = 1 / (var[:n] + 1e-6).sqrt()
        assert ((st[..., 1] - rstd).abs() / rstd).max() < 1e-4, n


def test_conv3x3_small_cout_beyond_2_31(L):
    """The VAE's RGB head (conv3x3_small_cout) reading a 3072^2 x 256 op16 tensor (2.4e9 elements)."""
    h = w = 3072
    c = 256
    x = _fill(torch.empty(h, w, c, device="cuda", dtype=L.operand_dtype()), 3)
    assert x.numel() > BIG
    wt = torch.randn(3, c, 3, 3, device="cuda") * 0.02
    bias = torch.randn(3, device="cuda")
    out = torch.empty(1, 3, h, w, device="cuda")
    L.conv3x3_small_cout(x, 1, h, w, c, wt.permute(0, 2, 3, 1).reshape(3, -1).contiguous(), bias, 3, out, nchw=True)
    for y in _rows(h, 101):
        lo, hi = max(0, y - 1), min(h, y + 2)
        slab = x[lo:hi].float().permute(2, 0, 1)[None]
        ref = F.conv2d(slab, wt, bias, padding=1)[0, :, y - lo]
        assert rel_err(out[0, :, y], ref) < 1e-5, y
    del x, out
    _free()


def test_im2col_s2_beyond_2_31(L):
    """The VAE encoder's stride-2 im2col at 3072^2 x 128: its op16 output has 2.7e9 elements."""
    h = w = 3072
    c = 128
    x = _fill(torch.empty(h, w, c, device="cuda"), 4)
    ho = wo = h // 2
    out = torch.empty(ho * wo, 9 * c, device="cuda", dtype=L.operand_dtype())
    assert out.numel() > BIG
    L.im2col_s2(x, 1, h, w, c, 0, out)
    ov = out.view(ho, wo, 9, c)
    zero_col = torch.zeros(1, c, device="cuda")
    for oy in _rows(ho, 53):
        for tap in range(9):
            yy, xs = 2 * oy + tap // 3, torch.arange(wo, device="cuda") * 2 + tap % 3
            row = torch.cat([x[yy], zero_col]) if yy < h else torch.zeros(w + 1, c, device="cuda")
            ref = row[xs.clamp(max=w)]
            assert rel_err(ov[oy, :, tap], ref) < _tol16(L), (oy, tap)
    del x, out
    _free()


def test_gemm_conv_gn_partials_beyond_2_31(L):
    """Implicit-GEMM 3x3 conv 256 -> 256 at 3072^2 (fp32 output of 2.4e9 elements) with the fused GroupNorm partial
    sums, finalised by gn_finalize: the epilogue's row and partial-slot offsets past 2^31."""
    h = w = 3072
    c, hw = 256, h * w
    dt = L.operand_dtype()
    x = _fill(torch.empty(h, w, c, device="cuda", dtype=dt), 5)
    wt = (torch.randn(c, c, 3, 3, device="cuda") * (9 * c) ** -0.5).to(dt)
    bias = 0.1 * torch.randn(c, device="cuda")
    out = torch.empty(hw, c, device="cuda")
    assert out.numel() > BIG
    slots = L.gemm_gn_slots(h, w)
    part = torch.zeros(slots * c * 2, device="cuda")
    L.gemm(x, wt.permute(0, 2, 3, 1).reshape(c, -1).contiguous(), out, M=hw, N=c, K=9 * c, bias=bias,
           conv=(1, h, w, c, 3), gn_partials=part)
    stats = torch.empty(64, device="cuda")
    L.gn_finalize(part, slots, c, None, 0, 0, 1, hw, 1e-6, stats)
    mean, rstd = _group_stats(out, hw, c)
    st = stats.view(32, 2).double()
    assert (st[:, 0] - mean).abs().max() < 1e-4 * (mean.abs().max() + 1)
    assert ((st[:, 1] - rstd).abs() / rstd).max() < 1e-4
    ov = out.view(h, w, c)
    for y in _rows(h, 127):
        lo, hi = max(0, y - 1), min(h, y + 2)
        slab = x[lo:hi].float().permute(2, 0, 1)[None]
        ref = F.conv2d(slab, wt.float(), bias, padding=1)[0, :, y - lo].t()
        assert rel_err(ov[y], ref) < 3e-5, y
    del x, out, part
    _free()


# ---------------------------------------------------------------- chunked tiled sampling, reduced networks
_SMALL = {}


def _small_pipe():
    no_tf32()
    if "p" not in _SMALL:
        _SMALL["p"] = build_synthetic_pipeline("cuda", seed=1234, small=True)
    return _SMALL["p"]


def _make_sampler(pipe, name):
    from diffbir_b200.sampler import DDIMSampler, EDMSampler, SpacedSampler
    betas, param = pipe.diffusion.betas, pipe.diffusion.parameterization
    if name == "spaced":
        return SpacedSampler(betas, param, False)
    if name == "ddim":
        return DDIMSampler(betas, param, False, eta=0)
    return EDMSampler(betas, param, False, name, s_churn=0, s_tmin=0, s_tmax=300, s_noise=1, eta=1, order=1)


def _conditions(cl, B, H, W, seed=17):
    g = torch.Generator().manual_seed(seed)
    ctxd = cl.unet_cfg["context_dim"]
    cond = dict(c_txt=torch.randn(B, 77, ctxd, generator=g).cuda(), c_img=torch.randn(B, 4, H, W, generator=g).cuda())
    unc = dict(c_txt=torch.randn(B, 77, ctxd, generator=g).cuda(), c_img=cond["c_img"].clone())
    return cond, unc, torch.randn(B, 4, H, W, generator=g).cuda()


def _sample(pipe, name, cap, cond, unc, xT, cfg, steps=4, tile=64, stride=16):
    smp = _make_sampler(pipe, name)
    smp.max_tile_forwards = cap
    torch.manual_seed(5)
    z = smp.sample(pipe.cldm, "cuda", steps, tuple(xT.shape), cond, unc, cfg, tiled=True, tile_size=tile,
                   tile_stride=stride, x_T=xT)
    return z.clone(), dict(smp.last_stats)


@pytest.mark.parametrize("sampler,cfg", [("spaced", 4.0), ("ddim", 4.0), ("edm_dpm++_2m", 4.0), ("spaced", 1.0)])
def test_chunked_tiled_sampling_bit_identical(sampler, cfg):
    """Latent 80 x 128 with 64-wide tiles at stride 16: a 2 x 5 tile grid, 10 tiles per branch, two images.
    Caps 6 and 8 split each branch into chunks of 3 (3, 3, 3, 1) and 4 (4, 4, 2) tiles; then one replay again."""
    pipe = _small_pipe()
    cl = pipe.cldm
    cl._build()
    B, H, W = 2, 80, 128
    cond, unc, xT = _conditions(cl, B, H, W)
    z0, st0 = _sample(pipe, sampler, 128, cond, unc, xT, cfg)
    assert st0["tiles"] == 10 and st0["chunks"] == 1
    nbr = 2 if cfg != 1.0 else 1
    # the last run is unchunked again: it must not see anything the chunked runs left in the engine
    for cap, chunks in ((6, 4 * nbr), (8, 3 * nbr), (128, 1)):
        z, st = _sample(pipe, sampler, cap, cond, unc, xT, cfg)
        print(f"{sampler} cfg {cfg}: cap {cap}: {st['chunks']} chunks of <= {st['forwards_per_step']} entries")
        assert st["chunks"] == chunks and st["forwards_per_step"] <= cap
        assert torch.isfinite(z).all() and torch.equal(z, z0), f"cap {cap}"


def test_engine_reused_across_batch_sizes():
    """One engine serves forwards of many batch sizes: chunked tiled sampling (6-entry replays), the generic
    ControlLDM.forward with 4 and 40 images and un-chunked tiled sampling (40 entries) in any order give the bits of
    a forward on a freshly released engine."""
    pipe = _small_pipe()
    cl = pipe.cldm
    cl._build()
    g = torch.Generator().manual_seed(23)
    n, L_ = 40, 64
    x = torch.randn(n, 4, L_, L_, generator=g).cuda()
    ci = torch.randn(n, 4, L_, L_, generator=g).cuda()
    ctx = torch.randn(n, 77, cl.unet_cfg["context_dim"], generator=g).cuda()
    t = torch.full((n,), 500, device="cuda")
    cl.engine.batch_invariant = True

    def generic(k):
        return cl(x[:k].contiguous(), t[:k], dict(c_txt=ctx[:k].contiguous(), c_img=ci[:k].contiguous())).clone()

    cl.release_engine_buffers()
    ref = generic(n)
    cond, unc, xT = _conditions(cl, 2, 80, 128)
    cl.release_engine_buffers()
    z_ref, _ = _sample(pipe, "ddim", 128, cond, unc, xT, 4.0)
    _sample(pipe, "ddim", 6, cond, unc, xT, 4.0)
    assert torch.equal(generic(n), ref)
    generic(4)
    assert torch.equal(generic(n), ref)
    _sample(pipe, "ddim", 6, cond, unc, xT, 4.0)
    z, st = _sample(pipe, "ddim", 128, cond, unc, xT, 4.0)
    assert st["chunks"] == 1 and torch.equal(z, z_ref)


def test_chunked_pipeline_uint8_bit_identical():
    """SwinIRPipeline.run at 640 x 1024 (latent 80 x 128, 512-pixel tiles at stride 128: 10 tiles per branch),
    unchunked and with caps 4 (chunks 4, 4, 2) and 6 (5, 5): identical latents and uint8 images."""
    pipe = _small_pipe()
    lq = synthetic_lq(640, 1024, seed=7)
    kw = dict(RUN_DEFAULTS, steps=4, cldm_tiled=True, cldm_tile_size=512, cldm_tile_stride=128)
    outs = []
    for cap in (128, 4, 6):
        pipe.max_tile_forwards = cap
        pipe.taps = {}
        torch.manual_seed(231)
        out = pipe.run(lq, **kw)
        outs.append((out, pipe.taps["z"].clone(), pipe.last_sampler.last_stats["chunks"]))
    pipe.max_tile_forwards = 128
    pipe.taps = None
    assert [o[2] for o in outs] == [1, 6, 4]
    for out, z, _ in outs[1:]:
        assert out.dtype == np.uint8 and np.array_equal(out, outs[0][0])
        assert torch.equal(z, outs[0][1])


def test_chunked_sampler_memory_bounded():
    """Cap 4 (one image): 4 tiles (8 units) and 16 tiles (32 units) replay the same 4-entry graph, so the sampler
    loop's peak memory differs by the latent-sized buffers only; without the cap the 16-tile run holds 32 entries."""
    pipe = _small_pipe()
    cl = pipe.cldm
    cl._build()

    def peak(side, cap):
        cond, unc, xT = _conditions(cl, 1, side, side, seed=side)
        cl.release_engine_buffers()
        _free()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        _, st = _sample(pipe, "spaced", cap, cond, unc, xT, 4.0, steps=2)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base, st

    p4, s4 = peak(80, 4)                   # 2 x 2 tiles
    p16, s16 = peak(112, 4)                # 4 x 4 tiles
    pu, su = peak(112, 128)                # 4 x 4 tiles, one replay of 32 entries
    cl.release_engine_buffers()
    assert (s4["tiles"], s16["tiles"]) == (4, 16) and s4["forwards_per_step"] == s16["forwards_per_step"] == 4
    assert su["chunks"] == 1 and su["forwards_per_step"] == 32
    # what may grow with the latent: x, x_next, noise, the blend output, the per-unit eps / condition tiles
    latent = 4 * 112 * 112 * 4
    unit_tiles = 2 * 16 * 4 * 64 * 64 * 4
    allow = 32 * latent + 4 * unit_tiles
    print(f"sampler-loop peak: 4 tiles {p4 / 2**20:.1f} MiB, 16 tiles {p16 / 2**20:.1f} MiB (cap 4), "
          f"16 tiles unchunked {pu / 2**20:.1f} MiB; allowance {allow / 2**20:.1f} MiB")
    assert p16 - p4 <= allow
    assert pu > p16 + 2 * allow


# ---------------------------------------------------------------- full configuration
_FULL = {}


def _full_pipe():
    no_tf32()
    if "p" not in _FULL:
        _SMALL.clear()
        _free()
        _FULL["p"] = build_synthetic_pipeline("cuda", seed=1234, small=False)
    return _FULL["p"]


def test_full_config_tiled_1024_chunked_bit_identical():
    """Full configuration at 1024^2 (latent 128^2, 9 tiles, 18 tile-forwards, 2 spaced steps): one replay of 18
    entries against cap 8, which splits each branch into chunks of 5 and 4 tiles replayed as a 6-entry graph (padded
    to an even size so the UNet / ControlNet twin layers keep their grouped launches). Same latent, same image."""
    pipe = _full_pipe()
    lq = synthetic_lq(1024, 1024, seed=4)
    kw = dict(RUN_DEFAULTS, steps=2, cldm_tiled=True, cldm_tile_size=512, cldm_tile_stride=256)
    outs = []
    for cap in (128, 8, 128):
        pipe.max_tile_forwards = cap
        pipe.taps = {}
        torch.manual_seed(231)
        out = pipe.run(lq, **kw)
        st = pipe.last_sampler.last_stats
        outs.append((out, pipe.taps["z"].clone(), st["chunks"], st["forwards_per_step"]))
    pipe.max_tile_forwards = 128
    pipe.taps = None
    assert [o[2:] for o in outs] == [(1, 18), (4, 6), (1, 18)]
    assert pipe.cldm.engine.twins_feasible(6, 64, 64) and not pipe.cldm.engine.twins_feasible(5, 64, 64)
    for out, z, _, _ in outs[1:]:
        assert np.array_equal(out, outs[0][0]) and torch.equal(z, outs[0][1])


def test_full_config_tiled_3072():
    """SwinIRPipeline at 3072^2 on one H100: tiled SwinIR, tiled sampling over 121 latent tiles (242 tile-forwards),
    2 spaced steps, un-tiled VAE. The default cap runs one 122-entry replay per branch; cap 64 runs four 62-entry
    replays. Both must finish with the same finite uint8 image."""
    pipe = _full_pipe()
    lq = synthetic_lq(3072, 3072, seed=8)
    kw = dict(RUN_DEFAULTS, steps=2, cldm_tiled=True, cleaner_tiled=True)
    outs = []
    for cap in (128, 64):
        pipe.max_tile_forwards = cap
        torch.cuda.reset_peak_memory_stats()
        torch.manual_seed(231)
        out = pipe.run(lq, **kw)
        st = pipe.last_sampler.last_stats
        print(f"3072^2 tiled, cap {cap}: {st['tiles']} tiles, {st['chunks']} chunks of {st['forwards_per_step']} entries, "
              f"peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB on {torch.cuda.get_device_name()}")
        outs.append((out, st["chunks"]))
    assert [c for _, c in outs] == [2, 4]
    out = outs[0][0]
    assert out.shape == (1, 3072, 3072, 3) and out.dtype == np.uint8 and 0 < out.std()
    assert np.array_equal(outs[1][0], out)
    pipe.max_tile_forwards = 128
    del pipe
    _FULL.clear()
    _free()
