"""-m gpu: per-kernel parity of the C-ABI entry points against torch fp32 (TF32 off) on the same
16-bit-rounded operands. Tolerances: fp32 outputs 2e-5 of max (accumulation order only);
16-bit outputs 1.5e-3 (one fp16 rounding, 2^-11) / 1e-2 for bf16 builds."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.gpu_util import no_tf32, rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from diffbir_b200 import lib
    lib.load()
    no_tf32()
    return lib


def g(seed=0):
    return torch.Generator(device="cuda").manual_seed(seed)


def rnd(*s, seed=0, scale=1.0):
    return torch.randn(*s, device="cuda", generator=g(seed)) * scale


def tol16(L):
    return 1.5e-3 if L.operand_dtype() == torch.float16 else 1e-2


@pytest.mark.parametrize("M,N,K,fbn", [(256, 64, 64, 0), (4109, 320, 320, 0), (2048, 640, 2560, 0),
                                         (512, 1280, 1280, 0), (1024, 320, 640, 160), (777, 200, 200, 0),
                                         (300, 24, 128, 0)])
def test_gemm_plain(L, M, N, K, fbn):
    dt = L.operand_dtype()
    a, b = rnd(M, K, seed=1).to(dt), rnd(N, K, seed=2, scale=K ** -0.5).to(dt)
    bias, res = rnd(N, seed=3), rnd(M, N, seed=4)
    out = torch.empty(M, N, device="cuda")
    out16 = torch.empty(M, N + 8, device="cuda", dtype=dt)
    L.gemm(a, b, out, M=M, N=N, K=K, bias=bias, residual=res, force_bn=fbn, alpha=0.7)
    L.gemm(a, b, out16, M=M, N=N, K=K, bias=bias, residual=res, force_bn=fbn, alpha=0.7, ldo=N + 8)
    ref = 0.7 * (a.float() @ b.float().t() + bias) + res
    assert rel_err(out, ref) < 2e-5
    assert rel_err(out16[:, :N], ref) < tol16(L)
    inplace = res.clone()
    L.gemm(a, b, inplace, M=M, N=N, K=K, bias=bias, residual=inplace, force_bn=fbn, alpha=0.7)
    assert torch.equal(inplace, out)


def test_gemm_bias_per_row_and_strides(L):
    dt = L.operand_dtype()
    M, N, K = 512, 1000, 512
    a = rnd(M, K, seed=1).to(dt)
    bfull = rnd(N, 2 * K, seed=2, scale=K ** -0.5).to(dt)
    bias = rnd(M, seed=3)
    out = torch.empty(M, N + 8, device="cuda", dtype=dt)
    L.gemm(a, bfull[:, K:], out, M=M, N=N, K=K, ldb=2 * K, ldo=N + 8, bias=bias, bias_per_row=True)
    ref = a.float() @ bfull[:, K:].float().t() + bias[:, None]
    assert rel_err(out[:, :N], ref) < tol16(L)


@pytest.mark.parametrize("M,C,fbn", [(4096, 320, 256), (300, 1280, 128), (1024, 640, 256), (200, 64, 256)])
def test_gemm_geglu(L, M, C, fbn):
    from diffbir_b200.engine.common import pack_geglu
    dt = L.operand_dtype()
    inner = 4 * C
    a = rnd(M, C, seed=1).to(dt)
    w = rnd(2 * inner, C, seed=2, scale=C ** -0.5)
    bias = rnd(2 * inner, seed=3)
    wp, bp = pack_geglu(w, bias, fbn, "cuda")
    out = torch.empty(M, inner, device="cuda", dtype=dt)
    L.gemm(a, wp, out, M=M, N=2 * inner, K=C, bias=bp, geglu=True, force_bn=fbn)
    hcat = a.float() @ w.to(dt).float().t() + bias
    ref = hcat[:, :inner] * F.gelu(hcat[:, inner:])
    assert rel_err(out, ref) < tol16(L)


@pytest.mark.parametrize("n,h,w,cin,cout,ks", [(2, 64, 64, 320, 320, 3), (2, 16, 16, 1280, 1280, 3),
                                                (2, 8, 8, 1280, 1280, 3), (1, 8, 8, 1280, 640, 3),
                                                (2, 32, 32, 1920, 640, 3), (1, 40, 72, 128, 192, 3),
                                                (1, 2, 2, 256, 256, 3), (3, 4, 4, 128, 64, 3),
                                                (2, 16, 16, 1280, 1280, 1)])
def test_gemm_conv(L, n, h, w, cin, cout, ks):
    dt = L.operand_dtype()
    x = rnd(n, h, w, cin, seed=1).to(dt)
    wt = rnd(cout, cin, ks, ks, seed=2, scale=(cin * ks * ks) ** -0.5).to(dt)
    bias, rv = rnd(cout, seed=3), rnd(n, cout, seed=4)
    res = rnd(n * h * w, cout, seed=5)
    wp = wt.permute(0, 2, 3, 1).reshape(cout, -1).contiguous()
    out = torch.empty(n * h * w, cout, device="cuda")
    L.gemm(x, wp, out, M=n * h * w, N=cout, K=ks * ks * cin, bias=bias, rowvec=rv, residual=res,
           conv=(n, h, w, cin, ks))
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), bias, padding=ks // 2) + rv[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1).reshape(n * h * w, cout) + res
    assert rel_err(out, ref) < 3e-5


@pytest.mark.parametrize("b,heads,sq,skv", [(2, 5, 4096, 4096), (2, 10, 1024, 1024), (2, 20, 256, 256),
                                             (2, 20, 64, 64), (2, 5, 4096, 77), (1, 20, 64, 77),
                                             (1, 1, 4, 4), (3, 2, 200, 333)])
def test_attention(L, b, heads, sq, skv):
    dt = L.operand_dtype()
    c = heads * 64
    self_attn = sq == skv
    if self_attn:
        qkv = rnd(b * sq, 3 * c, seed=1).to(dt)
        q, k, v = qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:]
        ldq = ldk = ldv = 3 * c
    else:
        q = rnd(b * sq, c, seed=1).to(dt)
        kv = rnd(b * skv, 2 * c, seed=2).to(dt)
        k, v = kv[:, :c], kv[:, c:]
        ldq, ldk, ldv = c, 2 * c, 2 * c
    out = torch.empty(b * sq, c, device="cuda", dtype=dt)
    L.attention(q, k, v, out, batch=b, heads=heads, sq=sq, skv=skv, ldq=ldq, ldk=ldk, ldv=ldv, ldo=c)

    def split(t, s):
        return t.float().reshape(b, s, heads, 64).permute(0, 2, 1, 3)
    ref = F.scaled_dot_product_attention(split(q, sq), split(k, skv), split(v, skv))
    ref = ref.permute(0, 2, 1, 3).reshape(b * sq, c)
    assert rel_err(out, ref) < 2 * tol16(L)
    # stream-K decomposition (tiles cut by CTA boundaries are combined through a workspace):
    # same result up to the combine's rounding, bit-identical across runs, tickets self-reset
    nws = L.attention_ws_bytes(b, heads, sq, skv)
    assert (nws > 0) == ((b, heads, sq, skv) == (2, 5, 4096, 4096))
    if nws:
        ws = torch.zeros(nws // 4, device="cuda")
        o1, o2 = torch.empty_like(out), torch.empty_like(out)
        for o in (o1, o2):
            L.attention(q, k, v, o, batch=b, heads=heads, sq=sq, skv=skv, ldq=ldq, ldk=ldk, ldv=ldv, ldo=c, ws=ws)
        assert rel_err(o1, ref) < 2 * tol16(L)
        assert torch.equal(o1, o2)
        assert (ws[:16384] == 0).all()


@pytest.mark.parametrize("n,h,w,c1,c2", [(2, 64, 64, 320, 0), (2, 16, 16, 1280, 640), (2, 32, 32, 640, 320),
                                          (1, 2, 2, 256, 256), (1, 128, 128, 128, 0)])
@pytest.mark.parametrize("up", [1, 2])
def test_groupnorm(L, n, h, w, c1, c2, up):
    dt = L.operand_dtype()
    c = c1 + c2
    s1 = rnd(n, h, w, c1, seed=1) * 2 + 0.5
    s2 = rnd(n, h, w, c2, seed=2) if c2 else None
    gamma, beta = 1 + 0.1 * rnd(c, seed=3), 0.1 * rnd(c, seed=4)
    stats = torch.empty(n * 64, device="cuda")
    ws = torch.zeros(L.gn_workspace_floats(n, h * w, c), device="cuda")
    out = torch.empty(n, h * up, w * up, c, device="cuda", dtype=dt)
    raw = torch.empty(n, h, w, c, device="cuda", dtype=dt) if up == 1 else None
    for _ in range(2):   # second pass checks the self-resetting tickets
        L.gn_stats(s1, s2, c1, c2, n, h * w, 1e-5, stats, ws)
    L.gn_apply(s1, s2, c1, c2, n, h, w, stats, gamma, beta, out, norm=True, silu=True, upsample=up, out_raw=raw)
    x = torch.cat([s1, s2], -1) if c2 else s1
    ref = F.silu(F.group_norm(x.permute(0, 3, 1, 2), 32, gamma, beta, 1e-5))
    if up == 2:
        ref = F.interpolate(ref, scale_factor=2, mode="nearest")
    ref = ref.permute(0, 2, 3, 1)
    assert rel_err(out, ref) < tol16(L)
    if raw is not None:
        assert rel_err(raw, x) < tol16(L)


@pytest.mark.parametrize("rows,c,ldo", [(8192, 320, 320), (100, 1280, 1280), (4096, 180, 192), (77, 640, 640)])
def test_layernorm(L, rows, c, ldo):
    dt = L.operand_dtype()
    ldx = ldo
    x = torch.zeros(rows, ldx, device="cuda")
    x[:, :c] = rnd(rows, c, seed=1) * 3 + 1
    gamma, beta = 1 + 0.1 * rnd(c, seed=2), 0.1 * rnd(c, seed=3)
    out = torch.full((rows, ldo), 7.0, device="cuda", dtype=dt)
    L.layernorm(x, ldx, rows, c, gamma, beta, out, ldo)
    ref = F.layer_norm(x[:, :c], (c,), gamma, beta, 1e-5)
    assert rel_err(out[:, :c], ref) < tol16(L)
    assert (out[:, c:] == 0).all()
    out32 = torch.empty(rows, ldo, device="cuda")
    L.layernorm(x, ldx, rows, c, gamma, beta, out32, ldo)
    assert rel_err(out32[:, :c], ref) < 1e-5


def test_small_convs_im2col_linear(L):
    dt = L.operand_dtype()
    n, h, w = 2, 32, 24
    x1, x2 = rnd(n, 4, h, w, seed=1), rnd(n, 4, h, w, seed=2)
    wt = rnd(320, 8, 3, 3, seed=3, scale=0.1)
    bias = rnd(320, seed=4)
    out = torch.empty(n * h * w, 320, device="cuda")
    L.conv3x3_small_cin(x1, x2, 4, 4, n, h, w, wt.permute(2, 3, 1, 0).reshape(-1, 320).contiguous(), bias, 320, out)
    ref = F.conv2d(torch.cat([x1, x2], 1), wt, bias, padding=1).permute(0, 2, 3, 1).reshape(-1, 320)
    assert rel_err(out, ref) < 1e-5
    for cout in (3, 4, 8):
        xin = rnd(n, h, w, 128, seed=5).to(dt)
        wt = rnd(cout, 128, 3, 3, seed=6, scale=0.03)
        bias = rnd(cout, seed=7)
        shift = rnd(cout, seed=8)
        o = torch.empty(n, cout, h, w, device="cuda")
        L.conv3x3_small_cout(xin, n, h, w, 128, wt.permute(0, 2, 3, 1).reshape(cout, -1).contiguous(), bias, cout, o,
                             nchw=True, post_scale=0.5, post_shift=shift)
        ref = F.conv2d(xin.float().permute(0, 3, 1, 2), wt, bias, padding=1) * 0.5 + shift.view(1, -1, 1, 1)
        assert rel_err(o, ref) < 1e-5
    # im2col stride 2, both paddings
    x = rnd(n, h, w, 64, seed=9)
    for pad_lo in (1, 0):
        ho, wo = h // 2, w // 2
        col = torch.empty(n * ho * wo, 9 * 64, device="cuda", dtype=dt)
        L.im2col_s2(x, n, h, w, 64, pad_lo, col)
        xp = x.permute(0, 3, 1, 2)
        xp = F.pad(xp, (1, 1, 1, 1)) if pad_lo else F.pad(xp, (0, 1, 0, 1))
        ref = F.unfold(xp, 3, stride=2)                               # [n, c*9, L] (c-major)
        ref = ref.view(n, 64, 9, ho * wo).permute(0, 3, 2, 1).reshape(n * ho * wo, 9 * 64)
        assert rel_err(col, ref) < tol16(L)
    # fp32 linear with silu in/out
    xm = rnd(50, 1280, seed=10)
    wl, bl = rnd(640, 1280, seed=11, scale=0.03), rnd(640, seed=12)
    y = torch.empty(50, 640, device="cuda")
    L.linear_f32(xm, 1280, 50, 1280, wl, bl, 640, y, 640, silu_in=True, silu_out=True)
    assert rel_err(y, F.silu(F.linear(F.silu(xm), wl, bl))) < 1e-5
    # timestep embedding
    t = torch.tensor([0.0, 1.0, 500.0, 999.0], device="cuda")
    te = torch.empty(4, 320, device="cuda")
    L.timestep_embedding(t, 4, 320, te)
    freqs = torch.exp(-math.log(10000.0) * torch.arange(160, dtype=torch.float32, device="cuda") / 160)
    args = t[:, None] * freqs[None]
    # one fp32 ulp in a frequency is worth 6e-5 rad at t = 999: both sides are "exact" to that
    assert rel_err(te, torch.cat([torch.cos(args), torch.sin(args)], -1)) < 2e-4
    # row softmax
    s = rnd(300, 1000, seed=13) * 4
    p16 = torch.empty(300, 1000, device="cuda", dtype=dt)
    L.softmax_rows(s, 1000, 300, 1000, 0.3, p16, 1000)
    assert rel_err(p16, torch.softmax(s * 0.3, -1)) < tol16(L)


def test_sampler_step_and_tiles_bit_exact(L, golden_dir):
    from oracle import sampling as osm
    x, ec, eu, nz = (rnd(1, 4, 24, 40, seed=i) for i in (1, 2, 3, 4))
    coef = torch.tensor([1.7, 0.9, 0.3, 0.6, 0.2, 0.8, 0, 0], device="cuda")
    out = torch.empty_like(x)
    L.sampler_step(ec, eu, 4.0, x, nz, coef, 0, x.numel(), out)
    e = eu + 4.0 * (ec - eu)
    x0 = coef[0] * x - coef[1] * e
    ref = (coef[2] * x0 + coef[3] * x) + coef[4] * nz
    assert torch.equal(out, ref)
    L.sampler_step(ec, eu, 4.0, x, nz, coef, 3, x.numel(), out)
    e2 = coef[5] * e + coef[1] * x
    x0 = (x - coef[1] * e2) / coef[0]
    ref = coef[2] * x0 + coef[3] * e2 + coef[4] * nz
    assert torch.equal(out, ref)
    # modes 1 (spaced, v: same update as mode 0) and 2 (DDIM, eps), each also without CFG (eps_uncond NULL)
    # and without noise (NULL: the last step)
    for ecu in (eu, None):
        for noise in (nz, None):
            e = ec if ecu is None else ecu + 4.0 * (ec - ecu)
            n_ = torch.zeros_like(x) if noise is None else noise
            L.sampler_step(ec, ecu, 4.0, x, noise, coef, 1, x.numel(), out)
            x0 = coef[0] * x - coef[1] * e
            assert torch.equal(out, (coef[2] * x0 + coef[3] * x) + coef[4] * n_)
            L.sampler_step(ec, ecu, 4.0, x, noise, coef, 2, x.numel(), out)
            x0 = (x - coef[1] * e) / coef[0]
            assert torch.equal(out, coef[2] * x0 + coef[3] * e + coef[4] * n_)
    # tile gather / blend against the reference-order accumulation of the oracle
    H, W, ts, stride = 24, 40, 16, 8
    wins = osm.sliding_windows(H, W, ts, stride)
    coords = torch.tensor([[a, c] for a, _, c, _ in wins], dtype=torch.int32, device="cuda")
    wts = torch.tensor(osm.gaussian_weights(ts, ts), dtype=torch.float32, device="cuda")
    full = rnd(2, 4, H, W, seed=5)
    tiles = torch.empty(len(wins), 2, 4, ts, ts, device="cuda")
    L.tile_gather(full, 2, 4, H, W, coords, len(wins), ts, tiles)
    for i, (a, b_, c, d) in enumerate(wins):
        assert torch.equal(tiles[i], full[..., a:b_, c:d])
    tiles = tiles * 1.37 + 0.1
    blended = torch.empty(2, 4, H, W, device="cuda")
    L.tile_blend(tiles, 2, 4, H, W, coords, len(wins), ts, wts, blended)
    acc, cnt = torch.zeros_like(full), torch.zeros_like(full)
    for i, (a, b_, c, d) in enumerate(wins):
        acc[..., a:b_, c:d] += tiles[i] * wts
        cnt[..., a:b_, c:d] += wts
    assert torch.equal(blended, acc / cnt)


@pytest.mark.parametrize("M,N,K,fbn", [(256, 64, 64, 64), (512, 1280, 1280, 0), (2048, 640, 2560, 0),
                                         (8192, 320, 320, 0), (4000, 320, 320, 160), (1024, 200, 448, 64),
                                         (2048, 1280, 640, 256)])
def test_gemm_cta_pair_plain(L, M, N, K, fbn):
    """CTA-pair path (2-CTA cluster sharing the B tile by TMA multicast): same fp32 result as the single-CTA
    path up to accumulation order (identical here: same k order), and vs the fp32 reference."""
    dt = L.operand_dtype()
    a, b = rnd(M, K, seed=1).to(dt), rnd(N, K, seed=2, scale=K ** -0.5).to(dt)
    bias, res = rnd(N, seed=3), rnd(M, N, seed=4)
    o1, o2 = torch.empty(M, N, device="cuda"), torch.empty(M, N, device="cuda")
    L.gemm(a, b, o1, M=M, N=N, K=K, bias=bias, residual=res, force_bn=fbn, alpha=0.7, cta_pair=1, split_k=1)
    L.gemm(a, b, o2, M=M, N=N, K=K, bias=bias, residual=res, force_bn=fbn, alpha=0.7, cta_pair=2, split_k=1)
    ref = 0.7 * (a.float() @ b.float().t() + bias) + res
    assert rel_err(o1, ref) < 2e-5
    assert torch.equal(o1, o2)
    o16 = torch.empty(M, N, device="cuda", dtype=dt)
    L.gemm(a, b, o16, M=M, N=N, K=K, bias=bias, act="gelu", force_bn=fbn, cta_pair=1)
    assert rel_err(o16, F.gelu(a.float() @ b.float().t() + bias)) < tol16(L)


@pytest.mark.parametrize("n,h,w,cin,cout,fbn,split", [(2, 64, 64, 320, 320, 0, 0), (2, 16, 16, 1280, 1280, 0, 0),
                                                       (2, 32, 32, 640, 640, 128, 0), (2, 32, 32, 1920, 640, 256, 0),
                                                       (2, 16, 16, 1280, 1280, 128, 3), (1, 40, 72, 128, 192, 64, 0)])
def test_gemm_cta_pair_conv(L, n, h, w, cin, cout, fbn, split):
    dt = L.operand_dtype()
    x = rnd(n, h, w, cin, seed=1).to(dt)
    wt = rnd(cout, cin, 3, 3, seed=2, scale=(cin * 9) ** -0.5).to(dt)
    bias, rv = rnd(cout, seed=3), rnd(n, cout, seed=4)
    res = rnd(n * h * w, cout, seed=5)
    wp = wt.permute(0, 2, 3, 1).reshape(cout, -1).contiguous()
    ws = torch.zeros(16 * 1024 * 1024 + 16384, device="cuda")
    slots = L.gemm_gn_slots(conv_h=h, conv_w=w)
    outs, parts = [], []
    for pair in (1, 2):
        out = torch.empty(n * h * w, cout, device="cuda")
        part = torch.zeros(n, slots, cout, 2, device="cuda")
        L.gemm(x, wp, out, M=n * h * w, N=cout, K=9 * cin, bias=bias, rowvec=rv, residual=res,
               conv=(n, h, w, cin, 3), force_bn=fbn, splitk_ws=ws, split_k=split if split else 1,
               gn_partials=part, cta_pair=pair)
        outs.append(out)
        parts.append(part)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), bias, padding=1) + rv[:, :, None, None]
    ref = ref.permute(0, 2, 3, 1).reshape(n * h * w, cout) + res
    assert rel_err(outs[0], ref) < 3e-5
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(parts[0], parts[1])
    assert (ws[:16384] == 0).all()


def test_gemm_cta_pair_geglu(L):
    from diffbir_b200.engine.common import pack_geglu
    dt = L.operand_dtype()
    M, C, fbn = 2048, 640, 128
    inner = 4 * C
    a = rnd(M, C, seed=1).to(dt)
    w = rnd(2 * inner, C, seed=2, scale=C ** -0.5)
    bias = rnd(2 * inner, seed=3)
    wp, bp = pack_geglu(w, bias, fbn, "cuda")
    o1 = torch.empty(M, inner, device="cuda", dtype=dt)
    o2 = torch.empty(M, inner, device="cuda", dtype=dt)
    L.gemm(a, wp, o1, M=M, N=2 * inner, K=C, bias=bp, geglu=True, force_bn=fbn, cta_pair=1)
    L.gemm(a, wp, o2, M=M, N=2 * inner, K=C, bias=bp, geglu=True, force_bn=fbn, cta_pair=2)
    hcat = a.float() @ w.to(dt).float().t() + bias
    assert rel_err(o1, hcat[:, :inner] * F.gelu(hcat[:, inner:])) < tol16(L)
    assert torch.equal(o1, o2)


@pytest.mark.parametrize("n,h,w,cin,cout,split", [(2, 8, 8, 1280, 1280, 0), (2, 8, 8, 1280, 1280, 7),
                                                   (2, 16, 16, 1280, 1280, 3), (1, 8, 8, 2560, 1280, 0)])
def test_gemm_split_k_deterministic(L, n, h, w, cin, cout, split):
    """Split-K (small-M, long-K layers): same result as the fp32 reference, bit-identical across
    runs (fixed summation order), workspace tickets self-reset."""
    dt = L.operand_dtype()
    x = rnd(n, h, w, cin, seed=1).to(dt)
    wt = rnd(cout, cin, 3, 3, seed=2, scale=(cin * 9) ** -0.5).to(dt)
    bias, res = rnd(cout, seed=3), rnd(n * h * w, cout, seed=5)
    wp = wt.permute(0, 2, 3, 1).reshape(cout, -1).contiguous()
    ws = torch.zeros(16 * 1024 * 1024 + 16384, device="cuda")
    outs = []
    for _ in range(3):
        out = torch.empty(n * h * w, cout, device="cuda")
        L.gemm(x, wp, out, M=n * h * w, N=cout, K=9 * cin, bias=bias, residual=res, conv=(n, h, w, cin, 3),
               splitk_ws=ws, split_k=split)
        outs.append(out)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), wt.float(), bias, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(n * h * w, cout) + res
    assert rel_err(outs[0], ref) < 3e-5
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
    assert (ws[:16384] == 0).all()


@pytest.mark.parametrize("n,h,w,c1,c2", [(2, 64, 64, 320, 0), (2, 16, 16, 1280, 640), (2, 8, 8, 1280, 1280),
                                          (1, 40, 72, 128, 64), (3, 8, 16, 64, 0)])
def test_fused_groupnorm_statistics(L, n, h, w, c1, c2):
    """GN statistics from the partial sums emitted by the producing GEMM epilogues (conv mode for
    source 1, matrix mode for source 2) == statistics of the stored tensors."""
    dt = L.operand_dtype()
    hw = h * w
    outs, parts = [], []
    for idx, c in enumerate([c1, c2]):
        if c == 0:
            outs.append(None); parts.append((None, 0)); continue
        cin = 64
        x = rnd(n, h, w, cin, seed=10 + idx).to(dt)
        res = rnd(n * hw, c, seed=20 + idx) * 2 + 0.3
        out = torch.empty(n * hw, c, device="cuda")
        if idx == 0:
            wt = rnd(c, 9 * cin, seed=30, scale=0.05).to(dt)
            slots = L.gemm_gn_slots(h, w)
            part = torch.zeros(n * slots * c * 2, device="cuda")
            L.gemm(x, wt, out, M=n * hw, N=c, K=9 * cin, residual=res, conv=(n, h, w, cin, 3), gn_partials=part)
        else:
            wt = rnd(c, cin, seed=31, scale=0.1).to(dt)
            slots = L.gemm_gn_slots(0, 0, hw)
            part = torch.zeros(n * slots * c * 2, device="cuda")
            L.gemm(x.view(n * hw, cin), wt, out, M=n * hw, N=c, K=cin, residual=res, gn_partials=part, gn_rows_per_img=hw)
        assert slots > 0
        outs.append(out); parts.append((part, slots))
    stats = torch.empty(n * 64, device="cuda")
    L.gn_finalize(parts[0][0], parts[0][1], c1, parts[1][0], parts[1][1], c2, n, hw, 1e-5, stats)
    full = outs[0].view(n, hw, c1) if c2 == 0 else torch.cat([outs[0].view(n, hw, c1), outs[1].view(n, hw, c2)], -1)
    c = c1 + c2
    g = full.view(n, hw, 32, c // 32).permute(0, 2, 1, 3).reshape(n, 32, -1).double()
    mean, var = g.mean(-1), g.var(-1, unbiased=False)
    st = stats.view(n, 32, 2)
    assert (st[..., 0].double() - mean).abs().max() < 1e-4 * (mean.abs().max() + 1)
    assert ((st[..., 1].double() - 1 / (var + 1e-5).sqrt()).abs() / (1 / (var + 1e-5).sqrt())).max() < 1e-4


@pytest.mark.parametrize("b,h,w,shift", [(1, 64, 64, 0), (1, 64, 64, 4), (2, 16, 24, 4), (1, 128, 64, 4)])
def test_window_attention_swinir(L, b, h, w, shift):
    """dbir_window_attention with SwinIR's 6 heads x 30 and shift mask -100, stand-alone (WindowAttention.forward
    + roll / partition / reverse / shift mask, swinir.py:120-151, 245-285) vs the oracle's op sequence in fp32 on
    the same 16-bit qkv."""
    from oracle.swinir import rel_pos_index, shift_mask
    heads, dh, ws = 6, 30, 8
    c = heads * dh
    g = torch.Generator().manual_seed(11)
    lib, dt = L, L.operand_dtype()
    ld = 544
    qkv = torch.zeros(b * h * w, ld, dtype=dt, device="cuda")
    qkv[:, :3 * c] = (torch.randn(b * h * w, 3 * c, generator=g) * 1.5).to("cuda", dt)
    table = (torch.randn(225, heads, generator=g) * 0.5).cuda()
    out = torch.zeros(b * h * w, 192, dtype=dt, device="cuda")
    lib.window_attention(qkv, ld, b, h, w, heads, dh, shift, table, -100.0, out, 192)
    # reference (fp32, on the fp16/bf16-rounded qkv)
    y = qkv[:, :3 * c].float().view(b, h, w, 3 * c)
    if shift:
        y = torch.roll(y, (-shift, -shift), (1, 2))
    win = y.view(b, h // ws, ws, w // ws, ws, 3 * c).permute(0, 1, 3, 2, 4, 5).reshape(-1, ws * ws, 3 * c)
    nwin = win.shape[0]
    t = win.view(nwin, ws * ws, 3, heads, dh).permute(2, 0, 3, 1, 4)
    q, k, v = t[0] * dh ** -0.5, t[1], t[2]
    attn = q @ k.transpose(-1, -2)
    bias = table[rel_pos_index(ws).to("cuda").view(-1)].view(ws * ws, ws * ws, heads).permute(2, 0, 1)
    attn = attn + bias[None]
    if shift:
        m = shift_mask(h, w, ws, shift, "cuda")
        attn = (attn.view(b, m.shape[0], heads, ws * ws, ws * ws) + m[None, :, None]).view(nwin, heads, ws * ws, ws * ws)
    o = (torch.softmax(attn, dim=-1) @ v).transpose(1, 2).reshape(nwin, ws * ws, c)
    o = o.view(b, h // ws, w // ws, ws, ws, c).permute(0, 1, 3, 2, 4, 5).reshape(b, h, w, c)
    if shift:
        o = torch.roll(o, (shift, shift), (1, 2))
    ref = o.reshape(b * h * w, c)
    err = rel_err(out[:, :c], ref)
    assert err < (4e-3 if dt == torch.float16 else 2e-2), err
    assert out[:, c:].abs().max().item() == 0.0      # pad columns untouched


@pytest.mark.parametrize("M,N,K,geglu", [(256, 320, 320, False), (1024, 640, 640, False), (256, 1280, 1280, False),
                                         (512, 2560, 320, True)])
def test_gemm_grouped_plain(L, M, N, K, geglu):
    """groups = 2 (twin UNet / ControlNet layers stacked along M, weights / bias stacked along N) is
    bit-identical to the two separate launches with the split pinned off (same per-row arithmetic)."""
    from diffbir_b200.engine.common import pack_geglu
    dt = L.operand_dtype()
    G = 2
    a = rnd(G * M, K, seed=1).to(dt)
    ws = [rnd(N, K, seed=10 + g, scale=K ** -0.5) for g in range(G)]
    bs = [rnd(N, seed=20 + g) for g in range(G)]
    kw = dict(split_k=1)
    if geglu:
        packed = [pack_geglu(w, b, 128, "cuda") for w, b in zip(ws, bs)]
        ws, bs = [p[0] for p in packed], [p[1] for p in packed]
        kw.update(geglu=True, force_bn=128)
        n_out, res = N // 2, None
    else:
        ws = [w.to(dt) for w in ws]
        n_out, res = N, rnd(G * M, N, seed=4)
    wcat, bcat = torch.cat(ws, 0).contiguous(), torch.cat(bs, 0).contiguous()
    out_dt = dt if geglu else torch.float32
    out = torch.empty(G * M, n_out, device="cuda", dtype=out_dt)
    L.gemm(a, wcat, out, M=G * M, N=N, K=K, bias=bcat, residual=res, groups=G, **kw)
    for g in range(G):
        sep = torch.empty(M, n_out, device="cuda", dtype=out_dt)
        L.gemm(a[g * M:(g + 1) * M], ws[g], sep, M=M, N=N, K=K, bias=bs[g],
               residual=None if res is None else res[g * M:(g + 1) * M], **kw)
        assert torch.equal(out[g * M:(g + 1) * M], sep), f"group {g}"


@pytest.mark.parametrize("n,h,w,cin,cout", [(2, 64, 64, 320, 320), (2, 8, 8, 1280, 1280), (1, 16, 16, 640, 1280)])
def test_gemm_grouped_conv(L, n, h, w, cin, cout):
    dt = L.operand_dtype()
    G = 2
    x = rnd(G * n, h, w, cin, seed=1).to(dt)
    wp = [rnd(cout, 9 * cin, seed=10 + g, scale=(9 * cin) ** -0.5).to(dt) for g in range(G)]
    bs = [rnd(cout, seed=20 + g) for g in range(G)]
    rv = rnd(G * n, cout, seed=4)
    M = n * h * w
    out = torch.empty(G * M, cout, device="cuda")
    slots = L.gemm_gn_slots(h, w)
    part = torch.zeros(G * n * slots * cout * 2, device="cuda")
    L.gemm(x, torch.cat(wp, 0).contiguous(), out, M=G * M, N=cout, K=9 * cin, bias=torch.cat(bs, 0).contiguous(),
           rowvec=rv, conv=(G * n, h, w, cin, 3), groups=G, split_k=1, gn_partials=part)
    for g in range(G):
        sep = torch.empty(M, cout, device="cuda")
        psep = torch.zeros(n * slots * cout * 2, device="cuda")
        L.gemm(x[g * n:(g + 1) * n], wp[g], sep, M=M, N=cout, K=9 * cin, bias=bs[g], rowvec=rv[g * n:(g + 1) * n],
               conv=(n, h, w, cin, 3), split_k=1, gn_partials=psep)
        assert torch.equal(out[g * M:(g + 1) * M], sep), f"group {g}"
        assert torch.equal(part.view(G, -1)[g], psep), f"group {g} statistics"


def test_norm_kernels_grouped(L):
    """gn_apply / layernorm with stacked twin problems pick gamma / beta by image / row group."""
    dt = L.operand_dtype()
    n, h, w, c = 2, 16, 16, 320
    x = rnd(2 * n, h, w, c, seed=1)
    gam, bet = rnd(2 * c, seed=2), rnd(2 * c, seed=3)
    stats = torch.empty(2 * n * 64, device="cuda")
    wsp = torch.zeros(L.gn_workspace_floats(2 * n, h * w, c), device="cuda")
    L.gn_stats(x, None, c, 0, 2 * n, h * w, 1e-5, stats, wsp)
    out = torch.empty(2 * n * h * w, c, device="cuda", dtype=dt)
    L.gn_apply(x, None, c, 0, 2 * n, h, w, stats, gam, bet, out, norm=True, silu=True, imgs_per_group=n)
    for g in range(2):
        sep = torch.empty(n * h * w, c, device="cuda", dtype=dt)
        L.gn_apply(x[g * n:(g + 1) * n].contiguous(), None, c, 0, n, h, w, stats[g * n * 64:(g + 1) * n * 64].contiguous(),
                   gam[g * c:(g + 1) * c].contiguous(), bet[g * c:(g + 1) * c].contiguous(), sep, norm=True, silu=True)
        assert torch.equal(out[g * n * h * w:(g + 1) * n * h * w], sep)
    rows = 512
    t = rnd(2 * rows, c, seed=5)
    o = torch.empty(2 * rows, c, device="cuda", dtype=dt)
    L.layernorm(t, c, 2 * rows, c, gam, bet, o, c, rows_per_group=rows)
    for g in range(2):
        sep = torch.empty(rows, c, device="cuda", dtype=dt)
        L.layernorm(t[g * rows:(g + 1) * rows], c, rows, c, gam[g * c:(g + 1) * c].contiguous(),
                    bet[g * c:(g + 1) * c].contiguous(), sep, c)
        assert torch.equal(o[g * rows:(g + 1) * rows], sep)


@pytest.mark.parametrize("b,h,w", [(1, 512, 512), (2, 200, 333), (1, 40, 50), (1, 17, 1030)])
def test_wavelet_fix_fused_epilogue(L, b, h, w):
    """dbir_wavelet_fix vs the reference op sequence (utils/common.py:29-77 + pipeline.py:306-320) as
    torch ops on the same device: fp32 result to accumulation-order level, uint8 output equal except where
    fixed*255 sits within rounding of an integer (truncation flips by one there)."""
    from diffbir_b200.utils.common import wavelet_reconstruction
    pad_s = torch.empty(b, 3, h + 8, w + 24, device="cuda").uniform_(-1.2, 1.2, generator=g(1))
    pad_t = torch.empty(b, 3, h + 16, w + 8, device="cuda").uniform_(0, 1, generator=g(2))
    sample, style = pad_s[:, :, :h, :w], pad_t[:, :, :h, :w]           # strided views, like the pipeline's crops
    ref = wavelet_reconstruction((sample + 1) / 2, style)
    out32 = torch.empty(b, 3, h, w, device="cuda")
    L.wavelet_fix(sample, style, out_f32=out32)
    assert (out32 - ref).abs().max().item() < 2e-6
    ref8 = (ref * 255.0).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    out8 = torch.empty(b, h, w, 3, dtype=torch.uint8, device="cuda")
    L.wavelet_fix(sample, style, out_u8=out8)
    diff = (out8.int() - ref8.int()).abs()
    assert diff.max().item() <= 1 and (diff != 0).float().mean().item() < 1e-3
    assert out8.min().item() == 0 and out8.max().item() == 255        # the clamp is exercised
