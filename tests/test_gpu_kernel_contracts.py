"""-m gpu: element-by-element contracts of the C-ABI kernels the stage-1 cleaners (SwinIR, RRDBNet, SCUNet) and
the VAE glue run, at the shapes, strides and argument combinations the engines pass.

Every reference is plain float64 torch on the same 16-bit-rounded operands the kernel reads, and every check
is per element: |out - ref| <= rtol * |ref| + atol, never max|err| / max|ref|, which would hide an error in a
small-magnitude region. Tolerances are bounds on the kernel's own fp32 arithmetic plus one final rounding;
each constant is derived where it is defined. Input gaps the kernel must not read are poisoned with NaN and
output gaps it must not write are pre-filled with a sentinel and checked unchanged. Where a plausible kernel
bug is cheap to restate in the reference, the wrong reference is checked to lie more than 10x outside the
tolerance, so the test is known to see that bug."""
import pytest
import torch
import torch.nn.functional as F

from tests.gpu_util import no_tf32

pytestmark = pytest.mark.gpu

U = 2.0 ** -24            # fp32 unit roundoff (round to nearest)
# wgmma accumulates in fp32 but aligns addends by truncation, so its per-add error is one fp32 ulp (2^-23) rather
# than half of one
U_TC = 2.0 ** -23
# __expf(x) (ex2.approx of x*log2e): the CUDA programming guide bounds its error by 2 + floor(1.173|x|) ulp
EXPF_ULP = 2.0 ** -23


@pytest.fixture(scope="module")
def L():
    from diffbir_b200 import lib
    lib.load()
    no_tf32()
    return lib


def gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def rnd(*s, seed=0, scale=1.0):
    return torch.randn(*s, device="cuda", generator=gen(seed)) * scale


def r16(L):
    """One rounding to the 16-bit operand format: half an ulp relative, 2^-11 (fp16) / 2^-8 (bf16)."""
    return 2.0 ** -11 if L.operand_dtype() == torch.float16 else 2.0 ** -8


def a16(L):
    """Absolute rounding error below the format's normal range: half the smallest fp16 subnormal (2^-25);
    bf16 shares fp32's exponent range, where that error (2^-134) is negligible."""
    return 2.0 ** -25 if L.operand_dtype() == torch.float16 else 0.0


def excess(out, ref, rtol, atol):
    """Largest |out - ref| / (rtol |ref| + atol (1 + rtol)); > 1 fails. NaN anywhere counts as a failure.
    atol bounds the kernel's fp32 error before the final rounding, which scales that error by up to 1 + rtol."""
    out, ref = out.double(), ref.double()
    bound = rtol * ref.abs() + atol * (1 + rtol)
    ratio = (out - ref).abs() / bound
    ratio = torch.where(torch.isnan(ratio) | torch.isnan(out), torch.full_like(ratio, float("inf")), ratio)
    return ratio.max().item() if ratio.numel() else 0.0


def check(out, ref, rtol, atol, what=""):
    e = excess(out, ref, rtol, atol)
    assert e <= 1.0, f"{what}: an element is {e:.3g}x outside |out - ref| <= rtol |ref| + atol"


def sees(wrong, ref, rtol, atol, what):
    """The wrong reference must lie > 10x outside the tolerance somewhere: the check can see that bug."""
    e = excess(wrong, ref, rtol, atol)
    assert e > 10.0, f"discrimination '{what}': the wrong reference lies only {e:.3g}x outside the tolerance"


def same_bits(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    if a.element_size() == 2:
        return torch.equal(a.view(torch.int16), b.view(torch.int16))
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def sentinel(L):
    """A 16-bit / fp32 value no kernel result here takes by accident."""
    return -12345.0 if L.operand_dtype() == torch.float16 else -1.2345e30


# ============================================================================================ window attention
def _rel_index():
    cord = torch.tensor([[i, j] for i in range(8) for j in range(8)])
    return cord[:, None, :] - cord[None, :, :] + 7                               # [64, 64, 2]


def window_attention_ref(qkv16, b, h, w, heads, dh, shift, table, mask_value, *, mask=True, region_shift=0,
                         transpose_table=False):
    """WMSA.forward (scunet.py:54-91) / WindowAttention + SwinTransformerBlock roll (swinir.py:120-151, 255-276) in
    fp64 on the 16-bit qkv. The shift mask is built the generate_mask way (boolean slices, scunet.py:33-52).
    Returns (out [b*h*w, heads*dh], atol [b*h*w, heads*dh]).
    Wrong variants: mask=False drops the mask, region_shift moves the region boundary by that many tokens,
    transpose_table reads the [225, heads] table as [heads, 225]."""
    c = heads * dh
    hw_, ww_ = h // 8, w // 8
    y = qkv16[:, :3 * c].double().view(b, h, w, 3 * c)
    if shift:
        y = torch.roll(y, (-shift, -shift), (1, 2))
    win = y.view(b, hw_, 8, ww_, 8, 3 * c).permute(0, 1, 3, 2, 4, 5).reshape(b, hw_ * ww_, 64, 3, heads, dh)
    q, k, v = (win[:, :, :, i].permute(0, 1, 3, 2, 4) for i in range(3))         # [b, nw, heads, 64, dh]
    scale = dh ** -0.5
    dot_abs = (q.abs() @ k.abs().transpose(-1, -2)) * scale                     # sum_d |q_d k_d| / sqrt(dh)
    sim = (q @ k.transpose(-1, -2)) * scale
    tab = table.double()                                                        # [225, heads]
    if transpose_table:
        tab = tab.reshape(-1).view(heads, 225).t()
    rel = _rel_index().to(qkv16.device)
    rpp = tab.t().reshape(heads, 15, 15)
    bias = rpp[:, rel[:, :, 0], rel[:, :, 1]]                                   # [heads, 64, 64]
    sim = sim + bias[None, None]
    if shift and mask:
        m = torch.zeros(hw_, ww_, 8, 8, 8, 8, dtype=torch.bool, device=qkv16.device)
        s = 8 - shift + region_shift
        m[-1, :, :s, :, s:, :] = True
        m[-1, :, s:, :, :s, :] = True
        m[:, -1, :, :s, :, s:] = True
        m[:, -1, :, s:, :, :s] = True
        m = m.reshape(1, hw_ * ww_, 1, 64, 64)
        if mask_value == float("-inf"):
            sim = sim.masked_fill(m, float("-inf"))
        else:
            sim = sim + m.double() * mask_value
    p = torch.softmax(sim, dim=-1)
    o = p @ v
    # Kernel error bound. Logit s_j: q pre-scaled by rsqrtf (2 ulp, 2^-22) and rounded (2^-24), a 32-term dot
    # product in four fma chains (<= 32 u), the bias add and a finite mask add (one rounding each on |s|):
    #   e_j <= (2^-22 + 33 u) * sum|q k| / sqrt(dh) + 2 u |s_j|.
    # exp(s_j - m): the subtraction rounds (u |x_j|), __expf adds (2 + 1.173 |x_j|) ulp, so the relative error of
    # p_j is d_j <= e_j + e_m + u |x_j| + (2 + 1.173 |x_j|) 2^-23 (e_m <= max_j e_j). The row sum l adds 64 u,
    # the 64 fma of P V 64 u of sum p|v|, the final scale one u: |o - ref| <= sum_j p_j |v_j| d_j
    # + (sum_j p_j d_j + 130 u) sum_j p_j |v_j|.
    fin = torch.isfinite(sim)
    simf = torch.where(fin, sim, torch.zeros_like(sim))
    e = (2.0 ** -22 + 33 * U) * dot_abs + 2 * U * simf.abs()
    e = torch.where(fin, e, torch.zeros_like(e))
    e_m = e.amax(-1, keepdim=True)
    x = (simf - sim.amax(-1, keepdim=True)).abs()
    d = e + e_m + U * x + (2 + 1.173 * x) * EXPF_ULP
    d = torch.where(fin, d, torch.zeros_like(d))
    pd = p * d
    pv = p @ v.abs()
    atol = pd @ v.abs() + (pd.sum(-1, keepdim=True) + 130 * U) * pv

    def back(t):
        t = t.permute(0, 1, 3, 2, 4).reshape(b, hw_, ww_, 8, 8, c).permute(0, 1, 3, 2, 4, 5).reshape(b, h, w, c)
        if shift:
            t = torch.roll(t, (shift, shift), (1, 2))
        return t.reshape(b * h * w, c)
    return back(o), back(atol)


WA_SCUNET = [(hd, s, geo) for hd in (1, 2, 4, 8) for s in (0, 4) for geo in ((1, 8, 8), (2, 16, 40), (1, 32, 24))]


def _run_window_attention(L, b, h, w, heads, dh, shift, mask_value, table_scale=0.5, q_scale=1.0, seed=0):
    dt = L.operand_dtype()
    c = heads * dh
    ldq = 3 * c
    ldo = max(c, 64)
    g = torch.Generator(device="cuda").manual_seed(100 + seed)
    qkv = (torch.randn(b * h * w, ldq, device="cuda", generator=g) * 1.5)
    qkv[:, :c] *= q_scale
    qkv = qkv.to(dt)
    table = torch.randn(225, heads, device="cuda", generator=g) * table_scale
    out = torch.full((b * h * w, ldo), sentinel(L), device="cuda", dtype=dt)
    L.window_attention(qkv, ldq, b, h, w, heads, dh, shift, table, mask_value, out, ldo)
    torch.cuda.synchronize()
    ref, atol = window_attention_ref(qkv, b, h, w, heads, dh, shift, table, mask_value)
    rtol, at = r16(L), atol + a16(L)
    check(out[:, :c], ref, rtol, at, f"window attention {heads}x{dh} shift {shift} {(b, h, w)}")
    assert (out[:, c:] == sentinel(L)).all(), "pad columns [heads*dim, ldo) were written"
    return qkv, table, ref, rtol, at


@pytest.mark.parametrize("heads,shift,geo", WA_SCUNET)
def test_window_attention_scunet(L, heads, shift, geo):
    """SCUNet's WMSA: (heads, 32) for trans_dim 32..256, mask -inf (engine/scunet.py:111, csrc/swin.cu:142-146),
    qkv ldq = 3 heads 32, output ldo = max(heads 32, 64) with the pad columns untouched. (1, 8, 8) is the
    single-window image SCUNet's deepest level sees for a 64x64 input."""
    b, h, w = geo
    qkv, table, ref, rtol, at = _run_window_attention(L, b, h, w, heads, 32, shift, float("-inf"), seed=heads)
    if shift:
        wrong, _ = window_attention_ref(qkv, b, h, w, heads, 32, shift, table, float("-inf"), mask=False)
        sees(wrong, ref, rtol, at, "mask off")
        wrong, _ = window_attention_ref(qkv, b, h, w, heads, 32, shift, table, float("-inf"), region_shift=1)
        sees(wrong, ref, rtol, at, "region boundary one token late")
        wrong, _ = window_attention_ref(qkv, b, h, w, heads, 32, shift, table, float("-inf"), region_shift=-1)
        sees(wrong, ref, rtol, at, "region boundary one token early")
    if heads > 1:      # with one head [heads, 225] and [225, heads] are the same array
        wrong, _ = window_attention_ref(qkv, b, h, w, heads, 32, shift, table, float("-inf"), transpose_table=True)
        sees(wrong, ref, rtol, at, "relative-position table transposed")


def test_window_attention_swinir_single_window(L):
    """SwinIR's 6 heads x 30 with mask -100 (engine/swinir.py:133) on a one-window image with shift 4: every
    token lies in the last window row and column."""
    qkv, table, ref, rtol, at = _run_window_attention(L, 2, 8, 8, 6, 30, 4, -100.0, seed=7)
    wrong, _ = window_attention_ref(qkv, 2, 8, 8, 6, 30, 4, table, -100.0, mask=False)
    sees(wrong, ref, rtol, at, "mask off")
    wrong, _ = window_attention_ref(qkv, 2, 8, 8, 6, 30, 4, table, -100.0, transpose_table=True)
    sees(wrong, ref, rtol, at, "relative-position table transposed")


@pytest.mark.parametrize("heads,dh,mask_value", [(4, 32, float("-inf")), (6, 30, -100.0)])
def test_window_attention_peaked(L, heads, dh, mask_value):
    """Peaked logits (standard deviation about 20: q and k have standard deviation 1.5, q is scaled by 9) where
    the softmax is nearly one-hot and the exp / max-shift arithmetic carries the result."""
    qkv, *_ = _run_window_attention(L, 1, 16, 24, heads, dh, 4, mask_value, q_scale=9.0, seed=11)
    c = heads * dh
    q, k = qkv[:, :c].double(), qkv[:, c:2 * c].double()
    s = (q[:, :dh] * k[:, :dh]).sum(-1) * dh ** -0.5        # same-token logits of head 0: their spread
    assert 10 < s.std().item() < 40


# ============================================================================================ flash attention
def flash_ref(q, k, v, *, lazy_block=None):
    """softmax(q k^T / 8) v per head in fp64 on the 16-bit operands ([sq, 64] x [skv, 64]) and the kernel's error
    bound. lazy_block=64 restates a kernel that forgets to rescale its running output when the row maximum
    moves between 64-key blocks (l is kept right)."""
    qd, kd, vd = q.double(), k.double(), v.double()
    s = qd @ kd.t()
    if lazy_block is None:
        p = torch.softmax(s / 8, -1)
        o = p @ vd
    else:
        m = torch.full((s.shape[0], 1), float("-inf"), dtype=s.dtype, device=s.device)
        l = torch.zeros_like(m)
        o = torch.zeros(s.shape[0], 64, dtype=s.dtype, device=s.device)
        for j0 in range(0, s.shape[1], lazy_block):
            sb = s[:, j0:j0 + lazy_block] / 8
            mn = torch.maximum(m, sb.amax(-1, keepdim=True))
            pb = torch.exp(sb - mn)
            l = l * torch.exp(m - mn) + pb.sum(-1, keepdim=True)
            o = o + pb @ vd[j0:j0 + lazy_block]                    # missing: o * exp(m - mn)
            m = mn
        return o / l, None
    # Bound. S = Q K^T on wgmma: 64-term fp32 accumulation, e_s <= 64 U_TC sum|q k|. exp2(fma(s, log2e/8,
    # -m log2e/8)): the fma and the rounded scale cost 2 u of the argument, ex2.approx 2^-22 relative, so
    # p_j carries d_j <= (e_s_j + e_s_max) / 8 + 2 u (|s_j| + |s_max|) / 8 + 2^-22. P is then rounded to 16 bit
    # for the P V product (r16 relative, plus the subnormal floor of fp16 on weights <= 1 after division by
    # l >= 1); l sums the unrounded p (skv u), O accumulates on wgmma (skv U_TC), 1/l and the scale 2 u:
    # |o - ref| <= sum_j p_j |v_j| (d_j + r16) + (sum_j p_j d_j + skv (u + U_TC) + 2^-21) sum_j p_j |v_j|
    # + a16 sum_j |v_j|. The lazy rescale (alpha on both O and l) cancels exactly.
    es = 64 * U_TC * (qd.abs() @ kd.abs().t())
    imax = s.argmax(-1, keepdim=True)
    d = (es + es.gather(-1, imax)) / 8 + 2 * U * (s.abs() + s.gather(-1, imax).abs()) / 8 + 2.0 ** -22
    return o, (p, d, vd.abs())


def flash_atol(parts, rp, ap):
    p, d, va = parts
    skv = p.shape[1]
    pv = p @ va
    return (p * (d + rp)) @ va + ((p * d).sum(-1, keepdim=True) + skv * (U + U_TC) + 2.0 ** -21) * pv + \
        ap * va.sum(0, keepdim=True)


def _peaked_qkv(L, b, heads, sq, skv, seed):
    """q, k, v [b*s, heads*64] where every query's dominant key is the LAST key (in the last, partial key block
    when skv % 64 != 0): q = z + 12 u, k_last = z' + 12 u for a shared unit vector u per head, so the planted
    logit / 8 is ~18 against a row of standard deviation ~1.8 and the row maximum moves late by > 5.5 (the
    kernel's lazy-rescale threshold of 2^8 in exp2 units)."""
    dt = L.operand_dtype()
    g = torch.Generator(device="cuda").manual_seed(seed)
    u = torch.randn(heads, 64, device="cuda", generator=g)
    u = u / u.norm(dim=-1, keepdim=True)
    q = torch.randn(b, sq, heads, 64, device="cuda", generator=g) + 12 * u
    k = torch.randn(b, skv, heads, 64, device="cuda", generator=g)
    k[:, -1] += 12 * u
    v = torch.randn(b, skv, heads, 64, device="cuda", generator=g)
    return [t.reshape(b * t.shape[1], heads * 64).to(dt) for t in (q, k, v)]


def _check_flash(L, q, k, v, out, b, heads, sq, skv, discriminate):
    rp, ap = r16(L), a16(L)
    seen = 0.0
    for bi in range(b):
        for hi in range(heads):
            qs = q[bi * sq:(bi + 1) * sq, hi * 64:(hi + 1) * 64]
            ks = k[bi * skv:(bi + 1) * skv, hi * 64:(hi + 1) * 64]
            vs = v[bi * skv:(bi + 1) * skv, hi * 64:(hi + 1) * 64]
            ref, parts = flash_ref(qs, ks, vs)
            atol = flash_atol(parts, rp, ap)
            check(out[bi * sq:(bi + 1) * sq, hi * 64:(hi + 1) * 64], ref, rp, atol,
                  f"attention b{bi} h{hi} sq {sq} skv {skv}")
            if discriminate:
                wrong, _ = flash_ref(qs, ks, vs, lazy_block=64)
                seen = max(seen, excess(wrong, ref, rp, atol))
    if discriminate:
        assert seen > 10.0, f"discrimination 'missing rescale': the wrong reference is only {seen:.3g}x outside"


@pytest.mark.parametrize("sq", [1, 127, 129])
@pytest.mark.parametrize("skv", [1, 63, 64, 65, 77, 129])
def test_attention_peaked_late_max(L, sq, skv):
    """Flash attention with the row maximum planted in the last key (the last, partial 64-key block): the
    online softmax must rescale the running output when the maximum moves. q / k / v are column slices of
    wider buffers (ld = 3 c) like the fused QKV projection (engine/cldm.py self-attention)."""
    b, heads = 2, 2
    c = heads * 64
    q0, k0, v0 = _peaked_qkv(L, b, heads, sq, skv, seed=sq * 1000 + skv)
    dt = L.operand_dtype()
    qb = torch.full((b * sq, 3 * c), float("nan"), device="cuda", dtype=dt)
    kvb = torch.full((b * skv, 3 * c), float("nan"), device="cuda", dtype=dt)
    qb[:, c:2 * c] = q0
    kvb[:, :c], kvb[:, 2 * c:] = k0, v0
    q, k, v = qb[:, c:2 * c], kvb[:, :c], kvb[:, 2 * c:]
    out_b = torch.full((b * sq, c + 64), sentinel(L), device="cuda", dtype=dt)
    L.attention(q, k, v, out_b[:, 64:], batch=b, heads=heads, sq=sq, skv=skv, ldq=3 * c, ldk=3 * c, ldv=3 * c,
                ldo=c + 64)
    torch.cuda.synchronize()
    _check_flash(L, q0, k0, v0, out_b[:, 64:], b, heads, sq, skv, discriminate=skv > 64)
    assert (out_b[:, :64] == sentinel(L)).all(), "columns before the output slice were written"


def test_attention_peaked_stream_k(L):
    """The one shape that takes the stream-K workspace path (2, 5, 4096, 4096; see test_gpu_kernels.py) with
    peaked logits: tiles cut by CTA boundaries are combined through the workspace with their own maxima."""
    b, heads, s = 2, 5, 4096
    c = heads * 64
    q, k, v = _peaked_qkv(L, b, heads, s, s, seed=5)
    nws = L.attention_ws_bytes(b, heads, s, s)
    assert nws > 0
    ws = torch.zeros(nws // 4, device="cuda")
    out = torch.empty(b * s, c, device="cuda", dtype=L.operand_dtype())
    L.attention(q, k, v, out, batch=b, heads=heads, sq=s, skv=s, ldq=c, ldk=c, ldv=c, ldo=c, ws=ws)
    torch.cuda.synchronize()
    _check_flash(L, q, k, v, out, b, heads, s, s, discriminate=True)
    assert (ws[:16384] == 0).all()


# ============================================================================================ GEMM epilogues
EPILOGUE_ACTS = (("none", 0.0), ("gelu", 0.0), ("lrelu", 0.2), ("lrelu", 0.01), ("lrelu", 0.0), ("silu", 0.0))
FORCE_BN = (32, 64, 128, 160, 256)          # every tile width dbir_gemm accepts (any N when forced)


def act_ref(z, act, slope):
    if act == "gelu":
        return F.gelu(z)
    if act == "lrelu":
        return F.leaky_relu(z, slope)
    if act == "silu":
        return F.silu(z)
    return z


def act_err(z, act):
    """(Lipschitz constant, evaluation error) of the kernel's fp32 activation at z.
    GELU: Abramowitz-Stegun 7.1.26 erf, |abs error| <= 1.5e-7 (csrc/common.cuh:347-352), so Phi is off by
    0.75e-7; rcp.approx / ex2.approx / 8 roundings add < 2^-20 of Phi <= 1; max GELU' = 1.129.
    SiLU: x / (1 + __expf(-x)): (2 + 1.173|x|) ulp of the exp, the add and the division: max SiLU' = 1.0998.
    LeakyReLU: one product rounding."""
    if act == "gelu":
        return 1.13, z.abs() * (0.75e-7 + 2.0 ** -20)
    if act == "silu":
        return 1.1, F.silu(z).abs() * ((2 + 1.173 * z.abs()) * EXPF_ULP + 2 * U)
    if act == "lrelu":
        return 1.0, U * z.abs()
    return 1.0, torch.zeros_like(z)


def gemm_ref(A, B, *, bias=None, rowvec_rows=None, act="none", slope=0.0, alpha=1.0, residual=None, k_terms=None,
             out16=False, L=None, bias_per_row=False):
    """fp64 out = residual + alpha act(A B^T + bias + rowvec) and its bound (rtol, atol).
    Pre-activation z: k fp32 adds on wgmma (k U_TC of sum |a b|), bias and row-vector adds (2 u of their
    magnitudes and of |z|). The activation passes that on with its Lipschitz constant and adds its own
    evaluation error; alpha and the residual add one rounding each of |alpha act| and |out|. A 16-bit output
    adds one final rounding (rtol r16, plus the fp16 subnormal floor)."""
    Ad, Bd = A.double(), B.double()
    z = Ad @ Bd.t()
    mag = Ad.abs() @ Bd.abs().t()
    add = torch.zeros_like(z)
    if bias is not None:
        add = add + (bias.double()[:, None] if bias_per_row else bias.double()[None, :])
    if rowvec_rows is not None:
        add = add + rowvec_rows.double()
    z = z + add
    k = A.shape[1] if k_terms is None else k_terms
    ez = k * U_TC * mag + 2 * U * (add.abs() + z.abs())
    lip, eact = act_err(z, act)
    y = alpha * act_ref(z, act, slope)
    out = y if residual is None else y + residual.double()
    atol = abs(alpha) * (lip * ez + eact) + U * (y.abs() + out.abs())
    rtol = 0.0
    if out16:
        rtol, atol = r16(L), atol + a16(L)
    return out, rtol, atol


def im2col3(x):
    """NHWC [n, h, w, C] -> [n*h*w, 9*C] with k = tap*C + c (the packed weights' order), zero padding 1."""
    n, h, w, C = x.shape
    xp = F.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1))
    cols = torch.stack([xp[:, :, ky:ky + h, kx:kx + w] for ky in range(3) for kx in range(3)], 1)   # [n, 9, C, h, w]
    return cols.permute(0, 3, 4, 1, 2).reshape(n * h * w, 9 * C)


@pytest.mark.parametrize("force_bn", FORCE_BN)
@pytest.mark.parametrize("mode", ["matrix", "conv"])
def test_gemm_epilogue_matrix(L, mode, force_bn):
    """Every epilogue combination, act in {none, gelu, lrelu 0.2 / 0.01 / 0.0, silu} x {fp32, 16-bit output} x
    alpha in {1, 0.2} x {no residual, residual through ldr > N at an offset pointer}, at one forced tile width.
    The output is a column slice (offset pointer, ldo > N) of a sentinel-filled buffer; the operand's row /
    pixel stride (lda) carries a NaN gap the kernel must not read; the residual's neighbouring columns are NaN.
    matrix: M = 300, K = 200 (partial M tile, partial last k-block); conv: 2 x 10 x 12 pixels, C = 64, K = 576."""
    dt = L.operand_dtype()
    N = 200
    if mode == "matrix":
        M, K = 300, 200
        lda = K + 16
        a_buf = torch.full((M, lda), float("nan"), device="cuda", dtype=dt)
        a_buf[:, :K] = rnd(M, K, seed=1).to(dt)
        A = a_buf[:, :K]
        conv = None
    else:
        n, h, w, C = 2, 10, 12, 64
        M, K = n * h * w, 9 * C
        lda = C + 64
        a_buf = torch.full((n, h, w, lda), float("nan"), device="cuda", dtype=dt)
        a_buf[..., :C] = rnd(n, h, w, C, seed=1).to(dt)
        A = im2col3(a_buf[..., :C].double())
        conv = (n, h, w, C, 3)
    B = rnd(N, K, seed=2, scale=K ** -0.5).to(dt)
    bias = rnd(N, seed=3)
    ldr, roff = N + 24, 8
    r_buf = torch.full((M, ldr), float("nan"), device="cuda")
    r_buf[:, roff:roff + N] = rnd(M, N, seed=4)
    res = r_buf[:, roff:]
    ooff = 8
    failures = []
    for act, slope in EPILOGUE_ACTS:
        for out_dt in (torch.float32, dt):
            for alpha in (1.0, 0.2):
                for with_res in (False, True):
                    ldo = N + 16
                    o_buf = torch.full((M, ldo), sentinel(L), device="cuda", dtype=out_dt)
                    L.gemm(a_buf, B, o_buf[:, ooff:], M=M, N=N, K=K, bias=bias, act=act, act_param=slope, alpha=alpha,
                           residual=res if with_res else None, ldr=ldr, lda=lda, ldo=ldo, conv=conv,
                           force_bn=force_bn, split_k=1)
                    ref, rtol, atol = gemm_ref(A, B, bias=bias, act=act, slope=slope, alpha=alpha,
                                               residual=res[:, :N] if with_res else None,
                                               out16=out_dt != torch.float32, L=L)
                    tag = f"{act}({slope}) {out_dt} alpha {alpha} residual {with_res}"
                    e = excess(o_buf[:, ooff:ooff + N], ref, rtol, atol)
                    if e > 1.0:
                        failures.append(f"{tag}: {e:.3g}x")
                    gap_ok = (o_buf[:, :ooff] == sentinel(L)).all() and (o_buf[:, ooff + N:] == sentinel(L)).all()
                    if not gap_ok:
                        failures.append(f"{tag}: wrote outside its column slice")
                    if with_res and act == "none" and alpha == 1.0 and out_dt == torch.float32:
                        # residual read with stride N from the residual pointer instead of ldr
                        flat = torch.nan_to_num(r_buf, nan=0.0).reshape(-1)[roff:roff + M * N].view(M, N)
                        wrong, _, _ = gemm_ref(A, B, bias=bias, residual=flat)
                        sees(wrong, ref, rtol, atol, "residual read with stride N")
    assert not failures, "; ".join(failures)


def test_gemm_rrdb_dense_block(L):
    """RRDBNet's dense block exactly as engine/bsrnet.py:84-88 calls it: one 16-bit [pixels, 192] concat buffer;
    conv k (k = 1..4) reads the first C = roundup64(64 + 32 (k-1)) channels through the pixel stride lda = 192
    and writes its 32 LeakyReLU(0.2) channels into cat[:, 64 + 32 (k-1):] with ldo = 192. Channels >= C are
    NaN; channels [cin, C) (convs 2 and 4: the zero-weight excess, which is also the slot being written) are
    finite, and refilling them with +-6e4 must give the same bits. The other slots must be unchanged."""
    from diffbir_b200.engine.common import pack_conv3x3
    dt = L.operand_dtype()
    n, h, w, nf, gc = 2, 12, 20, 64, 32
    Ctot = nf + 4 * gc
    M = n * h * w
    base = rnd(n, h, w, Ctot, seed=1).to(dt)
    for k in range(1, 5):
        cin = nf + (k - 1) * gc
        C = (cin + 63) // 64 * 64
        wt = rnd(gc, cin, 3, 3, seed=10 + k, scale=(9 * cin) ** -0.5)
        wp = pack_conv3x3(wt, "cuda", cin_pad=C)
        bias = rnd(gc, seed=20 + k)
        results = []
        for fill in ("finite", "large"):
            cat = base.clone()
            cat[..., C:] = float("nan")
            if C > cin:
                cat[..., cin:C] = base[..., cin:C] if fill == "finite" else \
                    (torch.sign(rnd(n, h, w, C - cin, seed=30)) * 6e4).to(dt)
            before = cat.clone()
            out = cat.view(M, Ctot)[:, cin:]
            L.gemm(cat, wp, out, M=M, N=gc, K=9 * C, bias=bias, act="lrelu", act_param=0.2, conv=(n, h, w, C, 3),
                   lda=Ctot, ldo=Ctot)
            torch.cuda.synchronize()
            got = cat.view(M, Ctot)
            A = im2col3(before[..., :cin].double())
            ref, rtol, atol = gemm_ref(A, wt.to(dt).permute(0, 2, 3, 1).reshape(gc, -1), bias=bias, act="lrelu",
                                       slope=0.2, out16=True, L=L, k_terms=9 * C)
            check(got[:, cin:cin + gc], ref, rtol, atol, f"dense conv {k} ({fill} excess)")
            keep = torch.ones(Ctot, dtype=torch.bool, device="cuda")
            keep[cin:cin + gc] = False
            assert same_bits(got[:, keep], before.view(M, Ctot)[:, keep]), f"conv {k} wrote outside its slot"
            results.append(got[:, cin:cin + gc].clone())
        assert same_bits(results[0], results[1]), f"conv {k}: the zero-weight excess channels changed the result"


def test_gemm_scunet_cb2_residual_stride(L):
    """SCUNet conv_block tail (engine/scunet.py:102): 3x3 conv of the [M, tp] operand into the first t columns of
    the 16-bit cat [M, c] (ldo = c) with the fp32 residual y [M, c] read through ldr = c (first t columns). The
    Swin half y[:, t:] is NaN (must not be read) and cat[:, t:] keeps its sentinel."""
    dt = L.operand_dtype()
    n, h, w, c = 2, 16, 24, 64
    t, tp = c // 2, 64
    M = n * h * w
    h16 = torch.zeros(n, h, w, tp, device="cuda", dtype=dt)
    h16[..., :t] = rnd(n, h, w, t, seed=1).to(dt)
    wt = rnd(t, t, 3, 3, seed=2, scale=(9 * t) ** -0.5)
    from diffbir_b200.engine.common import pack_conv3x3
    wp = pack_conv3x3(wt, "cuda", cin_pad=tp)
    y = torch.full((M, c), float("nan"), device="cuda")
    y[:, :t] = rnd(M, t, seed=3)
    cat = torch.full((M, c), sentinel(L), device="cuda", dtype=dt)
    L.gemm(h16, wp, cat, M=M, N=t, K=9 * tp, residual=y, ldr=c, conv=(n, h, w, tp, 3), ldo=c)
    torch.cuda.synchronize()
    A = im2col3(h16[..., :t].double())
    ref, rtol, atol = gemm_ref(A, wt.to(dt).permute(0, 2, 3, 1).reshape(t, -1), residual=y[:, :t], out16=True, L=L,
                               k_terms=9 * tp)
    check(cat[:, :t], ref, rtol, atol, "cb2")
    assert (cat[:, t:] == sentinel(L)).all()
    flat = torch.nan_to_num(y, nan=0.0).reshape(-1)[:M * t].view(M, t)
    wrong, _, _ = gemm_ref(A, wt.to(dt).permute(0, 2, 3, 1).reshape(t, -1), residual=flat)
    sees(wrong, ref, rtol, atol, "residual read with stride N")


@pytest.mark.parametrize("rows_per_vec", [50, 96, 200])
def test_gemm_rowvec_rows_per_vec(L, rows_per_vec):
    """Matrix-mode row vectors (time embedding per image) with rows_per_vec that does not divide the 128-row tile
    or the 32-row warp: a warp's rows take two different vectors."""
    dt = L.operand_dtype()
    M, N, K = 600, 96, 128
    A = rnd(M, K, seed=1).to(dt)
    B = rnd(N, K, seed=2, scale=K ** -0.5).to(dt)
    bias = rnd(N, seed=3)
    nvec = (M + rows_per_vec - 1) // rows_per_vec
    rv = rnd(nvec, N, seed=4)
    out = torch.empty(M, N, device="cuda")
    L.gemm(A, B, out, M=M, N=N, K=K, bias=bias, rowvec=rv, rows_per_vec=rows_per_vec, act="silu")
    rows = rv[torch.arange(M, device="cuda") // rows_per_vec]
    ref, rtol, atol = gemm_ref(A, B, bias=bias, rowvec_rows=rows, act="silu")
    check(out, ref, rtol, atol, f"rows_per_vec {rows_per_vec}")
    wrong, _, _ = gemm_ref(A, B, bias=bias, rowvec_rows=rv[torch.arange(M, device="cuda") // 128 % nvec], act="silu")
    sees(wrong, ref, rtol, atol, "row vector per 128-row tile")


def test_gemm_bias_per_row_fp32(L):
    """bias_per_row (transposed products: bias indexed by output row) with an fp32 output and a partial M tile."""
    dt = L.operand_dtype()
    M, N, K = 333, 256, 192
    A = rnd(M, K, seed=1).to(dt)
    B = rnd(N, K, seed=2, scale=K ** -0.5).to(dt)
    bias = rnd(M, seed=3)
    out = torch.empty(M, N, device="cuda")
    L.gemm(A, B, out, M=M, N=N, K=K, bias=bias, bias_per_row=True, alpha=0.2, act="gelu")
    ref, rtol, atol = gemm_ref(A, B, bias=bias, bias_per_row=True, alpha=0.2, act="gelu")
    check(out, ref, rtol, atol, "bias_per_row")


# ============================================================================================ elementwise / layout
@pytest.mark.parametrize("with_y,with_z", [(False, False), (False, True), (True, False), (True, True)])
def test_axpby_cast_bit_exact(L, with_y, with_z):
    """y = alpha x + z (engine/bsrnet.py:79-99, scunet.py:121-176): bit-identical to the unfused torch ops, the
    16-bit copy written with row stride ld16 > c and its gap left alone."""
    dt = L.operand_dtype()
    rows, c, ld16 = 1000, 64, 192
    x, z = rnd(rows, c, seed=1), rnd(rows, c, seed=2)
    y = torch.full((rows, c), 7.0, device="cuda") if with_y else None
    y16 = torch.full((rows, ld16), sentinel(L), device="cuda", dtype=dt)
    L.axpby_cast(x, 0.2, z if with_z else None, rows, c, y=y, y16=y16, ld16=ld16)
    ref = x * 0.2 + z if with_z else x * 0.2
    if with_y:
        assert same_bits(y, ref)
    assert same_bits(y16[:, :c], ref.to(dt))
    assert (y16[:, c:] == sentinel(L)).all()


def test_upsample2x_op16_bit_exact(L):
    """Nearest 2x upsample of a 16-bit NHWC tensor (engine/bsrnet.py:106, swinir.py:157)."""
    dt = L.operand_dtype()
    n, h, w, c = 2, 7, 13, 64
    x = rnd(n, h, w, c, seed=1).to(dt)
    out = torch.empty(n, 2 * h, 2 * w, c, device="cuda", dtype=dt)
    L.upsample2x_op16(x, n, h, w, c, out)
    assert same_bits(out, x.repeat_interleave(2, 1).repeat_interleave(2, 2))


@pytest.mark.parametrize("r,cpad", [(1, 8), (2, 16), (8, 200)])
def test_swin_stem_bit_exact(L, r, cpad):
    """(x - mean) * range, PixelUnshuffle(r), NCHW -> NHWC, channels [3 r^2, cpad) zero (engine/swinir.py:112)."""
    dt = L.operand_dtype()
    n, h, w = 2, 8 * 5, 8 * 3
    x = torch.rand(n, 3, h, w, device="cuda", generator=gen(1))
    mean = (0.4488, 0.4371, 0.4040)
    out = torch.full((n, h // r, w // r, cpad), sentinel(L), device="cuda", dtype=dt)
    L.swin_stem(x, n, h, w, r, mean, 255.0, cpad, out)
    t = (x - torch.tensor(mean, device="cuda").view(1, 3, 1, 1)) * 255.0
    ref = F.pixel_unshuffle(t, r).permute(0, 2, 3, 1)
    ref = F.pad(ref, (0, cpad - 3 * r * r)).to(dt)
    assert same_bits(out, ref)


@pytest.mark.parametrize("c", [3, 4, 8])
def test_layout_transposes_bit_exact(L, c):
    """NCHW <-> NHWC fp32 (latents and images, engine/vae.py:157-161) with hw not a multiple of 256."""
    n, hw = 2, 37 * 23
    x = rnd(n, c, hw, seed=c)
    nhwc = torch.empty(n, hw, c, device="cuda")
    L.nchw_to_nhwc(x, n, c, hw, nhwc)
    assert same_bits(nhwc, x.permute(0, 2, 1).contiguous())
    back = torch.empty(n, c, hw, device="cuda")
    L.nhwc_to_nchw(nhwc, n, c, hw, back)
    assert same_bits(back, x)


def silu_bound(x):
    """|silu_f(x) - silu(x)| for the fp32 input x: (2 + 1.173|x|) ulp of __expf, the add and the division."""
    return F.silu(x).abs() * ((2 + 1.173 * x.abs()) * EXPF_ULP + 2 * U)


@pytest.mark.parametrize("m,k,n", [(1001, 4, 4), (300, 8, 16), (13, 320, 1280), (5, 1280, 1280)])
def test_linear_f32(L, m, k, n):
    """y = silu(silu(x) W^T + b) in fp32: the row kernel (m >= 256, k, n <= 16: VAE quant convs,
    engine/vae.py:159,233) and the warp-per-feature kernel (time embedding, engine/cldm.py:229-239), with
    ldx > k (NaN gap), m not a multiple of 8 and ldy > n (sentinel gap)."""
    ldx, ldy = k + 4, n + 4
    xb = torch.full((m, ldx), float("nan"), device="cuda")
    xb[:, :k] = rnd(m, k, seed=1) * 3
    wt, b = rnd(n, k, seed=2, scale=k ** -0.5), rnd(n, seed=3)
    for silu in (False, True):
        y = torch.full((m, ldy), -7.0, device="cuda")
        L.linear_f32(xb, ldx, m, k, wt, b, n, y, ldy, silu_in=silu, silu_out=silu)
        x = xb[:, :k].double()
        xin = F.silu(x) if silu else x
        z = xin @ wt.double().t() + b.double()
        # k + 1 fp32 adds on sum |x w| + |b|, plus the input SiLU's error times |w|; the output SiLU passes that
        # on with slope <= 1.1 and adds its own
        ez = (k + 1) * U * (xin.abs() @ wt.double().abs().t() + b.double().abs())
        if silu:
            ez = ez + silu_bound(x) @ wt.double().abs().t()
            ref, atol = F.silu(z), 1.1 * ez + silu_bound(z)
        else:
            ref, atol = z, ez
        check(y[:, :n], ref, 0.0, atol, f"linear_f32 silu {silu}")
        assert (y[:, n:] == -7.0).all()


@pytest.mark.parametrize("c1,c2", [(3, 0), (4, 4), (12, 4)])
@pytest.mark.parametrize("cout", [64, 128, 320])
@pytest.mark.parametrize("w", [1, 31, 33, 72])
def test_conv3x3_small_cin(L, c1, c2, cout, w):
    """Stem conv of <= 16 input channels: RGB (c = 3, engine/bsrnet.py:75), latent + hint (4 + 4,
    engine/cldm.py:401) and 12 + 4, with in_scale / in_shift applied before the zero padding, on one-row
    images whose width leaves a partial 32-pixel strip."""
    n, h = 2, 1
    cin = c1 + c2
    x1, x2 = rnd(n, c1, h, w, seed=1), (rnd(n, c2, h, w, seed=2) if c2 else None)
    wt = rnd(cout, cin, 3, 3, seed=3, scale=(9 * cin) ** -0.5)
    bias = rnd(cout, seed=4)
    out = torch.full((n * h * w + 1, cout), -7.0, device="cuda")
    L.conv3x3_small_cin(x1, x2, c1, c2, n, h, w, wt.permute(2, 3, 1, 0).reshape(-1, cout).contiguous(), bias, cout,
                        out, in_scale=2.0, in_shift=-1.0)
    xin = torch.cat([x1, x2], 1) if c2 else x1
    A = im2col3((xin.double() * 2.0 - 1.0).permute(0, 2, 3, 1))
    Bm = wt.double().permute(0, 2, 3, 1).reshape(cout, -1)
    ref = A @ Bm.t() + bias.double()
    mag = A.abs() @ Bm.abs().t() + bias.double().abs()
    # 9 cin + 1 fp32 fma / adds on sum |x w| + |b|, and the (contracted) scale-shift rounds each input once
    check(out[:-1], ref, 0.0, (9 * cin + 2) * U * mag, f"small_cin {c1}+{c2} -> {cout}, w {w}")
    assert (out[-1] == -7.0).all(), "wrote past the last pixel"


@pytest.mark.parametrize("cout", [3, 4, 8])
def test_conv3x3_small_cout_nhwc(L, cout):
    """Head conv into NHWC fp32 without post_shift (the VAE encoder's conv_out before quant_conv,
    engine/vae.py:230) on a width that leaves a partial 4-pixel group."""
    dt = L.operand_dtype()
    n, h, w, cin = 2, 5, 11, 64
    x = rnd(n, h, w, cin, seed=1).to(dt)
    wt = rnd(cout, cin, 3, 3, seed=2, scale=(9 * cin) ** -0.5)
    bias = rnd(cout, seed=3)
    out = torch.full((n * h * w + 1, cout), -7.0, device="cuda")
    L.conv3x3_small_cout(x, n, h, w, cin, wt.permute(0, 2, 3, 1).reshape(cout, -1).contiguous(), bias, cout, out,
                         nchw=False, post_scale=0.5)
    A = im2col3(x.double())
    Bm = wt.double().permute(0, 2, 3, 1).reshape(cout, -1)
    ref = (A @ Bm.t() + bias.double()) * 0.5
    # 9 cin products summed in fp32 (8-term fma chains, then a 32-lane tree): 9 cin + 2 roundings incl. the
    # bias add and the scale
    atol = (9 * cin + 2) * U * (A.abs() @ Bm.abs().t() + bias.double().abs()) * 0.5
    check(out[:-1], ref, 0.0, atol, f"small_cout {cout} NHWC")
    assert (out[-1] == -7.0).all()


def test_softmax_rows_strided(L):
    """Row softmax (VAE mid attention, engine/vae.py:139) with lds, ldo > cols (NaN / sentinel gaps) and logits
    spanning a range of 80 within each row, so most probabilities are far below the row maximum."""
    dt = L.operand_dtype()
    rows, cols, lds, ldo = 300, 1000, 1032, 1016
    sb = torch.full((rows, lds), float("nan"), device="cuda")
    sb[:, :cols] = torch.rand(rows, cols, device="cuda", generator=gen(1)) * 80 - 40
    out = torch.full((rows, ldo), sentinel(L), device="cuda", dtype=dt)
    L.softmax_rows(sb, lds, rows, cols, 1.0, out, ldo)
    s = sb[:, :cols].double()
    ref = torch.softmax(s, -1)
    x = (s - s.amax(-1, keepdim=True)).abs()
    # each exp: the scaled argument rounds (u |x|), __expf (2 + 1.173|x|) ulp; the row sum adds cols u; 1/l and
    # the product 2 u; then one 16-bit rounding
    d = U * x + (2 + 1.173 * x) * EXPF_ULP
    rel = d + (ref * d).sum(-1, keepdim=True) + (cols + 2) * U
    check(out[:, :cols], ref, r16(L), rel * ref + a16(L), "softmax_rows")
    assert (out[:, cols:] == sentinel(L)).all()


@pytest.mark.parametrize("out_f32", [False, True])
def test_layernorm_offset_strided(L, out_f32):
    """LayerNorm of the Swin half of SCUNet's y (engine/scunet.py:107): input at an offset pointer with ldx > c,
    NaN in the skipped columns on both sides, output with ldo > c whose columns [c, ldo) are zero-filled."""
    dt = L.operand_dtype()
    rows, c, ldx, off, ldo = 1000, 96, 224, 96, 128
    xb = torch.full((rows, ldx), float("nan"), device="cuda")
    xb[:, off:off + c] = rnd(rows, c, seed=1) * 3 + 1
    gamma, beta = 1 + 0.1 * rnd(c, seed=2), 0.1 * rnd(c, seed=3)
    out = torch.full((rows, ldo), 7.0, device="cuda", dtype=torch.float32 if out_f32 else dt)
    L.layernorm(xb[:, off:], ldx, rows, c, gamma, beta, out, ldo)
    x = xb[:, off:off + c].double()
    mean = x.mean(-1, keepdim=True)
    var = x.var(-1, unbiased=False, keepdim=True)
    rstd = 1 / (var + 1e-5).sqrt()
    xh = (x - mean) * rstd
    ref = xh * gamma.double() + beta.double()
    # mean: c fp32 adds, (c + 1) u of mean |x|; rstd: c + 4 roundings of the variance (its mean error is second
    # order) halved by the root, plus rsqrtf's 2 ulp (2^-22); each output: the subtraction, two products and the
    # add (4 u of their magnitudes)
    dmean = (c + 1) * U * x.abs().mean(-1, keepdim=True)
    drstd = (c + 4) * U / 2 + 2.0 ** -22
    g = gamma.double().abs()
    atol = g * rstd * (dmean + U * (x - mean).abs()) + g * xh.abs() * (drstd + 2 * U) + U * ref.abs()
    if out_f32:
        check(out[:, :c], ref, 0.0, atol, "layernorm fp32")
    else:
        check(out[:, :c], ref, r16(L), atol + a16(L), "layernorm 16-bit")
    assert (out[:, c:] == 0).all(), "columns [c, ldo) must be zero-filled"


@pytest.mark.parametrize("norm,silu", [(False, False), (False, True), (True, False), (True, True)])
def test_gn_apply_modes(L, norm, silu):
    """gn_apply's modes: norm=False, silu=False is a plain cast (SwinIR RSTB tail, engine/swinir.py:141) and must
    be bit-exact; the others against fp64 GroupNorm(32, eps 1e-6, the VAE's Normalize) from gn_stats."""
    dt = L.operand_dtype()
    n, h, w, c = 2, 9, 14, 128
    x = rnd(n, h, w, c, seed=1) * 2 + 0.5
    gamma, beta = 1 + 0.1 * rnd(c, seed=2), 0.1 * rnd(c, seed=3)
    stats = torch.empty(n * 64, device="cuda")
    out = torch.empty(n, h, w, c, device="cuda", dtype=dt)
    if norm:
        ws = torch.zeros(L.gn_workspace_floats(n, h * w, c), device="cuda")
        L.gn_stats(x, None, c, 0, n, h * w, 1e-6, stats, ws)
        L.gn_apply(x, None, c, 0, n, h, w, stats, gamma, beta, out, norm=True, silu=silu)
    else:
        L.gn_apply(x, None, c, 0, n, h, w, None, None, None, out, norm=False, silu=silu)
    if not norm and not silu:
        assert same_bits(out, x.to(dt))
        return
    xd = x.double()
    if norm:
        gx = xd.view(n, h * w, 32, c // 32)
        mean = gx.mean((1, 3), keepdim=True)
        var = gx.var((1, 3), unbiased=False, keepdim=True)
        y = ((gx - mean) / (var + 1e-6).sqrt()).view(n, h, w, c) * gamma.double() + beta.double()
        # statistics: gn_stats sums fp32 partials over a tree about 10 levels deep and combines them in fp64, so
        # the mean is off by ~10 u (6e-7) of max |x| and rstd by as much relative: budget 1e-6 for each. The
        # apply: one fma with the folded a = gamma rstd, b = beta - mean a (3 u)
        ga = gamma.double().abs()
        rs = (1 / (var + 1e-6).sqrt()).view(n, 1, 1, 32).repeat_interleave(c // 32, -1)
        atol = ga * rs * (1e-6 * xd.abs().amax((1, 2), keepdim=True) + 1e-6 * (xd - mean.view(n, 1, 1, 32)
               .repeat_interleave(c // 32, -1)).abs()) + 3 * U * (y.abs() + ga * rs * xd.abs() + beta.double().abs())
    else:
        y, atol = xd, torch.zeros_like(xd)
    if silu:
        atol = 1.1 * atol + silu_bound(y)
        y = F.silu(y)
    check(out, y, r16(L), atol + a16(L), f"gn_apply norm {norm} silu {silu}")
