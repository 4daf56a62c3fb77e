"""Real-ESRGAN degradation on the engine (csrc/degrade.cu) against fp64 torch, the plain-torch oracle and
PyTorch's own fp32 ops on the same H100 (TF32 off). Each bar states the value measured on an H100 80GB HBM3."""
import math
import pickle
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from diffbir_b200 import lib as L
from oracle import degradation as od
from tests.gpu_util import no_tf32, psnr

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(autouse=True)
def _setup():
    no_tf32()
    L.load()


def _img(*shape, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.rand(*shape, generator=g, device=DEV)


# the last tile of a row or column can be short (w = 33: one column), and images can be barely larger than the
# reflect pad (19 > 21 // 2, 28 > 51 // 2), where the staged halo reaches furthest past the image
@pytest.mark.parametrize("k,shared,shape", [(21, False, (3, 3, 100, 77)), (21, True, (2, 3, 64, 33)),
                                            (51, True, (2, 3, 129, 95)), (51, False, (2, 3, 70, 200)),
                                            (21, False, (2, 3, 19, 19)), (51, True, (1, 3, 40, 28)),
                                            (51, False, (2, 3, 26, 33))])
def test_filter2d_matches_fp64(k, shared, shape):
    x = _img(*shape)
    kern = torch.rand(1 if shared else shape[0], k, k, device=DEV)
    kern /= kern.sum(dim=(1, 2), keepdim=True)
    out = torch.empty_like(x)
    L.filter2d(x, kern, out)
    ref = od.filter2d(x.double(), kern.double())
    err = (out.double() - ref).abs().max().item()
    print(f"filter2d k={k} shared={shared} {shape}: max |err| vs fp64 {err:.2e}")
    # fp32 accumulation of up to 2601 taps summing to 1; measured on an H100 80GB HBM3: k = 21 at most 6.3e-7,
    # k = 51 at most 1.55e-6
    assert err < 2e-6, err


def test_filter2d_threshold_mask_matches_fp64():
    x = _img(2, 3, 90, 64)
    kern = od.usm_kernel().to(DEV)
    blur, soft = torch.empty_like(x), torch.empty_like(x)
    L.filter2d(x, kern, blur)
    L.filter2d(x, kern, soft, sub=blur, threshold=10)
    mask = (torch.abs(x - blur) * 255 > 10).float()
    err = (soft.double() - od.filter2d(mask.double(), kern.double())).abs().max().item()
    print(f"filter2d threshold mask: max |err| vs fp64 {err:.2e}")
    assert err < 2e-6, err                 # measured on an H100: 1.38e-6


@pytest.mark.parametrize("mode", ["area", "bilinear", "bicubic"])
@pytest.mark.parametrize("hw,form,arg", [(512, "scale", 0.1484375), (128, "scale", 1.5), (96, "scale", 1),
                                         (512, "size", (76, 76)), (128, "size", (192, 160)), (96, "size", (96, 96))])
def test_resize_matches_fp64(mode, hw, form, arg):
    from diffbir_b200.dataset.batch_transform import resize
    x = _img(2, 3, hw, hw)
    kw = {"scale_factor": arg} if form == "scale" else {"size": arg}
    out = resize(x, mode, **({"scale": arg} if form == "scale" else {"size": arg}))
    ref = F.interpolate(x.double(), mode=mode, **kw)
    assert out.shape == ref.shape
    err = (out.double() - ref).abs().max().item()
    # Source coordinates are fp32, as in PyTorch's own fp32 kernels: at 512 -> 76 the fractional tap offset
    # carries ~ulp(512) of error, 2.3e-5 measured on an H100 (area, which has no fractional taps: < 1e-6).
    assert err < 3e-5, err
    assert (out - F.interpolate(x, mode=mode, **kw)).abs().max().item() < 3e-5
    # the ratio handed to the kernel is what the product computes (also called directly here)
    direct = torch.empty_like(out)
    rh = float(np.float32(1.0 / arg)) if form == "scale" else float(np.float32(hw) / np.float32(out.shape[2]))
    rw = float(np.float32(1.0 / arg)) if form == "scale" else float(np.float32(hw) / np.float32(out.shape[3]))
    L.resize(x, direct, mode, rh, rw)
    assert torch.equal(direct, out)


@pytest.mark.parametrize("gray", [False, True])
def test_gaussian_noise_is_torch_bit_for_bit(gray):
    b, c, h, w = 4, 3, 77, 130
    x = _img(b, c, h, w)
    u_sigma, u_gray = torch.rand(b, device=DEV), torch.tensor([0.1, 0.9, 0.3, 0.7], device=DEV)
    noise, ng = torch.randn(b, c, h, w, device=DEV), torch.randn(h, w, device=DEV)
    out = torch.empty_like(x)
    L.gaussian_noise(x, noise, ng if gray else None, u_sigma, 1, 29, u_gray, 0.4, out)
    sigma = (u_sigma * 29 + 1).view(b, 1, 1, 1)
    ref = noise * sigma / 255.
    if gray:
        g = (u_gray < 0.4).float().view(b, 1, 1, 1)
        ref = ref * (1 - g) + (ng * sigma / 255.).view(b, 1, h, w) * g
    assert torch.equal(out, torch.clamp(x + ref, 0, 1))


@pytest.mark.parametrize("gray", [False, True])
def test_poisson_noise_is_torch_bit_for_bit(gray):
    b, c, h, w = 3, 3, 61, 90
    x = _img(b, c, h, w)
    x[1] = torch.round(x[1] * 5) / 5            # few levels: vals = 8
    x[2] = x[2] * 0.3 + 0.2
    u_scale, u_gray = torch.rand(b, device=DEV), torch.tensor([0.1, 0.9, 0.3], device=DEV)

    def levels(img, gray_img):
        q = torch.empty(b, 1 if gray_img else c, h, w, device=DEV)
        hist = torch.empty(b, 256, dtype=torch.int32, device=DEV)
        vals, rate = torch.empty(b, device=DEV), torch.empty_like(q)
        L.noise_levels(img, q, hist, gray=gray_img)
        src = img
        if gray_img:
            src = (0.2989 * img[:, 0] + 0.587 * img[:, 1] + 0.114 * img[:, 2]).unsqueeze(1)
        ref_q = torch.clamp((src * 255.0).round(), 0, 255) / 255.
        assert torch.equal(q, ref_q)
        counts = [len(torch.unique(ref_q[i])) for i in range(b)]
        assert [int((hist[i] > 0).sum()) for i in range(b)] == counts
        assert hist.sum(1).tolist() == [q[0].numel()] * b
        L.poisson_rate(q, hist, vals, rate)
        ref_vals = torch.tensor([2 ** np.ceil(np.log2(n)) for n in counts], device=DEV, dtype=torch.float32)
        assert torch.equal(vals, ref_vals) and torch.equal(rate, q * ref_vals.view(b, 1, 1, 1))
        return q, torch.poisson(rate), vals

    extra = {}
    if gray:
        qg, dg, vg = levels(x, True)
        extra = dict(q_gray=qg, draw_gray=dg, vals_gray=vg, u_gray=u_gray, gray_prob=0.4)
    q, d, v = levels(x, False)
    out = torch.empty_like(x)
    L.poisson_noise(x, q, d, v, u_scale, 0.05, 2.95, out, **extra)
    noise = d / v.view(b, 1, 1, 1) - q
    if gray:
        g = (u_gray < 0.4).float().view(b, 1, 1, 1)
        noise = noise * (1 - g) + (dg / vg.view(b, 1, 1, 1) - qg).expand(b, 3, h, w) * g
    ref = torch.clamp(x + noise * (u_scale * 2.95 + 0.05).view(b, 1, 1, 1), 0, 1)
    assert torch.equal(out, ref)


def test_diffjpeg_matches_oracle():
    x = _img(4, 3, 133, 250)
    x = F.avg_pool2d(F.pad(x, (1, 1, 1, 1), mode="replicate"), 3, 1)     # some smooth content
    quality = torch.tensor([30.0, 49.5, 50.0, 94.7], device=DEV)
    out = torch.empty_like(x)
    L.diffjpeg(x, quality, out)
    ref = od.diffjpeg(x, quality.clone())
    diff = (out - ref).abs()
    frac = (diff > 1e-4).float().mean().item()
    print(f"diffjpeg: max |d| {diff.max().item():.3e}, share of pixels off by > 1e-4: {frac:.2e}")
    # bit-identical on an H100 (0 pixels differ); a coefficient on the other side of a rounding tie would move
    # one 8x8 block by one quantisation step, which this bar would tolerate in a few blocks
    assert frac < 2e-3, frac
    assert psnr(out, ref, peak=1.0) > 60
    clamped = torch.empty_like(x)
    L.diffjpeg(x * 1.4 - 0.2, quality, clamped, clamp_in=True)
    L.diffjpeg(torch.clamp(x * 1.4 - 0.2, 0, 1), quality, out)
    assert torch.equal(clamped, out)


@pytest.mark.parametrize("quality", [30, 37.3, 50, 71.9, 95])
def test_diffjpeg_scalar_quality_matches_oracle(quality):
    """A Python-number quality: the factor is the reference's double quality_to_factor, rounded once to fp32."""
    from diffbir_b200.dataset.diffjpeg import DiffJPEG
    x = F.avg_pool2d(F.pad(_img(2, 3, 70, 90, seed=6), (1, 1, 1, 1), mode="replicate"), 3, 1)
    out = DiffJPEG(differentiable=False)(x, quality)
    ref = od.diffjpeg(x, quality)
    frac = ((out - ref).abs() > 1e-4).float().mean().item()
    print(f"diffjpeg quality {quality}: max |d| {(out - ref).abs().max().item():.3e}, share off {frac:.2e}")
    # measured on an H100: no pixel off by more than 1e-4 (largest difference 1.8e-7) at any of these qualities
    assert frac < 2e-3, frac
    factor = torch.full((2,), float(np.float32(od.quality_to_factor(quality))), device=DEV)
    direct = torch.empty_like(x)
    L.diffjpeg(x, factor, direct, is_factor=True)
    assert torch.equal(direct, out)


def test_usm_and_epilogue_are_torch_bit_for_bit():
    img, blur, soft = _img(2, 3, 40, 50, seed=1), _img(2, 3, 40, 50, seed=2), _img(2, 3, 40, 50, seed=3)
    out = torch.empty_like(img)
    L.usm_blend(img, blur, soft, 0.5, out)
    res = img - blur
    assert torch.equal(out, soft * torch.clip(img + 0.5 * res, 0, 1) + (1 - soft) * img)
    x = _img(2, 3, 40, 50, seed=4) * 1.2 - 0.1
    lq = torch.empty_like(x)
    L.lq_levels(x, lq)
    assert torch.equal(lq, torch.clamp((x * 255.0).round(), 0, 255) / 255.0)
    lq_n, hq_n = torch.empty(2, 40, 50, 3, device=DEV), torch.empty(2, 40, 50, 3, device=DEV)
    L.pair_nhwc(lq, img, lq_n, hq_n)
    assert torch.equal(lq_n, lq.permute(0, 2, 3, 1)) and torch.equal(hq_n, (img * 2 - 1).permute(0, 2, 3, 1))


def test_usm_module_matches_oracle():
    from diffbir_b200.dataset.utils import USMSharp
    x = _img(2, 3, 128, 96, seed=5)
    m = USMSharp().to(x)
    ref = od.usm(x, od.usm_kernel().to(DEV))
    err = (m(x) - ref).abs().max().item()
    print(f"USMSharp vs oracle: max |err| {err:.2e}")
    # measured on an H100: 1.0e-6. The bar allows for a mask pixel right at the threshold flipping between the
    # two summation orders, which moves the output by up to one soft-mask tap weight times the residual.
    assert err < 1e-3, err


# ------------------------------------------------------------------------------ end to end
V21 = dict(use_sharpener=True, queue_size=16, resize_prob=[0.2, 0.7, 0.1], resize_range=[0.15, 1.5],
           gaussian_noise_prob=0.5, noise_range=[1, 30], poisson_scale_range=[0.05, 3], gray_noise_prob=0.4,
           jpeg_range=[30, 95], stage2_scale=4, second_blur_prob=0.8, resize_prob2=[0.3, 0.4, 0.3],
           resize_range2=[0.3, 1.2], gaussian_noise_prob2=0.5, noise_range2=[1, 25],
           poisson_scale_range2=[0.05, 2.5], gray_noise_prob2=0.4, jpeg_range2=[30, 95])


def v21_batch(b, size, seed):
    """A batch as RealESRGANDataset would give it (v2.1 kernel settings), built from private generators."""
    from diffbir_b200.dataset.degradation import circular_lowpass_kernel, random_mixed_kernels
    state = random.getstate(), np.random.get_state()
    random.seed(seed)
    np.random.seed(seed)
    types = ["iso", "aniso", "generalized_iso", "generalized_aniso", "plateau_iso", "plateau_aniso"]
    probs = [0.45, 0.25, 0.12, 0.03, 0.12, 0.03]
    ks = []
    for _ in range(b):
        row = []
        for sig in ([0.2, 3], [0.2, 1.5]):
            size_k = random.choice(range(7, 22, 2))
            k = random_mixed_kernels(types, probs, size_k, sig, sig, [-math.pi, math.pi], [0.5, 4], [1, 2], None)
            row.append(np.pad(k, (21 - size_k) // 2))
        row.append(circular_lowpass_kernel(np.random.uniform(np.pi / 3, np.pi), 11, pad_to=21))
        ks.append(row)
    hq = torch.from_numpy(np.random.RandomState(seed).rand(b, 3, size, size).astype(np.float32))
    random.setstate(state[0])
    np.random.set_state(state[1])
    hq = F.avg_pool2d(F.pad(hq, (2, 2, 2, 2), mode="replicate"), 5, 1)       # image-like local correlation
    k = [torch.from_numpy(np.stack([r[i] for r in ks])).float().to(DEV) for i in range(3)]
    return dict(hq=hq.to(DEV), kernel1=k[0], kernel2=k[1], sinc_kernel=k[2], txt=[f"{seed}:{i}" for i in range(b)])


def rng_states():
    return (pickle.dumps(random.getstate()), pickle.dumps(np.random.get_state()), torch.get_rng_state(),
            torch.cuda.get_rng_state())


def _seed(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_transform_matches_oracle_on_device(seed):
    from diffbir_b200.dataset.batch_transform import RealESRGANBatchTransform
    eng, ora = RealESRGANBatchTransform(**V21), od.BatchTransform(**V21)
    batches = [v21_batch(8, 512, 100 * seed + i) for i in range(3)]
    same, total, worst = 0, 0, float("inf")
    for i, batch in enumerate(batches):
        _seed(1000 * seed + i)
        hq_e, lq_e, txt_e = eng(batch)
        st_e = rng_states()
        _seed(1000 * seed + i)
        hq_o, lq_o, txt_o = ora(batch)
        st_o = rng_states()
        assert st_e[:2] == st_o[:2] and torch.equal(st_e[2], st_o[2]) and torch.equal(st_e[3], st_o[3])
        assert txt_e == txt_o
        assert (hq_e - hq_o).abs().max().item() < 1e-5
        le, lo = torch.round(lq_e * 255), torch.round(lq_o * 255)
        same += (le == lo).sum().item()
        total += le.numel()
        worst = min(worst, psnr(lq_e, lq_o, peak=1.0))
    frac = same / total
    print(f"seed {seed}: identical lq levels {frac:.6f}, worst lq PSNR {worst:.2f} dB, branches {ora.branches}")
    # measured on an H100 80GB HBM3 (seeds 0, 1, 2), two runs: 0.999997-0.999999 / 1.0 / 1.0 identical, worst PSNR
    # 100.2 dB (the oracle's cuDNN convolutions may pick a different summation order per run)
    assert frac > 0.9999 and worst > 80, (frac, worst)
