"""Plain-torch restatement of the Real-ESRGAN batch degradation (reference dataset/batch_transform.py,
degradation.py, diffjpeg.py, utils.py). Test infrastructure: runs on CPU or CUDA with stock torch ops, makes
the reference's random draws in the reference's order, and is what the engine is compared against on the
same device. The per-sample numpy kernel generators are shared with the product (they are already plain
numpy); the fixture pins them to the reference.
"""
from __future__ import annotations

import itertools
import random
from collections.abc import Sequence

import numpy as np
import torch
import torch.nn.functional as F

_STD_Y = [[16, 11, 10, 16, 24, 40, 51, 61], [12, 12, 14, 19, 26, 58, 60, 55], [14, 13, 16, 24, 40, 57, 69, 56],
          [14, 17, 22, 29, 51, 87, 80, 62], [18, 22, 37, 56, 68, 109, 103, 77], [24, 35, 55, 64, 81, 104, 113, 92],
          [49, 64, 78, 87, 103, 121, 120, 101], [72, 92, 95, 98, 112, 100, 103, 99]]


def filter2d(img, kernel):
    k = kernel.size(-1)
    b, c, h, w = img.shape
    x = F.pad(img, (k // 2,) * 4, mode="reflect")
    if kernel.size(0) == 1:
        return F.conv2d(x.view(b * c, 1, *x.shape[2:]), kernel.view(1, 1, k, k)).view(b, c, h, w)
    wt = kernel.view(b, 1, k, k).repeat(1, c, 1, 1).view(b * c, 1, k, k)
    return F.conv2d(x.view(1, b * c, *x.shape[2:]), wt, groups=b * c).view(b, c, h, w)


def usm_kernel(radius=51):
    import cv2
    g = cv2.getGaussianKernel(radius, 0)
    return torch.FloatTensor(np.dot(g, g.T)).unsqueeze_(0)


def usm(img, kernel, weight=0.5, threshold=10):
    blur = filter2d(img, kernel)
    res = img - blur
    soft = filter2d((torch.abs(res) * 255 > threshold).float(), kernel)
    sharp = torch.clip(img + weight * res, 0, 1)
    return soft * sharp + (1 - soft) * img


# ---------------------------------------------------------------- noise
def gaussian_noise(img, sigma_range, gray_prob):
    b, c, h, w = img.shape
    sigma = torch.rand(b, dtype=img.dtype, device=img.device) * (sigma_range[1] - sigma_range[0]) + sigma_range[0]
    gray = (torch.rand(b, dtype=img.dtype, device=img.device) < gray_prob).float().view(b, 1, 1, 1)
    sigma = sigma.view(b, 1, 1, 1)
    any_gray = torch.sum(gray) > 0
    if any_gray:
        ng = (torch.randn(h, w, dtype=img.dtype, device=img.device) * sigma / 255.).view(b, 1, h, w)
    noise = torch.randn(b, c, h, w, dtype=img.dtype, device=img.device) * sigma / 255.
    if any_gray:
        noise = noise * (1 - gray) + ng * gray
    return torch.clamp(img + noise, 0, 1), bool(any_gray)


def _levels(x):
    return torch.clamp((x * 255.0).round(), 0, 255) / 255.


def _shot(q):
    n = [len(torch.unique(q[i])) for i in range(q.size(0))]
    vals = q.new_tensor([2 ** np.ceil(np.log2(v)) for v in n]).view(-1, 1, 1, 1)
    return torch.poisson(q * vals) / vals - q


def poisson_noise(img, scale_range, gray_prob):
    b, c, h, w = img.shape
    scale = torch.rand(b, dtype=img.dtype, device=img.device) * (scale_range[1] - scale_range[0]) + scale_range[0]
    gray = (torch.rand(b, dtype=img.dtype, device=img.device) < gray_prob).float().view(b, 1, 1, 1)
    any_gray = torch.sum(gray) > 0
    if any_gray:
        r, g, bl = img.unbind(1)
        ng = _shot(_levels((0.2989 * r + 0.587 * g + 0.114 * bl).unsqueeze(1))).expand(b, 3, h, w)
    noise = _shot(_levels(img))
    if any_gray:
        noise = noise * (1 - gray) + ng * gray
    return torch.clamp(img + noise * scale.view(b, 1, 1, 1), 0, 1), bool(any_gray)


# ---------------------------------------------------------------- JPEG (differentiable=False)
def _jpeg_tables(device):
    y = torch.tensor(_STD_Y, dtype=torch.float32).T.contiguous()
    c = torch.full((8, 8), 99.0)
    c[:4, :4] = torch.tensor([[17, 18, 24, 47], [18, 21, 26, 66], [24, 26, 56, 99], [47, 66, 99, 99]],
                             dtype=torch.float32)
    cos = np.zeros((8, 8, 8, 8), dtype=np.float32)
    icos = np.zeros((8, 8, 8, 8), dtype=np.float32)
    for x, yy, u, v in itertools.product(range(8), repeat=4):
        cos[x, yy, u, v] = np.cos((2 * x + 1) * u * np.pi / 16) * np.cos((2 * yy + 1) * v * np.pi / 16)
        icos[x, yy, u, v] = np.cos((2 * u + 1) * x * np.pi / 16) * np.cos((2 * v + 1) * yy * np.pi / 16)
    alpha = np.array([1. / np.sqrt(2)] + [1] * 7)
    t = dict(y=y, c=c, cos=torch.from_numpy(cos), icos=torch.from_numpy(icos),
             scale=torch.from_numpy(np.outer(alpha, alpha) * 0.25).float(),
             alpha=torch.from_numpy(np.outer(alpha, alpha)).float(),
             rgb2ycc=torch.from_numpy(np.array([[0.299, 0.587, 0.114], [-0.168736, -0.331264, 0.5],
                                                [0.5, -0.418688, -0.081312]], dtype=np.float32).T),
             ycc2rgb=torch.from_numpy(np.array([[1., 0., 1.402], [1, -0.344136, -0.714136], [1, 1.772, 0]],
                                               dtype=np.float32).T))
    return {k: v.to(device) for k, v in t.items()}


def quality_to_factor(q):
    q = 5000. / q if q < 50 else 200. - q * 2
    return q / 100.


def diffjpeg(x, quality):
    """quality: a [b] tensor (factor per sample from tensor ops) or a number (factor in double on the host)."""
    t = _jpeg_tables(x.device)
    b = x.size(0)
    if isinstance(quality, (int, float)):
        factor = quality_to_factor(quality)
    else:
        factor = quality.clone()
        for i in range(factor.size(0)):
            factor[i] = quality_to_factor(factor[i])
        factor = factor.view(b, 1, 1, 1)
    h, w = x.shape[-2:]
    hp, wp = (16 - h % 16) % 16, (16 - w % 16) % 16
    x = F.pad(x, (0, wp, 0, hp), mode="constant", value=0)
    img = x.permute(0, 2, 3, 1) * 255
    ycc = (torch.tensordot(img, t["rgb2ycc"], dims=1) + torch.tensor([0., 128., 128.], device=x.device)).view(img.shape)
    planes = {"y": ycc[..., 0]}
    for j, name in ((1, "cb"), (2, "cr")):
        planes[name] = F.avg_pool2d(ycc[..., j].unsqueeze(1), kernel_size=2, stride=(2, 2),
                                    count_include_pad=False).squeeze(1)
    rec = {}
    for name, p in planes.items():
        ph, pw = p.shape[1:]
        blocks = p.reshape(b, ph // 8, 8, pw // 8, 8).permute(0, 1, 3, 2, 4).reshape(b, -1, 8, 8)
        coef = t["scale"] * torch.tensordot(blocks - 128, t["cos"], dims=2)
        table = (t["y"] if name == "y" else t["c"]).expand(b, 1, 8, 8) * factor
        deq = torch.round(coef.float() / table) * table
        pix = 0.25 * torch.tensordot(deq * t["alpha"], t["icos"], dims=2) + 128
        rec[name] = pix.view(b, ph // 8, pw // 8, 8, 8).permute(0, 1, 3, 2, 4).reshape(b, ph, pw)

    def up(c):
        hh, ww = c.shape[1:]
        return c.unsqueeze(-1).repeat(1, 1, 2, 2).view(-1, hh * 2, ww * 2)

    image = torch.cat([rec["y"].unsqueeze(3), up(rec["cb"]).unsqueeze(3), up(rec["cr"]).unsqueeze(3)], dim=3)
    rgb = torch.tensordot(image + torch.tensor([0, -128., -128.], device=x.device), t["ycc2rgb"], dims=1)
    rgb = rgb.view(image.shape).permute(0, 3, 1, 2)
    rgb = torch.min(255 * torch.ones_like(rgb), torch.max(torch.zeros_like(rgb), rgb)) / 255
    return rgb[:, :, :h, :w].contiguous()


# ---------------------------------------------------------------- the batch transform
class BatchTransform:
    """RealESRGANBatchTransform in plain torch; `branches` records the branch each stage took."""

    def __init__(self, **cfg):
        self.cfg = cfg
        self.kernel = usm_kernel() if cfg["use_sharpener"] else None
        self.branches = []

    def _updown(self, probs, rng):
        kind = random.choices(["up", "down", "keep"], probs)[0]
        self.branches.append(kind)
        if kind == "up":
            return np.random.uniform(1, rng[1])
        if kind == "down":
            return np.random.uniform(rng[0], 1)
        return 1

    def _mode(self):
        m = random.choice(["area", "bilinear", "bicubic"])
        self.branches.append(m)
        return m

    def _noise(self, out, gp, sr, pr, gray):
        kind = "gaussian" if np.random.uniform() < gp else "poisson"
        out, any_gray = (gaussian_noise(out, sr, gray) if kind == "gaussian" else poisson_noise(out, pr, gray))
        self.branches += [kind, "gray" if any_gray else "colour"]
        return out

    def _jpeg(self, out, rng):
        q = out.new_zeros(out.size(0)).uniform_(*rng)
        return diffjpeg(torch.clamp(out, 0, 1), q)

    @torch.no_grad()
    def __call__(self, batch):
        c = self.cfg
        hq = batch["hq"]
        if self.kernel is not None:
            hq = usm(hq, self.kernel.to(hq))
        oh, ow = hq.shape[2:4]
        out = filter2d(hq, batch["kernel1"].to(hq))
        scale = self._updown(c["resize_prob"], c["resize_range"])
        out = F.interpolate(out, scale_factor=scale, mode=self._mode())
        out = self._noise(out, c["gaussian_noise_prob"], c["noise_range"], c["poisson_scale_range"],
                          c["gray_noise_prob"])
        out = self._jpeg(out, c["jpeg_range"])
        if np.random.uniform() < c["second_blur_prob"]:
            self.branches.append("blur2")
            out = filter2d(out, batch["kernel2"].to(hq))
        s2 = c["stage2_scale"]
        if isinstance(s2, Sequence):
            self.branches.append("stage2_range")
            s2 = np.random.uniform(*s2)
        else:
            self.branches.append("stage2_scalar")
        h2, w2 = int(oh / s2), int(ow / s2)
        scale = self._updown(c["resize_prob2"], c["resize_range2"])
        out = F.interpolate(out, size=(int(h2 * scale), int(w2 * scale)), mode=self._mode())
        out = self._noise(out, c["gaussian_noise_prob2"], c["noise_range2"], c["poisson_scale_range2"],
                          c["gray_noise_prob2"])
        if np.random.uniform() < 0.5:
            self.branches.append("sinc_then_jpeg")
            out = filter2d(F.interpolate(out, size=(h2, w2), mode=self._mode()), batch["sinc_kernel"].to(hq))
            out = self._jpeg(out, c["jpeg_range2"])
        else:
            self.branches.append("jpeg_then_sinc")
            out = self._jpeg(out, c["jpeg_range2"])
            out = filter2d(F.interpolate(out, size=(h2, w2), mode=self._mode()), batch["sinc_kernel"].to(hq))
        if s2 != 1:
            out = F.interpolate(out, size=(oh, ow), mode="bicubic")
        lq = torch.clamp((out * 255.0).round(), 0, 255) / 255.0
        self._queue(hq, lq, batch["txt"])
        return ((self.gt * 2 - 1).float().permute(0, 2, 3, 1).contiguous(),
                self.lq.float().permute(0, 2, 3, 1).contiguous(), self.txt)

    def _queue(self, gt, lq, txt):
        b = lq.size(0)
        n = self.cfg["queue_size"]
        if not hasattr(self, "qlq"):
            self.qlq = torch.zeros(n, *lq.shape[1:]).to(lq)
            self.qgt = torch.zeros(n, *gt.shape[1:]).to(lq)
            self.qtxt, self.ptr = [None] * n, 0
        if self.ptr == n:
            self.branches.append("queue_full")
            idx = torch.randperm(n)
            self.qlq, self.qgt = self.qlq[idx], self.qgt[idx]
            self.qtxt = [self.qtxt[j] for j in idx]
            lq_out, gt_out, txt_out = self.qlq[:b].clone(), self.qgt[:b].clone(), self.qtxt[:b]
            self.qlq[:b], self.qgt[:b] = lq, gt
            self.qtxt[:b] = list(txt[:b])
            self.lq, self.gt, self.txt = lq_out, gt_out, txt_out
        else:
            self.branches.append("queue_fill")
            self.qlq[self.ptr:self.ptr + b], self.qgt[self.ptr:self.ptr + b] = lq, gt
            self.qtxt[self.ptr:self.ptr + b] = list(txt[:b])
            self.ptr += b
            self.lq, self.gt, self.txt = lq, gt, txt
