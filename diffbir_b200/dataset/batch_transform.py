"""Batch-level Real-ESRGAN degradation (reference dataset/batch_transform.py) on the engine.

`RealESRGANBatchTransform` makes the reference's random draws (Python `random`, numpy's global generator,
torch on the batch's device, torch's CPU generator for the queue shuffle) in the reference's order and with
the same shapes, so a seeded call draws the same degradation parameters and noise. Everything between the
draws runs in csrc/degrade.cu. The one host sync is where the reference branches on device data: whether any
sample of a noise step takes gray noise.
"""
from __future__ import annotations

import random
from typing import Any, Dict, List, Sequence, Union

import numpy as np
import torch

from ._device import require_cuda
from .degradation import random_add_gaussian_noise_pt, random_add_poisson_noise_pt
from .utils import DiffJPEG, USMSharp, filter2D

_MODES = ["area", "bilinear", "bicubic"]


def resize(x, mode, *, scale=None, size=None):
    """F.interpolate(x, scale_factor=scale | size=size, mode=mode) with align_corners=False, on `dbir_resize`.
    The scale_factor form gives floor(in * scale) and maps coordinates with 1/scale; the size form maps
    with in/out, as PyTorch does."""
    from .. import lib
    b, c, h, w = x.shape
    if scale is not None:
        ho, wo = int(h * scale), int(w * scale)
        rh = rw = float(np.float32(1.0 / scale))
    else:
        ho, wo = size
        rh, rw = float(np.float32(h) / np.float32(ho)), float(np.float32(w) / np.float32(wo))
    out = torch.empty(b, c, ho, wo, dtype=x.dtype, device=x.device)
    lib.resize(x, out, mode, rh, rw)
    return out


class BatchTransform:
    def __call__(self, batch: Any) -> Any:
        raise NotImplementedError


class IdentityBatchTransform(BatchTransform):
    def __call__(self, batch: Any) -> Any:
        return batch


class RealESRGANBatchTransform(BatchTransform):
    """Second-order degradation of a batch of HQ images into (hq, lq, txt) training pairs, with the
    training-pair queue that mixes degradations across batches (queue_size a multiple of the batch)."""

    def __init__(self, use_sharpener: bool, queue_size: int, resize_prob: Sequence[float],
                 resize_range: Sequence[float], gray_noise_prob: float, gaussian_noise_prob: float,
                 noise_range: Sequence[float], poisson_scale_range: Sequence[float], jpeg_range: Sequence[int],
                 second_blur_prob: float, stage2_scale: Union[float, Sequence[Union[float, int]]],
                 resize_prob2: Sequence[float], resize_range2: Sequence[float], gray_noise_prob2: float,
                 gaussian_noise_prob2: float, noise_range2: Sequence[float], poisson_scale_range2: Sequence[float],
                 jpeg_range2: Sequence[int]) -> None:
        super().__init__()
        assert isinstance(stage2_scale, (float, int)) or (
            isinstance(stage2_scale, Sequence) and len(stage2_scale) == 2
            and all(isinstance(x, (float, int)) for x in stage2_scale)
        ), f"stage2_scale can not be {type(stage2_scale)}"
        self.resize_prob, self.resize_range = resize_prob, resize_range
        self.gray_noise_prob, self.gaussian_noise_prob = gray_noise_prob, gaussian_noise_prob
        self.noise_range, self.poisson_scale_range, self.jpeg_range = noise_range, poisson_scale_range, jpeg_range
        self.second_blur_prob, self.stage2_scale = second_blur_prob, stage2_scale
        self.resize_prob2, self.resize_range2 = resize_prob2, resize_range2
        self.gray_noise_prob2, self.gaussian_noise_prob2 = gray_noise_prob2, gaussian_noise_prob2
        self.noise_range2, self.poisson_scale_range2, self.jpeg_range2 = noise_range2, poisson_scale_range2, jpeg_range2
        self.use_sharpener = use_sharpener
        self.usm_sharpener = USMSharp() if use_sharpener else None
        self.queue_size = queue_size
        self.jpeger = DiffJPEG(differentiable=False)

    # -- one degradation stage's pieces, each with the reference's draws
    @staticmethod
    def _updown(probs, rng):
        kind = random.choices(["up", "down", "keep"], probs)[0]
        if kind == "up":
            return np.random.uniform(1, rng[1])
        if kind == "down":
            return np.random.uniform(rng[0], 1)
        return 1

    @staticmethod
    def _noise(out, gaussian_prob, sigma_range, scale_range, gray_prob):
        if np.random.uniform() < gaussian_prob:
            return random_add_gaussian_noise_pt(out, sigma_range=sigma_range, clip=True, rounds=False,
                                                gray_prob=gray_prob)
        return random_add_poisson_noise_pt(out, scale_range=scale_range, gray_prob=gray_prob, clip=True,
                                           rounds=False)

    def _jpeg(self, out, rng):
        quality = out.new_zeros(out.size(0)).uniform_(*rng)
        return self.jpeger(out, quality=quality, clamp=True)

    @torch.no_grad()
    def _dequeue_and_enqueue(self):
        """Training-pair pool: once full, each batch is swapped for a random batch-sized draw from the pool, so
        one batch mixes the degradations of several calls."""
        b, c, h, w = self.lq.size()
        if not hasattr(self, "queue_lr"):
            assert self.queue_size % b == 0, f"queue size {self.queue_size} should be divisible by batch size {b}"
            self.queue_lr = torch.zeros(self.queue_size, c, h, w).to(self.lq)
            _, c, h, w = self.gt.size()
            self.queue_gt = torch.zeros(self.queue_size, c, h, w).to(self.lq)
            self.queue_txt = [None] * self.queue_size
            self.queue_ptr = 0
        if self.queue_ptr == self.queue_size:
            idx = torch.randperm(self.queue_size)
            self.queue_lr = self.queue_lr[idx]
            self.queue_gt = self.queue_gt[idx]
            self.queue_txt = [self.queue_txt[j] for j in idx]
            lq, gt, txt = self.queue_lr[0:b].clone(), self.queue_gt[0:b].clone(), self.queue_txt[0:b]
            self.queue_lr[0:b] = self.lq
            self.queue_gt[0:b] = self.gt
            self.queue_txt[0:b] = list(self.txt[0:b])
            self.lq, self.gt, self.txt = lq, gt, txt
        else:
            p = self.queue_ptr
            self.queue_lr[p: p + b] = self.lq
            self.queue_gt[p: p + b] = self.gt
            for i in range(b):
                self.queue_txt[p + i] = self.txt[i]
            self.queue_ptr = p + b

    @torch.no_grad()
    def __call__(self, batch: Dict[str, Union[torch.Tensor, str]]) -> tuple:
        """batch: hq [b, 3, h, w] in [0, 1] on CUDA, kernel1 / kernel2 / sinc_kernel [b, 21, 21], txt.
        Returns (hq NHWC in [-1, 1], lq NHWC in [0, 1] on 8-bit levels, txt)."""
        from .. import lib
        hq = batch["hq"]
        require_cuda(hq, "RealESRGANBatchTransform")
        hq = hq.float().contiguous()
        if self.use_sharpener:
            hq = self.usm_sharpener(hq)
        ori_h, ori_w = hq.size()[2:4]

        # first degradation: blur, resize, noise, JPEG
        out = filter2D(hq, batch["kernel1"])
        scale = self._updown(self.resize_prob, self.resize_range)
        out = resize(out, random.choice(_MODES), scale=scale)
        out = self._noise(out, self.gaussian_noise_prob, self.noise_range, self.poisson_scale_range,
                          self.gray_noise_prob)
        out = self._jpeg(out, self.jpeg_range)

        # second degradation: blur, resize, noise, then [resize back + sinc] and JPEG in a random order
        if np.random.uniform() < self.second_blur_prob:
            out = filter2D(out, batch["kernel2"])
        if isinstance(self.stage2_scale, Sequence):
            stage2_scale = np.random.uniform(*self.stage2_scale)
        else:
            stage2_scale = self.stage2_scale
        stage2_h, stage2_w = int(ori_h / stage2_scale), int(ori_w / stage2_scale)
        scale = self._updown(self.resize_prob2, self.resize_range2)
        out = resize(out, random.choice(_MODES), size=(int(stage2_h * scale), int(stage2_w * scale)))
        out = self._noise(out, self.gaussian_noise_prob2, self.noise_range2, self.poisson_scale_range2,
                          self.gray_noise_prob2)
        if np.random.uniform() < 0.5:
            out = resize(out, random.choice(_MODES), size=(stage2_h, stage2_w))
            out = filter2D(out, batch["sinc_kernel"])
            out = self._jpeg(out, self.jpeg_range2)
        else:
            out = self._jpeg(out, self.jpeg_range2)
            out = resize(out, random.choice(_MODES), size=(stage2_h, stage2_w))
            out = filter2D(out, batch["sinc_kernel"])
        if stage2_scale != 1:
            out = resize(out, "bicubic", size=(ori_h, ori_w))
        lq = torch.empty_like(out)
        lib.lq_levels(out, lq)

        self.gt, self.lq, self.txt = hq, lq, batch["txt"]
        self._dequeue_and_enqueue()
        b, c, h, w = self.lq.shape
        lq_nhwc = torch.empty(b, h, w, c, dtype=torch.float32, device=self.lq.device)
        hq_nhwc = torch.empty(b, h, w, c, dtype=torch.float32, device=self.lq.device)
        lib.pair_nhwc(self.lq.contiguous(), self.gt.contiguous(), lq_nhwc, hq_nhwc)
        return hq_nhwc, lq_nhwc, self.txt
