"""RealESRGANDataset (reference dataset/realesrgan.py): per-sample HQ crop, flips and the three blur kernels.

The per-sample work is numpy / PIL in dataloader workers, drawing from Python's `random` and numpy's global
generator in the reference's order; the batch degradation is RealESRGANBatchTransform on the engine.
"""
from __future__ import annotations

import io
import math
import random
import time
from typing import Any, Dict, List, Mapping, Optional, Sequence

import numpy as np
import torch
from PIL import Image
from torch.utils import data

from ..utils.common import instantiate_from_config
from .degradation import circular_lowpass_kernel, random_mixed_kernels
from .utils import augment, center_crop_arr, load_file_metas, random_crop_arr


class RealESRGANDataset(data.Dataset):

    def __init__(self, file_metas: List[Dict[str, str]], p_long_prompt: float, file_backend_cfg: Mapping[str, Any],
                 out_size: int, crop_type: str, use_hflip: bool, use_rot: bool,
                 blur_kernel_size: int, kernel_list: Sequence[str], kernel_prob: Sequence[float],
                 blur_sigma: Sequence[float], betag_range: Sequence[float], betap_range: Sequence[float],
                 sinc_prob: float,
                 blur_kernel_size2: int, kernel_list2: Sequence[str], kernel_prob2: Sequence[float],
                 blur_sigma2: Sequence[float], betag_range2: Sequence[float], betap_range2: Sequence[float],
                 sinc_prob2: float, final_sinc_prob: float, p_empty_prompt: float) -> None:
        super().__init__()
        self.file_metas = file_metas
        self.image_files = load_file_metas(file_metas)
        assert 0 <= p_long_prompt <= 1, f"p_long_prompt {p_long_prompt} should be a probability between [0, 1]"
        self.p_long_prompt = p_long_prompt
        self.file_backend = instantiate_from_config(file_backend_cfg)
        assert crop_type in ["none", "center", "random"]
        self.out_size, self.crop_type = out_size, crop_type
        # (blur_kernel_size, as in the reference, is not used: kernel sizes are drawn from kernel_range)
        self.blur_kernel_size, self.blur_kernel_size2 = blur_kernel_size, blur_kernel_size2
        self.stage1 = (kernel_list, kernel_prob, blur_sigma, betag_range, betap_range, sinc_prob)
        self.stage2 = (kernel_list2, kernel_prob2, blur_sigma2, betag_range2, betap_range2, sinc_prob2)
        self.final_sinc_prob = final_sinc_prob
        self.use_hflip, self.use_rot = use_hflip, use_rot
        self.kernel_range = [2 * v + 1 for v in range(3, 11)]      # 7, 9, ..., 21
        self.pulse_tensor = torch.zeros(21, 21).float()            # identity filter
        self.pulse_tensor[10, 10] = 1
        self.p_empty_prompt = p_empty_prompt

    def load_gt_image(self, image_path: str, max_retry: int = 5) -> Optional[np.ndarray]:
        """HWC RGB uint8 image of out_size x out_size, or None when it cannot be read or decoded."""
        image_bytes = None
        while image_bytes is None:
            if max_retry == 0:
                return None
            try:
                image_bytes = self.file_backend.get(image_path)
            except Exception:
                return None
            max_retry -= 1
            if image_bytes is None:
                time.sleep(0.5)
        try:
            image = Image.open(io.BytesIO(image_bytes)).convert("RGB")
        except Exception:
            return None
        if self.crop_type == "none":
            assert image.height == self.out_size and image.width == self.out_size
            return np.array(image)
        if image.height == self.out_size and image.width == self.out_size:
            return np.array(image)
        if self.crop_type == "center":
            return center_crop_arr(image, self.out_size)
        return random_crop_arr(image, self.out_size, min_crop_frac=0.7)

    def _blur_kernel(self, kernel_list, kernel_prob, blur_sigma, betag_range, betap_range, sinc_prob):
        """One stage's kernel, zero-padded to 21 x 21: a sinc with probability sinc_prob, else a mixed kernel."""
        size = random.choice(self.kernel_range)
        if np.random.uniform() < sinc_prob:
            omega_c = np.random.uniform(np.pi / 3, np.pi) if size < 13 else np.random.uniform(np.pi / 5, np.pi)
            kernel = circular_lowpass_kernel(omega_c, size, pad_to=False)
        else:
            kernel = random_mixed_kernels(kernel_list, kernel_prob, size, blur_sigma, blur_sigma,
                                          [-math.pi, math.pi], betag_range, betap_range, noise_range=None)
        p = (21 - size) // 2
        return np.pad(kernel, ((p, p), (p, p)))

    @torch.no_grad()
    def __getitem__(self, index: int) -> Dict[str, Any]:
        img_gt = None
        while img_gt is None:
            image_file = self.image_files[index]
            gt_path = image_file["image_path"]
            long = np.random.uniform() < self.p_long_prompt
            prompt = image_file["long_prompt"] if long else image_file["short_prompt"]
            img_gt = self.load_gt_image(gt_path)
            if img_gt is None:
                print(f"failed to load {gt_path}, try another image")
                index = random.randint(0, len(self) - 1)

        # BGR float32 in [0, 1], the layout the flips were written for
        img_hq = (img_gt[..., ::-1] / 255.0).astype(np.float32)
        if np.random.uniform() < self.p_empty_prompt:
            prompt = ""
        img_hq = augment(img_hq, self.use_hflip, self.use_rot)

        kernel = self._blur_kernel(*self.stage1)
        kernel2 = self._blur_kernel(*self.stage2)
        if np.random.uniform() < self.final_sinc_prob:
            size = random.choice(self.kernel_range)
            omega_c = np.random.uniform(np.pi / 3, np.pi)
            sinc_kernel = torch.FloatTensor(circular_lowpass_kernel(omega_c, size, pad_to=21))
        else:
            sinc_kernel = self.pulse_tensor

        img_hq = torch.from_numpy(img_hq[..., ::-1].transpose(2, 0, 1).copy()).float()
        return {"hq": img_hq, "kernel1": torch.FloatTensor(kernel), "kernel2": torch.FloatTensor(kernel2),
                "sinc_kernel": sinc_kernel, "txt": prompt}

    def __len__(self) -> int:
        return len(self.image_files)
