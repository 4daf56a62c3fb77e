"""Dataset helpers (reference dataset/utils.py): file lists, crops, flips, and the engine's filter2D / USMSharp."""
from __future__ import annotations

import math
import os
import random
from typing import Dict, List

import numpy as np
import torch
from PIL import Image

from ._device import require_cuda
from .diffjpeg import DiffJPEG  # noqa: F401  (the reference re-exports it from here)


def load_file_list(file_list_path: str) -> List[Dict[str, str]]:
    """One image path per non-empty line."""
    with open(file_list_path, "r") as fin:
        return [{"image_path": p, "prompt": ""} for p in (line.strip() for line in fin) if p]


def load_file_metas(file_metas: List[Dict[str, str]]) -> List[Dict[str, str]]:
    """Rows of each parquet file list, in file order, as {image_path, short_prompt, long_prompt}."""
    import pyarrow.parquet as pq
    files = []
    for meta in file_metas:
        path = meta["file_list"]
        assert os.path.splitext(path)[1].lower() == ".parquet", "only support parquet format"
        keys = (meta["image_path_key"], meta["short_prompt_key"], meta["long_prompt_key"])
        table = pq.read_table(path, columns=list(dict.fromkeys(keys)))
        cols = [table.column(k).to_pylist() for k in keys]
        files.extend({"image_path": p, "short_prompt": s, "long_prompt": l} for p, s, l in zip(*cols))
    return files


def _halve_while(pil_image, at_least):
    # box-downsample by powers of two first (what PIL's reducing_gap would do)
    while min(*pil_image.size) >= 2 * at_least:
        pil_image = pil_image.resize(tuple(x // 2 for x in pil_image.size), resample=Image.BOX)
    return pil_image


def center_crop_arr(pil_image, image_size):
    """Resize the short side to image_size (bicubic) and take the centre square."""
    pil_image = _halve_while(pil_image, image_size)
    scale = image_size / min(*pil_image.size)
    pil_image = pil_image.resize(tuple(round(x * scale) for x in pil_image.size), resample=Image.BICUBIC)
    arr = np.array(pil_image)
    y, x = (arr.shape[0] - image_size) // 2, (arr.shape[1] - image_size) // 2
    return arr[y: y + image_size, x: x + image_size]


def random_crop_arr(pil_image, image_size, min_crop_frac=0.8, max_crop_frac=1.0):
    """Resize the short side to a random size in [image_size/max_frac, image_size/min_frac], crop a random square."""
    short = random.randrange(math.ceil(image_size / max_crop_frac), math.ceil(image_size / min_crop_frac) + 1)
    pil_image = _halve_while(pil_image, short)
    scale = short / min(*pil_image.size)
    pil_image = pil_image.resize(tuple(round(x * scale) for x in pil_image.size), resample=Image.BICUBIC)
    arr = np.array(pil_image)
    y = random.randrange(arr.shape[0] - image_size + 1)
    x = random.randrange(arr.shape[1] - image_size + 1)
    return arr[y: y + image_size, x: x + image_size]


def augment(imgs, hflip=True, rotation=True, flows=None, return_status=False):
    """The same random horizontal flip, vertical flip and transpose (rotation) applied to every HWC array.
    Draws random.random() three times, in that order, each only when the option is on."""
    hflip = hflip and random.random() < 0.5
    vflip = rotation and random.random() < 0.5
    rot90 = rotation and random.random() < 0.5

    def one(img, flow=False):
        if hflip:
            img = np.ascontiguousarray(img[:, ::-1])
            if flow:
                img[:, :, 0] *= -1
        if vflip:
            img = np.ascontiguousarray(img[::-1])
            if flow:
                img[:, :, 1] *= -1
        if rot90:
            img = img.transpose(1, 0, 2)
            if flow:
                img = img[:, :, [1, 0]]
        return img

    single = not isinstance(imgs, list)
    out = [one(i) for i in ([imgs] if single else imgs)]
    out = out[0] if len(out) == 1 else out
    if flows is not None:
        fl = [one(f, True) for f in (flows if isinstance(flows, list) else [flows])]
        return out, (fl[0] if len(fl) == 1 else fl)
    return (out, (hflip, vflip, rot90)) if return_status else out


def filter2D(img, kernel):
    """cv2.filter2D-style correlation of a [b, c, h, w] batch with reflect padding; kernel [b, k, k] (one per
    sample) or [1, k, k] (one for the batch), k odd. Runs `dbir_filter2d`."""
    from .. import lib
    require_cuda(img, "filter2D")
    k = kernel.size(-1)
    if k % 2 != 1:
        raise ValueError("Wrong kernel size")
    b = img.size(0)
    kernel = kernel.to(device=img.device, dtype=torch.float32).reshape(-1, k, k).contiguous()
    if kernel.size(0) not in (1, b):
        raise ValueError(f"expected 1 or {b} kernels, got {kernel.size(0)}")
    img = img.float().contiguous()
    out = torch.empty_like(img)
    lib.filter2d(img, kernel, out)
    return out


class USMSharp(torch.nn.Module):
    """Unsharp masking: blend towards img + weight * (img - blur) where the residual exceeds threshold/255,
    with a soft mask; the blur is a radius x radius Gaussian (cv2.getGaussianKernel(radius, sigma) outer product)."""

    def __init__(self, radius=50, sigma=0):
        super().__init__()
        import cv2
        if radius % 2 == 0:
            radius += 1
        self.radius = radius
        g = cv2.getGaussianKernel(radius, sigma)
        self.register_buffer("kernel", torch.FloatTensor(np.dot(g, g.transpose())).unsqueeze_(0))

    def forward(self, img, weight=0.5, threshold=10):
        from .. import lib
        require_cuda(img, "USMSharp")
        img = img.float().contiguous()
        kernel = self.kernel.to(img.device)
        blur, soft, out = torch.empty_like(img), torch.empty_like(img), torch.empty_like(img)
        lib.filter2d(img, kernel, blur)
        lib.filter2d(img, kernel, soft, sub=blur, threshold=threshold)
        lib.usm_blend(img, blur, soft, weight, out)
        return out
