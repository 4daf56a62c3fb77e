"""Batched JPEG round trip (reference dataset/diffjpeg.py) on the engine: `dbir_diffjpeg`, one kernel."""
from __future__ import annotations

import torch
from torch import nn

from ._device import require_cuda


def quality_to_factor(quality):
    """JPEG quality -> scale of the standard quantisation tables."""
    q = 5000.0 / quality if quality < 50 else 200.0 - quality * 2
    return q / 100.0


class DiffJPEG(nn.Module):
    """Compress and decompress a batch with the standard tables scaled per sample (4:2:0 chroma, 16-pixel
    zero padding, rounding half to even). Only the non-differentiable rounding is built: the batch
    transform uses `differentiable=False`, and the engine has no backward pass."""

    def __init__(self, differentiable=True):
        super().__init__()
        if differentiable:
            raise NotImplementedError("DiffJPEG(differentiable=True) needs a backward pass, which the engine does "
                                      "not build; use differentiable=False")

    def forward(self, x, quality, clamp=False):
        """x: [b, 3, h, w] RGB in [0, 1] on CUDA; quality: a number or a [b] tensor. clamp=True clamps x to
        [0, 1] first (what the batch transform does before every JPEG step)."""
        from .. import lib
        require_cuda(x, "DiffJPEG")
        if x.dim() != 4 or x.shape[1] != 3 or x.dtype != torch.float32:
            raise ValueError("DiffJPEG expects a float32 [b, 3, h, w] batch")
        x = x.contiguous()
        b = x.shape[0]
        out = torch.empty_like(x)
        if isinstance(quality, (int, float)):
            # a number: the factor is computed in double on the host and the tables scaled by its fp32 value
            factor = torch.full((b,), quality_to_factor(quality), dtype=torch.float32, device=x.device)
            lib.diffjpeg(x, factor, out, clamp_in=clamp, is_factor=True)
        else:
            # a tensor: the factor is computed per sample on the device, in PyTorch's fp32 op order
            quality = quality.to(device=x.device, dtype=torch.float32).reshape(b).contiguous()
            lib.diffjpeg(x, quality, out, clamp_in=clamp)
        return out
