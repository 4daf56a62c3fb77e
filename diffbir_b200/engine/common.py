"""Shared engine plumbing: named workspace buffers and weight packing helpers."""
from __future__ import annotations

import os

from typing import Dict, Tuple

import torch

from .. import lib


class Workspace:
    """Named, grow-only device buffers. After one warm-up pass nothing is (re)allocated, which
    is what CUDA-graph capture needs (the C ABI never allocates)."""

    def __init__(self, device):
        self.device = device
        self._bufs: Dict[str, torch.Tensor] = {}
        self.on_grow = None      # called before a buffer is (re)allocated: captured graphs hold raw pointers

    def get(self, tag: str, shape, dtype, zero: bool = False) -> torch.Tensor:
        n = 1
        for s in shape:
            n *= int(s)
        key = f"{tag}:{dtype}"
        buf = self._bufs.get(key)
        if buf is None or buf.numel() < n:
            if torch.cuda.is_current_stream_capturing():
                raise RuntimeError(f"workspace buffer '{tag}' would be allocated during graph capture")
            if self.on_grow is not None:
                self.on_grow()
            buf = (torch.zeros if zero else torch.empty)(max(n, 1), dtype=dtype, device=self.device)
            self._bufs[key] = buf
        return buf[:n].view(*shape)

    def bytes(self) -> int:
        return sum(b.numel() * b.element_size() for b in self._bufs.values())


class GraphCache:
    """CUDA graphs of a fixed-shape function of device tensors, one per key (input shapes).
    First call per key: one eager run (sizes the workspace, lets dbir_gemm tune its plans -- it cannot
    time inside a capture), then capture; later calls copy the inputs into the static buffers and
    replay. Outputs live in the graph's memory pool and are overwritten by the next replay of the
    same graph, so a copy is returned. Graphs hold raw workspace pointers: `clear` is hooked to
    Workspace.on_grow."""

    def __init__(self, ws: "Workspace" = None):
        self._g = {}
        self.enabled = True
        if ws is not None:
            ws.on_grow = self._g.clear

    def clear(self):
        self._g.clear()

    def run(self, key, fn, *inputs: torch.Tensor):
        if not self.enabled or torch.cuda.is_current_stream_capturing():
            return fn(*inputs)
        hit = self._g.get(key)
        if hit is None:
            static_in = [t.clone() for t in inputs]
            fn(*static_in)                                   # eager warm-up (may grow the workspace -> clears the cache)
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            n0 = lib.launches()
            with torch.cuda.graph(graph):
                out = fn(*static_in)
            n = lib.launches() - n0
            lib.count_launch(-n)                             # capture executes nothing
            hit = (graph, static_in, out, n)
            self._g[key] = hit
        graph, static_in, out, n = hit
        for s, t in zip(static_in, inputs):
            s.copy_(t)
        graph.replay()
        lib.count_launch(n)
        return out.clone()


def op16(t: torch.Tensor, device) -> torch.Tensor:
    return t.to(device=device, dtype=lib.operand_dtype()).contiguous()


def f32(t: torch.Tensor, device) -> torch.Tensor:
    return t.to(device=device, dtype=torch.float32).contiguous()


def pack_conv3x3(w: torch.Tensor, device, cin_pad: int = 0) -> torch.Tensor:
    """[Cout, Cin, kh, kw] -> op16 [Cout, kh*kw*Cin'] with k = tap*Cin' + c (Cin zero-padded)."""
    co, ci, kh, kw = w.shape
    w = w.permute(0, 2, 3, 1)
    if cin_pad and cin_pad > ci:
        w = torch.nn.functional.pad(w, (0, cin_pad - ci))
        ci = cin_pad
    return op16(w.reshape(co, kh * kw * ci), device)


def pack_linear(w: torch.Tensor, device, k_pad: int = 0) -> torch.Tensor:
    if w.dim() == 4:
        w = w.reshape(w.shape[0], w.shape[1])
    if k_pad and k_pad > w.shape[1]:
        w = torch.nn.functional.pad(w, (0, k_pad - w.shape[1]))
    return op16(w, device)


def geglu_tile(c: int) -> int:
    """GEMM tile width used for the GEGLU projection of a width-c transformer block (the weights are packed
    per tile as [values | gates], so it is fixed at load time)."""
    # 256-wide tiles (128 values + 128 gates): at large batch the projection is bound by L2 -> SM operand
    # traffic, which a 256-wide tile (and a CTA pair sharing it) cuts against 128-wide ones. DBIR_GEGLU_TILE overrides.
    forced = int(os.environ.get("DBIR_GEGLU_TILE", "0"))       # A/B switch: 64 | 128 | 256
    for bn in ((forced,) if forced else ()) + (256, 128, 64):
        if (8 * c) % bn == 0:
            return bn
    return 64


def pack_geglu(w: torch.Tensor, b: torch.Tensor, bn: int, device) -> Tuple[torch.Tensor, torch.Tensor]:
    """Interleave value / gate rows per bn-row tile: tile j = [values j*hb.. | gates j*hb..]."""
    inner = w.shape[0] // 2
    hb = bn // 2
    assert inner % hb == 0
    wv, wg = w[:inner].view(inner // hb, hb, -1), w[inner:].view(inner // hb, hb, -1)
    wp = torch.cat([wv, wg], dim=1).reshape(2 * inner, -1)
    bv, bg = b[:inner].view(inner // hb, hb), b[inner:].view(inner // hb, hb)
    bp = torch.cat([bv, bg], dim=1).reshape(2 * inner)
    return op16(wp, device), f32(bp, device)
