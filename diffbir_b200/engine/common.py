"""Shared engine plumbing: named workspace buffers, checkpoint checks, weight packing helpers and the pre-norm
transformer block."""
from __future__ import annotations

from typing import Callable, Dict, Tuple

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

    def clear(self) -> None:
        """Drops every buffer (graphs that hold their pointers must be dropped with them)."""
        if self.on_grow is not None:
            self.on_grow()
        self._bufs.clear()


class GraphCache:
    """CUDA graphs of a fixed-shape function of device tensors, one per key (input shapes).
    First call per key: one eager run (sizes the workspace, lets dbir_gemm tune its plans -- it cannot
    time inside a capture), then capture; later calls copy the inputs into the static buffers and
    replay. Outputs live in the graph's memory pool and are overwritten by the next replay of the
    same graph, so a copy is returned. Graphs hold raw workspace pointers: `clear` is hooked to
    Workspace.on_grow."""

    def __init__(self, ws: "Workspace" = None):
        self._g = {}
        if ws is not None:
            ws.on_grow = self._g.clear

    def clear(self):
        self._g.clear()

    def run(self, key, fn, *inputs: torch.Tensor):
        if torch.cuda.is_current_stream_capturing():
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


def round_up(n: int, m: int = 64) -> int:
    return (n + m - 1) // m * m


def check_shapes(sd: Dict[str, torch.Tensor], shapes, what: str) -> None:
    """Every key of `shapes` is in the checkpoint `sd` with that shape (other keys are ignored)."""
    for k, shp in shapes.items():
        if k not in sd:
            raise KeyError(f"{what} checkpoint is missing {k}")
        if tuple(sd[k].shape) != tuple(shp):
            raise ValueError(f"{k}: {tuple(sd[k].shape)} != {shp}")


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


def pack_gathered(w: torch.Tensor, device, n_pad: int = 0) -> torch.Tensor:
    """[Cout, Cin, kh, kw] -> op16 [Cout', K] for a GEMM on dbir_patch_gather's patches: k = tap*Cin + c, K zero-padded
    to a multiple of 64, rows zero-padded to n_pad."""
    co = w.shape[0]
    flat = w.permute(0, 2, 3, 1).reshape(co, -1)
    return op16(torch.nn.functional.pad(flat, (0, round_up(flat.shape[1]) - flat.shape[1], 0, max(0, n_pad - co))),
                device)


def pack_swin_block(w: Dict[str, torch.Tensor], dst: str, sd: Dict[str, torch.Tensor], src: str, device,
                    k_pad: int = 0, hid_pad: int = 0) -> None:
    """Swin block `src` of a checkpoint (norm1, attn.qkv, attn.proj, attn.relative_position_bias_table, norm2,
    mlp.fc1, mlp.fc2) -> w[dst + prenorm_block's names] and w[dst + "rpb"]. GEMM K is zero-padded to k_pad, fc2's to
    hid_pad."""
    for i in (1, 2):
        w[f"{dst}ln{i}.w"] = f32(sd[f"{src}norm{i}.weight"], device)
        w[f"{dst}ln{i}.b"] = f32(sd[f"{src}norm{i}.bias"], device)
    for nm, key, kp in (("qkv", "attn.qkv", k_pad), ("proj", "attn.proj", k_pad), ("fc1", "mlp.fc1", k_pad),
                        ("fc2", "mlp.fc2", hid_pad)):
        w[dst + nm + ".w"] = pack_linear(sd[src + key + ".weight"], device, kp)
        w[dst + nm + ".b"] = f32(sd[src + key + ".bias"], device)
    w[dst + "rpb"] = f32(sd[src + "attn.relative_position_bias_table"], device)


def prenorm_block(W: Dict[str, torch.Tensor], p: str, t: torch.Tensor, bufs, M: int, c: int, hidden: int, lds,
                  act: str, eps: float, attend: Callable[[torch.Tensor, torch.Tensor], None]) -> None:
    """One pre-norm transformer block in place on the fp32 token stream t [M, c] (row stride lds[0]):
    t += proj(attention(qkv(LN1(t)))), then t += fc2(act(fc1(LN2(t)))).
    bufs = (ln16, qkv16, att16, hid16): op16 work buffers. lds = row strides of (t / ln16 / att16, qkv16, hid16);
    each is also the K of the GEMM that reads that buffer (weights zero-padded to it). attend(qkv16, att16) enqueues
    the attention. Weights: W[p + "ln1.w" / "ln1.b" / "qkv.w" / "qkv.b" / "proj.*" / "ln2.*" / "fc1.*" / "fc2.*"]."""
    ln16, qkv, att, hid = bufs
    ldt, ldqkv, ldh = lds
    lib.layernorm(t, ldt, M, c, W[p + "ln1.w"], W[p + "ln1.b"], ln16, ldt, eps=eps)
    lib.gemm(ln16, W[p + "qkv.w"], qkv, M=M, N=3 * c, K=ldt, bias=W[p + "qkv.b"], ldo=ldqkv)
    attend(qkv, att)
    lib.gemm(att, W[p + "proj.w"], t, M=M, N=c, K=ldt, bias=W[p + "proj.b"], residual=t, ldo=ldt, ldr=ldt)
    lib.layernorm(t, ldt, M, c, W[p + "ln2.w"], W[p + "ln2.b"], ln16, ldt, eps=eps)
    lib.gemm(ln16, W[p + "fc1.w"], hid, M=M, N=hidden, K=ldt, bias=W[p + "fc1.b"], act=act, ldo=ldh)
    lib.gemm(hid, W[p + "fc2.w"], t, M=M, N=c, K=ldh, bias=W[p + "fc2.b"], residual=t, ldo=ldt, ldr=ldt)


def geglu_tile(c: int) -> int:
    """GEMM tile width used for the GEGLU projection of a width-c transformer block (the weights are packed
    per tile as [values | gates], so it is fixed at load time)."""
    # 256-wide tiles (128 values + 128 gates): at large batch the projection is bound by L2 -> SM operand
    # traffic, which a 256-wide tile (and a CTA pair sharing it) cuts against 128-wide ones.
    for bn in (256, 128, 64):
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
