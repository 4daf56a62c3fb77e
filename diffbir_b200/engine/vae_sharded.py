"""AutoencoderKL encode / decode sharded over torch.distributed ranks by image rows (SURVEY §8f-1).

At 2048^2 the un-tiled VAE (encode 26 + decode 48 TFLOP) is the serial remainder of the 8-GPU tiled run:
every rank would redo it while the sampler loop shrinks with 1/N. Here each rank owns a horizontal band of
every activation and the result equals the un-sharded engine's (the reference's un-tiled semantics:
`AutoencoderKL.encode/decode`, vae.py:526-582 — NOT the approximate per-tile GroupNorm of utils/tilevae).

The network is stated once, in `vae.VaeWalk`; `ShardedVae` drives that walk over this rank's band, and
`BandWalk` overrides the few steps where a band differs from a whole image:

* **3x3 convolutions**: a band carries one halo row above and below ([n, hb + 2, W, C]); the rows a conv
  needs from the neighbours are exchanged on its 16-bit input (one small all-gather of the two edge rows
  per conv; image borders get zeros = the conv's zero padding). The conv runs over the whole band with the
  ordinary implicit-GEMM kernel; its outermost output rows are meaningless and never used.
* **GroupNorm**: per-rank (mean, variance) of the band's own rows, all-gathered and merged exactly
  (equal counts: mean of means, mean of variances + variance of means) — the statistics of the FULL image.
* **mid-block attention** (single head over all pixels, vae.py:232-282): queries stay local, the normalised
  input of all ranks is all-gathered once to form K and V.
* **stride-2 / nearest-2x resampling** keep the band structure (halo rows re-derived by the next exchange).

All ranks must hold the same input (they do: the pipeline's stage 1 and sampler are deterministic and
replicated / bit-identical) and all ranks return the full result (final all-gather of the bands).
Eager launches (NCCL calls between kernels), a few hundred per call: the price is ~4 ms of launch latency
against 130 + 90 ms of replicated encode + decode at 2048^2.
"""
from __future__ import annotations

import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import lib
from .common import Workspace
from .vae import VaeEngine, VaeWalk
from .vae_tiled import ProcessGroupGather


class BandWalk(VaeWalk):
    """The walk on this rank's band of every image: fp32 NHWC [nb, hb + 2, w, C], this rank's hb rows with one halo
    row above and below, so that the walk's h is hb + 2."""

    gn_partials = False         # a conv's partial sums would cover the halo rows

    def __init__(self, eng: VaeEngine, ws: Workspace, nb: int, rank: int, world: int, comm):
        super().__init__(eng, ws, nb)
        self.rank, self.world, self.comm = rank, world, comm

    def _exchange(self, band: torch.Tensor) -> None:
        """band [n, hb + 2, W, C] (any dtype): fills the halo rows 0 and hb + 1 with the neighbours' edge rows
        (zeros at the image border: the convolution's padding)."""
        edges = torch.stack([band[:, 1], band[:, -2]], 1)                   # [n, 2, W, C]: first / last own row
        allr = self.comm.all_gather(edges)                                   # [R, n, 2, W, C]
        if self.rank > 0:
            band[:, 0] = allr[self.rank - 1, :, 1]
        else:
            band[:, 0].zero_()
        if self.rank < self.world - 1:
            band[:, -1] = allr[self.rank + 1, :, 0]
        else:
            band[:, -1].zero_()

    def _halo(self, a16, h, w, c) -> None:
        self._exchange(a16.view(self.nb, h, w, c))

    def _down(self, key, c, h, w):
        """Output row r reads input rows 2r..2r+2: this rank's own rows plus ONE row of the lower neighbour (zeros
        at the image bottom). The result fills the new band's own rows; its halo rows wait for the next exchange."""
        n, hb, ws = self.nb, h - 2, self.ws
        xb = self.st["cur"].view(n, h, w, c)
        self._exchange(xb)
        src = xb[:, 1:].contiguous()                                      # [n, hb + 1, w, c]
        ho, wo = hb // 2, w // 2
        col = ws.get("col16", (n * ho * wo, 9 * c), self.op_dtype)
        lib.im2col_s2(src, n, hb + 1, w, c, 0, col)
        tmp = ws.get("down_tmp", (n, ho, wo, c), torch.float32)
        lib.gemm(col, self.w[key + ".weight"], tmp, M=n * ho * wo, N=c, K=9 * c, bias=self.w[key + ".bias"])
        self.st["cur"] = self.new(n * (ho + 2) * wo, c)
        self.st["cur"].view(n, ho + 2, wo, c)[:, 1:-1] = tmp
        return ho + 2, wo

    def _up(self, c, h, w):
        """The upsampled band's own 2 hb rows and one halo row each side, which the conv's exchange fills."""
        n, hb = self.nb, h - 2
        up_all = self.ws.get("up_all", (n, 2 * hb + 4, 2 * w, c), self.op_dtype)
        lib.gn_apply(self.st["cur"], None, c, 0, n, h, w, None, None, None, up_all, norm=False, silu=False, upsample=2)
        up16 = self.ws.get("a16", (n, 2 * hb + 2, 2 * w, c), self.op_dtype)
        up16.copy_(up_all[:, 1:-1])
        return up16, 2 * hb + 2, 2 * w

    def _attend(self, p, a16, x, c, h, w):
        """Local queries, keys / values of all ranks; proj_out per image on the band's own rows."""
        ws, W, n = self.ws, self.w, self.nb
        lw = (h - 2) * w
        hw = self.world * lw
        own = a16.view(n, h, w, c)[:, 1:-1].contiguous()                 # [n, hb, w, c]
        full = self.comm.all_gather(own).permute(1, 0, 2, 3, 4).reshape(n * hw, c).contiguous()   # global row order
        qk = ws.get("qk16", (n * hw, 2 * c), self.op_dtype)
        lib.gemm(full, W[p + "qk.w"], qk, M=n * hw, N=2 * c, K=c, bias=W[p + "qk.b"])
        o16 = ws.get("o16", (n * lw, c), self.op_dtype)
        self._softmax_av(p, qk, full, o16, c, hw, self.rank * lw, lw)
        xb = x.view(n, h, w, c)
        for b in range(n):
            xi = xb[b, 1:-1].reshape(lw, c)                                # contiguous interior of image b
            lib.gemm(o16[b * lw:(b + 1) * lw], W[p + "proj_out.weight"], xi, M=lw, N=c, K=c,
                     bias=W[p + "proj_out.bias"], residual=xi)


class ShardedVae:
    def __init__(self, base: VaeEngine, rank: int = None, world: int = None, comm=None):
        """Rank `rank` of `world` cooperating ranks (default: the torch.distributed ones) that all call with the same
        input; `comm.all_gather` (default: `ProcessGroupGather`) carries every exchange between them."""
        self.base, self.w, self.dev = base, base.w, base.dev
        self.ws = Workspace(self.dev)
        self.rank = dist.get_rank() if rank is None else rank
        self.world = dist.get_world_size() if world is None else world
        self.comm = ProcessGroupGather() if comm is None else comm

    # ------------------------------------------------------------------ applicability
    @staticmethod
    def usable(h_img: int, w_img: int) -> bool:
        """Bands of whole latent rows (>= 2 per rank) at every resolution level, widths the GEMM's GroupNorm-free
        conv path takes (any), and an initialised process group of more than one rank."""
        if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() < 2:
            return False
        world = dist.get_world_size()
        return h_img % (8 * world) == 0 and h_img // (8 * world) >= 2 and w_img % 8 == 0

    # ------------------------------------------------------------------ the driver
    def _gn_stats(self, x: torch.Tensor, n: int, c: int, eps: float) -> torch.Tensor:
        """x fp32 [n, hb + 2, W, c] -> (mean, rstd) of the FULL image per (image, group): stats [n*32*2]."""
        cpg = c // 32
        own = x.view(n, x.shape[1], x.shape[2], 32, cpg)[:, 1:-1]            # this rank's rows (strided view, no copy)
        var, mean = torch.var_mean(own, dim=(1, 2, 4), unbiased=False)       # [n, 32] each
        both = self.comm.all_gather(torch.stack([mean, var], -1).double())   # [R, n, 32, 2]
        gmean = both[..., 0].mean(0)
        gvar = both[..., 1].mean(0) + (both[..., 0] - gmean).pow(2).mean(0)  # equal counts per rank
        return torch.stack([gmean, (gvar + eps).rsqrt()], -1).float().reshape(-1).contiguous()

    def _run(self, net, x: torch.Tensor) -> torch.Tensor:
        """x fp32 NCHW: the whole input -> `net` (VaeWalk.encoder / .decoder) on this rank's band of its rows."""
        n, hb = x.shape[0], x.shape[2] // self.world
        band = F.pad(x, (0, 0, 1, 1))[:, :, self.rank * hb: self.rank * hb + hb + 2].contiguous()   # zero outside
        walk = BandWalk(self.base, self.ws, n, self.rank, self.world, self.comm)

        def answer(c, h, w, part, slots):                                   # no partial sums on a band
            return self._gn_stats(walk.st["cur"].view(n, h, w, c), n, c, 1e-6)
        return walk.run(net, band, answer)

    def _new(self, *shape) -> torch.Tensor:
        return torch.empty(*shape, dtype=torch.float32, device=self.dev)

    @torch.no_grad()
    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """z fp32 NCHW [n, 4, h, w] (already divided by the scale factor; identical on every rank) -> image fp32
        NCHW [n, 3, 8h, 8w] on every rank."""
        band = self._run(VaeWalk.decoder, self.base.post_quant(z, self._new))   # post_quant_conv on the whole latent
        n, oc, _, w = band.shape
        allb = self.comm.all_gather(band[:, :, 1:-1].contiguous())           # [R, n, 3, hb, w]
        return allb.permute(1, 2, 0, 3, 4).reshape(n, oc, -1, w).contiguous()

    @torch.no_grad()
    def encode_moments(self, img: torch.Tensor) -> torch.Tensor:
        """img fp32 NCHW [n, 3, H, W] in [-1, 1] (identical on every rank) -> moments fp32 NCHW [n, 8, H/8, W/8]."""
        m = self._run(VaeWalk.encoder, img)                                  # NHWC [n, hb + 2, w, 8]
        n, hb2, w, zc2 = m.shape
        q = torch.empty_like(m)
        lib.linear_f32(m, zc2, n * hb2 * w, zc2, self.w["quant_conv.weight"], self.w["quant_conv.bias"], zc2, q, zc2)
        allq = self.comm.all_gather(q[:, 1:-1].contiguous())                 # [R, n, hb, w, 8]
        return allq.permute(1, 4, 0, 2, 3).reshape(n, zc2, -1, w).contiguous()
