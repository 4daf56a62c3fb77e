"""Pipeline / SwinIRPipeline — drop-in counterparts of the reference's diffbir.pipeline
(pipeline.py:43-321, 369-397): same constructor, same 26-argument `run`, uint8 NHWC in/out.
The orchestration (resize, pads, crops, colour fix, quantisation) is the reference's, the
networks are the kernel engines behind diffbir_b200.model.{SwinIR, ControlLDM}.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
import torch.nn.functional as F

from . import lib
from .model import ControlLDM, Diffusion
from .sampler import DDIMSampler, DPMSolverSampler, EDMSampler, SpacedSampler
from .sampler.sampler import NoiseSource, randn, randn_like, tiled_run_chunked
from .utils.common import make_tiled_fn, sliding_windows, wavelet_reconstruction


def resize_short_edge_to(imgs: torch.Tensor, size: int) -> torch.Tensor:
    _, _, h, w = imgs.size()
    if h == w:
        out_h, out_w = size, size
    elif h < w:
        out_h, out_w = size, int(w * (size / h))
    else:
        out_h, out_w = int(h * (size / w)), size
    return F.interpolate(imgs, size=(out_h, out_w), mode="bicubic", antialias=True)


def pad_to_multiples_of(imgs: torch.Tensor, multiple: int) -> torch.Tensor:
    _, _, h, w = imgs.size()
    if h % multiple == 0 and w % multiple == 0:
        return imgs.clone()
    ph, pw = map(lambda x: (x + multiple - 1) // multiple * multiple - x, (h, w))
    return F.pad(imgs, pad=(0, pw, 0, ph), mode="constant", value=0)


def vae_tiling(img_hw, enc_tiled: bool, enc_tile: int, dec_tiled: bool, dec_tile: int) -> Tuple[bool, bool]:
    """Whether the VAE encode / decode of an (already padded) condition image of size img_hw run tiled
    (pipeline.py:105-115, 219-224): off for inputs smaller than a tile; an encoder tile size that is not a
    multiple of 8 is refused."""
    h, w = img_hw
    if enc_tiled and (h < enc_tile or w < enc_tile):
        print("[VAE Encoder]: the input size is tiny and unnecessary to tile.")
        enc_tiled = False
    if enc_tiled and enc_tile % 8 != 0:
        raise ValueError("VAE encoder tile size must be a multiple of 8")
    if dec_tiled and (h // 8 < dec_tile // 8 or w // 8 < dec_tile // 8):
        print("[VAE Decoder]: the input size is tiny and unnecessary to tile.")
        dec_tiled = False
    return enc_tiled, dec_tiled


class Pipeline:
    def __init__(self, cleaner, cldm: ControlLDM, diffusion: Diffusion, cond_fn, device: str) -> None:
        self.cleaner = cleaner
        self.cldm = cldm
        self.diffusion = diffusion
        self.cond_fn = cond_fn          # restoration guidance: dead code in the reference (SURVEY §2 #18)
        self.device = device
        self.output_size: Tuple[int, int] = None
        self.taps: Optional[dict] = None   # set to {} to capture intermediates (tests)
        self.fused_post = True             # colour fix + quantisation as one kernel (False: the torch op sequence)
        self.shard_vae = True              # cooperating ranks (tiled / batch-sharded sampling) shard the VAE (by image rows or by tiles)
        self.shard_batch = False           # un-tiled batches: shard (image, CFG branch) forwards over torch.distributed ranks
        self.shard_tiles = True            # tiled sampling: shard the tiles over torch.distributed ranks (Sampler.shard_tiles)
        self.shard_cleaner = False         # stage 1 shared by the ranks: a tiled cleaner by windows, an un-tiled one on rank 0
        self.max_tile_forwards = 128       # tiled sampling: most tile-forwards x images per graph replay (Sampler.max_tile_forwards)
        self.marks: Optional[list] = None  # set to [] to record (phase, CUDA event) boundaries (bench.py phases_ms)

    def _mark(self, name: str) -> None:
        if self.marks is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.marks.append((name, ev))

    def phases_ms(self) -> dict:
        """Milliseconds between consecutive marks of the last run (call after a synchronize)."""
        m = self.marks or []
        out = {}
        for (_, e0), (name, e1) in zip(m[:-1], m[1:]):
            out[name] = out.get(name, 0.0) + e0.elapsed_time(e1)
        return out

    def set_output_size(self, lq_size: Tuple[int]) -> None:
        h, w = lq_size[2:]
        self.output_size = (h, w)

    def apply_cleaner(self, lq, tiled, tile_size, tile_stride):
        raise NotImplementedError

    @torch.no_grad()
    def apply_cldm(self, cond_img, steps, strength, vae_encoder_tiled, vae_encoder_tile_size,
                   vae_decoder_tiled, vae_decoder_tile_size, cldm_tiled, cldm_tile_size,
                   cldm_tile_stride, pos_prompt, neg_prompt, cfg_scale, start_point_type,
                   sampler_type, noise_aug, rescale_cfg, s_churn, s_tmin, s_tmax, s_noise, eta,
                   order, x_T: Optional[torch.Tensor] = None, seeds: Optional[Sequence[int]] = None) -> torch.Tensor:
        """pipeline.py:71-233. pos_prompt: one prompt for every image, or one per image. seeds: one per image; image k
        then draws its noise from its own generators seeded seeds[k] (NoiseSource) instead of the global ones."""
        bs, _, h0, w0 = cond_img.shape
        source = None
        if seeds is not None:
            if len(seeds) != bs:
                raise ValueError(f"{len(seeds)} seeds for {bs} images")
            source = NoiseSource(seeds, self.device)
        if isinstance(pos_prompt, str):
            pos_prompts = [pos_prompt] * bs
        else:
            pos_prompts = list(pos_prompt)
            if len(pos_prompts) != bs:
                raise ValueError(f"{len(pos_prompts)} positive prompts for {bs} images")
        cond_img = pad_to_multiples_of(cond_img, multiple=64 if not vae_encoder_tiled and not cldm_tiled else 8)
        vae_encoder_tiled, vae_decoder_tiled = vae_tiling(cond_img.shape[2:], vae_encoder_tiled, vae_encoder_tile_size,
                                                          vae_decoder_tiled, vae_decoder_tile_size)
        # ranks that cooperate on this job (sharded tiles or batch units) also shard the VAE: the un-tiled one by
        # image rows, the tiled one by tiles (ControlLDM)
        import torch.distributed as dist
        coop = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1 and (
            (cldm_tiled and self.shard_tiles) or self.shard_batch)
        self.cldm.shard_vae = bool(coop and self.shard_vae)
        # The reference encodes the (identical) condition image twice (pipeline.py:117-128);
        # the latent is deterministic (posterior mode), so it is encoded once and shared.
        # Both prompts go through the text tower as one batch (pipeline.py:117-128 runs it twice).
        enc_tiling = dict(tiled=True, tile_size=vae_encoder_tile_size) if vae_encoder_tiled else {}
        if isinstance(pos_prompt, str):
            cond, uncond = self.cldm.prepare_condition_pair(cond_img, pos_prompts, [neg_prompt] * bs, **enc_tiling)
        else:       # image i's text rows as its run alone computes them, whatever else shares the call
            cond, uncond = self.cldm.prepare_condition_pairs(cond_img, pos_prompts, neg_prompt, **enc_tiling)
        self._mark("encode+clip")
        h1, w1 = cond["c_img"].shape[2:]
        if cldm_tiled and (h1 < cldm_tile_size // 8 or w1 < cldm_tile_size // 8):
            print("[Diffusion]: the input size is tiny and unnecessary to tile.")
            cldm_tiled = False
        if not cldm_tiled:
            cond["c_img"] = pad_to_multiples_of(cond["c_img"], multiple=8)
            uncond["c_img"] = pad_to_multiples_of(uncond["c_img"], multiple=8)
        elif cldm_tile_size % 64 != 0:
            raise ValueError("Diffusion tile size must be a multiple of 64")
        h2, w2 = cond["c_img"].shape[2:]
        if x_T is None:
            if start_point_type == "cond":
                x_T = self.diffusion.q_sample(
                    cond["c_img"],
                    torch.full((bs,), self.diffusion.num_timesteps - 1, dtype=torch.long, device=self.device),
                    randn(cond["c_img"].shape, self.device, source))
            else:
                x_T = randn((bs, 4, h2, w2), self.device, source)
        if noise_aug > 0:
            cond["c_img"] = self.diffusion.q_sample(
                x_start=cond["c_img"], t=torch.full(size=(bs,), fill_value=noise_aug, device=self.device),
                noise=randn_like(cond["c_img"], source))
            uncond["c_img"] = cond["c_img"].detach().clone()
        control_scales = self.cldm.control_scales
        self.cldm.control_scales = [strength] * 13
        betas, parameterization = self.diffusion.betas, self.diffusion.parameterization
        if sampler_type == "spaced":
            sampler = SpacedSampler(betas, parameterization, rescale_cfg)
        elif sampler_type == "ddim":
            sampler = DDIMSampler(betas, parameterization, rescale_cfg, eta=0)
        elif sampler_type.startswith("dpm"):
            sampler = DPMSolverSampler(betas, parameterization, rescale_cfg, sampler_type)
        elif sampler_type.startswith("edm"):
            sampler = EDMSampler(betas, parameterization, rescale_cfg, sampler_type, s_churn, s_tmin, s_tmax, s_noise, eta, order)
        else:
            raise NotImplementedError(sampler_type)
        sampler.shard_batch = self.shard_batch
        sampler.shard_tiles = self.shard_tiles
        sampler.max_tile_forwards = self.max_tile_forwards
        sampler.noise_source = source
        if cldm_tiled and tiled_run_chunked(len(sliding_windows(h2, w2, cldm_tile_size // 8, cldm_tile_stride // 8)),
                                            1 if cfg_scale == 1.0 else 2, bs, self.max_tile_forwards,
                                            sampler.shard_tiles):
            # an image too large for one replay: the encoder's full-resolution buffers are not needed again
            # before the decode, so the sampler's activations get their memory
            self.cldm.release_vae_buffers()
        z = sampler.sample(model=self.cldm, device=self.device, steps=steps, x_size=(bs, 4, h2, w2),
                           cond=cond, uncond=uncond, cfg_scale=cfg_scale, tiled=cldm_tiled,
                           tile_size=cldm_tile_size // 8, tile_stride=cldm_tile_stride // 8, x_T=x_T,
                           progress=True)
        self.last_sampler = sampler
        self._mark("sampler_loop")
        if sampler.last_stats.get("chunks", 1) > 1 or vae_decoder_tiled:
            # only images too large for one replay (or for the un-tiled decode) get here: hand the sampler's
            # activations back so that the full-resolution decode fits beside them -- a tiled decode keeps as much
            # of its state on the device as half the free memory allows; smaller runs keep their buffers and
            # graphs across calls
            self.cldm.release_engine_buffers()
        z = z[..., :h1, :w1].contiguous()
        dec_tiling = dict(tiled=True, tile_size=vae_decoder_tile_size // 8) if vae_decoder_tiled else {}
        x = self.cldm.vae_decode(z, **dec_tiling)
        self.cldm.shard_vae = False
        self._mark("vae_decode")
        x = x[:, :, :h0, :w0]
        self.cldm.control_scales = control_scales
        if self.taps is not None:
            self.taps.update(z=z, decoded=x, cond=cond, uncond=uncond)
        return x

    @torch.no_grad()
    def run(self, lq: np.ndarray, steps: int, strength: float, cleaner_tiled: bool,
            cleaner_tile_size: int, cleaner_tile_stride: int, vae_encoder_tiled: bool,
            vae_encoder_tile_size: int, vae_decoder_tiled: bool, vae_decoder_tile_size: int,
            cldm_tiled: bool, cldm_tile_size: int, cldm_tile_stride: int, pos_prompt: Union[str, List[str]],
            neg_prompt: str, cfg_scale: float, start_point_type: str, sampler_type: str,
            noise_aug: int, rescale_cfg: bool, s_churn: float, s_tmin: float, s_tmax: float,
            s_noise: float, eta: float, order: int, x_T: Optional[torch.Tensor] = None,
            seeds: Optional[Sequence[int]] = None) -> np.ndarray:
        """pipeline.py:235-321: uint8 [B,H,W,3] (numpy or pinned CPU tensor) -> uint8 numpy.

        pos_prompt: a str for every image (the reference's meaning) or a list of B prompts, one per image.
        seeds: one per image; every random draw of image k then comes from its own generators seeded seeds[k], in the
        order the run of that image alone makes after set_seed(seeds[k]) (sampler.NoiseSource). With the
        batch-invariant kernel plans (DBIR_DETERMINISTIC=1) image k's output is then that run's, bit for bit."""
        host = torch.from_numpy(lq) if isinstance(lq, np.ndarray) else lq
        lq_dev = host.to(self.device, non_blocking=True)                        # H2D
        out = self.run_device(lq_dev, steps, strength, cleaner_tiled, cleaner_tile_size,
                              cleaner_tile_stride, vae_encoder_tiled, vae_encoder_tile_size,
                              vae_decoder_tiled, vae_decoder_tile_size, cldm_tiled, cldm_tile_size,
                              cldm_tile_stride, pos_prompt, neg_prompt, cfg_scale, start_point_type,
                              sampler_type, noise_aug, rescale_cfg, s_churn, s_tmin, s_tmax, s_noise,
                              eta, order, x_T=x_T, seeds=seeds)
        return out.cpu().numpy()                                                # D2H

    @torch.no_grad()
    def run_device(self, lq_dev: torch.Tensor, steps, strength, cleaner_tiled, cleaner_tile_size,
                   cleaner_tile_stride, vae_encoder_tiled, vae_encoder_tile_size, vae_decoder_tiled,
                   vae_decoder_tile_size, cldm_tiled, cldm_tile_size, cldm_tile_stride, pos_prompt,
                   neg_prompt, cfg_scale, start_point_type, sampler_type, noise_aug, rescale_cfg,
                   s_churn, s_tmin, s_tmax, s_noise, eta, order, x_T=None, seeds=None) -> torch.Tensor:
        """Same as run() with the uint8 NHWC input and output resident on the device."""
        if self.marks is not None:
            self.marks.clear()
        self._mark("start")
        lq_tensor = lq_dev.to(torch.float32).div(255).clamp(0, 1).permute(0, 3, 1, 2).contiguous()
        self.set_output_size(lq_tensor.size())
        cond_img = self.shared_cleaner(lq_tensor, cleaner_tiled, cleaner_tile_size, cleaner_tile_stride)
        self._mark("swinir")
        assert all(x >= 512 for x in cond_img.shape[2:]), (
            "The resolution of stage-1 model output should be greater than 512, "
            "since it will be used as condition for stage-2 model.")
        if self.taps is not None:
            self.taps["clean"] = cond_img
        sample = self.apply_cldm(cond_img, steps, strength, vae_encoder_tiled, vae_encoder_tile_size,
                                 vae_decoder_tiled, vae_decoder_tile_size, cldm_tiled, cldm_tile_size,
                                 cldm_tile_stride, pos_prompt, neg_prompt, cfg_scale, start_point_type,
                                 sampler_type, noise_aug, rescale_cfg, s_churn, s_tmin, s_tmax, s_noise,
                                 eta, order, x_T=x_T, seeds=seeds)
        if tuple(sample.shape[2:]) == tuple(self.output_size) and sample.is_cuda and self.fused_post:
            # no resize (antialiased bicubic at scale 1 is the identity): colour fix + x255 / clamp /
            # truncate + NHWC in one kernel (dbir_wavelet_fix) instead of ~45 full-resolution passes
            out = torch.empty(sample.shape[0], sample.shape[2], sample.shape[3], 3, dtype=torch.uint8, device=sample.device)
            lib.wavelet_fix(sample.float(), cond_img.float(), out_u8=out)
        else:
            if sample.is_cuda and self.fused_post:
                fixed = torch.empty(sample.shape, dtype=torch.float32, device=sample.device)
                lib.wavelet_fix(sample.float(), cond_img.float(), out_f32=fixed)
            else:
                fixed = wavelet_reconstruction((sample + 1) / 2, cond_img)
            sample = F.interpolate(fixed, size=self.output_size, mode="bicubic", antialias=True)
            out = (sample * 255.0).clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
        self._mark("post")
        return out


    def shared_cleaner(self, lq: torch.Tensor, tiled: bool, tile_size: int, tile_stride: int) -> torch.Tensor:
        """apply_cleaner. With shard_cleaner set and more than one torch.distributed rank, every rank passes the same
        input and gets the same stage-1 output: a tiled cleaner runs each rank's share of the windows (make_tiled_fn's
        shard), an un-tiled one runs on rank 0, which broadcasts its output."""
        import torch.distributed as dist
        if not (self.shard_cleaner and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return self.apply_cleaner(lq, tiled, tile_size, tile_stride)
        if tiled and lq.size(2) >= tile_size and lq.size(3) >= tile_size:       # apply_cleaner's own test for tiling
            return self.apply_cleaner(lq, tiled, tile_size, tile_stride)
        out = self.apply_cleaner(lq, tiled, tile_size, tile_stride).contiguous() if dist.get_rank() == 0 else None
        meta = [(tuple(out.shape), out.dtype) if out is not None else None]
        dist.broadcast_object_list(meta, src=0)
        if out is None:
            out = torch.empty(meta[0][0], dtype=meta[0][1], device=lq.device)
        dist.broadcast(out, src=0)
        return out


class SwinIRPipeline(Pipeline):
    def apply_cleaner(self, lq: torch.Tensor, tiled: bool, tile_size: int, tile_stride: int) -> torch.Tensor:
        """pipeline.py:371-397. Un-tiled: resize the short edge to >= 512 first, pad to x64, crop.
        Tiled: Gaussian-blended `tile_size` windows through make_tiled_fn, resize afterwards (the
        reference's order in each branch). The un-tiled branch fits one GPU's memory; the tiled one is kept for
        parity of results with runs of the reference that used it."""
        if tiled and (lq.size(2) < tile_size or lq.size(3) < tile_size):
            print("[SwinIR]: the input size is tiny and unnecessary to tile.")
            tiled = False
        if tiled and tile_size % 64 != 0:
            raise ValueError("SwinIR (cleaner) tile size must be a multiple of 64")
        if not tiled:
            if min(lq.shape[2:]) < 512:
                lq = resize_short_edge_to(lq, size=512)
            h0, w0 = lq.shape[2:]
            lq = pad_to_multiples_of(lq, multiple=64)
            return self.cleaner(lq)[:, :, :h0, :w0]
        output = make_tiled_fn(self.cleaner, size=tile_size, stride=tile_stride, shard=self.shard_cleaner)(lq)
        if min(output.shape[2:]) < 512:
            output = resize_short_edge_to(output, size=512)
        return output


class BSRNetPipeline(Pipeline):
    """pipeline.py:324-366: the v2 blind-SR recipe. Stage 1 is RRDBNet (x4) on the LQ image itself, then an
    antialiased bicubic resize to the output size (upscale x LQ) or, for outputs under 512, short edge 512."""

    def __init__(self, cleaner, cldm: ControlLDM, diffusion: Diffusion, cond_fn, device: str, upscale: float) -> None:
        super().__init__(cleaner, cldm, diffusion, cond_fn, device)
        self.upscale = upscale

    def set_output_size(self, lq_size: Tuple[int]) -> None:
        h, w = lq_size[2:]
        self.output_size = (int(h * self.upscale), int(w * self.upscale))

    def apply_cleaner(self, lq: torch.Tensor, tiled: bool, tile_size: int, tile_stride: int) -> torch.Tensor:
        if tiled and (lq.size(2) < tile_size or lq.size(3) < tile_size):
            print("[BSRNet]: the input size is tiny and unnecessary to tile.")
            tiled = False
        model = make_tiled_fn(self.cleaner, tile_size, tile_stride, scale_type="up", scale=4,
                                                  shard=self.shard_cleaner) if tiled else self.cleaner
        up4 = model(lq)
        if min(self.output_size) < 512:
            return resize_short_edge_to(up4, size=512)
        return F.interpolate(up4, size=self.output_size, mode="bicubic", antialias=True)


class SCUNetPipeline(Pipeline):
    """pipeline.py:400-420: the v2 blind-denoising recipe. Stage 1 is SCUNet on the (pre-upscaled) LQ image, optionally
    over Gaussian-blended tiles; outputs under 512 are resized to short edge 512."""

    def apply_cleaner(self, lq: torch.Tensor, tiled: bool, tile_size: int, tile_stride: int) -> torch.Tensor:
        if tiled and (lq.size(2) < tile_size or lq.size(3) < tile_size):
            print("[SCUNet]: the input size is tiny and unnecessary to tile.")
            tiled = False
        model = make_tiled_fn(self.cleaner, tile_size, tile_stride, shard=self.shard_cleaner) if tiled else self.cleaner
        output = model(lq)
        if min(output.shape[2:]) < 512:
            output = resize_short_edge_to(output, size=512)
        return output
