"""Seeded synthetic checkpoints in the reference's state_dict layout.

There is no network for real weights, so bench / tests use random-init weights of the real
architecture.  Every tensor is drawn from its own generator (seed = crc32(key) ^ seed), so
the result does not depend on enumeration order and is identical on every machine with the
same torch CPU RNG.  Tensors the reference zero-initialises (zero_module) are re-randomised
with N(0, 1/fan_in) — otherwise eps == 0 and control == 0 and every parity check is vacuous
(SURVEY.md §8d).
"""
from __future__ import annotations

import zlib
from collections import OrderedDict
from typing import Callable, Dict, Optional, Tuple

import torch


def _gen(key: str, seed: int) -> torch.Generator:
    g = torch.Generator(device="cpu")
    g.manual_seed((zlib.crc32(key.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
    return g


def make_state_dict(shapes: "OrderedDict[str, Tuple[int, ...]]", seed: int = 1234,
                    zero_init: Optional[Callable[[str], bool]] = None,
                    prefix: str = "") -> "OrderedDict[str, torch.Tensor]":
    sd = OrderedDict()
    for key, shape in shapes.items():
        g = _gen(key, seed)
        if len(shape) >= 2:
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            if key.endswith("relative_position_bias_table") or "embedding" in key:
                t = torch.randn(shape, generator=g) * 0.02
            elif zero_init is not None and zero_init(key):
                t = torch.randn(shape, generator=g) * fan_in ** -0.5
            else:
                b = fan_in ** -0.5
                t = (torch.rand(shape, generator=g) * 2 - 1) * b
        elif len(shape) == 1 and key.endswith("weight"):      # norm gains
            t = 1.0 + 0.05 * torch.randn(shape, generator=g)
        elif len(shape) == 0:
            t = torch.tensor(2.6593)
        else:                                                  # biases / norm shifts
            t = 0.02 * torch.randn(shape, generator=g)
        sd[prefix + key] = t
    return sd


# ----------------------------------------------------------------------------------------
# Synthetic full pipelines (bench / tests): random-init weights of the real architecture,
# loaded through the same loaders a real checkpoint would take.
# ----------------------------------------------------------------------------------------
def synthetic_sd_checkpoint(unet_cfg=None, vae_cfg=None, clip_cfg=None, seed: int = 1234):
    """An SD-style checkpoint dict with the reference prefixes (cldm.py:37-41)."""
    from .. import arch
    unet_cfg = arch.UNET_CFG if unet_cfg is None else unet_cfg
    vae_cfg = arch.VAE_CFG if vae_cfg is None else vae_cfg
    clip_cfg = arch.CLIP_TEXT_CFG if clip_cfg is None else clip_cfg
    sd = OrderedDict()
    sd.update(make_state_dict(arch.unet_shapes(unet_cfg), seed, arch.is_zero_init, "model.diffusion_model."))
    sd.update(make_state_dict(arch.vae_shapes(vae_cfg), seed + 1, None, "first_stage_model."))
    sd.update(make_state_dict(arch.clip_text_shapes(clip_cfg), seed + 2, None, "cond_stage_model.model."))
    return sd


def build_synthetic_pipeline(device="cuda", seed: int = 1234, small: bool = False, v_prediction: bool = False):
    """SwinIRPipeline on synthetic weights. small=True uses the reduced test architectures;
    v_prediction=True uses the v2.1 diffusion settings (v-parameterization, zero terminal SNR:
    reference configs/inference/diffusion_v2.1.yaml)."""
    from .. import arch
    from ..model import ControlLDM, Diffusion, SwinIR
    from ..pipeline import SwinIRPipeline
    if small:
        ucfg = dict(arch.UNET_CFG, model_channels=64, context_dim=128)
        vcfg = dict(arch.VAE_CFG, ch=64)
        ccfg = dict(arch.CLIP_TEXT_CFG, width=128, heads=4, layers=3, vocab_size=512, embed_dim=128)
        scfg = dict(arch.SWINIR_CFG, depths=(2, 2), num_heads=(6, 6))
    else:
        ucfg, vcfg, ccfg, scfg = arch.UNET_CFG, arch.VAE_CFG, arch.CLIP_TEXT_CFG, arch.SWINIR_CFG
    cncfg = dict(ucfg, hint_channels=4)
    vae_yaml = dict(embed_dim=vcfg["embed_dim"],
                    ddconfig=dict(double_z=True, z_channels=vcfg["z_channels"], resolution=256,
                                  in_channels=vcfg["in_channels"], out_ch=vcfg["out_ch"], ch=vcfg["ch"],
                                  ch_mult=list(vcfg["ch_mult"]), num_res_blocks=vcfg["num_res_blocks"],
                                  attn_resolutions=[], dropout=0.0))
    clip_yaml = dict(embed_dim=ccfg["embed_dim"], layer="penultimate",
                     text_cfg=dict(context_length=ccfg["context_length"], vocab_size=ccfg["vocab_size"],
                                   width=ccfg["width"], heads=ccfg["heads"], layers=ccfg["layers"]))
    cldm = ControlLDM(ucfg, vae_yaml, clip_yaml, cncfg, 0.18215, device=device, synthetic_tokenizer=True)
    unused, missing = cldm.load_pretrained_sd(synthetic_sd_checkpoint(ucfg, vcfg, ccfg, seed))
    assert not missing, sorted(missing)[:3]
    cldm.load_controlnet_from_ckpt(make_state_dict(arch.unet_shapes(cncfg, True), seed + 3, arch.is_zero_init))
    swin = SwinIR(img_size=scfg["img_size"], patch_size=1, in_chans=3, embed_dim=scfg["embed_dim"],
                  depths=scfg["depths"], num_heads=scfg["num_heads"], window_size=8,
                  mlp_ratio=scfg["mlp_ratio"], sf=8, img_range=1.0, upsampler="nearest+conv",
                  resi_connection="1conv", unshuffle=True, unshuffle_scale=8, device=device)
    swin.load_state_dict(make_state_dict(arch.swinir_shapes(scfg), seed + 4))
    diffusion = Diffusion(linear_start=0.00085, linear_end=0.0120, timesteps=1000,
                          parameterization="v" if v_prediction else "eps", zero_snr=v_prediction)
    return SwinIRPipeline(swin, cldm, diffusion, None, device)


def synthetic_lq(h: int, w: int, batch: int = 1, seed: int = 0):
    """Image-like uint8 LQ input: uniform noise blurred with a Gaussian (SURVEY.md §8d config 2)."""
    import numpy as np
    import torch.nn.functional as F
    rng = np.random.default_rng(seed)
    x = torch.tensor(rng.random((batch, 3, h, w)), dtype=torch.float32)
    k = torch.arange(-9, 10, dtype=torch.float32)
    g = torch.exp(-k ** 2 / (2 * 3.0 ** 2))
    g = (g / g.sum())
    x = F.conv2d(F.pad(x, (9, 9, 0, 0), mode="reflect"), g.view(1, 1, 1, -1).repeat(3, 1, 1, 1), groups=3)
    x = F.conv2d(F.pad(x, (0, 0, 9, 9), mode="reflect"), g.view(1, 1, -1, 1).repeat(3, 1, 1, 1), groups=3)
    x = (x - x.min()) / (x.max() - x.min())
    return (x * 255).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous().numpy()


RUN_DEFAULTS = dict(steps=50, strength=1.0, cleaner_tiled=False, cleaner_tile_size=512, cleaner_tile_stride=256,
                    vae_encoder_tiled=False, vae_encoder_tile_size=256, vae_decoder_tiled=False,
                    vae_decoder_tile_size=256, cldm_tiled=False, cldm_tile_size=512, cldm_tile_stride=256,
                    pos_prompt="", neg_prompt="low quality, blurry, low-resolution, noisy, unsharp, weird textures",
                    cfg_scale=4.0, start_point_type="noise", sampler_type="spaced", noise_aug=0,
                    rescale_cfg=False, s_churn=0, s_tmin=0, s_tmax=300, s_noise=1, eta=1, order=1)


def synthetic_ram(seed: int = 1234):
    """RAM++ with seeded weights (arch.ram_shapes) plus a generated tag list tag0000.. and seeded per-class thresholds
    in [0.5, 1): (state_dict, tags, thresholds). Random weights give logits near 0, so the classes whose threshold
    lies just above 0.5 are the ones that fire."""
    from .. import arch
    n = arch.RAM_CFG["num_class"]
    thr = 0.5 + 0.5 * torch.rand(n, generator=_gen("ram_tag_list_threshold", seed))
    return make_state_dict(arch.ram_shapes(arch.RAM_CFG), seed), [f"tag{i:04d}" for i in range(n)], thr.tolist()


FACE_CLASS_GAIN = 15.0     # synthetic detector class heads: weight gain and face-logit bias (see synthetic_face_nets)
FACE_CLASS_BIAS = -1.4


def synthetic_face_nets(seed: int = 1234, class_gain: float = FACE_CLASS_GAIN, class_bias: float = FACE_CLASS_BIAS):
    """Seeded RetinaFace-ResNet50 and ParseNet state dicts (arch.retinaface_shapes / parsenet_shapes).
    - BatchNorm running variances are drawn in [1, 1.1): make_state_dict gives every norm shift 0.02 randn, and a
      variance must be positive.
    - The class heads' weights are scaled by `class_gain` and the face logits shifted by `class_bias`, so the score
      spreads over priors and only the strongest few pass 0.8. On a 128x160 synthetic_lq input at x4 that is 1-4
      faces, not none or thousands.
    - The landmark heads' biases place the five points of every prior where the 512 FFHQ template has them within
      a box of the prior's size, so detected faces have a plausible eye distance and alignment."""
    from .face import FACE_TEMPLATE_512
    from .. import arch
    det = make_state_dict(arch.retinaface_shapes(), seed + 11)
    parse = make_state_dict(arch.parsenet_shapes(), seed + 12)
    for sd in (det, parse):
        for k in sd:
            if k.endswith("running_var"):
                sd[k] = 1.0 + 0.1 * torch.rand(sd[k].shape, generator=_gen(k, seed))
    lm = torch.tensor(((FACE_TEMPLATE_512 - 256.0) / 512.0 / 0.1).reshape(-1), dtype=torch.float32)
    for i in range(3):
        det[f"ClassHead.{i}.conv1x1.weight"] *= class_gain
        det[f"ClassHead.{i}.conv1x1.bias"][1::2] += class_bias
        det[f"LandmarkHead.{i}.conv1x1.bias"] += torch.cat([lm, lm])
    return det, parse


def synthetic_llava(cfg: dict, seed: int = 1234, device="cuda", lm_head_scale: float = 1.0):
    """LLaVA-1.5 weights (arch.llava_shapes of cfg) drawn on `device` with the distributions of make_state_dict: at
    the 7B size a host generator would take minutes. Matrices are stored in fp16 (the checkpoints' dtype), vectors in
    fp32; each tensor has its own seeded device generator. lm_head is multiplied by lm_head_scale."""
    from .. import arch
    sd = OrderedDict()
    for key, shape in arch.llava_shapes(cfg).items():
        g = torch.Generator(device=device)
        g.manual_seed((zlib.crc32(key.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
        if len(shape) >= 2:
            fan_in = 1
            for d in shape[1:]:
                fan_in *= d
            if "embed" in key:
                t = torch.randn(shape, generator=g, device=device, dtype=torch.float16) * 0.02
            else:
                t = torch.rand(shape, generator=g, device=device, dtype=torch.float16).mul_(2).sub_(1).mul_(fan_in ** -0.5)
            if key == "lm_head.weight":
                t.mul_(lm_head_scale)
        elif key.endswith("weight"):
            t = 1.0 + 0.05 * torch.randn(shape, generator=g, device=device)
        else:
            t = 0.02 * torch.randn(shape, generator=g, device=device)
        sd[key] = t
    return sd
