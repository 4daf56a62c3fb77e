"""Command line of the reference's inference.py (same flags, same meaning) on the H100 engines.

  python inference.py --task sr --upscale 4 --version v2.1 --sampler spaced --steps 50 \
      --captioner none --pos_prompt '' --neg_prompt 'low quality, blurry' --cfg_scale 4.0 \
      --input inputs/ --output results/ --weights_dir /path/to/checkpoints

Differences from the reference (each refused with a message, never silently ignored): checkpoints are
read from --weights_dir (no downloads), `--synthetic` runs random-init weights of the real
architecture, the defaults of --sampler / --captioner are the ones this package runs ("spaced",
"none"), and tasks / samplers / captioners whose networks are outside the accelerated path raise
NotImplementedError (diffbir_b200/inference/loop.py:check_supported)."""
import random
from argparse import ArgumentParser, Namespace

import numpy as np
import torch

DEFAULT_POS_PROMPT = (
    "Cinematic, High Contrast, highly detailed, taken using a Canon EOS R camera, "
    "hyper detailed photo - realistic maximum detail, 32k, Color Grading, ultra HD, extreme meticulous detailing, "
    "skin pore detailing, hyper sharpness, perfect without deformations."
)
DEFAULT_NEG_PROMPT = (
    "painting, oil painting, illustration, drawing, art, sketch, oil painting, cartoon, "
    "CG Style, 3D render, unreal engine, blurring, dirty, messy, worst quality, low quality, frames, watermark, "
    "signature, jpeg artifacts, deformed, lowres, over-smooth."
)
SAMPLERS = ["dpm++_m2", "spaced", "ddim", "edm_euler", "edm_euler_a", "edm_heun", "edm_dpm_2", "edm_dpm_2_a", "edm_lms",
            "edm_dpm++_2s_a", "edm_dpm++_sde", "edm_dpm++_2m", "edm_dpm++_2m_sde", "edm_dpm++_3m_sde"]


def build_parser() -> ArgumentParser:
    p = ArgumentParser()
    # model parameters
    p.add_argument("--task", type=str, default="sr", choices=["sr", "face", "denoise", "unaligned_face"])
    p.add_argument("--upscale", type=float, default=4, help="Upscale factor of output.")
    p.add_argument("--version", type=str, default="v2.1", choices=["v1", "v2", "v2.1", "custom"])
    p.add_argument("--train_cfg", type=str, default="")
    p.add_argument("--ckpt", type=str, default="")
    # sampling parameters
    p.add_argument("--sampler", type=str, default="spaced", choices=SAMPLERS)
    p.add_argument("--steps", type=int, default=10)
    p.add_argument("--start_point_type", type=str, choices=["noise", "cond"], default="noise")
    # tiling
    p.add_argument("--cleaner_tiled", action="store_true")
    p.add_argument("--cleaner_tile_size", type=int, default=512)
    p.add_argument("--cleaner_tile_stride", type=int, default=256)
    p.add_argument("--vae_encoder_tiled", action="store_true")
    p.add_argument("--vae_encoder_tile_size", type=int, default=256)
    p.add_argument("--vae_decoder_tiled", action="store_true")
    p.add_argument("--vae_decoder_tile_size", type=int, default=256)
    p.add_argument("--cldm_tiled", action="store_true")
    p.add_argument("--cldm_tile_size", type=int, default=512)
    p.add_argument("--cldm_tile_stride", type=int, default=256)
    # prompts / guidance
    p.add_argument("--captioner", type=str, choices=["none", "llava", "ram"], default="none")
    p.add_argument("--pos_prompt", type=str, default=DEFAULT_POS_PROMPT)
    p.add_argument("--neg_prompt", type=str, default=DEFAULT_NEG_PROMPT)
    p.add_argument("--cfg_scale", type=float, default=6.0)
    p.add_argument("--rescale_cfg", action="store_true")
    p.add_argument("--noise_aug", type=int, default=0)
    p.add_argument("--s_churn", type=float, default=0)
    p.add_argument("--s_tmin", type=float, default=0)
    p.add_argument("--s_tmax", type=float, default=300)
    p.add_argument("--s_noise", type=float, default=1)
    p.add_argument("--eta", type=float, default=1)
    p.add_argument("--order", type=int, default=1)
    p.add_argument("--strength", type=float, default=1)
    p.add_argument("--batch_size", type=int, default=1)
    p.add_argument("--guidance", action="store_true")
    p.add_argument("--g_loss", type=str, default="w_mse", choices=["mse", "w_mse"])
    p.add_argument("--g_scale", type=float, default=0.0)
    # io
    p.add_argument("--input", type=str, required=True)
    p.add_argument("--n_samples", type=int, default=1)
    p.add_argument("--output", type=str, required=True)
    # common
    p.add_argument("--seed", type=int, default=231)
    p.add_argument("--device", type=str, default="cuda", choices=["cpu", "cuda", "mps"])
    p.add_argument("--precision", type=str, default="fp16", choices=["fp32", "fp16", "bf16"])
    p.add_argument("--llava_bit", type=str, default="4", choices=["16", "8", "4"])
    # this package only
    p.add_argument("--weights_dir", type=str, default="", help="Directory holding the reference's checkpoint files.")
    p.add_argument("--synthetic", action="store_true", help="Random-init weights of the real architecture.")
    return p


def parse_args(argv=None) -> Namespace:
    return build_parser().parse_args(argv)


def set_seed(seed: int) -> None:
    """accelerate.utils.set_seed: python, numpy and torch (CPU + CUDA) generators."""
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


def main(argv=None) -> None:
    args = parse_args(argv)
    if args.device == "cuda" and not torch.cuda.is_available():
        raise SystemExit("inference.py needs a CUDA device (sm_90a): there is no CPU fallback for the engines")
    set_seed(args.seed)
    from diffbir_b200.inference import (BFRInferenceLoop, BIDInferenceLoop, BSRInferenceLoop, CustomInferenceLoop,
                                        UnAlignedBFRInferenceLoop)
    loops = {"sr": BSRInferenceLoop, "face": BFRInferenceLoop, "denoise": BIDInferenceLoop,
             "unaligned_face": UnAlignedBFRInferenceLoop}
    if args.version == "custom":
        CustomInferenceLoop(args).run()
    else:
        loops[args.task](args).run()
    print("done!")


if __name__ == "__main__":
    main()
