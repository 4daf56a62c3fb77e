"""Checkpoint registry of the inference loops (reference: diffbir/inference/pretrained_models.py).

The reference downloads these files on first use; this package never touches the network: a loop
resolves the same registry keys to files in a local directory (`--weights_dir`, default
`$DIFFBIR_WEIGHTS_DIR` or ./weights) under the file names the reference's URLs end in."""
import os
from typing import Dict

# key -> file name (the basename of the reference's download URL for that key)
MODELS: Dict[str, str] = {
    # stage-1 cleaners
    "swinir_general": "general_swinir_v1.ckpt",
    "swinir_face": "face_swinir_v1.ckpt",
    "swinir_realesrgan": "realesrgan_s4_swinir_100k.pth",
    "bsrnet": "BSRNet.pth",
    "scunet_psnr": "scunet_color_real_psnr.pth",
    # Stable Diffusion 2.1 base (UNet + VAE + OpenCLIP text tower)
    "sd_v2.1": "v2-1_512-ema-pruned.ckpt",
    "sd_v2.1_zsnr": "sd2.1-base-zsnr-laionaes5.ckpt",
    # IRControlNet
    "v1_face": "v1_face.pth",
    "v1_general": "v1_general.pth",
    "v2": "v2.pth",
    "v2.1": "DiffBIR_v2.1.pt",
    # captioner (--captioner ram); its tag list and per-class thresholds sit next to it (utils/caption.py)
    "ram_plus": "ram_plus_swin_large_14m.pth",
}
UNSUPPORTED: Dict[str, str] = {}      # (every cleaner of the reference registry is built)


def default_weights_dir() -> str:
    return os.environ.get("DIFFBIR_WEIGHTS_DIR", "weights")


def resolve(key: str, weights_dir: str) -> str:
    if key in UNSUPPORTED:
        raise NotImplementedError(f"checkpoint '{key}' belongs to a cleaner outside the accelerated path")
    path = os.path.join(weights_dir, MODELS[key])
    if not os.path.isfile(path):
        raise FileNotFoundError(
            f"checkpoint '{key}' not found at {path}: place the file the reference downloads for this key "
            f"({MODELS[key]}) in --weights_dir (no network access here), or pass --synthetic")
    return path
