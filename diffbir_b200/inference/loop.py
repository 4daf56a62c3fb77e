"""InferenceLoop — drop-in counterpart of the reference's diffbir/inference/loop.py:30-243: same
constructor (an argparse Namespace with the flags of inference.py), same run() (folder of LQ images
-> `pipeline.run` with the 26 positional arguments -> PNGs + prompt.csv). Differences, all loud:
checkpoints come from a local directory (or `--synthetic` random-init weights), and the options
whose networks are outside the accelerated path raise NotImplementedError at construction."""
from __future__ import annotations

import csv
import os
from argparse import Namespace
from pathlib import Path
from typing import Generator, List

import numpy as np
import torch
import yaml
from PIL import Image

from ..utils.caption import Captioner, EmptyCaptioner
from ..utils.common import instantiate_from_config
from .pretrained_models import default_weights_dir, resolve

CONFIG_DIR = Path(__file__).resolve().parents[2] / "configs" / "inference"
SUPPORTED_SAMPLERS = ("dpm++_m2", "spaced", "ddim", "edm_euler", "edm_euler_a", "edm_heun", "edm_dpm_2", "edm_dpm_2_a", "edm_lms",
                      "edm_dpm++_2s_a", "edm_dpm++_sde", "edm_dpm++_2m", "edm_dpm++_2m_sde", "edm_dpm++_3m_sde")


def load_config(name: str) -> dict:
    with open(CONFIG_DIR / name) as f:
        return yaml.safe_load(f)


class _StubGlobal:
    """Stands in for a pickled global that is not needed to read the tensors (Lightning callbacks,
    hyper-parameter containers, ...)."""

    def __init__(self, *a, **k):
        pass

    def __setstate__(self, state):
        pass

    def __call__(self, *a, **k):
        return self


class _TensorOnlyPickle:
    """pickle_module for torch.load: resolves torch / numpy / stdlib container globals, stubs the rest.
    Lightning-style SD checkpoints (v2-1_512-ema-pruned.ckpt, ...) carry non-tensor globals that
    weights_only=True rejects; the reference uses a plain torch.load (utils/common.py:104-111)."""
    import pickle as _pickle
    __name__ = "diffbir_b200_tensor_only_pickle"
    _SAFE = ("torch", "collections", "numpy", "builtins", "_codecs", "copyreg")

    class Unpickler(_pickle.Unpickler):
        def find_class(self, module, name):
            if module.split(".")[0] in _TensorOnlyPickle._SAFE and not (module == "builtins" and name in (
                    "eval", "exec", "compile", "open", "__import__", "getattr", "setattr")):
                return super().find_class(module, name)
            return _StubGlobal

    @staticmethod
    def load(f, **kw):
        return _TensorOnlyPickle.Unpickler(f, **kw).load()


def load_checkpoint(path: str) -> dict:
    """torch.load on CPU + the unwrapping of utils/common.py:104-120 (state_dict wrapper, module. prefix).
    Tries the safe tensors-only loader first; checkpoints with foreign pickled globals are re-read with
    an unpickler that keeps the tensors and stubs everything else."""
    import pickle
    try:
        sd = torch.load(path, map_location="cpu", weights_only=True)
    except pickle.UnpicklingError:
        sd = torch.load(path, map_location="cpu", weights_only=False, pickle_module=_TensorOnlyPickle)
    if "state_dict" in sd:
        sd = sd["state_dict"]
    if sd and next(iter(sd)).startswith("module."):
        sd = {k[len("module."):]: v for k, v in sd.items()}
    return sd


def check_supported(args: Namespace) -> None:
    """Everything this package cannot honour is refused here, before any model is built."""
    if args.device != "cuda":
        raise NotImplementedError(f"--device {args.device}: the engines are CUDA (sm_90a) only, there is no CPU path")
    if args.sampler not in SUPPORTED_SAMPLERS:
        raise NotImplementedError(f"--sampler {args.sampler}: not one of {SUPPORTED_SAMPLERS}")
    if args.captioner == "llava" and str(getattr(args, "llava_bit", "4")) != "16":
        from ..utils.caption import llava_bit_message
        raise NotImplementedError(llava_bit_message(getattr(args, "llava_bit", "4")))
    if args.captioner not in ("none", "ram", "llava"):
        raise NotImplementedError(f"--captioner {args.captioner}: captioners are outside the path; pass --captioner none "
                                  "and a --pos_prompt")
    if args.guidance:
        raise NotImplementedError("--guidance: restoration guidance is not wired into the reference's samplers either")
    if args.precision == "fp32":
        raise NotImplementedError("--precision fp32: the kernels take 16-bit operands (fp32 accumulate / residual stream)")
    # stage-2 images are at least 512 on both sides, so a tile of 512 or less always tiles; larger tiles are left to the
    # pipeline, which (like the reference) runs un-tiled when the image is smaller than a tile
    if (args.vae_encoder_tiled and args.vae_encoder_tile_size <= 512) or (args.vae_decoder_tiled and args.vae_decoder_tile_size <= 512):
        raise NotImplementedError("Tiled-VAE is outside the path (SURVEY.md §8f); the VAE engines run un-tiled")


def prompt_with_caption(caption: str, pos_prompt: str) -> str:
    """loop.py:167-169: the caption, then the user's positive prompt, empty parts dropped."""
    return ", ".join([text for text in [caption, pos_prompt] if text])


class InferenceLoop:
    captioner: Captioner = EmptyCaptioner("cuda")      # replaced by load_captioner

    def __init__(self, args: Namespace) -> None:
        self.args = args
        check_supported(args)
        self.loop_ctx = {}
        self.pipeline = None
        self.weights_dir = getattr(args, "weights_dir", None) or default_weights_dir()
        self.synthetic = bool(getattr(args, "synthetic", False))
        self.load_cleaner()
        self.load_cldm()
        self.load_captioner()
        self.cond_fn = None
        self.load_pipeline()

    # ------------------------------------------------------------------ models
    def load_cleaner(self) -> None:
        raise NotImplementedError

    def load_pipeline(self) -> None:
        raise NotImplementedError

    def load_captioner(self) -> None:
        """loop.py:119-129: --captioner none -> no caption, ram -> RAM++ tags, llava -> a LLaVA-1.5 description, each
        on the engine."""
        if self.args.captioner == "llava":
            from ..utils.caption import LLaVACaptioner
            self.captioner = LLaVACaptioner(self.args.device, self.args.llava_bit, self.weights_dir, self.synthetic,
                                            self.args.seed)
        elif self.args.captioner == "ram":
            from ..utils.caption import RAMCaptioner
            self.captioner = RAMCaptioner(self.args.device, self.weights_dir, self.synthetic, self.args.seed)
        else:
            self.captioner = EmptyCaptioner(self.args.device)

    def _operand_check(self) -> None:
        from .. import lib
        want = {"fp16": torch.float16, "bf16": torch.bfloat16}[self.args.precision]
        have = lib.operand_dtype()
        if want != have:
            raise RuntimeError(f"--precision {self.args.precision} but libdiffbir_b200.so was built for {have} operands "
                               "(rebuild with -DDBIR_OPERAND_BF16 for bf16)")

    def load_cldm(self) -> None:
        """loop.py:47-99: SD weights by version, ControlNet weights by version / task, diffusion config."""
        from ..model import ControlLDM, Diffusion  # noqa: F401  (targets of the YAML reflection)
        a = self.args
        self._operand_check()
        self.cldm = instantiate_from_config(load_config("cldm.yaml"), device=a.device,
                                            synthetic_tokenizer=self.synthetic)
        if self.synthetic:
            from ..utils import synth
            from .. import arch
            unused, missing = self.cldm.load_pretrained_sd(
                synth.synthetic_sd_checkpoint(arch.UNET_CFG, arch.VAE_CFG, arch.CLIP_TEXT_CFG, a.seed))
            assert not missing
            self.cldm.load_controlnet_from_ckpt(
                synth.make_state_dict(arch.unet_shapes(arch.CONTROLNET_CFG, True), a.seed + 3, arch.is_zero_init))
        else:
            sd_key = "sd_v2.1_zsnr" if a.version == "v2.1" else "sd_v2.1"
            unused, missing = self.cldm.load_pretrained_sd(load_checkpoint(resolve(sd_key, self.weights_dir)))
            print(f"load pretrained stable diffusion, unused weights: {unused}, missing weights: {missing}")
            if a.version == "v1":
                if a.task == "face":
                    ck = "v1_face"
                elif a.task in ("sr", "denoise"):
                    ck = "v1_general"
                else:
                    raise ValueError(f"DiffBIR v1 doesn't support task: {a.task}, please use v2 or v2.1 by passing '--version'")
            else:
                ck = "v2" if a.version == "v2" else "v2.1"
            self.cldm.load_controlnet_from_ckpt(load_checkpoint(resolve(ck, self.weights_dir)))
            print("load controlnet weight")
        cfg = "diffusion.yaml" if a.version in ("v1", "v2") else "diffusion_v2.1.yaml"
        self.diffusion = instantiate_from_config(load_config(cfg))

    # ------------------------------------------------------------------ io
    def setup(self) -> None:
        self.save_dir = self.args.output
        os.makedirs(self.save_dir, exist_ok=True)

    def load_lq(self) -> Generator[Image.Image, None, None]:
        img_exts = [".png", ".jpg", ".jpeg"]
        assert os.path.isdir(self.args.input), "Please put your low-quality images in a folder."
        for file_name in sorted(os.listdir(self.args.input)):
            stem, ext = os.path.splitext(file_name)
            if ext not in img_exts:
                print(f"{file_name} is not an image, continue")
                continue
            file_path = os.path.join(self.args.input, file_name)
            lq = Image.open(file_path).convert("RGB")
            print(f"load lq: {file_path}")
            self.loop_ctx["file_stem"] = stem
            yield lq

    def after_load_lq(self, lq: Image.Image) -> np.ndarray:
        return np.array(lq)

    # ------------------------------------------------------------------ run
    @torch.no_grad()
    def run(self) -> None:
        a = self.args
        self.setup()
        for lq in self.load_lq():
            caption = self.captioner(lq)                 # fp32 logits; nothing here runs under autocast
            pos_prompt = prompt_with_caption(caption, a.pos_prompt)
            neg_prompt = a.neg_prompt
            lq = self.after_load_lq(lq)
            n_samples, batch_size = a.n_samples, a.batch_size
            num_batches = (n_samples + batch_size - 1) // batch_size
            samples: List[np.ndarray] = []
            for i in range(num_batches):
                n_inputs = min((i + 1) * batch_size, n_samples) - i * batch_size
                batch_samples = self.pipeline.run(
                    np.tile(lq[None], (n_inputs, 1, 1, 1)), a.steps, a.strength, a.cleaner_tiled, a.cleaner_tile_size,
                    a.cleaner_tile_stride, a.vae_encoder_tiled, a.vae_encoder_tile_size, a.vae_decoder_tiled,
                    a.vae_decoder_tile_size, a.cldm_tiled, a.cldm_tile_size, a.cldm_tile_stride, pos_prompt, neg_prompt,
                    a.cfg_scale, a.start_point_type, a.sampler, a.noise_aug, a.rescale_cfg, a.s_churn, a.s_tmin,
                    a.s_tmax, a.s_noise, a.eta, a.order)
                samples.extend(list(batch_samples))
            self.save(samples, pos_prompt, neg_prompt)

    def save(self, samples: List[np.ndarray], pos_prompt: str, neg_prompt: str) -> None:
        file_stem = self.loop_ctx["file_stem"]
        assert len(samples) == self.args.n_samples
        for i, sample in enumerate(samples):
            file_name = f"{file_stem}_{i}.png" if self.args.n_samples > 1 else f"{file_stem}.png"
            save_path = os.path.join(self.save_dir, file_name)
            Image.fromarray(sample).save(save_path)
            print(f"save result to {save_path}")
        append_prompt_row(self.save_dir, file_stem, pos_prompt, neg_prompt)


def append_prompt_row(save_dir: str, file_stem: str, pos_prompt: str, neg_prompt: str) -> None:
    """One row of <save_dir>/prompt.csv, the header written with the first row."""
    csv_path = os.path.join(save_dir, "prompt.csv")
    new = not os.path.exists(csv_path)
    with open(csv_path, "a", newline="") as f:
        w = csv.writer(f)
        if new:
            w.writerow(["file_name", "pos_prompt", "neg_prompt"])
        w.writerow([file_stem, pos_prompt, neg_prompt])
