"""CustomInferenceLoop (reference: diffbir/inference/custom_loop.py:19-93): `--version custom --train_cfg <yaml>
--ckpt <controlnet.pt>` — a user's own stage-2 training run. The networks are whatever the training YAML names
(`model.cldm`, `model.swinir`, `model.diffusion`, same `target:` / `params:` reflection), the weights are the paths the
YAML's `train:` block holds (`sd_path`, `swinir_path`) plus `--ckpt`; stage 1 is SwinIR, upscaling is a bicubic resize
of the LQ image. The YAML is read with PyYAML (the reference's training configs use no OmegaConf interpolation).
`--synthetic` only swaps the BPE vocabulary file for the hash tokenizer (random-weight checkpoints in the tests)."""
from argparse import Namespace
from typing import Optional

import numpy as np
import yaml
from PIL import Image

from ..pipeline import SwinIRPipeline
from ..utils.common import instantiate_from_config
from .loop import InferenceLoop, batch_images_setup, check_supported, load_checkpoint
from .ranks import Ranks


class CustomInferenceLoop(InferenceLoop):
    def __init__(self, args: Namespace, ranks: Optional[Ranks] = None) -> None:
        self.args = args
        self.ranks = ranks
        check_supported(args)
        batch_images_setup(args)
        if not args.train_cfg or not args.ckpt:
            raise ValueError("--version custom needs --train_cfg (the stage-2 training YAML) and --ckpt (ControlNet weights)")
        with open(args.train_cfg) as f:
            self.train_cfg = yaml.safe_load(f)
        self.loop_ctx = {}
        self.pipeline = None
        self.load_cleaner()
        self.load_cldm()
        self.cond_fn = None
        self.load_pipeline()

    def _train_path(self, key: str) -> str:
        path = (self.train_cfg.get("train") or {}).get(key)
        if not path:
            raise ValueError(f"{self.args.train_cfg}: train.{key} is empty (custom_loop.py:{'39' if key == 'sd_path' else '70'} loads it)")
        return path

    def load_cldm(self) -> None:
        """custom_loop.py:36-65: ControlLDM from model.cldm, SD weights from train.sd_path, ControlNet from --ckpt."""
        from ..model import ControlLDM, Diffusion  # noqa: F401  (targets of the YAML reflection)
        self._operand_check()
        self.cldm = instantiate_from_config(self.train_cfg["model"]["cldm"], device=self.args.device,
                                            synthetic_tokenizer=bool(getattr(self.args, "synthetic", False)))
        unused, missing = self.cldm.load_pretrained_sd(load_checkpoint(self._train_path("sd_path")))
        print(f"load pretrained stable diffusion, unused weights: {unused}, missing weights: {missing}")
        self.cldm.load_controlnet_from_ckpt(load_checkpoint(self.args.ckpt))
        print("load controlnet weight")
        self.diffusion = instantiate_from_config(self.train_cfg["model"]["diffusion"])

    def load_cleaner(self) -> None:
        """custom_loop.py:67-79."""
        from ..model import SwinIR  # noqa: F401
        self.cleaner = instantiate_from_config(self.train_cfg["model"]["swinir"], device=self.args.device)
        self.cleaner.load_state_dict(load_checkpoint(self._train_path("swinir_path")), strict=True)

    def load_pipeline(self) -> None:
        self.pipeline = SwinIRPipeline(self.cleaner, self.cldm, self.diffusion, self.cond_fn, self.args.device)

    def after_load_lq(self, lq: Image.Image) -> np.ndarray:
        lq = lq.resize(tuple(int(x * self.args.upscale) for x in lq.size), Image.BICUBIC)
        return super().after_load_lq(lq)
