"""Captioners of the inference loops (reference diffbir/utils/caption.py): the caption is prepended to the positive
prompt (loop.py: pos_prompt = ", ".join([caption, pos_prompt])).

RAMCaptioner runs RAM++ (ram_plus_swin_large_14m.pth) on engine.ram.RamPlusEngine. Weights come from the local
registry (`ram_plus` in --weights_dir). The tag names and per-class thresholds are the reference's data files
ram_tag_list.txt and ram_tag_list_threshold.txt, read from the same directory.
"""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

import numpy as np
import torch
from PIL import Image

TAG_LIST = "ram_tag_list.txt"
THRESHOLDS = "ram_tag_list_threshold.txt"


class Captioner:
    def __init__(self, device) -> None:
        self.device = device

    def __call__(self, image: Image.Image) -> str:
        raise NotImplementedError


class EmptyCaptioner(Captioner):
    def __call__(self, image: Image.Image) -> str:
        return ""


def read_tag_files(weights_dir: str, classes: int) -> Tuple[List[str], List[float]]:
    """The RAM++ tag list (one name per line) and per-class thresholds (one float per line) from weights_dir."""
    paths = [os.path.join(weights_dir, TAG_LIST), os.path.join(weights_dir, THRESHOLDS)]
    missing = [p for p in paths if not os.path.isfile(p)]
    if missing:
        raise FileNotFoundError(f"RAM++ needs {TAG_LIST} and {THRESHOLDS} (the reference's ram/data files) next to "
                                f"its checkpoint in --weights_dir; missing: {', '.join(missing)}")
    with open(paths[0], encoding="utf-8") as f:
        tags = f.read().splitlines()
    with open(paths[1], encoding="utf-8") as f:
        thresholds = [float(s.strip()) for s in f if s.strip()]
    if len(tags) != classes or len(thresholds) != classes:
        raise ValueError(f"{TAG_LIST} / {THRESHOLDS}: {len(tags)} tags and {len(thresholds)} thresholds, "
                         f"expected {classes} of each")
    return tags, thresholds


def preprocess(image: Image.Image, size: int = 384) -> torch.Tensor:
    """ram/transform.py up to its Normalize (which the engine folds into the patch embed): RGB, PIL bilinear resize
    to size x size, / 255 -> fp32 [1, 3, size, size]."""
    img = image.convert("RGB").resize((size, size), Image.BILINEAR)
    return torch.from_numpy(np.asarray(img, dtype=np.float32) / 255.0).permute(2, 0, 1).unsqueeze(0).contiguous()


def decide(logits: torch.Tensor, thresholds: torch.Tensor, tags: List[str]) -> str:
    """generate_tag's decision (sigmoid(logit) > class threshold, ram_plus.py:322-336) joined with ", " in tag-list
    order, as RAMCaptioner's `.replace(" | ", ", ")` gives."""
    keep = (torch.sigmoid(logits.float().cpu()) > thresholds.cpu()).nonzero().flatten().tolist()
    return ", ".join(tags[i] for i in keep)


class RAMCaptioner(Captioner):
    def __init__(self, device, weights_dir: Optional[str] = None, synthetic: bool = False, seed: int = 1234) -> None:
        super().__init__(device)
        from .. import arch
        from ..engine.ram import RamPlusEngine
        from ..inference.pretrained_models import default_weights_dir, resolve
        classes = arch.RAM_CFG["num_class"]
        if synthetic:
            from .synth import synthetic_ram
            sd, tags, thresholds = synthetic_ram(seed)
        else:
            from ..inference.loop import load_checkpoint
            weights_dir = weights_dir or default_weights_dir()
            tags, thresholds = read_tag_files(weights_dir, classes)
            sd = load_checkpoint(resolve("ram_plus", weights_dir))
        self.tags = tags
        self.thresholds = torch.tensor(thresholds, dtype=torch.float32)
        self.engine = RamPlusEngine(sd, device=device)
        self.size = arch.RAM_CFG["img_size"]

    @torch.no_grad()
    def __call__(self, image: Image.Image) -> str:
        x = preprocess(image, self.size).to(self.engine.dev)
        return decide(self.engine.forward(x)[0], self.thresholds, self.tags)
