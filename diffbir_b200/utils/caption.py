"""Captioners of the inference loops (reference diffbir/utils/caption.py): the caption is prepended to the positive
prompt (loop.py: pos_prompt = ", ".join([caption, pos_prompt])).

RAMCaptioner runs RAM++ (ram_plus_swin_large_14m.pth) on engine.ram.RamPlusEngine. Weights come from the local
registry (`ram_plus` in --weights_dir). The tag names and per-class thresholds are the reference's data files
ram_tag_list.txt and ram_tag_list_threshold.txt, read from the same directory.

LLaVACaptioner runs LLaVA-1.5-7B (fp16 weights, --llava_bit 16) on engine.llava.LlavaEngine: the registry
directories llava_v1.5_7b (config, SentencePiece tokenizer, shards) and clip_vit_l14_336 (the vision tower).
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


# ---- LLaVA-1.5-7B (reference utils/caption.py:52-145, --llava_bit 16) -------------------------------------------------
# The llava_v1 conversation template with the fixed question; mm_use_im_start_end is false, so the image is `<image>\n`
# in front of the question (caption.py:85-99, llava/conversation.py conv_vicuna_v1).
LLAVA_QUESTION = "Please give me a very short description of this image."
LLAVA_PROMPT = ("A chat between a curious human and an artificial intelligence assistant. The assistant gives helpful, "
                "detailed, and polite answers to the human's questions. USER: <image>\n" + LLAVA_QUESTION +
                " ASSISTANT:")
IMAGE_TOKEN = "<image>"
CLIP_BACKGROUND = (122, 116, 104)                 # expand2square's fill: int(image_mean * 255)


def expand2square(img: Image.Image, background=CLIP_BACKGROUND) -> Image.Image:
    """llava/mm_utils.py expand2square: pad the shorter side (centred, floor on the leading edge)."""
    w, h = img.size
    if w == h:
        return img
    side = max(w, h)
    out = Image.new(img.mode, (side, side), background)
    out.paste(img, (0, (w - h) // 2) if w > h else ((h - w) // 2, 0))
    return out


def preprocess_llava(image: Image.Image, size: int = 336) -> torch.Tensor:
    """process_images with image_aspect_ratio "pad" up to CLIPImageProcessor's normalisation (which the engine folds
    into the vision tower): RGB, expand2square, PIL bicubic resize to size x size (the shortest edge of a square; the
    centre crop is then the identity), / 255 -> fp32 [1, 3, size, size]."""
    img = expand2square(image.convert("RGB")).resize((size, size), Image.BICUBIC)
    x = np.asarray(img, dtype=np.uint8).astype(np.float64) * (1 / 255)
    return torch.from_numpy(x.astype(np.float32)).permute(2, 0, 1).unsqueeze(0).contiguous()


def clip_normalize(x: torch.Tensor) -> torch.Tensor:
    """CLIPImageProcessor's normalisation of preprocess_llava's output: the pixel_values the reference feeds CLIP."""
    from ..engine.llava import CLIP_MEAN, CLIP_STD
    return (x - torch.tensor(CLIP_MEAN).view(1, 3, 1, 1)) / torch.tensor(CLIP_STD).view(1, 3, 1, 1)


def splice_image_token(chunk_ids: List[List[int]], bos: int, image_index: int = -200) -> List[int]:
    """tokenizer_image_token (llava/mm_utils.py): every chunk between <image> markers is tokenised on its own (with
    BOS when the tokenizer adds one); the leading BOS is kept once and image_index goes between the chunks."""
    out: List[int] = []
    offset = 0
    if chunk_ids and chunk_ids[0] and chunk_ids[0][0] == bos:
        offset = 1
        out.append(bos)
    for i, ids in enumerate(chunk_ids):
        if i:
            out.append(image_index)
        out.extend(ids[offset:])
    return out


class ByteTokenizer:
    """Stand-in for LLaMA's tokenizer that needs no file (--synthetic): LLaMA's byte-fallback layout, <unk> = 0,
    <s> = 1, </s> = 2 and ids 3 .. 258 the bytes 0x00 .. 0xFF. Text encodes to UTF-8 bytes; ids past the byte range
    decode to a word " w<id>" so a caption of random weights stays printable."""
    bos, eos, unk = 1, 2, 0

    def encode(self, text: str, add_bos: bool = True) -> List[int]:
        return ([self.bos] if add_bos else []) + [3 + b for b in text.encode("utf-8")]

    def decode(self, ids: List[int]) -> str:
        """batch_decode(skip_special_tokens=True)."""
        out, run = [], bytearray()
        for i in ids:
            if i in (self.bos, self.eos, self.unk):
                continue
            if 3 <= i < 259:
                run.append(i - 3)
                continue
            out.append(run.decode("utf-8", errors="replace"))
            run = bytearray()
            out.append(f" w{i}")
        out.append(run.decode("utf-8", errors="replace"))
        return "".join(out)


class SentencePieceTokenizer:
    """The model's slow LlamaTokenizer (transformers 4.37, use_fast=False) on its tokenizer.model: add_bos_token and
    legacy from tokenizer_config.json (4.37 defaults: add BOS, legacy). Non-legacy mode encodes "▁" + text without
    SentencePiece's own dummy prefix (the unk-prefix trick of LlamaTokenizer._tokenize)."""

    def __init__(self, model_dir: str):
        import json
        import sentencepiece as spm
        self.sp = spm.SentencePieceProcessor(model_file=os.path.join(model_dir, "tokenizer.model"))
        conf = {}
        path = os.path.join(model_dir, "tokenizer_config.json")
        if os.path.isfile(path):
            with open(path, encoding="utf-8") as f:
                conf = json.load(f)
        self.add_bos = conf.get("add_bos_token", True)
        self.legacy = conf.get("legacy", None)
        self.legacy = True if self.legacy is None else bool(self.legacy)
        self.bos, self.eos, self.unk = self.sp.bos_id(), self.sp.eos_id(), self.sp.unk_id()

    def encode(self, text: str, add_bos: Optional[bool] = None) -> List[int]:
        if self.legacy or not text:
            ids = self.sp.encode(text)
        else:
            unk = self.sp.id_to_piece(self.unk)
            n = len(self.sp.encode(unk, out_type=str))
            ids = self.sp.encode(unk + "▁" + text.replace("▁", " "))[n:]
        return ([self.bos] if (self.add_bos if add_bos is None else add_bos) else []) + ids

    def decode(self, ids: List[int]) -> str:
        return self.sp.decode([i for i in ids if i not in (self.bos, self.eos, self.unk)])


def llava_prompt_ids(tokenizer) -> List[int]:
    return splice_image_token([tokenizer.encode(c) for c in LLAVA_PROMPT.split(IMAGE_TOKEN)], tokenizer.bos)


def load_llava_weights(weights_dir: str):
    """(state_dict, cfg, tokenizer directory) from the registry directories llava_v1.5_7b and clip_vit_l14_336."""
    import json
    from .. import arch
    from ..inference.pretrained_models import resolve
    model_dir = resolve("llava_v1.5_7b", weights_dir)
    with open(os.path.join(model_dir, "config.json"), encoding="utf-8") as f:
        config = json.load(f)
    sd = read_shards(model_dir)
    clip_sd, clip_config = None, None
    if not any(k.startswith("model.vision_tower.") for k in sd):
        clip_dir = resolve("clip_vit_l14_336", weights_dir)
        clip_sd = read_shards(clip_dir)
        conf = os.path.join(clip_dir, "config.json")
        if os.path.isfile(conf):
            with open(conf, encoding="utf-8") as f:
                clip_config = json.load(f)
    cfg = arch.llava_config(config, clip_config)
    return arch.llava_state_dict(sd, clip_sd, cfg), cfg, model_dir


def read_shards(directory: str) -> dict:
    """Every tensor of a Hugging Face checkpoint directory: *.safetensors or pytorch_model*.bin shards (an index
    file, if present, names them)."""
    import glob
    import json
    for index, kind in (("model.safetensors.index.json", "st"), ("pytorch_model.bin.index.json", "bin")):
        path = os.path.join(directory, index)
        if os.path.isfile(path):
            with open(path, encoding="utf-8") as f:
                files = sorted(set(json.load(f)["weight_map"].values()))
            files = [os.path.join(directory, n) for n in files]
            break
    else:
        files = sorted(glob.glob(os.path.join(directory, "*.safetensors")))
        kind = "st"
        if not files:
            files, kind = sorted(glob.glob(os.path.join(directory, "*.bin"))), "bin"
    if not files:
        raise FileNotFoundError(f"{directory}: no *.safetensors or *.bin checkpoint shards")
    sd = {}
    for path in files:
        if kind == "st":
            from safetensors.torch import load_file
            sd.update(load_file(path))
        else:
            sd.update(torch.load(path, map_location="cpu", weights_only=True))
    return sd


class LLaVACaptioner(Captioner):
    """LLaVA-1.5-7B with fp16 weights (--llava_bit 16) on engine.llava.LlavaEngine, greedy, at most 512 new tokens.
    The bitsandbytes 4-bit (NF4) and 8-bit (LLM.int8) variants are not built."""

    def __init__(self, device, llava_bit: str = "16", weights_dir: Optional[str] = None, synthetic: bool = False,
                 seed: int = 1234) -> None:
        super().__init__(device)
        if str(llava_bit) != "16":
            raise NotImplementedError(llava_bit_message(llava_bit))
        from .. import arch
        from ..engine.llava import LlavaEngine
        if synthetic:
            from .synth import synthetic_llava
            cfg = dict(arch.LLAVA_CFG)
            self.tokenizer = ByteTokenizer()
            sd = synthetic_llava(cfg, seed, device)
        else:
            from ..inference.pretrained_models import default_weights_dir
            sd, cfg, model_dir = load_llava_weights(weights_dir or default_weights_dir())
            self.tokenizer = SentencePieceTokenizer(model_dir)
        self.cfg = cfg
        self.prompt_ids = llava_prompt_ids(self.tokenizer)
        self.engine = LlavaEngine(sd, self.prompt_ids, cfg, device=device)
        del sd
        self.size = cfg["image"]

    @torch.no_grad()
    def __call__(self, image: Image.Image) -> str:
        ids = self.engine.generate(preprocess_llava(image, self.size).to(self.engine.dev))
        return self.tokenizer.decode(ids).strip()


def llava_bit_message(llava_bit) -> str:
    return (f"--captioner llava --llava_bit {llava_bit}: the bitsandbytes 4-/8-bit LLaVA is not built; pass "
            "--llava_bit 16 (fp16 weights, ~14 GB)")
