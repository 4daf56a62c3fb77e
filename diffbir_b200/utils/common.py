"""Host-side helpers with the reference's names and semantics (diffbir/utils/common.py):
sliding windows, Gaussian tile weights, wavelet colour fix, config instantiation."""
from __future__ import annotations

import importlib
from typing import Any, List, Mapping, Tuple

import numpy as np
import torch
import torch.nn.functional as F


def get_obj_from_str(string: str) -> Any:
    module, cls = string.rsplit(".", 1)
    if module == "diffbir.model" or module.startswith("diffbir.model."):
        module = "diffbir_b200.model"          # reference YAML targets resolve to this package
    return getattr(importlib.import_module(module), cls)


def instantiate_from_config(config: Mapping[str, Any], **extra) -> Any:
    """`target:` / `params:` reflection of utils/common.py:15-26 (same YAML files)."""
    if "target" not in config:
        raise KeyError("Expected key `target` to instantiate.")
    return get_obj_from_str(config["target"])(**config.get("params", dict()), **extra)


def sliding_windows(h: int, w: int, tile_size: int, tile_stride: int) -> List[Tuple[int, int, int, int]]:
    """Row-major windows; the last one is snapped to the border (utils/common.py:123-138)."""
    his = list(range(0, h - tile_size + 1, tile_stride))
    if (h - tile_size) % tile_stride != 0:
        his.append(h - tile_size)
    wis = list(range(0, w - tile_size + 1, tile_stride))
    if (w - tile_size) % tile_stride != 0:
        wis.append(w - tile_size)
    return [(hi, hi + tile_size, wi, wi + tile_size) for hi in his for wi in wis]


def gaussian_weights(tile_width: int, tile_height: int) -> np.ndarray:
    """Gaussian tile mask, var 0.01; x midpoint (W-1)/2, y midpoint H/2 — the asymmetry is the
    reference's (utils/common.py:142-169) and is kept."""
    var = 0.01
    xs, ys = np.arange(tile_width), np.arange(tile_height)
    xp = np.exp(-(xs - (tile_width - 1) / 2) ** 2 / (tile_width * tile_width) / (2 * var)) / np.sqrt(2 * np.pi * var)
    yp = np.exp(-(ys - tile_height / 2) ** 2 / (tile_height * tile_height) / (2 * var)) / np.sqrt(2 * np.pi * var)
    return np.outer(yp, xp)


def make_tiled_fn(fn, size: int, stride: int, scale_type: str = "up", scale: int = 1, channel=None,
                  weight: str = "gaussian", dtype=None, device=None, progress: bool = False, shard: bool = False):
    """Image-tiling wrapper of utils/common.py:172-232: the first argument is cut into row-major
    `size` x `size` windows (last one snapped to the border), `fn(tile) * w` and `w` are accumulated
    in that order, the result is `out / count`. Weights are built in fp64 and cast to the output
    dtype exactly like the reference; extra arguments get the window as hi/hi_end/wi/wi_end.

    shard: with a torch.distributed group of more than one rank, every rank passes the same input, runs
    the windows it owns (window t belongs to rank t % world), and one all-gather hands every rank all
    window outputs, which it blends in the order above: the result is bit-identical to one rank's. `fn`
    must return the output dtype."""
    def tiled_fn(x: torch.Tensor, *args, **kwargs) -> torch.Tensor:
        sc = (lambda n: int(n * scale)) if scale_type == "up" else (lambda n: int(n // scale))
        b, c, h, w = x.size()
        out_dtype, out_device = dtype or x.dtype, device or x.device
        out = torch.zeros((b, channel or c, sc(h), sc(w)), dtype=out_dtype, device=out_device)
        count = torch.zeros_like(out, dtype=torch.float32)
        ws = sc(size)
        wnp = gaussian_weights(ws, ws)[None, None] if weight == "gaussian" else np.ones((1, 1, ws, ws))
        weights = torch.tensor(wnp, dtype=out_dtype, device=out_device)
        wins = sliding_windows(h, w, size, stride)

        def run(t):
            hi, hi_end, wi, wi_end = wins[t]
            if len(args) or len(kwargs):
                kwargs.update(dict(hi=hi, hi_end=hi_end, wi=wi, wi_end=wi_end))
            return fn(x[..., hi:hi_end, wi:wi_end], *args, **kwargs)

        import torch.distributed as dist
        shared = None
        if shard and dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            from ..sampler.sampler import tile_slots, tiles_of_rank
            world, slots = dist.get_world_size(), tile_slots(len(wins), dist.get_world_size())
            send = torch.zeros((slots, b, channel or c, ws, ws), dtype=out_dtype, device=out_device)
            for s, t in enumerate(tiles_of_rank(len(wins), dist.get_rank(), world)):
                send[s] = run(t)
            # one buffer of every rank's slots (rank-major); ranks without a window still send their zero slots
            shared = torch.empty((world * slots,) + tuple(send.shape[1:]), dtype=out_dtype, device=out_device)
            dist.all_gather_into_tensor(shared, send)
            del send
        for t, (hi, hi_end, wi, wi_end) in enumerate(wins):
            oh, oh_end, ow, ow_end = map(sc, (hi, hi_end, wi, wi_end))
            y = run(t) if shared is None else shared[(t % world) * slots + t // world]     # window t: rank t % world
            out[..., oh:oh_end, ow:ow_end] += y * weights
            count[..., oh:oh_end, ow:ow_end] += weights
        return out / count

    return tiled_fn


def wavelet_blur(image: torch.Tensor, radius: int) -> torch.Tensor:
    k = torch.tensor([[0.0625, 0.125, 0.0625], [0.125, 0.25, 0.125], [0.0625, 0.125, 0.0625]],
                     dtype=image.dtype, device=image.device)[None, None].repeat(3, 1, 1, 1)
    image = F.pad(image, (radius, radius, radius, radius), mode="replicate")
    return F.conv2d(image, k, groups=3, dilation=radius)


def wavelet_decomposition(image: torch.Tensor, levels: int = 5):
    high = torch.zeros_like(image)
    low = image
    for i in range(levels):
        low = wavelet_blur(image, 2 ** i)
        high = high + (image - low)
        image = low
    return high, low


def wavelet_reconstruction(content_feat: torch.Tensor, style_feat: torch.Tensor) -> torch.Tensor:
    """High frequencies of the sample + low frequencies of the stage-1 image
    (utils/common.py:66-77)."""
    ch, _ = wavelet_decomposition(content_feat)
    _, sl = wavelet_decomposition(style_feat)
    return ch + sl


def load_file_from_url(url: str, model_dir=None, progress: bool = True, file_name=None) -> str:
    """utils/common.py:81-110 without the download: the file the URL names (or `file_name`) must already be in
    `model_dir` (default: $DIFFBIR_WEIGHTS_DIR or ./weights) — there is no network access on this path."""
    import os
    from urllib.parse import urlparse
    from ..inference.pretrained_models import default_weights_dir
    model_dir = default_weights_dir() if model_dir is None else model_dir
    path = os.path.abspath(os.path.join(model_dir, file_name or os.path.basename(urlparse(url).path)))
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} not found: place the file of {url} there (downloads are not performed)")
    return path


def load_model_from_url(url: str):
    """utils/common.py:113-120: the checkpoint behind a registry URL (or bare file name) as a flat state_dict
    (`state_dict` wrapper and `module.` prefix removed), read from the local weights directory."""
    from ..inference.loop import load_checkpoint
    return load_checkpoint(load_file_from_url(url))


class VRAMPeakMonitor:
    """utils/common.py:261-280: context manager around a loading / inference phase; prints the peak allocation when
    DIFFBIR_TRACE_VRAM=1 (the reference's TRACE_VRAM switch). Works without a CUDA device (then it does nothing)."""

    def __init__(self, tag: str) -> None:
        self.tag = tag

    def __enter__(self):
        self.peak_before = torch.cuda.max_memory_allocated() / 1024 ** 3 if torch.cuda.is_available() else 0.0
        return self

    def __exit__(self, exc_type, exc_value, traceback):
        import os
        if torch.cuda.is_available():
            torch.cuda.synchronize()
            if os.environ.get("DIFFBIR_TRACE_VRAM", "0") == "1":
                peak_after = torch.cuda.max_memory_allocated() / 1024 ** 3
                print(f"\033[93mVRAM peak before {self.tag}: {self.peak_before:.2f} GB, after: {peak_after:.2f} GB\033[0m")
        return False


def to(obj, device):
    """utils/common.py:310-319: moves the tensors of a nested dict / tuple / list."""
    if torch.is_tensor(obj):
        return obj.to(device)
    if isinstance(obj, dict):
        return {k: to(v, device) for k, v in obj.items()}
    if isinstance(obj, tuple):
        return tuple(to(v, device) for v in obj)
    if isinstance(obj, list):
        return [to(v, device) for v in obj]
    return obj
