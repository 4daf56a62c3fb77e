"""fp32 CPU restatement of the reference's LLaVA-1.5 captioner (utils/caption.py:52-145): CLIP ViT-L/14-336 up to
mm_vision_select_layer = -2 with the patch features, the mlp2x_gelu projector, the image features spliced in at the
-200 position, LLaMA (RMSNorm, rotate_half RoPE, causal attention with a KV cache, SwiGLU MLP) and greedy decoding.
Weights are an arch.llava_state_dict; pixel_values are CLIPImageProcessor's output."""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
import torch.nn.functional as F

V = "model.vision_tower.vision_tower.vision_model."


def _w(sd, k):
    return sd[k].float()


def vision_features(sd: dict, cfg: dict, pixel_values: torch.Tensor) -> torch.Tensor:
    """[1, 3, 336, 336] -> [576, v_width]: hidden_states[select_layer] without the class token."""
    vw, heads = cfg["v_width"], cfg["v_heads"]
    x = F.conv2d(pixel_values.float(), _w(sd, V + "embeddings.patch_embedding.weight"), stride=cfg["patch"])
    x = x.flatten(2).transpose(1, 2)[0]
    x = torch.cat([_w(sd, V + "embeddings.class_embedding")[None], x]) + _w(sd, V + "embeddings.position_embedding.weight")
    x = F.layer_norm(x, (vw,), _w(sd, V + "pre_layrnorm.weight"), _w(sd, V + "pre_layrnorm.bias"), cfg["v_eps"])
    n_run = cfg["v_layers"] + cfg["select_layer"] + 1
    for i in range(n_run):
        p = f"{V}encoder.layers.{i}."
        lin = lambda t, nm: F.linear(t, _w(sd, p + nm + ".weight"), _w(sd, p + nm + ".bias"))  # noqa: E731
        h = F.layer_norm(x, (vw,), _w(sd, p + "layer_norm1.weight"), _w(sd, p + "layer_norm1.bias"), cfg["v_eps"])
        q, k, v = (lin(h, f"self_attn.{n}_proj").view(-1, heads, vw // heads).transpose(0, 1) for n in "qkv")
        a = torch.softmax(q @ k.transpose(1, 2) * (vw // heads) ** -0.5, -1) @ v
        x = x + lin(a.transpose(0, 1).reshape(-1, vw), "self_attn.out_proj")
        h = F.layer_norm(x, (vw,), _w(sd, p + "layer_norm2.weight"), _w(sd, p + "layer_norm2.bias"), cfg["v_eps"])
        h = lin(h, "mlp.fc1")
        x = x + lin(h * torch.sigmoid(1.702 * h), "mlp.fc2")
    return x[1:]


def project(sd: dict, feats: torch.Tensor) -> torch.Tensor:
    h = F.gelu(F.linear(feats, _w(sd, "model.mm_projector.0.weight"), _w(sd, "model.mm_projector.0.bias")))
    return F.linear(h, _w(sd, "model.mm_projector.2.weight"), _w(sd, "model.mm_projector.2.bias"))


def splice(sd: dict, ids: List[int], image_features: torch.Tensor, image_index: int = -200) -> torch.Tensor:
    """prepare_inputs_labels_for_multimodal for one image: text embeddings with the features at the -200 slot."""
    i0 = ids.index(image_index)
    emb = _w(sd, "model.embed_tokens.weight")
    pre = emb[torch.tensor(ids[:i0], dtype=torch.long)]
    post = emb[torch.tensor(ids[i0 + 1:], dtype=torch.long)]
    return torch.cat([pre, image_features, post])


def _rms(x, w, eps):
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def _rope(x: torch.Tensor, pos: torch.Tensor, theta: float) -> torch.Tensor:
    """x [heads, n, 128] at positions pos [n]: rotate_half form."""
    d = x.shape[-1]
    inv = 1.0 / (theta ** (torch.arange(0, d, 2, device=x.device).float() / d))
    f = pos.float()[:, None] * inv[None]
    emb = torch.cat([f, f], -1)
    rot = torch.cat([-x[..., d // 2:], x[..., :d // 2]], -1)
    return x * emb.cos() + rot * emb.sin()


def llm_forward(sd: dict, cfg: dict, x: torch.Tensor, cache: Optional[list], pos0: int) -> Tuple[torch.Tensor, list]:
    """Embeddings x [n, hidden] at positions pos0 .. pos0+n-1 with a KV cache (list of (k, v) per layer, [heads, t,
    128]) -> (logits [n, vocab], the extended cache)."""
    heads, hd, eps = cfg["heads"], cfg["hidden"] // cfg["heads"], cfg["rms_eps"]
    n = x.shape[0]
    pos = torch.arange(pos0, pos0 + n, device=x.device)
    cache = cache if cache is not None else [None] * cfg["layers"]
    out_cache = []
    for i in range(cfg["layers"]):
        p = f"model.layers.{i}."
        h = _rms(x, _w(sd, p + "input_layernorm.weight"), eps)
        q, k, v = (F.linear(h, _w(sd, p + f"self_attn.{m}_proj.weight")).view(n, heads, hd).transpose(0, 1) for m in "qkv")
        q, k = _rope(q, pos, cfg["rope_theta"]), _rope(k, pos, cfg["rope_theta"])
        if cache[i] is not None:
            k, v = torch.cat([cache[i][0], k], 1), torch.cat([cache[i][1], v], 1)
        out_cache.append((k, v))
        t = k.shape[1]
        s = q @ k.transpose(1, 2) / math.sqrt(hd)
        keypos = torch.arange(t, device=x.device)
        s = s.masked_fill(keypos[None, None, :] > pos[None, :, None], float("-inf"))
        a = (torch.softmax(s, -1) @ v).transpose(0, 1).reshape(n, -1)
        x = x + F.linear(a, _w(sd, p + "self_attn.o_proj.weight"))
        h = _rms(x, _w(sd, p + "post_attention_layernorm.weight"), eps)
        g = F.linear(h, _w(sd, p + "mlp.gate_proj.weight"))
        u = F.linear(h, _w(sd, p + "mlp.up_proj.weight"))
        x = x + F.linear(F.silu(g) * u, _w(sd, p + "mlp.down_proj.weight"))
    x = _rms(x, _w(sd, "model.norm.weight"), eps)
    return F.linear(x, _w(sd, "lm_head.weight")), out_cache


@torch.no_grad()
def greedy(sd: dict, cfg: dict, pixel_values: torch.Tensor, ids: List[int], max_new: int,
           forced: Optional[List[int]] = None):
    """Greedy decoding (temperature 0, one beam) with a KV cache, stopping after EOS or max_new tokens. forced: feed
    these tokens instead of the argmax (teacher forcing). -> (tokens, logits [steps, vocab], image features)."""
    feats = project(sd, vision_features(sd, cfg, pixel_values))
    x = splice(sd, ids, feats)
    logits, cache = llm_forward(sd, cfg, x, None, 0)
    pos = x.shape[0]
    rows, toks = [logits[-1]], []
    while True:
        t = int(rows[-1].argmax()) if forced is None else int(forced[len(toks)])
        toks.append(t)
        if len(toks) >= max_new or (forced is None and t == cfg["eos"]):
            break
        step, cache = llm_forward(sd, cfg, _w(sd, "model.embed_tokens.weight")[t][None], cache, pos)
        pos += 1
        rows.append(step[-1])
    return toks, torch.stack(rows), feats
