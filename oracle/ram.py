"""ORACLE (test infrastructure): fp32 functional restatement of RAM++ tagging (reference ram/models/ram_plus.py
RAM_plus.generate_tag with vit="swin_l", image_size=384), driven by the reference's state_dict keys.

Swin-L (ram/models/swin_transformer.py): 4x4 patch embed + LN, four stages of Swin blocks (window 12, shift 6 on odd
blocks; stage 4's 12x12 map is one un-shifted window), PatchMerging between stages, final LN and the token mean as
the cls token; image_proj; the per-image reweighting of the 51 description embeddings per class; wordvec_proj +
ReLU; two BERT layers of cross-attention only (4 heads, post-LN eps 1e-12, GELU FFN); fc.

Pinned by tests/test_ram.py against tests/golden/ram_small.npz, generated from the reference module.
"""
from __future__ import annotations

from typing import Dict

import torch
import torch.nn.functional as F

from .swinir import swin_block

SD = Dict[str, torch.Tensor]
IMAGENET_MEAN = (0.485, 0.456, 0.406)       # ram/transform.py
IMAGENET_STD = (0.229, 0.224, 0.225)


def normalize(x01: torch.Tensor) -> torch.Tensor:
    """ToTensor() output in [0, 1] -> Normalize(ImageNet mean / std) (ram/transform.py)."""
    m = torch.tensor(IMAGENET_MEAN, dtype=x01.dtype, device=x01.device).view(1, 3, 1, 1)
    s = torch.tensor(IMAGENET_STD, dtype=x01.dtype, device=x01.device).view(1, 3, 1, 1)
    return (x01 - m) / s


def patch_merge(sd: SD, p: str, x: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """PatchMerging.forward — swin_transformer.py:310-331."""
    b, _, c = x.shape
    x = x.view(b, h, w, c)
    x = torch.cat([x[:, 0::2, 0::2], x[:, 1::2, 0::2], x[:, 0::2, 1::2], x[:, 1::2, 1::2]], -1).view(b, -1, 4 * c)
    x = F.layer_norm(x, (4 * c,), sd[p + "norm.weight"], sd[p + "norm.bias"], 1e-5)
    return F.linear(x, sd[p + "reduction.weight"])


def swin_l(sd: SD, x: torch.Tensor, stages=None) -> torch.Tensor:
    """SwinTransformer.forward (swin_transformer.py:562-576) on a normalised [B, 3, 384, 384] image ->
    [B, 145, 1536] = [token mean | normed stage-4 tokens]. stages (optional list) receives each stage's output."""
    from diffbir_b200.arch import RAM_CFG, ram_stages
    p = "visual_encoder."
    t = F.conv2d(x, sd[p + "patch_embed.proj.weight"], sd[p + "patch_embed.proj.bias"], stride=4)
    b, c, h, w = t.shape
    t = t.flatten(2).transpose(1, 2)
    t = F.layer_norm(t, (c,), sd[p + "patch_embed.norm.weight"], sd[p + "patch_embed.norm.bias"], 1e-5)
    plan = ram_stages(RAM_CFG)
    for i, (c, r, heads, ws, shifts) in enumerate(plan):
        for bi, shift in enumerate(shifts):
            t = swin_block(sd, f"{p}layers.{i}.blocks.{bi}.", t, r, r, ws, heads, shift)
        if stages is not None:
            stages.append(t)
        if i < len(plan) - 1:
            t = patch_merge(sd, f"{p}layers.{i}.downsample.", t, r, r)
    t = F.layer_norm(t, (t.shape[-1],), sd[p + "norm.weight"], sd[p + "norm.bias"], 1e-5)
    return torch.cat([t.mean(1, keepdim=True), t], 1)


def reweight(sd: SD, cls: torch.Tensor, per_class: int = 51) -> torch.Tensor:
    """generate_tag's description reweighting — ram_plus.py:293-307. cls [B, 512] -> [B, classes, 512]."""
    label = sd["label_embed"]
    cls = cls / cls.norm(dim=-1, keepdim=True)
    logits = (sd["reweight_scale"].exp() * cls @ label.t()).view(cls.shape[0], -1, per_class)
    p = F.softmax(logits, dim=2)
    return (p.unsqueeze(-1) * label.view(-1, per_class, label.shape[-1]).unsqueeze(0)).sum(2)


def tagging_head(sd: SD, q: torch.Tensor, kv: torch.Tensor, heads: int = 4, layers: int = 2) -> torch.Tensor:
    """BertModel(mode='tagging') without embeddings or self-attention (ram_plus.py:196-199, bert.py:376-458):
    per layer cross-attention (all-ones encoder mask) + post-LN, GELU FFN + post-LN, eps 1e-12."""
    b, n, hid = q.shape
    dh = hid // heads
    for l in range(layers):
        p = f"tagging_head.encoder.layer.{l}."
        a = p + "crossattention."
        qq = F.linear(q, sd[a + "self.query.weight"], sd[a + "self.query.bias"]).view(b, n, heads, dh).transpose(1, 2)
        kk = F.linear(kv, sd[a + "self.key.weight"], sd[a + "self.key.bias"]).view(b, -1, heads, dh).transpose(1, 2)
        vv = F.linear(kv, sd[a + "self.value.weight"], sd[a + "self.value.bias"]).view(b, -1, heads, dh).transpose(1, 2)
        att = torch.softmax(qq @ kk.transpose(-1, -2) / dh ** 0.5, dim=-1)
        ctx = (att @ vv).transpose(1, 2).reshape(b, n, hid)
        h1 = F.layer_norm(F.linear(ctx, sd[a + "output.dense.weight"], sd[a + "output.dense.bias"]) + q, (hid,),
                          sd[a + "output.LayerNorm.weight"], sd[a + "output.LayerNorm.bias"], 1e-12)
        f = F.gelu(F.linear(h1, sd[p + "intermediate.dense.weight"], sd[p + "intermediate.dense.bias"]))
        q = F.layer_norm(F.linear(f, sd[p + "output.dense.weight"], sd[p + "output.dense.bias"]) + h1, (hid,),
                         sd[p + "output.LayerNorm.weight"], sd[p + "output.LayerNorm.bias"], 1e-12)
    return q


def ram_forward(sd: SD, x: torch.Tensor, stages=None):
    """Normalised image [B, 3, 384, 384] -> (image_embeds [B, 145, 512], logits [B, classes])."""
    emb = F.linear(swin_l(sd, x, stages), sd["image_proj.weight"], sd["image_proj.bias"])
    label = F.relu(F.linear(reweight(sd, emb[:, 0]), sd["wordvec_proj.weight"], sd["wordvec_proj.bias"]))
    h = tagging_head(sd, label, emb)
    return emb, F.linear(h, sd["fc.weight"], sd["fc.bias"]).squeeze(-1)


def caption(logits: torch.Tensor, thresholds: torch.Tensor, tags) -> str:
    """generate_tag's decision + RAMCaptioner's join (ram_plus.py:322-336, diffbir/utils/caption.py:166-171)."""
    keep = (torch.sigmoid(logits.float()) > thresholds.float()).nonzero().flatten().tolist()
    return ", ".join(tags[i] for i in keep)
