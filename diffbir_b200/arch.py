"""Architecture descriptions: block plans and parameter shapes, in the reference's state_dict
key layout, derived from the reference's YAML configs (configs/inference/*.yaml).

The block plan is what the engine walks to enqueue kernels; the shape tables drive the
synthetic-checkpoint generator (bench / tests use random-init weights of the real
architecture) and the strict checkpoint loaders.  Mirrors the constructor logic of
UNetModel (model/unet.py:412-682), ControlNet (model/controlnet.py:52-312),
Encoder/Decoder (model/vae.py:306-345, 456-524), SwinIR (model/swinir.py:648-812) and the
OpenCLIP text tower (model/open_clip/transformer.py).
"""
from __future__ import annotations

from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

Shapes = "OrderedDict[str, Tuple[int, ...]]"

UNET_CFG = dict(in_channels=4, out_channels=4, model_channels=320, attention_resolutions=(4, 2, 1),
                num_res_blocks=2, channel_mult=(1, 2, 4, 4), num_head_channels=64,
                transformer_depth=1, context_dim=1024)
CONTROLNET_CFG = dict(UNET_CFG, hint_channels=4)
VAE_CFG = dict(embed_dim=4, z_channels=4, in_channels=3, out_ch=3, ch=128, ch_mult=(1, 2, 4, 4),
               num_res_blocks=2)
SWINIR_CFG = dict(img_size=64, in_chans=3, embed_dim=180, depths=(6,) * 8, num_heads=(6,) * 8,
                  window_size=8, mlp_ratio=2, sf=8, img_range=1.0, unshuffle_scale=8, num_feat=64)
CLIP_TEXT_CFG = dict(context_length=77, vocab_size=49408, width=1024, heads=16, layers=24,
                     embed_dim=1024)


# ------------------------------------------------------------------------------- UNet plan
@dataclass
class Layer:
    kind: str                 # conv_in | res | attn | down | up
    prefix: str               # state_dict prefix, ends with '.'
    cin: int
    cout: int


@dataclass
class Block:
    prefix: str
    layers: List[Layer] = field(default_factory=list)
    cout: int = 0


@dataclass
class UNetPlan:
    cfg: dict
    input_blocks: List[Block]
    middle: Block
    output_blocks: List[Block]            # empty for ControlNet
    skip_channels: List[int]              # channels of hs[i] (== zero-conv widths, + middle)
    is_controlnet: bool


def unet_plan(cfg: dict, controlnet: bool = False) -> UNetPlan:
    mc = cfg["model_channels"]
    mult = tuple(cfg["channel_mult"])
    nres = cfg["num_res_blocks"]
    attn_res = tuple(cfg["attention_resolutions"])
    in_ch = cfg["in_channels"] + (cfg.get("hint_channels", 0) if controlnet else 0)
    blocks = [Block("input_blocks.0.", [Layer("conv_in", "input_blocks.0.0.", in_ch, mc)], mc)]
    chans = [mc]
    ch, ds = mc, 1
    for level, m in enumerate(mult):
        for _ in range(nres):
            i = len(blocks)
            p = f"input_blocks.{i}."
            layers = [Layer("res", p + "0.", ch, m * mc)]
            ch = m * mc
            if ds in attn_res:
                layers.append(Layer("attn", p + "1.", ch, ch))
            blocks.append(Block(p, layers, ch))
            chans.append(ch)
        if level != len(mult) - 1:
            i = len(blocks)
            p = f"input_blocks.{i}."
            blocks.append(Block(p, [Layer("down", p + "0.", ch, ch)], ch))
            chans.append(ch)
            ds *= 2
    middle = Block("middle_block.", [Layer("res", "middle_block.0.", ch, ch),
                                     Layer("attn", "middle_block.1.", ch, ch),
                                     Layer("res", "middle_block.2.", ch, ch)], ch)
    skip_channels = list(chans) + [ch]
    outs: List[Block] = []
    if not controlnet:
        stack = list(chans)
        for level, m in list(enumerate(mult))[::-1]:
            for i in range(nres + 1):
                ich = stack.pop()
                k = len(outs)
                p = f"output_blocks.{k}."
                layers = [Layer("res", p + "0.", ch + ich, mc * m)]
                ch = mc * m
                if ds in attn_res:
                    layers.append(Layer("attn", p + f"{len(layers)}.", ch, ch))
                if level and i == nres:
                    layers.append(Layer("up", p + f"{len(layers)}.", ch, ch))
                    ds //= 2
                outs.append(Block(p, layers, ch))
    return UNetPlan(cfg, blocks, middle, outs, skip_channels, controlnet)


def _res_shapes(s: Shapes, p: str, cin: int, cout: int, emb: int):
    s[p + "in_layers.0.weight"] = (cin,)
    s[p + "in_layers.0.bias"] = (cin,)
    s[p + "in_layers.2.weight"] = (cout, cin, 3, 3)
    s[p + "in_layers.2.bias"] = (cout,)
    s[p + "emb_layers.1.weight"] = (cout, emb)
    s[p + "emb_layers.1.bias"] = (cout,)
    s[p + "out_layers.0.weight"] = (cout,)
    s[p + "out_layers.0.bias"] = (cout,)
    s[p + "out_layers.3.weight"] = (cout, cout, 3, 3)
    s[p + "out_layers.3.bias"] = (cout,)
    if cin != cout:
        s[p + "skip_connection.weight"] = (cout, cin, 1, 1)
        s[p + "skip_connection.bias"] = (cout,)


def _attn_shapes(s: Shapes, p: str, c: int, ctx: int, depth: int):
    s[p + "norm.weight"] = (c,)
    s[p + "norm.bias"] = (c,)
    s[p + "proj_in.weight"] = (c, c)
    s[p + "proj_in.bias"] = (c,)
    for d in range(depth):
        q = f"{p}transformer_blocks.{d}."
        s[q + "attn1.to_q.weight"] = (c, c)
        s[q + "attn1.to_k.weight"] = (c, c)
        s[q + "attn1.to_v.weight"] = (c, c)
        s[q + "attn1.to_out.0.weight"] = (c, c)
        s[q + "attn1.to_out.0.bias"] = (c,)
        s[q + "ff.net.0.proj.weight"] = (8 * c, c)
        s[q + "ff.net.0.proj.bias"] = (8 * c,)
        s[q + "ff.net.2.weight"] = (c, 4 * c)
        s[q + "ff.net.2.bias"] = (c,)
        s[q + "attn2.to_q.weight"] = (c, c)
        s[q + "attn2.to_k.weight"] = (c, ctx)
        s[q + "attn2.to_v.weight"] = (c, ctx)
        s[q + "attn2.to_out.0.weight"] = (c, c)
        s[q + "attn2.to_out.0.bias"] = (c,)
        for nm in ("norm1", "norm2", "norm3"):
            s[q + nm + ".weight"] = (c,)
            s[q + nm + ".bias"] = (c,)
    s[p + "proj_out.weight"] = (c, c)
    s[p + "proj_out.bias"] = (c,)


def unet_shapes(cfg: dict, controlnet: bool = False) -> Shapes:
    plan = unet_plan(cfg, controlnet)
    mc, emb = cfg["model_channels"], cfg["model_channels"] * 4
    ctx, depth = cfg["context_dim"], cfg.get("transformer_depth", 1)
    s: Shapes = OrderedDict()
    s["time_embed.0.weight"] = (emb, mc)
    s["time_embed.0.bias"] = (emb,)
    s["time_embed.2.weight"] = (emb, emb)
    s["time_embed.2.bias"] = (emb,)

    def add(block: Block):
        for l in block.layers:
            if l.kind == "conv_in":
                s[l.prefix + "weight"] = (l.cout, l.cin, 3, 3)
                s[l.prefix + "bias"] = (l.cout,)
            elif l.kind == "res":
                _res_shapes(s, l.prefix, l.cin, l.cout, emb)
            elif l.kind == "attn":
                _attn_shapes(s, l.prefix, l.cin, ctx, depth)
            elif l.kind == "down":
                s[l.prefix + "op.weight"] = (l.cout, l.cin, 3, 3)
                s[l.prefix + "op.bias"] = (l.cout,)
            elif l.kind == "up":
                s[l.prefix + "conv.weight"] = (l.cout, l.cin, 3, 3)
                s[l.prefix + "conv.bias"] = (l.cout,)

    for i, b in enumerate(plan.input_blocks):
        add(b)
        if controlnet:
            s[f"zero_convs.{i}.0.weight"] = (b.cout, b.cout, 1, 1)
            s[f"zero_convs.{i}.0.bias"] = (b.cout,)
    add(plan.middle)
    if controlnet:
        s["middle_block_out.0.weight"] = (plan.middle.cout, plan.middle.cout, 1, 1)
        s["middle_block_out.0.bias"] = (plan.middle.cout,)
    else:
        for b in plan.output_blocks:
            add(b)
        s["out.0.weight"] = (mc,)
        s["out.0.bias"] = (mc,)
        s["out.2.weight"] = (cfg["out_channels"], mc, 3, 3)
        s["out.2.bias"] = (cfg["out_channels"],)
    return s


# Tensors the reference constructors zero-initialise (zero_module): re-randomised in synthetic
# checkpoints so parity checks are not vacuous (SURVEY.md headline fact 5).
def is_zero_init(key: str) -> bool:
    return (".out_layers.3." in key or ".proj_out." in key or key.startswith("out.2.")
            or key.startswith("zero_convs.") or key.startswith("middle_block_out."))


# ------------------------------------------------------------------------------- VAE
def _vae_res(s: Shapes, p: str, cin: int, cout: int):
    s[p + "norm1.weight"] = (cin,)
    s[p + "norm1.bias"] = (cin,)
    s[p + "conv1.weight"] = (cout, cin, 3, 3)
    s[p + "conv1.bias"] = (cout,)
    s[p + "norm2.weight"] = (cout,)
    s[p + "norm2.bias"] = (cout,)
    s[p + "conv2.weight"] = (cout, cout, 3, 3)
    s[p + "conv2.bias"] = (cout,)
    if cin != cout:
        s[p + "nin_shortcut.weight"] = (cout, cin, 1, 1)
        s[p + "nin_shortcut.bias"] = (cout,)


def _vae_attn(s: Shapes, p: str, c: int):
    s[p + "norm.weight"] = (c,)
    s[p + "norm.bias"] = (c,)
    for nm in ("q", "k", "v", "proj_out"):
        s[p + nm + ".weight"] = (c, c, 1, 1)
        s[p + nm + ".bias"] = (c,)


def vae_shapes(cfg: dict) -> Shapes:
    ch, mult, nres = cfg["ch"], tuple(cfg["ch_mult"]), cfg["num_res_blocks"]
    z = cfg["z_channels"]
    s: Shapes = OrderedDict()
    # encoder
    p = "encoder."
    s[p + "conv_in.weight"] = (ch, cfg["in_channels"], 3, 3)
    s[p + "conv_in.bias"] = (ch,)
    in_mult = (1,) + mult
    block_in = ch
    for lvl in range(len(mult)):
        block_in = ch * in_mult[lvl]
        block_out = ch * mult[lvl]
        for j in range(nres):
            _vae_res(s, f"{p}down.{lvl}.block.{j}.", block_in, block_out)
            block_in = block_out
        if lvl != len(mult) - 1:
            s[f"{p}down.{lvl}.downsample.conv.weight"] = (block_in, block_in, 3, 3)
            s[f"{p}down.{lvl}.downsample.conv.bias"] = (block_in,)
    _vae_res(s, p + "mid.block_1.", block_in, block_in)
    _vae_attn(s, p + "mid.attn_1.", block_in)
    _vae_res(s, p + "mid.block_2.", block_in, block_in)
    s[p + "norm_out.weight"] = (block_in,)
    s[p + "norm_out.bias"] = (block_in,)
    s[p + "conv_out.weight"] = (2 * z, block_in, 3, 3)
    s[p + "conv_out.bias"] = (2 * z,)
    # decoder
    p = "decoder."
    block_in = ch * mult[-1]
    s[p + "conv_in.weight"] = (block_in, z, 3, 3)
    s[p + "conv_in.bias"] = (block_in,)
    _vae_res(s, p + "mid.block_1.", block_in, block_in)
    _vae_attn(s, p + "mid.attn_1.", block_in)
    _vae_res(s, p + "mid.block_2.", block_in, block_in)
    for lvl in reversed(range(len(mult))):
        block_out = ch * mult[lvl]
        for j in range(nres + 1):
            _vae_res(s, f"{p}up.{lvl}.block.{j}.", block_in, block_out)
            block_in = block_out
        if lvl != 0:
            s[f"{p}up.{lvl}.upsample.conv.weight"] = (block_in, block_in, 3, 3)
            s[f"{p}up.{lvl}.upsample.conv.bias"] = (block_in,)
    s[p + "norm_out.weight"] = (block_in,)
    s[p + "norm_out.bias"] = (block_in,)
    s[p + "conv_out.weight"] = (cfg["out_ch"], block_in, 3, 3)
    s[p + "conv_out.bias"] = (cfg["out_ch"],)
    s["quant_conv.weight"] = (2 * cfg["embed_dim"], 2 * z, 1, 1)
    s["quant_conv.bias"] = (2 * cfg["embed_dim"],)
    s["post_quant_conv.weight"] = (z, cfg["embed_dim"], 1, 1)
    s["post_quant_conv.bias"] = (z,)
    return s


# ------------------------------------------------------------------------------- SwinIR
def swinir_shapes(cfg: dict) -> Shapes:
    """Parameters only; the reference state_dict additionally carries the int64
    relative_position_index and fp32 attn_mask buffers (see swinir_buffers)."""
    c, ws = cfg["embed_dim"], cfg["window_size"]
    nf = cfg.get("num_feat", 64)
    hidden = int(c * cfg["mlp_ratio"])
    in_ch = cfg["in_chans"] * cfg["unshuffle_scale"] ** 2
    s: Shapes = OrderedDict()
    s["conv_first.1.weight"] = (c, in_ch, 3, 3)
    s["conv_first.1.bias"] = (c,)
    s["patch_embed.norm.weight"] = (c,)
    s["patch_embed.norm.bias"] = (c,)
    for li, depth in enumerate(cfg["depths"]):
        heads = cfg["num_heads"][li]
        for bi in range(depth):
            p = f"layers.{li}.residual_group.blocks.{bi}."
            s[p + "norm1.weight"] = (c,)
            s[p + "norm1.bias"] = (c,)
            s[p + "attn.relative_position_bias_table"] = ((2 * ws - 1) ** 2, heads)
            s[p + "attn.qkv.weight"] = (3 * c, c)
            s[p + "attn.qkv.bias"] = (3 * c,)
            s[p + "attn.proj.weight"] = (c, c)
            s[p + "attn.proj.bias"] = (c,)
            s[p + "norm2.weight"] = (c,)
            s[p + "norm2.bias"] = (c,)
            s[p + "mlp.fc1.weight"] = (hidden, c)
            s[p + "mlp.fc1.bias"] = (hidden,)
            s[p + "mlp.fc2.weight"] = (c, hidden)
            s[p + "mlp.fc2.bias"] = (c,)
        s[f"layers.{li}.conv.weight"] = (c, c, 3, 3)
        s[f"layers.{li}.conv.bias"] = (c,)
    s["norm.weight"] = (c,)
    s["norm.bias"] = (c,)
    s["conv_after_body.weight"] = (c, c, 3, 3)
    s["conv_after_body.bias"] = (c,)
    s["conv_before_upsample.0.weight"] = (nf, c, 3, 3)
    s["conv_before_upsample.0.bias"] = (nf,)
    ups = {2: 1, 4: 2, 8: 3}[cfg["sf"]]
    for i in range(1, ups + 1):
        s[f"conv_up{i}.weight"] = (nf, nf, 3, 3)
        s[f"conv_up{i}.bias"] = (nf,)
    s["conv_hr.weight"] = (nf, nf, 3, 3)
    s["conv_hr.bias"] = (nf,)
    s["conv_last.weight"] = (cfg["in_chans"], nf, 3, 3)
    s["conv_last.bias"] = (cfg["in_chans"],)
    return s


# ------------------------------------------------------------------------------- CLIP text
def clip_text_shapes(cfg: dict) -> Shapes:
    w = cfg["width"]
    s: Shapes = OrderedDict()
    s["positional_embedding"] = (cfg["context_length"], w)
    s["text_projection"] = (w, cfg["embed_dim"])
    s["logit_scale"] = ()
    for i in range(cfg["layers"]):
        p = f"transformer.resblocks.{i}."
        s[p + "ln_1.weight"] = (w,)
        s[p + "ln_1.bias"] = (w,)
        s[p + "attn.in_proj_weight"] = (3 * w, w)
        s[p + "attn.in_proj_bias"] = (3 * w,)
        s[p + "attn.out_proj.weight"] = (w, w)
        s[p + "attn.out_proj.bias"] = (w,)
        s[p + "ln_2.weight"] = (w,)
        s[p + "ln_2.bias"] = (w,)
        s[p + "mlp.c_fc.weight"] = (4 * w, w)
        s[p + "mlp.c_fc.bias"] = (4 * w,)
        s[p + "mlp.c_proj.weight"] = (w, 4 * w)
        s[p + "mlp.c_proj.bias"] = (w,)
    s["token_embedding.weight"] = (cfg["vocab_size"], w)
    s["ln_final.weight"] = (w,)
    s["ln_final.bias"] = (w,)
    return s


# ------------------------------------------------------------------------------- RRDBNet (BSRNet)
RRDBNET_CFG = dict(in_nc=3, out_nc=3, nf=64, nb=23, gc=32, sf=4)      # configs/inference/bsrnet.yaml


def rrdbnet_shapes(cfg: dict) -> Shapes:
    """state_dict of the reference's RRDBNet (model/bsrnet.py:36-104): conv_first, nb x RRDB of three
    5-conv dense blocks, trunk_conv, upconv1 (+ upconv2 when sf == 4), HRconv, conv_last."""
    nf, gc = cfg["nf"], cfg["gc"]
    s: Shapes = OrderedDict()
    s["conv_first.weight"] = (nf, cfg["in_nc"], 3, 3)
    s["conv_first.bias"] = (nf,)
    for b in range(cfg["nb"]):
        for r in (1, 2, 3):
            p = f"RRDB_trunk.{b}.RDB{r}."
            for k in range(1, 5):
                s[p + f"conv{k}.weight"] = (gc, nf + (k - 1) * gc, 3, 3)
                s[p + f"conv{k}.bias"] = (gc,)
            s[p + "conv5.weight"] = (nf, nf + 4 * gc, 3, 3)
            s[p + "conv5.bias"] = (nf,)
    names = ["trunk_conv", "upconv1"] + (["upconv2"] if cfg["sf"] == 4 else []) + ["HRconv"]
    for nm in names:
        s[nm + ".weight"] = (nf, nf, 3, 3)
        s[nm + ".bias"] = (nf,)
    s["conv_last.weight"] = (cfg["out_nc"], nf, 3, 3)
    s["conv_last.bias"] = (cfg["out_nc"],)
    return s


# ------------------------------------------------------------------------------- SCUNet
SCUNET_CFG = dict(in_nc=3, config=(4, 4, 4, 4, 4, 4, 4), dim=64)       # configs/inference/scunet.yaml


def scunet_stages(cfg: dict):
    """(module name, channels = conv_dim + trans_dim, number of ConvTransBlocks, first index inside the module)
    for the seven stages of SCUNet (model/scunet.py:176-212); the up stages start with their ConvTranspose2d."""
    d, n = cfg["dim"], cfg["config"]
    return [("m_down1", d, n[0], 0), ("m_down2", 2 * d, n[1], 0), ("m_down3", 4 * d, n[2], 0), ("m_body", 8 * d, n[3], 0),
            ("m_up3", 4 * d, n[4], 1), ("m_up2", 2 * d, n[5], 1), ("m_up1", d, n[6], 1)]


def scunet_shapes(cfg: dict) -> Shapes:
    """state_dict of the reference's SCUNet (model/scunet.py:163-219)."""
    d = cfg["dim"]
    s: Shapes = OrderedDict()
    s["m_head.0.weight"] = (d, cfg["in_nc"], 3, 3)
    for name, c, nblk, first in scunet_stages(cfg):
        if first:                                                  # ConvTranspose2d(2c -> c, 2, 2): [Cin, Cout, 2, 2]
            s[f"{name}.0.weight"] = (2 * c, c, 2, 2)
        t = c // 2                                                 # conv_dim == trans_dim
        for i in range(nblk):
            p = f"{name}.{first + i}."
            s[p + "trans_block.ln1.weight"] = (t,)
            s[p + "trans_block.ln1.bias"] = (t,)
            s[p + "trans_block.msa.relative_position_params"] = (t // 32, 15, 15)
            s[p + "trans_block.msa.embedding_layer.weight"] = (3 * t, t)
            s[p + "trans_block.msa.embedding_layer.bias"] = (3 * t,)
            s[p + "trans_block.msa.linear.weight"] = (t, t)
            s[p + "trans_block.msa.linear.bias"] = (t,)
            s[p + "trans_block.ln2.weight"] = (t,)
            s[p + "trans_block.ln2.bias"] = (t,)
            s[p + "trans_block.mlp.0.weight"] = (4 * t, t)
            s[p + "trans_block.mlp.0.bias"] = (4 * t,)
            s[p + "trans_block.mlp.2.weight"] = (t, 4 * t)
            s[p + "trans_block.mlp.2.bias"] = (t,)
            s[p + "conv1_1.weight"] = (c, c, 1, 1)
            s[p + "conv1_1.bias"] = (c,)
            s[p + "conv1_2.weight"] = (c, c, 1, 1)
            s[p + "conv1_2.bias"] = (c,)
            s[p + "conv_block.0.weight"] = (t, t, 3, 3)
            s[p + "conv_block.2.weight"] = (t, t, 3, 3)
        if name.startswith("m_down"):                              # Conv2d(c -> 2c, 2, 2)
            s[f"{name}.{nblk}.weight"] = (2 * c, c, 2, 2)
    s["m_tail.0.weight"] = (cfg["in_nc"], d, 3, 3)
    return s


# ------------------------------------------------------------------------------- RAM++ (captioner)
# RAM_plus(image_size=384, vit="swin_l") (ram/models/ram_plus.py:90-179): Swin-L at 384^2 (configs/swin/
# config_swinL_384.json), the 2-layer cross-attention-only BERT tagging head (configs/q2l_config.json,
# encoder_width 512) and 4585 classes x 51 description embeddings.
RAM_CFG = dict(img_size=384, patch_size=4, embed_dim=192, depths=(2, 2, 18, 2), num_heads=(6, 12, 24, 48),
               window_size=12, mlp_ratio=4, vision_width=1536, embed=512, hidden=768, bert_heads=4,
               intermediate=3072, bert_layers=2, num_class=4585, des_per_class=51)


def ram_stages(cfg: dict):
    """(channels, token-map side, heads, window, block shifts) per Swin stage. A stage whose map is no larger than
    the window runs one un-shifted window of the map's size (swin_transformer.py:195-198)."""
    out = []
    side = cfg["img_size"] // cfg["patch_size"]
    for i, (depth, heads) in enumerate(zip(cfg["depths"], cfg["num_heads"])):
        r = side >> i
        ws, shift = cfg["window_size"], cfg["window_size"] // 2
        if r <= ws:
            ws, shift = r, 0
        out.append((cfg["embed_dim"] << i, r, heads, ws, tuple(0 if b % 2 == 0 else shift for b in range(depth))))
    return out


def ram_shapes(cfg: dict) -> Shapes:
    """Parameters of RAM_plus in its state_dict order, without the relative_position_index / attn_mask buffers
    the checkpoint loader drops (ram/models/utils.py:241-270)."""
    s: Shapes = OrderedDict()
    e, hid, inter = cfg["embed"], cfg["hidden"], cfg["intermediate"]
    s["label_embed"] = (cfg["num_class"] * cfg["des_per_class"], e)
    s["reweight_scale"] = ()
    c0, p = cfg["embed_dim"], "visual_encoder."
    s[p + "patch_embed.proj.weight"] = (c0, 3, cfg["patch_size"], cfg["patch_size"])
    s[p + "patch_embed.proj.bias"] = (c0,)
    s[p + "patch_embed.norm.weight"] = (c0,)
    s[p + "patch_embed.norm.bias"] = (c0,)
    stages = ram_stages(cfg)
    for i, (c, _, heads, ws, shifts) in enumerate(stages):
        for b in range(len(shifts)):
            q = f"{p}layers.{i}.blocks.{b}."
            s[q + "norm1.weight"] = (c,)
            s[q + "norm1.bias"] = (c,)
            s[q + "attn.relative_position_bias_table"] = ((2 * ws - 1) ** 2, heads)
            s[q + "attn.qkv.weight"] = (3 * c, c)
            s[q + "attn.qkv.bias"] = (3 * c,)
            s[q + "attn.proj.weight"] = (c, c)
            s[q + "attn.proj.bias"] = (c,)
            s[q + "norm2.weight"] = (c,)
            s[q + "norm2.bias"] = (c,)
            s[q + "mlp.fc1.weight"] = (cfg["mlp_ratio"] * c, c)
            s[q + "mlp.fc1.bias"] = (cfg["mlp_ratio"] * c,)
            s[q + "mlp.fc2.weight"] = (c, cfg["mlp_ratio"] * c)
            s[q + "mlp.fc2.bias"] = (c,)
        if i < len(stages) - 1:
            s[f"{p}layers.{i}.downsample.reduction.weight"] = (2 * c, 4 * c)
            s[f"{p}layers.{i}.downsample.norm.weight"] = (4 * c,)
            s[f"{p}layers.{i}.downsample.norm.bias"] = (4 * c,)
    s[p + "norm.weight"] = (cfg["vision_width"],)
    s[p + "norm.bias"] = (cfg["vision_width"],)
    for l in range(cfg["bert_layers"]):
        q = f"tagging_head.encoder.layer.{l}."
        s[q + "crossattention.self.query.weight"] = (hid, hid)
        s[q + "crossattention.self.query.bias"] = (hid,)
        s[q + "crossattention.self.key.weight"] = (hid, e)
        s[q + "crossattention.self.key.bias"] = (hid,)
        s[q + "crossattention.self.value.weight"] = (hid, e)
        s[q + "crossattention.self.value.bias"] = (hid,)
        s[q + "crossattention.output.dense.weight"] = (hid, hid)
        s[q + "crossattention.output.dense.bias"] = (hid,)
        s[q + "crossattention.output.LayerNorm.weight"] = (hid,)
        s[q + "crossattention.output.LayerNorm.bias"] = (hid,)
        s[q + "intermediate.dense.weight"] = (inter, hid)
        s[q + "intermediate.dense.bias"] = (inter,)
        s[q + "output.dense.weight"] = (hid, inter)
        s[q + "output.dense.bias"] = (hid,)
        s[q + "output.LayerNorm.weight"] = (hid,)
        s[q + "output.LayerNorm.bias"] = (hid,)
    s["wordvec_proj.weight"] = (hid, e)
    s["wordvec_proj.bias"] = (hid,)
    s["fc.weight"] = (1, hid)
    s["fc.bias"] = (1,)
    s["image_proj.weight"] = (e, cfg["vision_width"])
    s["image_proj.bias"] = (e,)
    return s


def ram_state_dict(ckpt: dict, cfg: dict = None) -> dict:
    """The strict RAM++ loader: unwraps the checkpoint's `model` entry, drops the relative_position_index / attn_mask
    buffers and renames vision_multi -> tagging_head as ram/models/utils.py:241-270 does, then checks every key and
    shape of ram_shapes. A relative-position bias table of another window size is refused (the reference would
    interpolate it; the Swin-L checkpoint already holds 23^2-row tables)."""
    cfg = RAM_CFG if cfg is None else cfg
    sd = ckpt["model"] if "model" in ckpt else ckpt
    sd = {k.replace("vision_multi", "tagging_head"): v for k, v in sd.items()
          if "relative_position_index" not in k and "attn_mask" not in k}
    rows = (2 * cfg["window_size"] - 1) ** 2
    for k, v in sd.items():
        if k.endswith("relative_position_bias_table") and v.shape[0] != rows:
            raise ValueError(f"{k}: {v.shape[0]} rows, expected {rows} ((2 * {cfg['window_size']} - 1)^2); "
                             "relative-position tables of other window sizes are not interpolated")
    from .engine.common import check_shapes          # imported here: this module needs neither torch nor the library
    check_shapes(sd, ram_shapes(cfg), "RAM++")
    return sd


# ---- face detector and face parser of the unaligned-face loop (facexlib 0.3 key layout) --------------------------
RETINAFACE_CFG = dict(min_sizes=((16, 32), (64, 128), (256, 512)), steps=(8, 16, 32), variance=(0.1, 0.2),
                      in_channel=256, out_channel=256, layers=(3, 4, 6, 3))
PARSENET_CFG = dict(in_size=512, base_ch=64, min_feat_size=32, res_depth=10, parsing_ch=19, ch_range=(32, 256))
BN_EPS = 1e-5


def _bn(s: Shapes, p: str, c: int):
    for nm in ("weight", "bias", "running_mean", "running_var"):
        s[f"{p}.{nm}"] = (c,)


def retinaface_shapes(cfg: dict = None) -> Shapes:
    """RetinaFace(cfg_re50): `body.*` = torchvision resnet50 up to layer4 (stride on conv2), `fpn.output{1,2,3}` 1x1 and
    `fpn.merge{1,2}` 3x3 conv + BN, `ssh{1,2,3}` conv + BN branches, then the per-level 1x1 heads."""
    cfg = RETINAFACE_CFG if cfg is None else cfg
    s = OrderedDict()
    s["body.conv1.weight"] = (64, 3, 7, 7)
    _bn(s, "body.bn1", 64)
    cin = 64
    for li, blocks in enumerate(cfg["layers"]):
        w = 64 << li
        for b in range(blocks):
            p = f"body.layer{li + 1}.{b}."
            s[p + "conv1.weight"] = (w, cin, 1, 1)
            _bn(s, p + "bn1", w)
            s[p + "conv2.weight"] = (w, w, 3, 3)
            _bn(s, p + "bn2", w)
            s[p + "conv3.weight"] = (4 * w, w, 1, 1)
            _bn(s, p + "bn3", 4 * w)
            if b == 0:
                s[p + "downsample.0.weight"] = (4 * w, cin, 1, 1)
                _bn(s, p + "downsample.1", 4 * w)
            cin = 4 * w
    ic, oc = cfg["in_channel"], cfg["out_channel"]
    for i, c in enumerate((2 * ic, 4 * ic, 8 * ic)):
        s[f"fpn.output{i + 1}.0.weight"] = (oc, c, 1, 1)
        _bn(s, f"fpn.output{i + 1}.1", oc)
    for i in (1, 2):
        s[f"fpn.merge{i}.0.weight"] = (oc, oc, 3, 3)
        _bn(s, f"fpn.merge{i}.1", oc)
    for i in (1, 2, 3):
        for nm, ci, co in (("conv3X3", oc, oc // 2), ("conv5X5_1", oc, oc // 4), ("conv5X5_2", oc // 4, oc // 4),
                           ("conv7X7_2", oc // 4, oc // 4), ("conv7x7_3", oc // 4, oc // 4)):
            s[f"ssh{i}.{nm}.0.weight"] = (co, ci, 3, 3)
            _bn(s, f"ssh{i}.{nm}.1", co)
    for head, k in (("ClassHead", 2), ("BboxHead", 4), ("LandmarkHead", 10)):
        for i in range(3):
            s[f"{head}.{i}.conv1x1.weight"] = (2 * k, oc, 1, 1)
            s[f"{head}.{i}.conv1x1.bias"] = (2 * k,)
    return s


def parsenet_blocks(cfg: dict = None):
    """(key prefix, cin, cout, scale) of every ResidualBlock of ParseNet(in_size=out_size=512), in forward order."""
    cfg = PARSENET_CFG if cfg is None else cfg
    lo, hi = cfg["ch_range"]
    clip = lambda x: max(lo, min(x, hi))            # noqa: E731
    steps = (cfg["in_size"] // min(cfg["in_size"], cfg["min_feat_size"])).bit_length() - 1
    out, head = [], cfg["base_ch"]
    for i in range(steps):
        out.append((f"encoder.{i + 1}.", clip(head), clip(head * 2), "down"))
        head *= 2
    for i in range(cfg["res_depth"]):
        out.append((f"body.{i}.", clip(head), clip(head), "none"))
    for i in range(steps):
        out.append((f"decoder.{i}.", clip(head), clip(head // 2), "up"))
        head //= 2
    return out


def parsenet_shapes(cfg: dict = None) -> Shapes:
    """ParseNet: ConvLayer keys `<p>conv2d.weight` (+ `.bias` without BN), BN under `<p>norm.norm.*`; a ResidualBlock
    has `conv1`, `conv2` (BN) and, unless it keeps size and width, a `shortcut_func` conv (bias, no norm)."""
    cfg = PARSENET_CFG if cfg is None else cfg
    s = OrderedDict()
    s["encoder.0.conv2d.weight"] = (cfg["base_ch"], 3, 3, 3)
    s["encoder.0.conv2d.bias"] = (cfg["base_ch"],)
    for p, ci, co, scale in parsenet_blocks(cfg):
        if scale != "none" or ci != co:
            s[p + "shortcut_func.conv2d.weight"] = (co, ci, 3, 3)
            s[p + "shortcut_func.conv2d.bias"] = (co,)
        s[p + "conv1.conv2d.weight"] = (co, ci, 3, 3)
        _bn(s, p + "conv1.norm.norm", co)
        s[p + "conv2.conv2d.weight"] = (co, co, 3, 3)
        _bn(s, p + "conv2.norm.norm", co)
    last = parsenet_blocks(cfg)[-1][2]
    for nm, co in (("out_img_conv", 3), ("out_mask_conv", cfg["parsing_ch"])):
        s[nm + ".conv2d.weight"] = (co, last, 3, 3)
        s[nm + ".conv2d.bias"] = (co,)
    return s


def _strict(ckpt: dict, shapes: Shapes, what: str) -> dict:
    if "state_dict" in ckpt and not hasattr(ckpt["state_dict"], "shape"):
        ckpt = ckpt["state_dict"]
    sd = {(k[len("module."):] if k.startswith("module.") else k): v for k, v in ckpt.items()
          if not k.endswith("num_batches_tracked")}
    missing = [k for k in shapes if k not in sd]
    extra = [k for k in sd if k not in shapes]
    bad = [f"{k} {tuple(sd[k].shape)} != {tuple(shapes[k])}" for k in shapes
           if k in sd and tuple(sd[k].shape) != tuple(shapes[k])]
    if missing or extra or bad:
        raise ValueError(f"{what} checkpoint does not match: missing {missing}, unexpected {extra}, mis-shaped {bad}")
    return sd


def retinaface_state_dict(ckpt: dict, cfg: dict = None) -> dict:
    """Strict loader of detection_Resnet50_Final.pth: `module.` stripped, num_batches_tracked ignored, every missing,
    unexpected or mis-shaped key named."""
    return _strict(ckpt, retinaface_shapes(cfg), "RetinaFace")


def parsenet_state_dict(ckpt: dict, cfg: dict = None) -> dict:
    """Strict loader of parsing_parsenet.pth (same rules as retinaface_state_dict)."""
    return _strict(ckpt, parsenet_shapes(cfg), "ParseNet")


def fold_bn(w, sd: dict, bn: str, bias=None, eps: float = BN_EPS):
    """Eval-mode BatchNorm folded into the preceding conv, in fp32: (w * g / sqrt(var + eps), (b - mean) * that + beta)."""
    import torch
    scale = sd[bn + ".weight"].float() / torch.sqrt(sd[bn + ".running_var"].float() + eps)
    b = torch.zeros_like(scale) if bias is None else bias.float()
    return w.float() * scale.view(-1, *([1] * (w.dim() - 1))), (b - sd[bn + ".running_mean"].float()) * scale + \
        sd[bn + ".bias"].float()


# ---- LLaVA-1.5-7B captioner (reference utils/caption.py:52-145, llava/model/*) --------------------------------------
# LLM: LLaMA-7B (Vicuna-7B v1.5); vision tower: CLIP ViT-L/14-336; projector mlp2x_gelu. Keys in the layout of the
# llava-v1.5-7b shards, the vision tower under model.vision_tower.vision_tower.vision_model.* (CLIPVisionTower).
LLAVA_CFG = dict(vocab=32000, hidden=4096, layers=32, heads=32, intermediate=11008, rms_eps=1e-5, rope_theta=10000.0,
                 bos=1, eos=2, image=336, patch=14, v_width=1024, v_layers=24, v_heads=16, v_intermediate=4096,
                 v_eps=1e-5, select_layer=-2)
LLAVA_HEAD_DIM = 128
VISION_PREFIX = "model.vision_tower.vision_tower."


def llava_config(config: dict, clip_config: Optional[dict] = None) -> dict:
    """Sizes from llava-v1.5-7b's config.json (and the CLIP directory's config.json, if any). Anything but the v1.5
    settings the engine implements is refused with a message naming the setting."""
    def need(key, want, ok):
        got = config.get(key, want)
        if not ok(got):
            raise NotImplementedError(f"LLaVA config.json: {key} = {got!r}; only {want!r} (LLaVA-1.5) is built")
    need("mm_projector_type", "mlp2x_gelu", lambda v: v == "mlp2x_gelu")
    need("image_aspect_ratio", "pad", lambda v: v == "pad")
    need("mm_vision_select_layer", -2, lambda v: v == -2)
    need("mm_vision_select_feature", "patch", lambda v: v == "patch")
    need("mm_use_im_start_end", False, lambda v: not v)
    need("rope_scaling", None, lambda v: v is None)
    heads = config["num_attention_heads"]
    need("num_key_value_heads", heads, lambda v: v == heads)
    if config["hidden_size"] != heads * LLAVA_HEAD_DIM:
        raise NotImplementedError(f"LLaVA config.json: hidden_size {config['hidden_size']} != {heads} heads x 128")
    cfg = dict(LLAVA_CFG, vocab=config["vocab_size"], hidden=config["hidden_size"], layers=config["num_hidden_layers"],
               heads=heads, intermediate=config["intermediate_size"], rms_eps=config.get("rms_norm_eps", 1e-5),
               rope_theta=float(config.get("rope_theta", 10000.0)), bos=config.get("bos_token_id", 1),
               eos=config.get("eos_token_id", 2))
    if "mm_hidden_size" in config:
        cfg["v_width"] = config["mm_hidden_size"]
    if clip_config is not None:
        v = clip_config.get("vision_config", clip_config)
        if v.get("hidden_act", "quick_gelu") != "quick_gelu":
            raise NotImplementedError(f"CLIP config.json: hidden_act {v['hidden_act']!r}; only quick_gelu is built")
        cfg.update(image=v.get("image_size", 336), patch=v.get("patch_size", 14), v_width=v["hidden_size"],
                   v_layers=v["num_hidden_layers"], v_heads=v["num_attention_heads"],
                   v_intermediate=v["intermediate_size"], v_eps=v.get("layer_norm_eps", 1e-5))
    return cfg


def llava_shapes(cfg: dict) -> Shapes:
    s: Shapes = OrderedDict()
    d, f, vw = cfg["hidden"], cfg["intermediate"], cfg["v_width"]
    s["model.embed_tokens.weight"] = (cfg["vocab"], d)
    for i in range(cfg["layers"]):
        p = f"model.layers.{i}."
        for nm in ("q_proj", "k_proj", "v_proj", "o_proj"):
            s[p + f"self_attn.{nm}.weight"] = (d, d)
        s[p + "mlp.gate_proj.weight"] = (f, d)
        s[p + "mlp.up_proj.weight"] = (f, d)
        s[p + "mlp.down_proj.weight"] = (d, f)
        s[p + "input_layernorm.weight"] = (d,)
        s[p + "post_attention_layernorm.weight"] = (d,)
    s["model.norm.weight"] = (d,)
    s["lm_head.weight"] = (cfg["vocab"], d)
    s["model.mm_projector.0.weight"] = (d, vw)
    s["model.mm_projector.0.bias"] = (d,)
    s["model.mm_projector.2.weight"] = (d, d)
    s["model.mm_projector.2.bias"] = (d,)
    v = VISION_PREFIX + "vision_model."
    side = cfg["image"] // cfg["patch"]
    s[v + "embeddings.class_embedding"] = (vw,)
    s[v + "embeddings.patch_embedding.weight"] = (vw, 3, cfg["patch"], cfg["patch"])
    s[v + "embeddings.position_embedding.weight"] = (side * side + 1, vw)
    s[v + "pre_layrnorm.weight"] = (vw,)
    s[v + "pre_layrnorm.bias"] = (vw,)
    for i in range(cfg["v_layers"]):
        p = f"{v}encoder.layers.{i}."
        for nm in ("q_proj", "k_proj", "v_proj", "out_proj"):
            s[p + f"self_attn.{nm}.weight"] = (vw, vw)
            s[p + f"self_attn.{nm}.bias"] = (vw,)
        for nm in ("layer_norm1", "layer_norm2"):
            s[p + nm + ".weight"] = (vw,)
            s[p + nm + ".bias"] = (vw,)
        s[p + "mlp.fc1.weight"] = (cfg["v_intermediate"], vw)
        s[p + "mlp.fc1.bias"] = (cfg["v_intermediate"],)
        s[p + "mlp.fc2.weight"] = (vw, cfg["v_intermediate"])
        s[p + "mlp.fc2.bias"] = (vw,)
    s[v + "post_layernorm.weight"] = (vw,)
    s[v + "post_layernorm.bias"] = (vw,)
    return s


def llava_state_dict(llava_sd: dict, clip_sd: Optional[dict] = None, cfg: dict = None) -> dict:
    """The strict LLaVA loader. llava_sd: the merged llava-v1.5-7b shards; clip_sd: the CLIP ViT-L/14-336 checkpoint
    (its vision_model.* keys become the vision tower; the text tower and projections it also holds are not used), or
    None when the shards carry model.vision_tower.*. Buffers the checkpoints may hold (rotary inv_freq, position_ids)
    are dropped; every other key must be one of llava_shapes, with its shape."""
    cfg = LLAVA_CFG if cfg is None else cfg
    buffers = ("rotary_emb.inv_freq", "position_ids")
    sd = {k: v for k, v in llava_sd.items() if not k.endswith(buffers)}
    if clip_sd is not None:
        if any(k.startswith("model.vision_tower.") for k in sd):
            raise ValueError("LLaVA checkpoint carries model.vision_tower.* and a CLIP checkpoint was given too")
        sd.update({VISION_PREFIX + k: v for k, v in clip_sd.items()
                   if k.startswith("vision_model.") and not k.endswith(buffers)})
    shapes = llava_shapes(cfg)
    missing = [k for k in shapes if k not in sd]
    extra = [k for k in sd if k not in shapes]
    bad = [f"{k} {tuple(sd[k].shape)} != {tuple(shapes[k])}" for k in shapes
           if k in sd and tuple(sd[k].shape) != tuple(shapes[k])]
    if missing or extra or bad:
        raise ValueError(f"LLaVA checkpoint does not match: missing {missing[:8]}{' ...' if len(missing) > 8 else ''}, "
                         f"unexpected {extra[:8]}{' ...' if len(extra) > 8 else ''}, mis-shaped {bad[:8]}")
    return sd
