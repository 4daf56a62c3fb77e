"""RAM++ tagging (the `--captioner ram` captioner) on the sm_90a kernels.

Replaces RAM_plus.generate_tag up to its logits (reference ram/models/ram_plus.py:280-320) for
RAM_plus(image_size=384, vit="swin_l"):

- Swin-L (ram/models/swin_transformer.py): the 4x4 stride-4 patch embed is dbir_swin_stem (r = 4, ImageNet mean
  subtracted) + a GEMM whose packed weights carry ImageNet's 1/std; Swin blocks are LN - qkv GEMM - 12x12 window
  attention (tensor cores) - proj GEMM + residual - LN - fc1 GEMM + GELU - fc2 GEMM + residual on a fp32 token
  stream; PatchMerging is dbir_swin_patch_merge + the reduction GEMM; the final LN feeds dbir_token_mean, which
  writes [cls = token mean | tokens] as image_proj's operand.
- dbir_label_reweight builds the [B, 4585, 512] operand of wordvec_proj (+ ReLU in the GEMM epilogue).
- The tagging head's two cross-attention layers: Q / K GEMMs, V^T by a bias-per-row GEMM, then per image and head
  S = Q K^T into rows padded to 160 keys, dbir_softmax_rows over the 145 real keys and P V (the VAE mid attention's
  path); output dense + residual, post-LN (eps 1e-12), GELU FFN, post-LN; fc as a GEMM padded to 8 outputs.

label_embed (233 835 x 512) is stored in the 16-bit operand format, 240 MB, read once per batch.
One CUDA-graph replay per batch size; logits come back fp32.
"""
from __future__ import annotations

import math
from typing import Dict

import torch

from .. import arch, lib
from .common import GraphCache, Workspace, f32, op16, pack_linear, pack_swin_block, prenorm_block, round_up

IMAGENET_MEAN = (0.485, 0.456, 0.406)      # ram/transform.py
IMAGENET_STD = (0.229, 0.224, 0.225)
HEAD_DIM = 32
KEYS_PAD = 160                             # 145 image tokens, padded for 16-byte GEMM rows


class RamPlusEngine:
    def __init__(self, sd: Dict[str, torch.Tensor], cfg: dict = None, device="cuda"):
        self.cfg = dict(arch.RAM_CFG if cfg is None else cfg)
        cfg = self.cfg
        sd = arch.ram_state_dict(sd, cfg)
        self.dev = torch.device(device)
        self.ws = Workspace(self.dev)
        self.graphs = GraphCache(self.ws)
        self.op_dtype = lib.operand_dtype()
        self.stages = arch.ram_stages(cfg)
        side = cfg["img_size"] // cfg["patch_size"]
        self.tokens = (side >> (len(self.stages) - 1)) ** 2           # 144 stage-4 tokens
        for c, _, heads, _, _ in self.stages:
            assert c == heads * HEAD_DIM and c % 64 == 0, "Swin-L stages are heads x 32 wide"
        dev, w = self.dev, {}
        p = "visual_encoder."
        pe = sd[p + "patch_embed.proj.weight"].float()
        c0, r = pe.shape[0], cfg["patch_size"]
        self.stem_c = 3 * r * r
        self.stem_cp = round_up(self.stem_c)                            # 48 -> 64
        std = torch.tensor(IMAGENET_STD).view(1, 3, 1, 1)
        w["pe.w"] = pack_linear((pe / std).reshape(c0, self.stem_c), dev, self.stem_cp)   # (c, dy, dx) = unshuffle order
        w["pe.b"] = f32(sd[p + "patch_embed.proj.bias"], dev)
        w["pe.norm.w"] = f32(sd[p + "patch_embed.norm.weight"], dev)
        w["pe.norm.b"] = f32(sd[p + "patch_embed.norm.bias"], dev)
        for i, (c, _, _, _, shifts) in enumerate(self.stages):
            for b in range(len(shifts)):
                pack_swin_block(w, f"{i}.{b}.", sd, f"{p}layers.{i}.blocks.{b}.", dev)
            if i < len(self.stages) - 1:
                q = f"{p}layers.{i}.downsample."
                w[f"{i}.merge.w"] = f32(sd[q + "norm.weight"], dev)
                w[f"{i}.merge.b"] = f32(sd[q + "norm.bias"], dev)
                w[f"{i}.reduction.w"] = pack_linear(sd[q + "reduction.weight"], dev)
        w["norm.w"] = f32(sd[p + "norm.weight"], dev)
        w["norm.b"] = f32(sd[p + "norm.bias"], dev)
        w["image_proj.w"] = pack_linear(sd["image_proj.weight"], dev)
        w["image_proj.b"] = f32(sd["image_proj.bias"], dev)
        w["label"] = op16(sd["label_embed"], dev)
        self.reweight_scale = math.exp(float(sd["reweight_scale"]))
        w["wordvec.w"] = pack_linear(sd["wordvec_proj.weight"], dev)
        w["wordvec.b"] = f32(sd["wordvec_proj.bias"], dev)
        for l in range(cfg["bert_layers"]):
            q, o = f"tagging_head.encoder.layer.{l}.", f"bert{l}."
            for src, dst in (("crossattention.self.query", "q"), ("crossattention.self.key", "k"),
                             ("crossattention.self.value", "v"), ("crossattention.output.dense", "dense"),
                             ("intermediate.dense", "inter"), ("output.dense", "out")):
                w[o + dst + ".w"] = pack_linear(sd[q + src + ".weight"], dev)
                w[o + dst + ".b"] = f32(sd[q + src + ".bias"], dev)
            for src, dst in (("crossattention.output.LayerNorm", "ln1"), ("output.LayerNorm", "ln2")):
                w[o + dst + ".w"] = f32(sd[q + src + ".weight"], dev)
                w[o + dst + ".b"] = f32(sd[q + src + ".bias"], dev)
        fcw = torch.zeros(8, cfg["hidden"])                              # 1 output padded to 8 (16-byte rows)
        fcw[0] = sd["fc.weight"][0]
        fcb = torch.zeros(8)
        fcb[0] = sd["fc.bias"][0]
        w["fc.w"], w["fc.b"] = op16(fcw, dev), f32(fcb, dev)
        self.w = w

    # ------------------------------------------------------------------ public
    def forward(self, x: torch.Tensor) -> torch.Tensor:
        """x fp32 NCHW [B, 3, 384, 384]: the ToTensor() image in [0, 1] (ImageNet normalisation is folded into the
        patch embed) -> fp32 logits [B, classes]. One CUDA-graph replay per batch size."""
        s = self.cfg["img_size"]
        assert x.is_cuda and x.dtype == torch.float32 and x.is_contiguous() and tuple(x.shape[1:]) == (3, s, s)
        return self.graphs.run(tuple(x.shape), self._forward, x)

    def image_embeds(self, batch: int) -> torch.Tensor:
        """image_proj's output [B, 145, 512] (fp32) of the last forward of this batch size."""
        return self.ws.get("emb", (batch * (self.tokens + 1), self.cfg["embed"]), torch.float32).view(
            batch, self.tokens + 1, -1).clone()

    def stage_output(self, batch: int, i: int) -> torch.Tensor:
        """Swin stage i's output tokens [B, L_i, C_i] (fp32) of the last forward of this batch size."""
        c, r = self.stages[i][0], self.stages[i][1]
        return self.ws.get(f"t{i}", (batch * r * r, c), torch.float32).view(batch, r * r, c).clone()

    # ------------------------------------------------------------------ graph body
    def _forward(self, x: torch.Tensor) -> torch.Tensor:
        cfg, ws, W, dt = self.cfg, self.ws, self.w, self.op_dtype
        nb = x.shape[0]
        emb = self._encoder(x)
        e, hid, nc = cfg["embed"], cfg["hidden"], cfg["num_class"]
        nkv = self.tokens + 1
        emb16 = ws.get("emb16", (nb * nkv, e), dt)
        lib.axpby_cast(emb, 1.0, None, nb * nkv, e, y16=emb16, ld16=e)
        rw16 = ws.get("rw16", (nb * nc, e), dt)
        lib.label_reweight(emb, nkv * e, nb, W["label"], nc, cfg["des_per_class"], self.reweight_scale, rw16, e)
        M = nb * nc
        h = ws.get("h", (M, hid), torch.float32)
        h16 = ws.get("h16", (M, hid), dt)
        lib.gemm(rw16, W["wordvec.w"], h, M=M, N=hid, K=e, bias=W["wordvec.b"], act="lrelu", act_param=0.0)
        lib.axpby_cast(h, 1.0, None, M, hid, y16=h16, ld16=hid)
        for l in range(cfg["bert_layers"]):
            self._bert_layer(f"bert{l}.", h, h16, emb16, nb)
        logits8 = ws.get("logits8", (M, 8), torch.float32)
        lib.gemm(h16, W["fc.w"], logits8, M=M, N=8, K=hid, bias=W["fc.b"])
        return logits8[:, 0].reshape(nb, nc)

    def _encoder(self, x: torch.Tensor) -> torch.Tensor:
        """Swin-L + image_proj -> fp32 image_embeds [B*145, 512] (workspace 'emb')."""
        cfg, ws, W, dt = self.cfg, self.ws, self.w, self.op_dtype
        nb, _, s, _ = x.shape
        r = cfg["patch_size"]
        side = s // r
        M = nb * side * side
        c0 = self.stages[0][0]
        stem = ws.get("stem16", (M, self.stem_cp), dt)
        lib.swin_stem(x, nb, s, s, r, IMAGENET_MEAN, 1.0, self.stem_cp, stem)
        pe = ws.get("pe", (M, c0), torch.float32)
        lib.gemm(stem, W["pe.w"], pe, M=M, N=c0, K=self.stem_cp, bias=W["pe.b"])
        t = ws.get("t0", (M, c0), torch.float32)
        lib.layernorm(pe, c0, M, c0, W["pe.norm.w"], W["pe.norm.b"], t, c0)
        for i, (c, side, heads, win, shifts) in enumerate(self.stages):
            M = nb * side * side
            hidden = cfg["mlp_ratio"] * c
            bufs = (ws.get("ln16", (M, c), dt), ws.get("qkv16", (M, 3 * c), dt), ws.get("att16", (M, c), dt),
                    ws.get("hid16", (M, hidden), dt))
            for b, shift in enumerate(shifts):
                o = f"{i}.{b}."
                prenorm_block(W, o, t, bufs, M, c, hidden, (c, 3 * c, hidden), "gelu", 1e-5,
                              lambda qkv, att: lib.window_attention(qkv, 3 * c, nb, side, side, heads, HEAD_DIM, shift,
                                                                    W[o + "rpb"], -100.0, att, c, window=win))
            if i < len(self.stages) - 1:
                m16 = ws.get("merge16", (M // 4, 4 * c), dt)
                lib.swin_patch_merge(t, c, nb, side, side, c, W[f"{i}.merge.w"], W[f"{i}.merge.b"], m16, 4 * c)
                t = ws.get(f"t{i + 1}", (M // 4, 2 * c), torch.float32)
                lib.gemm(m16, W[f"{i}.reduction.w"], t, M=M // 4, N=2 * c, K=4 * c)
        c, L = self.stages[-1][0], self.tokens
        normed = ws.get("normed", (nb * L, c), torch.float32)
        lib.layernorm(t, c, nb * L, c, W["norm.w"], W["norm.b"], normed, c)
        tok16 = ws.get("tok16", (nb * (L + 1), c), dt)
        lib.token_mean(normed, c, nb, L, c, tok16, c)
        emb = ws.get("emb", (nb * (L + 1), cfg["embed"]), torch.float32)
        lib.gemm(tok16, W["image_proj.w"], emb, M=nb * (L + 1), N=cfg["embed"], K=c, bias=W["image_proj.b"])
        return emb

    def _bert_layer(self, o: str, h: torch.Tensor, h16: torch.Tensor, emb16: torch.Tensor, nb: int):
        """One tagging-head layer (bert.py:376-458, mode 'tagging') in place on h (fp32) and its op16 copy h16."""
        cfg, ws, W, dt = self.cfg, self.ws, self.w, self.op_dtype
        hid, e, nc, heads = cfg["hidden"], cfg["embed"], cfg["num_class"], cfg["bert_heads"]
        dh = hid // heads
        nkv = self.tokens + 1
        M = nb * nc
        q16 = ws.get("q16", (M, hid), dt)
        lib.gemm(h16, W[o + "q.w"], q16, M=M, N=hid, K=hid, bias=W[o + "q.b"])
        k16 = ws.get("k16", (nb * nkv, hid), dt)
        lib.gemm(emb16, W[o + "k.w"], k16, M=nb * nkv, N=hid, K=e, bias=W[o + "k.b"])
        vt = ws.get("vt16", (hid, KEYS_PAD), dt)                      # V^T of one image: [hid, keys]
        p16 = ws.get("p16", (nc, KEYS_PAD), dt)
        s32 = ws.get("s32", (nc, KEYS_PAD), torch.float32)
        vt[:, nkv:].zero_()
        p16[:, nkv:].zero_()
        ctx = ws.get("ctx16", (M, hid), dt)
        for b in range(nb):
            lib.gemm(W[o + "v.w"], emb16[b * nkv:(b + 1) * nkv], vt, M=hid, N=nkv, K=e, bias=W[o + "v.b"],
                     bias_per_row=True, ldo=KEYS_PAD)
            for hd in range(heads):
                cs = slice(hd * dh, (hd + 1) * dh)
                lib.gemm(q16[b * nc:(b + 1) * nc, cs], k16[b * nkv:(b + 1) * nkv, cs], s32, M=nc, N=nkv, K=dh,
                         lda=hid, ldb=hid, ldo=KEYS_PAD)
                lib.softmax_rows(s32, KEYS_PAD, nc, nkv, dh ** -0.5, p16, KEYS_PAD)
                lib.gemm(p16, vt[cs], ctx[b * nc:(b + 1) * nc, cs], M=nc, N=dh, K=KEYS_PAD, ldo=hid)
        pre = ws.get("bert_pre", (M, hid), torch.float32)                  # sum before each post-LN
        lib.gemm(ctx, W[o + "dense.w"], pre, M=M, N=hid, K=hid, bias=W[o + "dense.b"], residual=h)
        a = ws.get("bert_a", (M, hid), torch.float32)
        lib.layernorm(pre, hid, M, hid, W[o + "ln1.w"], W[o + "ln1.b"], a, hid, eps=1e-12)
        a16 = ws.get("bert_a16", (M, hid), dt)
        lib.axpby_cast(a, 1.0, None, M, hid, y16=a16, ld16=hid)
        f16 = ws.get("bert_f16", (M, cfg["intermediate"]), dt)
        lib.gemm(a16, W[o + "inter.w"], f16, M=M, N=cfg["intermediate"], K=hid, bias=W[o + "inter.b"], act="gelu")
        lib.gemm(f16, W[o + "out.w"], pre, M=M, N=hid, K=cfg["intermediate"], bias=W[o + "out.b"], residual=a)
        lib.layernorm(pre, hid, M, hid, W[o + "ln2.w"], W[o + "ln2.b"], h, hid, eps=1e-12)
        lib.axpby_cast(h, 1.0, None, M, hid, y16=h16, ld16=hid)
