"""LLaVA-1.5-7B (the `--captioner llava --llava_bit 16` captioner) on the sm_90a kernels.

Replaces LlavaLlamaForCausalLM.generate with greedy decoding (reference utils/caption.py:52-145 with
llava/model/llava_arch.py, clip_encoder.py, multimodal_projector/builder.py and transformers' LLaMA):

- Vision tower, CLIP ViT-L/14-336 up to the output of layer 23 of 24 (mm_vision_select_layer = -2, patch
  features): dbir_swin_stem (r = 14, CLIP mean subtracted) + a GEMM whose packed weight carries CLIP's 1/std and
  whose residual operand adds the position embeddings; pre-LN blocks of dbir_layernorm, fused-QKV GEMM,
  dbir_attention (head_dim 64, 577 tokens), out-proj GEMM + residual, fc1 GEMM + quick_gelu, fc2 GEMM + residual.
- Projector mlp2x_gelu: two GEMMs, the second writing straight into the LLM's residual stream at the <image> slot.
- LLM prefill over the whole prompt: RMSNorm, fused-QKV GEMM, dbir_rope_kv into the KV cache, dbir_attention_causal,
  o_proj GEMM + residual, RMSNorm, gate/up GEMM with the SwiGLU epilogue, down GEMM + residual; lm_head on the last
  row, argmax. Vision, projector and prefill are one CUDA graph (the prompt length is a constant).
- Decode: one CUDA-graph replay per token (embedding gather, 32 layers of RMSNorm / dbir_gemv / dbir_rope_kv /
  dbir_attention_decode, lm_head dbir_gemv, dbir_argmax advancing the device position). The GEMV reads the same
  packed weights as the prefill GEMMs: one device copy of every weight. The host reads each token back through a
  pinned copy to stop at EOS.

The KV cache holds prompt length + max_new_tokens rows. A new image needs no clearing: prefill rewrites rows
0 .. L-1 and every step attends only to the rows written for this image.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from .. import arch, lib

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)     # CLIPImageProcessor image_mean / image_std
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
IMAGE_TOKEN_INDEX = -200                            # llava/constants.py
VISION_HEAD_DIM = 64


def swiglu_tile(inter: int) -> int:
    """Tile width of the packed gate/up weight (force_bn of dbir_gemm's geglu = 2, pack of dbir_gemv)."""
    for bn in (256, 128, 64):
        if (2 * inter) % bn == 0:
            return bn
    raise ValueError(f"intermediate size {inter}: gate/up rows must tile by 64")


class LlavaEngine:
    def __init__(self, sd: Dict[str, torch.Tensor], prompt_ids: Sequence[int], cfg: dict = None, device="cuda",
                 max_new_tokens: int = 512):
        """sd: a llava_state_dict (CPU or device tensors). Its entries are popped while they are packed, so weights
        already on the device in the operand format are kept, not copied. prompt_ids: the prompt's token ids with one
        IMAGE_TOKEN_INDEX where the image features go."""
        self.cfg = cfg = dict(arch.LLAVA_CFG if cfg is None else cfg)
        self.dev = dev = torch.device(device)
        self.dt = dt = lib.operand_dtype()
        ids = list(prompt_ids)
        if ids.count(IMAGE_TOKEN_INDEX) != 1:
            raise ValueError("the prompt must hold exactly one image token")
        i0 = ids.index(IMAGE_TOKEN_INDEX)
        side = cfg["image"] // cfg["patch"]
        self.patches = side * side
        self.pre, self.post = ids[:i0], ids[i0 + 1:]
        self.L = L = len(self.pre) + self.patches + len(self.post)
        self.max_new = max_new_tokens
        self.cap = L + max_new_tokens
        self.v_run = cfg["v_layers"] + cfg["select_layer"] + 1        # hidden_states[-2]: 23 of 24 layers
        d, f, vw, H = cfg["hidden"], cfg["intermediate"], cfg["v_width"], cfg["heads"]
        assert vw == cfg["v_heads"] * VISION_HEAD_DIM and d == H * arch.LLAVA_HEAD_DIM
        self.bn = swiglu_tile(f)

        def take(k):
            return sd.pop(k)

        def o16(t):
            return t.to(device=dev, dtype=dt).contiguous()

        def f32(t):
            return t.to(device=dev, dtype=torch.float32).contiguous()

        w = {}
        v = arch.VISION_PREFIX + "vision_model."
        r = cfg["patch"]
        self.stem_c = 3 * r * r
        self.stem_cp = -(-self.stem_c // 64) * 64                      # 588 -> 640
        pe = take(v + "embeddings.patch_embedding.weight").to(dev, torch.float32)
        pe = pe / torch.tensor(CLIP_STD, device=dev).view(1, 3, 1, 1)
        w["pe"] = o16(torch.nn.functional.pad(pe.reshape(vw, self.stem_c), (0, self.stem_cp - self.stem_c)))
        pos = f32(take(v + "embeddings.position_embedding.weight"))
        self.vemb = torch.empty(self.patches + 1, vw, device=dev)
        self.vemb[0] = f32(take(v + "embeddings.class_embedding")) + pos[0]      # constant class-token row
        w["pos"] = pos[1:].contiguous()
        w["pre.w"], w["pre.b"] = f32(take(v + "pre_layrnorm.weight")), f32(take(v + "pre_layrnorm.bias"))
        for i in range(cfg["v_layers"]):
            p = f"{v}encoder.layers.{i}."
            keys = [k for k in sd if k.startswith(p)]
            if i >= self.v_run:                                          # layers past the selected one never run
                for k in keys:
                    del sd[k]
                continue
            o = f"v{i}."
            w[o + "qkv.w"] = o16(torch.cat([take(p + f"self_attn.{n}_proj.weight").to(dev) for n in "qkv"]))
            w[o + "qkv.b"] = f32(torch.cat([take(p + f"self_attn.{n}_proj.bias").to(dev) for n in "qkv"]))
            for src, dst in (("self_attn.out_proj", "out"), ("mlp.fc1", "fc1"), ("mlp.fc2", "fc2")):
                w[o + dst + ".w"], w[o + dst + ".b"] = o16(take(p + src + ".weight")), f32(take(p + src + ".bias"))
            for nm in ("layer_norm1", "layer_norm2"):
                w[o + nm + ".w"], w[o + nm + ".b"] = f32(take(p + nm + ".weight")), f32(take(p + nm + ".bias"))
        for k in [k for k in sd if k.startswith(v + "post_layernorm")]:
            del sd[k]
        for i in (0, 2):
            w[f"mm{i}.w"] = o16(take(f"model.mm_projector.{i}.weight"))
            w[f"mm{i}.b"] = f32(take(f"model.mm_projector.{i}.bias"))
        w["embed"] = o16(take("model.embed_tokens.weight"))
        hb = self.bn // 2
        for i in range(cfg["layers"]):
            p, o = f"model.layers.{i}.", f"l{i}."
            w[o + "qkv"] = o16(torch.cat([take(p + f"self_attn.{n}_proj.weight").to(dev, dt) for n in "qkv"]))
            w[o + "o"] = o16(take(p + "self_attn.o_proj.weight"))
            up = take(p + "mlp.up_proj.weight").to(dev, dt).view(f // hb, hb, d)       # values
            gate = take(p + "mlp.gate_proj.weight").to(dev, dt).view(f // hb, hb, d)   # gates
            w[o + "gu"] = torch.cat([up, gate], dim=1).reshape(2 * f, d).contiguous()
            del up, gate
            w[o + "down"] = o16(take(p + "mlp.down_proj.weight"))
            w[o + "ln1"] = f32(take(p + "input_layernorm.weight"))
            w[o + "ln2"] = f32(take(p + "post_attention_layernorm.weight"))
        w["norm"] = f32(take("model.norm.weight"))
        w["lm_head"] = o16(take("lm_head.weight"))
        assert not sd, f"unused weights: {sorted(sd)[:4]}"
        self.w = w

        # ---- buffers: every shape is fixed by the config and the prompt, allocated once
        nv = self.patches + 1
        e = lambda *s, dtype=torch.float32: torch.empty(*s, device=dev, dtype=dtype)  # noqa: E731
        self.img = e(1, 3, cfg["image"], cfg["image"])
        self.stem16 = e(self.patches, self.stem_cp, dtype=dt)
        self.t = e(nv, vw)
        self.ln16 = e(nv, vw, dtype=dt)
        self.vqkv16 = e(nv, 3 * vw, dtype=dt)
        self.vatt16 = e(nv, vw, dtype=dt)
        self.vhid16 = e(nv, cfg["v_intermediate"], dtype=dt)
        self.feat16 = e(self.patches, vw, dtype=dt)
        self.phid16 = e(self.patches, d, dtype=dt)
        self.vattn_ws = torch.zeros(max(lib.attention_ws_bytes(1, cfg["v_heads"], nv, nv), 1), dtype=torch.uint8,
                                    device=dev)
        self.h = e(L, d)
        self.x16 = e(L, d, dtype=dt)
        self.qkv = e(L, 3 * d)
        self.q16 = e(L, d, dtype=dt)
        self.att16 = e(L, d, dtype=dt)
        self.gu16 = e(L, f, dtype=dt)
        self.kc = torch.zeros(cfg["layers"], self.cap, H, arch.LLAVA_HEAD_DIM, device=dev, dtype=dt)
        self.vc = torch.zeros_like(self.kc)
        self.logits = e(cfg["vocab"])
        self.ids_pre = torch.tensor(self.pre or [0], dtype=torch.int32, device=dev)
        self.ids_post = torch.tensor(self.post or [0], dtype=torch.int32, device=dev)
        self.tok = torch.zeros(1, dtype=torch.int32, device=dev)
        self.state = torch.tensor([L, L + 1], dtype=torch.int32, device=dev)      # (position fed, cache length)
        self.state0 = self.state.clone()
        self.zero = torch.zeros(1, dtype=torch.int32, device=dev)
        self.dec_ws = torch.empty(lib.attention_decode_ws_bytes(H, self.cap), dtype=torch.uint8, device=dev)
        self.tok_host = torch.zeros(1, dtype=torch.int32, pin_memory=True)
        self._graphs = None

    # ------------------------------------------------------------------ public
    @torch.no_grad()
    def generate(self, x: torch.Tensor, use_graphs: bool = True, max_new_tokens: Optional[int] = None) -> List[int]:
        """x: fp32 [1, 3, 336, 336], the padded, resized image / 255 (CLIP normalisation is folded into the
        vision tower). Greedy decoding: the generated ids, ending with EOS when it came within max_new_tokens."""
        assert x.shape == self.img.shape
        n = self.max_new if max_new_tokens is None else min(max_new_tokens, self.max_new)
        self.img.copy_(x)
        if use_graphs and self._graphs is None:
            self._graphs = (self._capture(self._prefill), self._capture(self._decode_step))
        run_prefill = self._graphs[0].replay if use_graphs else self._prefill
        run_step = self._graphs[1].replay if use_graphs else self._decode_step
        run_prefill()
        out = []
        while True:
            self.tok_host.copy_(self.tok, non_blocking=True)
            torch.cuda.current_stream().synchronize()
            t = int(self.tok_host[0])
            out.append(t)
            if t == self.cfg["eos"] or len(out) >= n:
                return out
            run_step()

    @torch.no_grad()
    def prefill_logits(self, x: torch.Tensor) -> torch.Tensor:
        """fp32 logits of the prompt's last position (eager prefill)."""
        self.img.copy_(x)
        self._prefill()
        return self.logits.clone()

    @torch.no_grad()
    def forced_logits(self, x: torch.Tensor, tokens: Sequence[int], use_graphs: bool = False) -> torch.Tensor:
        """Teacher forcing: after the prefill, feed `tokens` one decode step each; row i = the logits after
        tokens[:i] (row 0 = the prefill's)."""
        self.img.copy_(x)
        if use_graphs and self._graphs is None:
            self._graphs = (self._capture(self._prefill), self._capture(self._decode_step))
        (self._graphs[0].replay if use_graphs else self._prefill)()
        rows = [self.logits.clone()]
        for t in tokens[:-1]:
            self.tok.fill_(int(t))
            (self._graphs[1].replay if use_graphs else self._decode_step)()
            rows.append(self.logits.clone())
        return torch.stack(rows)

    @torch.no_grad()
    def image_features(self, x: torch.Tensor) -> torch.Tensor:
        """The projector's output for one image (fp32 [576, hidden], eager)."""
        self.img.copy_(x)
        out = torch.empty(self.patches, self.cfg["hidden"], device=self.dev)
        self._vision()
        self._project(out)
        return out

    # ------------------------------------------------------------------ graph bodies
    def _capture(self, fn) -> torch.cuda.CUDAGraph:
        fn()                                   # eager run first: dbir_gemm times its plans outside a capture
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        return g

    def _vision(self):
        cfg, W = self.cfg, self.w
        vw, nv, P = cfg["v_width"], self.patches + 1, self.patches
        s = cfg["image"]
        lib.swin_stem(self.img, 1, s, s, cfg["patch"], CLIP_MEAN, 1.0, self.stem_cp, self.stem16)
        lib.gemm(self.stem16, W["pe"], self.vemb[1:], M=P, N=vw, K=self.stem_cp, residual=W["pos"])
        t = self.t
        lib.layernorm(self.vemb, vw, nv, vw, W["pre.w"], W["pre.b"], t, vw, eps=cfg["v_eps"])
        heads, ld = cfg["v_heads"], 3 * vw
        for i in range(self.v_run):
            o = f"v{i}."
            lib.layernorm(t, vw, nv, vw, W[o + "layer_norm1.w"], W[o + "layer_norm1.b"], self.ln16, vw, eps=cfg["v_eps"])
            lib.gemm(self.ln16, W[o + "qkv.w"], self.vqkv16, M=nv, N=3 * vw, K=vw, bias=W[o + "qkv.b"])
            q = self.vqkv16
            lib.attention(q, q[:, vw:], q[:, 2 * vw:], self.vatt16, batch=1, heads=heads, sq=nv, skv=nv, ldq=ld,
                          ldk=ld, ldv=ld, ldo=vw, ws=self.vattn_ws)
            lib.gemm(self.vatt16, W[o + "out.w"], t, M=nv, N=vw, K=vw, bias=W[o + "out.b"], residual=t)
            lib.layernorm(t, vw, nv, vw, W[o + "layer_norm2.w"], W[o + "layer_norm2.b"], self.ln16, vw, eps=cfg["v_eps"])
            lib.gemm(self.ln16, W[o + "fc1.w"], self.vhid16, M=nv, N=cfg["v_intermediate"], K=vw, bias=W[o + "fc1.b"],
                     act="quick_gelu")
            lib.gemm(self.vhid16, W[o + "fc2.w"], t, M=nv, N=vw, K=cfg["v_intermediate"], bias=W[o + "fc2.b"],
                     residual=t)
        lib.axpby_cast(t[1:], 1.0, None, P, vw, y16=self.feat16, ld16=vw)          # select_feature "patch"

    def _project(self, out: torch.Tensor):
        """mlp2x_gelu on the selected patch features -> fp32 rows of `out` (the <image> slot of the stream)."""
        W, d, P = self.w, self.cfg["hidden"], self.patches
        lib.gemm(self.feat16, W["mm0.w"], self.phid16, M=P, N=d, K=self.cfg["v_width"], bias=W["mm0.b"], act="gelu")
        lib.gemm(self.phid16, W["mm2.w"], out, M=P, N=d, K=d, bias=W["mm2.b"])

    def _prefill(self):
        cfg, W = self.cfg, self.w
        d, f, H, L = cfg["hidden"], cfg["intermediate"], cfg["heads"], self.L
        self._vision()
        i0, P = len(self.pre), self.patches
        self._project(self.h[i0:i0 + P])
        if self.pre:
            lib.embed_gather(W["embed"], cfg["vocab"], self.ids_pre, len(self.pre), d, self.h, d)
        if self.post:
            lib.embed_gather(W["embed"], cfg["vocab"], self.ids_post, len(self.post), d, self.h[i0 + P:], d)
        h, x16 = self.h, self.x16
        for i in range(cfg["layers"]):
            o = f"l{i}."
            lib.rmsnorm(h, d, L, d, W[o + "ln1"], x16, d, eps=cfg["rms_eps"])
            lib.gemm(x16, W[o + "qkv"], self.qkv, M=L, N=3 * d, K=d)
            lib.rope_kv(self.qkv, 3 * d, L, H, self.zero, self.q16, d, self.kc[i], self.vc[i], theta=cfg["rope_theta"])
            lib.attention_causal(self.q16, d, self.kc[i], self.vc[i], H, L, self.att16, d)
            lib.gemm(self.att16, W[o + "o"], h, M=L, N=d, K=d, residual=h)
            lib.rmsnorm(h, d, L, d, W[o + "ln2"], x16, d, eps=cfg["rms_eps"])
            lib.gemm(x16, W[o + "gu"], self.gu16, M=L, N=2 * f, K=d, geglu=2, force_bn=self.bn)
            lib.gemm(self.gu16, W[o + "down"], h, M=L, N=d, K=f, residual=h)
        lib.rmsnorm(h[L - 1:], d, 1, d, W["norm"], x16, d, eps=cfg["rms_eps"])
        lib.gemv(W["lm_head"], x16, self.logits, N=cfg["vocab"], K=d)
        lib.argmax(self.logits, cfg["vocab"], self.tok)
        self.state.copy_(self.state0)

    def _decode_step(self):
        cfg, W = self.cfg, self.w
        d, f, H = cfg["hidden"], cfg["intermediate"], cfg["heads"]
        h, x16 = self.h[:1], self.x16[:1]             # the prompt's rows are no longer needed
        qkv, q16, att16, gu16 = self.qkv[:1], self.q16[:1], self.att16[:1], self.gu16[:1]
        lib.embed_gather(W["embed"], cfg["vocab"], self.tok, 1, d, h, d)
        for i in range(cfg["layers"]):
            o = f"l{i}."
            lib.rmsnorm(h, d, 1, d, W[o + "ln1"], x16, d, eps=cfg["rms_eps"])
            lib.gemv(W[o + "qkv"], x16, qkv, N=3 * d, K=d)
            lib.rope_kv(qkv, 3 * d, 1, H, self.state[0:1], q16, d, self.kc[i], self.vc[i], theta=cfg["rope_theta"])
            lib.attention_decode(q16, self.kc[i], self.vc[i], H, self.cap, self.state[1:2], self.dec_ws, att16)
            lib.gemv(W[o + "o"], att16, h, N=d, K=d, epilogue="residual", residual=h)
            lib.rmsnorm(h, d, 1, d, W[o + "ln2"], x16, d, eps=cfg["rms_eps"])
            lib.gemv(W[o + "gu"], x16, gu16, N=2 * f, K=d, epilogue="swiglu", pack=self.bn)
            lib.gemv(W[o + "down"], gu16, h, N=d, K=f, epilogue="residual", residual=h)
        lib.rmsnorm(h, d, 1, d, W["norm"], x16, d, eps=cfg["rms_eps"])
        lib.gemv(W["lm_head"], x16, self.logits, N=cfg["vocab"], K=d)
        lib.argmax(self.logits, cfg["vocab"], self.tok, advance=self.state)
