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
- Batched decode (generate_list, up to MAX_SEQS images): every image shares the prompt length, so all sequences sit
  at the same position at every step. Each image's prefill runs on its own (the graph above) and its KV rows are
  copied into that sequence's cache; then one CUDA-graph replay per token decodes all of them: dbir_gemv_rows reads
  each weight row once for every sequence, dbir_rope_kv_seqs / dbir_attention_decode_seqs write and read each
  sequence's cache, dbir_argmax_rows picks each one's token. Every row's arithmetic is the single-sequence kernels',
  so each caption has the bits of generate on its image. A sequence that has emitted EOS keeps decoding until the
  last one stops; its extra tokens are dropped.

The KV cache holds prompt length + max_new_tokens rows. A new image needs no clearing: prefill rewrites rows
0 .. L-1 and every step attends only to the rows written for this image.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch

from .. import arch, lib
from .common import f32, op16, prenorm_block, round_up

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


class _Seqs:
    """Buffers and decode graphs of batched decoding; sized for `cap_seqs` sequences, used by any B up to it."""

    def __init__(self, eng: "LlavaEngine", cap_seqs: int):
        cfg, dev, dt = eng.cfg, eng.dev, eng.dt
        d, f, H = cfg["hidden"], cfg["intermediate"], cfg["heads"]
        e = lambda *s, dtype=torch.float32: torch.empty(*s, device=dev, dtype=dtype)  # noqa: E731
        self.cap_seqs = cap_seqs
        self.h, self.x16 = e(cap_seqs, d), e(cap_seqs, d, dtype=dt)
        self.qkv, self.q16, self.att16 = e(cap_seqs, 3 * d), e(cap_seqs, d, dtype=dt), e(cap_seqs, d, dtype=dt)
        self.gu16 = e(cap_seqs, f, dtype=dt)
        self.logits = e(cap_seqs, cfg["vocab"])
        self.tok = torch.zeros(cap_seqs, dtype=torch.int32, device=dev)
        self.kc = torch.zeros(cfg["layers"], cap_seqs, eng.cap, H, arch.LLAVA_HEAD_DIM, device=dev, dtype=dt)
        self.vc = torch.zeros_like(self.kc)
        self.stride = eng.cap * H * arch.LLAVA_HEAD_DIM              # elements between two sequences' caches
        self.ws = torch.empty(cap_seqs * lib.attention_decode_ws_bytes(H, eng.cap), dtype=torch.uint8, device=dev)
        self.tok_host = torch.zeros(cap_seqs, dtype=torch.int32, pin_memory=True)
        self.graphs: Dict[int, torch.cuda.CUDAGraph] = {}


class LlavaEngine:
    MAX_SEQS = 8                                    # most sequences one batched decode step takes (dbir_gemv_rows)

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

        take = sd.pop
        w = {}
        v = arch.VISION_PREFIX + "vision_model."
        r = cfg["patch"]
        self.stem_c = 3 * r * r
        self.stem_cp = round_up(self.stem_c)                           # 588 -> 640
        pe = take(v + "embeddings.patch_embedding.weight").to(dev, torch.float32)
        pe = pe / torch.tensor(CLIP_STD, device=dev).view(1, 3, 1, 1)
        w["pe"] = op16(torch.nn.functional.pad(pe.reshape(vw, self.stem_c), (0, self.stem_cp - self.stem_c)), dev)
        pos = f32(take(v + "embeddings.position_embedding.weight"), dev)
        self.vemb = torch.empty(self.patches + 1, vw, device=dev)
        self.vemb[0] = f32(take(v + "embeddings.class_embedding"), dev) + pos[0]      # constant class-token row
        w["pos"] = pos[1:].contiguous()
        w["pre.w"], w["pre.b"] = f32(take(v + "pre_layrnorm.weight"), dev), f32(take(v + "pre_layrnorm.bias"), dev)
        for i in range(cfg["v_layers"]):
            p = f"{v}encoder.layers.{i}."
            keys = [k for k in sd if k.startswith(p)]
            if i >= self.v_run:                                          # layers past the selected one never run
                for k in keys:
                    del sd[k]
                continue
            o = f"v{i}."                                                # prenorm_block's names
            w[o + "qkv.w"] = op16(torch.cat([take(p + f"self_attn.{n}_proj.weight").to(dev) for n in "qkv"]), dev)
            w[o + "qkv.b"] = f32(torch.cat([take(p + f"self_attn.{n}_proj.bias").to(dev) for n in "qkv"]), dev)
            for src, dst in (("self_attn.out_proj", "proj"), ("mlp.fc1", "fc1"), ("mlp.fc2", "fc2")):
                w[o + dst + ".w"] = op16(take(p + src + ".weight"), dev)
                w[o + dst + ".b"] = f32(take(p + src + ".bias"), dev)
            for src, dst in (("layer_norm1", "ln1"), ("layer_norm2", "ln2")):
                w[o + dst + ".w"] = f32(take(p + src + ".weight"), dev)
                w[o + dst + ".b"] = f32(take(p + src + ".bias"), dev)
        for k in [k for k in sd if k.startswith(v + "post_layernorm")]:
            del sd[k]
        for i in (0, 2):
            w[f"mm{i}.w"] = op16(take(f"model.mm_projector.{i}.weight"), dev)
            w[f"mm{i}.b"] = f32(take(f"model.mm_projector.{i}.bias"), dev)
        w["embed"] = op16(take("model.embed_tokens.weight"), dev)
        hb = self.bn // 2
        for i in range(cfg["layers"]):
            p, o = f"model.layers.{i}.", f"l{i}."
            w[o + "qkv"] = op16(torch.cat([take(p + f"self_attn.{n}_proj.weight").to(dev, dt) for n in "qkv"]), dev)
            w[o + "o"] = op16(take(p + "self_attn.o_proj.weight"), dev)
            up = take(p + "mlp.up_proj.weight").to(dev, dt).view(f // hb, hb, d)       # values
            gate = take(p + "mlp.gate_proj.weight").to(dev, dt).view(f // hb, hb, d)   # gates
            w[o + "gu"] = torch.cat([up, gate], dim=1).reshape(2 * f, d).contiguous()
            del up, gate
            w[o + "down"] = op16(take(p + "mlp.down_proj.weight"), dev)
            w[o + "ln1"] = f32(take(p + "input_layernorm.weight"), dev)
            w[o + "ln2"] = f32(take(p + "post_attention_layernorm.weight"), dev)
        w["norm"] = f32(take("model.norm.weight"), dev)
        w["lm_head"] = op16(take("lm_head.weight"), dev)
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
        self._seqs: Optional[_Seqs] = None

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
    def generate_list(self, xs: Sequence[torch.Tensor], max_new_tokens: Optional[int] = None,
                      use_graphs: bool = True) -> List[List[int]]:
        """generate for each of up to MAX_SEQS images, decoded together: list i is what generate(xs[i]) returns."""
        B = len(xs)
        if B == 1:
            return [self.generate(xs[0], use_graphs, max_new_tokens)]
        n = self.max_new if max_new_tokens is None else min(max_new_tokens, self.max_new)
        S = self._seq_buffers(B)
        if use_graphs and B not in S.graphs:
            # before the prefills: the capture's eager run is a decode step of whatever the buffers hold
            self.state.copy_(self.state0)
            S.graphs[B] = self._capture(lambda: self._decode_step_seqs(S, B))
        self.prefill_seqs(xs, use_graphs)
        run_step = S.graphs[B].replay if use_graphs else (lambda: self._decode_step_seqs(S, B))
        out: List[List[int]] = [[] for _ in range(B)]
        done = [False] * B
        while True:
            S.tok_host[:B].copy_(S.tok[:B], non_blocking=True)
            torch.cuda.current_stream().synchronize()
            for b in range(B):
                if not done[b]:
                    t = int(S.tok_host[b])
                    out[b].append(t)
                    done[b] = t == self.cfg["eos"] or len(out[b]) >= n
            if all(done):
                return out
            run_step()

    def _seq_buffers(self, B: int) -> _Seqs:
        if not 1 <= B <= self.MAX_SEQS:
            raise ValueError(f"{B} sequences: batched decoding takes 1 .. {self.MAX_SEQS}")
        if self._seqs is None or self._seqs.cap_seqs < B:
            self._seqs = None                       # free the smaller buffers (and their graphs) first
            self._seqs = _Seqs(self, B)
        return self._seqs

    @torch.no_grad()
    def prefill_seqs(self, xs: Sequence[torch.Tensor], use_graphs: bool = True) -> _Seqs:
        """The prefill of each image on its own; its KV rows and first token go to sequence b of the batch buffers.
        Leaves the shared position / length at the first decode step."""
        S = self._seq_buffers(len(xs))
        if use_graphs and self._graphs is None:
            self._graphs = (self._capture(self._prefill), self._capture(self._decode_step))
        run_prefill = self._graphs[0].replay if use_graphs else self._prefill
        L = self.L
        for b, x in enumerate(xs):
            assert x.shape == self.img.shape
            self.img.copy_(x)
            run_prefill()
            S.kc[:, b, :L].copy_(self.kc[:, :L])
            S.vc[:, b, :L].copy_(self.vc[:, :L])
            S.tok[b:b + 1].copy_(self.tok)
        return S

    @torch.no_grad()
    def forced_logits_seqs(self, xs: Sequence[torch.Tensor], tokens: Sequence[Sequence[int]]) -> torch.Tensor:
        """Teacher forcing of B sequences decoded together (eager): [len(tokens[b]) - 1, B, vocab], row i = sequence b's
        logits after feeding tokens[b][:i + 1] (rows 1.. of forced_logits on image b)."""
        B = len(xs)
        S = self.prefill_seqs(xs, use_graphs=False)
        rows = []
        steps = len(tokens[0])
        for i in range(steps - 1):
            S.tok[:B].copy_(torch.tensor([int(t[i]) for t in tokens], dtype=torch.int32))
            self._decode_step_seqs(S, B)
            rows.append(S.logits[:B].clone())
        return torch.stack(rows) if rows else torch.empty(0, B, self.cfg["vocab"], device=self.dev)

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
        heads, ld, vi = cfg["v_heads"], 3 * vw, cfg["v_intermediate"]

        def attend(q, att):
            lib.attention(q, q[:, vw:], q[:, 2 * vw:], att, batch=1, heads=heads, sq=nv, skv=nv, ldq=ld, ldk=ld, ldv=ld,
                          ldo=vw, ws=self.vattn_ws)
        bufs = (self.ln16, self.vqkv16, self.vatt16, self.vhid16)
        for i in range(self.v_run):
            prenorm_block(W, f"v{i}.", t, bufs, nv, vw, vi, (vw, ld, vi), "quick_gelu", cfg["v_eps"], attend)
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

    def _decode_step_seqs(self, S: _Seqs, B: int):
        """_decode_step for sequences 0 .. B-1 of S, all at the shared position."""
        cfg, W = self.cfg, self.w
        d, f, H, V = cfg["hidden"], cfg["intermediate"], cfg["heads"], cfg["vocab"]
        h, x16, qkv, q16, att16, gu16 = S.h[:B], S.x16[:B], S.qkv[:B], S.q16[:B], S.att16[:B], S.gu16[:B]
        lib.embed_gather(W["embed"], V, S.tok, B, d, h, d)
        for i in range(cfg["layers"]):
            o = f"l{i}."
            lib.rmsnorm(h, d, B, d, W[o + "ln1"], x16, d, eps=cfg["rms_eps"])
            lib.gemv_rows(W[o + "qkv"], x16, qkv, M=B, N=3 * d, K=d, ldx=d, ldy=3 * d)
            lib.rope_kv_seqs(qkv, 3 * d, B, H, self.state[0:1], q16, d, S.kc[i], S.vc[i], S.stride,
                             theta=cfg["rope_theta"])
            lib.attention_decode_seqs(q16, d, S.kc[i], S.vc[i], S.stride, B, H, self.cap, self.state[1:2], S.ws, att16, d)
            lib.gemv_rows(W[o + "o"], att16, h, M=B, N=d, K=d, ldx=d, ldy=d, epilogue="residual", residual=h, ldr=d)
            lib.rmsnorm(h, d, B, d, W[o + "ln2"], x16, d, eps=cfg["rms_eps"])
            lib.gemv_rows(W[o + "gu"], x16, gu16, M=B, N=2 * f, K=d, ldx=d, ldy=f, epilogue="swiglu", pack=self.bn)
            lib.gemv_rows(W[o + "down"], gu16, h, M=B, N=d, K=f, ldx=f, ldy=d, epilogue="residual", residual=h, ldr=d)
        lib.rmsnorm(h, d, B, d, W["norm"], x16, d, eps=cfg["rms_eps"])
        lib.gemv_rows(W["lm_head"], x16, S.logits, M=B, N=V, K=d, ldx=d, ldy=V)
        lib.argmax_rows(S.logits, V, B, V, S.tok, advance=self.state)
