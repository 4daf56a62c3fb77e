"""OpenCLIP ViT-H text tower (penultimate layer) — supporting component, kept in PyTorch ops
(SURVEY.md §2 row 14: runs twice per image, out of scope for hand-written kernels).
Same role / key layout as the reference's FrozenOpenCLIPEmbedder (model/clip.py:9-61): weights
live under 'model.' (token_embedding, positional_embedding, transformer.resblocks.*, ln_final).
"""
from __future__ import annotations

import gzip
import html
import os
from functools import lru_cache
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from ..engine.common import GraphCache


class TextTower:
    def __init__(self, sd: Dict[str, torch.Tensor], heads: int = 16, layer: str = "penultimate",
                 device="cuda"):
        self.dev = torch.device(device)
        self.sd = {k: v.to(self.dev, torch.float32) for k, v in sd.items() if k != "text_projection"}
        self.heads = heads
        self.skip_last = 1 if layer == "penultimate" else 0
        self.n_layers = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("transformer.resblocks."))
        self.context_length = sd["positional_embedding"].shape[0]
        self.graphs = GraphCache() if self.dev.type == "cuda" else None

    @torch.no_grad()
    def __call__(self, tokens: torch.Tensor) -> torch.Tensor:
        """tokens int64 [B, 77] -> fp32 [B, 77, width] (model/clip.py:37-59). On CUDA the ~280 small
        library kernels of the tower are replayed as one CUDA graph per batch shape."""
        tokens = tokens.to(self.dev)
        if self.graphs is None:
            return self._forward(tokens)
        return self.graphs.run(tuple(tokens.shape), self._forward, tokens)

    def _forward(self, tokens: torch.Tensor) -> torch.Tensor:
        sd = self.sd
        x = sd["token_embedding.weight"][tokens] + sd["positional_embedding"]
        b, n, c = x.shape
        dh = c // self.heads
        for i in range(self.n_layers - self.skip_last):
            p = f"transformer.resblocks.{i}."
            h = F.layer_norm(x, (c,), sd[p + "ln_1.weight"], sd[p + "ln_1.bias"], 1e-5)
            qkv = F.linear(h, sd[p + "attn.in_proj_weight"], sd[p + "attn.in_proj_bias"])
            q, k, v = (t.reshape(b, n, self.heads, dh).transpose(1, 2) for t in qkv.chunk(3, dim=-1))
            o = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(b, n, c)
            x = x + F.linear(o, sd[p + "attn.out_proj.weight"], sd[p + "attn.out_proj.bias"])
            h = F.layer_norm(x, (c,), sd[p + "ln_2.weight"], sd[p + "ln_2.bias"], 1e-5)
            h = F.gelu(F.linear(h, sd[p + "mlp.c_fc.weight"], sd[p + "mlp.c_fc.bias"]))
            x = x + F.linear(h, sd[p + "mlp.c_proj.weight"], sd[p + "mlp.c_proj.bias"])
        return F.layer_norm(x, (c,), sd["ln_final.weight"], sd["ln_final.bias"], 1e-5)


# ------------------------------------------------------------------------------- tokenizer
@lru_cache()
def _bytes_to_unicode():
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, [chr(c) for c in cs]))


class BpeTokenizer:
    """CLIP byte-pair tokenizer (same vocabulary file as open_clip: bpe_simple_vocab_16e6.txt.gz,
    which is data and must be supplied — path via DIFFBIR_BPE_VOCAB or the constructor)."""

    def __init__(self, bpe_path: str, context_length: int = 77):
        import regex as re
        merges = gzip.open(bpe_path).read().decode("utf-8").split("\n")[1:49152 - 256 - 2 + 1]
        merges = [tuple(m.split()) for m in merges]
        self.byte_encoder = _bytes_to_unicode()
        vocab = list(self.byte_encoder.values())
        vocab = vocab + [v + "</w>" for v in vocab] + ["".join(m) for m in merges]
        vocab += ["<start_of_text>", "<end_of_text>"]
        self.encoder = dict(zip(vocab, range(len(vocab))))
        self.ranks = dict(zip(merges, range(len(merges))))
        self.cache = {"<start_of_text>": "<start_of_text>", "<end_of_text>": "<end_of_text>"}
        self.pat = re.compile(r"""<start_of_text>|<end_of_text>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+""",
                              re.IGNORECASE)
        self.context_length = context_length
        self.sot, self.eot = self.encoder["<start_of_text>"], self.encoder["<end_of_text>"]

    def _bpe(self, token):
        if token in self.cache:
            return self.cache[token]
        word = tuple(token[:-1]) + (token[-1] + "</w>",)
        while len(word) > 1:
            pairs = {(word[i], word[i + 1]) for i in range(len(word) - 1)}
            best = min(pairs, key=lambda p: self.ranks.get(p, float("inf")))
            if best not in self.ranks:
                break
            a, b = best
            new, i = [], 0
            while i < len(word):
                if i < len(word) - 1 and word[i] == a and word[i + 1] == b:
                    new.append(a + b)
                    i += 2
                else:
                    new.append(word[i])
                    i += 1
            word = tuple(new)
        out = " ".join(word)
        self.cache[token] = out
        return out

    def __call__(self, texts: List[str]) -> torch.Tensor:
        res = torch.zeros(len(texts), self.context_length, dtype=torch.long)
        for i, text in enumerate(texts):
            text = " ".join(html.unescape(html.unescape(text)).split()).strip().lower()
            ids = [self.sot]
            for tok in self.pat.findall(text):
                tok = "".join(self.byte_encoder[b] for b in tok.encode("utf-8"))
                ids.extend(self.encoder[t] for t in self._bpe(tok).split(" "))
            ids.append(self.eot)
            if len(ids) > self.context_length:
                ids = ids[: self.context_length]
                ids[-1] = self.eot
            res[i, : len(ids)] = torch.tensor(ids)
        return res


class SyntheticTokenizer:
    """Stand-in used only with synthetic checkpoints (no vocabulary file in the sandbox): maps
    words to stable pseudo-ids. Never used silently: ControlLDM requires synthetic_tokenizer=True."""

    def __init__(self, vocab_size: int = 49408, context_length: int = 77):
        self.vocab_size, self.context_length = vocab_size, context_length

    def __call__(self, texts: List[str]) -> torch.Tensor:
        import zlib
        res = torch.zeros(len(texts), self.context_length, dtype=torch.long)
        for i, text in enumerate(texts):
            ids = [self.vocab_size - 2]
            ids += [zlib.crc32(w.encode()) % (self.vocab_size - 2) for w in text.lower().split()]
            ids = ids[: self.context_length - 1] + [self.vocab_size - 1]
            res[i, : len(ids)] = torch.tensor(ids)
        return res


def find_bpe_vocab() -> Optional[str]:
    for p in (os.environ.get("DIFFBIR_BPE_VOCAB"), "weights/bpe_simple_vocab_16e6.txt.gz"):
        if p and os.path.exists(p):
            return p
    return None
