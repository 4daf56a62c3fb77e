"""LLaVA-1.5-7B captioner (LlavaEngine) at the full size with synthetic weights (timings do not depend on the values):

- the card and its power limit;
- vision tower + projector ms and LLM prefill ms (CUDA-graph replays, device events, median);
- ms per decode token over >= 200 tokens: the graph replays back to back, and the captioner's loop with its pinned
  token copy and host synchronisation after every replay (the difference is the per-token EOS check);
- the bytes a decode step must read (weights + KV cache at the mean length) and the rate achieved, against a
  measured device-to-device copy;
- the device memory the engine adds;
- the decode step with dbir_gemv against the same step with dbir_gemm at M = 1 (split-K workspace, its own plans),
  in alternating windows of the same run.

    python tools/measure_llava.py [--tokens 256] [--rounds 5]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def event_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def decode_step_gemm(eng, ws):
    """The decode step with every matrix-vector product as a dbir_gemm at M = 1 (split-K allowed)."""
    from diffbir_b200 import lib
    cfg, W = eng.cfg, eng.w
    d, f, H = cfg["hidden"], cfg["intermediate"], cfg["heads"]
    h, x16 = eng.h[:1], eng.x16[:1]
    qkv, q16, att16, gu16 = eng.qkv[:1], eng.q16[:1], eng.att16[:1], eng.gu16[:1]
    lib.embed_gather(W["embed"], cfg["vocab"], eng.tok, 1, d, h, d)
    for i in range(cfg["layers"]):
        o = f"l{i}."
        lib.rmsnorm(h, d, 1, d, W[o + "ln1"], x16, d, eps=cfg["rms_eps"])
        lib.gemm(x16, W[o + "qkv"], qkv, M=1, N=3 * d, K=d, splitk_ws=ws)
        lib.rope_kv(qkv, 3 * d, 1, H, eng.state[0:1], q16, d, eng.kc[i], eng.vc[i], theta=cfg["rope_theta"])
        lib.attention_decode(q16, eng.kc[i], eng.vc[i], H, eng.cap, eng.state[1:2], eng.dec_ws, att16)
        lib.gemm(att16, W[o + "o"], h, M=1, N=d, K=d, residual=h, splitk_ws=ws)
        lib.rmsnorm(h, d, 1, d, W[o + "ln2"], x16, d, eps=cfg["rms_eps"])
        lib.gemm(x16, W[o + "gu"], gu16, M=1, N=2 * f, K=d, geglu=2, force_bn=eng.bn, splitk_ws=ws)
        lib.gemm(gu16, W[o + "down"], h, M=1, N=d, K=f, residual=h, splitk_ws=ws)
    lib.rmsnorm(h, d, 1, d, W["norm"], x16, d, eps=cfg["rms_eps"])
    lib.gemm(x16, W["lm_head"], eng.logits[None], M=1, N=cfg["vocab"], K=d, splitk_ws=ws)
    lib.argmax(eng.logits, cfg["vocab"], eng.tok, advance=eng.state)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "measure_llava.py needs a CUDA device"
    assert a.tokens >= 200
    from diffbir_b200 import arch, lib
    from diffbir_b200.engine.llava import LlavaEngine
    from diffbir_b200.utils.caption import ByteTokenizer, llava_prompt_ids
    from diffbir_b200.utils.synth import synthetic_llava
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    cfg = dict(arch.LLAVA_CFG)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    eng = LlavaEngine(synthetic_llava(cfg, 1), llava_prompt_ids(ByteTokenizer()), cfg, max_new_tokens=a.tokens + 8)
    torch.cuda.synchronize()
    load_s = time.perf_counter() - t0
    x = torch.rand(1, 3, 336, 336, generator=torch.Generator().manual_seed(0)).cuda()
    eng.generate(x, max_new_tokens=4)                 # captures the prefill and decode graphs
    resident = torch.cuda.memory_allocated() - base
    peak = torch.cuda.max_memory_allocated() - base

    # vision + projector as a graph of its own; the prefill graph holds them too
    feats = torch.empty(eng.patches, cfg["hidden"], device="cuda")

    def vision():
        eng._vision()
        eng._project(feats)
    vision()
    torch.cuda.synchronize()
    gv = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gv):
        vision()
    gp, gd = eng._graphs
    vis_ms = sorted(event_ms(gv.replay, 10) for _ in range(a.rounds))[a.rounds // 2]
    pre_ms = sorted(event_ms(gp.replay, 5) for _ in range(a.rounds))[a.rounds // 2]

    # decode: graph replays back to back (no host sync) and the captioner's loop (sync + pinned copy per token)
    def replays():
        gp.replay()
        for _ in range(a.tokens):
            gd.replay()
    raw = []
    loop = []
    for _ in range(a.rounds):
        gp.replay()
        torch.cuda.synchronize()
        raw.append(event_ms(lambda: [gd.replay() for _ in range(a.tokens)], 1) / a.tokens)
        gp.replay()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.tokens):
            gd.replay()
            eng.tok_host.copy_(eng.tok, non_blocking=True)
            torch.cuda.current_stream().synchronize()
        loop.append((time.perf_counter() - t0) * 1e3 / a.tokens)
    raw_ms, loop_ms = sorted(raw)[a.rounds // 2], sorted(loop)[a.rounds // 2]

    # bytes a decode step reads: every LLM weight once (embedding: one row), KV rows at the mean length
    d, H = cfg["hidden"], cfg["heads"]
    es = torch.finfo(lib.operand_dtype()).bits // 8
    wbytes = sum(t.numel() * t.element_size() for k, t in eng.w.items() if k.startswith("l") or k in ("lm_head", "norm"))
    wbytes += d * es
    mean_len = eng.L + a.tokens / 2
    kv = 2 * cfg["layers"] * mean_len * H * 128 * es
    step_bytes = wbytes + kv
    buf = torch.empty(2 ** 30, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(buf)
    dst.copy_(buf)
    copy_ms = sorted(event_ms(lambda: dst.copy_(buf), 10) for _ in range(a.rounds))[a.rounds // 2]
    copy_gbs = 2 * buf.numel() / copy_ms / 1e6                  # read + write
    del buf, dst

    # GEMV vs GEMM at M = 1, alternating windows
    ws = torch.zeros(256 * 2 ** 20, dtype=torch.uint8, device="cuda")
    gp.replay()
    decode_step_gemm(eng, ws)                         # eager: dbir_gemm picks its plans outside the capture
    torch.cuda.synchronize()
    gg = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gg):
        decode_step_gemm(eng, ws)
    gemv_t, gemm_t = [], []
    n = 100
    for _ in range(a.rounds):
        gp.replay()
        gemv_t.append(event_ms(gd.replay, n))
        gp.replay()
        gemm_t.append(event_ms(gg.replay, n))
    gemv_ms, gemm_ms = sorted(gemv_t)[a.rounds // 2], sorted(gemm_t)[a.rounds // 2]

    res = dict(card=card, operands=str(lib.operand_dtype()), prompt_tokens=eng.L, weights_load_s=round(load_s, 1),
               vision_projector_ms=round(vis_ms, 3), prefill_total_ms=round(pre_ms, 3),
               llm_prefill_ms=round(pre_ms - vis_ms, 3), decode_tokens=a.tokens,
               decode_ms_per_token_graph=round(raw_ms, 4), decode_ms_per_token_with_eos_check=round(loop_ms, 4),
               eos_check_ms_per_token=round(loop_ms - raw_ms, 4),
               step_bytes_gb=round(step_bytes / 1e9, 3), weight_bytes_gb=round(wbytes / 1e9, 3),
               kv_bytes_gb_at_mean_len=round(kv / 1e9, 3), achieved_gbs=round(step_bytes / raw_ms / 1e6, 1),
               d2d_copy_gbs=round(copy_gbs, 1), achieved_over_copy=round(step_bytes / raw_ms / 1e6 / copy_gbs, 3),
               added_resident_gib=round(resident / 2 ** 30, 2), added_peak_gib=round(peak / 2 ** 30, 2),
               decode_step_gemv_ms=round(gemv_ms, 4), decode_step_gemm_m1_ms=round(gemm_ms, 4),
               gemm_over_gemv=round(gemm_ms / gemv_ms, 3), rounds=a.rounds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
