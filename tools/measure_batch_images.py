"""Folder throughput of `inference.py --batch_images N` and the batched LLaVA decode step.

  python tools/measure_batch_images.py [--images 16] [--steps 50] [--caption_tokens 40] [--rounds 3] [--repeats 7]

One process builds the CLI's loop on synthetic weights (full SD-2.1 config, v2.1 recipe, 128^2 inputs x4 = 512^2
outputs, spaced sampler, CFG 4) and restores a folder of `--images` inputs at N = 1, 4 and 8, without a captioner and
with `--captioner llava --llava_bit 16` (synthetic LLaVA-1.5-7B). N = 1 runs the ControlNet+UNet engine with its
default plans, as `python inference.py` does; N > 1 with the batch-invariant plans it pins. Random LLaVA weights
almost never emit EOS, so every caption is cut at `--caption_tokens` tokens (about the length of a real short
description) to keep the captioner's share realistic. Each configuration is warmed up on the folder once, then
timed `--rounds` times in alternation (host clock around a run that ends in a device synchronise, PNG writes
included); the median round is reported as MPix/s of output, with the slowest and fastest rounds.

Then the LLaVA decode step alone: one CUDA-graph replay per token for B = 1, 2, 4, 8 sequences, device events over
100 replays from the prompt's end, `--repeats` windows taken in alternation over B; the median window per B is
reported, and the B = 8 / B = 1 ratio of each repeat (median, min, max). Prints one JSON line with the card's name
and power limit."""
import argparse
import json
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import torch  # noqa: E402
from PIL import Image  # noqa: E402

import inference as cli  # noqa: E402
from diffbir_b200.inference import BSRInferenceLoop  # noqa: E402
from diffbir_b200.utils.caption import EmptyCaptioner  # noqa: E402
from diffbir_b200.utils.synth import synthetic_lq  # noqa: E402


def median(v):
    v = sorted(v)
    n = len(v)
    return v[n // 2] if n % 2 else (v[n // 2 - 1] + v[n // 2]) / 2


def decode_step_ms(eng, B: int, reps: int = 100) -> float:
    """One window: the prefill(s), then `reps` decode-step replays timed with device events."""
    xs = [torch.rand(1, 3, 336, 336, generator=torch.Generator().manual_seed(b)).cuda() for b in range(B)]
    if B == 1:
        eng.generate(xs[0], max_new_tokens=2)
        step = eng._graphs[1].replay
        eng._graphs[0].replay()
    else:
        eng.generate_list(xs, max_new_tokens=2)
        S = eng.prefill_seqs(xs)
        step = S.graphs[B].replay
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        step()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=16)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--caption_tokens", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=7)
    opt = ap.parse_args()
    assert torch.cuda.is_available(), "measure_batch_images.py needs a CUDA device"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    root = Path(tempfile.mkdtemp(prefix="measure_batch_images_"))
    try:
        (root / "in").mkdir()
        for i in range(opt.images):
            Image.fromarray(synthetic_lq(128, 128, seed=i)[0]).save(root / "in" / f"{i:03d}.png")
        flags = ["--task", "sr", "--version", "v2.1", "--upscale", "4", "--sampler", "spaced", "--steps", str(opt.steps),
                 "--cfg_scale", "4.0", "--synthetic", "--input", str(root / "in")]
        loop = BSRInferenceLoop(cli.parse_args(flags + ["--batch_images", "4", "--output", "-"]))
        loop.pipeline.cldm._build()
        eng = loop.pipeline.cldm.engine
        captioners = {"none": EmptyCaptioner("cuda")}
        loop.args = cli.parse_args(flags + ["--captioner", "llava", "--llava_bit", "16", "--output", "-"])
        loop.load_captioner()
        captioners["llava"] = loop.captioner
        llava = loop.captioner.engine
        llava.max_new = opt.caption_tokens
        configs = [(cap, n) for cap in ("none", "llava") for n in (1, 4, 8)]

        def run(cap, n, out):
            loop.args = cli.parse_args(flags + ["--captioner", cap, "--llava_bit", "16", "--batch_images", str(n),
                                                "--output", str(out)])
            loop.captioner = captioners[cap]
            eng.deterministic = n > 1           # N = 1: the plain CLI's plans
            cli.set_seed(loop.args.seed)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            loop.run()
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        times = {c: [] for c in configs}
        for c in configs:                        # warm-up: every graph and plan of the timed runs
            run(*c, root / "warm")
            shutil.rmtree(root / "warm")
        for r in range(opt.rounds):
            for c in configs:
                times[c].append(run(*c, root / f"out{r}"))
                shutil.rmtree(root / f"out{r}")
        mpix = opt.images * 512 * 512 / 1e6
        res = dict(card=card, images=opt.images, size="512x512", steps=opt.steps, caption_tokens=opt.caption_tokens,
                   rounds=opt.rounds)
        for cap, n in configs:
            t = times[(cap, n)]
            res[f"mpix_s_{cap}_n{n}"] = round(mpix / median(t), 3)
            res[f"mpix_s_{cap}_n{n}_slowest_fastest"] = [round(mpix / max(t), 3), round(mpix / min(t), 3)]
        for cap in ("none", "llava"):
            for n in (4, 8):
                res[f"speedup_{cap}_n{n}"] = round(res[f"mpix_s_{cap}_n{n}"] / res[f"mpix_s_{cap}_n1"], 3)
        llava.max_new = 512
        windows = {b: [] for b in (1, 2, 4, 8)}
        for _ in range(opt.repeats):
            for b in windows:
                windows[b].append(decode_step_ms(llava, b))
        for b, ms in windows.items():
            res[f"llava_decode_step_ms_b{b}"] = round(median(ms), 3)
        ratios = [w8 / w1 for w8, w1 in zip(windows[8], windows[1])]
        res["llava_decode_b8_over_b1"] = round(median(ratios), 3)
        res["llava_decode_b8_over_b1_min_max"] = [round(min(ratios), 3), round(max(ratios), 3)]
        res["decode_repeats"] = opt.repeats
        print(json.dumps(res))
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
