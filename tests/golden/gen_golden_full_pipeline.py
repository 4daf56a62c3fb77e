"""A WHOLE run of the reference at the FULL configuration — BASELINE configs[2]: SwinIRPipeline.run on one 512 x 512 image,
full SwinIR + SD-2.1 UNet + ControlNet + VAE + OpenCLIP text tower (random-init weights from the seeded generator, loaded
through the reference's own loaders), 50-step DDIM (eta 0, batched CFG), cfg 4.0, seed 231, on the CPU in fp32:

    python tests/golden/gen_golden_full_pipeline.py [--oracle] [--spaced] [--v21]   # needs /root/reference; ~10 min of CPU (+ ~10 with --oracle)

-> tests/golden/full_pipeline_ddim.npz (the uint8 result). DDIM with eta 0 draws no per-step noise, so the CPU-drawn x_T
(`torch.manual_seed(231); torch.randn(1, 4, 64, 64)`) is the only randomness and a GPU run can be fed the same one.
`--oracle` also replays the run through the oracle's restatement of the pipeline and prints the difference (too slow for
the CPU test suite).
`--spaced` does the same for configs[1] (50-step spaced sampler, image seed 0); its per-step noise comes from the CPU
generator, which a GPU run cannot reproduce, so that variant only serves the oracle comparison and writes no fixture;
`--v21` uses configs/inference/diffusion_v2.1.yaml (v-parameterization, zero terminal SNR) with the cosine CFG ramp.
The BPE vocabulary file is not in the sandbox: both sides use the hash tokenizer (SyntheticTokenizer, 49 408 entries).
"""
import contextlib
import sys
import time
from pathlib import Path

import numpy as np
import torch
import yaml

sys.path.insert(0, str(Path(__file__).resolve().parent))
from _ref_import import use_reference  # noqa: E402

use_reference()
from diffbir_b200 import arch  # noqa: E402
from diffbir_b200.model.clip import SyntheticTokenizer  # noqa: E402
from diffbir_b200.utils.synth import RUN_DEFAULTS, make_state_dict, synthetic_lq, synthetic_sd_checkpoint  # noqa: E402

OUT = Path(__file__).resolve().parent
REF = Path("/root/reference")


@torch.no_grad()
def main():
    import diffbir.model.clip as rclip
    import diffbir.pipeline as rpipe
    from diffbir.utils.common import instantiate_from_config
    tok = SyntheticTokenizer(arch.CLIP_TEXT_CFG["vocab_size"])
    rclip.tokenize = tok
    rpipe.VRAMPeakMonitor = lambda *a, **k: contextlib.nullcontext()
    load = lambda name: yaml.safe_load(open(REF / "configs" / "inference" / name))      # noqa: E731
    t0 = time.time()
    cldm = instantiate_from_config(load("cldm.yaml")).eval()
    sd = synthetic_sd_checkpoint(arch.UNET_CFG, arch.VAE_CFG, arch.CLIP_TEXT_CFG, 1234)
    unused, missing = cldm.load_pretrained_sd(sd)
    assert all("attn_mask" in k or "logit_scale" in k or "text_projection" in k for k in missing), sorted(missing)[:5]
    csd = make_state_dict(arch.unet_shapes(arch.CONTROLNET_CFG, True), 1237, arch.is_zero_init)
    cldm.load_controlnet_from_ckpt(csd)
    swin = instantiate_from_config(load("swinir.yaml")).eval()
    ssd = make_state_dict(arch.swinir_shapes(arch.SWINIR_CFG), 1238)
    missing_s, unexpected_s = swin.load_state_dict(ssd, strict=False)
    assert not unexpected_s and all(k.endswith(("relative_position_index", "attn_mask")) for k in missing_s)
    v21 = "--v21" in sys.argv
    diffusion = instantiate_from_config(load("diffusion_v2.1.yaml" if v21 else "diffusion.yaml"))
    print(f"reference models built in {time.time() - t0:.0f}s", flush=True)
    spaced = "--spaced" in sys.argv
    lq = synthetic_lq(512, 512, seed=0 if spaced else 3)
    r = dict(RUN_DEFAULTS, sampler_type="spaced" if spaced else "ddim", rescale_cfg=v21)
    pipe = rpipe.SwinIRPipeline(swin, cldm, diffusion, None, "cpu")
    torch.manual_seed(231)
    t0 = time.time()
    y = pipe.run(lq, r["steps"], r["strength"], r["cleaner_tiled"], r["cleaner_tile_size"], r["cleaner_tile_stride"],
                 r["vae_encoder_tiled"], r["vae_encoder_tile_size"], r["vae_decoder_tiled"], r["vae_decoder_tile_size"],
                 r["cldm_tiled"], r["cldm_tile_size"], r["cldm_tile_stride"], r["pos_prompt"], r["neg_prompt"],
                 r["cfg_scale"], r["start_point_type"], r["sampler_type"], r["noise_aug"], r["rescale_cfg"], r["s_churn"],
                 r["s_tmin"], r["s_tmax"], r["s_noise"], r["eta"], r["order"])
    print(f"reference SwinIRPipeline.run, full config, 50-step {r['sampler_type']}: {time.time() - t0:.0f}s, output {y.shape} {y.dtype} "
          f"mean {y.mean():.2f} std {y.std():.2f}", flush=True)
    if not spaced and not v21:
        np.savez_compressed(OUT / "full_pipeline_ddim.npz", out=y)
        print("wrote full_pipeline_ddim.npz", flush=True)
    if "--oracle" not in sys.argv:
        return
    del cldm, swin, pipe
    from oracle import cldm as ocl
    from oracle import sampling as osm
    from oracle import swinir as osw
    part = lambda pre: {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}      # noqa: E731
    usd, vsd, clipsd = part("model.diffusion_model."), part("first_stage_model."), part("cond_stage_model.model.")
    scales = {"s": [1.0] * 13}
    torch.manual_seed(231)
    t0 = time.time()
    out = osm.swinir_pipeline_run(
        lq, cleaner=lambda im: osw.swinir_forward(ssd, im), encode_img=lambda im: ocl.vae_encode_mode(vsd, im, 0.18215),
        encode_txt=lambda txt: ocl.clip_text_encode(clipsd, tok(txt), heads=arch.CLIP_TEXT_CFG["heads"]),
        decode=lambda z: ocl.vae_decode(vsd, z / 0.18215),
        model=lambda x, t, c: ocl.cldm_forward(usd, csd, x, t, c["c_txt"], c["c_img"], scales["s"]),
        betas=diffusion.betas, parameterization=diffusion.parameterization, rescale_cfg=r["rescale_cfg"], steps=50, strength=1.0, pos_prompt=r["pos_prompt"], neg_prompt=r["neg_prompt"],
        cfg_scale=4.0, sampler=r["sampler_type"], set_strength=lambda s: scales.update(s=[s] * 13))
    diff = np.abs(out.astype(int) - y.astype(int))
    mse = (diff.astype(np.float64) ** 2).mean()
    psnr = float("inf") if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)
    print(f"oracle pipeline replay ({time.time() - t0:.0f}s) vs the reference run, full config, 50-step {r['sampler_type']}{' (v2.1 diffusion, CFG ramp)' if v21 else ''}: "
          f"{100 * (diff > 0).mean():.3f} % of pixels differ, max |diff| {diff.max()}, PSNR {psnr:.1f} dB", flush=True)


if __name__ == "__main__":
    main()
