"""The two v2 recipes at FULL width, reference vs the product's host code (no fixture, a log):

    python tests/golden/gen_golden_full_recipes.py      # needs /root/reference; ~20 min of CPU

  * blind super-resolution: BSRNetPipeline (23-block RRDBNet x4 on a 128 x 160 image -> 512 x 640) + DPM-Solver++ m2, eps
  * blind denoising: SCUNetPipeline (28-block SCUNet on a 512 x 512 image) + EDM dpm++_2m on the v / zero-SNR diffusion

each 20 steps, cfg 4.0, seed 231, all networks at the sizes of configs/inference/*.yaml with seeded random-init weights.
The reference's own pipeline runs first; then this package's pipeline + sampler classes run with the oracle networks
plugged in where the kernel engines sit (the harness of tests/test_oracle_golden.py), and the uint8 images are compared.
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

REF = Path("/root/reference")
STEPS = 20


@torch.no_grad()
def main():
    import diffbir.model.clip as rclip
    import diffbir.pipeline as rpipe
    from diffbir.utils.common import instantiate_from_config
    tok = SyntheticTokenizer(arch.CLIP_TEXT_CFG["vocab_size"])
    rclip.tokenize = tok
    rpipe.VRAMPeakMonitor = lambda *a, **k: contextlib.nullcontext()
    load = lambda name: yaml.safe_load(open(REF / "configs" / "inference" / name))      # noqa: E731
    cldm = instantiate_from_config(load("cldm.yaml")).eval()
    sd = synthetic_sd_checkpoint(arch.UNET_CFG, arch.VAE_CFG, arch.CLIP_TEXT_CFG, 1234)
    cldm.load_pretrained_sd(sd)
    csd = make_state_dict(arch.unet_shapes(arch.CONTROLNET_CFG, True), 1237, arch.is_zero_init)
    cldm.load_controlnet_from_ckpt(csd)
    rr = instantiate_from_config(load("bsrnet.yaml")).eval()
    rsd = make_state_dict(arch.rrdbnet_shapes(arch.RRDBNET_CFG), 78)
    rr.load_state_dict(rsd, strict=True)
    scu = instantiate_from_config(load("scunet.yaml")).eval()
    scsd = make_state_dict(arch.scunet_shapes(arch.SCUNET_CFG), 79)
    scu.load_state_dict(scsd, strict=True)
    d_eps = instantiate_from_config(load("diffusion.yaml"))
    d_v = instantiate_from_config(load("diffusion_v2.1.yaml"))
    cases = (("BSRNetPipeline + dpm++_m2 (eps)", lambda: rpipe.BSRNetPipeline(rr, cldm, d_eps, None, "cpu", 4.0), synthetic_lq(128, 160, seed=3), "dpm++_m2"),
             ("SCUNetPipeline + edm_dpm++_2m (v, zero SNR)", lambda: rpipe.SCUNetPipeline(scu, cldm, d_v, None, "cpu"), synthetic_lq(512, 512, seed=3), "edm_dpm++_2m"))
    refs = []
    for name, make, lq, sampler in cases:
        r = dict(RUN_DEFAULTS, steps=STEPS, sampler_type=sampler)
        torch.manual_seed(231)
        t0 = time.time()
        y = make().run(lq, r["steps"], r["strength"], r["cleaner_tiled"], r["cleaner_tile_size"], r["cleaner_tile_stride"],
                       r["vae_encoder_tiled"], r["vae_encoder_tile_size"], r["vae_decoder_tiled"], r["vae_decoder_tile_size"],
                       r["cldm_tiled"], r["cldm_tile_size"], r["cldm_tile_stride"], r["pos_prompt"], r["neg_prompt"],
                       r["cfg_scale"], r["start_point_type"], r["sampler_type"], r["noise_aug"], r["rescale_cfg"], r["s_churn"],
                       r["s_tmin"], r["s_tmax"], r["s_noise"], r["eta"], r["order"])
        print(f"reference {name}, full config, {STEPS} steps: {time.time() - t0:.0f}s, output {y.shape} mean {y.mean():.2f} std {y.std():.2f}", flush=True)
        refs.append(y)
    del cldm, rr, scu
    # ---- this package's host code on the oracle networks
    sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
    from diffbir_b200.model import Diffusion
    from diffbir_b200.pipeline import BSRNetPipeline, SCUNetPipeline
    from oracle import bsrnet as ob
    from oracle import scunet as osc
    from tests.test_oracle_golden import _OracleCldm
    part = lambda pre: {k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)}      # noqa: E731
    ocldm = _OracleCldm(part("model.diffusion_model."), csd, part("first_stage_model."), part("cond_stage_model.model."), tok,
                        arch.CLIP_TEXT_CFG["heads"])
    mk = lambda p, z: Diffusion(linear_start=0.00085, linear_end=0.0120, timesteps=1000, parameterization=p, zero_snr=z)   # noqa: E731
    mine = ((lambda: BSRNetPipeline(lambda im: ob.rrdbnet_forward(rsd, im), ocldm, mk("eps", False), None, "cpu", upscale=4.0)),
            (lambda: SCUNetPipeline(lambda im: osc.scunet_forward(scsd, im), ocldm, mk("v", True), None, "cpu")))
    for (name, _, lq, sampler), make, ref in zip(cases, mine, refs):
        torch.manual_seed(231)
        t0 = time.time()
        out = make().run(lq, **dict(RUN_DEFAULTS, steps=STEPS, sampler_type=sampler))
        diff = np.abs(out.astype(int) - ref.astype(int))
        mse = (diff.astype(np.float64) ** 2).mean()
        psnr = float("inf") if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)
        print(f"product host code + oracle networks ({time.time() - t0:.0f}s) vs the reference run, {name}: "
              f"{100 * (diff > 0).mean():.3f} % of pixels differ, max |diff| {diff.max()}, PSNR {psnr:.1f} dB", flush=True)


if __name__ == "__main__":
    main()
