"""Generates tests/golden/tilevae_small.npz by running the REFERENCE Tiled-VAE hook (utils/tilevae/tilevae.py,
non-fast mode with color_fix=True, exactly as model/cldm.py:92-141 builds it) on the VAE_SMALL weights, in fp64.

    python tests/golden/gen_golden_tilevae.py

Contents:
* plan_{enc,dec}_{h}_{w}_{tile}_{in,out}: VAEHook.split_tiles boxes ([x0, x1, y0, y1] rows) over a grid of sizes;
* enc_*: the input's (seed, shape, range) for tests/tilevae_oracle.fixture_input, which rebuilds it, with its
  fp64 sum as a check; the tile size and the moments (quant_conv of the hook);
* dec_*: the same for the latent (already divided by the scale factor), the tile size in latent pixels and the
  decoded image, kept at every `dec_stride`-th pixel in both directions (5 is coprime with the x8 output grid, so
  every tile seam is sampled);
* enc_fallback: an input no larger than 2 * pad + tile, which the hook runs un-tiled.
"""
import contextlib
import io
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "oracle" / "_shims"))
sys.path.insert(0, str(Path(__file__).resolve().parent))
from _ref_import import use_reference  # noqa: E402

use_reference()

from diffbir_b200 import arch  # noqa: E402
from diffbir_b200.utils.synth import make_state_dict  # noqa: E402
from tests.small_cfg import VAE_SMALL  # noqa: E402
from tests.tilevae_oracle import fixture_input  # noqa: E402

OUT = Path(__file__).resolve().parent
DEC_STRIDE = 5
# encoder inputs are multiples of 8 (the pipeline pads them so)
PLAN_GRID = [(h, w, t) for h in (64, 96, 136, 200, 328) for w in (72, 200, 328, 520) for t in (32, 64, 96)]
PLAN_GRID_DEC = [(h, w, t) for h in (20, 26, 40, 64, 97) for w in (23, 37, 56, 128) for t in (8, 12, 16, 32)]


@torch.no_grad()
def main():
    import diffbir.model  # noqa: F401  (before utils.tilevae: the other order is a circular import)
    from diffbir.model.vae import AutoencoderKL
    from diffbir.utils.tilevae import VAEHook

    vcfg = dict(ddconfig=dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3,
                              ch=VAE_SMALL["ch"], ch_mult=list(VAE_SMALL["ch_mult"]),
                              num_res_blocks=VAE_SMALL["num_res_blocks"], attn_resolutions=[], dropout=0.0),
                embed_dim=4)
    vae = AutoencoderKL(**vcfg).eval()
    vae.load_state_dict(make_state_dict(arch.vae_shapes(VAE_SMALL), 3), strict=True)
    vae.double()        # fp64 reference: the fixture carries the hook's semantics, not fp32 rounding noise

    def hook(net, tile, dec):
        return VAEHook(net, tile_size=tile, is_decoder=dec, fast_decoder=False, fast_encoder=False, color_fix=True)

    quiet = contextlib.redirect_stdout(io.StringIO())
    out = {"dec_stride": np.int64(DEC_STRIDE)}
    with quiet:
        for grid, dec in ((PLAN_GRID, False), (PLAN_GRID_DEC, True)):
            for h, w, t in grid:
                ins, outs = hook(None, t, dec).split_tiles(h, w)
                key = f"plan_{'dec' if dec else 'enc'}_{h}_{w}_{t}"
                out[key + "_in"] = np.array(ins, dtype=np.int32)
                out[key + "_out"] = np.array(outs, dtype=np.int32)

        def source(name, seed, shape, lo, hi):
            x = fixture_input(seed, shape, lo, hi)
            out.update({f"{name}_seed": np.int64(seed), f"{name}_shape": np.array(shape, np.int64),
                        f"{name}_range": np.array([lo, hi], np.float64), f"{name}_sum": np.float64(x.double().sum())})
            return x.double()

        for name, (seed, n, h, w, t) in dict(enc_a=(31, 1, 200, 328, 64), enc_b=(32, 2, 136, 200, 48),
                                             enc_fallback=(33, 1, 96, 120, 64)).items():
            img = source(name, seed, (n, 3, h, w), -1.0, 1.0)
            mom = vae.quant_conv(hook(vae.encoder, t, False)(img).double())
            out.update({f"{name}_tile": np.int64(t), f"{name}_moments": mom.float().numpy()})
        for name, (seed, n, h, w, t) in dict(dec_a=(41, 1, 40, 56, 16), dec_b=(42, 2, 26, 37, 8)).items():
            z = source(name, seed, (n, 4, h, w), -2.0, 2.0)
            x = hook(vae.decoder, t, True)(vae.post_quant_conv(z))
            out.update({f"{name}_tile": np.int64(t),
                        f"{name}_dec": x[..., ::DEC_STRIDE, ::DEC_STRIDE].float().contiguous().numpy()})
    np.savez_compressed(OUT / "tilevae_small.npz", **out)
    for k in sorted(out):
        if not k.startswith("plan_"):
            print(k, getattr(out[k], "shape", out[k]))
    print(f"{(OUT / 'tilevae_small.npz').stat().st_size} bytes")


if __name__ == "__main__":
    main()
