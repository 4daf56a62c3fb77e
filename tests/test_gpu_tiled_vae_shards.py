"""-m gpu, one device: the tiled VAE sharded over R emulated ranks in one process. R TiledVae instances share one
VaeEngine, each with its own rank, workspace and a communicator of threads that meet at a barrier; every rank's
output must be bit-identical to the single-rank TiledVae's, and each rank's last_stats must show its share."""
import numpy as np
import pytest
import torch

from diffbir_b200 import arch
from diffbir_b200.utils.synth import make_state_dict
from tests import tilevae_oracle as otv
from tests.gpu_util import no_tf32, run_ranks
from tests.small_cfg import VAE_SMALL

pytestmark = pytest.mark.gpu


def _sharded(base, world, method, x, tile, budget=None):
    from diffbir_b200.engine.vae_tiled import TiledVae

    def run(r, comm):
        tv = TiledVae(base, r, world, comm)
        tv.state_budget = budget
        return getattr(tv, method)(x, tile), dict(tv.last_stats)

    res, _ = run_ranks(world, run)
    return [out for out, _ in res], [st for _, st in res]


def _expected_share(plan, world, n_img, decoder, wave_pixels):
    from diffbir_b200.engine.vae_tiled import tiles_of_ranks
    up = 8 if decoder else 1
    out = []
    for mine in tiles_of_ranks(plan, world):
        waves = 0
        for (th, tw), tiles in plan.classes.items():
            k = len([t for t in tiles if t in mine])
            per = max(1, wave_pixels // (n_img * th * tw * up * up))
            waves += -(-k // per)
        out.append((len(mine), waves))
    return out


def _check(base, single, world, case_input, tile, decoder, budget=None):
    from diffbir_b200.engine.vae import VaeWalk
    from diffbir_b200.engine.vae_tiled import TiledVae, plan_vae_tiles
    method = "decode" if decoder else "encode_moments"
    ref = getattr(single, method)(case_input, tile)
    ref_stats = dict(single.last_stats)
    outs, stats = _sharded(base, world, method, case_input, tile, budget)
    plan = plan_vae_tiles(case_input.shape[2], case_input.shape[3], tile, decoder)
    share = _expected_share(plan, world, case_input.shape[0], decoder, TiledVae.wave_pixels)
    stops = VaeWalk.stops(base.cfg, decoder)
    print(f"{method} {tuple(case_input.shape)} tile {tile}, R={world}: single {ref_stats}; ranks "
          f"{[(s['owned'], s['waves'], s['spills']) for s in stats]}")
    assert ref_stats["exchanges"] == 0 and ref_stats["owned"] == ref_stats["tiles"] == len(plan.in_boxes)
    for r in range(world):
        assert torch.equal(outs[r], ref), f"rank {r}: max diff {(outs[r] - ref).abs().max().item():.3e}"
        assert torch.equal(outs[r].signbit(), ref.signbit())
        st = stats[r]
        assert (st["owned"], st["waves"]) == share[r]
        assert st["tiles"] == len(plan.in_boxes) and st["groupnorms"] == stops and st["exchanges"] == stops + 1
        if budget == 0 and st["owned"]:
            assert st["spills"] > 0
    assert sum(s["owned"] for s in stats) == len(plan.in_boxes)
    return stats


@pytest.fixture(scope="module")
def fx(golden_dir):
    return np.load(golden_dir / "tilevae_small.npz")


@pytest.fixture(scope="module")
def small():
    from diffbir_b200.engine.vae import VaeEngine
    from diffbir_b200.engine.vae_tiled import TiledVae
    no_tf32()
    base = VaeEngine(make_state_dict(arch.vae_shapes(VAE_SMALL), 3), VAE_SMALL, "cuda")
    return base, TiledVae(base)


@pytest.mark.parametrize("world", [2, 3, 5])
@pytest.mark.parametrize("case", ["enc_a", "enc_b", "dec_a", "dec_b"])
def test_emulated_ranks_bit_identical(fx, small, case, world):
    base, single = small
    x = otv.fixture_source(fx, case).cuda()
    _check(base, single, world, x, int(fx[case + "_tile"]), case.startswith("dec"))


def test_more_ranks_than_tiles(fx, small):
    """enc_b has 6 tiles: on 8 ranks two own none and still take part in every exchange."""
    base, single = small
    x = otv.fixture_source(fx, "enc_b").cuda()
    stats = _check(base, single, 8, x, int(fx["enc_b_tile"]), False)
    assert sum(1 for s in stats if s["owned"] == 0) == 2


def test_all_state_staged(fx, small):
    """state_budget 0 on every rank: each stages its own waves through the host, the bits stay."""
    base, single = small
    for case in ("enc_a", "dec_a"):
        x = otv.fixture_source(fx, case).cuda()
        _check(base, single, 3, x, int(fx[case + "_tile"]), case.startswith("dec"), budget=0)


def test_fallbacks_stay_replicated(fx, small):
    """Inputs no larger than 2 * pad + tile run un-tiled on every rank, with no exchange."""
    from diffbir_b200.engine.vae_tiled import TiledVae
    base, _ = small
    x = otv.fixture_source(fx, "enc_fallback").cuda()          # 96 x 120: one tile through the tiled path

    class _NoComm:
        def all_gather(self, t):
            raise AssertionError("a fallback must not exchange")

    tv = TiledVae(base, 1, 3, _NoComm())
    out = tv.encode_moments(x, int(fx["enc_fallback_tile"]))
    assert tv.last_stats["tiles"] == tv.last_stats["owned"] == 1 and tv.last_stats["exchanges"] == 0
    assert torch.equal(out, TiledVae(base).encode_moments(x, int(fx["enc_fallback_tile"])))
    z = torch.randn(1, 4, 30, 20, device="cuda")
    assert torch.equal(tv.decode(z, 8), base.decode(z))


def test_full_config_768x1280_four_ranks():
    """Full SD VAE: 768 x 1280 image with 256-pixel encoder tiles and its 96 x 160 latent with 256-pixel decoder
    tiles, 15 tiles each over 4 emulated ranks."""
    from diffbir_b200.engine.vae import VaeEngine
    from diffbir_b200.engine.vae_tiled import TiledVae
    no_tf32()
    base = VaeEngine(make_state_dict(arch.vae_shapes(arch.VAE_CFG), 77), arch.VAE_CFG, "cuda")
    single = TiledVae(base)
    g = torch.Generator().manual_seed(5)
    img = (torch.rand(1, 3, 768, 1280, generator=g) * 2 - 1).cuda()
    z = (torch.randn(1, 4, 96, 160, generator=g) * 0.8).cuda()
    _check(base, single, 4, img, 256, False)
    _check(base, single, 4, z, 256 // 8, True)
