"""-m gpu, one device: the row-sharded VAE over R emulated ranks in one process. R ShardedVae instances share one
VaeEngine, each with its own rank, workspace and a communicator of threads that meet at a barrier. Every rank must
return the same bits, in the single-GPU engine's shape and within the fp16 noise floor of its result: the merged
GroupNorm statistics differ from the single-GPU ones in their last bits, which flips 16-bit operand roundings, while a
halo or ownership bug shows up as O(1) errors along the band borders."""
import pytest
import torch

from diffbir_b200 import arch
from diffbir_b200.utils.synth import make_state_dict
from tests.gpu_util import no_tf32, rel_err, rel_rms, run_ranks
from tests.small_cfg import VAE_SMALL

pytestmark = pytest.mark.gpu

CFGS = dict(small=(VAE_SMALL, 3), full=(arch.VAE_CFG, 77))
# (config, ranks, images, image height, image width): heights of whole latent rows, at least 2 per rank, as
# ShardedVae.usable asks
CASES = [
    ("small", 2, 2, 64, 96),
    ("small", 3, 1, 48, 40),        # a 6 x 5 latent: 30 tokens in the mid attention, not a multiple of 8
    ("small", 4, 1, 128, 48),
    ("full", 4, 1, 1024, 256),
]


def case_inputs(n, h, w):
    g = torch.Generator().manual_seed(h * w + n)
    img = (torch.rand(n, 3, h, w, generator=g) * 2 - 1).cuda()
    z = (torch.randn(n, 4, h // 8, w // 8, generator=g) * 0.8).cuda()
    return img, z


def sharded(base, world, method, x):
    """Every rank's ShardedVae(base).method(x), and the hub that carried their all-gathers."""
    from diffbir_b200.engine.vae_sharded import ShardedVae
    return run_ranks(world, lambda r, comm: getattr(ShardedVae(base, r, world, comm), method)(x))


@pytest.fixture(scope="module")
def engines():
    from diffbir_b200.engine.vae import VaeEngine
    no_tf32()
    made = {}

    def get(name):
        if name not in made:
            cfg, seed = CFGS[name]
            made[name] = VaeEngine(make_state_dict(arch.vae_shapes(cfg), seed), cfg, "cuda")
        return made[name]
    return get


@pytest.mark.parametrize("method", ["encode_moments", "decode"])
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-R{c[1]}-n{c[2]}-{c[3]}x{c[4]}")
def test_row_shards_match_one_gpu(engines, case, method):
    name, world, n, h, w = case
    base = engines(name)
    img, z = case_inputs(n, h, w)
    x = img if method == "encode_moments" else z
    ref = getattr(base, method)(x)
    outs, hub = sharded(base, world, method, x)
    rel, rms = rel_err(outs[0], ref), rel_rms(outs[0], ref)
    print(f"{method} {tuple(x.shape)} over {world} ranks: max rel {rel:.2e}, rel rms {rms:.2e}, "
          f"{len(hub.shapes[0])} all-gathers per rank")
    for r in range(world):
        assert torch.equal(outs[r], outs[0]), f"rank {r} differs from rank 0"
    assert outs[0].shape == ref.shape
    assert rel < 1e-2 and rms < 4e-3
