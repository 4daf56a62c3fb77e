"""diffbir.dataset on the CPU: the kernel generators, the dataset's __getitem__ and the plain-torch oracle against
the reference fixture (tests/golden/gen_golden_degradation.py), the alias names, and the refusals."""
import math
import random
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent / "golden"))
import gen_golden_degradation as gen  # noqa: E402


@pytest.fixture(scope="module")
def fx(golden_dir):
    return np.load(golden_dir / "degradation_small.npz")


def test_kernel_generators_match_reference(fx):
    from diffbir_b200.dataset import degradation as deg
    for seed in range(4):
        for kt in gen.KERNEL_TYPES:
            for size in (21, 7):
                gen.seed_all(seed)
                k = deg.random_mixed_kernels([kt], [1.0], size, [0.2, 3], [0.2, 3], [-math.pi, math.pi], [0.5, 4],
                                             [1, 2], None)
                assert np.array_equal(k, fx[f"k_{kt}_{size}_{seed}"]), (kt, size, seed)
        gen.seed_all(seed)
        k = deg.circular_lowpass_kernel(np.random.uniform(np.pi / 5, np.pi), 13, pad_to=21)
        assert np.array_equal(k, fx[f"k_sinc_{seed}"])


def test_dataset_getitem_matches_reference(fx, tmp_path):
    from diffbir_b200.dataset.realesrgan import RealESRGANDataset
    ds = RealESRGANDataset(file_metas=gen.write_dataset(tmp_path), **gen.DATASET)
    assert len(ds) == 2
    for i in gen.ITEM_SEEDS:
        gen.seed_all(i)
        item = ds[i % 2]
        assert gen.sha(item["hq"].numpy().tobytes()) == str(fx[f"item_{i}_hq"]), i
        for k in ("kernel1", "kernel2", "sinc_kernel"):
            assert item[k].dtype == torch.float32 and np.array_equal(item[k].numpy(), fx[f"item_{i}_{k}"]), (i, k)
        assert item["txt"] == str(fx[f"item_{i}_txt"])
        assert gen.rng_digests() == list(fx[f"item_{i}_rng"]), i


def _oracle_runs(fx):
    from oracle.degradation import BatchTransform
    from diffbir_b200.dataset.degradation import circular_lowpass_kernel, random_mixed_kernels
    for entry in fx["chosen"]:
        name, seed = str(entry).split(":")
        t, calls = gen.run_calls(lambda: BatchTransform(**gen.CONFIGS[name]), int(seed), random_mixed_kernels,
                                 circular_lowpass_kernel, None)
        yield name, int(seed), t, calls


def test_oracle_transform_matches_reference(fx):
    for name, seed, _, calls in _oracle_runs(fx):
        for j, c in enumerate(calls):
            p = f"tf_{name}_{seed}_{j}"
            assert c["hq"] == str(fx[p + "_hq"]), p
            assert np.array_equal(c["lq"], fx[p + "_lq"]), p
            assert c["txt"] == list(fx[p + "_txt"]), p
            assert c["rng"] == list(fx[p + "_rng"]), p


def test_fixture_seeds_cover_every_branch(fx):
    seen = set()
    for _, _, t, _ in _oracle_runs(fx):
        seen |= set(t.branches)
    assert seen >= gen.ALL_BRANCHES, gen.ALL_BRANCHES - seen
    assert set(fx["branches"]) >= gen.ALL_BRANCHES


def test_alias_names_resolve_to_product():
    import diffbir.dataset.batch_transform as bt
    import diffbir.dataset.degradation as dg
    import diffbir.dataset.diffjpeg as dj
    import diffbir.dataset.file_backend as fb
    import diffbir.dataset.realesrgan as rs
    import diffbir.dataset.utils as ut
    from diffbir_b200 import dataset as p
    import diffbir_b200.dataset.batch_transform  # noqa: F401
    import diffbir_b200.dataset.realesrgan  # noqa: F401
    assert bt.RealESRGANBatchTransform is p.batch_transform.RealESRGANBatchTransform
    assert bt.IdentityBatchTransform is p.batch_transform.IdentityBatchTransform
    assert rs.RealESRGANDataset is p.realesrgan.RealESRGANDataset
    assert dj.DiffJPEG is p.diffjpeg.DiffJPEG and ut.DiffJPEG is p.diffjpeg.DiffJPEG
    assert ut.USMSharp is p.utils.USMSharp and ut.filter2D is p.utils.filter2D
    assert dg.random_mixed_kernels is p.degradation.random_mixed_kernels
    assert fb.HardDiskBackend is p.file_backend.HardDiskBackend
    from diffbir.utils.common import instantiate_from_config
    assert isinstance(instantiate_from_config({"target": "diffbir.dataset.file_backend.HardDiskBackend"}),
                      p.file_backend.HardDiskBackend)


def test_codeformer_dataset_is_refused():
    from diffbir.dataset.codeformer import CodeformerDataset
    with pytest.raises(NotImplementedError, match="no GPU path"):
        CodeformerDataset(file_list="x", file_backend_cfg={}, out_size=512, crop_type="none")


def test_cpu_tensors_are_refused():
    from diffbir_b200.dataset.batch_transform import IdentityBatchTransform, RealESRGANBatchTransform
    from diffbir_b200.dataset.degradation import random_add_gaussian_noise_pt, random_add_poisson_noise_pt
    from diffbir_b200.dataset.diffjpeg import DiffJPEG
    from diffbir_b200.dataset.utils import USMSharp, filter2D
    x = torch.rand(1, 3, 32, 32)
    k = torch.ones(1, 5, 5) / 25
    for call in (lambda: filter2D(x, k), lambda: USMSharp()(x), lambda: DiffJPEG(differentiable=False)(x, 50),
                 lambda: random_add_gaussian_noise_pt(x, (1, 2)), lambda: random_add_poisson_noise_pt(x, (1, 2)),
                 lambda: RealESRGANBatchTransform(**gen.CONFIGS["scalar"])(
                     dict(hq=x, kernel1=k, kernel2=k, sinc_kernel=k, txt=["a"]))):
        with pytest.raises(RuntimeError, match="CUDA engine"):
            call()
    batch = {"hq": x}
    assert IdentityBatchTransform()(batch) is batch
    with pytest.raises(NotImplementedError, match="backward"):
        DiffJPEG()
