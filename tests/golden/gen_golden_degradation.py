"""Fixture for diffbir.dataset, produced by the REFERENCE modules (dataset/degradation.py, batch_transform.py,
realesrgan.py) on the CPU:

    python tests/golden/gen_golden_degradation.py      # needs /root/reference; writes degradation_small.npz

- `k_<type>_<seed>`: random_mixed_kernels of each kernel type (size 21 and 7) and circular_lowpass_kernel.
- `item_<i>_*`: RealESRGANDataset.__getitem__ over a two-image parquet list of synthetic PNGs (rebuilt by
  `write_dataset` below, which the test calls too), with the v2.1 kernel settings; hq as a SHA-1.
- `tf_<cfg>_<call>_*`: RealESRGANBatchTransform calls on one instance per configuration (queue of two batches,
  so the first two calls fill it and the next two draw from it), 2 x 96^2 batches. lq is stored as its 8-bit
  levels, hq as the SHA-1 of its fp32 bytes, and the Python / numpy / torch-CPU generator states after each call
  as SHA-1 digests. The seeds are chosen (with the oracle's branch recorder) so that together they take every
  branch; `branches` lists them.
"""
import hashlib
import math
import pickle
import random
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from _ref_import import ROOT, use_reference  # noqa: E402

OUT = Path(__file__).resolve().parent
SIZE, BATCH, CALLS = 96, 2, 4
KERNEL_TYPES = ["iso", "aniso", "generalized_iso", "generalized_aniso", "plateau_iso", "plateau_aniso"]
V21 = dict(use_sharpener=True, queue_size=2 * BATCH, resize_prob=[0.2, 0.7, 0.1], resize_range=[0.15, 1.5],
           gaussian_noise_prob=0.5, noise_range=[1, 30], poisson_scale_range=[0.05, 3], gray_noise_prob=0.4,
           jpeg_range=[30, 95], second_blur_prob=0.8, resize_prob2=[0.3, 0.4, 0.3],
           resize_range2=[0.3, 1.2], gaussian_noise_prob2=0.5, noise_range2=[1, 25], poisson_scale_range2=[0.05, 2.5],
           gray_noise_prob2=0.4, jpeg_range2=[30, 95])
# stage2_scale 4 (v2.1) needs ~150 px so the smallest stage-2 image still exceeds the 21-tap reflect pad
CONFIGS = {"scalar": dict(V21, stage2_scale=2), "range": dict(V21, stage2_scale=[1.5, 2.5])}
DATASET = dict(p_long_prompt=0.2, file_backend_cfg={"target": "diffbir.dataset.file_backend.HardDiskBackend"},
               out_size=64, crop_type="none", use_hflip=True, use_rot=True, blur_kernel_size=21,
               kernel_list=KERNEL_TYPES, kernel_prob=[0.45, 0.25, 0.12, 0.03, 0.12, 0.03], sinc_prob=0.1,
               blur_sigma=[0.2, 3], betag_range=[0.5, 4], betap_range=[1, 2], blur_kernel_size2=21,
               kernel_list2=KERNEL_TYPES, kernel_prob2=[0.45, 0.25, 0.12, 0.03, 0.12, 0.03], sinc_prob2=0.1,
               blur_sigma2=[0.2, 1.5], betag_range2=[0.5, 4], betap_range2=[1, 2], final_sinc_prob=0.8,
               p_empty_prompt=0.2)
ITEM_SEEDS = list(range(12))
ALL_BRANCHES = {"up", "down", "keep", "area", "bilinear", "bicubic", "gaussian", "poisson", "gray", "colour",
                "sinc_then_jpeg", "jpeg_then_sinc", "stage2_scalar", "stage2_range", "queue_fill", "queue_full"}


def sha(b: bytes) -> str:
    return hashlib.sha1(b).hexdigest()


def rng_digests():
    return [sha(pickle.dumps(random.getstate())), sha(pickle.dumps(np.random.get_state())),
            sha(torch.get_rng_state().numpy().tobytes())]


def seed_all(s):
    random.seed(s)
    np.random.seed(s)
    torch.manual_seed(s)


def write_dataset(root: Path):
    """Two 64x64 RGB PNGs and a parquet list naming them (the rows the dataset reads)."""
    import pyarrow as pa
    import pyarrow.parquet as pq
    from PIL import Image
    rs = np.random.RandomState(7)
    paths = []
    for i in range(2):
        p = root / f"img{i}.png"
        Image.fromarray(rs.randint(0, 256, (64, 64, 3), dtype=np.uint8)).save(p)
        paths.append(str(p))
    pq.write_table(pa.table({"image_path": paths, "llava_short": ["a cat", "a dog"],
                             "llava_long": ["a long cat", "a long dog"]}), root / "files.parquet")
    return [dict(file_list=str(root / "files.parquet"), image_path_key="image_path",
                 short_prompt_key="llava_short", long_prompt_key="llava_long")]


def transform_inputs(seed, mixed, lowpass):
    """hq and the three kernels of one batch, from a private generator (no global state touched)."""
    rs = np.random.RandomState(1000 + seed)
    hq = torch.from_numpy(rs.rand(BATCH, 3, SIZE, SIZE).astype(np.float32))
    k1, k2, sinc = [], [], []
    state = random.getstate(), np.random.get_state()
    random.seed(2000 + seed)
    np.random.seed(2000 + seed)
    for _ in range(BATCH):
        k1.append(np.pad(mixed(KERNEL_TYPES, [1 / 6] * 6, 11, [0.2, 3], [0.2, 3], [-math.pi, math.pi], [0.5, 4],
                               [1, 2], None), 5))
        k2.append(np.pad(mixed(KERNEL_TYPES, [1 / 6] * 6, 21, [0.2, 1.5], [0.2, 1.5], [-math.pi, math.pi], [0.5, 4],
                               [1, 2], None), 0))
        sinc.append(lowpass(np.random.uniform(np.pi / 3, np.pi), 9, pad_to=21))
    random.setstate(state[0])
    np.random.set_state(state[1])
    f = lambda a: torch.from_numpy(np.stack(a)).float()  # noqa: E731
    return dict(hq=hq, kernel1=f(k1), kernel2=f(k2), sinc_kernel=f(sinc), txt=[f"t{seed}_{i}" for i in range(BATCH)])


def run_calls(make, cfg_seed, mixed, lowpass, transform_cls, record=None):
    t = make()
    seed_all(cfg_seed)
    out = []
    for call in range(CALLS):
        hq, lq, txt = t(transform_inputs(cfg_seed * 10 + call, mixed, lowpass))
        out.append(dict(hq=sha(hq.numpy().tobytes()), lq=torch.round(lq * 255).to(torch.uint8).numpy(),
                        txt=list(txt), rng=rng_digests()))
    return t, out


def choose_seeds():
    """Greedy: seeds (per configuration) until the oracle's branch recorder has seen every branch."""
    from oracle.degradation import BatchTransform
    from diffbir_b200.dataset.degradation import circular_lowpass_kernel, random_mixed_kernels
    seen, chosen = set(), []
    for seed in range(200):
        for name, cfg in CONFIGS.items():
            t, _ = run_calls(lambda: BatchTransform(**cfg), seed, random_mixed_kernels, circular_lowpass_kernel,
                             None)
            new = set(t.branches) - seen
            if new:
                seen |= new
                chosen.append((name, seed))
        if seen >= ALL_BRANCHES:
            return chosen, sorted(seen)
    raise SystemExit(f"no covering seeds: missing {ALL_BRANCHES - seen}")


def main():
    import tempfile
    sys.path.insert(0, str(ROOT))
    chosen, branches = choose_seeds()
    use_reference()
    from diffbir.dataset import degradation as rdeg
    from diffbir.dataset.batch_transform import RealESRGANBatchTransform
    from diffbir.dataset.realesrgan import RealESRGANDataset
    fx = {"branches": np.array(branches), "chosen": np.array([f"{n}:{s}" for n, s in chosen])}
    for seed in range(4):
        for kt in KERNEL_TYPES:
            for size in (21, 7):
                seed_all(seed)
                fx[f"k_{kt}_{size}_{seed}"] = rdeg.random_mixed_kernels([kt], [1.0], size, [0.2, 3], [0.2, 3],
                                                                        [-math.pi, math.pi], [0.5, 4], [1, 2], None)
        seed_all(seed)
        fx[f"k_sinc_{seed}"] = rdeg.circular_lowpass_kernel(np.random.uniform(np.pi / 5, np.pi), 13, pad_to=21)
    with tempfile.TemporaryDirectory() as d:
        ds = RealESRGANDataset(file_metas=write_dataset(Path(d)), **DATASET)
        for i in ITEM_SEEDS:
            seed_all(i)
            item = ds[i % 2]
            fx[f"item_{i}_hq"] = np.array(sha(item["hq"].numpy().tobytes()))
            for k in ("kernel1", "kernel2", "sinc_kernel"):
                fx[f"item_{i}_{k}"] = item[k].numpy()
            fx[f"item_{i}_txt"] = np.array(item["txt"])
            fx[f"item_{i}_rng"] = np.array(rng_digests())
    for name, seed in chosen:
        _, calls = run_calls(lambda: RealESRGANBatchTransform(**CONFIGS[name]), seed, rdeg.random_mixed_kernels,
                             rdeg.circular_lowpass_kernel, None)
        for j, c in enumerate(calls):
            p = f"tf_{name}_{seed}_{j}"
            fx[p + "_hq"], fx[p + "_lq"] = np.array(c["hq"]), c["lq"]
            fx[p + "_txt"], fx[p + "_rng"] = np.array(c["txt"]), np.array(c["rng"])
    np.savez_compressed(OUT / "degradation_small.npz", **fx)
    print("wrote degradation_small.npz:", chosen, branches)


if __name__ == "__main__":
    main()
