"""-m gpu, >= 2 GPUs: the tiled VAE sharded over NCCL ranks is bit-identical to the single-rank tiled VAE on every rank,
and a tiled SwinIRPipeline.run gives the same uint8 image with the tiled VAE sharded or replicated
(tools/run_tiled_vae_multi.py under torchrun). On one GPU, tests/test_gpu_tiled_vae_shards.py emulates the ranks."""
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def test_sharded_tiled_vae_bit_identical():
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    n = 2 if n < 4 else 4
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
                        "--master-addr", "127.0.0.1", "--master-port", "29533",
                        str(ROOT / "tools" / "run_tiled_vae_multi.py")],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-4000:], r.stderr[-3000:])
    assert r.returncode == 0
