"""The dataset's batch ops run on the engine only (there is no CPU path)."""
import torch


def require_cuda(t: torch.Tensor, what: str) -> None:
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError(f"{what} runs on the CUDA engine (sm_90a) only: move the batch to a CUDA device first "
                           f"(got {'a CPU tensor' if isinstance(t, torch.Tensor) else type(t).__name__})")
