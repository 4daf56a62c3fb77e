"""inference.py under torchrun: one process per GPU of the box, in one of two modes (`--distribute`).

images     the sorted input images are dealt round-robin (rank r restores images r, r + W, r + 2W, ... of W ranks).
           Each rank runs the whole restoration of its images (captioner, cleaner, sampler, VAE) and writes their
           PNGs; the prompt.csv rows are gathered to rank 0, which writes them in input order. Image k is restored
           right after set_seed(seed + k), so every output is independent of the world size. That differs from the
           plain single-process run for k >= 1, which seeds once and draws through the folder. The ranks meet once,
           at the end, over a gloo group whose timeout (WAIT) covers a rank that finishes hours before the slowest.
cooperate  every rank works on every image, seeded once as in the single-process run, and the outputs are that
           run's with DBIR_DETERMINISTIC=1 (see below): rank 0 runs the captioner and broadcasts the prompt; stage 1 is sharded by windows when tiled and
           runs on rank 0 (broadcast) otherwise; tiled sampling and the tiled VAE are sharded by tiles, an un-tiled
           sampler by (image, CFG branch) forwards (ranks beyond 2 x batch_size idle). The un-tiled VAE stays
           replicated. Rank 0 writes every file.

Under torchrun the ControlNet+UNet engine uses its batch-invariant plans (DBIR_DETERMINISTIC=1), so no result
depends on which process computed it; the other engines pass no split-K workspace, so the timing-based tuner's
choices (tile width, CTA pairs) never change their bits."""
from __future__ import annotations

import os
from datetime import timedelta
from typing import Callable, List, Optional, Tuple

MODES = ("images", "cooperate")
# How long a rank waits at a host-side meeting point (images mode's prompt.csv gather) for the slowest rank. The NCCL
# group keeps torch's default timeout: its collectives are per-step exchanges of ranks that work in lock step.
WAIT = timedelta(days=7)


def torchrun_env(environ=os.environ) -> Optional[Tuple[int, int, int]]:
    """(rank, local rank, world size) when launched by torchrun, else None."""
    if not all(k in environ for k in ("WORLD_SIZE", "RANK", "LOCAL_RANK")):
        return None
    return int(environ["RANK"]), int(environ["LOCAL_RANK"]), int(environ["WORLD_SIZE"])


class Ranks:
    """What one rank of a torchrun'd inference.py does; the loops consult it where the single-process run acts
    alone (which images, seeding, captions, file writes)."""

    def __init__(self, mode: str, rank: int, world: int, seed: int, set_seed: Callable[[int], None],
                 host_group=None) -> None:
        if mode not in MODES:
            raise ValueError(f"--distribute {mode}: not one of {MODES}")
        self.mode, self.rank, self.world, self.seed, self.set_seed = mode, rank, world, seed, set_seed
        self.host_group = host_group                        # gloo group for waits of any length (None: the default group)
        self.rows: List[Tuple[int, List[str]]] = []         # images mode: (image index, prompt.csv row)

    @property
    def writes(self) -> bool:
        """Whether this rank saves the images it restores."""
        return self.mode == "images" or self.rank == 0

    @property
    def captions(self) -> bool:
        """Whether this rank runs (and so loads) the captioner."""
        return self.mode == "images" or self.rank == 0

    def takes(self, k: int) -> bool:
        """Whether this rank restores input image k (its index among the sorted image files)."""
        return self.mode == "cooperate" or k % self.world == self.rank

    def start_image(self, k: int) -> None:
        if self.mode == "images":
            self.set_seed(self.seed + k)

    def caption(self, captioner, lq) -> str:
        if self.mode == "images":
            return captioner(lq)
        import torch.distributed as dist
        box = [captioner(lq) if self.rank == 0 else None]
        dist.broadcast_object_list(box, src=0)
        return box[0]

    def prompt_row(self, save_dir: str, k: int, file_stem: str, pos_prompt: str, neg_prompt: str) -> None:
        from .loop import append_prompt_row
        if self.mode == "images":
            self.rows.append((k, [file_stem, pos_prompt, neg_prompt]))
        else:
            append_prompt_row(save_dir, file_stem, pos_prompt, neg_prompt)

    def finish(self, save_dir: str) -> None:
        """images mode: rank 0 appends every rank's prompt.csv rows in input order (a stable sort keeps the order
        of an image's own rows: its faces, then the photo)."""
        if self.mode != "images":
            return
        import torch.distributed as dist
        from .loop import append_prompt_row
        parts = [None] * self.world
        dist.all_gather_object(parts, self.rows, group=self.host_group)
        if self.rank == 0:
            for _, row in sorted((r for p in parts for r in p), key=lambda r: r[0]):
                append_prompt_row(save_dir, *row)
        self.rows = []

    def configure(self, pipelines) -> None:
        """Sets how the pipelines' stages use the other ranks."""
        for p in pipelines:
            if self.mode == "images":            # each rank's images are its own: no collective anywhere
                p.shard_tiles = p.shard_batch = p.shard_vae = p.shard_cleaner = False
            else:
                p.shard_tiles = p.shard_batch = p.shard_vae = p.shard_cleaner = True
                p.cldm.shard_vae_rows = False


def launch(args, set_seed: Callable[[int], None]) -> Optional[Ranks]:
    """Under torchrun: binds this process to its GPU, pins process-independent kernel plans and opens the NCCL
    group. Without torchrun's variables nothing is done (and torch.distributed is not touched)."""
    env = torchrun_env()
    if env is None:
        return None
    if args.distribute == "cooperate" and args.task == "unaligned_face" and args.version != "custom":
        raise NotImplementedError("--task unaligned_face restores each face on its own: use --distribute images")
    rank, local, world = env
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(local)
    os.environ["DBIR_DETERMINISTIC"] = "1"
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    host_group = dist.new_group(backend="gloo", timeout=WAIT)
    return Ranks(args.distribute, rank, world, args.seed, set_seed, host_group)


def close() -> None:
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized():
        dist.destroy_process_group()
