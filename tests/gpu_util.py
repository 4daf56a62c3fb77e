"""Helpers shared by the -m gpu parity tests."""
import threading

import torch


def no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def rel_err(x, ref):
    """max |x - ref| / max |ref|"""
    x, ref = x.float(), ref.float()
    return ((x - ref).abs().max() / (ref.abs().max() + 1e-20)).item()


def rel_rms(x, ref):
    x, ref = x.double(), ref.double()
    return ((x - ref).pow(2).mean().sqrt() / (ref.pow(2).mean().sqrt() + 1e-30)).item()


def psnr(x, ref, peak=None):
    x, ref = x.double(), ref.double()
    mse = (x - ref).pow(2).mean().item()
    peak = ref.abs().max().item() if peak is None else peak
    return float("inf") if mse == 0 else 10 * torch.log10(torch.tensor(peak * peak / mse)).item()


def to_dev(sd, dev="cuda"):
    return {k: v.to(dev) for k, v in sd.items()}


class Hub:
    """all_gather among threads that emulate ranks on one device: each rank leaves its tensor and waits for the
    others; the gathered copy is taken on the device's default stream, which every thread launches on, so it follows
    every rank's writes. A failing rank aborts the barrier and the timeout bounds a wait, so a fault cannot hang the
    test. `shapes[r]` lists the shapes rank r sent, in order."""

    def __init__(self, world: int, timeout: float = 300.0):
        self.bar = threading.Barrier(world, timeout=timeout)
        self.sent = [None] * world
        self.shapes = [[] for _ in range(world)]

    def comm(self, rank: int):
        hub = self

        class _Comm:
            def all_gather(self, t):
                hub.shapes[rank].append(tuple(t.shape))
                hub.sent[rank] = t
                hub.bar.wait()
                out = torch.stack(hub.sent, 0)
                hub.bar.wait()                   # nobody replaces its tensor before every rank has copied
                return out
        return _Comm()


def run_ranks(world: int, fn):
    """fn(rank, comm) on `world` threads, one per emulated rank, each with its communicator of one Hub -> (every
    rank's result, the hub). Fails if a rank raised or did not finish."""
    hub = Hub(world)
    outs, errs = [None] * world, []

    def run(r):
        try:
            outs[r] = fn(r, hub.comm(r))
        except BaseException as e:              # noqa: BLE001 -- reported below
            errs.append((r, e))
            hub.bar.abort()

    threads = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    torch.cuda.synchronize()
    assert not errs, errs
    assert not any(t.is_alive() for t in threads)
    return outs, hub
