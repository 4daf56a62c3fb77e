"""NumPy restatement of the device Brownian tree (csrc/brownian.cu), vectorised over elements.

Counter-based Philox4x32-10 on uint32, Box-Muller in float64, and the dyadic bisection walk of [lo, hi]: every
element walks the same nodes (they depend on t only), with its own draws keyed by (seed, node, element)."""
import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = 0x9E3779B9, 0xBB67AE85
LEAF = 0x80000000                                  # tag bit of a leaf draw (counter word 3)


def philox4x32_10(ctr, key):
    """ctr: 4 uint32 arrays (or scalars) broadcast together, key: 2 ints -> 4 uint32 arrays."""
    c = [np.asarray(v, dtype=np.uint64) for v in ctr]
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    mask = np.uint64(0xFFFFFFFF)
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & mask,
             (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1), p0 & mask]
    return [np.broadcast_to(v, np.broadcast(*c).shape).astype(np.uint32) for v in c]


def normal_from_words(w):
    """Box-Muller on one Philox block: 52 bits of (w0, w1) -> u1 in (0, 1), w2 -> u2 in [0, 1)."""
    k = (w[0].astype(np.uint64) << np.uint64(20)) | (w[1].astype(np.uint64) >> np.uint64(12))
    u1 = (k.astype(np.float64) + 0.5) * 2.0 ** -52
    u2 = w[2].astype(np.float64) * 2.0 ** -32
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(2.0 * np.pi * u2)


def draw_words(n, seed, node, leaf=False, t=0.0):
    """Philox words of elements 0 .. n-1 at a node (interior / root) or of the leaf draw at time t."""
    e = np.arange(n, dtype=np.uint64)
    key = int(seed)
    if leaf:
        key ^= int(np.float64(t).view(np.uint64))
    hi = (int(node) >> 32) | (LEAF if leaf else 0)
    return philox4x32_10([e & np.uint64(0xFFFFFFFF), e >> np.uint64(32), int(node) & 0xFFFFFFFF, hi],
                         (key & 0xFFFFFFFF, key >> 32))


def draw(n, seed, node, leaf=False, t=0.0):
    return normal_from_words(draw_words(n, seed, node, leaf, t))


def tree_depth(lo, hi, tol=1e-6):
    """Fewest bisections of [lo, hi] that leave leaves no wider than tol."""
    d = 0
    while (hi - lo) / 2.0 ** d > tol:
        d += 1
    return d


def _bridge(a, b, wa, wb, t, z):
    if t <= a:
        return wa
    if t >= b:
        return wb
    return wa + (t - a) / (b - a) * (wb - wa) + np.sqrt((t - a) * (b - t) / (b - a)) * z


def point(n, seed, lo, hi, t, depth):
    """W(t) of elements 0 .. n-1 (float64): W(lo) = 0, W(hi) = sqrt(hi - lo) * (draw of node 0)."""
    t = min(max(float(t), lo), hi)
    a, b, wa, wb, node = lo, hi, np.zeros(n), np.sqrt(hi - lo) * draw(n, seed, 0), 1
    for _ in range(depth):
        m = 0.5 * (a + b)
        wm = _bridge(a, b, wa, wb, m, draw(n, seed, node))
        if t < m:
            b, wb, node = m, wm, 2 * node
        else:
            a, wa, node = m, wm, 2 * node + 1
    return _bridge(a, b, wa, wb, t, draw(n, seed, node, leaf=True, t=t))


def increment(n, seed, lo, hi, t0, t1, depth):
    """W(t1) - W(t0) rounded to float32, as dbir_brownian_increment writes it."""
    return (point(n, seed, lo, hi, t1, depth) - point(n, seed, lo, hi, t0, depth)).astype(np.float32)


class RestatedTree:
    """Drop-in for diffbir_b200.sampler.edm.DeviceBrownianTree with this restatement behind it (CPU tensors)."""

    def __init__(self, x, lo, hi, seed):
        import torch
        self.n, self.shape, self.device = x.numel(), x.shape, x.device
        self.lo, self.hi, self.seed = float(lo), float(hi), int(seed)
        self.depth = tree_depth(self.lo, self.hi)
        self.torch = torch

    def __call__(self, t0, t1):
        w = increment(self.n, self.seed, self.lo, self.hi, float(t0), float(t1), self.depth)
        return self.torch.from_numpy(w).view(self.shape).to(self.device)
