// Brownian tree generated on the device: the noise source of the `dpm++_sde` step rule (reference
// k_diffusion.py:70-120, 548-586), which queries W over [sigma_i, sigma_mid] and [sigma_i, sigma_next] of every step.
// The two intervals overlap, so both queries must read one Brownian path.
//
// W is a Brownian motion on [lo, hi] with W(lo) = 0, independent per element. A query W(t) walks the dyadic bisection
// of [lo, hi] for `depth` levels. At node k (heap numbering: 1 is the midpoint of [lo, hi], 2k / 2k + 1 its halves'
// midpoints) the midpoint value is a Brownian-bridge draw between the node's end values. W(hi) is the draw of node 0.
// Below the last level, W(t) is one more bridge draw between the leaf's ends, with t mixed into the key.
// Every draw is a normal from counter-based Philox4x32-10 (Salmon et al., SC'11) and Box-Muller:
//   counter = (element lo32, element hi32, node lo32, node hi32 | leaf << 31), key = seed (leaf: seed ^ bits(t)).
// No state is kept between calls, so the same query gives the same bits every time, an element's value does not depend
// on the tensor's size, and W(t1) - W(t0) is a difference of point values (additive up to rounding).
// The walk runs in fp64: the increments that matter are small differences of values of size sqrt(hi - lo).
#include "common.cuh"
#include "../../include/diffbir_b200.h"

namespace {

constexpr int THREADS = 128;
constexpr uint32_t LEAF = 0x80000000u;

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) {
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
  }
  return c;
}

// 52 bits of (w0, w1) -> u1 in (0, 1) (never 0: |z| <= 8.6), w2 -> u2 in [0, 1)
__device__ __forceinline__ double box_muller(uint4 w) {
  const unsigned long long k = (static_cast<unsigned long long>(w.x) << 20) | (w.y >> 12);
  const double u1 = (static_cast<double>(k) + 0.5) * 0x1p-52;
  const double u2 = static_cast<double>(w.z) * 0x1p-32;
  return sqrt(-2.0 * log(u1)) * cospi(2.0 * u2);
}

struct Key {
  uint32_t e0, e1;              // element index
  unsigned long long seed;
};

__device__ __forceinline__ uint4 words(const Key& k, unsigned long long node, bool leaf, double t) {
  const unsigned long long key = leaf ? k.seed ^ static_cast<unsigned long long>(__double_as_longlong(t)) : k.seed;
  const uint4 c = make_uint4(k.e0, k.e1, static_cast<uint32_t>(node),
                             static_cast<uint32_t>(node >> 32) | (leaf ? LEAF : 0u));
  return philox4x32_10(c, static_cast<uint32_t>(key), static_cast<uint32_t>(key >> 32));
}

// W(t) given W(a) = wa, W(b) = wb: mean on the chord, variance (t - a)(b - t) / (b - a); exact at the ends
__device__ __forceinline__ double bridge(double a, double b, double wa, double wb, double t, double z) {
  if (t <= a) return wa;
  if (t >= b) return wb;
  return wa + (t - a) / (b - a) * (wb - wa) + sqrt((t - a) * (b - t) / (b - a)) * z;
}

struct Walk {
  double a, b, wa, wb;
  unsigned long long node;
  __device__ __forceinline__ void split(double t, double z) {
    const double m = 0.5 * (a + b);
    const double wm = bridge(a, b, wa, wb, m, z);
    if (t < m) {
      b = m, wb = wm, node = 2 * node;
    } else {
      a = m, wa = wm, node = 2 * node + 1;
    }
  }
};

// W(t1) - W(t0) of element e of the tree seeded `seed`
__device__ __forceinline__ float increment(long long e, unsigned long long seed, double lo, double hi, double t0,
                                           double t1, int depth) {
  const Key k{static_cast<uint32_t>(e), static_cast<uint32_t>(e >> 32), seed};
  t0 = fmin(fmax(t0, lo), hi);
  t1 = fmin(fmax(t1, lo), hi);
  const double w_hi = sqrt(hi - lo) * box_muller(words(k, 0, false, 0.0));
  Walk p{lo, hi, 0.0, w_hi, 1}, q = p;
  // both walks share their nodes down to where t0 and t1 part: one draw per shared node
  for (int l = 0; l < depth; ++l) {
    const double zp = box_muller(words(k, p.node, false, 0.0));
    const double zq = q.node == p.node ? zp : box_muller(words(k, q.node, false, 0.0));
    p.split(t0, zp);
    q.split(t1, zq);
  }
  const double w0 = bridge(p.a, p.b, p.wa, p.wb, t0, box_muller(words(k, p.node, true, t0)));
  const double w1 = bridge(q.a, q.b, q.wa, q.wb, t1, box_muller(words(k, q.node, true, t1)));
  return static_cast<float>(w1 - w0);
}

__global__ void __launch_bounds__(THREADS)
brownian_increment_kernel(float* __restrict__ out, long long n, unsigned long long seed, double lo, double hi,
                          double t0, double t1, int depth) {
  const long long e = static_cast<long long>(blockIdx.x) * THREADS + threadIdx.x;
  if (e >= n) return;
  out[e] = increment(e, seed, lo, hi, t0, t1, depth);
}

// one tree per sample: element e of sample b is element e of the tree seeded seeds[b]
__global__ void __launch_bounds__(THREADS)
brownian_increment_samples_kernel(float* __restrict__ out, long long n, const unsigned long long* __restrict__ seeds,
                                  double lo, double hi, double t0, double t1, int depth) {
  const long long e = static_cast<long long>(blockIdx.x) * THREADS + threadIdx.x;
  const int b = blockIdx.y;
  if (e >= n) return;
  out[b * n + e] = increment(e, seeds[b], lo, hi, t0, t1, depth);
}

__global__ void __launch_bounds__(THREADS)
brownian_draws_kernel(uint32_t* __restrict__ w_out, double* __restrict__ z_out, long long n, unsigned long long seed,
                      unsigned long long node, int leaf, double t) {
  const long long e = static_cast<long long>(blockIdx.x) * THREADS + threadIdx.x;
  if (e >= n) return;
  const uint4 w = words(Key{static_cast<uint32_t>(e), static_cast<uint32_t>(e >> 32), seed}, node, leaf != 0, t);
  if (w_out) reinterpret_cast<uint4*>(w_out)[e] = w;
  if (z_out) z_out[e] = box_muller(w);
}

unsigned blocks(long long n) { return static_cast<unsigned>((n + THREADS - 1) / THREADS); }

}  // namespace

extern "C" int dbir_brownian_increment(float* out, int64_t n, uint64_t seed, double lo, double hi, double t0,
                                       double t1, int32_t depth, void* stream) {
  DBIR_REQUIRE(out && n > 0 && n <= (1LL << 31) * THREADS, "dbir_brownian_increment: bad output (n = %lld)",
               static_cast<long long>(n));
  DBIR_REQUIRE(lo <= hi && depth >= 0 && depth <= 62, "dbir_brownian_increment: bad tree [%g, %g], depth %d", lo, hi,
               depth);
  brownian_increment_kernel<<<blocks(n), THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      out, n, seed, lo, hi, t0, t1, depth);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_brownian_increment_samples(float* out, int64_t n, int32_t samples, const uint64_t* seeds, double lo,
                                               double hi, double t0, double t1, int32_t depth, void* stream) {
  DBIR_REQUIRE(out && seeds && n > 0 && n <= (1LL << 31) * THREADS && samples > 0 && samples <= 65535,
               "dbir_brownian_increment_samples: bad output (n = %lld, samples = %d)", static_cast<long long>(n), samples);
  DBIR_REQUIRE(lo <= hi && depth >= 0 && depth <= 62, "dbir_brownian_increment_samples: bad tree [%g, %g], depth %d", lo,
               hi, depth);
  brownian_increment_samples_kernel<<<dim3(blocks(n), samples), THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      out, n, reinterpret_cast<const unsigned long long*>(seeds), lo, hi, t0, t1, depth);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_brownian_draws(uint32_t* words_out, double* normals, int64_t n, uint64_t seed, uint64_t node,
                                   int32_t leaf, double t, void* stream) {
  DBIR_REQUIRE((words_out || normals) && n > 0 && n <= (1LL << 31) * THREADS, "dbir_brownian_draws: bad output");
  DBIR_REQUIRE(node < (1ULL << 63), "dbir_brownian_draws: node index needs more than 63 bits");
  brownian_draws_kernel<<<blocks(n), THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      words_out, normals, n, seed, node, leaf, t);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}
