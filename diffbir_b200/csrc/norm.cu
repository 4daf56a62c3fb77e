// GroupNorm (32 groups) statistics + apply and LayerNorm, fp32 math, NHWC activations.
//
// GroupNorm replaces GroupNorm32 / Normalize (reference util.py:191-193 eps 1e-5,
// attention.py:48-51 and vae.py:18-21 eps 1e-6). The input may be a *virtual concat* of two
// NHWC tensors along C (UNet output blocks normalise cat([h, skip+control]),
// controlnet.py:39-44); groups that straddle the boundary are handled because statistics
// are first taken per channel. The apply pass writes the 16-bit tensor-core operand that the
// implicit-GEMM convolution reads through TMA (optionally 2x nearest-upsampled:
// unet.py:76-78, vae.py:37-40), fused with SiLU.
//
// LayerNorm replaces nn.LayerNorm in BasicTransformerBlock (attention.py:257-259) and
// SwinIR (swinir.py:208,214,722,783), eps 1e-5, writing the 16-bit operand of the next GEMM.
#include "common.cuh"
#include "../../include/diffbir_b200.h"

namespace {

constexpr int GN_THREADS = 256;
constexpr int GN_WARPS = GN_THREADS / 32;

__device__ __forceinline__ const float* cat_ptr(const float* s1, const float* s2, int c1, int c2,
                                                long long pix, int c) {
  // element (pix, c) of the virtual concat [pix, c1 + c2]
  return c < c1 ? s1 + pix * c1 + c : s2 + pix * c2 + (c - c1);
}

// Stage 1: per-group sum / sum of squares over a chunk of pixels.
// grid = (chunks, N). A warp sweeps 128-channel slabs (one float4 per lane, coalesced) over the
// chunk's pixels keeping per-lane register sums, folds them into 32 per-group shared-memory
// accumulators, and the CTA writes 64 floats: partial[N][chunks][32][2].
// The last CTA of each image (atomic ticket, self-resetting) combines the chunk partials in fp64
// in a fixed order -> deterministic mean / rstd.
__global__ void __launch_bounds__(GN_THREADS)
gn_stats_kernel(const float* __restrict__ s1, const float* __restrict__ s2, int c1, int c2,
                int hw, int pix_per_chunk, float* __restrict__ partial,
                unsigned int* __restrict__ tickets, float* __restrict__ stats, float eps) {
  pdl_trigger();
  pdl_wait();
  const int C = c1 + c2;
  const int cpg = C / 32;
  const int n = blockIdx.y;
  const int chunk = blockIdx.x;
  const int chunks = gridDim.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int p_begin = chunk * pix_per_chunk;
  const int p_end = min(hw, p_begin + pix_per_chunk);
  __shared__ float s_grp[GN_WARPS][32][2];
  __shared__ float s_ch[GN_WARPS][128][2];
  __shared__ bool s_last;
  for (int i = threadIdx.x; i < GN_WARPS * 64; i += GN_THREADS) (&s_grp[0][0][0])[i] = 0.f;
  __syncthreads();

  for (int cb = 0; cb < C; cb += 128) {
    const int c = cb + lane * 4;
    float sum[4] = {0.f, 0.f, 0.f, 0.f}, sq[4] = {0.f, 0.f, 0.f, 0.f};
    if (c < C) {
      // 4 pixels per step, all four loads in flight before the first add (the chunk is sized so a
      // warp usually owns exactly 4 pixels: one memory latency per slab instead of four)
      int p = p_begin + warp;
      for (; p + 3 * GN_WARPS < p_end; p += 4 * GN_WARPS) {
        float4 v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
          v[u] = *reinterpret_cast<const float4*>(cat_ptr(s1, s2, c1, c2, static_cast<long long>(n) * hw + p + u * GN_WARPS, c));
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          sum[0] += v[u].x; sum[1] += v[u].y; sum[2] += v[u].z; sum[3] += v[u].w;
          sq[0] += v[u].x * v[u].x; sq[1] += v[u].y * v[u].y; sq[2] += v[u].z * v[u].z; sq[3] += v[u].w * v[u].w;
        }
      }
      for (; p < p_end; p += GN_WARPS) {
        // c1, c2 are multiples of 4, so a float4 never straddles the concat boundary
        const float4 v = *reinterpret_cast<const float4*>(cat_ptr(s1, s2, c1, c2, static_cast<long long>(n) * hw + p, c));
        sum[0] += v.x; sum[1] += v.y; sum[2] += v.z; sum[3] += v.w;
        sq[0] += v.x * v.x; sq[1] += v.y * v.y; sq[2] += v.z * v.z; sq[3] += v.w * v.w;
      }
    }
    // fold the slab's channels into groups without atomics (fixed order => deterministic):
    // lane l owns group (cb / cpg + l) for this slab
#pragma unroll
    for (int j = 0; j < 4; ++j) { s_ch[warp][lane * 4 + j][0] = sum[j]; s_ch[warp][lane * 4 + j][1] = sq[j]; }
    __syncwarp();
    const int g = cb / cpg + lane;
    const int c_lo = max(g * cpg, cb), c_hi = min(min((g + 1) * cpg, cb + 128), C);
    if (g < 32 && c_lo < c_hi) {
      float a = 0.f, b = 0.f;
      for (int cc = c_lo; cc < c_hi; ++cc) { a += s_ch[warp][cc - cb][0]; b += s_ch[warp][cc - cb][1]; }
      s_grp[warp][g][0] += a;
      s_grp[warp][g][1] += b;
    }
    __syncwarp();
  }
  __syncthreads();
  float* my_partial = partial + (static_cast<long long>(n) * chunks + chunk) * 64;
  if (threadIdx.x < 64) {
    float a = 0.f;
#pragma unroll
    for (int w = 0; w < GN_WARPS; ++w) a += (&s_grp[w][0][0])[threadIdx.x];
    my_partial[threadIdx.x] = a;
  }

  // ---- last-CTA-of-the-image finalisation (fixed summation order) ----
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int t = atomicAdd(&tickets[n], 1u);
    s_last = (t == static_cast<unsigned int>(chunks) - 1);
    if (s_last) tickets[n] = 0;   // self-reset for the next launch
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const float* img_partial = partial + static_cast<long long>(n) * chunks * 64;
  for (int g = warp; g < 32; g += GN_WARPS) {
    double a = 0.0, b = 0.0;
    for (int ch = lane; ch < chunks; ch += 32) {
      a += static_cast<double>(__ldcg(img_partial + ch * 64 + g * 2));
      b += static_cast<double>(__ldcg(img_partial + ch * 64 + g * 2 + 1));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      b += __shfl_xor_sync(0xffffffffu, b, o);
    }
    if (lane == 0) {
      const double cnt = static_cast<double>(hw) * cpg;
      const double mean = a / cnt;
      double var = b / cnt - mean * mean;
      if (var < 0.0) var = 0.0;
      stats[(n * 32 + g) * 2 + 0] = static_cast<float>(mean);
      stats[(n * 32 + g) * 2 + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
    }
  }
}

// Finalisation of statistics whose partial sums were emitted by the producing GEMM epilogues
// (dbir_gemm gn_partials): grid (32 groups, N), fixed-order fp64 combine.
constexpr int FIN_THREADS = 256;
// This thread's share of the (slot, channel) partial pairs of one source, four loads in flight per
// round: the kernel is a dependent link of every GroupNorm chain and was bound by the L2 latency of
// its one-load-at-a-time loop, not by bytes (fixed order per thread => deterministic).
template <int SPLIT>
__device__ __forceinline__ void fin_accumulate(const float* __restrict__ base, int c, int lo, int w, int total, int part,
                                               double& a, double& b) {
  for (int i0 = part * FIN_THREADS + threadIdx.x; i0 < total; i0 += 4 * SPLIT * FIN_THREADS) {
    float2 v[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = i0 + u * SPLIT * FIN_THREADS;
      v[u] = make_float2(0.f, 0.f);
      if (i < total) {
        const int sl = i / w, cc = lo + i % w;
        v[u] = __ldcg(reinterpret_cast<const float2*>(base + (static_cast<long long>(sl) * c + cc) * 2));
      }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) { a += v[u].x; b += v[u].y; }
  }
}

// SPLIT > 1: a (SPLIT,1,1) cluster shares one (group, image); every CTA reduces an interleaved share of the
// partial pairs, the shares meet in CTA 0 through distributed shared memory in rank order (deterministic).
// A VAE layer at 512^2 has 8192 row slots x 4 channels per group: one CTA per group would read its
// 8.4 MB with only 32 CTAs in the grid, and 16x that at 2048^2.
template <int SPLIT>
__global__ void __launch_bounds__(FIN_THREADS)
gn_finalize_kernel(const float* __restrict__ p1, int slots1, int c1, const float* __restrict__ p2,
                   int slots2, int c2, int hw, float eps, float* __restrict__ stats) {
  pdl_trigger();
  pdl_wait();
  const int g = blockIdx.x / SPLIT, part = blockIdx.x % SPLIT, n = blockIdx.y;
  const int C = c1 + c2, cpg = C / 32;
  const int ch0 = g * cpg, ch1 = ch0 + cpg;
  double a = 0.0, b = 0.0;
  // source 1: channels [ch0, ch1) ∩ [0, c1)
  {
    const int lo = min(ch0, c1), hi = min(ch1, c1), w = hi - lo;
    const int total = w * slots1;
    const float* base = p1 + static_cast<long long>(n) * slots1 * c1 * 2;
    fin_accumulate<SPLIT>(base, c1, lo, w, total, part, a, b);
  }
  if (c2 > 0) {
    const int lo = max(ch0, c1) - c1, hi = max(ch1, c1) - c1, w = hi - lo;
    const int total = w * slots2;
    const float* base = p2 + static_cast<long long>(n) * slots2 * c2 * 2;
    fin_accumulate<SPLIT>(base, c2, lo, w, total, part, a, b);
  }
  // fixed-order tree: xor-shuffles inside each warp, then thread 0 adds the 8 warp sums in warp order
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  __shared__ double sa[FIN_THREADS / 32], sb[FIN_THREADS / 32];
  __shared__ double s_part[2];
  if ((threadIdx.x & 31) == 0) { sa[threadIdx.x >> 5] = a; sb[threadIdx.x >> 5] = b; }
  __syncthreads();
  double ta = 0.0, tb = 0.0;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int i = 0; i < FIN_THREADS / 32; ++i) { ta += sa[i]; tb += sb[i]; }
    s_part[0] = ta; s_part[1] = tb;
  }
  if constexpr (SPLIT > 1) {
    cluster_sync_all();                       // every CTA's s_part is written and visible cluster-wide
    if (part == 0 && threadIdx.x == 0) {
      ta = 0.0; tb = 0.0;
      for (int r = 0; r < SPLIT; ++r) {
        const uint32_t peer = mapa_u32(smem_u32(s_part), static_cast<uint32_t>(r));
        double pa, pb;
        asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(pa) : "r"(peer) : "memory");
        asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(pb) : "r"(peer + 8) : "memory");
        ta += pa; tb += pb;
      }
    }
    cluster_sync_all();                       // peers stay resident until CTA 0 has read their shares
  }
  if (part == 0 && threadIdx.x == 0) {
    const double cnt = static_cast<double>(hw) * cpg;
    const double mean = ta / cnt;
    double var = tb / cnt - mean * mean;
    if (var < 0.0) var = 0.0;
    stats[(n * 32 + g) * 2 + 0] = static_cast<float>(mean);
    stats[(n * 32 + g) * 2 + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  }
}

// Stage 2: y = silu?(x * a[c] + b[c]) -> op16, optional 2x nearest upsample, optional raw copy.
// grid = (pixel chunks, N)
__global__ void __launch_bounds__(256)
gn_apply_kernel(const float* __restrict__ s1, const float* __restrict__ s2, int c1, int c2,
                int h, int w, const float* __restrict__ stats, const float* __restrict__ gamma,
                const float* __restrict__ beta, int do_norm, int do_silu, int up,
                op_t* __restrict__ out, op_t* __restrict__ out_raw, int pix_per_cta, int imgs_per_group) {
  extern __shared__ float s_ab[];   // [C][2]
  pdl_trigger();
  pdl_wait();
  const int C = c1 + c2;
  const int n = blockIdx.y;
  const int hw = h * w;
  if (do_norm) {
    const int cpg = C / 32;
    const int goff = imgs_per_group > 0 ? (n / imgs_per_group) * C : 0;     // stacked twin problems
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      const int g = c / cpg;
      const float mean = stats[(n * 32 + g) * 2], rstd = stats[(n * 32 + g) * 2 + 1];
      const float a = gamma[goff + c] * rstd;
      s_ab[2 * c] = a;
      s_ab[2 * c + 1] = beta[goff + c] - mean * a;
    }
    __syncthreads();
  }
  const int V = C / 4;
  const int p_begin = blockIdx.x * pix_per_cta;
  const int p_end = min(hw, p_begin + pix_per_cta);
  const long long total = static_cast<long long>(p_end - p_begin) * V;
  // four 16-byte loads in flight per thread before the first use: at 512^2 x 128 channels (VAE) the pass
  // streams 134 MB from HBM and the one-load-per-iteration loop reached 2.7 TB/s (ncu, 41 % of the copy peak)
  constexpr int U = 4;
  for (long long i0 = threadIdx.x; i0 < total; i0 += static_cast<long long>(U) * blockDim.x) {
    float4 v[U];
    int pp[U], cc[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const long long i = i0 + static_cast<long long>(u) * blockDim.x;
      pp[u] = -1;
      if (i < total) {
        pp[u] = p_begin + static_cast<int>(i / V);
        cc[u] = static_cast<int>(i % V) * 4;
        v[u] = *reinterpret_cast<const float4*>(cat_ptr(s1, s2, c1, c2, static_cast<long long>(n) * hw + pp[u], cc[u]));
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (pp[u] < 0) continue;
      const int p = pp[u], c = cc[u];
      const long long pix = static_cast<long long>(n) * hw + p;
      float y[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
      uint2 raw;
      raw.x = pack2(v[u].x, v[u].y); raw.y = pack2(v[u].z, v[u].w);
      if (do_norm) {
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = y[j] * s_ab[2 * (c + j)] + s_ab[2 * (c + j) + 1];
      }
      if (do_silu) {
#pragma unroll
        for (int j = 0; j < 4; ++j) y[j] = silu_f(y[j]);
      }
      uint2 o;
      o.x = pack2(y[0], y[1]); o.y = pack2(y[2], y[3]);
      if (up == 1) {
        *reinterpret_cast<uint2*>(out + pix * C + c) = o;
        if (out_raw) *reinterpret_cast<uint2*>(out_raw + pix * C + c) = raw;
      } else {
        const int py = p / w, px = p % w;
        const int W2 = w * 2;
        const long long base = (static_cast<long long>(n) * (h * 2) + py * 2) * W2 + px * 2;
        *reinterpret_cast<uint2*>(out + (base) * C + c) = o;
        *reinterpret_cast<uint2*>(out + (base + 1) * C + c) = o;
        *reinterpret_cast<uint2*>(out + (base + W2) * C + c) = o;
        *reinterpret_cast<uint2*>(out + (base + W2 + 1) * C + c) = o;
      }
    }
  }
}

// LayerNorm over the last dim; one warp per row; C <= 1280, C % 4 == 0.
// Output op16 with row stride ldo >= C; columns [C, ldo) are zero-filled (K padding).
template <bool F32OUT>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, long long ldx, int rows, int C,
                 const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                 void* __restrict__ out_v, long long ldo, int rows_per_group) {
  pdl_trigger();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long row = static_cast<long long>(blockIdx.x) * (blockDim.x >> 5) + warp;
  if (row >= rows) return;
  if (rows_per_group > 0) {                      // stacked twin problems: this row's gamma / beta set
    const long long goff = (row / rows_per_group) * C;
    gamma += goff; beta += goff;
  }
  const float* xr = x + row * ldx;
  constexpr int MAXV = 10;
  float4 v[MAXV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = (lane + 32 * i) * 4;
    if (c < C) {
      v[i] = *reinterpret_cast<const float4*>(xr + c);
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    } else {
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  s = warp_sum(s);
  const float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = (lane + 32 * i) * 4;
    if (c < C) {
      const float a = v[i].x - mean, b = v[i].y - mean, d = v[i].z - mean, e = v[i].w - mean;
      q += (a * a + b * b) + (d * d + e * e);
    }
  }
  q = warp_sum(q);
  const float rstd = rsqrtf(q / C + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    const int c = (lane + 32 * i) * 4;
    if (c < C) {
      const float4 g = *reinterpret_cast<const float4*>(gamma + c);
      const float4 b = *reinterpret_cast<const float4*>(beta + c);
      const float y0 = (v[i].x - mean) * rstd * g.x + b.x, y1 = (v[i].y - mean) * rstd * g.y + b.y;
      const float y2 = (v[i].z - mean) * rstd * g.z + b.z, y3 = (v[i].w - mean) * rstd * g.w + b.w;
      if (F32OUT) {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(out_v) + row * ldo + c) = make_float4(y0, y1, y2, y3);
      } else {
        uint2 o;
        o.x = pack2(y0, y1); o.y = pack2(y2, y3);
        *reinterpret_cast<uint2*>(reinterpret_cast<op_t*>(out_v) + row * ldo + c) = o;
      }
    } else if (c < ldo) {
      if (F32OUT) *reinterpret_cast<float4*>(reinterpret_cast<float*>(out_v) + row * ldo + c) = make_float4(0.f, 0.f, 0.f, 0.f);
      else *reinterpret_cast<uint2*>(reinterpret_cast<op_t*>(out_v) + row * ldo + c) = make_uint2(0u, 0u);
    }
  }
}

}  // namespace

extern "C" int64_t dbir_gn_workspace_floats(int32_t n, int32_t hw, int32_t c) {
  // tickets + partials [n][chunks <= 1024][32][2]
  (void)hw; (void)c;
  return 64 + ((static_cast<int64_t>(n) + 3) / 4) * 4 + static_cast<int64_t>(n) * 1024 * 64 + 64;
}

static int gn_chunks(int n, int hw, int* pix_per_chunk) {
  // The chunking is a function of the image size only (never of the batch): the fp32 partial sums
  // and hence the statistics of an image have the same bits whatever batch it is normalised in.
  // 32 pixels per chunk (4 per warp, loaded together) for images of >= 2048 pixels, 8 (one per warp)
  // below; at most 1024 chunks per image (the partial buffer).
  (void)n;
  int ppc = hw >= 2048 ? 32 : 8;
  int chunks = (hw + ppc - 1) / ppc;
  if (chunks > 1024) { ppc = (hw + 1023) / 1024; chunks = (hw + ppc - 1) / ppc; }
  *pix_per_chunk = ppc;
  return chunks;
}

extern "C" int dbir_gn_stats(const float* src1, const float* src2, int32_t c1, int32_t c2,
                             int32_t n, int32_t hw, float eps, float* stats, float* workspace,
                             void* stream) {
  const int C = c1 + c2;
  DBIR_REQUIRE(src1 && stats && workspace, "dbir_gn_stats: null pointer");
  DBIR_REQUIRE(c1 % 4 == 0 && c2 % 4 == 0 && C % 32 == 0, "dbir_gn_stats: bad channels %d+%d", c1, c2);
  DBIR_REQUIRE(c2 == 0 || src2, "dbir_gn_stats: src2 missing");
  int ppc;
  const int chunks = gn_chunks(n, hw, &ppc);
  unsigned int* tickets = reinterpret_cast<unsigned int*>(workspace);
  float* partial = workspace + 64 + ((n + 3) / 4) * 4;
  DBIR_CHECK_CUDA(dbir_launch(gn_stats_kernel, dim3(chunks, n), dim3(GN_THREADS), 0,
                              reinterpret_cast<cudaStream_t>(stream), src1, src2, c1, c2, hw, ppc, partial, tickets,
                              stats, eps));
  return 0;
}

extern "C" int dbir_gn_finalize(const float* partials1, int32_t slots1, int32_t c1, const float* partials2,
                                int32_t slots2, int32_t c2, int32_t n, int32_t hw, float eps, float* stats,
                                void* stream) {
  DBIR_REQUIRE(partials1 && stats && slots1 > 0 && (c1 + c2) % 32 == 0, "dbir_gn_finalize: bad args");
  DBIR_REQUIRE(c2 == 0 || (partials2 && slots2 > 0), "dbir_gn_finalize: second source missing");
  // pairs per (group, image): a function of the image size and width only, never of the batch
  const long long per_group = static_cast<long long>((c1 + c2) / 32) * (slots1 > slots2 ? slots1 : slots2);
  const int split = per_group <= 4096 ? 1 : per_group <= 8192 ? 2 : per_group <= 16384 ? 4 : 8;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
#define DBIR_FIN(S)                                                                                             \
  DBIR_CHECK_CUDA(dbir_launch_cluster(gn_finalize_kernel<S>, dim3(32 * S, n), dim3(FIN_THREADS), 0, st, S, partials1, \
                                      slots1, c1, partials2, slots2, c2, hw, eps, stats))
  switch (split) {
    case 1: DBIR_FIN(1); break;
    case 2: DBIR_FIN(2); break;
    case 4: DBIR_FIN(4); break;
    default: DBIR_FIN(8); break;
  }
#undef DBIR_FIN
  return 0;
}

extern "C" int dbir_gn_apply(const float* src1, const float* src2, int32_t c1, int32_t c2,
                             int32_t n, int32_t h, int32_t w, const float* stats,
                             const float* gamma, const float* beta, int32_t do_norm,
                             int32_t do_silu, int32_t upsample, void* out, void* out_raw,
                             int32_t imgs_per_group, void* stream) {
  const int C = c1 + c2;
  DBIR_REQUIRE(src1 && out, "dbir_gn_apply: null pointer");
  DBIR_REQUIRE(c1 % 4 == 0 && c2 % 4 == 0, "dbir_gn_apply: channels must be multiples of 4");
  DBIR_REQUIRE(!do_norm || (stats && gamma && beta && C % 32 == 0), "dbir_gn_apply: norm args");
  DBIR_REQUIRE(upsample == 1 || upsample == 2, "dbir_gn_apply: upsample must be 1 or 2");
  DBIR_REQUIRE(!(upsample == 2 && out_raw), "dbir_gn_apply: raw copy unsupported with upsample");
  const int hw = h * w;
  const int target = 4 * dbir_sm_count();
  int ctas = (target + n - 1) / n;
  int ppc = (hw + ctas - 1) / ctas;
  if (ppc < 1) ppc = 1;
  ctas = (hw + ppc - 1) / ppc;
  const size_t smem = do_norm ? static_cast<size_t>(C) * 2 * sizeof(float) : 0;
  DBIR_CHECK_CUDA(dbir_launch(gn_apply_kernel, dim3(ctas, n), dim3(256), smem, reinterpret_cast<cudaStream_t>(stream),
                              src1, src2, c1, c2, h, w, stats, gamma, beta, do_norm, do_silu, upsample,
                              reinterpret_cast<op_t*>(out), reinterpret_cast<op_t*>(out_raw), ppc, imgs_per_group));
  return 0;
}

extern "C" int dbir_layernorm(const float* x, int64_t ldx, int32_t rows, int32_t c,
                              const float* gamma, const float* beta, float eps, void* out,
                              int64_t ldo, int32_t out_kind, int32_t rows_per_group, void* stream) {
  DBIR_REQUIRE(x && gamma && beta && out, "dbir_layernorm: null pointer");
  DBIR_REQUIRE(c % 4 == 0 && c <= 1280 && ldo >= c && ldo % 4 == 0 && ldo <= 1280,
               "dbir_layernorm: unsupported width %d (ldo %lld)", c, (long long)ldo);
  const int rows_per_cta = 8;
  const int grid = (rows + rows_per_cta - 1) / rows_per_cta;
  const long long ldx_ = ldx, ldo_ = ldo;
  if (out_kind == 0)
    DBIR_CHECK_CUDA(dbir_launch(layernorm_kernel<true>, dim3(grid), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
                                x, ldx_, rows, c, gamma, beta, eps, out, ldo_, rows_per_group));
  else
    DBIR_CHECK_CUDA(dbir_launch(layernorm_kernel<false>, dim3(grid), dim3(256), 0, reinterpret_cast<cudaStream_t>(stream),
                                x, ldx_, rows, c, gamma, beta, eps, out, ldo_, rows_per_group));
  return 0;
}
