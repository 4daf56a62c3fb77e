// The LLaVA captioner's language model (LLaMA-7B / Vicuna-7B v1.5, reference llava/model/language_model/llava_llama.py
// on transformers' LlamaModel): RMSNorm, RoPE with the KV-cache write, causal prefill attention and decode-step
// attention at head_dim 128, the M = 1 matrix-vector product of a decode step with its epilogues, greedy argmax and
// the token-embedding gather. Positions and lengths that change per generated token are read from device int32
// scalars, so one captured decode graph replays for every token. The M > 1 products run on dbir_gemm.
#include "common.cuh"
#include "../../include/diffbir_b200.h"

namespace {

constexpr int HD = 128;                       // head_dim of every LLaMA-7B head

// Sum of one value per thread over a 256-thread CTA in a fixed order (warp butterflies, then warps 0..7).
__device__ __forceinline__ float block_sum256(float v, float* red) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) t += red[i];
  return t;
}

// LlamaRMSNorm: out = w * x / sqrt(mean(x^2) + eps), fp32 row in, op16 row out. One CTA per row.
__global__ void __launch_bounds__(256)
rmsnorm_kernel(const float* __restrict__ x, long long ldx, int c, const float* __restrict__ w, float eps,
               op_t* __restrict__ out, long long ldo) {
  __shared__ float red[8];
  pdl_trigger();
  pdl_wait();
  const float* xr = x + blockIdx.x * ldx;
  float s = 0.f;
  for (int k = threadIdx.x * 4; k < c; k += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(xr + k);
    s += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
  }
  const float rstd = rsqrtf(block_sum256(s, red) / c + eps);
  op_t* orow = out + blockIdx.x * ldo;
  for (int k = threadIdx.x * 4; k < c; k += 1024) {
    const float4 v = *reinterpret_cast<const float4*>(xr + k);
    const float4 g = *reinterpret_cast<const float4*>(w + k);
    uint2 o;
    o.x = pack2(v.x * rstd * g.x, v.y * rstd * g.y);
    o.y = pack2(v.z * rstd * g.z, v.w * rstd * g.w);
    *reinterpret_cast<uint2*>(orow + k) = o;
  }
}

// RoPE (rotate_half form, LlamaRotaryEmbedding with base theta) on q and k of the fused QKV rows, in fp32, and the
// cache write. Row i sits at position p0[0] + i. CTA (row, head), 64 threads: thread d rotates the pair (d, d + 64).
__global__ void __launch_bounds__(64)
rope_kv_kernel(const float* __restrict__ qkv, long long ldqkv, int heads, const int* __restrict__ p0, float theta,
               op_t* __restrict__ q, long long ldq, op_t* __restrict__ kc, op_t* __restrict__ vc) {
  pdl_trigger();
  pdl_wait();
  const int row = blockIdx.x, h = blockIdx.y, d = threadIdx.x;
  const int pos = p0[0] + row;
  const float inv_freq = 1.0f / powf(theta, static_cast<float>(2 * d) / HD);
  float sn, cs;
  sincosf(static_cast<float>(pos) * inv_freq, &sn, &cs);
  const long long C = static_cast<long long>(heads) * HD;
  const float* qr = qkv + row * ldqkv + h * HD;
  const float* kr = qr + C;
  const float* vr = qr + 2 * C;
  const float q0 = qr[d], q1 = qr[d + 64], k0 = kr[d], k1 = kr[d + 64];
  op_t* qo = q + row * ldq + h * HD;
  qo[d] = f2op(q0 * cs - q1 * sn);
  qo[d + 64] = f2op(q1 * cs + q0 * sn);
  const long long slot = (static_cast<long long>(pos) * heads + h) * HD;
  kc[slot + d] = f2op(k0 * cs - k1 * sn);
  kc[slot + d + 64] = f2op(k1 * cs + k0 * sn);
  vc[slot + d] = f2op(vr[d]);
  vc[slot + d + 64] = f2op(vr[d + 64]);
}

__device__ __forceinline__ void mma_16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." DBIR_WGMMA_AB ".f32 "
               "{%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// ---- causal prefill attention (LlamaAttention with the causal mask, queries at positions 0 .. sq-1) ----
// CTA (64-query block, head), 4 warps x 16 query rows on mma.sync m16n8k16 with an online softmax over 64-key
// tiles up to the diagonal. K is staged row-major, V transposed, both op16 in shared memory with padded rows
// (272-byte K rows, 144-byte V^T rows) so every fragment load is bank-conflict free.
constexpr int CA_Q = 64, CA_K = 64;
constexpr int K_LD = HD + 8, VT_LD = CA_K + 8;

__device__ __forceinline__ uint32_t lds32(const op_t* p) { return *reinterpret_cast<const uint32_t*>(p); }
__device__ __forceinline__ uint32_t ldg32(const op_t* p) { return *reinterpret_cast<const uint32_t*>(p); }

__global__ void __launch_bounds__(128)
attention_causal_kernel(const op_t* __restrict__ q, long long ldq, const op_t* __restrict__ kc,
                        const op_t* __restrict__ vc, int heads, int sq, op_t* __restrict__ out, long long ldo) {
  __shared__ __align__(16) op_t s_k[CA_K][K_LD];
  __shared__ __align__(16) op_t s_vt[HD][VT_LD];
  pdl_trigger();
  pdl_wait();
  const int qb = blockIdx.x, h = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  const int r0 = qb * CA_Q + warp * 16 + g, r1 = r0 + 8;     // this thread's two query rows
  uint32_t qa[HD / 16][4];
  {
    const op_t* q0 = q + static_cast<long long>(min(r0, sq - 1)) * ldq + h * HD;
    const op_t* q1 = q + static_cast<long long>(min(r1, sq - 1)) * ldq + h * HD;
#pragma unroll
    for (int ks = 0; ks < HD / 16; ++ks) {
      qa[ks][0] = ldg32(q0 + ks * 16 + 2 * tq);
      qa[ks][1] = ldg32(q1 + ks * 16 + 2 * tq);
      qa[ks][2] = ldg32(q0 + ks * 16 + 8 + 2 * tq);
      qa[ks][3] = ldg32(q1 + ks * 16 + 8 + 2 * tq);
    }
  }
  float o[HD / 8][4];
#pragma unroll
  for (int d = 0; d < HD / 8; ++d) o[d][0] = o[d][1] = o[d][2] = o[d][3] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  const float sl2 = 0.08838834764831845f * 1.4426950408889634f;    // head_dim^-0.5 * log2(e)
  const long long kstride = static_cast<long long>(heads) * HD;
  for (int kb = 0; kb <= qb; ++kb) {
    __syncthreads();                                 // the previous tile has been consumed
    for (int t = tid; t < CA_K * (HD / 8); t += 128) {
      const int key = t / (HD / 8), ch = (t % (HD / 8)) * 8;
      const int gk = kb * CA_K + key;
      uint4 kv = make_uint4(0u, 0u, 0u, 0u), vv = kv;
      if (gk < sq) {
        kv = *reinterpret_cast<const uint4*>(kc + gk * kstride + h * HD + ch);
        vv = *reinterpret_cast<const uint4*>(vc + gk * kstride + h * HD + ch);
      }
      *reinterpret_cast<uint4*>(&s_k[key][ch]) = kv;
      const op_t* v = reinterpret_cast<const op_t*>(&vv);
#pragma unroll
      for (int e = 0; e < 8; ++e) s_vt[ch + e][key] = v[e];
    }
    __syncthreads();
    float s[CA_K / 8][4];
#pragma unroll
    for (int j = 0; j < CA_K / 8; ++j) {
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < HD / 16; ++ks)
        mma_16816(s[j], qa[ks], lds32(&s_k[j * 8 + g][ks * 16 + 2 * tq]), lds32(&s_k[j * 8 + g][ks * 16 + 8 + 2 * tq]));
    }
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int j = 0; j < CA_K / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int key = kb * CA_K + j * 8 + 2 * tq + e;
        float v0 = s[j][e] * sl2, v1 = s[j][2 + e] * sl2;
        if (key > r0) v0 = -INFINITY;                // causal mask (keys beyond sq lie beyond every real row)
        if (key > r1) v1 = -INFINITY;
        s[j][e] = v0; s[j][2 + e] = v1;
        mx0 = fmaxf(mx0, v0); mx1 = fmaxf(mx1, v1);
      }
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    // key 0 is never masked, so mx0 / mx1 are finite from the first tile on
    const float c0 = exp2f(m0 - mx0), c1 = exp2f(m1 - mx1);
    m0 = mx0; m1 = mx1;
    float ls0 = 0.f, ls1 = 0.f;
#pragma unroll
    for (int j = 0; j < CA_K / 8; ++j) {
      s[j][0] = exp2f(s[j][0] - m0); s[j][1] = exp2f(s[j][1] - m0);
      s[j][2] = exp2f(s[j][2] - m1); s[j][3] = exp2f(s[j][3] - m1);
      ls0 += s[j][0] + s[j][1];
      ls1 += s[j][2] + s[j][3];
    }
    ls0 += __shfl_xor_sync(0xffffffffu, ls0, 1); ls0 += __shfl_xor_sync(0xffffffffu, ls0, 2);
    ls1 += __shfl_xor_sync(0xffffffffu, ls1, 1); ls1 += __shfl_xor_sync(0xffffffffu, ls1, 2);
    l0 = l0 * c0 + ls0;
    l1 = l1 * c1 + ls1;
#pragma unroll
    for (int d = 0; d < HD / 8; ++d) { o[d][0] *= c0; o[d][1] *= c0; o[d][2] *= c1; o[d][3] *= c1; }
#pragma unroll
    for (int kk = 0; kk < CA_K / 16; ++kk) {
      const uint32_t pa[4] = {pack2(s[2 * kk][0], s[2 * kk][1]), pack2(s[2 * kk][2], s[2 * kk][3]),
                              pack2(s[2 * kk + 1][0], s[2 * kk + 1][1]), pack2(s[2 * kk + 1][2], s[2 * kk + 1][3])};
#pragma unroll
      for (int d = 0; d < HD / 8; ++d)
        mma_16816(o[d], pa, lds32(&s_vt[d * 8 + g][kk * 16 + 2 * tq]), lds32(&s_vt[d * 8 + g][kk * 16 + 8 + 2 * tq]));
    }
  }
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  if (r0 < sq) {
    op_t* orow = out + static_cast<long long>(r0) * ldo + h * HD + 2 * tq;
#pragma unroll
    for (int d = 0; d < HD / 8; ++d) *reinterpret_cast<uint32_t*>(orow + d * 8) = pack2(o[d][0] * inv0, o[d][1] * inv0);
  }
  if (r1 < sq) {
    op_t* orow = out + static_cast<long long>(r1) * ldo + h * HD + 2 * tq;
#pragma unroll
    for (int d = 0; d < HD / 8; ++d) *reinterpret_cast<uint32_t*>(orow + d * 8) = pack2(o[d][2] * inv1, o[d][3] * inv1);
  }
}

// ---- decode-step attention: one query row per head against the first len[0] cache rows ----
// Pass 1: CTA (head, split) takes keys [split * 64, split * 64 + 64) and writes its running max, sum of
// exponentials and un-normalised output to the workspace; splits past the length exit. Pass 2: CTA per head
// combines the splits in index order (deterministic).
constexpr int DEC_CHUNK = 64;

__global__ void __launch_bounds__(128)
attention_decode_part_kernel(const op_t* __restrict__ q, const op_t* __restrict__ kc, const op_t* __restrict__ vc,
                             int heads, const int* __restrict__ len, float* __restrict__ ws) {
  __shared__ float s_p[DEC_CHUNK];
  __shared__ float s_red[2];
  pdl_trigger();
  pdl_wait();
  const int h = blockIdx.x, split = blockIdx.y, nsplit = gridDim.y;
  const int L = len[0];
  const int k0 = split * DEC_CHUNK;
  if (k0 >= L) return;
  const int nk = min(DEC_CHUNK, L - k0);
  const int tid = threadIdx.x;
  const long long kstride = static_cast<long long>(heads) * HD;
  // scores: 16 threads per key (8 dims each), 8 keys per pass
  {
    const int sub = tid & 15, kk = tid >> 4;
    const uint4 qv = *reinterpret_cast<const uint4*>(q + h * HD + sub * 8);
    const uint32_t* qw = reinterpret_cast<const uint32_t*>(&qv);
    for (int j = kk; j < DEC_CHUNK; j += 8) {
      float acc = 0.f;
      if (j < nk) {
        const uint4 kv = *reinterpret_cast<const uint4*>(kc + (k0 + j) * kstride + h * HD + sub * 8);
        const uint32_t* kw = reinterpret_cast<const uint32_t*>(&kv);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 a = unpack2(qw[e]), b = unpack2(kw[e]);
          acc = fmaf(a.x, b.x, acc);
          acc = fmaf(a.y, b.y, acc);
        }
      }
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
      if (sub == 0) s_p[j] = j < nk ? acc * (0.08838834764831845f * 1.4426950408889634f) : -INFINITY;
    }
  }
  __syncthreads();
  if (tid < 32) {
    const float a = s_p[tid], b = s_p[tid + 32];
    const float m = warp_max(fmaxf(a, b));
    const float ea = exp2f(a - m), eb = exp2f(b - m);
    s_p[tid] = ea;
    s_p[tid + 32] = eb;
    const float l = warp_sum(ea + eb);
    if (tid == 0) { s_red[0] = m; s_red[1] = l; }
  }
  __syncthreads();
  float acc = 0.f;
  const op_t* vcol = vc + h * HD + tid;
  for (int j = 0; j < nk; ++j) acc = fmaf(s_p[j], op2f(vcol[(k0 + j) * kstride]), acc);
  float* w = ws + (static_cast<long long>(h) * nsplit + split) * (HD + 2);
  w[2 + tid] = acc;
  if (tid == 0) { w[0] = s_red[0]; w[1] = s_red[1]; }
}

__global__ void __launch_bounds__(128)
attention_decode_combine_kernel(const float* __restrict__ ws, const int* __restrict__ len, int nsplit,
                                op_t* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int h = blockIdx.x, tid = threadIdx.x;
  const int used = (len[0] + DEC_CHUNK - 1) / DEC_CHUNK;
  const float* w = ws + static_cast<long long>(h) * nsplit * (HD + 2);
  float m = -INFINITY;
  for (int s = 0; s < used; ++s) m = fmaxf(m, w[s * (HD + 2)]);
  float l = 0.f, acc = 0.f;
  for (int s = 0; s < used; ++s) {
    const float c = exp2f(w[s * (HD + 2)] - m);
    l = fmaf(c, w[s * (HD + 2) + 1], l);
    acc = fmaf(c, w[s * (HD + 2) + 2 + tid], acc);
  }
  out[h * HD + tid] = f2op(acc / l);
}

// ---- y = W x for one input row (decode step) ----
// One warp per output (SwiGLU: per value / gate row pair), 16-byte loads of the op16 weight row, fp32
// accumulation in a fixed order (lane-strided partial sums, then a butterfly). x is read through L1.
// mode 0: y = Wx; 1: y = Wx + residual; 2: SwiGLU over rows packed per `pack`-row tile as [values | gates]:
// y[c] = v(c) * silu(g(c)) with v / g the rows of c's tile (dbir_gemm's geglu = 2 packing).
constexpr int GEMV_WARPS = 8;

template <int MODE>
__global__ void __launch_bounds__(GEMV_WARPS * 32)
gemv_kernel(const op_t* __restrict__ w, long long ldw, const op_t* __restrict__ x, int n_out, int K, int pack,
            const float* residual, void* y, int out_kind) {
  pdl_trigger();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x * GEMV_WARPS + warp;
  if (c >= n_out) return;
  long long ra = c, rb = 0;
  if (MODE == 2) {
    const int hb = pack / 2, t = c / hb, j = c % hb;
    ra = static_cast<long long>(t) * pack + j;
    rb = ra + hb;
  }
  const op_t* wa = w + ra * ldw;
  const op_t* wb = w + rb * ldw;
  float sa = 0.f, sb = 0.f;
#pragma unroll 4
  for (int k = lane * 8; k < K; k += 256) {
    const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + k));
    const uint4 av = __ldcs(reinterpret_cast<const uint4*>(wa + k));
    const uint32_t* xw = reinterpret_cast<const uint32_t*>(&xv);
    const uint32_t* aw = reinterpret_cast<const uint32_t*>(&av);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 xf = unpack2(xw[e]), af = unpack2(aw[e]);
      sa = fmaf(af.x, xf.x, sa);
      sa = fmaf(af.y, xf.y, sa);
    }
    if (MODE == 2) {
      const uint4 bv = __ldcs(reinterpret_cast<const uint4*>(wb + k));
      const uint32_t* bw = reinterpret_cast<const uint32_t*>(&bv);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 xf = unpack2(xw[e]), bf = unpack2(bw[e]);
        sb = fmaf(bf.x, xf.x, sb);
        sb = fmaf(bf.y, xf.y, sb);
      }
    }
  }
  sa = warp_sum(sa);
  if (MODE == 2) sb = warp_sum(sb);
  if (lane == 0) {
    float v = sa;
    if (MODE == 1) v += residual[c];
    if (MODE == 2) v = sa * silu_f(sb);
    if (out_kind == 0) static_cast<float*>(y)[c] = v;
    else static_cast<op_t*>(y)[c] = f2op(v);
  }
}

// First maximum of n fp32 logits -> *token; then every advance[i] += 1 (the decode step's position / length).
__global__ void __launch_bounds__(1024)
argmax_kernel(const float* __restrict__ logits, int n, int* __restrict__ token, int* advance, int n_advance) {
  __shared__ float s_v[32];
  __shared__ int s_i[32];
  pdl_trigger();
  pdl_wait();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int i = tid; i < n; i += 1024) {
    const float v = logits[i];
    if (v > best) { best = v; bi = i; }         // increasing i per thread: keeps the first maximum
  }
  auto merge = [&](float ov, int oi) {
    if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
  };
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    merge(ov, oi);
  }
  if (lane == 0) { s_v[warp] = best; s_i[warp] = bi; }
  __syncthreads();
  if (warp == 0) {
    best = s_v[lane]; bi = s_i[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      merge(ov, oi);
    }
    if (lane == 0) {
      *token = bi == 0x7fffffff ? 0 : bi;       // all-NaN logits: token 0
      for (int i = 0; i < n_advance; ++i) advance[i] += 1;
    }
  }
}

// out row i (fp32) = embed_tokens[ids[i]] (op16).
__global__ void __launch_bounds__(256)
embed_gather_kernel(const op_t* __restrict__ table, int vocab, const int* __restrict__ ids, int dim,
                    float* __restrict__ out, long long ldo) {
  pdl_trigger();
  pdl_wait();
  const int id = min(max(ids[blockIdx.x], 0), vocab - 1);
  const op_t* src = table + static_cast<long long>(id) * dim;
  float* dst = out + blockIdx.x * ldo;
  for (int k = threadIdx.x * 2; k < dim; k += 512) {
    const float2 v = unpack2(*reinterpret_cast<const uint32_t*>(src + k));
    *reinterpret_cast<float2*>(dst + k) = v;
  }
}

inline cudaStream_t ST(void* s) { return reinterpret_cast<cudaStream_t>(s); }
inline bool al16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

}  // namespace

extern "C" int dbir_rmsnorm(const float* x, int64_t ldx, int32_t rows, int32_t c, const float* w, float eps, void* out,
                            int64_t ldo, void* stream) {
  DBIR_REQUIRE(x && w && out && rows > 0 && c > 0 && c % 4 == 0 && ldx % 4 == 0 && ldo % 4 == 0 && al16(x) && al16(w),
               "dbir_rmsnorm: bad args (c, ldx, ldo multiples of 4, 16-byte aligned rows)");
  DBIR_CHECK_CUDA(dbir_launch(rmsnorm_kernel, dim3(rows), dim3(256), 0, ST(stream), x, static_cast<long long>(ldx), c,
                              w, eps, reinterpret_cast<op_t*>(out), static_cast<long long>(ldo)));
  return 0;
}

extern "C" int dbir_rope_kv(const float* qkv, int64_t ldqkv, int32_t rows, int32_t heads, const int32_t* p0,
                            float theta, void* q, int64_t ldq, void* k_cache, void* v_cache, void* stream) {
  DBIR_REQUIRE(qkv && p0 && q && k_cache && v_cache && rows > 0 && heads > 0 && ldqkv >= 3LL * heads * HD &&
                   ldq >= static_cast<int64_t>(heads) * HD,
               "dbir_rope_kv: bad args");
  DBIR_CHECK_CUDA(dbir_launch(rope_kv_kernel, dim3(rows, heads), dim3(HD / 2), 0, ST(stream), qkv,
                              static_cast<long long>(ldqkv), heads, p0, theta, reinterpret_cast<op_t*>(q),
                              static_cast<long long>(ldq), reinterpret_cast<op_t*>(k_cache),
                              reinterpret_cast<op_t*>(v_cache)));
  return 0;
}

extern "C" int dbir_attention_causal(const void* q, int64_t ldq, const void* k_cache, const void* v_cache, int32_t heads,
                                     int32_t sq, void* out, int64_t ldo, void* stream) {
  DBIR_REQUIRE(q && k_cache && v_cache && out && heads > 0 && sq > 0 && ldq % 2 == 0 && ldo % 2 == 0 &&
                   al16(k_cache) && al16(v_cache),
               "dbir_attention_causal: bad args");
  DBIR_CHECK_CUDA(dbir_launch(attention_causal_kernel, dim3((sq + CA_Q - 1) / CA_Q, heads), dim3(128), 0, ST(stream),
                              reinterpret_cast<const op_t*>(q), static_cast<long long>(ldq),
                              reinterpret_cast<const op_t*>(k_cache), reinterpret_cast<const op_t*>(v_cache), heads, sq,
                              reinterpret_cast<op_t*>(out), static_cast<long long>(ldo)));
  return 0;
}

extern "C" int64_t dbir_attention_decode_ws_bytes(int32_t heads, int32_t capacity) {
  return static_cast<int64_t>(heads) * ((capacity + DEC_CHUNK - 1) / DEC_CHUNK) * (HD + 2) * 4;
}

extern "C" int dbir_attention_decode(const void* q, const void* k_cache, const void* v_cache, int32_t heads,
                                     int32_t capacity, const int32_t* len, void* ws, int64_t ws_bytes, void* out,
                                     void* stream) {
  DBIR_REQUIRE(q && k_cache && v_cache && len && ws && out && heads > 0 && capacity > 0 && al16(q) && al16(k_cache),
               "dbir_attention_decode: bad args");
  DBIR_REQUIRE(ws_bytes >= dbir_attention_decode_ws_bytes(heads, capacity),
               "dbir_attention_decode: workspace of %lld bytes, need %lld", (long long)ws_bytes,
               (long long)dbir_attention_decode_ws_bytes(heads, capacity));
  const int nsplit = (capacity + DEC_CHUNK - 1) / DEC_CHUNK;
  DBIR_CHECK_CUDA(dbir_launch(attention_decode_part_kernel, dim3(heads, nsplit), dim3(128), 0, ST(stream),
                              reinterpret_cast<const op_t*>(q), reinterpret_cast<const op_t*>(k_cache),
                              reinterpret_cast<const op_t*>(v_cache), heads, len, static_cast<float*>(ws)));
  DBIR_CHECK_CUDA(dbir_launch(attention_decode_combine_kernel, dim3(heads), dim3(HD), 0, ST(stream),
                              static_cast<const float*>(ws), len, nsplit, reinterpret_cast<op_t*>(out)));
  return 0;
}

extern "C" int dbir_gemv(const void* w, int64_t ldw, const void* x, int32_t N, int32_t K, int32_t epilogue,
                         int32_t pack, const float* residual, void* y, int32_t out_kind, void* stream) {
  DBIR_REQUIRE(w && x && y && N > 0 && K > 0 && K % 8 == 0 && ldw >= K && ldw % 8 == 0 && al16(w) && al16(x),
               "dbir_gemv: bad args (K and ldw multiples of 8, 16-byte aligned operands)");
  DBIR_REQUIRE(epilogue >= 0 && epilogue <= 2 && (out_kind == 0 || out_kind == 1), "dbir_gemv: bad epilogue / out_kind");
  DBIR_REQUIRE(epilogue != 1 || residual, "dbir_gemv: epilogue 1 needs a residual");
  DBIR_REQUIRE(epilogue != 2 || (pack >= 2 && pack % 2 == 0 && N % pack == 0),
               "dbir_gemv: SwiGLU needs the tile width `pack` (even, dividing N)");
  const int n_out = epilogue == 2 ? N / 2 : N;
  const dim3 grid((n_out + GEMV_WARPS - 1) / GEMV_WARPS), block(GEMV_WARPS * 32);
  const op_t* wp = reinterpret_cast<const op_t*>(w);
  const op_t* xp = reinterpret_cast<const op_t*>(x);
  const long long l = ldw;
  if (epilogue == 0)
    DBIR_CHECK_CUDA(dbir_launch(gemv_kernel<0>, grid, block, 0, ST(stream), wp, l, xp, n_out, K, pack, residual, y, out_kind));
  else if (epilogue == 1)
    DBIR_CHECK_CUDA(dbir_launch(gemv_kernel<1>, grid, block, 0, ST(stream), wp, l, xp, n_out, K, pack, residual, y, out_kind));
  else
    DBIR_CHECK_CUDA(dbir_launch(gemv_kernel<2>, grid, block, 0, ST(stream), wp, l, xp, n_out, K, pack, residual, y, out_kind));
  return 0;
}

extern "C" int dbir_argmax(const float* logits, int32_t n, int32_t* token, int32_t* advance, int32_t n_advance,
                           void* stream) {
  DBIR_REQUIRE(logits && token && n > 0 && n_advance >= 0 && (n_advance == 0 || advance), "dbir_argmax: bad args");
  DBIR_CHECK_CUDA(dbir_launch(argmax_kernel, dim3(1), dim3(1024), 0, ST(stream), logits, n, token, advance, n_advance));
  return 0;
}

extern "C" int dbir_embed_gather(const void* table, int32_t vocab, const int32_t* ids, int32_t n, int32_t dim, float* out,
                                 int64_t ldo, void* stream) {
  DBIR_REQUIRE(table && ids && out && n > 0 && vocab > 0 && dim % 2 == 0 && ldo % 2 == 0, "dbir_embed_gather: bad args");
  DBIR_CHECK_CUDA(dbir_launch(embed_gather_kernel, dim3(n), dim3(256), 0, ST(stream), reinterpret_cast<const op_t*>(table),
                              vocab, ids, dim, out, static_cast<long long>(ldo)));
  return 0;
}
