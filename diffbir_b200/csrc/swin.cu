// SwinIR window multi-head self-attention (W-MSA / SW-MSA), one CTA per (8x8 window, head).
//
// Replaces WindowAttention.forward (reference swinir.py:120-151) together with the data
// movement around it in SwinTransformerBlock.forward (swinir.py:255-276): torch.roll,
// window_partition, window_reverse and the reverse roll are folded into the gather/scatter
// addressing; the shift mask (swinir.py:222-243, -100 across region borders) is evaluated
// analytically; the relative-position bias is gathered from the [ (2w-1)^2, heads ] table.
//
// 64 threads, thread == query token. The head's K and V rows (64 x 30, zero-padded to 32) are
// staged in shared memory as fp32 and read as warp-wide broadcasts (LDS.128, conflict-free);
// the query row, the 64 scores, the softmax and the 30 outputs stay in registers. HBM-/latency-
// bound (6 MB of qkv + 2 MB of output per 512^2 image, 0.19 GFLOP): the grid of
// windows x heads = 384 CTAs at 512^2 fills the 132 SMs where one CTA per window (64 CTAs with
// two query rows per lane) leaves most of them idle.
#include "common.cuh"
#include "../../include/diffbir_b200.h"

namespace {

constexpr int WS = 8;
constexpr int NTOK = WS * WS;   // 64

template <int HEADS, int DH>
__global__ void __launch_bounds__(NTOK)
swin_window_attn_kernel(const op_t* __restrict__ qkv, long long ldq, int H, int W, int shift,
                        const float* __restrict__ bias_table, op_t* __restrict__ out,
                        long long ldo, float mask_value) {
  constexpr int C = HEADS * DH;
  constexpr int DP = 32;                          // DH padded for float4 rows
  static_assert(DH <= DP && DH % 2 == 0, "head_dim must be even and <= 32");
  constexpr int NB = (2 * WS - 1) * (2 * WS - 1);
  __shared__ __align__(16) float s_k[NTOK][DP];
  __shared__ __align__(16) float s_v[NTOK][DP];
  __shared__ float s_bias[NB];
  __shared__ int s_reg[NTOK];

  pdl_trigger();
  pdl_wait();                                     // qkv comes from the predecessor GEMM
  const int head = blockIdx.x % HEADS;
  int wid = blockIdx.x / HEADS;
  const int wins_x = W / WS, wins_y = H / WS;
  const int wx = wid % wins_x; wid /= wins_x;
  const int wy = wid % wins_y; wid /= wins_y;
  const int b = wid;
  const int i = threadIdx.x;                      // query token of this thread
  const int iy = i / WS, ix = i % WS;

  // token -> global row (roll by -shift folded in) and mask region
  const int sy = wy * WS + iy, sx = wx * WS + ix;              // coordinates in the shifted frame
  const int gy = (sy + shift) % H, gx = (sx + shift) % W;      // original position
  const long long row = (static_cast<long long>(b) * H + gy) * W + gx;
  int reg_i = 0;
  if (shift > 0) {
    const int rh = sy < H - WS ? 0 : (sy < H - shift ? 1 : 2);
    const int rw = sx < W - WS ? 0 : (sx < W - shift ? 1 : 2);
    reg_i = rh * 3 + rw;
  }
  s_reg[i] = reg_i;
  for (int t = i; t < NB; t += NTOK) s_bias[t] = bias_table[t * HEADS + head];

  // this token's q (registers, pre-scaled), k and v (shared, fp32)
  const op_t* base = qkv + row * ldq + head * DH;
  const float scale = rsqrtf(static_cast<float>(DH));
  float q[DP];
#pragma unroll
  for (int d = 0; d < DH; d += 2) {
    const float2 tq = unpack2(*reinterpret_cast<const uint32_t*>(base + d));
    const float2 tk = unpack2(*reinterpret_cast<const uint32_t*>(base + C + d));
    const float2 tv = unpack2(*reinterpret_cast<const uint32_t*>(base + 2 * C + d));
    q[d] = tq.x * scale; q[d + 1] = tq.y * scale;
    s_k[i][d] = tk.x; s_k[i][d + 1] = tk.y;
    s_v[i][d] = tv.x; s_v[i][d + 1] = tv.y;
  }
#pragma unroll
  for (int d = DH; d < DP; ++d) { q[d] = 0.f; s_k[i][d] = 0.f; s_v[i][d] = 0.f; }
  __syncthreads();

  unsigned long long masked = 0ull;               // bit j: token j lies in another mask region
  if (shift > 0) {
#pragma unroll 8
    for (int j = 0; j < NTOK; ++j) masked |= static_cast<unsigned long long>(s_reg[j] != reg_i) << j;
  }
  const int bias_base = (iy + WS - 1) * (2 * WS - 1) + (ix + WS - 1);
  float sc[NTOK];
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < NTOK; ++j) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll
    for (int d = 0; d < DP; d += 4) {
      const float4 k4 = *reinterpret_cast<const float4*>(&s_k[j][d]);
      a0 = fmaf(q[d], k4.x, a0); a1 = fmaf(q[d + 1], k4.y, a1);
      a2 = fmaf(q[d + 2], k4.z, a2); a3 = fmaf(q[d + 3], k4.w, a3);
    }
    float acc = (a0 + a1) + (a2 + a3);
    acc += s_bias[bias_base - ((j / WS) * (2 * WS - 1) + (j % WS))];
    if ((masked >> j) & 1ull) acc += mask_value;       // -100 (SwinIR, swinir.py:241) or -inf (SCUNet, scunet.py:77)
    sc[j] = acc;
    m = fmaxf(m, acc);
  }
  float l = 0.f;
#pragma unroll
  for (int j = 0; j < NTOK; ++j) { sc[j] = __expf(sc[j] - m); l += sc[j]; }
  const float inv = 1.0f / l;
  float o[DP];
#pragma unroll
  for (int d = 0; d < DP; ++d) o[d] = 0.f;
#pragma unroll
  for (int j = 0; j < NTOK; ++j) {
    const float pj = sc[j];
#pragma unroll
    for (int d = 0; d < DP; d += 4) {
      const float4 v4 = *reinterpret_cast<const float4*>(&s_v[j][d]);
      o[d] = fmaf(pj, v4.x, o[d]); o[d + 1] = fmaf(pj, v4.y, o[d + 1]);
      o[d + 2] = fmaf(pj, v4.z, o[d + 2]); o[d + 3] = fmaf(pj, v4.w, o[d + 3]);
    }
  }
  op_t* orow = out + row * ldo + head * DH;
#pragma unroll
  for (int d = 0; d < DH; d += 2)
    *reinterpret_cast<uint32_t*>(orow + d) = pack2(o[d] * inv, o[d + 1] * inv);
}

// ---- 12 x 12 windows, head_dim 32 (Swin-L, the RAM++ image encoder: ram/models/swin_transformer.py:68-273) ----
// One CTA per (window, head), 9 warps x 16 query rows on mma.sync m16n8k16 (fp32 accumulate). With 144 keys a
// thread-per-query design would hold 144 scores plus q and o in registers and spill; here a thread holds the
// 18 x 4 score fragments of its two rows, softmaxes them in registers (quad shuffles) and feeds them straight back
// as the A fragments of P V. Q and K are staged row-major, V transposed, all op16 in shared memory; rows padded so
// every fragment load is bank-conflict free (80-byte Q / K rows, 304-byte V^T rows).
constexpr int WS12 = 12;
constexpr int NTOK12 = WS12 * WS12;           // 144
constexpr int QK_LD = 40;                     // 32 dims + 8 pad (op16 elements)
constexpr int VT_LD = NTOK12 + 8;             // 144 keys + 8 pad

__device__ __forceinline__ void mma_16816(float* d, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32." DBIR_WGMMA_AB ".f32 "
               "{%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint32_t lds32(const op_t* p) { return *reinterpret_cast<const uint32_t*>(p); }

__global__ void __launch_bounds__(9 * 32)
swin_window12_attn_kernel(const op_t* __restrict__ qkv, long long ldq, int H, int W, int heads, int shift,
                          const float* __restrict__ bias_table, op_t* __restrict__ out, long long ldo,
                          float mask_value) {
  constexpr int DH = 32;
  constexpr int TW = 2 * WS12 - 1;            // 23
  constexpr int NB = TW * TW;
  __shared__ __align__(16) op_t s_q[NTOK12][QK_LD];
  __shared__ __align__(16) op_t s_k[NTOK12][QK_LD];
  __shared__ __align__(16) op_t s_vt[DH][VT_LD];
  __shared__ float s_bias[NB];
  __shared__ long long s_row[NTOK12];
  __shared__ int s_pos[NTOK12];               // y * 23 + x of the token inside the window
  __shared__ int s_reg[NTOK12];               // shift-mask region

  pdl_trigger();
  pdl_wait();                                 // qkv comes from the predecessor GEMM
  const int head = blockIdx.x % heads;
  int wid = blockIdx.x / heads;
  const int wins_x = W / WS12, wins_y = H / WS12;
  const int wx = wid % wins_x; wid /= wins_x;
  const int wy = wid % wins_y; wid /= wins_y;
  const int b = wid;
  const int tid = threadIdx.x;
  if (tid < NTOK12) {
    const int iy = tid / WS12, ix = tid % WS12;
    const int sy = wy * WS12 + iy, sx = wx * WS12 + ix;        // shifted frame
    const int gy = (sy + shift) % H, gx = (sx + shift) % W;    // original position (roll by -shift folded in)
    s_row[tid] = (static_cast<long long>(b) * H + gy) * W + gx;
    s_pos[tid] = iy * TW + ix;
    int reg = 0;
    if (shift > 0) {
      const int rh = sy < H - WS12 ? 0 : (sy < H - shift ? 1 : 2);
      const int rw = sx < W - WS12 ? 0 : (sx < W - shift ? 1 : 2);
      reg = rh * 3 + rw;
    }
    s_reg[tid] = reg;
  }
  for (int t = tid; t < NB; t += blockDim.x) s_bias[t] = bias_table[t * heads + head];
  __syncthreads();
  const long long C = static_cast<long long>(heads) * DH;
  for (int t = tid; t < NTOK12 * 4; t += blockDim.x) {
    const int tok = t >> 2, ch = (t & 3) * 8;
    const op_t* base = qkv + s_row[tok] * ldq + head * DH + ch;
    *reinterpret_cast<uint4*>(&s_q[tok][ch]) = *reinterpret_cast<const uint4*>(base);
    *reinterpret_cast<uint4*>(&s_k[tok][ch]) = *reinterpret_cast<const uint4*>(base + C);
    const uint4 v4 = *reinterpret_cast<const uint4*>(base + 2 * C);
    const op_t* v = reinterpret_cast<const op_t*>(&v4);
#pragma unroll
    for (int e = 0; e < 8; ++e) s_vt[ch + e][tok] = v[e];
  }
  __syncthreads();

  const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  const int r0 = warp * 16 + g, r1 = r0 + 8;  // the two query rows of this thread
  uint32_t qa[2][4];
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    qa[ks][0] = lds32(&s_q[r0][ks * 16 + 2 * tq]);
    qa[ks][1] = lds32(&s_q[r1][ks * 16 + 2 * tq]);
    qa[ks][2] = lds32(&s_q[r0][ks * 16 + 8 + 2 * tq]);
    qa[ks][3] = lds32(&s_q[r1][ks * 16 + 8 + 2 * tq]);
  }
  constexpr int NT = NTOK12 / 8;              // 18 key tiles
  float s[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
      mma_16816(s[j], qa[ks], lds32(&s_k[j * 8 + g][ks * 16 + 2 * tq]), lds32(&s_k[j * 8 + g][ks * 16 + 8 + 2 * tq]));
  }
  const float scale = 0.17677669529663687f;   // head_dim ** -0.5
  const int pb0 = s_pos[r0] + (WS12 - 1) * (TW + 1), pb1 = s_pos[r1] + (WS12 - 1) * (TW + 1);
  const int reg0 = s_reg[r0], reg1 = s_reg[r1];
  float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int key = j * 8 + 2 * tq + e;
      const int kp = s_pos[key], kr = s_reg[key];
      float v0 = fmaf(s[j][e], scale, s_bias[pb0 - kp]);
      float v1 = fmaf(s[j][2 + e], scale, s_bias[pb1 - kp]);
      if (kr != reg0) v0 += mask_value;       // regions differ only when shift > 0
      if (kr != reg1) v1 += mask_value;
      s[j][e] = v0; s[j][2 + e] = v1;
      m0 = fmaxf(m0, v0); m1 = fmaxf(m1, v1);
    }
  }
  m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1)); m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
  m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
  float l0 = 0.f, l1 = 0.f;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    s[j][0] = __expf(s[j][0] - m0); s[j][1] = __expf(s[j][1] - m0);
    s[j][2] = __expf(s[j][2] - m1); s[j][3] = __expf(s[j][3] - m1);
    l0 += s[j][0] + s[j][1];
    l1 += s[j][2] + s[j][3];
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);

  float o[4][4];
#pragma unroll
  for (int d = 0; d < 4; ++d) o[d][0] = o[d][1] = o[d][2] = o[d][3] = 0.f;
#pragma unroll
  for (int kk = 0; kk < NT / 2; ++kk) {       // 16 keys per step: score tiles 2kk, 2kk+1 are P's A fragment
    const uint32_t pa[4] = {pack2(s[2 * kk][0], s[2 * kk][1]), pack2(s[2 * kk][2], s[2 * kk][3]),
                            pack2(s[2 * kk + 1][0], s[2 * kk + 1][1]), pack2(s[2 * kk + 1][2], s[2 * kk + 1][3])};
#pragma unroll
    for (int d = 0; d < 4; ++d)
      mma_16816(o[d], pa, lds32(&s_vt[d * 8 + g][kk * 16 + 2 * tq]), lds32(&s_vt[d * 8 + g][kk * 16 + 8 + 2 * tq]));
  }
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  op_t* o0 = out + s_row[r0] * ldo + head * DH + 2 * tq;
  op_t* o1 = out + s_row[r1] * ldo + head * DH + 2 * tq;
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    *reinterpret_cast<uint32_t*>(o0 + d * 8) = pack2(o[d][0] * inv0, o[d][1] * inv0);
    *reinterpret_cast<uint32_t*>(o1 + d * 8) = pack2(o[d][2] * inv1, o[d][3] * inv1);
  }
}

}  // namespace

extern "C" int dbir_window_attention(const void* qkv, int64_t ldq, int32_t batch, int32_t h, int32_t w, int32_t heads,
                                     int32_t head_dim, int32_t window, int32_t shift, const float* bias_table,
                                     float mask_value, void* out, int64_t ldo, void* stream) {
  DBIR_REQUIRE(qkv && bias_table && out, "dbir_window_attention: null pointer");
  if (window == WS12) {
    DBIR_REQUIRE(head_dim == 32 && heads > 0, "dbir_window_attention: 12 x 12 windows need head_dim 32 (got %d x %d)",
                 heads, head_dim);
    DBIR_REQUIRE(h % WS12 == 0 && w % WS12 == 0 && ldq % 8 == 0 && ldo % 2 == 0 && shift >= 0 && shift < WS12 &&
                     reinterpret_cast<uintptr_t>(qkv) % 16 == 0,
                 "dbir_window_attention: bad geometry for 12 x 12 windows");
    const int nwin12 = batch * (h / WS12) * (w / WS12);
    DBIR_CHECK_CUDA(dbir_launch(swin_window12_attn_kernel, dim3(nwin12 * heads), dim3(9 * 32), 0,
                                reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const op_t*>(qkv),
                                static_cast<long long>(ldq), h, w, heads, shift, bias_table,
                                reinterpret_cast<op_t*>(out), static_cast<long long>(ldo), mask_value));
    return 0;
  }
  DBIR_REQUIRE(window == 8, "dbir_window_attention: built for 8 x 8 and 12 x 12 windows");
  DBIR_REQUIRE(h % 8 == 0 && w % 8 == 0 && ldq % 2 == 0 && ldo % 2 == 0 && shift >= 0 && shift < 8,
               "dbir_window_attention: bad geometry");
  const int nwin = batch * (h / 8) * (w / 8);
#define DBIR_WIN(H_, D_)                                                                                             \
  if (heads == H_ && head_dim == D_) {                                                                                \
    DBIR_CHECK_CUDA(dbir_launch(swin_window_attn_kernel<H_, D_>, dim3(nwin * H_), dim3(NTOK), 0,                      \
                                reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const op_t*>(qkv),          \
                                static_cast<long long>(ldq), h, w, shift, bias_table, reinterpret_cast<op_t*>(out),   \
                                static_cast<long long>(ldo), mask_value));                                            \
    return 0;                                                                                                         \
  }
  DBIR_WIN(6, 30)      // SwinIR stage 1 (configs/inference/swinir.yaml)
  DBIR_WIN(1, 32)      // SCUNet levels: trans_dim 32 / 64 / 128 / 256, head_dim 32 (scunet.py:167-168)
  DBIR_WIN(2, 32)
  DBIR_WIN(4, 32)
  DBIR_WIN(8, 32)
#undef DBIR_WIN
  dbir_set_error("dbir_window_attention: unsupported heads x head_dim %d x %d", heads, head_dim);
  return -2;
}
