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

}  // namespace

extern "C" int dbir_window_attention(const void* qkv, int64_t ldq, int32_t batch, int32_t h, int32_t w, int32_t heads,
                                     int32_t head_dim, int32_t window, int32_t shift, const float* bias_table,
                                     float mask_value, void* out, int64_t ldo, void* stream) {
  DBIR_REQUIRE(qkv && bias_table && out, "dbir_window_attention: null pointer");
  DBIR_REQUIRE(window == 8, "dbir_window_attention: built for 8 x 8 windows");
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

extern "C" int dbir_swin_window_attention(const void* qkv, int64_t ldq, int32_t batch, int32_t h,
                                          int32_t w, int32_t heads, int32_t head_dim,
                                          int32_t window, int32_t shift, const float* bias_table,
                                          void* out, int64_t ldo, void* stream) {
  return dbir_window_attention(qkv, ldq, batch, h, w, heads, head_dim, window, shift, bias_table, -100.0f, out, ldo, stream);
}
