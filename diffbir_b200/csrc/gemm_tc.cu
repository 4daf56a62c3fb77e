// wgmma / TMA GEMM with an implicit-GEMM 3x3 convolution mode (sm_90a).
//
//   D[M, N] = A[M, K] * B[N, K]^T   (16-bit operands, fp32 accumulate in registers)
//
// A is either a plain row-major [M, K] matrix (Linear layers, 1x1 convs on NHWC
// activations) or an NHWC activation tensor read through a 4-D TMA box, one box per
// filter tap, with the hardware's out-of-bounds zero fill providing the conv padding
// (replaces nn.Conv2d 3x3/pad 1 at reference unet.py:149-153,173-180, vae.py:77-86,
// swinir.py:472,797-811). B is the packed weight [N, K] (K = taps*C, tap-major).
//
// One CTA computes a 128 x BN tile: warps 0-7 are two consumer warpgroups (tile rows 0-63 / 64-127,
// wgmma with both operands in shared memory, accumulators in registers), warp 8 is the TMA producer.
// After the mainloop the accumulators go to the freed stage memory as swizzled 32 x 32 fp32 blocks and
// the same eight warps run the epilogue on them (thread == accumulator row).
//
// Epilogue (per warp, 32 rows x 32 columns at a time): accumulator block -> bias / per-image row
// vector (time embedding) / GELU / LeakyReLU / SiLU / GEGLU gating / alpha -> + fp32 residual
// tile (TMA-loaded, double buffered) -> swizzled shared-memory tile -> TMA bulk store
// (from the accumulator block itself). Threads never touch global memory for the output, and the TMA
// unit clips overhanging rows / columns (M, N tails, conv tiles that overhang the image).
//   out = residual + alpha * act(acc + bias + rowvec),  fp32 or 16-bit, any row stride.
#include "common.cuh"
#include "../../include/diffbir_b200.h"
#include <stdlib.h>
#include <array>
#include <map>
#include <mutex>
#include <type_traits>
#include <utility>
#include <vector>

namespace {

constexpr int BM = 128;
constexpr int BK = 64;                 // 64 x 16-bit = 128 B = one swizzle atom row
constexpr int A_SUB_BYTES = BM * BK * 2;    // one 64-wide k-block of A
constexpr int EPI_TILE_BYTES = 32 * 32 * 4;   // one warp's 32x32 fp32 staging tile

struct GemmParams {
  int M, N, num_kb;
  // conv geometry (mode 1)
  int mode;                // 0 plain, 1 conv taps over NHWC
  int H, W, NI;            // image size / count
  int bw, bh, bni;         // box extents (bw*bh*bni == 128)
  int tiles_x, tiles_y;    // tiles per image row / column
  int cblocks;             // C / 64
  int kw, pad;             // filter width (taps = kw*kw), padding
  int wbw, wbh;            // per-warp sub-box (32 rows) extents in w / h
  // epilogue
  int out_kind;            // 0 fp32, 1 16-bit operand
  const float* bias;
  const float* rowvec;     // [NI or M/rows_per_vec, N]
  int rows_per_vec;
  int has_residual;
  float alpha;
  int act;                 // 0 none, 1 gelu(erf), 2 leaky relu (slope in act_param), 3 silu, 4 quick_gelu
  float act_param;
  int geglu;               // 1: tile holds [BN/2 values | BN/2 gates], out = values * gelu(gates); 2: the same
                           // packing, out = values * silu(gates) (SwiGLU); output width N/2
  int bias_per_row;        // bias indexed by output row instead of column
  // grouped launch: G same-shape problems back to back along M; group g's weights / bias start at row g*N
  int group_span;          // m-tiles (plain) or images (conv) per group; 0 = one problem
  // split-K: grid.z CTAs share one output tile; partial tiles go through `ws`, the last CTA to
  // arrive (ticket) sums them in fixed order (deterministic) and runs the epilogue.
  int splits, kb_per_split;
  float* ws;
  unsigned int* tickets;
  // fused GroupNorm statistics of the OUTPUT tensor: per (image, 32-row slot, channel) sum / sum of
  // squares over the warp's rows -> stats[(img * nslots + slot) * N + col][2] (fp32 outputs only)
  float* stats;
  int stats_nslots, stats_rows_per_img, stats_slots_x;
};

__device__ __forceinline__ float apply_act(float v, int act, float prm) {
  if (act == 1) return gelu_erf_f(v);
  if (act == 2) return v > 0.f ? v : v * prm;
  // 3: silu x * sigmoid(x), 4: quick_gelu x * sigmoid(1.702 x) (CLIP MLP); -1.0f * v == -v, so silu is unchanged
  return v / (1.0f + __expf((act == 4 ? -1.702f : -1.0f) * v));
}

__device__ __forceinline__ void sts_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ float4 lds_v4(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}

// Per-warp epilogue state: which 32 rows of the tile, their sub-box origin, staging buffers.
struct EpiCtx {
  const CUtensorMap* tm_out;
  const CUtensorMap* tm_res;
  uint32_t cur;            // shared address of the chunk being finished: its accumulator block, reused as the
                           // output staging tile
  uint32_t res_base;       // this warp's two residual staging tiles
  uint32_t res_bar;        // shared address of this warp's two residual-load mbarriers
  int row0;                // plain mode: first global row of this warp
  int x, y, n;             // conv mode: origin of this warp's sub-box
  long long stats_base;    // element offset of this warp's (image, slot) row in the stats buffer, < 0: none
  int grp_off;             // grouped launch: row offset of this CTA's problem in the stacked bias
  __device__ __forceinline__ uint32_t res_buf(int b) const { return res_base + b * EPI_TILE_BYTES; }
  __device__ __forceinline__ uint32_t bar(int b) const { return res_bar + b * 8; }
};

__device__ __forceinline__ void mbar_wait_s(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  long long t0 = 0;
  while (true) {
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
        : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    if (ok) return;
    if (t0 == 0) t0 = clock64();
    else if (clock64() - t0 > 4000000000LL) __trap();     // no printf: see mbar_wait
  }
}

__device__ __forceinline__ void epi_issue_residual(const GemmParams& p, EpiCtx& e, int lane, int chunk_idx,
                                                   int gc0) {
  // lane 0 only
  if (lane == 0) {
    const int b = chunk_idx & 1;
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(e.bar(b)), "r"(EPI_TILE_BYTES) : "memory");
    if (p.mode == 0) {
      asm volatile(
          "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::
              "r"(e.res_buf(b)), "l"(reinterpret_cast<uint64_t>(e.tm_res)), "r"(e.bar(b)), "r"(gc0), "r"(e.row0)
          : "memory");
    } else {
      asm volatile(
          "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::
              "r"(e.res_buf(b)), "l"(reinterpret_cast<uint64_t>(e.tm_res)), "r"(e.bar(b)), "r"(gc0), "r"(e.x),
          "r"(e.y), "r"(e.n)
          : "memory");
    }
  }
}

// Finishes one 32-column chunk held as fp32 in v[] (thread == row): epilogue math, residual,
// staging, TMA store. `chunk_idx` counts chunks processed by this warp (buffer parity),
// `gc0` is the first *output* column, `next_gc0` (< 0: none) the column of the chunk after next
// whose residual tile can start loading into the buffer this chunk frees.
__device__ __forceinline__ void finish_chunk(const GemmParams& p, EpiCtx& e, float* v, int lane, int chunk_idx,
                                             int gc0, int ncols, int next_gc0, long long out_row, int vec_idx,
                                             bool raw_math, bool have_pre = false, float pre = 0.f) {
  const int b = chunk_idx & 1;
  if (raw_math && have_pre) {
    // bias + row vector of this chunk were fetched while the mainloop ran (lane == column)
#pragma unroll
    for (int j = 0; j < 32; ++j) v[j] += __shfl_sync(0xffffffffu, pre, j);
    if (p.act) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = apply_act(v[j], p.act, p.act_param);
    }
    if (p.alpha != 1.0f) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] *= p.alpha;
    }
  } else if (raw_math) {
    if (p.bias && p.bias_per_row) {
      const float bv = out_row >= 0 ? __ldg(p.bias + out_row) : 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] += bv;
    } else if (p.bias || p.rowvec) {
      // acc + (bias + rowvec): the same association as the prefetched path above, so a sample's bits do not
      // depend on whether its warp's 32 rows share one row vector (tiny images: several images per warp)
      const bool rv_on = p.rowvec && out_row >= 0;
      const float* rv = p.rowvec + static_cast<long long>(vec_idx) * p.N + gc0;
      if (ncols == 32) {
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          float4 t = p.bias ? __ldg(reinterpret_cast<const float4*>(p.bias + e.grp_off + gc0 + j)) : make_float4(0.f, 0.f, 0.f, 0.f);
          if (rv_on) {
            const float4 r = __ldg(reinterpret_cast<const float4*>(rv + j));
            t.x += r.x; t.y += r.y; t.z += r.z; t.w += r.w;
          }
          v[j] += t.x; v[j + 1] += t.y; v[j + 2] += t.z; v[j + 3] += t.w;
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j)
          if (j < ncols) {
            float t = p.bias ? __ldg(p.bias + e.grp_off + gc0 + j) : 0.f;
            if (rv_on) t += __ldg(rv + j);
            v[j] += t;
          }
      }
    }
    if (p.act) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] = apply_act(v[j], p.act, p.act_param);
    }
    if (p.alpha != 1.0f) {
#pragma unroll
      for (int j = 0; j < 32; ++j) v[j] *= p.alpha;
    }
  }
  const int sw = lane & 7;
  if (p.has_residual) {
    mbar_wait_s(e.bar(b), (chunk_idx >> 1) & 1);
    const uint32_t rrow = e.res_buf(b) + lane * 128;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 t = lds_v4(rrow + ((j ^ sw) << 4));
      v[4 * j] += t.x; v[4 * j + 1] += t.y; v[4 * j + 2] += t.z; v[4 * j + 3] += t.w;
    }
    fence_proxy_async_smem();                       // generic reads before the async overwrite
    __syncwarp();                                   // every lane has read the residual tile
    if (next_gc0 >= 0) epi_issue_residual(p, e, lane, chunk_idx + 2, next_gc0);
  }
  __syncwarp();                                   // every lane has read the chunk out of its block
  if (p.out_kind == 0) {
    const uint32_t orow = e.cur + lane * 128;          // 128-byte rows, SWIZZLE_128B
#pragma unroll
    for (int j = 0; j < 8; ++j)
      sts_v4(orow + ((j ^ sw) << 4), __float_as_uint(v[4 * j]), __float_as_uint(v[4 * j + 1]),
             __float_as_uint(v[4 * j + 2]), __float_as_uint(v[4 * j + 3]));
  } else {
    const uint32_t orow = e.cur + lane * 64;           // 64-byte rows, SWIZZLE_64B
    const int sw2 = (lane >> 1) & 3;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      sts_v4(orow + ((j ^ sw2) << 4), pack2(v[8 * j], v[8 * j + 1]), pack2(v[8 * j + 2], v[8 * j + 3]),
             pack2(v[8 * j + 4], v[8 * j + 5]), pack2(v[8 * j + 6], v[8 * j + 7]));
  }
  fence_proxy_async_smem();
  __syncwarp();
  if (p.stats && e.stats_base >= 0 && p.out_kind == 0) {
    // column sums over the warp's valid rows, read back from the staged tile (lane == column)
    const uint32_t valid = __ballot_sync(0xffffffffu, out_row >= 0);
    float sa = 0.f, sb = 0.f;
    const uint32_t col_off = static_cast<uint32_t>(lane & 3) * 4;
    const int chunk = lane >> 2;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      float x;
      asm volatile("ld.shared.f32 %0, [%1];" : "=f"(x) : "r"(e.cur + i * 128 + (((chunk ^ (i & 7))) << 4) + col_off) : "memory");
      if ((valid >> i) & 1u) { sa += x; sb += x * x; }
    }
    if (lane < ncols)
      *reinterpret_cast<float2*>(p.stats + (e.stats_base + gc0 + lane) * 2) = make_float2(sa, sb);
  }
  if (lane == 0) {
    if (p.mode == 0) tma_store_2d(e.tm_out, e.cur, gc0, e.row0);
    else tma_store_4d(e.tm_out, e.cur, gc0, e.x, e.y, e.n);
    bulk_commit();
  }
}

constexpr int EW = 8;                        // epilogue warps == the two consumer warpgroups
constexpr int PRODUCER_WARP = EW;
constexpr int GEMM_THREADS = 32 * EW + 32;
constexpr int CSTEP = 64;                    // two warps per 32-row quarter take alternate 32-column chunks

template <int BN>
__device__ __forceinline__ void wgmma_tile(float* d, uint64_t da, uint64_t db) {
  if constexpr (BN == 32) wgmma_ss_n32(d, da, db);
  else if constexpr (BN == 64) wgmma_ss_n64(d, da, db);
  else if constexpr (BN == 128) wgmma_ss_n128(d, da, db);
  else if constexpr (BN == 160) wgmma_ss_n160(d, da, db);
  else wgmma_ss_n256(d, da, db);
}

// Accumulator block (32-column chunk c, 32-row quarter q): [32 rows][32 fp32], 128-byte rows with the
// 16-byte units XOR-swizzled by (row & 7) -- the layout of the SWIZZLE_128B output / residual boxes.
__device__ __forceinline__ uint32_t acc_block(uint32_t base, int c, int q) {
  return base + static_cast<uint32_t>(c * 4 + q) * EPI_TILE_BYTES;
}
// thread == row `lane` of the block: its 32 values
__device__ __forceinline__ void acc_ld32(uint32_t blk, int lane, float* v) {
  const uint32_t row = blk + lane * 128;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float4 t = lds_v4(row + ((j ^ (lane & 7)) << 4));
    v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
  }
}

template <int BN, int STAGES>
struct GemmSmem {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int PIPE = STAGES * (A_SUB_BYTES + B_STAGE_BYTES);
  static constexpr int EPI = BN * BM * 4 + EW * 2 * EPI_TILE_BYTES;     // accumulator blocks + residual tiles
  static constexpr int DATA = PIPE > EPI ? PIPE : EPI;
  static constexpr int TOTAL = DATA + 1024 + 512;                        // + alignment slack, barriers
};

// PAIR: the two CTAs of a (2,1,1) cluster (adjacent M tiles, same N tile) each load half of the B tile
// and multicast it to both, so B crosses the L2 fabric once per pair; a stage is refilled only after
// the consumers of both CTAs released it.
template <int BN, int STAGES, bool PAIR>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tma_a, const __grid_constant__ CUtensorMap tma_b,
               const __grid_constant__ CUtensorMap tma_out, const __grid_constant__ CUtensorMap tma_res,
               const GemmParams p) {
  using L = GemmSmem<BN, STAGES>;
  constexpr int B_ROWS = PAIR ? BN / 2 : BN;          // B rows loaded by this CTA
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * A_SUB_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::DATA);
  uint64_t* empty = full + STAGES;
  uint64_t* res_bars = empty + STAGES;                // [EW warps][2]
  uint32_t* split_flag = reinterpret_cast<uint32_t*>(res_bars + 2 * EW);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t cta_rank = PAIR ? cluster_ctarank() : 0u;
  const int m_tile = blockIdx.x;
  const int n_tile = blockIdx.y;
  const int tile_lin = blockIdx.y * gridDim.x + blockIdx.x;
  const int kb0 = blockIdx.z * p.kb_per_split;
  const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);

  // tile origin
  int n0 = 0, y0 = 0, x0 = 0;
  if (p.mode == 1) {
    int t = m_tile;
    int tx = t % p.tiles_x; t /= p.tiles_x;
    int ty = t % p.tiles_y; t /= p.tiles_y;
    x0 = tx * p.bw; y0 = ty * p.bh; n0 = t * p.bni;
  }

  // grouped launch: this CTA's problem -> row offset into the stacked weights / bias
  int grp_off = 0;
  if (p.group_span > 0) grp_off = ((p.mode == 1 ? n0 : m_tile) / p.group_span) * p.N;

  if (warp == PRODUCER_WARP && lane == 0) {
    tma_prefetch_desc(&tma_a);
    tma_prefetch_desc(&tma_b);
    tma_prefetch_desc(&tma_out);
    if (p.has_residual) tma_prefetch_desc(&tma_res);
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], PAIR ? 4 : 2); }
    for (int i = 0; i < 2 * EW; ++i) mbar_init(&res_bars[i], 1);
    fence_mbar_init();
  }
  // PAIR: the peer's barriers must be live before any multicast complete_tx or remote arrive
  if constexpr (PAIR) cluster_sync_all();
  else __syncthreads();
  pdl_trigger();        // the next kernel may start its prologue
  pdl_wait();           // A operand / residual come from predecessor kernels

  const int n_iters = kb1 - kb0;
  if (warp == PRODUCER_WARP) {
    // ---------------- TMA producer: warp-uniform loop, one elected lane issues -------------
    const int b_row = grp_off + n_tile * BN + static_cast<int>(cta_rank) * B_ROWS;
    // conv mode: (channel block, tap column, tap row) of the next k-block, advanced incrementally
    // (integer divisions in this loop cost more than the TMA issue itself)
    int cb = 0, tx = 0, ty = 0;
    if (p.mode == 1) {
      const int tap0 = kb0 / p.cblocks;
      cb = kb0 - tap0 * p.cblocks;
      ty = tap0 / p.kw;
      tx = tap0 - ty * p.kw;
    }
    int s = 0;
    uint32_t ph = 0;
    for (int it = 0; it < n_iters; ++it) {
      const int kc = (kb0 + it) * BK;
      // conv: A is addressed by (channel block, tap offset) instead of k
      const int ac = cb * BK, ax = x0 + tx - p.pad, ay = y0 + ty - p.pad;
      if (p.mode == 1 && ++cb == p.cblocks) { cb = 0; if (++tx == p.kw) { tx = 0; ++ty; } }
      mbar_wait(&empty[s], ph ^ 1);
      if (elect_one()) {
        mbar_expect_tx(&full[s], A_SUB_BYTES + L::B_STAGE_BYTES);
        uint8_t* a_dst = sA + s * A_SUB_BYTES;
        uint8_t* b_dst = sB + s * L::B_STAGE_BYTES;
        if (p.mode == 0) tma_load_2d(a_dst, &tma_a, &full[s], kc, m_tile * BM);
        else tma_load_4d(a_dst, &tma_a, &full[s], ac, ax, ay, n0);
        if constexpr (PAIR) tma_load_2d_mc(b_dst + cta_rank * (B_ROWS * BK * 2), &tma_b, &full[s], kc, b_row, 3);
        else tma_load_2d(b_dst, &tma_b, &full[s], kc, b_row);
      }
      __syncwarp();
      if (++s == STAGES) { s = 0; ph ^= 1; }
    }
  } else {
    // ---------------- consumers, then epilogue: warps 0..7, row quarter = warp % 4 -------------
    const int q = warp & 3;
    const int ew = warp;                    // epilogue warp index
    const int c_first = (ew >> 2) * 32;     // warps 4..7 start at column 32
    const int r = q * 32 + lane;            // accumulator row within the tile
    long long out_row = -1;                 // global output row (bias_per_row / rowvec index), -1 = masked
    int vec_idx = 0;
    EpiCtx e;
    e.tm_out = &tma_out; e.tm_res = &tma_res;
    e.grp_off = grp_off;
    e.res_bar = smem_u32(res_bars + ew * 2);
    e.row0 = m_tile * BM + q * 32;
    e.x = e.y = e.n = 0;
    if (p.mode == 0) {
      const long long gr = static_cast<long long>(m_tile) * BM + r;
      if (gr < p.M) { out_row = gr; vec_idx = static_cast<int>(gr) / p.rows_per_vec; }   // 32-bit: gr < M
    } else {
      const int bx = r % p.bw;
      const int by = (r / p.bw) % p.bh;
      const int bn = r / (p.bw * p.bh);
      const int x = x0 + bx, y = y0 + by, n = n0 + bn;
      if (x < p.W && y < p.H && n < p.NI) {
        out_row = (static_cast<long long>(n) * p.H + y) * p.W + x;
        vec_idx = n;
      }
      const int r0 = q * 32;                // this warp's sub-box origin
      e.x = x0 + r0 % p.bw;
      e.y = y0 + (r0 / p.bw) % p.bh;
      e.n = n0 + r0 / (p.bw * p.bh);
    }
    // Per-column addends (bias + the row vector of this warp's image) of every chunk this warp will
    // finish, fetched now so that their L2 latency hides behind the mainloop: lane == column, one
    // register per chunk. Needs one row vector for the whole warp (images of >= 32 rows).
    constexpr int MAX_PRE = BN / CSTEP + 1;
    float pre[MAX_PRE];
    bool have_pre = false;
    if (!p.geglu && !p.bias_per_row && (p.bias || p.rowvec)) {
      const bool any_row = __any_sync(0xffffffffu, out_row >= 0);
      // masked lanes of lane 0 would make v0 meaningless: take the vector of the first valid row
      const unsigned vm = __ballot_sync(0xffffffffu, out_row >= 0);
      const int vsel = any_row ? __shfl_sync(0xffffffffu, vec_idx, __ffs(vm) - 1) : 0;
      const bool uniform = !p.rowvec || !any_row || __all_sync(0xffffffffu, out_row < 0 || vec_idx == vsel);
      if (uniform) {
        have_pre = true;
#pragma unroll
        for (int i = 0; i < MAX_PRE; ++i) {
          const int col = n_tile * BN + c_first + i * CSTEP + lane;
          float x = 0.f;
          if (c_first + i * CSTEP < BN && col < p.N) {
            if (p.bias) x = __ldg(p.bias + grp_off + col);
            if (p.rowvec && any_row) x += __ldg(p.rowvec + static_cast<long long>(vsel) * p.N + col);
          }
          pre[i] = x;
        }
      }
    }
    // GEGLU: value / gate biases of every chunk this warp finishes (lane == column), fetched while the
    // mainloop runs and broadcast through shared memory later
    constexpr int MAX_G = (BN / 2) / CSTEP + 1;
    float pa[MAX_G], pg[MAX_G];
    if (p.geglu) {
#pragma unroll
      for (int i = 0; i < MAX_G; ++i) {
        const int c = c_first + i * CSTEP + lane;
        const bool live = p.bias && c_first + i * CSTEP < BN / 2 && n_tile * (BN / 2) + c < p.N / 2;
        pa[i] = live ? __ldg(p.bias + grp_off + n_tile * BN + c) : 0.f;
        pg[i] = live ? __ldg(p.bias + grp_off + n_tile * BN + BN / 2 + c) : 0.f;
      }
    }

    // ---------------- mainloop: this warpgroup's 64 rows x BN, one 64-wide k-block per stage ----------
    const int wg = warp >> 2;
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    {
      const uint64_t a_desc0 = wgmma_desc_sw128(smem_u32(sA)) + static_cast<uint64_t>((wg * 64 * 128) >> 4);
      const uint64_t b_desc0 = wgmma_desc_sw128(smem_u32(sB));
      const uint32_t peer_empty = PAIR ? mapa_u32(smem_u32(&empty[0]), cta_rank ^ 1u) : 0u;
      const bool signal = (threadIdx.x & 127) == 0;       // one arrival per warpgroup
      auto release = [&](int st) {
        if (signal) {
          mbar_arrive(&empty[st]);
          if constexpr (PAIR) mbar_arrive_cluster(peer_empty + st * 8);
        }
      };
      int s = 0, prev = -1;
      uint32_t ph = 0;
      for (int it = 0; it < n_iters; ++it) {
        mbar_wait(&full[s], ph);
        wgmma_fence();
        const uint64_t da = a_desc0 + static_cast<uint64_t>((s * A_SUB_BYTES) >> 4);
        const uint64_t db = b_desc0 + static_cast<uint64_t>((s * L::B_STAGE_BYTES) >> 4);
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) wgmma_tile<BN>(acc, da + 2 * k, db + 2 * k);
        wgmma_commit();
        wgmma_wait<1>();                    // the previous stage's MMAs have retired: hand it back
        if (prev >= 0) release(prev);
        prev = s;
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_reg_fence(acc, BN / 2);
      if (prev >= 0) release(prev);
    }
    // every MMA of both warpgroups has retired -> the stage memory is free: accumulators -> blocks
    asm volatile("bar.sync 1, %0;" ::"n"(32 * EW) : "memory");
    const uint32_t acc_base = smem_u32(smem);
    {
      const int rw = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // first of this thread's two rows
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = rw + 8 * h, rr = row & 31;
          const uint32_t addr = acc_block(acc_base, col >> 5, row >> 5) + rr * 128 +
                                ((((col & 31) >> 2) ^ (rr & 7)) << 4) + (col & 3) * 4;
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(acc[4 * j + 2 * h]),
                       "f"(acc[4 * j + 2 * h + 1]) : "memory");
        }
      }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(32 * EW) : "memory");
    e.res_base = acc_base + BN * BM * 4 + ew * (2 * EPI_TILE_BYTES);
    // GroupNorm-statistics row of this warp, computed only now: the epilogue is its first reader, and the wide
    // tiles sit at the 168-register limit, where a 64-bit value held across the mainloop makes ptxas spill
    e.stats_base = -1;
    if (p.stats) {
      if (p.mode == 0) {
        const int img = e.row0 / p.stats_rows_per_img, slot = (e.row0 % p.stats_rows_per_img) / 32;
        if (e.row0 < p.M) e.stats_base = (static_cast<long long>(img) * p.stats_nslots + slot) * p.N;
      } else if (e.x < p.W && e.y < p.H && e.n < p.NI) {
        const int slot = (e.y / p.wbh) * p.stats_slots_x + e.x / p.wbw;
        e.stats_base = (static_cast<long long>(e.n) * p.stats_nslots + slot) * p.N;
      }
    }

    constexpr int OUT_COLS = BN;            // accumulator columns that produce output (GEGLU: BN/2)
    const bool finalize = p.splits == 1;
    if (!p.geglu) {
      const int col_base = n_tile * BN;
      // prefetch the first two residual tiles
      if (finalize && p.has_residual) {
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int cc = c_first + c * CSTEP;
          if (cc < OUT_COLS && col_base + cc < p.N) epi_issue_residual(p, e, lane, c, col_base + cc);
        }
      }
      int ci = 0;
#pragma unroll 1
      for (int c0 = c_first; c0 < BN; c0 += CSTEP) {
        float v[32];
        e.cur = acc_block(acc_base, c0 >> 5, q);
        __syncwarp();
        acc_ld32(e.cur, lane, v);
        const int gc0 = col_base + c0;
        if (p.splits > 1) {
          // raw partial -> workspace [tile][split][col][row]: coalesced across the warp's rows
          float* wcol = p.ws + ((static_cast<long long>(tile_lin) * p.splits + blockIdx.z) * BN + c0) * BM + r;
#pragma unroll
          for (int j = 0; j < 32; ++j) __stcg(wcol + j * BM, v[j]);
          continue;
        }
        if (gc0 >= p.N) continue;
        const int ncols = min(32, p.N - gc0);
        const int ngc = gc0 + 2 * CSTEP;
        finish_chunk(p, e, v, lane, ci, gc0, ncols, (c0 + 2 * CSTEP < BN && ngc < p.N) ? ngc : -1, out_row, vec_idx, true,
                     have_pre, pre[(c0 - c_first) / CSTEP]);
        ++ci;
      }
      if (p.splits > 1) {
        __threadfence();
        asm volatile("bar.sync 1, %0;" ::"n"(32 * EW) : "memory");
        if (threadIdx.x == 0) {
          const unsigned int t = atomicAdd(&p.tickets[tile_lin], 1u);
          const bool last = (t == static_cast<unsigned int>(p.splits) - 1);
          if (last) p.tickets[tile_lin] = 0;        // self-reset for the next launch
          *split_flag = last ? 1u : 0u;
        }
        asm volatile("bar.sync 1, %0;" ::"n"(32 * EW) : "memory");
        if (*split_flag) {
          __threadfence();
          if (p.has_residual) {
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int cc = c_first + c * CSTEP;
              if (cc < BN && col_base + cc < p.N) epi_issue_residual(p, e, lane, c, col_base + cc);
            }
          }
          int cj = 0;
#pragma unroll 1
          for (int c0 = c_first; c0 < BN; c0 += CSTEP) {
            const int gc0 = col_base + c0;
            if (gc0 >= p.N) continue;
            const int ncols = min(32, p.N - gc0);
            const int ngc = gc0 + 2 * CSTEP;
            float v[32];
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = 0.f;
            for (int z = 0; z < p.splits; ++z) {     // fixed summation order
              const float* wcol = p.ws + ((static_cast<long long>(tile_lin) * p.splits + z) * BN + c0) * BM + r;
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] += __ldcg(wcol + j * BM);
            }
            e.cur = acc_block(acc_base, c0 >> 5, q);
            finish_chunk(p, e, v, lane, cj, gc0, ncols, (c0 + 2 * CSTEP < BN && ngc < p.N) ? ngc : -1, out_row, vec_idx, true,
                         have_pre, pre[(c0 - c_first) / CSTEP]);
            ++cj;
          }
        }
      }
    } else {
      // GEGLU: tile columns [0, BN/2) are values, [BN/2, BN) the matching gates
      // (weights are packed that way); output column = n_tile*BN/2 + c.
      constexpr int HB = BN / 2;
      const int n_half = p.N / 2;
      if constexpr (HB % 32 == 0) {
        // Value / gate biases of this warp's chunks go through its (unused: GEGLU has no residual) residual
        // staging tile and come back as broadcast LDS.128: 16 loads per chunk instead of 64 shuffles.
        const uint32_t bb = e.res_buf(0);
#pragma unroll
        for (int i = 0; i < MAX_G; ++i) {
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(bb + (i * 64 + lane) * 4), "f"(pa[i]) : "memory");
          asm volatile("st.shared.f32 [%0], %1;" ::"r"(bb + (i * 64 + 32 + lane) * 4), "f"(pg[i]) : "memory");
        }
        __syncwarp();
        // one chunk of values * act(gates); false once the chunks of this warp are done. SWIGLU (geglu = 2) runs
        // as a rolled loop so that the GEGLU path keeps its code unchanged.
        auto chunk = [&](int i, int& ci, auto swiglu) -> bool {
          const int c0 = c_first + i * CSTEP;
          if (c0 >= HB) return false;
          float av[32], ag[32];
          e.cur = acc_block(acc_base, c0 >> 5, q);
          __syncwarp();
          acc_ld32(e.cur, lane, av);
          acc_ld32(acc_block(acc_base, (HB + c0) >> 5, q), lane, ag);
          const int gc0 = n_tile * HB + c0;   // output column
          if (gc0 >= n_half) return true;
          const int ncols = min(32, n_half - gc0);
          float v[32];
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            const float4 ba = lds_v4(bb + i * 256 + jj * 16), bg = lds_v4(bb + i * 256 + 128 + jj * 16);
            float a0, a1, a2, a3, g0, g1, g2, g3, y0, y1, y2, y3;
            fadd2(a0, a1, av[4 * jj], av[4 * jj + 1], ba.x, ba.y);
            fadd2(a2, a3, av[4 * jj + 2], av[4 * jj + 3], ba.z, ba.w);
            fadd2(g0, g1, ag[4 * jj], ag[4 * jj + 1], bg.x, bg.y);
            fadd2(g2, g3, ag[4 * jj + 2], ag[4 * jj + 3], bg.z, bg.w);
            if constexpr (decltype(swiglu)::value) {
              y0 = silu_f(g0); y1 = silu_f(g1); y2 = silu_f(g2); y3 = silu_f(g3);
            } else {
              gelu_erf_f2(g0, g1, y0, y1);
              gelu_erf_f2(g2, g3, y2, y3);
            }
            fmul2(v[4 * jj], v[4 * jj + 1], a0, a1, y0, y1);
            fmul2(v[4 * jj + 2], v[4 * jj + 3], a2, a3, y2, y3);
          }
          finish_chunk(p, e, v, lane, ci, gc0, ncols, -1, out_row, vec_idx, false);
          ++ci;
          return true;
        };
        int ci = 0;
        if (p.geglu == 2) {
#pragma unroll 1
          for (int i = 0; i < MAX_G; ++i)
            if (!chunk(i, ci, std::true_type{})) break;
        } else {
#pragma unroll
          for (int i = 0; i < MAX_G; ++i)
            if (!chunk(i, ci, std::false_type{})) break;
        }
      }
    }
    if (lane == 0) bulk_wait_read<0>();     // staging tiles must outlive the bulk stores' reads
    __syncwarp();
  }
  if constexpr (PAIR) cluster_sync_all();     // neither CTA may retire while the other can still signal it
}

template <int BN, int STAGES, bool PAIR>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& to, const CUtensorMap& tr,
           const GemmParams& p, dim3 grid, cudaStream_t st) {
  constexpr int smem = GemmSmem<BN, STAGES>::TOTAL;
  static_assert(smem <= 227 * 1024, "pipeline does not fit in shared memory");
  static_assert((2 * STAGES + 2 * EW) * 8 + 8 <= 512, "barriers do not fit");
  static bool configured = false;
  if (!configured) {
    DBIR_CHECK_CUDA(cudaFuncSetAttribute(gemm_tc_kernel<BN, STAGES, PAIR>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    configured = true;
  }
  DBIR_CHECK_CUDA(dbir_launch_cluster(gemm_tc_kernel<BN, STAGES, PAIR>, grid, dim3(GEMM_THREADS), smem, st,
                                      PAIR ? 2u : 1u, ta, tb, to, tr, p));
  return 0;
}

// Tile width, CTA pairing and split-K factor from a cost model in SM cycles. Every kernel of the
// family runs one CTA per SM (two warpgroups of register accumulators and a ~200 KB stage ring):
//   * one 64-wide k-block costs max(MMA time, pipeline overhead): 128 x BN x 64 MACs at the dense
//     16-bit rate of 2048 MACs per cycle per SM take 4*BN cycles; a stage round trip (barrier wait,
//     wgmma issue, release) ~200 cycles;
//   * a CTA pair loads half of B per CTA (multicast): less L2 traffic per k-block, more set-up;
//   * epilogue ~1200 + 24*BN cycles; split-K adds a workspace round trip; CTAs are spread over `sms`
//     SMs, a partial last wave costs a full one.
// The first call of each problem signature replaces this estimate with a measurement (see below).
struct TilePlan { int bn, splits, kb_per_split, pair; };

struct PlanQuery {
  int m_tiles, N, num_kb, geglu, forced_bn, split_req, pair_req;
  long long ws_floats_avail;
};

// Calls f(plan, modelled cost) for every plan the kernel family can run for this problem.
template <typename F>
void for_each_plan(const PlanQuery& q, F f) {
  const int cands[5] = {256, 160, 128, 64, 32};
  const int sms = dbir_sm_count();
  // CTA pairs (2-CTA clusters sharing B): 0 never, 1 whenever the shape allows, -1 free choice
  const int pair_mode = q.pair_req == 1 ? 1 : q.pair_req == 2 ? 0 : -1;
  const bool can_pair = pair_mode != 0 && !(q.m_tiles & 1);
  for (int i = 0; i < 10; ++i) {
    const int bn = cands[i % 5];
    const int pair = 1 - i / 5;
    if (pair && (!can_pair || bn < 64)) continue;
    if (!pair && pair_mode == 1 && can_pair && bn >= 64) continue;     // forced pairing
    if (q.forced_bn > 0 && bn != q.forced_bn) continue;
    if (q.forced_bn <= 0) {
      if (q.geglu && bn < 64) continue;
      if (bn > 64 && q.N % bn != 0) continue;                          // ragged N only with the narrow tiles
    }
    const long long tiles = static_cast<long long>(q.m_tiles) * ((q.N + bn - 1) / bn);
    for (int s = 1; s <= 16; ++s) {
      if (s > 1) {
        if (q.split_req == 1 || q.geglu || q.ws_floats_avail <= 0) break;
        if (q.num_kb / s < 6) break;
        if (tiles > 16384 || tiles * s * 128LL * bn > q.ws_floats_avail) break;
        if (tiles * (s - 1) >= 2LL * sms) break;       // already two waves without it
      }
      if (q.split_req > 1 && s != q.split_req) continue;
      const int kbs = (q.num_kb + s - 1) / s;
      if (static_cast<long long>(kbs) * (s - 1) >= q.num_kb) continue;   // an empty split
      const long long ctas = tiles * s;
      const double waves = static_cast<double>((ctas + sms - 1) / sms);
      const double mma = 4.0 * bn;
      const double ovh = pair ? 180.0 : 200.0;
      const double main = kbs * (ovh > mma ? ovh : mma) * (pair ? 0.97 : 1.0);
      double epi = 1200.0 + 24.0 * bn;
      if (s > 1) epi += 30.0 * bn + 6.0 * bn * s;
      f(TilePlan{bn, s, kbs, pair}, waves * (2500.0 + (pair ? 900.0 : 0.0) + main + epi));
    }
  }
}

TilePlan pick_plan(const PlanQuery& q) {
  TilePlan best{64, 1, q.num_kb, 0};
  double best_cost = -1.0;
  for_each_plan(q, [&](const TilePlan& t, double cost) {
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = t; }
  });
  return best;
}

// ---- plan cache + on-device autotuning ---------------------------------------------------------
// The first dbir_gemm call for a problem signature outside stream capture times every plan the model
// rates within 3x of its best (cold L2: the real layers stream their weights from HBM) on the
// caller's own operands, with the outputs redirected to scratch, and caches the winner. Split-K
// factors change the fp32 summation order, so results can differ at rounding level between
// processes; DBIR_GEMM_AUTOTUNE=0 keeps the deterministic model choice.
using PlanKey = std::array<long long, 20>;
std::mutex g_plan_mu;                     // guards the cache
std::mutex g_tune_mu;                     // serialises tuning (shared scratch / events, meaningful timings)
std::map<PlanKey, TilePlan> g_plan_cache;

bool autotune_enabled() {
  static const int on = [] { const char* e = getenv("DBIR_GEMM_AUTOTUNE"); return e ? atoi(e) : 1; }();
  return on != 0;
}

PlanKey make_key(const dbir_gemm_args* a) {
  PlanKey k{};
  int i = 0;
  k[i++] = a->M; k[i++] = a->N; k[i++] = a->K; k[i++] = a->a_mode;
  k[i++] = a->img_n; k[i++] = a->img_h; k[i++] = a->img_w; k[i++] = a->img_c; k[i++] = a->ksize;
  k[i++] = a->out_kind; k[i++] = a->geglu; k[i++] = a->force_bn; k[i++] = a->split_k; k[i++] = a->cta_pair;
  k[i++] = a->residual != nullptr; k[i++] = a->gn_partials != nullptr;
  k[i++] = a->splitk_ws ? a->splitk_ws_bytes : 0;
  k[i++] = a->lda; k[i++] = a->ldo; k[i++] = a->act * 8 + (a->groups > 1 ? a->groups : 1);
  return k;
}

int gemm_impl(const dbir_gemm_args* a, cudaStream_t st, const TilePlan* forced);

struct TuneScratch {
  void* out = nullptr; size_t out_cap = 0;
  void* part = nullptr; size_t part_cap = 0;
  void* flush = nullptr;
  static constexpr size_t FLUSH_BYTES = 128u << 20;     // > 2.5x the 50 MB L2
  cudaEvent_t ev[3][2] = {};
  bool ready = false;
};
TuneScratch g_ts;

bool tune_reserve(void** ptr, size_t* cap, size_t need) {
  if (need <= *cap) return true;
  if (*ptr) cudaFree(*ptr);
  *ptr = nullptr; *cap = 0;
  if (cudaMalloc(ptr, need) != cudaSuccess) { cudaGetLastError(); return false; }
  *cap = need;
  return true;
}

// Returns true and the fastest measured plan, or false if tuning could not run (keeps the model's plan).
bool tune_plan(const dbir_gemm_args* a, cudaStream_t st, const PlanQuery& q, TilePlan* out_plan) {
  TuneScratch& ts = g_ts;
  if (!ts.ready) {
    if (cudaMalloc(&ts.flush, TuneScratch::FLUSH_BYTES) != cudaSuccess) { cudaGetLastError(); return false; }
    for (auto& e : ts.ev) for (auto& x : e) if (cudaEventCreate(&x) != cudaSuccess) return false;
    ts.ready = true;
  }
  const int eb = a->out_kind == 0 ? 4 : 2;
  const size_t out_bytes = static_cast<size_t>(a->M) * a->ldo * eb;
  if (!tune_reserve(&ts.out, &ts.out_cap, out_bytes)) return false;
  dbir_gemm_args t = *a;
  t.out = ts.out;
  if (a->gn_partials) {
    const long long imgs = a->a_mode == 1 ? a->img_n : a->M / a->gn_rows_per_img;
    const long long slots = a->a_mode == 1 ? dbir_gemm_gn_slots(a->img_h, a->img_w, 0)
                                           : dbir_gemm_gn_slots(0, 0, a->gn_rows_per_img);
    if (slots <= 0 || !tune_reserve(&ts.part, &ts.part_cap, static_cast<size_t>(imgs) * slots * a->N * 8)) return false;
    t.gn_partials = ts.part;
  }
  std::vector<std::pair<double, TilePlan>> cands;
  double best_model = -1.0;
  for_each_plan(q, [&](const TilePlan& p, double c) {
    cands.emplace_back(c, p);
    if (best_model < 0 || c < best_model) best_model = c;
  });
  float best_ms = -1.f;
  for (const auto& c : cands) {
    if (c.first > 3.0 * best_model) continue;
    if (gemm_impl(&t, st, &c.second) != 0) continue;              // warm-up (also validates the plan)
    bool ok = true;
    for (int r = 0; r < 3 && ok; ++r) {
      ok = cudaMemsetAsync(ts.flush, r, TuneScratch::FLUSH_BYTES, st) == cudaSuccess &&
           cudaEventRecord(ts.ev[r][0], st) == cudaSuccess && gemm_impl(&t, st, &c.second) == 0 &&
           cudaEventRecord(ts.ev[r][1], st) == cudaSuccess;
    }
    if (!ok || cudaEventSynchronize(ts.ev[2][1]) != cudaSuccess) { cudaGetLastError(); continue; }
    float ms = -1.f;
    for (int r = 0; r < 3; ++r) {
      float x = 0.f;
      if (cudaEventElapsedTime(&x, ts.ev[r][0], ts.ev[r][1]) == cudaSuccess && (ms < 0 || x < ms)) ms = x;
    }
    if (ms > 0 && (best_ms < 0 || ms < best_ms)) { best_ms = ms; *out_plan = c.second; }
  }
  return best_ms > 0;
}

TilePlan choose_plan(const dbir_gemm_args* a, cudaStream_t st, const PlanQuery& q) {
  if (!autotune_enabled()) return pick_plan(q);
  const PlanKey key = make_key(a);
  {
    std::lock_guard<std::mutex> lk(g_plan_mu);
    auto it = g_plan_cache.find(key);
    if (it != g_plan_cache.end()) return it->second;
  }
  TilePlan plan = pick_plan(q);
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) { cudaGetLastError(); return plan; }
  if (cs != cudaStreamCaptureStatusNone) return plan;       // cannot time inside a capture: model plan, not cached
  std::lock_guard<std::mutex> tune_lk(g_tune_mu);
  {
    std::lock_guard<std::mutex> lk(g_plan_mu);          // another thread may have tuned it meanwhile
    auto it = g_plan_cache.find(key);
    if (it != g_plan_cache.end()) return it->second;
  }
  TilePlan tuned = plan;
  if (tune_plan(a, st, q, &tuned)) plan = tuned;
  std::lock_guard<std::mutex> lk(g_plan_mu);
  g_plan_cache[key] = plan;
  return plan;
}

}  // namespace

extern "C" int dbir_gemm(const dbir_gemm_args* a, void* stream) {
  return gemm_impl(a, reinterpret_cast<cudaStream_t>(stream), nullptr);
}
/* The analytic model's plan for a tile grid (host only, no launch): out[0..3] = BN, splits, k-blocks per
 * split, CTA pair flag. Lets the CPU test suite check the planner's invariants. */
extern "C" int dbir_gemm_model_plan(int32_t m_tiles, int32_t N, int32_t num_kb, int32_t geglu, int32_t force_bn,
                                    int32_t split_k, int32_t cta_pair, int64_t ws_floats, int32_t* out) {
  DBIR_REQUIRE(m_tiles > 0 && N > 0 && num_kb > 0 && out, "dbir_gemm_model_plan: bad arguments");
  const TilePlan t = pick_plan(PlanQuery{m_tiles, N, num_kb, geglu, force_bn, split_k, cta_pair, ws_floats});
  out[0] = t.bn; out[1] = t.splits; out[2] = t.kb_per_split; out[3] = t.pair;
  return 0;
}

namespace {
int gemm_impl(const dbir_gemm_args* a, cudaStream_t st, const TilePlan* forced) {
  DBIR_REQUIRE(a != nullptr, "dbir_gemm: null args");
  DBIR_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0, "dbir_gemm: bad shape M=%d N=%d K=%d", a->M,
               a->N, a->K);
  DBIR_REQUIRE(a->a && a->b && a->out, "dbir_gemm: null pointer");
  DBIR_REQUIRE(a->K % 8 == 0, "dbir_gemm: K=%d must be a multiple of 8 (16-byte rows)", a->K);
  const int eb = a->out_kind == 0 ? 4 : 2;
  DBIR_REQUIRE((a->ldo * eb) % 16 == 0, "dbir_gemm: output row stride must be a multiple of 16 bytes (ldo=%lld)",
               (long long)a->ldo);
  DBIR_REQUIRE(!a->residual || a->ldr % 4 == 0, "dbir_gemm: residual row stride must be a multiple of 4");

  GemmParams p{};
  p.M = a->M; p.N = a->N;
  p.mode = a->a_mode;
  p.out_kind = a->out_kind;
  p.bias = a->bias; p.rowvec = a->rowvec;
  p.rows_per_vec = a->rows_per_vec > 0 ? a->rows_per_vec : a->M;
  p.has_residual = a->residual != nullptr;
  p.alpha = a->alpha; p.act = a->act; p.act_param = a->act_param; p.geglu = a->geglu;
  p.bias_per_row = a->bias_per_row;
  const int groups = a->groups > 1 ? a->groups : 1;
  if (groups > 1) {
    DBIR_REQUIRE(!a->bias_per_row, "dbir_gemm: groups and bias_per_row are exclusive");
    DBIR_REQUIRE(a->N % 4 == 0, "dbir_gemm: grouped launches need N %% 4 == 0 (stacked bias alignment)");
    if (a->a_mode == 0)
      DBIR_REQUIRE(a->M % groups == 0 && (a->M / groups) % BM == 0,
                   "dbir_gemm: grouped launch needs M/groups (= %d) to be a multiple of %d rows", a->M / groups, BM);
    else
      DBIR_REQUIRE(a->img_n % groups == 0, "dbir_gemm: grouped conv needs img_n %% groups == 0");
  }
  if (a->geglu)
    DBIR_REQUIRE(a->force_bn >= 64 && a->force_bn != 160 && a->N % a->force_bn == 0 && !a->residual,
                 "dbir_gemm: GEGLU needs force_bn in {64,128,256} dividing N (weights are packed per tile)");
  const int n_out = a->geglu ? a->N / 2 : a->N;

  CUtensorMap ta, tb, to, tr;
  int m_tiles;
  if (a->a_mode == 0) {
    const long long lda = a->lda > 0 ? a->lda : a->K;
    DBIR_REQUIRE(lda % 8 == 0, "dbir_gemm: lda must be a multiple of 8");
    uint64_t dims[2] = {static_cast<uint64_t>(a->K), static_cast<uint64_t>(a->M)};
    uint64_t strides[1] = {static_cast<uint64_t>(lda) * 2};
    uint32_t box[2] = {BK, BM};
    if (dbir_make_tmap(&ta, a->a, 2, dims, strides, box, 2, 1)) return -3;
    p.num_kb = (a->K + BK - 1) / BK;
    m_tiles = (a->M + BM - 1) / BM;
    if (groups > 1) p.group_span = (a->M / groups) / BM;
    // output / residual: 32 x 32 element boxes per epilogue warp
    uint64_t odims[2] = {static_cast<uint64_t>(n_out), static_cast<uint64_t>(a->M)};
    uint64_t ostr[1] = {static_cast<uint64_t>(a->ldo) * eb};
    uint32_t obox[2] = {32, 32};
    if (dbir_make_tmap(&to, a->out, 2, odims, ostr, obox, eb, eb == 4 ? 1 : 2)) return -3;
    tr = to;
    if (a->residual) {
      uint64_t rstr[1] = {static_cast<uint64_t>(a->ldr) * 4};
      if (dbir_make_tmap(&tr, a->residual, 2, odims, rstr, obox, 4, 1)) return -3;
    }
  } else {
    const int C = a->img_c, H = a->img_h, W = a->img_w, NI = a->img_n;
    const int taps = a->ksize * a->ksize;
    DBIR_REQUIRE(a->ksize == 3 || a->ksize == 1, "dbir_gemm: ksize must be 1 or 3");
    DBIR_REQUIRE(C % BK == 0, "dbir_gemm: conv channels C=%d must be a multiple of 64", C);
    DBIR_REQUIRE(a->K == taps * C, "dbir_gemm: K=%d != taps*C=%d", a->K, taps * C);
    DBIR_REQUIRE(static_cast<long long>(NI) * H * W == a->M, "dbir_gemm: M != N*H*W");
    int bw = 1;
    while (bw < W && bw < 128) bw <<= 1;
    int bh = 1;
    while (bh < H && bw * bh < 128) bh <<= 1;
    int bni = 128 / (bw * bh);
    p.H = H; p.W = W; p.NI = NI;
    p.bw = bw; p.bh = bh; p.bni = bni;
    p.tiles_x = (W + bw - 1) / bw;
    p.tiles_y = (H + bh - 1) / bh;
    p.cblocks = C / BK;
    p.kw = a->ksize; p.pad = a->ksize / 2;
    uint64_t dims[4] = {static_cast<uint64_t>(C), static_cast<uint64_t>(W),
                        static_cast<uint64_t>(H), static_cast<uint64_t>(NI)};
    // lda > 0: the pixels of `a` are lda elements apart and the conv reads their first C channels (dense
    // concat buffers: RRDBNet's cat((x, x1, ..)) lives in one [pixels, nf + 4 gc] tensor, bsrnet.py:51-56)
    const uint64_t ps = static_cast<uint64_t>(a->lda > 0 ? a->lda : C);
    DBIR_REQUIRE(ps >= static_cast<uint64_t>(C) && ps % 8 == 0, "dbir_gemm: conv pixel stride lda=%lld must be >= C and a multiple of 8",
                 (long long)a->lda);
    uint64_t strides[3] = {ps * 2, static_cast<uint64_t>(W) * ps * 2, static_cast<uint64_t>(H) * W * ps * 2};
    uint32_t box[4] = {BK, static_cast<uint32_t>(bw), static_cast<uint32_t>(bh),
                       static_cast<uint32_t>(bni)};
    if (dbir_make_tmap(&ta, a->a, 4, dims, strides, box, 2, 1)) return -3;
    p.num_kb = taps * p.cblocks;
    m_tiles = p.tiles_x * p.tiles_y * ((NI + bni - 1) / bni);
    if (groups > 1) {
      DBIR_REQUIRE((NI / groups) % bni == 0, "dbir_gemm: grouped conv: a %d-image tile would straddle two groups", bni);
      p.group_span = NI / groups;
    }
    // per-warp sub-box of 32 pixels: (wbw x wbh x wbn)
    const int wbw = bw < 32 ? bw : 32;
    const int wbh = bh < 32 / wbw ? bh : 32 / wbw;
    const int wbn = 32 / (wbw * wbh);
    p.wbw = wbw; p.wbh = wbh;
    uint64_t odims[4] = {static_cast<uint64_t>(n_out), static_cast<uint64_t>(W), static_cast<uint64_t>(H),
                         static_cast<uint64_t>(NI)};
    uint64_t ostr[3] = {static_cast<uint64_t>(a->ldo) * eb, static_cast<uint64_t>(W) * a->ldo * eb,
                        static_cast<uint64_t>(H) * W * a->ldo * eb};
    uint32_t obox[4] = {32, static_cast<uint32_t>(wbw), static_cast<uint32_t>(wbh), static_cast<uint32_t>(wbn)};
    if (dbir_make_tmap(&to, a->out, 4, odims, ostr, obox, eb, eb == 4 ? 1 : 2)) return -3;
    tr = to;
    if (a->residual) {
      uint64_t rstr[3] = {static_cast<uint64_t>(a->ldr) * 4, static_cast<uint64_t>(W) * a->ldr * 4,
                          static_cast<uint64_t>(H) * W * a->ldr * 4};
      if (dbir_make_tmap(&tr, a->residual, 4, odims, rstr, obox, 4, 1)) return -3;
    }
  }

  if (a->gn_partials) {
    DBIR_REQUIRE(a->out_kind == 0 && !a->geglu, "dbir_gemm: gn_partials needs an fp32, non-GEGLU output");
    p.stats = reinterpret_cast<float*>(a->gn_partials);
    if (a->a_mode == 0) {
      DBIR_REQUIRE(a->gn_rows_per_img > 0 && a->gn_rows_per_img % 32 == 0 && a->M % a->gn_rows_per_img == 0,
                   "dbir_gemm: gn_partials in matrix mode needs rows-per-image that is a multiple of 32");
      p.stats_rows_per_img = a->gn_rows_per_img;
      p.stats_nslots = a->gn_rows_per_img / 32;
    } else {
      DBIR_REQUIRE(p.bw * p.bh >= 32, "dbir_gemm: gn_partials needs images of at least 32 pixels");
      p.stats_slots_x = (p.W + p.wbw - 1) / p.wbw;
      p.stats_nslots = p.stats_slots_x * ((p.H + p.wbh - 1) / p.wbh);
    }
  }
  constexpr long long TICKET_FLOATS = 16384;
  const long long ws_floats = a->splitk_ws ? a->splitk_ws_bytes / 4 - TICKET_FLOATS : 0;
  // CTA pairs share one weight tile between two adjacent m-tiles: in a grouped launch a pair must not
  // straddle two problems
  int pair_req = a->cta_pair;
  if (groups > 1 && ((m_tiles / groups) & 1)) pair_req = 2;
  const PlanQuery pq{m_tiles, a->N, p.num_kb, a->geglu, a->force_bn, a->split_k, pair_req, ws_floats};
  const TilePlan plan = forced ? *forced : choose_plan(a, st, pq);
  const int bn = plan.bn;
  p.splits = plan.splits;
  p.kb_per_split = plan.kb_per_split;
  if (plan.splits > 1) {
    p.tickets = reinterpret_cast<unsigned int*>(a->splitk_ws);
    p.ws = reinterpret_cast<float*>(a->splitk_ws) + TICKET_FLOATS;
  }
  {
    const long long ldb = a->ldb > 0 ? a->ldb : a->K;
    uint64_t dims[2] = {static_cast<uint64_t>(a->K), static_cast<uint64_t>(a->N) * groups};
    uint64_t strides[1] = {static_cast<uint64_t>(ldb) * 2};
    uint32_t box[2] = {BK, static_cast<uint32_t>(plan.pair ? bn / 2 : bn)};
    if (dbir_make_tmap(&tb, a->b, 2, dims, strides, box, 2, 1)) return -3;
  }
  dim3 grid(m_tiles, (a->N + bn - 1) / bn, plan.splits);
  // <BN, STAGES, PAIR>: stage rings of 160-224 KB, one CTA per SM
#define DBIR_GO(BN_, ST_) return plan.pair ? launch<BN_, ST_, true>(ta, tb, to, tr, p, grid, st) \
                                           : launch<BN_, ST_, false>(ta, tb, to, tr, p, grid, st)
  switch (bn) {
    case 32:  if (plan.pair) break; return launch<32, 8, false>(ta, tb, to, tr, p, grid, st);
    case 64:  DBIR_GO(64, 8);
    case 128: DBIR_GO(128, 6);
    case 160: DBIR_GO(160, 6);
    case 256: DBIR_GO(256, 4);
    default: break;
  }
#undef DBIR_GO
  dbir_set_error("dbir_gemm: unsupported tile width %d (pair %d)", bn, plan.pair);
  return -2;
}
}  // namespace

extern "C" int32_t dbir_gemm_gn_slots(int32_t conv_h, int32_t conv_w, int32_t rows_per_img) {
  if (conv_h > 0 && conv_w > 0) {
    int bw = 1;
    while (bw < conv_w && bw < 128) bw <<= 1;
    int bh = 1;
    while (bh < conv_h && bw * bh < 128) bh <<= 1;
    const int wbw = bw < 32 ? bw : 32;
    const int wbh = bh < 32 / wbw ? bh : 32 / wbw;
    if (wbw * wbh < 32) return -1;
    return ((conv_w + wbw - 1) / wbw) * ((conv_h + wbh - 1) / wbh);
  }
  return rows_per_img > 0 && rows_per_img % 32 == 0 ? rows_per_img / 32 : -1;
}
