// Flash attention for head_dim 64 on wgmma (self- and cross-attention of the SpatialTransformer:
// reference attention.py:189-216 `F.scaled_dot_product_attention`, with the head split/merge copies
// of :196-214 folded into TMA coordinates).
//
//   O[b, i, h*64:(h+1)*64] = softmax_j(Q_h[i] . K_h[j] / 8) V_h[j]
//
// Q/K/V are 16-bit matrices [B, S, ld] (any row stride / column offset, e.g. slices of a fused
// QKV projection). One CTA = one (128-query tile, head, batch), keys in steps of 64:
//   warp 8      TMA producer (Q once per tile, K/V steps of 64 keys, 4 stages)
//   warps 0-7   two consumer warpgroups, 64 query rows each: S = Q K^T (wgmma, both operands in
//               shared memory, S in registers), online softmax in fp32 with exp2 on the accumulator
//               fragment (row reductions over the 4 lanes that share a row), then O += P V with P
//               taken from registers (16-bit) and V read transposed from shared memory.
// The running max is only raised when a row max grows by more than 2^8 (any reference point is a
// valid softmax shift; P stays < 2^8 and l carries the same scale), so O is rescaled rarely.
// Two CTAs are resident per SM (80 KB shared memory each).
#include "common.cuh"
#include "../../include/diffbir_b200.h"

namespace {

constexpr int TQ = 128;      // queries per CTA
constexpr int TK = 64;       // keys per step
constexpr int DH = 64;
constexpr int KV_STAGES = 4;
constexpr int Q_BYTES = TQ * DH * 2;       // 16 KB
constexpr int KV_BYTES = TK * DH * 2;      // 8 KB per K or V step
constexpr int ATTN_THREADS = 288;          // two consumer warpgroups + the producer warp
constexpr int CTAS_PER_SM = 2;
constexpr float RESCALE_LOG2 = 8.0f;
struct AttnParams {
  int sq, skv, heads;
  void* out;
  long long ldo;       // elements per output row
  float scale_log2;    // dh^-0.5 * log2(e)
  // work decomposition: CTA c runs the global steps [c * total / ctas, (c + 1) * total / ctas) of the
  // linearised (tile, key step) space, tile = (batch * heads + head) * q_tiles + q_tile. With
  // ctas == tiles every CTA owns one whole tile; otherwise ("stream-K") tiles cut by a CTA boundary
  // are finished through `ws`: each part stores its unnormalised O, reference max and row sum, the
  // last part to arrive (ticket) combines them in part order and writes the output.
  int q_tiles, n_steps, tiles, parts_max;
  long long total_steps;
  unsigned int* tickets;   // [tiles], zero on entry, self-resetting
  float* ws;               // [tiles][parts_max][WS_ROW planes][128 rows]
};
constexpr int WS_ROW = DH + 2;   // O[64], m_ref, l

struct __align__(8) AttnBarriers {
  uint64_t q_full, q_empty;
  uint64_t kv_full[KV_STAGES];
  uint64_t kv_empty[KV_STAGES];
  uint32_t last_flag;
};

constexpr int ATTN_SMEM = Q_BYTES + 2 * KV_STAGES * KV_BYTES + 256;

__device__ __forceinline__ int sk_bound(const AttnParams& p, int c) {
  if (p.parts_max == 0) return c * p.n_steps;           // one whole tile per CTA
  return static_cast<int>(static_cast<long long>(c) * p.total_steps / static_cast<long long>(gridDim.x));
}
// CTA whose range contains global step x
__device__ __forceinline__ int sk_owner(const AttnParams& p, int x) {
  int c = static_cast<int>(static_cast<long long>(x) * static_cast<long long>(gridDim.x) / p.total_steps);
  while (sk_bound(p, c + 1) <= x) ++c;
  while (sk_bound(p, c) > x) --c;
  return c;
}

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// SK = false: one whole tile per CTA (grid == tiles), the partial-tile machinery compiles away.
template <bool SK>
__global__ void __launch_bounds__(ATTN_THREADS, CTAS_PER_SM)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tma_q, const __grid_constant__ CUtensorMap tma_k,
                const __grid_constant__ CUtensorMap tma_v, const AttnParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Q_BYTES;
  uint8_t* sV = sK + KV_STAGES * KV_BYTES;
  AttnBarriers* bar = reinterpret_cast<AttnBarriers*>(sV + KV_STAGES * KV_BYTES);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_steps = p.n_steps;
  const int g_begin = SK ? sk_bound(p, blockIdx.x) : static_cast<int>(blockIdx.x) * n_steps;
  const int g_end = SK ? sk_bound(p, blockIdx.x + 1) : g_begin + n_steps;

  if (threadIdx.x == 0 && (smem_u32(smem) & 1023u) != 0) __trap();   // swizzled operands need 1024-byte alignment
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tma_q); tma_prefetch_desc(&tma_k); tma_prefetch_desc(&tma_v);
    mbar_init(&bar->q_full, 1);
    mbar_init(&bar->q_empty, 2);
    for (int s = 0; s < KV_STAGES; ++s) { mbar_init(&bar->kv_full[s], 1); mbar_init(&bar->kv_empty[s], 2); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_trigger();
  pdl_wait();

  // Every role walks the same list of segments (tile, key steps [a, e)) of this CTA's range; `it`
  // counts the CTA's key steps across segments and selects pipeline stages / barrier phases.
  if (warp == 8) {
    int it = 0, seg = 0;
    for (int g = g_begin; g < g_end; ++seg) {
      const int tile = g / n_steps;
      const int a = g - tile * n_steps;
      const int e = min(g_end, (tile + 1) * n_steps) - tile * n_steps;
      const int qt = tile % p.q_tiles, bh = tile / p.q_tiles;
      const int head = bh % p.heads, b = bh / p.heads;
      if (seg > 0) mbar_wait(&bar->q_empty, (seg - 1) & 1);     // QK MMAs of the previous tile retired
      if (elect_one()) {
        mbar_expect_tx(&bar->q_full, Q_BYTES);
        tma_load_3d(sQ, &tma_q, &bar->q_full, head * DH, qt * TQ, b);
      }
      __syncwarp();
      for (int j = a; j < e; ++j, ++it) {
        const int s = it % KV_STAGES;
        mbar_wait(&bar->kv_empty[s], ((it / KV_STAGES) & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&bar->kv_full[s], 2 * KV_BYTES);
          tma_load_3d(sK + s * KV_BYTES, &tma_k, &bar->kv_full[s], head * DH, j * TK, b);
          tma_load_3d(sV + s * KV_BYTES, &tma_v, &bar->kv_full[s], head * DH, j * TK, b);
        }
        __syncwarp();
      }
      g += e - a;
    }
  } else {
    const int wg = warp >> 2;
    const int rl0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);    // tile rows rl0 and rl0 + 8
    const int cq = 2 * (lane & 3);                              // column of fragment pair j: 8 j + cq
    const bool signal = (threadIdx.x & 127) == 0;               // one arrival per warpgroup
    const float sl2 = p.scale_log2;
    const uint64_t q_desc = wgmma_desc_sw128(smem_u32(sQ)) + static_cast<uint64_t>((wg * 64 * 128) >> 4);
    const uint64_t k_desc0 = wgmma_desc_sw128(smem_u32(sK));
    const uint64_t v_desc0 = wgmma_desc_sw128(smem_u32(sV));
    int it = 0, seg = 0;
    for (int g = g_begin; g < g_end; ++seg) {
      const int tile = g / n_steps;
      const int a = g - tile * n_steps;
      const int e = min(g_end, (tile + 1) * n_steps) - tile * n_steps;
      const int qt = tile % p.q_tiles, bh = tile / p.q_tiles;
      const int head = bh % p.heads, b = bh / p.heads;
      float m_ref[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // per row: softmax reference point, sum
      float o[DH / 2];
#pragma unroll
      for (int i = 0; i < DH / 2; ++i) o[i] = 0.f;
      mbar_wait(&bar->q_full, seg & 1);

      for (int j = a; j < e; ++j, ++it) {
        const int st = it % KV_STAGES;
        const int valid = min(TK, p.skv - j * TK);
        mbar_wait(&bar->kv_full[st], (it / KV_STAGES) & 1);
        float s[TK / 2];
#pragma unroll
        for (int i = 0; i < TK / 2; ++i) s[i] = 0.f;
        wgmma_fence();
        const uint64_t k_desc = k_desc0 + static_cast<uint64_t>((st * KV_BYTES) >> 4);
#pragma unroll
        for (int k = 0; k < DH / 16; ++k) wgmma_ss_n64(s, q_desc + 2 * k, k_desc + 2 * k);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(s, TK / 2);
        if (j == e - 1 && signal) mbar_arrive(&bar->q_empty);     // Q may be replaced
        if (valid < TK) {
#pragma unroll
          for (int i = 0; i < TK / 2; ++i)
            if (8 * (i >> 2) + cq + (i & 1) >= valid) s[i] = -INFINITY;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float mx = -INFINITY;
#pragma unroll
          for (int jj = 0; jj < TK / 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
          mx = quad_max(mx);
          if (j == a) {
            m_ref[h] = mx;
          } else if ((mx - m_ref[h]) * sl2 > RESCALE_LOG2) {
            const float alpha = ex2_approx((m_ref[h] - mx) * sl2);
#pragma unroll
            for (int jj = 0; jj < DH / 8; ++jj) {
              o[4 * jj + 2 * h] *= alpha;
              o[4 * jj + 2 * h + 1] *= alpha;
            }
            l_run[h] *= alpha;
            m_ref[h] = mx;
          }
        }
        // P = exp2(s * scale - m_ref * scale) in 16 bit, laid out as the A fragments of the PV MMAs
        const float nmb[2] = {-m_ref[0] * sl2, -m_ref[1] * sl2};
        uint32_t pa[TK / 16][4];
        float ls[2] = {0.f, 0.f};
#pragma unroll
        for (int i = 0; i < TK / 2; i += 2) {
          const int h = (i >> 1) & 1;
          const float x0 = ex2_approx(fmaf(s[i], sl2, nmb[h]));
          const float x1 = ex2_approx(fmaf(s[i + 1], sl2, nmb[h]));
          ls[h] += x0 + x1;
          pa[i >> 3][(i >> 1) & 3] = pack2(x0, x1);
        }
        l_run[0] += ls[0];
        l_run[1] += ls[1];
        wgmma_fence();
        const uint64_t v_desc = v_desc0 + static_cast<uint64_t>((st * KV_BYTES) >> 4);
#pragma unroll
        for (int kk = 0; kk < TK / 16; ++kk) wgmma_rs_n64_tb(o, pa[kk], v_desc + static_cast<uint64_t>((kk * 16 * 128) >> 4));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(o, DH / 2);
        if (signal) mbar_arrive(&bar->kv_empty[st]);
      }
      l_run[0] = quad_sum(l_run[0]);
      l_run[1] = quad_sum(l_run[1]);

      const bool whole = !SK || (a == 0 && e == n_steps);
      float inv[2] = {1.0f / l_run[0], 1.0f / l_run[1]};
      bool store = whole;
      if (!whole) {
        // part of a tile that a CTA boundary cuts: publish (O, m_ref, l), the last part combines
        const int t0 = tile * n_steps;
        const int c_lo = sk_owner(p, t0), c_hi = sk_owner(p, t0 + n_steps - 1);
        const int parts = c_hi - c_lo + 1, part = static_cast<int>(blockIdx.x) - c_lo;
        // part layout [WS_ROW planes][128 rows]
        float* wp = p.ws + (static_cast<long long>(tile) * p.parts_max + part) * (TQ * WS_ROW);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int rl = rl0 + 8 * h;
#pragma unroll
          for (int jj = 0; jj < DH / 8; ++jj) {
            __stcg(wp + (8 * jj + cq) * TQ + rl, o[4 * jj + 2 * h]);
            __stcg(wp + (8 * jj + cq + 1) * TQ + rl, o[4 * jj + 2 * h + 1]);
          }
          if ((lane & 3) == 0) {
            __stcg(wp + DH * TQ + rl, m_ref[h]);
            __stcg(wp + (DH + 1) * TQ + rl, l_run[h]);
          }
        }
        __threadfence();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (threadIdx.x == 0) {
          const unsigned int t = atomicAdd(&p.tickets[tile], 1u);
          const bool last = t == static_cast<unsigned int>(parts) - 1;
          if (last) p.tickets[tile] = 0;           // self-reset for the next launch
          bar->last_flag = last ? 1u : 0u;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (bar->last_flag) {
          __threadfence();
          const float* base = p.ws + static_cast<long long>(tile) * p.parts_max * (TQ * WS_ROW);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int rl = rl0 + 8 * h;
            float m_all = -INFINITY;
            for (int i = 0; i < parts; ++i)
              m_all = fmaxf(m_all, __ldcg(base + static_cast<long long>(i) * TQ * WS_ROW + DH * TQ + rl));
#pragma unroll
            for (int jj = 0; jj < DH / 8; ++jj) { o[4 * jj + 2 * h] = 0.f; o[4 * jj + 2 * h + 1] = 0.f; }
            float l_all = 0.f;
            for (int i = 0; i < parts; ++i) {        // fixed order: deterministic
              const float* pr = base + static_cast<long long>(i) * TQ * WS_ROW;
              const float wgt = ex2_approx((__ldcg(pr + DH * TQ + rl) - m_all) * sl2);
              l_all += __ldcg(pr + (DH + 1) * TQ + rl) * wgt;
#pragma unroll
              for (int jj = 0; jj < DH / 8; ++jj) {
                o[4 * jj + 2 * h] += __ldcg(pr + (8 * jj + cq) * TQ + rl) * wgt;
                o[4 * jj + 2 * h + 1] += __ldcg(pr + (8 * jj + cq + 1) * TQ + rl) * wgt;
              }
            }
            inv[h] = 1.0f / l_all;
          }
          store = true;
        }
        asm volatile("bar.sync 1, 256;" ::: "memory");      // last_flag is reused by the next segment
      }
      if (store) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int qi = qt * TQ + rl0 + 8 * h;
          if (qi >= p.sq) continue;
          op_t* o_ptr = reinterpret_cast<op_t*>(p.out) + (static_cast<long long>(b) * p.sq + qi) * p.ldo + head * DH + cq;
#pragma unroll
          for (int jj = 0; jj < DH / 8; ++jj)
            *reinterpret_cast<uint32_t*>(o_ptr + 8 * jj) = pack2(o[4 * jj + 2 * h] * inv[h], o[4 * jj + 2 * h + 1] * inv[h]);
        }
      }
      g += e - a;
    }
  }
}

int make_qkv_map(CUtensorMap* m, const void* base, int batch, int s, long long ld, int width, int box_rows) {
  uint64_t dims[3] = {static_cast<uint64_t>(width), static_cast<uint64_t>(s),
                      static_cast<uint64_t>(batch)};
  uint64_t strides[2] = {static_cast<uint64_t>(ld) * 2, static_cast<uint64_t>(s) * ld * 2};
  uint32_t box[3] = {DH, static_cast<uint32_t>(box_rows), 1};
  return dbir_make_tmap(m, base, 3, dims, strides, box, 2, 1);
}

}  // namespace

namespace {
// Stream-K decomposition: used when whole tiles would leave the last wave of CTA slots (two per SM)
// mostly empty, e.g. 320 tiles on 264 slots. Returns the grid size; *parts_max = 0 without stream-K.
int attn_plan(int batch, int heads, int sq, int skv, int* parts_max) {
  const int q_tiles = (sq + TQ - 1) / TQ, n_steps = (skv + TK - 1) / TK;
  const long long tiles = static_cast<long long>(batch) * heads * q_tiles;
  const long long slots = static_cast<long long>(CTAS_PER_SM) * dbir_sm_count();
  *parts_max = 0;
  // (the ticket array holds 16384 tiles; such grids are many waves deep and need no balancing)
  if (n_steps < 8 || tiles * n_steps < slots * 4 || tiles > 16384) return static_cast<int>(tiles);
  const long long waves = (tiles + slots - 1) / slots;
  // a single, partly filled wave is left alone: its CTAs mostly have an SM to themselves
  if (waves < 2 || static_cast<double>(tiles) / static_cast<double>(waves * slots) >= 0.8) return static_cast<int>(tiles);
  const long long ctas = slots * (waves - 1);                        // the work of the ragged wave is spread out
  const long long per_min = tiles * n_steps / ctas;                  // >= 4 here
  *parts_max = static_cast<int>((n_steps - 1 + per_min - 1) / per_min + 1);
  return static_cast<int>(ctas);
}
constexpr long long ATTN_TICKET_BYTES = 1 << 16;     // 16384 tiles
}  // namespace

extern "C" int64_t dbir_attention_ws_bytes(int32_t batch, int32_t heads, int32_t sq, int32_t skv) {
  if (batch <= 0 || heads <= 0 || sq <= 0 || skv <= 0) return 0;
  int parts_max = 0;
  attn_plan(batch, heads, sq, skv, &parts_max);
  if (parts_max == 0) return 0;
  const long long tiles = static_cast<long long>(batch) * heads * ((sq + TQ - 1) / TQ);
  return ATTN_TICKET_BYTES + tiles * parts_max * TQ * WS_ROW * 4;
}

extern "C" int dbir_attention(const void* q, const void* k, const void* v, void* out,
                              int32_t batch, int32_t heads, int32_t sq, int32_t skv,
                              int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                              void* ws, int64_t ws_bytes, void* stream) {
  DBIR_REQUIRE(q && k && v && out, "dbir_attention: null pointer");
  DBIR_REQUIRE(batch > 0 && heads > 0 && sq > 0 && skv > 0, "dbir_attention: bad shape");
  DBIR_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0,
               "dbir_attention: row strides must be multiples of 8 elements");
  CUtensorMap mq, mk, mv;
  const int width = heads * DH;
  if (make_qkv_map(&mq, q, batch, sq, ldq, width, TQ)) return -3;
  if (make_qkv_map(&mk, k, batch, skv, ldk, width, TK)) return -3;
  if (make_qkv_map(&mv, v, batch, skv, ldv, width, TK)) return -3;
  AttnParams p{};
  p.sq = sq; p.skv = skv; p.heads = heads;
  p.out = out; p.ldo = ldo;
  p.scale_log2 = 0.125f * 1.4426950408889634f;
  p.q_tiles = (sq + TQ - 1) / TQ;
  p.n_steps = (skv + TK - 1) / TK;
  const long long tiles = static_cast<long long>(batch) * heads * p.q_tiles;
  DBIR_REQUIRE(tiles * ((skv + TK - 1) / TK) < (1LL << 30), "dbir_attention: problem too large");
  p.tiles = static_cast<int>(tiles);
  p.total_steps = tiles * p.n_steps;
  int parts_max = 0;
  int ctas = attn_plan(batch, heads, sq, skv, &parts_max);
  if (parts_max > 0 && (!ws || ws_bytes < ATTN_TICKET_BYTES + tiles * parts_max * TQ * WS_ROW * 4)) {
    ctas = static_cast<int>(tiles);       // no (or too small a) workspace: whole tiles per CTA
    parts_max = 0;
  }
  p.parts_max = parts_max;
  if (parts_max > 0) {
    p.tickets = reinterpret_cast<unsigned int*>(ws);
    p.ws = reinterpret_cast<float*>(reinterpret_cast<char*>(ws) + ATTN_TICKET_BYTES);
  }
  static bool configured = false;
  if (!configured) {
    DBIR_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATTN_SMEM));
    DBIR_CHECK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, ATTN_SMEM));
    configured = true;
  }
  if (parts_max > 0)
    DBIR_CHECK_CUDA(dbir_launch(attn_fwd_kernel<true>, dim3(ctas), dim3(ATTN_THREADS), ATTN_SMEM,
                                reinterpret_cast<cudaStream_t>(stream), mq, mk, mv, p));
  else
    DBIR_CHECK_CUDA(dbir_launch(attn_fwd_kernel<false>, dim3(ctas), dim3(ATTN_THREADS), ATTN_SMEM,
                                reinterpret_cast<cudaStream_t>(stream), mq, mk, mv, p));
  return 0;
}
