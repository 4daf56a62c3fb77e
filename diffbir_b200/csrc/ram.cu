// RAM++ (the `--captioner ram` image tagger, reference ram/models/ram_plus.py) memory-bound kernels: Swin patch
// merging with its LayerNorm, the cls token (mean of the normed stage-4 tokens) and the per-image reweighting of
// the 51 description embeddings of every class. The rest of RAM++ runs on dbir_gemm / dbir_layernorm /
// dbir_window_attention / dbir_softmax_rows.
#include "common.cuh"
#include "../../include/diffbir_b200.h"

namespace {

// Sum of one value per thread over a 256-thread CTA in a fixed order (warp butterflies, then warps 0..7).
__device__ __forceinline__ float block_sum256(float v, float* red) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  v = warp_sum(v);
  __syncthreads();                            // red may still be read by the previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) t += red[i];
  return t;
}

// PatchMerging (swin_transformer.py:294-331): out row (b, oy, ox) = LN([x0 | x1 | x2 | x3]) over 4C with
// x0 = x[2oy, 2ox], x1 = x[2oy+1, 2ox], x2 = x[2oy, 2ox+1], x3 = x[2oy+1, 2ox+1]. One CTA per output row; two
// passes (mean, then the centred variance) over the fp32 stream, op16 out for the 4C -> 2C reduction GEMM.
__global__ void __launch_bounds__(256)
patch_merge_ln_kernel(const float* __restrict__ x, long long ldx, int H, int W, int C,
                      const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                      op_t* __restrict__ out, long long ldo) {
  __shared__ float red[8];
  pdl_trigger();
  pdl_wait();
  const int Wo = W / 2, Ho = H / 2;
  const long long orow = blockIdx.x;
  const int ox = static_cast<int>(orow % Wo), oy = static_cast<int>((orow / Wo) % Ho);
  const long long b = orow / (static_cast<long long>(Wo) * Ho);
  const float* x00 = x + ((b * H + 2 * oy) * W + 2 * ox) * ldx;
  const long long step_y = static_cast<long long>(W) * ldx;
  // element k of the concat: quarter q = k / C takes row offset (q & 1) down, (q >> 1) right
  auto at = [&](int k) {
    const int q = k / C;
    return *reinterpret_cast<const float4*>(x00 + (q & 1) * step_y + (q >> 1) * ldx + (k - q * C));
  };
  const int C4 = 4 * C;
  float s = 0.f;
  for (int k = threadIdx.x * 4; k < C4; k += 1024) {
    const float4 v = at(k);
    s += (v.x + v.y) + (v.z + v.w);
  }
  const float mean = block_sum256(s, red) / C4;
  float q2 = 0.f;
  for (int k = threadIdx.x * 4; k < C4; k += 1024) {
    const float4 v = at(k);
    const float a = v.x - mean, bb = v.y - mean, d = v.z - mean, e = v.w - mean;
    q2 += (a * a + bb * bb) + (d * d + e * e);
  }
  const float rstd = rsqrtf(block_sum256(q2, red) / C4 + eps);
  op_t* orow_p = out + orow * ldo;
  for (int k = threadIdx.x * 4; k < C4; k += 1024) {
    const float4 v = at(k);
    const float4 g = *reinterpret_cast<const float4*>(gamma + k);
    const float4 bt = *reinterpret_cast<const float4*>(beta + k);
    uint2 o;
    o.x = pack2((v.x - mean) * rstd * g.x + bt.x, (v.y - mean) * rstd * g.y + bt.y);
    o.y = pack2((v.z - mean) * rstd * g.z + bt.z, (v.w - mean) * rstd * g.w + bt.w);
    *reinterpret_cast<uint2*>(orow_p + k) = o;
  }
}

// [cls | tokens] operand of image_proj (swin_transformer.py:571-576): out row b*(L+1) = mean of x rows b*L ..
// b*L+L-1, summed in token order; out rows b*(L+1)+1+i = x row b*L+i. One thread per (image, channel).
__global__ void __launch_bounds__(256)
token_mean_kernel(const float* __restrict__ x, long long ldx, int L, int C, op_t* __restrict__ out, long long ldo) {
  pdl_trigger();
  pdl_wait();
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long long b = blockIdx.y;
  const float* xc = x + b * L * ldx + c;
  op_t* oc = out + b * (L + 1) * ldo + c;
  float s = 0.f;
  for (int i = 0; i < L; ++i) {
    const float v = xc[i * ldx];
    s += v;
    oc[(i + 1) * ldo] = f2op(v);
  }
  oc[0] = f2op(s / L);
}

// generate_tag's description reweighting (ram_plus.py:291-309) for one class, every image of the batch:
// cls <- cls / |cls|, l_j = scale * cls . e_j over the class's descriptions e_j (j < per_class), p = softmax(l),
// out = sum_j p_j e_j. One CTA per class, so each class's block of label_embed is read from HBM once per batch
// (the second pass and the other images hit L1 / L2). Fixed summation orders throughout.
constexpr int RW_DIM = 512;
constexpr int RW_MAX_DESC = 64;

__global__ void __launch_bounds__(256)
label_reweight_kernel(const float* __restrict__ cls, long long ld_cls, int batch, const op_t* __restrict__ label,
                      int classes, int per_class, float scale, op_t* __restrict__ out, long long ldo) {
  __shared__ float s_cls[RW_DIM];
  __shared__ float s_p[RW_MAX_DESC];
  __shared__ float red[8];
  pdl_trigger();
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, tid = threadIdx.x;
  const int cidx = blockIdx.x;
  const op_t* blk = label + static_cast<long long>(cidx) * per_class * RW_DIM;
  for (int b = 0; b < batch; ++b) {
    const float* cr = cls + b * ld_cls;
    const float a0 = cr[tid], a1 = cr[tid + 256];
    const float nrm = sqrtf(block_sum256(a0 * a0 + a1 * a1, red));
    s_cls[tid] = a0 / nrm;
    s_cls[tid + 256] = a1 / nrm;
    __syncthreads();
    for (int j = warp; j < per_class; j += 8) {
      const op_t* e = blk + static_cast<long long>(j) * RW_DIM;
      float acc = 0.f;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int d0 = half * 256 + lane * 8;
        const uint4 u = *reinterpret_cast<const uint4*>(e + d0);
        const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 f = unpack2(w4[i]);
          acc = fmaf(f.x, s_cls[d0 + 2 * i], acc);
          acc = fmaf(f.y, s_cls[d0 + 2 * i + 1], acc);
        }
      }
      acc = warp_sum(acc);
      if (lane == 0) s_p[j] = scale * acc;
    }
    __syncthreads();
    if (warp == 0) {                          // softmax over the descriptions (per_class <= 64: two per lane)
      const float x0 = lane < per_class ? s_p[lane] : -INFINITY;
      const float x1 = lane + 32 < per_class ? s_p[lane + 32] : -INFINITY;
      const float m = warp_max(fmaxf(x0, x1));
      const float e0 = lane < per_class ? __expf(x0 - m) : 0.f;
      const float e1 = lane + 32 < per_class ? __expf(x1 - m) : 0.f;
      const float inv = 1.0f / warp_sum(e0 + e1);
      __syncwarp();
      if (lane < per_class) s_p[lane] = e0 * inv;
      if (lane + 32 < per_class) s_p[lane + 32] = e1 * inv;
    }
    __syncthreads();
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j < per_class; ++j) {
      const float2 f = unpack2(*reinterpret_cast<const uint32_t*>(blk + static_cast<long long>(j) * RW_DIM + 2 * tid));
      o0 = fmaf(s_p[j], f.x, o0);
      o1 = fmaf(s_p[j], f.y, o1);
    }
    *reinterpret_cast<uint32_t*>(out + (static_cast<long long>(b) * classes + cidx) * ldo + 2 * tid) = pack2(o0, o1);
    __syncthreads();                          // s_cls / s_p are rewritten for the next image
  }
}

}  // namespace

extern "C" int dbir_swin_patch_merge(const float* x, int64_t ldx, int32_t n, int32_t h, int32_t w, int32_t c,
                                     const float* gamma, const float* beta, float eps, void* out, int64_t ldo,
                                     void* stream) {
  DBIR_REQUIRE(x && gamma && beta && out, "dbir_swin_patch_merge: null pointer");
  DBIR_REQUIRE(n > 0 && h % 2 == 0 && w % 2 == 0 && h > 0 && w > 0 && c % 4 == 0 && ldx >= c && ldx % 4 == 0 &&
                   ldo >= 4 * c && ldo % 4 == 0,
               "dbir_swin_patch_merge: bad geometry");
  const long long rows = static_cast<long long>(n) * (h / 2) * (w / 2);
  DBIR_CHECK_CUDA(dbir_launch(patch_merge_ln_kernel, dim3(static_cast<unsigned>(rows)), dim3(256), 0,
                              reinterpret_cast<cudaStream_t>(stream), x, static_cast<long long>(ldx), h, w, c, gamma,
                              beta, eps, reinterpret_cast<op_t*>(out), static_cast<long long>(ldo)));
  return 0;
}

extern "C" int dbir_token_mean(const float* x, int64_t ldx, int32_t n, int32_t tokens, int32_t c, void* out,
                               int64_t ldo, void* stream) {
  DBIR_REQUIRE(x && out && n > 0 && tokens > 0 && c > 0 && ldx >= c && ldo >= c, "dbir_token_mean: bad args");
  DBIR_CHECK_CUDA(dbir_launch(token_mean_kernel, dim3((c + 255) / 256, n), dim3(256), 0,
                              reinterpret_cast<cudaStream_t>(stream), x, static_cast<long long>(ldx), tokens, c,
                              reinterpret_cast<op_t*>(out), static_cast<long long>(ldo)));
  return 0;
}

extern "C" int dbir_label_reweight(const float* cls, int64_t ld_cls, int32_t batch, const void* label_embed,
                                   int32_t classes, int32_t per_class, int32_t dim, float scale, void* out,
                                   int64_t ldo, void* stream) {
  DBIR_REQUIRE(cls && label_embed && out && batch > 0 && classes > 0, "dbir_label_reweight: bad args");
  DBIR_REQUIRE(dim == RW_DIM && per_class > 0 && per_class <= RW_MAX_DESC && ldo >= dim && ldo % 2 == 0 &&
                   reinterpret_cast<uintptr_t>(label_embed) % 16 == 0,
               "dbir_label_reweight: built for 512-wide embeddings and at most 64 descriptions per class");
  DBIR_CHECK_CUDA(dbir_launch(label_reweight_kernel, dim3(classes), dim3(256), 0,
                              reinterpret_cast<cudaStream_t>(stream), cls, static_cast<long long>(ld_cls), batch,
                              reinterpret_cast<const op_t*>(label_embed), classes, per_class, scale,
                              reinterpret_cast<op_t*>(out), static_cast<long long>(ldo)));
  return 0;
}
