// Face detector (RetinaFace-ResNet50) and face parser (ParseNet) of the unaligned-face loop: the memory-bound
// kernels around dbir_gemm. Convolutions that dbir_gemm's conv mode does not take (7x7, stride 2, reflection
// padding, nearest-2x up-sampled input) are a patch gather into a 16-bit operand matrix plus a matrix-mode GEMM.
#include "common.cuh"
#include "../../include/diffbir_b200.h"

namespace {

constexpr int kThreads = 256;

inline unsigned blocks_for(long long n) {
  const long long b = (n + kThreads - 1) / kThreads;
  return static_cast<unsigned>(b < (1LL << 20) ? b : (1LL << 20));
}

// uint8 HWC pixels -> op16 [(n*h*w), 3]: out[c] = (src[c'] * scale - shift[c]) / div, c' = 2 - c when reverse.
__global__ void __launch_bounds__(kThreads)
face_input_kernel(const uint8_t* __restrict__ img, long long pixels, float scale, float s0, float s1, float s2,
                  float div, int reverse, op_t* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < pixels * 3;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % 3);
    const long long px = i / 3;
    const float v = static_cast<float>(img[px * 3 + (reverse ? 2 - c : c)]);
    const float sh = c == 0 ? s0 : (c == 1 ? s1 : s2);
    out[i] = f2op(__fdiv_rn(__fsub_rn(__fmul_rn(v, scale), sh), div));
  }
}

// Source coordinate of padded coordinate p on an axis of length n (zero padding: -1 = outside).
__device__ __forceinline__ int src_coord(int p, int n, int reflect) {
  if (p < 0) return reflect ? -p : -1;
  if (p >= n) return reflect ? 2 * (n - 1) - p : -1;
  return p;
}

// Patch matrix of a ksize x ksize convolution: out[(b, oy, ox), tap * C + c] = x[b, sy, sx, c], taps row-major,
// columns [ksize^2 C, kpad) zero. The source is the image nearest-2x up-sampled when up2 (so sy, sx address the
// up-sampled grid and read pixel (sy >> 1, sx >> 1)). VEC = 8: 16-byte chunks (C % 8 == 0).
template <int VEC>
__global__ void __launch_bounds__(kThreads)
patch_gather_kernel(const op_t* __restrict__ x, long long ldx, int H, int W, int C, int ksize, int stride,
                    int reflect, int up2, int Ho, int Wo, int kpad, long long rows, op_t* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int pad = ksize / 2, Hs = up2 ? 2 * H : H, Ws = up2 ? 2 * W : W;
  const int chunks = kpad / VEC, kreal = ksize * ksize * C;
  const long long total = rows * chunks;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / chunks;
    const int k = static_cast<int>(i - row * chunks) * VEC;
    op_t* dst = out + row * kpad + k;
    int sy = -1, sx = -1, c = 0;
    if (k < kreal) {
      const int tap = k / C;
      c = k - tap * C;
      const int ox = static_cast<int>(row % Wo), oy = static_cast<int>((row / Wo) % Ho);
      sy = src_coord(oy * stride + tap / ksize - pad, Hs, reflect);
      sx = src_coord(ox * stride + tap % ksize - pad, Ws, reflect);
    }
    if (sy < 0 || sx < 0) {
      if constexpr (VEC == 8) *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
      else *dst = f2op(0.f);
      continue;
    }
    if (up2) { sy >>= 1; sx >>= 1; }
    const long long b = row / (static_cast<long long>(Wo) * Ho);
    const op_t* src = x + ((b * H + sy) * W + sx) * ldx + c;
    if constexpr (VEC == 8) *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
    else *dst = *src;
  }
}

// 3x3 / stride 2 / pad 1 max pool on op16 NHWC, 8 channels per thread (padding never wins, as -inf).
__global__ void __launch_bounds__(kThreads)
maxpool3s2_kernel(const op_t* __restrict__ x, int H, int W, int C, int Ho, int Wo, long long rows,
                  op_t* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int chunks = C / 8;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < rows * chunks;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / chunks;
    const int c = static_cast<int>(i - row * chunks) * 8;
    const int ox = static_cast<int>(row % Wo), oy = static_cast<int>((row / Wo) % Ho);
    const long long b = row / (static_cast<long long>(Wo) * Ho);
    float m[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) m[j] = -INFINITY;
    for (int dy = 0; dy < 3; ++dy) {
      const int y = 2 * oy - 1 + dy;
      if (y < 0 || y >= H) continue;
      for (int dx = 0; dx < 3; ++dx) {
        const int xx = 2 * ox - 1 + dx;
        if (xx < 0 || xx >= W) continue;
        const uint4 u = *reinterpret_cast<const uint4*>(x + ((b * H + y) * W + xx) * C + c);
        const uint32_t w4[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 f = unpack2(w4[j]);
          m[2 * j] = fmaxf(m[2 * j], f.x);
          m[2 * j + 1] = fmaxf(m[2 * j + 1], f.y);
        }
      }
    }
    uint4 o;
    o.x = pack2(m[0], m[1]);
    o.y = pack2(m[2], m[3]);
    o.z = pack2(m[4], m[5]);
    o.w = pack2(m[6], m[7]);
    *reinterpret_cast<uint4*>(out + row * C + c) = o;
  }
}

// PyTorch's nearest source index for F.interpolate(size=out): identity, dst >> 1 at exactly 2x, else
// min(floor(dst * (float)in / out), in - 1).
__device__ __forceinline__ int nearest_src(int dst, int in, int outn) {
  if (outn == in) return dst;
  if (outn == 2 * in) return dst >> 1;
  const float scale = static_cast<float>(in) / static_cast<float>(outn);
  const int s = static_cast<int>(floorf(__fmul_rn(static_cast<float>(dst), scale)));
  return s < in - 1 ? s : in - 1;
}

// FPN top-down step: out = a + nearest_resize(b, size of a); a fp32 NHWC, b op16 NHWC, out op16. 4 channels / thread.
__global__ void __launch_bounds__(kThreads)
fpn_add_up_kernel(const float* __restrict__ a, const op_t* __restrict__ bsrc, int H, int W, int Hb, int Wb, int C,
                  long long rows, op_t* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int chunks = C / 4;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < rows * chunks;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / chunks;
    const int c = static_cast<int>(i - row * chunks) * 4;
    const int xx = static_cast<int>(row % W), y = static_cast<int>((row / W) % H);
    const long long n = row / (static_cast<long long>(W) * H);
    const int sy = nearest_src(y, Hb, H), sx = nearest_src(xx, Wb, W);
    const float4 av = *reinterpret_cast<const float4*>(a + row * C + c);
    const uint2 bu = *reinterpret_cast<const uint2*>(bsrc + ((n * Hb + sy) * Wb + sx) * C + c);
    const float2 b0 = unpack2(bu.x), b1 = unpack2(bu.y);
    uint2 o;
    o.x = pack2(__fadd_rn(av.x, b0.x), __fadd_rn(av.y, b0.y));
    o.y = pack2(__fadd_rn(av.z, b1.x), __fadd_rn(av.w, b1.y));
    *reinterpret_cast<uint2*>(out + row * C + c) = o;
  }
}

// Bottleneck tail: y = relu(x) (x = conv + bias + identity from the GEMM epilogue), fp32 y and op16 y16.
__global__ void __launch_bounds__(kThreads)
relu_cast_kernel(const float* __restrict__ x, long long n4, float* __restrict__ y, op_t* __restrict__ y16) {
  pdl_trigger();
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(x)[i];
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    if (y) reinterpret_cast<float4*>(y)[i] = v;
    uint2 o;
    o.x = pack2(v.x, v.y);
    o.y = pack2(v.z, v.w);
    reinterpret_cast<uint2*>(y16)[i] = o;
  }
}

// RetinaFace decode. Prior p = 2 * r + anchor, r = head row (levels back to back, row-major pixels); the prior box is
// PriorBox's (double, rounded to float); box / landmark decode with variances (0.1, 0.2), scaled to input pixels.
// head columns: [class logits 2 x 2 | box 2 x 4 | landmarks 2 x 10]. out [P, 15] = x1 y1 x2 y2 score l1x .. l5y.
__global__ void __launch_bounds__(kThreads)
retinaface_decode_kernel(const float* __restrict__ head, int H, int W, long long priors, float* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const long long p = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (p >= priors) return;
  const long long r = p >> 1;
  const int a = static_cast<int>(p & 1);
  long long off = 0;
  int step = 8, ms = 16, fw = 1, lvl = 0;
  for (lvl = 0; lvl < 3; ++lvl) {
    step = 8 << lvl;
    const int fh = (H + step - 1) / step;
    fw = (W + step - 1) / step;
    if (r < off + static_cast<long long>(fh) * fw) break;
    off += static_cast<long long>(fh) * fw;
  }
  ms = (16 << (2 * lvl)) << a;                          // (16, 32), (64, 128), (256, 512)
  const long long local = r - off;
  const int i = static_cast<int>(local / fw), j = static_cast<int>(local % fw);
  const float pcx = static_cast<float>((j + 0.5) * step / W), pcy = static_cast<float>((i + 0.5) * step / H);
  const float pw = static_cast<float>(static_cast<double>(ms) / W), ph = static_cast<float>(static_cast<double>(ms) / H);
  const float* h = head + r * 32;
  const float l0 = h[2 * a], l1 = h[2 * a + 1];
  const float m = fmaxf(l0, l1);
  const float e0 = expf(__fsub_rn(l0, m)), e1 = expf(__fsub_rn(l1, m));
  const float* bx = h + 4 + 4 * a;
  const float cx = __fadd_rn(pcx, __fmul_rn(__fmul_rn(bx[0], 0.1f), pw));
  const float cy = __fadd_rn(pcy, __fmul_rn(__fmul_rn(bx[1], 0.1f), ph));
  const float bw = __fmul_rn(pw, expf(__fmul_rn(bx[2], 0.2f)));
  const float bh = __fmul_rn(ph, expf(__fmul_rn(bx[3], 0.2f)));
  const float x1 = __fsub_rn(cx, __fdiv_rn(bw, 2.f)), y1 = __fsub_rn(cy, __fdiv_rn(bh, 2.f));
  const float fW = static_cast<float>(W), fH = static_cast<float>(H);
  float* o = out + p * 15;
  o[0] = __fmul_rn(x1, fW);
  o[1] = __fmul_rn(y1, fH);
  o[2] = __fmul_rn(__fadd_rn(bw, x1), fW);
  o[3] = __fmul_rn(__fadd_rn(bh, y1), fH);
  o[4] = __fdiv_rn(e1, __fadd_rn(e0, e1));
  const float* lm = h + 12 + 10 * a;
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    o[5 + 2 * k] = __fmul_rn(__fadd_rn(pcx, __fmul_rn(__fmul_rn(lm[2 * k], 0.1f), pw)), fW);
    o[6 + 2 * k] = __fmul_rn(__fadd_rn(pcy, __fmul_rn(__fmul_rn(lm[2 * k + 1], 0.1f), ph)), fH);
  }
}

// ParseNet mask: argmax over `classes` logits (first maximum wins, as torch.argmax) -> 255 for the face classes of
// FaceRestoreHelper's MASK_COLORMAP (1-13 and 15), else 0.
constexpr uint32_t kFaceClasses = 0x0000BFFEu;

__global__ void __launch_bounds__(kThreads)
parse_mask_kernel(const float* __restrict__ logits, long long ld, long long rows, int classes,
                  uint8_t* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < rows;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float* l = logits + i * ld;
    int best = 0;
    float bv = l[0];
    for (int k = 1; k < classes; ++k) {
      const float v = l[k];
      if (v > bv) { bv = v; best = k; }
    }
    out[i] = ((kFaceClasses >> best) & 1u) ? 255 : 0;
  }
}

}  // namespace

extern "C" int dbir_face_input(const uint8_t* img, int32_t n, int32_t h, int32_t w, float scale, float shift0,
                               float shift1, float shift2, float div, int32_t reverse, void* out, void* stream) {
  DBIR_REQUIRE(img && out && n > 0 && h > 0 && w > 0 && div != 0.f, "dbir_face_input: bad args");
  const long long px = static_cast<long long>(n) * h * w;
  DBIR_CHECK_CUDA(dbir_launch(face_input_kernel, dim3(blocks_for(3 * px)), dim3(kThreads), 0,
                              reinterpret_cast<cudaStream_t>(stream), img, px, scale, shift0, shift1, shift2, div,
                              static_cast<int>(reverse != 0), reinterpret_cast<op_t*>(out)));
  return 0;
}

extern "C" int dbir_patch_gather(const void* x, int64_t ldx, int32_t n, int32_t h, int32_t w, int32_t c,
                                 int32_t ksize, int32_t stride, int32_t reflect, int32_t up2, int32_t kpad, void* out,
                                 void* stream) {
  DBIR_REQUIRE(x && out && n > 0 && h > 0 && w > 0 && c > 0 && ldx >= c, "dbir_patch_gather: bad args");
  DBIR_REQUIRE((ksize == 1 || ksize == 3 || ksize == 7) && (stride == 1 || stride == 2),
               "dbir_patch_gather: ksize must be 1, 3 or 7 and stride 1 or 2");
  DBIR_REQUIRE(kpad % 64 == 0 && kpad >= ksize * ksize * c, "dbir_patch_gather: kpad=%d must be a multiple of 64 "
               ">= ksize^2 * C", kpad);
  const int hs = up2 ? 2 * h : h, ws = up2 ? 2 * w : w, pad = ksize / 2;
  DBIR_REQUIRE(!reflect || (pad < hs && pad < ws), "dbir_patch_gather: reflection padding wider than the image");
  const int ho = (hs + 2 * pad - ksize) / stride + 1, wo = (ws + 2 * pad - ksize) / stride + 1;
  const long long rows = static_cast<long long>(n) * ho * wo;
  auto st = reinterpret_cast<cudaStream_t>(stream);
  const op_t* xp = reinterpret_cast<const op_t*>(x);
  op_t* op = reinterpret_cast<op_t*>(out);
  if (c % 8 == 0 && ldx % 8 == 0) {
    DBIR_CHECK_CUDA(dbir_launch(patch_gather_kernel<8>, dim3(blocks_for(rows * (kpad / 8))), dim3(kThreads), 0, st,
                                xp, static_cast<long long>(ldx), h, w, c, ksize, stride, reflect != 0 ? 1 : 0,
                                up2 != 0 ? 1 : 0, ho, wo, kpad, rows, op));
  } else {
    DBIR_CHECK_CUDA(dbir_launch(patch_gather_kernel<1>, dim3(blocks_for(rows * kpad)), dim3(kThreads), 0, st, xp,
                                static_cast<long long>(ldx), h, w, c, ksize, stride, reflect != 0 ? 1 : 0,
                                up2 != 0 ? 1 : 0, ho, wo, kpad, rows, op));
  }
  return 0;
}

extern "C" int dbir_maxpool3s2(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, void* out, void* stream) {
  DBIR_REQUIRE(x && out && n > 0 && h > 0 && w > 0 && c % 8 == 0, "dbir_maxpool3s2: bad args (C %% 8 == 0)");
  const int ho = (h - 1) / 2 + 1, wo = (w - 1) / 2 + 1;
  const long long rows = static_cast<long long>(n) * ho * wo;
  DBIR_CHECK_CUDA(dbir_launch(maxpool3s2_kernel, dim3(blocks_for(rows * (c / 8))), dim3(kThreads), 0,
                              reinterpret_cast<cudaStream_t>(stream), reinterpret_cast<const op_t*>(x), h, w, c, ho,
                              wo, rows, reinterpret_cast<op_t*>(out)));
  return 0;
}

extern "C" int dbir_fpn_add_up(const float* a, const void* b, int32_t n, int32_t h, int32_t w, int32_t hb, int32_t wb,
                               int32_t c, void* out, void* stream) {
  DBIR_REQUIRE(a && b && out && n > 0 && h > 0 && w > 0 && hb > 0 && wb > 0 && c % 4 == 0,
               "dbir_fpn_add_up: bad args (C %% 4 == 0)");
  const long long rows = static_cast<long long>(n) * h * w;
  DBIR_CHECK_CUDA(dbir_launch(fpn_add_up_kernel, dim3(blocks_for(rows * (c / 4))), dim3(kThreads), 0,
                              reinterpret_cast<cudaStream_t>(stream), a, reinterpret_cast<const op_t*>(b), h, w, hb,
                              wb, c, rows, reinterpret_cast<op_t*>(out)));
  return 0;
}

extern "C" int dbir_relu_cast(const float* x, int64_t numel, float* y, void* y16, void* stream) {
  DBIR_REQUIRE(x && y16 && numel > 0 && numel % 4 == 0, "dbir_relu_cast: bad args (numel %% 4 == 0)");
  DBIR_CHECK_CUDA(dbir_launch(relu_cast_kernel, dim3(blocks_for(numel / 4)), dim3(kThreads), 0,
                              reinterpret_cast<cudaStream_t>(stream), x, static_cast<long long>(numel / 4), y,
                              reinterpret_cast<op_t*>(y16)));
  return 0;
}

extern "C" int dbir_retinaface_decode(const float* head, int32_t h, int32_t w, float* out, void* stream) {
  DBIR_REQUIRE(head && out && h > 0 && w > 0, "dbir_retinaface_decode: bad args");
  long long rows = 0;
  for (int s = 8; s <= 32; s *= 2) rows += static_cast<long long>((h + s - 1) / s) * ((w + s - 1) / s);
  const long long priors = 2 * rows;
  DBIR_CHECK_CUDA(dbir_launch(retinaface_decode_kernel, dim3(static_cast<unsigned>((priors + kThreads - 1) / kThreads)),
                              dim3(kThreads), 0, reinterpret_cast<cudaStream_t>(stream), head, h, w, priors, out));
  return 0;
}

extern "C" int dbir_parse_mask(const float* logits, int64_t ld, int64_t rows, int32_t classes, uint8_t* out,
                               void* stream) {
  DBIR_REQUIRE(logits && out && rows > 0 && classes > 0 && classes <= 32 && ld >= classes,
               "dbir_parse_mask: bad args");
  DBIR_CHECK_CUDA(dbir_launch(parse_mask_kernel, dim3(blocks_for(rows)), dim3(kThreads), 0,
                              reinterpret_cast<cudaStream_t>(stream), logits, static_cast<long long>(ld),
                              static_cast<long long>(rows), classes, out));
  return 0;
}
