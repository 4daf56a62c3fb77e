// Real-ESRGAN second-order degradation (reference dataset/batch_transform.py:142-285) on sm_90a.
//
// Every buffer is fp32 NCHW and owned by the caller; the random draws (torch.rand / randn / poisson /
// uniform_) stay with the caller, so a seeded run consumes exactly the reference's generator states.
// What lies between the draws runs here:
//
//   filter2d        utils.py:162-187 (reflect pad, odd k, one kernel or one per sample); optionally of the
//                   USM threshold mask |x - sub| * 255 > thr computed while the tile is staged (utils.py:205)
//   resize          F.interpolate, align_corners=False, no antialias: area (adaptive_avg_pool2d bins),
//                   bilinear, bicubic (A = -0.75, clamped taps)
//   gaussian_noise  degradation.py:461-554, one [h, w] gray field shared by the batch and scaled per sample
//   noise_levels /  degradation.py:610-724: uint8 levels + a 256-bin histogram per sample, vals = 2^ceil(log2
//   poisson_rate /  (distinct levels)) on the device, rate = level * vals for torch.poisson, then the noise,
//   poisson_noise   the gray mix, the scale and the clip
//   diffjpeg        diffjpeg.py:450-492 (differentiable=False), one 16x16 macroblock per step
//   usm_blend       utils.py:206-210
//   lq_levels /     batch_transform.py:271,279-281
//   pair_nhwc
//
// The elementwise steps reproduce PyTorch's CUDA op order with explicitly rounded intrinsics (no FMA
// contraction): a tensor divided by a Python scalar is computed by PyTorch on CUDA as a product with the
// fp32 reciprocal, so `x / 255.` is `x * (1.f / 255.f)` here too.
#include "common.cuh"
#include "../../include/diffbir_b200.h"

namespace {

constexpr float INV255 = 1.0f / 255.0f;
constexpr float INV100 = 1.0f / 100.0f;

__device__ __forceinline__ int reflect(int i, int n) {
  return i < 0 ? -i : (i >= n ? 2 * (n - 1) - i : i);
}

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

// ---------------------------------------------------------------------------------------------
// filter2d: one CTA per 32x32 output tile of one (sample, channel) plane. The tile plus its k-1 halo
// (reflect-padded) and the k*k taps are staged in shared memory; each thread accumulates four rows
// of one column, so a warp reads 32 consecutive words per tap (no bank conflicts).
// ---------------------------------------------------------------------------------------------
constexpr int FT = 32;            // output tile side
constexpr int FROWS = 4;          // rows per thread (blockDim = 32 x 8)
constexpr int KMAX = 63;

__global__ void __launch_bounds__(256)
filter2d_kernel(const float* __restrict__ x, const float* __restrict__ sub, float thr, int c, int h, int w,
                const float* __restrict__ kern, long long kstride, int k, float* __restrict__ out) {
  extern __shared__ float sm[];
  const int sw = FT + k - 1;
  float* tile = sm;
  float* taps = sm + sw * sw;
  const int plane = blockIdx.z, smp = plane / c, r = k / 2;
  const long long base = static_cast<long long>(plane) * h * w;
  const int x0 = blockIdx.x * FT, y0 = blockIdx.y * FT;
  const int tid = threadIdx.y * 32 + threadIdx.x;
  const float* kp = kern + smp * kstride;
  for (int i = tid; i < k * k; i += 256) taps[i] = kp[i];
  // Tile positions past the image's last row / column plus r feed only outputs outside the image (never
  // written); they are zero-filled rather than read, so every staged coordinate lies in [-r, n-1+r] and one
  // reflection (r < n) maps it into the image.
  const int ylast = h - 1 + r - (y0 - r), xlast = w - 1 + r - (x0 - r);
  for (int i = tid; i < sw * sw; i += 256) {
    const int by = i / sw, bx = i - by * sw;
    if (by > ylast || bx > xlast) {
      tile[i] = 0.f;
      continue;
    }
    const int gy = reflect(y0 - r + by, h), gx = reflect(x0 - r + bx, w);
    const long long o = base + static_cast<long long>(gy) * w + gx;
    float v = x[o];
    if (sub != nullptr) v = __fmul_rn(fabsf(__fsub_rn(v, sub[o])), 255.f) > thr ? 1.f : 0.f;
    tile[i] = v;
  }
  __syncthreads();
  float acc[FROWS];
#pragma unroll
  for (int j = 0; j < FROWS; ++j) acc[j] = 0.f;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int ky = 0; ky < k; ++ky) {
    const float* row = tile + (ty + ky) * sw + tx;
    const float* wk = taps + ky * k;
#pragma unroll 4
    for (int kx = 0; kx < k; ++kx) {
      const float wt = wk[kx];
#pragma unroll
      for (int j = 0; j < FROWS; ++j) acc[j] = fmaf(wt, row[j * 8 * sw + kx], acc[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < FROWS; ++j) {
    const int gy = y0 + ty + 8 * j, gx = x0 + tx;
    if (gy < h && gx < w) out[base + static_cast<long long>(gy) * w + gx] = acc[j];
  }
}

// ---------------------------------------------------------------------------------------------
// resize: one thread per output element; formulas and op order of ATen's CUDA upsample kernels.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float cubic1(float x, float a) { return ((a + 2) * x - (a + 3)) * x * x + 1; }
__device__ __forceinline__ float cubic2(float x, float a) { return ((a * x - 5 * a) * x + 8 * a) * x - 4 * a; }

__device__ __forceinline__ float cubic_interp(float x0, float x1, float x2, float x3, float t) {
  const float a = -0.75f;
  const float c0 = cubic2(t + 1.0f, a), c1 = cubic1(t, a);
  const float u = 1.0f - t;
  const float c2 = cubic1(u, a), c3 = cubic2(u + 1.0f, a);
  return x0 * c0 + x1 * c1 + x2 * c2 + x3 * c3;
}

__global__ void resize_kernel(const float* __restrict__ x, long long planes, int hin, int win, int hout, int wout,
                              int mode, float rh, float rw, float* __restrict__ out) {
  const long long total = planes * hout * wout;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int ox = static_cast<int>(i % wout);
    const int oy = static_cast<int>((i / wout) % hout);
    const long long p = i / (static_cast<long long>(wout) * hout);
    const float* src = x + p * hin * win;
    float v;
    if (mode == 0) {                                   // area == adaptive_avg_pool2d
      const int ys = static_cast<int>(static_cast<long long>(oy) * hin / hout);
      const int ye = static_cast<int>((static_cast<long long>(oy + 1) * hin + hout - 1) / hout);
      const int xs = static_cast<int>(static_cast<long long>(ox) * win / wout);
      const int xe = static_cast<int>((static_cast<long long>(ox + 1) * win + wout - 1) / wout);
      float s = 0.f;
      for (int yy = ys; yy < ye; ++yy)
        for (int xx = xs; xx < xe; ++xx) s += src[static_cast<long long>(yy) * win + xx];
      v = s / (ye - ys) / (xe - xs);
    } else if (mode == 1) {                            // bilinear
      float hr = rh * (oy + 0.5f) - 0.5f;
      hr = hr < 0 ? 0.f : hr;
      float wr = rw * (ox + 0.5f) - 0.5f;
      wr = wr < 0 ? 0.f : wr;
      const int h1 = min(static_cast<int>(hr), hin - 1), w1 = min(static_cast<int>(wr), win - 1);
      const int h1p = h1 < hin - 1 ? 1 : 0, w1p = w1 < win - 1 ? 1 : 0;
      const float h1l = hr - h1, h0l = 1.0f - h1l, w1l = wr - w1, w0l = 1.0f - w1l;
      const float* r0 = src + static_cast<long long>(h1) * win + w1;
      const float* r1 = r0 + static_cast<long long>(h1p) * win;
      v = h0l * (w0l * r0[0] + w1l * r0[w1p]) + h1l * (w0l * r1[0] + w1l * r1[w1p]);
    } else {                                           // bicubic
      const float hr = rh * (oy + 0.5f) - 0.5f, wr = rw * (ox + 0.5f) - 0.5f;
      const int iy = static_cast<int>(floorf(hr)), ix = static_cast<int>(floorf(wr));
      const float ty = hr - iy, tx = wr - ix;
      float rows[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float* rp = src + static_cast<long long>(min(max(iy - 1 + j, 0), hin - 1)) * win;
        rows[j] = cubic_interp(rp[min(max(ix - 1, 0), win - 1)], rp[min(max(ix, 0), win - 1)],
                               rp[min(max(ix + 1, 0), win - 1)], rp[min(max(ix + 2, 0), win - 1)], tx);
      }
      v = cubic_interp(rows[0], rows[1], rows[2], rows[3], ty);
    }
    out[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// noise. Per-sample parameters come from uniform draws u: param = u * span + lo, gray = u_gray < p.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float draw_param(const float* u, int s, float lo, float span) {
  return __fadd_rn(__fmul_rn(u[s], span), lo);
}
__device__ __forceinline__ float gray_flag(const float* u, int s, float p) { return u[s] < p ? 1.f : 0.f; }

__global__ void gaussian_noise_kernel(const float* __restrict__ img, const float* __restrict__ noise,
                                      const float* __restrict__ noise_gray, const float* __restrict__ u_sigma,
                                      float lo, float span, const float* __restrict__ u_gray, float gray_prob,
                                      int c, long long hw, long long total, float* __restrict__ out) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int s = static_cast<int>(i / (c * hw));
    const float sigma = draw_param(u_sigma, s, lo, span);
    float n = __fmul_rn(__fmul_rn(noise[i], sigma), INV255);
    if (noise_gray != nullptr) {
      const float g = gray_flag(u_gray, s, gray_prob);
      const float ng = __fmul_rn(__fmul_rn(noise_gray[i % hw], sigma), INV255);
      n = __fadd_rn(__fmul_rn(n, __fsub_rn(1.f, g)), __fmul_rn(ng, g));
    }
    out[i] = clamp01(__fadd_rn(img[i], n));
  }
}

__device__ __forceinline__ float levels_of(float v, int* level) {
  const float r = fminf(fmaxf(rintf(__fmul_rn(v, 255.f)), 0.f), 255.f);
  *level = r == r ? static_cast<int>(r) : -1;
  return __fmul_rn(r, INV255);
}

// q = clamp(round(x * 255), 0, 255) / 255 per element (gray: of rgb_to_grayscale(x)); hist[s][level] += 1.
__global__ void noise_levels_kernel(const float* __restrict__ img, int c, long long hw, int gray,
                                    float* __restrict__ q, int* __restrict__ hist) {
  __shared__ int bins[256];
  const int s = blockIdx.y;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) bins[i] = 0;
  __syncthreads();
  const long long per = gray ? hw : c * hw;
  const float* src = img + static_cast<long long>(s) * c * hw;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < per;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float v = src[i];
    if (gray) {                    // torchvision rgb_to_grayscale: (0.2989 r + 0.587 g) + 0.114 b
      v = __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, v), __fmul_rn(0.587f, src[i + hw])),
                    __fmul_rn(0.114f, src[i + 2 * hw]));
    }
    int lv;
    q[s * per + i] = levels_of(v, &lv);
    if (lv >= 0) atomicAdd(&bins[lv], 1);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x)
    if (bins[i]) atomicAdd(&hist[s * 256 + i], bins[i]);
}

// vals[s] = 2^ceil(log2(number of non-empty bins)); rate = q * vals.
__global__ void poisson_rate_kernel(const float* __restrict__ q, const int* __restrict__ hist, long long per,
                                    float* __restrict__ vals, float* __restrict__ rate) {
  const int s = blockIdx.y;
  // blockDim.x == 256: one bin per thread
  const int total = __syncthreads_count(hist[s * 256 + threadIdx.x] != 0);
  int p2 = 1;
  while (p2 < total) p2 <<= 1;
  const float v = static_cast<float>(p2);
  if (blockIdx.x == 0 && threadIdx.x == 0) vals[s] = v;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < per;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    rate[s * per + i] = __fmul_rn(q[s * per + i], v);
}

// noise = draw / vals - q (gray: mixed with the gray field's), * scale; out = clip(img + noise, 0, 1).
__global__ void poisson_noise_kernel(const float* __restrict__ img, const float* __restrict__ q,
                                     const float* __restrict__ draw, const float* __restrict__ vals,
                                     const float* __restrict__ q_gray, const float* __restrict__ draw_gray,
                                     const float* __restrict__ vals_gray, const float* __restrict__ u_scale,
                                     float lo, float span, const float* __restrict__ u_gray, float gray_prob,
                                     int c, long long hw, long long total, float* __restrict__ out) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int s = static_cast<int>(i / (c * hw));
    float n = __fsub_rn(__fdiv_rn(draw[i], vals[s]), q[i]);
    if (q_gray != nullptr) {
      const long long gi = s * hw + i % hw;
      const float g = gray_flag(u_gray, s, gray_prob);
      const float ng = __fsub_rn(__fdiv_rn(draw_gray[gi], vals_gray[s]), q_gray[gi]);
      n = __fadd_rn(__fmul_rn(n, __fsub_rn(1.f, g)), __fmul_rn(ng, g));
    }
    n = __fmul_rn(n, draw_param(u_scale, s, lo, span));
    out[i] = clamp01(__fadd_rn(img[i], n));
  }
}

// ---------------------------------------------------------------------------------------------
// DiffJPEG. The 8x8 DCT basis T[x][y][u][v] = cos((2x+1)u pi/16) cos((2y+1)v pi/16) is built per CTA in
// double (rounded to fp32 like the reference's numpy table) twice: indexed [xy][uv] for the forward
// transform and [uv][xy] for the inverse, so both walks read consecutive words across a warp.
// Quantisation tables: ITU-T T.81 Annex K.1 / K.2; luminance is used transposed, chrominance is symmetric.
// ---------------------------------------------------------------------------------------------
__constant__ float kYTable[64] = {
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57,
    69, 56, 14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64,
    81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
__constant__ float kCTable4[16] = {17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 99, 47, 66, 99, 99};

__device__ __forceinline__ float qtable(int chroma, int u, int v) {
  if (chroma) return (u < 4 && v < 4) ? kCTable4[u * 4 + v] : 99.f;
  return kYTable[v * 8 + u];
}

// quality -> factor exactly as PyTorch evaluates quality_to_factor on a CUDA scalar tensor
__device__ __forceinline__ float jpeg_factor(float q) {
  const float f = q < 50.f ? __fmul_rn(__frcp_rn(q), 5000.f) : __fsub_rn(200.f, __fmul_rn(q, 2.f));
  return __fmul_rn(f, INV100);
}

constexpr int JT = 256;

__global__ void __launch_bounds__(JT)
diffjpeg_kernel(const float* __restrict__ x, const float* __restrict__ quality, int is_factor, int b, int h, int w,
                int clamp_in, float* __restrict__ out) {
  __shared__ float tf[64 * 64];      // tf[xy * 64 + uv]
  __shared__ float ti[64 * 64];      // ti[uv * 64 + xy]
  __shared__ double cosv[64];        // cos((2p+1) f pi / 16) at [p * 8 + f]
  __shared__ float ycc[3][256];      // Y, Cb, Cr of the macroblock (16 x 16)
  __shared__ float blk[6][64];       // 4 Y blocks, Cb, Cr (8x8 after subsampling), then coefficients
  __shared__ float rec[6][64];
  const int tid = threadIdx.x;
  if (tid < 64) cosv[tid] = cos(static_cast<double>((2 * (tid >> 3) + 1) * (tid & 7)) * 3.141592653589793 / 16);
  __syncthreads();
  for (int i = tid; i < 4096; i += JT) {
    const int xy = i >> 6, uv = i & 63;
    const float t = __double2float_rn(cosv[(xy >> 3) * 8 + (uv >> 3)] * cosv[(xy & 7) * 8 + (uv & 7)]);
    tf[i] = t;
    ti[uv * 64 + xy] = t;
  }
  const int hp = (h + 15) / 16, wp = (w + 15) / 16;
  const long long nmb = static_cast<long long>(b) * hp * wp;
  for (long long mb = blockIdx.x; mb < nmb; mb += gridDim.x) {
    const int s = static_cast<int>(mb / (static_cast<long long>(hp) * wp));
    const int rem = static_cast<int>(mb % (static_cast<long long>(hp) * wp));
    const int y0 = (rem / wp) * 16, x0 = (rem % wp) * 16;
    const float factor = is_factor ? quality[s] : jpeg_factor(quality[s]);
    const long long plane = static_cast<long long>(h) * w;
    const float* src = x + static_cast<long long>(s) * 3 * plane;
    __syncthreads();                                   // previous macroblock done with the buffers
    {                                                  // x * 255 -> YCbCr (zero padding to x16)
      const int py = tid >> 4, px = tid & 15, gy = y0 + py, gx = x0 + px;
      float r = 0.f, g = 0.f, bl = 0.f;
      if (gy < h && gx < w) {
        const long long o = static_cast<long long>(gy) * w + gx;
        r = src[o]; g = src[o + plane]; bl = src[o + 2 * plane];
        if (clamp_in) { r = clamp01(r); g = clamp01(g); bl = clamp01(bl); }
      }
      r = __fmul_rn(r, 255.f); g = __fmul_rn(g, 255.f); bl = __fmul_rn(bl, 255.f);
      ycc[0][tid] = fmaf(0.114f, bl, fmaf(0.587f, g, __fmul_rn(0.299f, r)));
      ycc[1][tid] = __fadd_rn(fmaf(0.5f, bl, fmaf(-0.331264f, g, __fmul_rn(-0.168736f, r))), 128.f);
      ycc[2][tid] = __fadd_rn(fmaf(-0.081312f, bl, fmaf(-0.418688f, g, __fmul_rn(0.5f, r))), 128.f);
    }
    __syncthreads();
    for (int i = tid; i < 384; i += JT) {              // split into 8x8 blocks; 2x2 chroma average
      const int k = i >> 6, xy = i & 63, bx = xy >> 3, by = xy & 7;
      float v;
      if (k < 4) {
        v = ycc[0][((k >> 1) * 8 + bx) * 16 + (k & 1) * 8 + by];
      } else {
        const float* cp = ycc[k - 3] + (2 * bx) * 16 + 2 * by;
        v = __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(cp[0], cp[1]), cp[16]), cp[17]), 4.f);
      }
      blk[k][xy] = __fsub_rn(v, 128.f);
    }
    __syncthreads();
    for (int i = tid; i < 384; i += JT) {              // DCT, quantise, round, dequantise, * alpha
      const int k = i >> 6, uv = i & 63, u = uv >> 3, v = uv & 7;
      float acc = 0.f;
#pragma unroll 8
      for (int xy = 0; xy < 64; ++xy) acc = fmaf(blk[k][xy], tf[xy * 64 + uv], acc);
      const double au = u ? 1.0 : 1.0 / sqrt(2.0), av = v ? 1.0 : 1.0 / sqrt(2.0);
      const float coef = __fmul_rn(__double2float_rn(au * av * 0.25), acc);
      const float tab = __fmul_rn(qtable(k >= 4, u, v), factor);
      const float qv = rintf(__fdiv_rn(coef, tab));
      rec[k][uv] = __fmul_rn(__fmul_rn(qv, tab), __double2float_rn(au * av));
    }
    __syncthreads();
    for (int i = tid; i < 384; i += JT) {              // inverse DCT
      const int k = i >> 6, xy = i & 63;
      float acc = 0.f;
#pragma unroll 8
      for (int uv = 0; uv < 64; ++uv) acc = fmaf(rec[k][uv], ti[uv * 64 + xy], acc);
      blk[k][xy] = __fadd_rn(__fmul_rn(0.25f, acc), 128.f);
    }
    __syncthreads();
    {                                                  // chroma repeat, YCbCr -> RGB, clamp, / 255, crop
      const int py = tid >> 4, px = tid & 15, gy = y0 + py, gx = x0 + px;
      if (gy < h && gx < w) {
        const float yv = blk[((py >> 3) << 1) | (px >> 3)][(py & 7) * 8 + (px & 7)];
        const int ci = (py >> 1) * 8 + (px >> 1);
        const float cb = __fsub_rn(blk[4][ci], 128.f), cr = __fsub_rn(blk[5][ci], 128.f);
        const float rgb[3] = {fmaf(1.402f, cr, yv), fmaf(-0.714136f, cr, fmaf(-0.344136f, cb, yv)),
                              fmaf(1.772f, cb, yv)};
        float* dst = out + static_cast<long long>(s) * 3 * plane + static_cast<long long>(gy) * w + gx;
#pragma unroll
        for (int ch = 0; ch < 3; ++ch) dst[ch * plane] = __fmul_rn(fminf(255.f, fmaxf(0.f, rgb[ch])), INV255);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// small elementwise tails
// ---------------------------------------------------------------------------------------------
__global__ void usm_blend_kernel(const float* __restrict__ img, const float* __restrict__ blur,
                                 const float* __restrict__ soft, float weight, long long n, float* __restrict__ out) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float im = img[i], m = soft[i];
    const float res = __fsub_rn(im, blur[i]);
    const float sharp = clamp01(__fadd_rn(im, __fmul_rn(weight, res)));
    out[i] = __fadd_rn(__fmul_rn(m, sharp), __fmul_rn(__fsub_rn(1.f, m), im));
  }
}

__global__ void lq_levels_kernel(const float* __restrict__ x, long long n, float* __restrict__ out) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = __fmul_rn(fminf(fmaxf(rintf(__fmul_rn(x[i], 255.f)), 0.f), 255.f), INV255);
}

__global__ void pair_nhwc_kernel(const float* __restrict__ lq, const float* __restrict__ hq, int c, long long hw,
                                 long long n, float* __restrict__ lq_out, float* __restrict__ hq_out) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {      // i indexes the NHWC output
    const int ch = static_cast<int>(i % c);
    const long long pix = (i / c) % hw, s = i / (c * hw);
    const long long src = (s * c + ch) * hw + pix;
    lq_out[i] = lq[src];
    hq_out[i] = __fsub_rn(__fmul_rn(hq[src], 2.f), 1.f);
  }
}

int grid_for(long long n, int threads) {
  const long long cap = static_cast<long long>(dbir_sm_count()) * 16;
  long long g = (n + threads - 1) / threads;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

extern "C" int dbir_filter2d(const float* x, const float* sub, float threshold, int32_t b, int32_t c, int32_t h,
                             int32_t w, const float* kernel, int64_t kernel_stride, int32_t k, float* out,
                             void* stream) {
  DBIR_REQUIRE(x && kernel && out && x != out, "dbir_filter2d: need distinct input and output");
  DBIR_REQUIRE(b > 0 && c > 0 && static_cast<long long>(b) * c <= 65535, "dbir_filter2d: bad batch");
  DBIR_REQUIRE(k % 2 == 1 && k >= 1 && k <= KMAX, "dbir_filter2d: kernel size must be odd and <= 63");
  DBIR_REQUIRE(h > k / 2 && w > k / 2, "dbir_filter2d: reflect padding needs h and w > k / 2");
  const int sw = FT + k - 1;
  const int smem = (sw * sw + k * k) * static_cast<int>(sizeof(float));
  static bool configured = false;
  if (!configured) {
    const int most = ((FT + KMAX - 1) * (FT + KMAX - 1) + KMAX * KMAX) * static_cast<int>(sizeof(float));
    DBIR_CHECK_CUDA(cudaFuncSetAttribute(filter2d_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, most));
    configured = true;
  }
  dim3 grid((w + FT - 1) / FT, (h + FT - 1) / FT, b * c);
  filter2d_kernel<<<grid, dim3(32, 8), smem, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, sub, threshold, c, h, w, kernel, kernel_stride, k, out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_resize(const float* x, int64_t planes, int32_t hin, int32_t win, int32_t hout, int32_t wout,
                           int32_t mode, float ratio_h, float ratio_w, float* out, void* stream) {
  DBIR_REQUIRE(x && out && x != out, "dbir_resize: need distinct input and output");
  DBIR_REQUIRE(planes > 0 && hin > 0 && win > 0 && hout > 0 && wout > 0, "dbir_resize: bad shape");
  DBIR_REQUIRE(mode >= 0 && mode <= 2, "dbir_resize: mode is 0 area, 1 bilinear, 2 bicubic");
  const long long n = planes * hout * wout;
  resize_kernel<<<grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, planes, hin, win, hout, wout, mode, ratio_h, ratio_w, out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_gaussian_noise(const float* img, const float* noise, const float* noise_gray, const float* u_sigma,
                                   float sigma_lo, float sigma_span, const float* u_gray, float gray_prob, int32_t b,
                                   int32_t c, int64_t hw, float* out, void* stream) {
  DBIR_REQUIRE(img && noise && u_sigma && out && b > 0 && c > 0 && hw > 0, "dbir_gaussian_noise: bad arguments");
  DBIR_REQUIRE(noise_gray == nullptr || u_gray != nullptr, "dbir_gaussian_noise: the gray field needs u_gray");
  const long long n = static_cast<long long>(b) * c * hw;
  gaussian_noise_kernel<<<grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      img, noise, noise_gray, u_sigma, sigma_lo, sigma_span, u_gray, gray_prob, c, hw, n, out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_noise_levels(const float* img, int32_t b, int32_t c, int64_t hw, int32_t gray, float* q,
                                 int32_t* hist, void* stream) {
  DBIR_REQUIRE(img && q && hist && b > 0 && b <= 65535 && c > 0 && hw > 0, "dbir_noise_levels: bad arguments");
  DBIR_REQUIRE(!gray || c == 3, "dbir_noise_levels: the gray level image needs 3 channels");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DBIR_CHECK_CUDA(cudaMemsetAsync(hist, 0, sizeof(int32_t) * 256 * b, st));
  const long long per = gray ? hw : c * hw;
  const int gx = (grid_for(per * b, 256) + b - 1) / b;
  noise_levels_kernel<<<dim3(gx, b), 256, 0, st>>>(img, c, hw, gray, q, reinterpret_cast<int*>(hist));
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_poisson_rate(const float* q, const int32_t* hist, int32_t b, int64_t per_sample, float* vals,
                                 float* rate, void* stream) {
  DBIR_REQUIRE(q && hist && vals && rate && b > 0 && b <= 65535 && per_sample > 0, "dbir_poisson_rate: bad arguments");
  const int gx = (grid_for(per_sample * b, 256) + b - 1) / b;
  poisson_rate_kernel<<<dim3(gx, b), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      q, reinterpret_cast<const int*>(hist), per_sample, vals, rate);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_poisson_noise(const float* img, const float* q, const float* draw, const float* vals,
                                  const float* q_gray, const float* draw_gray, const float* vals_gray,
                                  const float* u_scale, float scale_lo, float scale_span, const float* u_gray,
                                  float gray_prob, int32_t b, int32_t c, int64_t hw, float* out, void* stream) {
  DBIR_REQUIRE(img && q && draw && vals && u_scale && out && b > 0 && c > 0 && hw > 0,
               "dbir_poisson_noise: bad arguments");
  DBIR_REQUIRE(q_gray == nullptr || (draw_gray && vals_gray && u_gray), "dbir_poisson_noise: incomplete gray field");
  const long long n = static_cast<long long>(b) * c * hw;
  poisson_noise_kernel<<<grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      img, q, draw, vals, q_gray, draw_gray, vals_gray, u_scale, scale_lo, scale_span, u_gray, gray_prob, c, hw, n,
      out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_diffjpeg(const float* x, const float* quality, int32_t quality_is_factor, int32_t b, int32_t h,
                             int32_t w, int32_t clamp_in, float* out, void* stream) {
  DBIR_REQUIRE(x && quality && out && b > 0 && h > 0 && w > 0, "dbir_diffjpeg: bad arguments");
  const long long nmb = static_cast<long long>(b) * ((h + 15) / 16) * ((w + 15) / 16);
  const long long cap = static_cast<long long>(dbir_sm_count()) * 8;
  const int grid = static_cast<int>(nmb < cap ? nmb : cap);
  diffjpeg_kernel<<<grid, JT, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, quality, quality_is_factor, b, h, w,
                                                                          clamp_in, out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_usm_blend(const float* img, const float* blur, const float* soft, float weight, int64_t n,
                              float* out, void* stream) {
  DBIR_REQUIRE(img && blur && soft && out && n > 0, "dbir_usm_blend: bad arguments");
  usm_blend_kernel<<<grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(img, blur, soft, weight, n,
                                                                                          out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_lq_levels(const float* x, int64_t n, float* out, void* stream) {
  DBIR_REQUIRE(x && out && n > 0, "dbir_lq_levels: bad arguments");
  lq_levels_kernel<<<grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, n, out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_pair_nhwc(const float* lq, const float* hq, int32_t b, int32_t c, int64_t hw, float* lq_out,
                              float* hq_out, void* stream) {
  DBIR_REQUIRE(lq && hq && lq_out && hq_out && b > 0 && c > 0 && hw > 0, "dbir_pair_nhwc: bad arguments");
  const long long n = static_cast<long long>(b) * c * hw;
  pair_nhwc_kernel<<<grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(lq, hq, c, hw, n, lq_out,
                                                                                          hq_out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}
