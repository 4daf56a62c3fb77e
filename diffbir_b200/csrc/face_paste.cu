// Face paste-back of the unaligned-face loop (FaceRestoreHelper.paste_faces_to_input_image, reference
// utils/face.py) on sm_90a, byte-identical to the host cv2 / numpy recipe:
//
//   paste_square      cv2.warpAffine(ones(512, 512) f32, inv, (w, h)) then cv2.erode(2x2), and its fp64 sum
//   paste_soft        cv2.erode((2e)x(2e)) then cv2.GaussianBlur(2e+1, sigma 0) of the square (f32)
//   paste_parse_blur  two cv2.GaussianBlur((101, 101), 11) of the fp64 parse mask, its 10-pixel frame zeroed, / 255
//   paste_compose     cv2.warpAffine of the restored face (u8) and of the parse mask (f64, flags=3 = bilinear),
//                     square * face (f32), min(pm, soft) and out = mask * pasted + (1 - mask) * out (f64)
//   paste_begin/_end  the fp64 frame from the u8 background, and its astype(uint8) truncation
//
// Each per-face kernel covers a region of interest (ROI) of the frame, a rectangle (x0, y0, rw, rh) that holds
// every pixel where the face's square, soft mask or warped parse mask can be non-zero; outside it those images are
// exactly 0, so the ROI buffers read 0 there. Borders are always those of the full frame (h, w).
//
// cv2 recipes (OpenCV 4.13 with its AVX2 / AVX-512 dispatch, as pinned by tests/test_face_paste.py):
//  - warpAffine inverts the 2x3 map in double (host side here), then per destination pixel computes
//    X = (round((m1*y + m2) * 1024) + 16 + round(m0*x*1024)) >> 5 (and Y alike): 1/32-pixel positions. The
//    bilinear weights of fraction (fy, fx) are (32-fy)(32-fx)/1024 etc., exact in float; u8 uses them times 32768
//    with a +2^14 >> 15 rounding; f32 and f64 sum w00, w01, w10, w11 products in that order, unfused. Taps
//    outside the source read 0.
//  - erode with a k x k rectangle takes the minimum over [y - k/2, y + k - 1 - k/2] (same in x); taps outside
//    the frame are skipped. An empty kernel is the 3 x 3 rectangle.
//  - GaussianBlur is separable with reflect-101 borders. Row pass: s = k0*x0, then s = fma(k_j, x_j, s) in tap
//    order. Column pass: s = k_r * x_c, then for i = 1..r, s += k_{r+i} * (x_{c-i} + x_{c+i}), fused (fma) for
//    f32 columns below 8 * (w / 8) (cv2's 8-wide vector loop) and unfused for the f32 columns of the 4-wide
//    loop behind it and for f64. Frames whose width is not a multiple of 4 have scalar tail columns whose order
//    is not restated here; the host refuses them before launching.
// Every rounding step is an explicit intrinsic, so nvcc contraction cannot change the order.
#include "common.cuh"
#include "../../include/diffbir_b200.h"

namespace {

struct Map {
  double m[6];  // the destination -> source map (cv2's inverted warpAffine matrix)
};

struct Roi {
  int x0, y0, rw, rh;
};

__device__ __forceinline__ void src_pos(const Map& mp, int x, int y, int& X, int& Y) {
  const int adx = __double2int_rn(__dmul_rn(__dmul_rn(mp.m[0], static_cast<double>(x)), 1024.0));
  const int ady = __double2int_rn(__dmul_rn(__dmul_rn(mp.m[3], static_cast<double>(x)), 1024.0));
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(mp.m[1], static_cast<double>(y)), mp.m[2]), 1024.0));
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(mp.m[4], static_cast<double>(y)), mp.m[5]), 1024.0));
  X = (X0 + 16 + adx) >> 5;
  Y = (Y0 + 16 + ady) >> 5;
}

// The four bilinear weights (in 1/1024) of fractions fy, fx in 1/32: w00, w01, w10, w11.
__device__ __forceinline__ void weights(int fy, int fx, int w[4]) {
  w[0] = (32 - fy) * (32 - fx);
  w[1] = (32 - fy) * fx;
  w[2] = fy * (32 - fx);
  w[3] = fy * fx;
}

__device__ __forceinline__ bool inside(int y, int x, int n) { return y >= 0 && y < n && x >= 0 && x < n; }

__device__ __forceinline__ float warp_ones(const Map& mp, int x, int y, int fs) {
  int X, Y, w[4];
  src_pos(mp, x, y, X, Y);
  const int ix = X >> 5, iy = Y >> 5;
  weights(Y & 31, X & 31, w);
  const float p[4] = {inside(iy, ix, fs) ? 1.f : 0.f, inside(iy, ix + 1, fs) ? 1.f : 0.f,
                      inside(iy + 1, ix, fs) ? 1.f : 0.f, inside(iy + 1, ix + 1, fs) ? 1.f : 0.f};
  float s = __fmul_rn(p[0], w[0] * (1.f / 1024.f));
#pragma unroll
  for (int k = 1; k < 4; ++k) s = __fadd_rn(s, __fmul_rn(p[k], w[k] * (1.f / 1024.f)));
  return s;
}

__device__ __forceinline__ int reflect101(int i, int n) {
  i = i < 0 ? -i : i;
  return i >= n ? 2 * (n - 1) - i : i;
}

// ---------------------------------------------------------------------------------------------
// square: 2x2 erode (anchor 1: the window is [y-1, y] x [x-1, x]) of the warped ones, recomputed per tap; the fp64
// sum of the ROI goes to *sum (one atomic per CTA).
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
square_kernel(Map mp, int fs, int h, int w, Roi r, float* __restrict__ square, double* __restrict__ sum) {
  __shared__ double part[8];
  const int rx = blockIdx.x * 32 + threadIdx.x, ry = blockIdx.y * 8 + threadIdx.y;
  double v = 0.0;
  if (rx < r.rw && ry < r.rh) {
    const int x = r.x0 + rx, y = r.y0 + ry;
    float m = INFINITY;
    for (int yy = y - 1; yy <= y; ++yy)
      for (int xx = x - 1; xx <= x; ++xx)
        if (yy >= 0 && xx >= 0) m = fminf(m, warp_ones(mp, xx, yy, fs));
    square[static_cast<long long>(ry) * r.rw + rx] = m;
    v = m;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (threadIdx.x == 0) part[threadIdx.y] = v;
  __syncthreads();
  if (threadIdx.x == 0 && threadIdx.y == 0) {
    double t = 0.0;
    for (int i = 0; i < 8; ++i) t += part[i];
    atomicAdd(sum, t);
  }
}

// ---------------------------------------------------------------------------------------------
// Separable passes over ROI buffers [batch][rh][rw]; `dir` 0 runs along x, 1 along y. A tap outside the ROI but
// inside the frame reads 0 (the image is 0 there).
// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T roi_at(const T* p, const Roi& r, int y, int x) {
  const int ry = y - r.y0, rx = x - r.x0;
  return (ry >= 0 && ry < r.rh && rx >= 0 && rx < r.rw) ? p[static_cast<long long>(ry) * r.rw + rx] : T(0);
}

// erode with the window [c + lo, c + hi] along `dir`; taps outside the frame are skipped
__global__ void __launch_bounds__(256)
erode_kernel(const float* __restrict__ in, int h, int w, Roi r, int lo, int hi, int dir, float* __restrict__ out) {
  const int rx = blockIdx.x * 32 + threadIdx.x, ry = blockIdx.y * 8 + threadIdx.y;
  if (rx >= r.rw || ry >= r.rh) return;
  const int x = r.x0 + rx, y = r.y0 + ry, n = dir ? h : w, c = dir ? y : x;
  float m = INFINITY;
  for (int t = max(c + lo, 0); t <= min(c + hi, n - 1); ++t) m = fminf(m, dir ? roi_at(in, r, t, x) : roi_at(in, r, y, t));
  out[static_cast<long long>(ry) * r.rw + rx] = m;
}

__device__ __forceinline__ float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ double fma_rn(double a, double b, double c) { return __fma_rn(a, b, c); }
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add_rn(double a, double b) { return __dadd_rn(a, b); }

// Row pass of GaussianBlur: s = k0 * x(c - r), then s = fma(k_j, x(c - r + j), s). Tin is the source element
// (u8 parse masks are read as their fp64 values). Batched over blockIdx.z with a per-item stride of rh * rw.
template <typename Tin, typename T>
__global__ void __launch_bounds__(256)
blur_rows_kernel(const Tin* __restrict__ in, int w, Roi r, const T* __restrict__ taps, int k, T* __restrict__ out) {
  const int rx = blockIdx.x * 32 + threadIdx.x, ry = blockIdx.y * 8 + threadIdx.y;
  if (rx >= r.rw || ry >= r.rh) return;
  const long long plane = static_cast<long long>(blockIdx.z) * r.rh * r.rw;
  const Tin* src = in + plane;
  const int x = r.x0 + rx, y = r.y0 + ry, rad = k / 2;
  T s = mul_rn(taps[0], static_cast<T>(roi_at(src, r, y, reflect101(x - rad, w))));
  for (int j = 1; j < k; ++j) s = fma_rn(taps[j], static_cast<T>(roi_at(src, r, y, reflect101(x - rad + j, w))), s);
  out[plane + static_cast<long long>(ry) * r.rw + rx] = s;
}

// Column pass: s = k_r * x(c), then s += k_{r+i} * (x(c - i) + x(c + i)), fused for columns x < fused_below.
// finish = 1 (the parse mask's last pass): the 10-pixel frame of the image is zeroed and the rest divided by 255.
template <typename T>
__global__ void __launch_bounds__(256)
blur_cols_kernel(const T* __restrict__ in, int h, int w, Roi r, const T* __restrict__ taps, int k, int fused_below,
                 int finish, T* __restrict__ out) {
  const int rx = blockIdx.x * 32 + threadIdx.x, ry = blockIdx.y * 8 + threadIdx.y;
  if (rx >= r.rw || ry >= r.rh) return;
  const long long plane = static_cast<long long>(blockIdx.z) * r.rh * r.rw;
  const T* src = in + plane;
  const int x = r.x0 + rx, y = r.y0 + ry, rad = k / 2;
  const bool fused = x < fused_below;
  T s = mul_rn(taps[rad], roi_at(src, r, y, x));
  for (int i = 1; i <= rad; ++i) {
    const T ab = add_rn(roi_at(src, r, reflect101(y - i, h), x), roi_at(src, r, reflect101(y + i, h), x));
    s = fused ? fma_rn(taps[rad + i], ab, s) : add_rn(s, mul_rn(taps[rad + i], ab));
  }
  if (finish) s = (y < 10 || y >= h - 10 || x < 10 || x >= w - 10) ? T(0) : static_cast<T>(__ddiv_rn(s, 255.0));
  out[plane + static_cast<long long>(ry) * r.rw + rx] = s;
}

// ---------------------------------------------------------------------------------------------
// compose: one thread per ROI pixel of sample blockIdx.z.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
compose_kernel(const uint8_t* __restrict__ faces, long long face_stride, const double* __restrict__ pms,
               long long pm_stride, const float* __restrict__ square, const float* __restrict__ soft, Map mp, int fs,
               int h, int w, Roi r, double* __restrict__ out) {
  const int rx = blockIdx.x * 32 + threadIdx.x, ry = blockIdx.y * 8 + threadIdx.y;
  if (rx >= r.rw || ry >= r.rh) return;
  const uint8_t* face = faces + blockIdx.z * face_stride;
  const double* pm = pms + blockIdx.z * pm_stride;
  const int x = r.x0 + rx, y = r.y0 + ry;
  int X, Y, wt[4];
  src_pos(mp, x, y, X, Y);
  const int ix = X >> 5, iy = Y >> 5;
  weights(Y & 31, X & 31, wt);
  const int ty[4] = {iy, iy, iy + 1, iy + 1}, tx[4] = {ix, ix + 1, ix, ix + 1};
  bool in[4];
#pragma unroll
  for (int t = 0; t < 4; ++t) in[t] = inside(ty[t], tx[t], fs);
  // the parse mask: fp64 taps, float weights, unfused sum in tap order
  double pmv = 0.0;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const double p = in[t] ? pm[static_cast<long long>(ty[t]) * fs + tx[t]] : 0.0;
    const double term = __dmul_rn(p, static_cast<double>(wt[t] * (1.f / 1024.f)));
    pmv = t == 0 ? term : __dadd_rn(pmv, term);
  }
  const long long ri = static_cast<long long>(ry) * r.rw + rx;
  const float sq = square[ri], sf = soft[ri];
  const double mask = pmv < static_cast<double>(sf) ? pmv : static_cast<double>(sf);
  const double keep = __dsub_rn(1.0, mask);
  double* o = out + (static_cast<long long>(blockIdx.z) * h * w + static_cast<long long>(y) * w + x) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    int acc = 0;
#pragma unroll
    for (int t = 0; t < 4; ++t)
      if (in[t]) acc += face[(static_cast<long long>(ty[t]) * fs + tx[t]) * 3 + c] * (wt[t] << 5);
    const int fc = min((acc + (1 << 14)) >> 15, 255);
    const float pasted = __fmul_rn(sq, static_cast<float>(fc));
    o[c] = __dadd_rn(__dmul_rn(mask, static_cast<double>(pasted)), __dmul_rn(keep, o[c]));
  }
}

__global__ void begin_kernel(const uint8_t* __restrict__ img, long long n, double* __restrict__ out) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    out[i] = img[i];
}

__global__ void end_kernel(const double* __restrict__ in, long long n, uint8_t* __restrict__ img) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    img[i] = static_cast<uint8_t>(__double2int_rz(in[i]));
}

int grid_for(long long n, int threads) {
  const long long cap = static_cast<long long>(dbir_sm_count()) * 16;
  long long g = (n + threads - 1) / threads;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

dim3 roi_grid(const Roi& r, int batch) { return dim3((r.rw + 31) / 32, (r.rh + 7) / 8, batch); }

bool roi_ok(const Roi& r, int h, int w) {
  return r.rw > 0 && r.rh > 0 && r.x0 >= 0 && r.y0 >= 0 && r.x0 + r.rw <= w && r.y0 + r.rh <= h &&
         (r.rh + 7) / 8 <= 65535;
}

Map load_map(const double* m) {
  Map mp;
  for (int i = 0; i < 6; ++i) mp.m[i] = m[i];
  return mp;
}

}  // namespace

extern "C" int dbir_paste_square(const double* map, int32_t face_size, int32_t h, int32_t w, int32_t x0, int32_t y0,
                                 int32_t rw, int32_t rh, float* square, double* sum, void* stream) {
  const Roi r{x0, y0, rw, rh};
  DBIR_REQUIRE(map && square && sum && face_size > 0 && roi_ok(r, h, w), "dbir_paste_square: bad arguments");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DBIR_CHECK_CUDA(cudaMemsetAsync(sum, 0, sizeof(double), st));
  square_kernel<<<roi_grid(r, 1), dim3(32, 8), 0, st>>>(load_map(map), face_size, h, w, r, square, sum);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_paste_soft(const float* square, int32_t h, int32_t w, int32_t x0, int32_t y0, int32_t rw,
                               int32_t rh, int32_t edge, const float* taps, float* tmp, float* soft, void* stream) {
  const Roi r{x0, y0, rw, rh};
  DBIR_REQUIRE(square && tmp && soft && square != soft && roi_ok(r, h, w) && edge >= 0,
               "dbir_paste_soft: bad arguments");
  DBIR_REQUIRE(edge == 0 || edge >= 3, "dbir_paste_soft: edge 1 and 2 (3- and 5-tap blurs) are not restated");
  DBIR_REQUIRE(w % 4 == 0, "dbir_paste_soft: the frame width must be a multiple of 4");
  DBIR_REQUIRE(edge == 0 || (taps && 2 * edge < w && 2 * edge < h), "dbir_paste_soft: bad blur");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const dim3 g = roi_grid(r, 1), b(32, 8);
  // cv2.erode with (2e)x(2e) ones: anchor e, window [-e, e-1]; edge 0 is the empty kernel, i.e. 3x3 ([-1, 1])
  const int lo = edge ? -edge : -1, hi = edge ? edge - 1 : 1;
  erode_kernel<<<g, b, 0, st>>>(square, h, w, r, lo, hi, 0, tmp);
  erode_kernel<<<g, b, 0, st>>>(tmp, h, w, r, lo, hi, 1, soft);
  if (edge > 0) {     // a 1-tap GaussianBlur is the identity
    const int k = 2 * edge + 1;
    blur_rows_kernel<float, float><<<g, b, 0, st>>>(soft, w, r, taps, k, tmp);
    blur_cols_kernel<float><<<g, b, 0, st>>>(tmp, h, w, r, taps, k, w / 8 * 8, 0, soft);
  }
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_paste_parse_blur(const uint8_t* masks, int32_t n, int32_t size, const double* taps, int32_t k,
                                     double* tmp, double* out, void* stream) {
  DBIR_REQUIRE(masks && taps && tmp && out && tmp != out && n > 0 && n <= 65535 && k % 2 == 1 && k / 2 < size &&
                   size > 20,
               "dbir_paste_parse_blur: bad arguments");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const Roi r{0, 0, size, size};
  const dim3 g = roi_grid(r, n), b(32, 8);
  blur_rows_kernel<uint8_t, double><<<g, b, 0, st>>>(masks, size, r, taps, k, tmp);
  blur_cols_kernel<double><<<g, b, 0, st>>>(tmp, size, size, r, taps, k, 0, 0, out);
  blur_rows_kernel<double, double><<<g, b, 0, st>>>(out, size, r, taps, k, tmp);
  blur_cols_kernel<double><<<g, b, 0, st>>>(tmp, size, size, r, taps, k, 0, 1, out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_paste_compose(const uint8_t* faces, int64_t face_stride, const double* pms, int64_t pm_stride,
                                  int32_t samples, const float* square, const float* soft, const double* map,
                                  int32_t face_size, int32_t h, int32_t w, int32_t x0, int32_t y0, int32_t rw,
                                  int32_t rh, double* out, void* stream) {
  const Roi r{x0, y0, rw, rh};
  DBIR_REQUIRE(faces && pms && square && soft && map && out && samples > 0 && samples <= 65535 && face_size > 0 &&
                   roi_ok(r, h, w),
               "dbir_paste_compose: bad arguments");
  compose_kernel<<<roi_grid(r, samples), dim3(32, 8), 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      faces, face_stride, pms, pm_stride, square, soft, load_map(map), face_size, h, w, r, out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_paste_begin(const uint8_t* img, int64_t n, double* out, void* stream) {
  DBIR_REQUIRE(img && out && n > 0, "dbir_paste_begin: bad arguments");
  begin_kernel<<<grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(img, n, out);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int dbir_paste_end(const double* in, int64_t n, uint8_t* img, void* stream) {
  DBIR_REQUIRE(in && img && n > 0, "dbir_paste_end: bad arguments");
  end_kernel<<<grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(in, n, img);
  DBIR_CHECK_CUDA(cudaGetLastError());
  return 0;
}
