// painter_b200 — the MATLAB scores of Painter's derain and SIDD evaluations on the device (painter_b200/task_metrics.py
// derain_scores, sidd_scores, ycbcr_y), restated from the two scripts and MATLAB's documented algorithms:
//
//  derain  Painter/eval/derain/evaluate_PSNR_SSIM.m on the PNGs painter_inference_derain.py writes: u = uint8(trunc(
//          clip(x, 0, 1) * 255)), the Y channel of rgb2ycbcr, compute_psnr (peak 255) and SSIM_index (11 x 11 Gaussian
//          window, sigma 1.5, 'valid' filtering, C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2, mean of the map)
//  SIDD    Painter/eval/sidd/eval_sidd.m on the Idenoised.mat painter_inference_sidd.py saves: x = single(clip(r, 0, 1)),
//          y = single(g) / 255, psnr (peak 1) and ssim on the H x W x 3 block as a volume (separable Gaussian, sigma
//          1.5, 11 taps, replicate padding, 'same' output; C1 = 0.01^2, C2 = 0.03^2; mean of the H x W x 3 map)
//
// Layout.  CTA (tile, image) covers a 16 x 16 pixel tile.  It fills a 26 x 26 shared halo once (derain: the Y channels
// of rows / columns r0 .. r0 + 25, clamped at the far border, which only the positions outside the 'valid' map would
// read; SIDD: one channel at a time, rows / columns r0 - 5 .. r0 + 20 clamped to the image, which is the replicate
// padding), then filters the five quantities x, y, x^2, y^2, xy as two separable fp64 passes through shared memory.
// SIDD's depth pass on 3 planes with replicate padding is a 3 x 3 matrix M[c][d] (the sum of the taps whose clamped
// source plane is d), applied after the 2-D passes.  The tile's squared-error sum and SSIM-map sum go to
// partials[image][tile]; the image's last CTA (counter) adds them in tile order.  Every element-wise term is an
// explicitly rounded fp64 operation (no FMA contraction) and every sum has a fixed order, so results are bitwise
// reproducible; no kernel synchronises with the host.
#include "host_common.h"
#include "metrics.cuh"

namespace pk {

constexpr int kMTaps = 11;
constexpr int kMRad = kMTaps / 2;
constexpr int kMTile = 16;
constexpr int kMHalo = kMTile + kMTaps - 1;                 // 26
constexpr int kMThreads = kMTile * kMTile;

// MATLAB rgb2ycbcr on uint8, Y only: K1 R + K2 G + K3 B + 16 with Ki = (1/255) * {65.481, 128.553, 24.966}, summed
// left to right, rounded half away from zero (round()) and saturated.  194 of the 2^24 colours are exact ties in
// rationals; their fp64 value, and so Y, depends on this order.
__device__ __forceinline__ uint8_t ycbcr_y(int r, int g, int b) {
  const double inv = 1.0 / 255.0;
  const double k1 = __dmul_rn(inv, 65.481), k2 = __dmul_rn(inv, 128.553), k3 = __dmul_rn(inv, 24.966);
  double v = __dadd_rn(__dmul_rn(k1, static_cast<double>(r)), __dmul_rn(k2, static_cast<double>(g)));
  v = __dadd_rn(v, __dmul_rn(k3, static_cast<double>(b)));
  v = round(__dadd_rn(v, 16.0));
  return static_cast<uint8_t>(fmin(fmax(v, 0.0), 255.0));
}

// The PNG value painter_inference_derain.py writes for one fp64 channel value: trunc(clip(x, 0, 1) * 255).
__device__ __forceinline__ int derain_u8(double x) {
  return static_cast<int>(__dmul_rn(fmin(fmax(x, 0.0), 1.0), 255.0));
}

__global__ void __launch_bounds__(256) ycbcr_y_kernel(const uint8_t* __restrict__ rgb, long long npix,
                                                      uint8_t* __restrict__ out) {
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < npix; i += static_cast<long long>(gridDim.x) * 256)
    out[i] = ycbcr_y(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]);
}

struct GaussSmem {
  double a[kMHalo * kMHalo], b[kMHalo * kMHalo];   // the halo of x and y
  double h[5][kMHalo][kMTile];                     // row pass of x, y, x^2, y^2, xy
  double tap[kMTaps];
  double red[2][kMThreads / 32];
  bool last;
};

// Both passes of the separable filter over the halo in s.a, s.b: f[0..4] = the filtered x, y, x^2, y^2, xy at this
// thread's pixel (row ty, column tx of the tile; halo rows ty .. ty + 10, columns tx .. tx + 10).
__device__ __forceinline__ void gauss_2d(GaussSmem& s, double (&f)[5]) {
  for (int i = threadIdx.x; i < kMHalo * kMTile; i += kMThreads) {
    const int row = i / kMTile, col = i % kMTile;
    double q[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int k = 0; k < kMTaps; ++k) {
      const double t = s.tap[k];
      const double a = s.a[row * kMHalo + col + k], b = s.b[row * kMHalo + col + k];
      q[0] = __dadd_rn(q[0], __dmul_rn(t, a));
      q[1] = __dadd_rn(q[1], __dmul_rn(t, b));
      q[2] = __dadd_rn(q[2], __dmul_rn(t, __dmul_rn(a, a)));
      q[3] = __dadd_rn(q[3], __dmul_rn(t, __dmul_rn(b, b)));
      q[4] = __dadd_rn(q[4], __dmul_rn(t, __dmul_rn(a, b)));
    }
#pragma unroll
    for (int j = 0; j < 5; ++j) s.h[j][row][col] = q[j];
  }
  __syncthreads();
  const int ty = threadIdx.x / kMTile, tx = threadIdx.x % kMTile;
#pragma unroll
  for (int j = 0; j < 5; ++j) f[j] = 0.0;
#pragma unroll
  for (int k = 0; k < kMTaps; ++k) {
    const double t = s.tap[k];
#pragma unroll
    for (int j = 0; j < 5; ++j) f[j] = __dadd_rn(f[j], __dmul_rn(t, s.h[j][ty + k][tx]));
  }
}

// SSIM map value from the filtered means mu_x, mu_y and second moments.
__device__ __forceinline__ double ssim_value(double mx, double my, double mxx, double myy, double mxy, double c1,
                                             double c2) {
  const double mx2 = __dmul_rn(mx, mx), my2 = __dmul_rn(my, my), mxmy = __dmul_rn(mx, my);
  const double sx = __dsub_rn(mxx, mx2), sy = __dsub_rn(myy, my2), sxy = __dsub_rn(mxy, mxmy);
  const double num = __dmul_rn(__dadd_rn(__dmul_rn(2.0, mxmy), c1), __dadd_rn(__dmul_rn(2.0, sxy), c2));
  const double den = __dmul_rn(__dadd_rn(__dadd_rn(mx2, my2), c1), __dadd_rn(__dadd_rn(sx, sy), c2));
  return __ddiv_rn(num, den);
}

// The tile's two sums to partials[image][tile]; true in thread 0 of the image's last CTA, with s[] the image's sums
// over its tiles in tile order.  INT_SSE: the first sum is an integer in every tile (exact in fp64) and is added in
// int64, so the image's total is exact as well.
template <bool INT_SSE>
__device__ __forceinline__ bool finish_tiles(GaussSmem& sm, double (&v)[2], unsigned* counters, double* partials,
                                             int tiles, double (&s)[2]) {
  block_sum<2, kMThreads>(v, sm.red);
  double* part = partials + (static_cast<size_t>(blockIdx.y) * gridDim.x + blockIdx.x) * 2;
  if (threadIdx.x == 0) {
    part[0] = v[0];
    part[1] = v[1];
    __threadfence();
    sm.last = atomicAdd(&counters[blockIdx.y], 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!sm.last || threadIdx.x != 0) return false;
  __threadfence();
  const volatile double* all = partials + static_cast<size_t>(blockIdx.y) * gridDim.x * 2;
  long long e = 0;
  s[0] = s[1] = 0.0;
  for (int k = 0; k < tiles; ++k) {
    if (INT_SSE) e += static_cast<long long>(all[2 * k]);
    else s[0] += all[2 * k];
    s[1] += all[2 * k + 1];
  }
  if (INT_SSE) s[0] = static_cast<double>(e);     // below 2^53: 65025 H W
  return true;
}

// Derain.  Tiles cover the H x W image: every pixel adds (Yp - Yg)^2 to the squared-error sum (an integer, exact in the
// tile's fp64 sum and added across tiles in int64), and the SSIM window whose top-left corner it is, when that window
// lies inside the image (the (H - 10) x (W - 10) 'valid' map), adds its map value.
__global__ void __launch_bounds__(kMThreads)
derain_scores_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base,
                     const double* __restrict__ taps, unsigned* __restrict__ counters, double* __restrict__ partials,
                     double c1, double c2, double* __restrict__ psnr, double* __restrict__ ssim) {
  __shared__ GaussSmem sm;
  const MetricItem it = metric_item(items, base, blockIdx.y);
  const double* X = static_cast<const double*>(it.pred);
  const uint8_t* G = static_cast<const uint8_t*>(it.gt);
  const int H = it.H, W = it.W;
  const int tiles_w = (W + kMTile - 1) / kMTile;
  const int tiles = tiles_w * ((H + kMTile - 1) / kMTile);
  const int t = blockIdx.x;
  double v[2] = {0.0, 0.0};
  if (t < tiles) {                                  // uniform over the CTA
    const int r0 = (t / tiles_w) * kMTile, c0 = (t % tiles_w) * kMTile;
    if (threadIdx.x < kMTaps) sm.tap[threadIdx.x] = taps[threadIdx.x];
    for (int i = threadIdx.x; i < kMHalo * kMHalo; i += kMThreads) {
      const int r = min(r0 + i / kMHalo, H - 1), c = min(c0 + i % kMHalo, W - 1);
      const size_t p = (static_cast<size_t>(r) * W + c) * 3;
      sm.a[i] = ycbcr_y(derain_u8(X[p]), derain_u8(X[p + 1]), derain_u8(X[p + 2]));
      sm.b[i] = ycbcr_y(G[p], G[p + 1], G[p + 2]);
    }
    __syncthreads();
    const int ty = threadIdx.x / kMTile, tx = threadIdx.x % kMTile;
    const int r = r0 + ty, c = c0 + tx;
    if (r < H && c < W) {
      const double d = sm.a[ty * kMHalo + tx] - sm.b[ty * kMHalo + tx];
      v[0] = d * d;                                 // exact: |d| <= 255
    }
    double f[5];
    gauss_2d(sm, f);
    if (r < H - 2 * kMRad && c < W - 2 * kMRad) v[1] = ssim_value(f[0], f[1], f[2], f[3], f[4], c1, c2);
  }
  double s[2];
  if (!finish_tiles<true>(sm, v, counters, partials, tiles, s)) return;
  const double rmse = sqrt(s[0] / (static_cast<double>(H) * W));
  psnr[blockIdx.y] = 20.0 * log10(255.0 / rmse);
  ssim[blockIdx.y] = s[1] / (static_cast<double>(H - 2 * kMRad) * (W - 2 * kMRad));
}

// SIDD.  Tiles cover the H x W image with 'same' output: every pixel adds its three squared errors and its three SSIM
// map values.  consts: the kMTaps taps, then the 3 x 3 depth matrix (row c: output plane c).
__global__ void __launch_bounds__(kMThreads)
sidd_scores_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base,
                   const double* __restrict__ consts, unsigned* __restrict__ counters, double* __restrict__ partials,
                   double c1, double c2, double* __restrict__ psnr, double* __restrict__ ssim) {
  __shared__ GaussSmem sm;
  const MetricItem it = metric_item(items, base, blockIdx.y);
  const double* X = static_cast<const double*>(it.pred);
  const uint8_t* G = static_cast<const uint8_t*>(it.gt);
  const int H = it.H, W = it.W;
  const int tiles_w = (W + kMTile - 1) / kMTile;
  const int tiles = tiles_w * ((H + kMTile - 1) / kMTile);
  const int t = blockIdx.x;
  double v[2] = {0.0, 0.0};
  if (t < tiles) {                                  // uniform over the CTA
    const int r0 = (t / tiles_w) * kMTile, c0 = (t % tiles_w) * kMTile;
    const int ty = threadIdx.x / kMTile, tx = threadIdx.x % kMTile;
    const bool inside = r0 + ty < H && c0 + tx < W;
    if (threadIdx.x < kMTaps) sm.tap[threadIdx.x] = consts[threadIdx.x];
    double f[3][5];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      if (ch) __syncthreads();                      // the previous channel's passes are done with the halo
      for (int i = threadIdx.x; i < kMHalo * kMHalo; i += kMThreads) {
        const int r = min(max(r0 - kMRad + i / kMHalo, 0), H - 1);
        const int c = min(max(c0 - kMRad + i % kMHalo, 0), W - 1);
        const size_t p = (static_cast<size_t>(r) * W + c) * 3 + ch;
        sm.a[i] = static_cast<double>(__double2float_rn(fmin(fmax(X[p], 0.0), 1.0)));
        sm.b[i] = static_cast<double>(__fdiv_rn(static_cast<float>(G[p]), 255.0f));
      }
      __syncthreads();
      if (inside) {
        const int q = (ty + kMRad) * kMHalo + tx + kMRad;
        const double d = __dsub_rn(sm.a[q], sm.b[q]);
        v[0] = __dadd_rn(v[0], __dmul_rn(d, d));
      }
      gauss_2d(sm, f[ch]);
    }
    if (inside) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        double m[5];
#pragma unroll
        for (int j = 0; j < 5; ++j) {
          m[j] = __dmul_rn(consts[kMTaps + 3 * c], f[0][j]);
          m[j] = __dadd_rn(m[j], __dmul_rn(consts[kMTaps + 3 * c + 1], f[1][j]));
          m[j] = __dadd_rn(m[j], __dmul_rn(consts[kMTaps + 3 * c + 2], f[2][j]));
        }
        v[1] = __dadd_rn(v[1], ssim_value(m[0], m[1], m[2], m[3], m[4], c1, c2));
      }
    }
  }
  double s[2];
  if (!finish_tiles<false>(sm, v, counters, partials, tiles, s)) return;
  const double n = 3.0 * H * W;
  psnr[blockIdx.y] = 10.0 * log10(1.0 / (s[0] / n));
  ssim[blockIdx.y] = s[1] / n;
}

}  // namespace pk

using namespace pk;

extern "C" int pk_ycbcr_y(const uint8_t* rgb, long long npix, uint8_t* out, void* stream) {
  PK_CHECK(rgb && out && npix > 0, "pk_ycbcr_y: null pointer or empty image");
  const long long want = (npix + 255) / 256, cap = static_cast<long long>(sm_count()) * 8;
  const unsigned grid = static_cast<unsigned>(want < cap ? want : cap);
  ycbcr_y_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(rgb, npix, out);
  PK_LAUNCH_CHECK("pk_ycbcr_y");
  return 0;
}

static long long matlab_tiles(int max_h, int max_w) {
  if (max_h < 1 || max_w < 1) return 0;
  return static_cast<long long>((max_h + kMTile - 1) / kMTile) * ((max_w + kMTile - 1) / kMTile);
}

extern "C" long long pk_derain_ws_doubles(int max_h, int max_w) { return matlab_tiles(max_h, max_w) * 2; }
extern "C" long long pk_sidd_ws_doubles(int max_h, int max_w) { return matlab_tiles(max_h, max_w) * 2; }

extern "C" int pk_derain_scores(const long long* items, const void* base, int n, int max_h, int max_w,
                                const double* taps, unsigned* counters_zeroed, double* partials, double c1, double c2,
                                double* psnr, double* ssim, void* stream) {
  PK_CHECK(items && base && taps && counters_zeroed && partials && psnr && ssim && n >= 1 && n <= 65535,
           "pk_derain_scores: null pointer or n outside 1..65535");
  PK_CHECK(max_h >= kMTaps && max_w >= kMTaps, "pk_derain_scores: images must be at least 11 x 11");
  const long long tiles = matlab_tiles(max_h, max_w);
  PK_CHECK(tiles < (1ll << 31), "pk_derain_scores: image too large");
  const dim3 grid(static_cast<unsigned>(tiles), static_cast<unsigned>(n));
  derain_scores_kernel<<<grid, kMThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      items, static_cast<const uint8_t*>(base), taps, counters_zeroed, partials, c1, c2, psnr, ssim);
  PK_LAUNCH_CHECK("pk_derain_scores");
  return 0;
}

extern "C" int pk_sidd_scores(const long long* items, const void* base, int n, int max_h, int max_w,
                              const double* consts, unsigned* counters_zeroed, double* partials, double c1, double c2,
                              double* psnr, double* ssim, void* stream) {
  PK_CHECK(items && base && consts && counters_zeroed && partials && psnr && ssim && n >= 1 && n <= 65535,
           "pk_sidd_scores: null pointer or n outside 1..65535");
  const long long tiles = matlab_tiles(max_h, max_w);
  PK_CHECK(tiles >= 1 && tiles < (1ll << 31), "pk_sidd_scores: empty or too large image");
  const dim3 grid(static_cast<unsigned>(tiles), static_cast<unsigned>(n));
  sidd_scores_kernel<<<grid, kMThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      items, static_cast<const uint8_t*>(base), consts, counters_zeroed, partials, c1, c2, psnr, ssim);
  PK_LAUNCH_CHECK("pk_sidd_scores");
  return 0;
}
