// painter_b200 — task metrics on the device (painter_b200/task_metrics.py): the scores the reference computes in Python
// from the eval scripts' PNG files, computed from run_batch's device outputs instead.
//
//  palette decode + confusion matrix   Painter/eval/ade20k_semantic/ADE20kSemSegEvaluatorCustom.py:86-101,114-141 and
//                                      coco_panoptic/COCOPanoSemSegEvaluatorCustom.py (post_process_segm_output, then
//                                      np.bincount((K + 1) * pred + gt))
//  depth errors                        Painter/eval/nyuv2_depth/eval_with_pngs.py:50-71,148-209 (compute_errors on the
//                                      valid, Eigen-cropped pixels of each image)
//  PSNR / SSIM                         Painter/eval/lol/painter_inference_lol.py:163-166 (skimage 0.19's
//                                      peak_signal_noise_ratio / structural_similarity(multichannel=True))
//
// Exactness.  The palette distances of the reference are fp32 sums of integers (or, for 'mean', of halves of the even
// integers |d| + d^2) below 2^24, so they are exact and the integer scores below order the colours identically; argmin
// keeps the first minimum, as torch.argmin does.  The confusion matrix is a sum of integers (uint32 per-CTA bins,
// 64-bit atomics into the result), independent of scheduling.  The depth and restoration kernels compute every
// element-wise term in the reference's precision with explicitly rounded operations (no FMA contraction) and sum the
// terms in fp64 in a fixed order: per thread, a fixed tree per CTA, and the CTAs of an image in index order, so every
// result is bitwise reproducible.  No kernel synchronises with the host.
#include <climits>

#include "host_common.h"
#include "metrics.cuh"

namespace pk {

constexpr int kMaxPalette = 200;

// ------------------------------------------------------------------------------------------------------------------
// Palette decode.  Colours are packed as r | g << 8 | b << 16; nrm[k] = |P_k|^2.  Scores (the reference's fp32 distance
// times one, one and two): abs sum |c - P_k| = SAD; square sum (c - P_k)^2 = |c|^2 - 2 c.P_k + |P_k|^2; mean
// sum (|d| + d^2) = SAD + square.  Strict < keeps the first minimum.
template <int DIST>
__device__ __forceinline__ int palette_class(uint32_t c, int cn, const uint32_t* pal, const int* nrm, int K) {
  int best = INT_MAX, idx = 0;
#pragma unroll 4
  for (int k = 0; k < K; ++k) {
    const uint32_t p = pal[k];
    int s;
    if (DIST == PK_DIST_ABS) {
      s = static_cast<int>(__vsadu4(c, p));
    } else {
      s = cn - 2 * static_cast<int>(__dp4a(c, p, 0u)) + nrm[k];
      if (DIST == PK_DIST_MEAN) s += static_cast<int>(__vsadu4(c, p));
    }
    if (s < best) {
      best = s;
      idx = k;
    }
  }
  return idx;
}

__device__ __forceinline__ uint32_t load_rgb(const uint8_t* px, size_t i, int* cn) {
  const uint32_t r = px[3 * i], g = px[3 * i + 1], b = px[3 * i + 2];
  *cn = static_cast<int>(r * r + g * g + b * b);
  return r | (g << 8) | (b << 16);
}

__device__ __forceinline__ void stage_palette(const uint8_t* palette, int K, uint32_t* pal, int* nrm) {
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const uint32_t r = palette[3 * k], g = palette[3 * k + 1], b = palette[3 * k + 2];
    pal[k] = r | (g << 8) | (b << 16);
    nrm[k] = static_cast<int>(r * r + g * g + b * b);
  }
}

template <int DIST>
__global__ void __launch_bounds__(256)
palette_classes_kernel(const uint8_t* __restrict__ segm, long long npix, const uint8_t* __restrict__ palette, int K,
                       uint8_t* __restrict__ out) {
  __shared__ uint32_t pal[kMaxPalette];
  __shared__ int nrm[kMaxPalette];
  stage_palette(palette, K, pal, nrm);
  __syncthreads();
  for (long long i = blockIdx.x * 256ll + threadIdx.x; i < npix; i += static_cast<long long>(gridDim.x) * 256) {
    int cn;
    const uint32_t c = load_rgb(segm, static_cast<size_t>(i), &cn);
    out[i] = static_cast<uint8_t>(palette_class<DIST>(c, cn, pal, nrm, K));
  }
}

// Confusion matrix: CTA (x, image) decodes a grid-stride share of the image's pixels and counts cell (K+1) * pred + gt
// (gt = K for the ignore label) in uint32 shared bins; lanes of a warp that hit the same cell add once.  The bins are
// flushed into the int64 matrix with 64-bit atomics (integer sums: the result does not depend on the order).
constexpr int kConfThreads = 512;
template <int DIST>
__global__ void __launch_bounds__(kConfThreads)
semseg_confusion_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base,
                        const uint8_t* __restrict__ palette, int K, int ignore_label,
                        unsigned long long* __restrict__ conf) {
  extern __shared__ uint32_t smem[];
  uint32_t* pal = smem;
  int* nrm = reinterpret_cast<int*>(smem + K);
  uint32_t* bins = smem + 2 * K;
  const MetricItem it = metric_item(items, base, blockIdx.y);
  const long long npix = static_cast<long long>(it.H) * it.W;
  const long long first = static_cast<long long>(blockIdx.x) * kConfThreads;
  if (first >= npix) return;                       // uniform over the CTA
  const int cells = (K + 1) * (K + 1);
  stage_palette(palette, K, pal, nrm);
  for (int c = threadIdx.x; c < cells; c += kConfThreads) bins[c] = 0;
  __syncthreads();
  const uint8_t* px = static_cast<const uint8_t*>(it.pred);
  const uint8_t* gt = static_cast<const uint8_t*>(it.gt);
  const long long stride = static_cast<long long>(gridDim.x) * kConfThreads;
  for (long long b0 = first; b0 < npix; b0 += stride) {          // b0 is warp-uniform: every lane takes part
    const long long i = b0 + threadIdx.x;
    int cell = -1;
    if (i < npix) {
      int cn;
      const uint32_t c = load_rgb(px, static_cast<size_t>(i), &cn);
      const int pred = palette_class<DIST>(c, cn, pal, nrm, K);
      const int g = gt[i];
      const int gc = g == ignore_label ? K : (g < K ? g : K);   // labels >= K are refused on the host
      cell = (K + 1) * pred + gc;
    }
    const unsigned peers = __match_any_sync(0xffffffffu, cell);
    if (cell >= 0 && (threadIdx.x & 31) == static_cast<unsigned>(__ffs(peers) - 1))
      atomicAdd(&bins[cell], static_cast<uint32_t>(__popc(peers)));
  }
  __syncthreads();
  for (int c = threadIdx.x; c < cells; c += kConfThreads) {
    const uint32_t v = bins[c];
    if (v) atomicAdd(&conf[c], static_cast<unsigned long long>(v));
  }
}

// ------------------------------------------------------------------------------------------------------------------
// NYUv2 depth: one CTA per image.  pred = float(v) / 1000 clamped into [min, max], gt = float(g) / 1000; on the pixels
// with min < gt < max (and inside rows 45:471, columns 41:601 with the Eigen crop) the fp32 terms of compute_errors,
// summed in fp64.  out[i] = {d1, d2, d3, AbsRel, SqRel, RMSE, RMSElog, SILog, log10}.
constexpr int kDepthThreads = 512;
__global__ void __launch_bounds__(kDepthThreads)
depth_errors_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base, float min_d, float max_d,
                    int eigen_crop, double* __restrict__ out) {
  __shared__ double red[10][kDepthThreads / 32];
  const MetricItem it = metric_item(items, base, blockIdx.x);
  const int* pred = static_cast<const int*>(it.pred);
  const uint16_t* gtv = static_cast<const uint16_t*>(it.gt);
  const int H = it.H, W = it.W;
  const int r0 = eigen_crop ? 45 : 0, r1 = eigen_crop ? min(471, H) : H;
  const int c0 = eigen_crop ? 41 : 0, c1 = eigen_crop ? min(601, W) : W;
  const int cw = c1 - c0;
  const long long n_box = r1 > r0 && cw > 0 ? static_cast<long long>(r1 - r0) * cw : 0;
  // v: count, d1, d2, d3, sum |d|/gt, sum d^2/gt, sum d^2, sum e, sum e^2, sum |log10 p - log10 gt|
  double v[10];
#pragma unroll
  for (int j = 0; j < 10; ++j) v[j] = 0.0;
  int cnt = 0, n1 = 0, n2 = 0, n3 = 0;
  for (long long k = threadIdx.x; k < n_box; k += kDepthThreads) {
    const long long idx = static_cast<long long>(r0 + k / cw) * W + c0 + k % cw;
    const float gt = __fdiv_rn(static_cast<float>(gtv[idx]), 1000.0f);
    if (!(gt > min_d && gt < max_d)) continue;
    float p = __fdiv_rn(static_cast<float>(pred[idx]), 1000.0f);
    if (p < min_d) p = min_d;
    if (p > max_d) p = max_d;
    const float th = fmaxf(__fdiv_rn(gt, p), __fdiv_rn(p, gt));
    ++cnt;
    n1 += th < 1.25f;
    n2 += th < 1.5625f;
    n3 += th < 1.953125f;
    const float d = __fsub_rn(gt, p);
    const float d2 = __fmul_rn(d, d);
    v[4] += __fdiv_rn(fabsf(d), gt);
    v[5] += __fdiv_rn(d2, gt);
    v[6] += d2;
    const float e = __fsub_rn(logf(p), logf(gt));
    v[7] += e;
    v[8] += __fmul_rn(e, e);
    v[9] += fabsf(__fsub_rn(log10f(p), log10f(gt)));
  }
  v[0] = cnt;
  v[1] = n1;
  v[2] = n2;
  v[3] = n3;
  block_sum<10, kDepthThreads>(v, red);
  if (threadIdx.x == 0) {
    const double n = v[0];
    double* o = out + static_cast<size_t>(blockIdx.x) * 9;
    o[0] = v[1] / n;
    o[1] = v[2] / n;
    o[2] = v[3] / n;
    o[3] = v[4] / n;
    o[4] = v[5] / n;
    o[5] = sqrt(v[6] / n);
    o[6] = sqrt(v[8] / n);
    const double me = v[7] / n;
    o[7] = sqrt(v[8] / n - me * me) * 100.0;
    o[8] = v[9] / n;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// PSNR / SSIM.  x = clip(restored, 0, 1) (fp64 [H, W, 3]), y = gt / 255. (uint8 [H, W, 3]).  CTA (tile, image) covers a
// 16 x 16 pixel tile: every pixel adds its squared errors to the MSE sum and, more than 3 pixels from every border,
// its S-map values of the three channels (a 7 x 7 window that never reaches the border, so the reflect padding of the
// reference's filter is never read).  The CTA's four sums go to partials[image][tile]; the image's last CTA to finish
// (counter) adds them in tile order and writes psnr[i], ssim[i].
constexpr int kSsimTile = 16;
constexpr int kSsimThreads = kSsimTile * kSsimTile;

__device__ __forceinline__ double unit_x(const double* x, size_t i) { return fmin(fmax(x[i], 0.0), 1.0); }
__device__ __forceinline__ double unit_y(const uint8_t* y, size_t i) { return static_cast<double>(y[i]) / 255.0; }

__global__ void __launch_bounds__(kSsimThreads)
restoration_scores_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base,
                          unsigned* __restrict__ counters, double* __restrict__ partials, double c1, double c2,
                          double* __restrict__ psnr, double* __restrict__ ssim) {
  __shared__ double red[4][kSsimThreads / 32];
  __shared__ bool last;
  const MetricItem it = metric_item(items, base, blockIdx.y);
  const double* X = static_cast<const double*>(it.pred);
  const uint8_t* Y = static_cast<const uint8_t*>(it.gt);
  const int H = it.H, W = it.W;
  const int tiles_w = (W + kSsimTile - 1) / kSsimTile;
  const int tiles = tiles_w * ((H + kSsimTile - 1) / kSsimTile);
  const int t = blockIdx.x;
  double v[4] = {0.0, 0.0, 0.0, 0.0};
  if (t < tiles) {
    const int r = (t / tiles_w) * kSsimTile + threadIdx.x / kSsimTile;
    const int c = (t % tiles_w) * kSsimTile + threadIdx.x % kSsimTile;
    if (r < H && c < W) {
      const size_t p = (static_cast<size_t>(r) * W + c) * 3;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const double d = __dsub_rn(unit_x(X, p + ch), unit_y(Y, p + ch));
        v[0] += __dmul_rn(d, d);
      }
      if (r >= 3 && r < H - 3 && c >= 3 && c < W - 3) {
        const double cov_norm = 49.0 / 48.0;
#pragma unroll 1
        for (int ch = 0; ch < 3; ++ch) {
          // scipy's uniform_filter: the 7-tap mean along the rows, then along the columns
          double ux = 0.0, uy = 0.0, uxx = 0.0, uyy = 0.0, uxy = 0.0;
#pragma unroll 1
          for (int dc = -3; dc <= 3; ++dc) {
            double sx = 0.0, sy = 0.0, sxx = 0.0, syy = 0.0, sxy = 0.0;
#pragma unroll
            for (int dr = -3; dr <= 3; ++dr) {
              const size_t q = (static_cast<size_t>(r + dr) * W + (c + dc)) * 3 + ch;
              const double a = unit_x(X, q), b = unit_y(Y, q);
              sx += a;
              sy += b;
              sxx += __dmul_rn(a, a);
              syy += __dmul_rn(b, b);
              sxy += __dmul_rn(a, b);
            }
            ux += sx / 7.0;
            uy += sy / 7.0;
            uxx += sxx / 7.0;
            uyy += syy / 7.0;
            uxy += sxy / 7.0;
          }
          ux /= 7.0;
          uy /= 7.0;
          uxx /= 7.0;
          uyy /= 7.0;
          uxy /= 7.0;
          const double vx = __dmul_rn(cov_norm, __dsub_rn(uxx, __dmul_rn(ux, ux)));
          const double vy = __dmul_rn(cov_norm, __dsub_rn(uyy, __dmul_rn(uy, uy)));
          const double vxy = __dmul_rn(cov_norm, __dsub_rn(uxy, __dmul_rn(ux, uy)));
          const double a1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), c1);
          const double a2 = __dadd_rn(__dmul_rn(2.0, vxy), c2);
          const double b1 = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), c1);
          const double b2 = __dadd_rn(__dadd_rn(vx, vy), c2);
          const double sv = __dmul_rn(a1, a2) / __dmul_rn(b1, b2);
          if (ch == 0) v[1] += sv;           // constant indices keep v in registers
          else if (ch == 1) v[2] += sv;
          else v[3] += sv;
        }
      }
    }
  }
  block_sum<4, kSsimThreads>(v, red);
  double* part = partials + (static_cast<size_t>(blockIdx.y) * gridDim.x + t) * 4;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) part[j] = v[j];
    __threadfence();
    last = atomicAdd(&counters[blockIdx.y], 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  const volatile double* all = partials + static_cast<size_t>(blockIdx.y) * gridDim.x * 4;
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int k = 0; k < tiles; ++k) {
#pragma unroll
    for (int j = 0; j < 4; ++j) s[j] += all[k * 4 + j];
  }
  const double mse = s[0] / (3.0 * H * W);
  psnr[blockIdx.y] = 10.0 * log10(1.0 / mse);
  const double n_in = static_cast<double>(H - 6) * (W - 6);
  ssim[blockIdx.y] = (s[1] / n_in + s[2] / n_in + s[3] / n_in) / 3.0;
}

}  // namespace pk

using namespace pk;

extern "C" int pk_palette_classes(const uint8_t* segm, long long npix, const uint8_t* palette, int K, int dist_type,
                                  uint8_t* out, void* stream) {
  PK_CHECK(segm && palette && out && npix > 0, "pk_palette_classes: null pointer or empty image");
  PK_CHECK(K >= 1 && K <= kMaxPalette, "pk_palette_classes: palette size %d outside 1..%d", K, kMaxPalette);
  PK_CHECK(dist_type >= PK_DIST_ABS && dist_type <= PK_DIST_MEAN, "pk_palette_classes: unknown dist_type %d",
           dist_type);
  const long long want = (npix + 255) / 256, cap = static_cast<long long>(sm_count()) * 8;
  const unsigned grid = static_cast<unsigned>(want < cap ? want : cap);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (dist_type == PK_DIST_ABS)
    palette_classes_kernel<PK_DIST_ABS><<<grid, 256, 0, st>>>(segm, npix, palette, K, out);
  else if (dist_type == PK_DIST_SQUARE)
    palette_classes_kernel<PK_DIST_SQUARE><<<grid, 256, 0, st>>>(segm, npix, palette, K, out);
  else
    palette_classes_kernel<PK_DIST_MEAN><<<grid, 256, 0, st>>>(segm, npix, palette, K, out);
  PK_LAUNCH_CHECK("pk_palette_classes");
  return 0;
}

extern "C" int pk_semseg_confusion(const long long* items, const void* base, int n, long long max_pix,
                                   const uint8_t* palette, int K, int dist_type, int ignore_label, long long* conf,
                                   void* stream) {
  PK_CHECK(items && base && palette && conf && n >= 1 && n <= 65535 && max_pix > 0,
           "pk_semseg_confusion: bad arguments (null pointer, n outside 1..65535 or max_pix < 1)");
  PK_CHECK(K >= 1 && K <= kMaxPalette, "pk_semseg_confusion: palette size %d outside 1..%d", K, kMaxPalette);
  PK_CHECK(dist_type >= PK_DIST_ABS && dist_type <= PK_DIST_MEAN, "pk_semseg_confusion: unknown dist_type %d",
           dist_type);
  const size_t smem = (2 * static_cast<size_t>(K) + static_cast<size_t>(K + 1) * (K + 1)) * 4;
  const size_t smem_max = (2 * kMaxPalette + (kMaxPalette + 1) * (kMaxPalette + 1)) * 4;
  static bool attr_set[3] = {false, false, false};   // per process: kernels are shared by every device's context
  void (*kernels[3])(const long long*, const uint8_t*, const uint8_t*, int, int, unsigned long long*) = {
      semseg_confusion_kernel<PK_DIST_ABS>, semseg_confusion_kernel<PK_DIST_SQUARE>,
      semseg_confusion_kernel<PK_DIST_MEAN>};
  if (!attr_set[dist_type]) {
    PK_CHECK(cudaFuncSetAttribute(kernels[dist_type], cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(smem_max)) == cudaSuccess,
             "pk_semseg_confusion: %zu bytes of shared memory not available", smem_max);
    attr_set[dist_type] = true;
  }
  // about 64 pixels per thread: the bins are zeroed and flushed once per CTA
  const long long per_cta = static_cast<long long>(kConfThreads) * 64;
  const dim3 grid(static_cast<unsigned>((max_pix + per_cta - 1) / per_cta), static_cast<unsigned>(n));
  kernels[dist_type]<<<grid, kConfThreads, smem, static_cast<cudaStream_t>(stream)>>>(
      items, static_cast<const uint8_t*>(base), palette, K, ignore_label, reinterpret_cast<unsigned long long*>(conf));
  PK_LAUNCH_CHECK("pk_semseg_confusion");
  return 0;
}

extern "C" int pk_depth_errors(const long long* items, const void* base, int n, float min_depth, float max_depth,
                               int eigen_crop, double* out, void* stream) {
  PK_CHECK(items && base && out && n >= 1, "pk_depth_errors: null pointer or no image");
  PK_CHECK(min_depth < max_depth, "pk_depth_errors: min_depth %g >= max_depth %g", min_depth, max_depth);
  depth_errors_kernel<<<n, kDepthThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      items, static_cast<const uint8_t*>(base), min_depth, max_depth, eigen_crop != 0, out);
  PK_LAUNCH_CHECK("pk_depth_errors");
  return 0;
}

extern "C" long long pk_restoration_ws_doubles(int max_h, int max_w) {
  if (max_h < 1 || max_w < 1) return 0;
  const long long tiles = static_cast<long long>((max_h + kSsimTile - 1) / kSsimTile) * ((max_w + kSsimTile - 1) / kSsimTile);
  return tiles * 4;
}

extern "C" int pk_restoration_scores(const long long* items, const void* base, int n, int max_h, int max_w,
                                     unsigned* counters_zeroed, double* partials, double c1, double c2, double* psnr,
                                     double* ssim, void* stream) {
  PK_CHECK(items && base && counters_zeroed && partials && psnr && ssim && n >= 1 && n <= 65535,
           "pk_restoration_scores: null pointer or n outside 1..65535");
  PK_CHECK(max_h >= 7 && max_w >= 7, "pk_restoration_scores: images must be at least 7 x 7");
  const long long tiles = pk_restoration_ws_doubles(max_h, max_w) / 4;
  PK_CHECK(tiles < (1ll << 31), "pk_restoration_scores: image too large");
  const dim3 grid(static_cast<unsigned>(tiles), static_cast<unsigned>(n));
  restoration_scores_kernel<<<grid, kSsimThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      items, static_cast<const uint8_t*>(base), counters_zeroed, partials, c1, c2, psnr, ssim);
  PK_LAUNCH_CHECK("pk_restoration_scores");
  return 0;
}
