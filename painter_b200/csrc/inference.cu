// painter_b200 — device-side pre/post-processing of the inference wrappers (SURVEY §8 f.2): everything the reference
// does in numpy / PIL-free torch around the forward of seggpt_engine.inference_image / inference_video
// (SegGPT/SegGPT_inference/seggpt_engine.py:56-181) and of the Painter eval scripts' run_one_image
// (Painter/eval/{ade20k_semantic, coco_panoptic, mmpose_custom, nyuv2_depth, sidd, lol, derain}/painter_inference_*.py),
// so that a frame costs one small H2D copy, the forward, and one D2H copy of the finished image (uint8 / int32 PNG,
// or the float64 restoration result).
//
// The reference does this arithmetic in float64 (numpy broadcasting of the float64 mean/std arrays, torch-CPU
// F.interpolate on the float64 tensor); the kernels below keep float64 wherever the reference result is consumed as
// float64, so results are bit-comparable.  Where torch-CPU's compiled kernels contract a multiply and an add into one
// fused multiply-add the kernels say so with __fma_rn; everything else is an explicitly rounded __dmul_rn / __dadd_rn.
// All kernels are HBM-bound streaming passes over <= a few MB on the caller's stream (graph-capturable).
#include "common.cuh"
#include "host_common.h"
#include "../../include/painter_b200.h"

namespace pk {

__constant__ double c_mean[3] = {0.485, 0.456, 0.406};
__constant__ double c_std[3] = {0.229, 0.224, 0.225};

// Source pixel in [0, 1] as a double: uint8 / 255. (np.array(PIL) / 255.), float32 or float64 as stored.
__device__ __forceinline__ double load_unit(const void* src, int dtype, size_t idx) {
  if (dtype == 0) return static_cast<double>(static_cast<const uint8_t*>(src)[idx]) / 255.0;
  if (dtype == 1) return static_cast<double>(static_cast<const float*>(src)[idx]);
  return static_cast<const double*>(src)[idx];
}

// canvas[p, c, y, x] (fp32 NCHW, [P, 3, 2S, S]) = ((y < S ? top[p] : bottom[p])[y % S, x, c] - mean[c]) / std[c]
// top / bottom: per-member pointers to HWC images [S, S, 3] in [0,1] (or uint8); seggpt_engine.py:75-91 (stitch,
// normalise), :29-34 (nhwc -> nchw, .float()).
constexpr int kCanvasMembers = 16;
struct CanvasSrc {
  const void* top[kCanvasMembers];
  const void* bottom[kCanvasMembers];
  int top_dtype[kCanvasMembers];
  int bottom_dtype[kCanvasMembers];
};
__global__ void __launch_bounds__(256)
stitch_normalize_kernel(const CanvasSrc src, float* __restrict__ out, int P, int S) {
  const size_t total = static_cast<size_t>(P) * 3 * 2 * S * S;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % S);
    size_t r = i / S;
    const int y = static_cast<int>(r % (2 * S));
    r /= (2 * S);
    const int c = static_cast<int>(r % 3), p = static_cast<int>(r / 3);
    const bool is_top = y < S;
    const int yy = is_top ? y : y - S;
    const size_t sidx = (static_cast<size_t>(yy) * S + x) * 3 + c;
    const double v = is_top ? load_unit(src.top[p], src.top_dtype[p], sidx)
                            : load_unit(src.bottom[p], src.bottom_dtype[p], sidx);
    out[i] = static_cast<float>(__dsub_rn(v, c_mean[c]) / c_std[c]);
  }
}

// nhwc (fp64 or fp32, already normalised) -> nchw fp32: torch.einsum('nhwc->nchw', x).float() (seggpt_engine.py:29-34)
__global__ void __launch_bounds__(256)
nhwc_to_nchw_f32_kernel(const void* __restrict__ in, int in_is_f64, float* __restrict__ out, int n, int H, int W) {
  const size_t total = static_cast<size_t>(n) * 3 * H * W;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % W);
    size_t r = i / W;
    const int y = static_cast<int>(r % H);
    r /= H;
    const int c = static_cast<int>(r % 3), b = static_cast<int>(r / 3);
    const size_t s = ((static_cast<size_t>(b) * H + y) * W + x) * 3 + c;
    out[i] = in_is_f64 ? static_cast<float>(static_cast<const double*>(in)[s]) : static_cast<const float*>(in)[s];
  }
}

// How the de-normalised bottom half is finished (the eval scripts differ only here before the resize):
//   kClip255   clip(x * 255, 0, 255)      ade20k_semantic, coco_panoptic, mmpose_custom, seggpt_engine.py:48-52
//   kClip10000 clip(x * 10000, 0, 10000)  nyuv2_depth/painter_inference_depth.py
//   kPlain     x                          sidd / lol / derain (no clip)
enum DenormFinish { kClip255 = 0, kClip10000 = 1, kPlain = 2 };

// out[b, y, x, c] (fp64 [B, H/2, W, 3]) = finish(pred_pixel(sample b * src_stride, y + H/2, x, c) * std[c] + mean[c])
// patch: patchified prediction [*, h*w, p*p*3] fp32 (inner order (pr, pc, c), models_painter.py:355-368);
// = unpatchify -> 'nchw->nhwc' -> bottom half -> de-normalise (seggpt_engine.py:48-52).  Optionally (kClip255 only)
// also writes bin[b, y, x] = (mean_c(out) > 128) (the video path's next-frame target, seggpt_engine.py:164-169).
// Every sample gets the same arithmetic whatever B and src_stride are, so sample b equals a B = 1 call on it alone.
template <int kFinish>
__global__ void __launch_bounds__(256)
seg_postprocess_kernel(const float* __restrict__ patch, double* __restrict__ out, float* __restrict__ bin, int B,
                       int src_stride, int h, int w, int p) {
  const int H = h * p, W = w * p, Hh = H / 2;
  const size_t per = static_cast<size_t>(Hh) * W;
  const size_t total = per * B;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t b = i / per, j = i % per;
    const int x = static_cast<int>(j % W), y = static_cast<int>(j / W) + Hh;
    const int ti = y / p, tj = x / p, pr = y % p, pc = x % p;
    const float* src = patch + b * src_stride * (static_cast<size_t>(h) * w * p * p * 3) +
                       (static_cast<size_t>(ti) * w + tj) * (p * p * 3) + (pr * p + pc) * 3;
    double s = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      // explicit IEEE mul / add: numpy rounds the product before the addition (no fused multiply-add)
      double v = __dadd_rn(__dmul_rn(static_cast<double>(src[c]), c_std[c]), c_mean[c]);
      if (kFinish == kClip255) {
        v = __dmul_rn(v, 255.0);
        v = v < 0.0 ? 0.0 : (v > 255.0 ? 255.0 : v);
      } else if (kFinish == kClip10000) {
        v = __dmul_rn(v, 10000.0);
        v = v < 0.0 ? 0.0 : (v > 10000.0 ? 10000.0 : v);
      }
      out[i * 3 + c] = v;
      s += v;
    }
    if (kFinish == kClip255 && bin) bin[i] = (s / 3.0 > 128.0) ? 1.f : 0.f;
  }
}

// ATen nearest (legacy) source index: upsample_nearest's nearest_idx with scale = float(in) / out
__device__ __forceinline__ int nearest_idx(int dst, int in_size, int out_size) {
  if (out_size == in_size) return dst;
  if (out_size == 2 * in_size) return dst >> 1;
  const float scale = static_cast<float>(in_size) / static_cast<float>(out_size);
  const int s = static_cast<int>(floorf(dst * scale));
  return s < in_size - 1 ? s : in_size - 1;
}
// dst[y, x, c] (uint8 [OH, OW, 3]) = uint8(image[y, x, c] * (0.6 * nearest(seg)[y, x, c] / 255 + 0.4))
// (seggpt_engine.py:97-102: F.interpolate(mode='nearest') to the original size, alpha blend, astype(uint8)).
// The *_at functions compute output element i of one image; ragged_finish_kernel calls them with each image's own
// source sample, size and output.
__device__ __forceinline__ void nearest_blend_at(const double* __restrict__ seg, int SH, int SW,
                                                 const uint8_t* __restrict__ image, uint8_t* __restrict__ dst, int OH,
                                                 int OW, size_t i) {
  const int c = static_cast<int>(i % 3);
  const size_t r = i / 3;
  const int x = static_cast<int>(r % OW), y = static_cast<int>(r / OW);
  const int sy = nearest_idx(y, SH, OH), sx = nearest_idx(x, SW, OW);
  const double o = seg[(static_cast<size_t>(sy) * SW + sx) * 3 + c];
  const double v = __dmul_rn(static_cast<double>(image[i]), __dadd_rn(__dmul_rn(0.6, o) / 255.0, 0.4));
  dst[i] = static_cast<uint8_t>(v);   // numpy astype(uint8): truncation (values are within [0, 255])
}

// One axis of ATen's linear interpolation (align_corners=False, scale = in / out from the sizes):
// compute_source_index_and_lambda.  src = scale * (dst + 0.5) - 0.5 (one fused multiply-add in torch-CPU's build),
// clamped at 0; i1 = i0 + 1 inside the image; l1 = src - i0, l0 = 1 - l1.  An unchanged size copies (l1 = 0).
struct LinearTap {
  int i0, i1;
  double l0, l1;
};
__device__ __forceinline__ LinearTap linear_tap(int dst, int in_size, int out_size, double scale) {
  LinearTap t;
  if (in_size == out_size) {
    t.i0 = t.i1 = dst;
    t.l0 = 1.0;
    t.l1 = 0.0;
    return t;
  }
  double f = __fma_rn(scale, static_cast<double>(dst) + 0.5, -0.5);
  if (f < 0.0) f = 0.0;
  t.i0 = static_cast<int>(f);
  if (t.i0 > in_size - 1) t.i0 = in_size - 1;
  t.i1 = t.i0 + (t.i0 < in_size - 1 ? 1 : 0);
  t.l1 = __dadd_rn(f, -static_cast<double>(t.i0));
  t.l1 = t.l1 < 0.0 ? 0.0 : (t.l1 > 1.0 ? 1.0 : t.l1);
  t.l0 = __dadd_rn(1.0, -t.l1);
  return t;
}

// dst[y, x, c] (uint8 [OH, OW, 3]) = uint8(int(bilinear(seg)[y, x, c]))   (painter_inference_segm.py:89-92:
// F.interpolate(mode='bilinear', align_corners=False) on the float64 tensor, .int(), astype(uint8))
__device__ __forceinline__ void bilinear_u8_at(const double* __restrict__ seg, int SH, int SW,
                                               uint8_t* __restrict__ dst, int OH, int OW, size_t i) {
  const double sch = static_cast<double>(SH) / OH, scw = static_cast<double>(SW) / OW;
  const int c = static_cast<int>(i % 3);
  const size_t r = i / 3;
  const int x = static_cast<int>(r % OW), y = static_cast<int>(r / OW);
  const LinearTap ty = linear_tap(y, SH, OH, sch), tx = linear_tap(x, SW, OW, scw);
  auto at = [&](int yy, int xx) { return seg[(static_cast<size_t>(yy) * SW + xx) * 3 + c]; };
  const double v = ty.l0 * (tx.l0 * at(ty.i0, tx.i0) + tx.l1 * at(ty.i0, tx.i1)) +
                   ty.l1 * (tx.l0 * at(ty.i1, tx.i0) + tx.l1 * at(ty.i1, tx.i1));
  dst[i] = static_cast<uint8_t>(static_cast<int>(v));
}

// dst[y, x] (int32 [OH, OW]) = int(mean_c(bilinear(src)[y, x, c]))   (nyuv2_depth/painter_inference_depth.py:
// F.interpolate(mode='bilinear') on the float64 tensor, .mean(-1), .int()).  torch-CPU evaluates the 2 x 2 sum in one
// of two forms, both reproduced here with the fused multiply-adds of its build:
//   cl_form = 0 (its generic kernel)        (v00 l0x + v01 l1x) l0y + (v10 l0x + v11 l1x) l1y
//   cl_form = 1 (its channels-last kernel)  v00 (l0y l0x) + v01 (l0y l1x) + v10 (l1y l0x) + v11 (l1y l1x), left to right
// The mean is torch's sum over the 3 channels in order, then / 3.
__device__ __forceinline__ void depth_finish_at(const double* __restrict__ src, int SH, int SW,
                                                int32_t* __restrict__ dst, int OH, int OW, int cl_form, size_t i) {
  const double sch = static_cast<double>(SH) / OH, scw = static_cast<double>(SW) / OW;
  const int x = static_cast<int>(i % OW), y = static_cast<int>(i / OW);
  const LinearTap ty = linear_tap(y, SH, OH, sch), tx = linear_tap(x, SW, OW, scw);
  const double* r0 = src + static_cast<size_t>(ty.i0) * SW * 3;
  const double* r1 = src + static_cast<size_t>(ty.i1) * SW * 3;
  const double w00 = __dmul_rn(ty.l0, tx.l0), w01 = __dmul_rn(ty.l0, tx.l1);
  const double w10 = __dmul_rn(ty.l1, tx.l0), w11 = __dmul_rn(ty.l1, tx.l1);
  double s = 0.0;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double v00 = r0[tx.i0 * 3 + c], v01 = r0[tx.i1 * 3 + c];
    const double v10 = r1[tx.i0 * 3 + c], v11 = r1[tx.i1 * 3 + c];
    double v;
    if (cl_form) {
      v = __fma_rn(v11, w11, __fma_rn(v10, w10, __fma_rn(v00, w00, __dmul_rn(v01, w01))));
    } else {
      const double t0 = __fma_rn(v00, tx.l0, __dmul_rn(v01, tx.l1));
      const double t1 = __fma_rn(v10, tx.l0, __dmul_rn(v11, tx.l1));
      v = __fma_rn(t0, ty.l0, __dmul_rn(t1, ty.l1));
    }
    s = c == 0 ? v : __dadd_rn(s, v);
  }
  dst[i] = static_cast<int32_t>(__ddiv_rn(s, 3.0));   // .int(): truncation (values are within [0, 10000])
}

// ATen's nearest source index in its generic kernel (HelperInterpNearest): scale = double(in) / out, then
// floorf(scale * dst) of the product rounded to float.  Its channels-last kernel uses nearest_idx above instead.
__device__ __forceinline__ int nearest_idx_generic(int dst, int in_size, double scale) {
  const int s = static_cast<int>(floorf(static_cast<float>(__dmul_rn(scale, static_cast<double>(dst)))));
  return s < in_size - 1 ? s : in_size - 1;
}

// dst[y, x, c] (uint8 [OH, OW, 3]) = uint8(int(nearest(src)[y, x, c]))   (coco_panoptic/painter_inference_pano_inst.py,
// mmpose_custom/painter_inference_pose.py: F.interpolate(mode='nearest') on the float64 tensor, .int(), astype(uint8)).
// cl_form = 1: torch-CPU's channels-last kernel (which it takes for 3 channels when OH + OW <= 128), else its generic
// kernel; the two compute the source index differently.
__device__ __forceinline__ void nearest_u8_at(const double* __restrict__ src, int SH, int SW,
                                              uint8_t* __restrict__ dst, int OH, int OW, int cl_form, size_t i) {
  const double sch = static_cast<double>(SH) / OH, scw = static_cast<double>(SW) / OW;
  const int c = static_cast<int>(i % 3);
  const size_t r = i / 3;
  const int x = static_cast<int>(r % OW), y = static_cast<int>(r / OW);
  const int sy = cl_form ? nearest_idx(y, SH, OH) : nearest_idx_generic(y, SH, sch);
  const int sx = cl_form ? nearest_idx(x, SW, OW) : nearest_idx_generic(x, SW, scw);
  dst[i] = static_cast<uint8_t>(static_cast<int>(src[(static_cast<size_t>(sy) * SW + sx) * 3 + c]));
}

// ATen's cubic convolution weights (get_cubic_upsample_coefficients, A = -0.75) of the 4 taps around a source
// position with fractional part t, with the fused multiply-adds of torch-CPU's build:
//   w(x) = ((A + 2) x - (A + 3)) x x + 1      for the two inner taps (x = t, 1 - t)
//   w(x) = ((A x - 5A) x + 8A) x - 4A         for the two outer taps (x = t + 1, (1 - t) + 1)
__device__ __forceinline__ double cubic_inner(double x) {
  const double A = -0.75;
  return __dadd_rn(__dmul_rn(__dmul_rn(__fma_rn(A + 2.0, x, -(A + 3.0)), x), x), 1.0);
}
__device__ __forceinline__ double cubic_outer(double x) {
  const double A = -0.75;
  return __dadd_rn(__dmul_rn(__fma_rn(__fma_rn(A, x, -5.0 * A), x, 8.0 * A), x), -4.0 * A);
}
// One axis of ATen's bicubic (align_corners=False, scale = in / out): src = scale * (dst + 0.5) - 0.5 (not clamped),
// i = min(floorf(src), in - 1) (floorf of the value rounded to float, as ATen does), t = clamp(src - i, 0, 1); taps
// i - 1 .. i + 2 clamped to the border.
struct CubicTaps {
  int idx[4];
  double w[4];
};
__device__ __forceinline__ CubicTaps cubic_taps(int dst, int in_size, double scale) {
  CubicTaps k;
  const double f = __fma_rn(scale, static_cast<double>(dst) + 0.5, -0.5);
  int i = static_cast<int>(floorf(static_cast<float>(f)));
  if (i > in_size - 1) i = in_size - 1;
  double t = __dadd_rn(f, -static_cast<double>(i));
  t = t < 0.0 ? 0.0 : (t > 1.0 ? 1.0 : t);
  const double u = __dadd_rn(1.0, -t);
  k.w[0] = cubic_outer(__dadd_rn(t, 1.0));
  k.w[1] = cubic_inner(t);
  k.w[2] = cubic_inner(u);
  k.w[3] = cubic_outer(__dadd_rn(u, 1.0));
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int v = i - 1 + j;
    k.idx[j] = v < 0 ? 0 : (v > in_size - 1 ? in_size - 1 : v);
  }
  return k;
}
// ATen's 4-tap weighted sum: fma(v3, w3, fma(v2, w2, fma(v0, w0, v1 w1)))
__device__ __forceinline__ double cubic_sum(const double v[4], const double w[4]) {
  return __fma_rn(v[3], w[3], __fma_rn(v[2], w[2], __fma_rn(v[0], w[0], __dmul_rn(v[1], w[1]))));
}

// dst[y, x, c] (fp64 [OH, OW, 3]) = bicubic(src)[y, x, c]   (sidd / lol / derain painter_inference_*.py:
// F.interpolate(mode='bicubic', align_corners=False) on the float64 tensor, no clipping).  As in ATen, each of the 4
// source rows is first summed along x, then the 4 row sums along y.
__device__ __forceinline__ void bicubic_f64_at(const double* __restrict__ src, int SH, int SW,
                                               double* __restrict__ dst, int OH, int OW, size_t i) {
  const double sch = static_cast<double>(SH) / OH, scw = static_cast<double>(SW) / OW;
  const int c = static_cast<int>(i % 3);
  const size_t r = i / 3;
  const int x = static_cast<int>(r % OW), y = static_cast<int>(r / OW);
  const CubicTaps ky = cubic_taps(y, SH, sch), kx = cubic_taps(x, SW, scw);
  double rows[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const double* row = src + static_cast<size_t>(ky.idx[j]) * SW * 3 + c;
    double v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = row[kx.idx[k] * 3];
    rows[j] = cubic_sum(v, kx.w);
  }
  dst[i] = cubic_sum(rows, ky.w);
}

// Ragged finish of a batch: one CTA row (blockIdx.y) per descriptor row [src sample, OH, OW, cl_form, offset lo, hi]
// (PK_RAG_FIELDS), grid-stride over that image's output elements.  src sample s is src + s * SH * SW * 3; the image's
// output starts at dst + offset (elements of the output type), and for the blend the source image at image + offset.
template <int kOp>
__global__ void __launch_bounds__(256)
ragged_finish_kernel(const double* __restrict__ src, int SH, int SW, const int* __restrict__ items,
                     const uint8_t* __restrict__ image, void* __restrict__ dst) {
  const int* it = items + static_cast<size_t>(blockIdx.y) * PK_RAG_FIELDS;
  const int OH = it[1], OW = it[2], cl_form = it[3];
  const size_t off = static_cast<size_t>(static_cast<uint32_t>(it[4])) |
                     (static_cast<size_t>(static_cast<uint32_t>(it[5])) << 32);
  const double* s = src + static_cast<size_t>(it[0]) * SH * SW * 3;
  const size_t total = static_cast<size_t>(OH) * OW * (kOp == PK_FIN_DEPTH ? 1 : 3);
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    if constexpr (kOp == PK_FIN_BILINEAR_U8) {
      bilinear_u8_at(s, SH, SW, static_cast<uint8_t*>(dst) + off, OH, OW, i);
    } else if constexpr (kOp == PK_FIN_NEAREST_U8) {
      nearest_u8_at(s, SH, SW, static_cast<uint8_t*>(dst) + off, OH, OW, cl_form, i);
    } else if constexpr (kOp == PK_FIN_DEPTH) {
      depth_finish_at(s, SH, SW, static_cast<int32_t*>(dst) + off, OH, OW, cl_form, i);
    } else if constexpr (kOp == PK_FIN_BICUBIC_F64) {
      bicubic_f64_at(s, SH, SW, static_cast<double*>(dst) + off, OH, OW, i);
    } else {
      nearest_blend_at(s, SH, SW, image + off, static_cast<uint8_t*>(dst) + off, OH, OW, i);
    }
  }
}

static inline int stream_grid(size_t total) {
  size_t g = (total + 255) / 256;
  const size_t cap = static_cast<size_t>(sm_count()) * 16;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace pk

using namespace pk;

extern "C" int pk_stitch_normalize(const void* const* top, const int* top_dtype, const void* const* bottom,
                                   const int* bottom_dtype, float* out, int P, int S, void* stream) {
  PK_CHECK(top && bottom && top_dtype && bottom_dtype && out && P >= 1 && S > 0, "pk_stitch_normalize: bad arguments");
  for (int p = 0; p < P; ++p)
    PK_CHECK(top[p] && bottom[p] && top_dtype[p] >= 0 && top_dtype[p] <= 2 && bottom_dtype[p] >= 0 &&
                 bottom_dtype[p] <= 2, "pk_stitch_normalize: bad member %d", p);
  // the member pointers travel as a kernel parameter of kCanvasMembers entries: one launch per chunk of members
  const size_t per = static_cast<size_t>(3) * 2 * S * S;
  for (int p0 = 0; p0 < P; p0 += kCanvasMembers) {
    const int n = P - p0 < kCanvasMembers ? P - p0 : kCanvasMembers;
    CanvasSrc src;
    for (int p = 0; p < n; ++p) {
      src.top[p] = top[p0 + p];
      src.bottom[p] = bottom[p0 + p];
      src.top_dtype[p] = top_dtype[p0 + p];
      src.bottom_dtype[p] = bottom_dtype[p0 + p];
    }
    stitch_normalize_kernel<<<stream_grid(n * per), 256, 0, static_cast<cudaStream_t>(stream)>>>(src, out + p0 * per, n,
                                                                                                  S);
    PK_LAUNCH_CHECK("pk_stitch_normalize");
  }
  return 0;
}

extern "C" int pk_nhwc_to_nchw_f32(const void* in, int in_is_f64, float* out, int n, int H, int W, void* stream) {
  PK_CHECK(in && out && n > 0 && H > 0 && W > 0, "pk_nhwc_to_nchw_f32: bad arguments");
  const size_t total = static_cast<size_t>(n) * 3 * H * W;
  nhwc_to_nchw_f32_kernel<<<stream_grid(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(in, in_is_f64, out, n, H,
                                                                                             W);
  PK_LAUNCH_CHECK("pk_nhwc_to_nchw_f32");
  return 0;
}

extern "C" int pk_denorm_bottom_batched(const float* patch, double* out, float* bin_or_null, int B, int src_stride,
                                        int h, int w, int p, int finish, void* stream) {
  PK_CHECK(patch && out && B >= 1 && src_stride >= 1 && h > 0 && w > 0 && p > 0 && h % 2 == 0 && finish >= kClip255 &&
               finish <= kPlain, "pk_denorm_bottom_batched: bad arguments");
  PK_CHECK(!bin_or_null || finish == kClip255, "pk_denorm_bottom_batched: the binarised mask needs finish 0 (x 255)");
  const int grid = stream_grid(static_cast<size_t>(B) * h * p / 2 * w * p);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (finish == kClip255)
    seg_postprocess_kernel<kClip255><<<grid, 256, 0, st>>>(patch, out, bin_or_null, B, src_stride, h, w, p);
  else if (finish == kClip10000)
    seg_postprocess_kernel<kClip10000><<<grid, 256, 0, st>>>(patch, out, bin_or_null, B, src_stride, h, w, p);
  else
    seg_postprocess_kernel<kPlain><<<grid, 256, 0, st>>>(patch, out, bin_or_null, B, src_stride, h, w, p);
  PK_LAUNCH_CHECK("pk_denorm_bottom_batched");
  return 0;
}

extern "C" int pk_finish_ragged(int op, const double* src, int SH, int SW, const int* items, int n, int max_pix,
                                const uint8_t* image, void* dst, void* stream) {
  PK_CHECK(src && items && dst && SH > 0 && SW > 0 && n >= 1 && n <= 65535 && max_pix > 0,
           "pk_finish_ragged: bad arguments (1 <= n <= 65535 images, max_pix > 0)");
  PK_CHECK(op >= PK_FIN_BILINEAR_U8 && op <= PK_FIN_NEAREST_BLEND, "pk_finish_ragged: unknown op %d", op);
  PK_CHECK((op == PK_FIN_NEAREST_BLEND) == (image != nullptr),
           "pk_finish_ragged: the source images are given for the blend (op %d) and only for it", PK_FIN_NEAREST_BLEND);
  // max_pix only sizes the grid (every loop is grid-stride): CTAs per image cover the largest image's elements
  const size_t per = static_cast<size_t>(max_pix) * (op == PK_FIN_DEPTH ? 1 : 3);
  const size_t cap = static_cast<size_t>(sm_count()) * 16;
  size_t gx = (per + 255) / 256, gcap = (cap + n - 1) / n;
  gx = gx < gcap ? gx : gcap;
  const dim3 grid(static_cast<unsigned>(gx < 1 ? 1 : gx), static_cast<unsigned>(n));
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  switch (op) {
    case PK_FIN_BILINEAR_U8:
      ragged_finish_kernel<PK_FIN_BILINEAR_U8><<<grid, 256, 0, st>>>(src, SH, SW, items, image, dst);
      break;
    case PK_FIN_NEAREST_U8:
      ragged_finish_kernel<PK_FIN_NEAREST_U8><<<grid, 256, 0, st>>>(src, SH, SW, items, image, dst);
      break;
    case PK_FIN_DEPTH:
      ragged_finish_kernel<PK_FIN_DEPTH><<<grid, 256, 0, st>>>(src, SH, SW, items, image, dst);
      break;
    case PK_FIN_BICUBIC_F64:
      ragged_finish_kernel<PK_FIN_BICUBIC_F64><<<grid, 256, 0, st>>>(src, SH, SW, items, image, dst);
      break;
    default:
      ragged_finish_kernel<PK_FIN_NEAREST_BLEND><<<grid, 256, 0, st>>>(src, SH, SW, items, image, dst);
  }
  PK_LAUNCH_CHECK("pk_finish_ragged");
  return 0;
}
