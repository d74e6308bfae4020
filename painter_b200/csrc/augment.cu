// painter_b200 — the pixel arithmetic of the training recipe's paired augmentations (Painter/main_train.py:232-262
// applied by Painter/data/pairdataset.py:106-190), batched over samples with per-sample descriptors.  The host keeps
// decoding and every random draw; these kernels reproduce what PIL and torch-CPU compute from those draws, bit for bit:
//
//   resized crop   F.resized_crop on a PIL image = crop + Image.resize(S x S, BICUBIC | NEAREST), Pillow's
//                  ImagingResample: separable, horizontal pass first (over the rows the vertical pass reads;
//                  vertical first for very tall, narrow sources, see vertical_first) into a uint8-clipped
//                  intermediate; double coefficients (Keys a = -0.5, support 2 * max(scale, 1), normalised by their
//                  sum) in 22-bit fixed point, accumulated from 1 << 21, >> 22, clipped.  NEAREST
//                  is Pillow's affine scale path (source positions accumulated in double).  The flip is folded into
//                  the store.
//   color jitter   ColorJitter on PIL in the drawn op order: Image.blend in float32 (truncate, clip), L by the ITU-R
//                  601 integer weights, contrast around int(mean(L) + 0.5) of the current image, hue through
//                  Pillow's uint8 HSV.  One CTA per image: contrast needs the whole image's mean between ops.
//   normalise      ToTensor + Normalize: (u / 255 - mean) / std in fp32, into the top or bottom half of the canvas.
//   second crop    RandomResizedCrop on the fp32 canvas: torch-CPU interpolate(bicubic, antialias=True) (float
//                  weights, separable, horizontal first; torch-CPU contracts the filter and the accumulation to FMA)
//                  or upsample_nearest2d (float scale).  Samples without a second crop take the full box in nearest
//                  mode, which is an exact copy.
//
// No expression here may be contracted differently from the arithmetic it restates: every floating-point step is an
// explicit _rn intrinsic (or an explicit fma where torch-CPU uses one).
#include "common.cuh"
#include "host_common.h"
#include "../../include/painter_b200.h"

namespace pk {

// ------------------------------------------------------------------------------------------------ resized crop (PIL)
__device__ __forceinline__ double pil_bicubic(double x) {
  if (x < 0.0) x = -x;
  if (x < 1.0)   // ((a + 2) x - (a + 3)) x x + 1
    return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, x), 2.5), x), x), 1.0);
  if (x < 2.0)   // (((x - 5) x + 8) x - 4) a
    return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), -0.5);
  return 0.0;
}

struct CropJob {
  long long off;          // byte offset of the decoded H x W x 3 image in the source buffer
  int H, W, top, left, h, w, mode, flip;
  long long tmp_off;      // byte offset of this job's first-pass intermediate in the scratch buffer
};
__device__ __forceinline__ CropJob load_crop_job(const int* t, int j) {
  const int* r = t + j * PK_AUG_CROP_FIELDS;
  CropJob c;
  c.off = static_cast<long long>(static_cast<unsigned>(r[0])) | (static_cast<long long>(r[1]) << 32);
  c.H = r[2]; c.W = r[3]; c.top = r[4]; c.left = r[5]; c.h = r[6]; c.w = r[7]; c.mode = r[8]; c.flip = r[9];
  c.tmp_off = static_cast<long long>(static_cast<unsigned>(r[10])) | (static_cast<long long>(r[11]) << 32);
  return c;
}

// one thread per (job, axis, output index): bounds + fixed-point coefficients (bicubic) or the source index (nearest)
__global__ void __launch_bounds__(128)
crop_coeffs_kernel(const int* __restrict__ jobs, int S, int KP, int* __restrict__ coef, int2* __restrict__ bounds) {
  const int xx = blockIdx.x * blockDim.x + threadIdx.x;
  const int axis = blockIdx.y;               // 0: x (columns), 1: y (rows)
  const int j = blockIdx.z;
  if (xx >= S) return;
  const CropJob c = load_crop_job(jobs, j);
  const int in = axis == 0 ? c.w : c.h;
  const size_t row = (static_cast<size_t>(j) * 2 + axis) * S + xx;
  if (c.mode == 1) {
    // ImagingScaleAffine: xo = a0 / 2, then xo += a0 per output pixel
    const double a0 = __ddiv_rn(static_cast<double>(in), static_cast<double>(S));
    double xo = __dmul_rn(a0, 0.5);
    for (int k = 0; k < xx; ++k) xo = __dadd_rn(xo, a0);
    const int xin = xo < 0.0 ? -1 : static_cast<int>(xo);
    bounds[row] = make_int2(xin >= 0 && xin < in ? xin : -1, 1);
    return;
  }
  const double scale = __ddiv_rn(static_cast<double>(in), static_cast<double>(S));
  const double fscale = scale < 1.0 ? 1.0 : scale;
  const double support = __dmul_rn(2.0, fscale);
  const double center = __dmul_rn(__dadd_rn(static_cast<double>(xx), 0.5), scale);
  const double ss = __ddiv_rn(1.0, fscale);
  int xmin = static_cast<int>(__dadd_rn(__dsub_rn(center, support), 0.5));
  if (xmin < 0) xmin = 0;
  int xmax = static_cast<int>(__dadd_rn(__dadd_rn(center, support), 0.5));
  if (xmax > in) xmax = in;
  xmax -= xmin;
  int* k = coef + row * KP;
  double ww = 0.0;
  for (int x = 0; x < xmax; ++x)
    ww = __dadd_rn(ww, pil_bicubic(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss)));
  for (int x = 0; x < KP; ++x) {
    int q = 0;
    if (x < xmax) {
      double w = pil_bicubic(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss));
      if (ww != 0.0) w = __ddiv_rn(w, ww);
      const double f = __dmul_rn(w, 4194304.0);   // 1 << 22
      q = static_cast<int>(w < 0 ? __dadd_rn(-0.5, f) : __dadd_rn(0.5, f));
    }
    k[x] = q;
  }
  bounds[row] = make_int2(xmin, xmax);
}

__device__ __forceinline__ unsigned char clip8(int v) {
  v >>= 22;
  return static_cast<unsigned char>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// Pillow runs the vertical pass first for a source more than 100 times taller than wide that it shrinks vertically
// (found by comparing both orders against Image.resize; the order changes the uint8-rounded intermediate)
__device__ __forceinline__ bool vertical_first(const CropJob& c, int S) { return c.h > S && 100LL * c.w < c.h; }

// first pass of the bicubic jobs, into a uint8-clipped intermediate: horizontal over rows [y0, y1) of the crop
// (tmp [y1 - y0, S]), or vertical over columns [x0, x1) (tmp [S, x1 - x0])
__global__ void __launch_bounds__(256)
crop_pass1_kernel(const unsigned char* __restrict__ src, const int* __restrict__ jobs, int S, int KP,
                  const int* __restrict__ coef, const int2* __restrict__ bounds, unsigned char* __restrict__ tmp) {
  const int j = blockIdx.z;
  const CropJob c = load_crop_job(jobs, j);
  if (c.mode != 0) return;
  const bool vfirst = vertical_first(c, S);
  const int axis = vfirst ? 1 : 0;
  const int2* b1 = bounds + (static_cast<size_t>(j) * 2 + axis) * S;          // the pass's own taps
  const int2* b2 = bounds + (static_cast<size_t>(j) * 2 + (1 - axis)) * S;    // the span the other pass reads
  const int* k1 = coef + (static_cast<size_t>(j) * 2 + axis) * S * KP;
  const int lo = b2[0].x, span = b2[S - 1].x + b2[S - 1].y - lo;
  unsigned char* out = tmp + c.tmp_off;
  const unsigned char* in = src + c.off;
  const int n = span * S;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    // hfirst: i = row * S + xx (row of the span, output column); vfirst: i = yy * span + col
    const int a = vfirst ? i % span : i % S;            // position along the span / output index of this pass
    const int o = vfirst ? i / span : i / S;
    const int2 b = b1[vfirst ? o : a];
    const int* k = k1 + static_cast<size_t>(vfirst ? o : a) * KP;
    const unsigned char* p;
    long long step;
    if (vfirst) {
      p = in + (static_cast<size_t>(c.top + b.x) * c.W + c.left + lo + a) * 3;
      step = static_cast<long long>(c.W) * 3;
    } else {
      p = in + (static_cast<size_t>(c.top + lo + o) * c.W + c.left + b.x) * 3;
      step = 3;
    }
    int s0 = 1 << 21, s1 = 1 << 21, s2 = 1 << 21;
    for (int x = 0; x < b.y; ++x) {
      const int w = k[x];
      const unsigned char* q = p + x * step;
      s0 += q[0] * w;
      s1 += q[1] * w;
      s2 += q[2] * w;
    }
    unsigned char* r = out + static_cast<size_t>(i) * 3;
    r[0] = clip8(s0); r[1] = clip8(s1); r[2] = clip8(s2);
  }
}

// second pass (bicubic: from the intermediate) or the nearest gather (from the source), flip folded into the store
__global__ void __launch_bounds__(256)
crop_pass2_kernel(const unsigned char* __restrict__ src, const int* __restrict__ jobs, int S, int KP,
                  const int* __restrict__ coef, const int2* __restrict__ bounds, const unsigned char* __restrict__ tmp,
                  unsigned char* __restrict__ dst) {
  const int j = blockIdx.z;
  const CropJob c = load_crop_job(jobs, j);
  const int2* bx = bounds + static_cast<size_t>(j) * 2 * S;
  const int2* by = bx + S;
  const bool vfirst = c.mode == 0 && vertical_first(c, S);
  const int axis = vfirst ? 0 : 1;
  const int2* b2 = bounds + (static_cast<size_t>(j) * 2 + axis) * S;
  const int* k2 = coef + (static_cast<size_t>(j) * 2 + axis) * S * KP;
  const int lo = b2[0].x, span = b2[S - 1].x + b2[S - 1].y - lo;
  unsigned char* out = dst + static_cast<size_t>(j) * S * S * 3;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < S * S; i += gridDim.x * blockDim.x) {
    const int yy = i / S, xx = i - yy * S;
    unsigned char* o = out + (static_cast<size_t>(yy) * S + (c.flip ? S - 1 - xx : xx)) * 3;
    if (c.mode == 1) {
      const int sy = by[yy].x, sx = bx[xx].x;
      if (sy < 0 || sx < 0) { o[0] = o[1] = o[2] = 0; continue; }
      const unsigned char* p = src + c.off + (static_cast<size_t>(c.top + sy) * c.W + c.left + sx) * 3;
      o[0] = p[0]; o[1] = p[1]; o[2] = p[2];
      continue;
    }
    // hfirst: vertical taps over tmp [span rows, S]; vfirst: horizontal taps over tmp [S, span columns]
    const int2 b = b2[vfirst ? xx : yy];
    const int* k = k2 + static_cast<size_t>(vfirst ? xx : yy) * KP;
    const unsigned char* p = vfirst ? tmp + c.tmp_off + (static_cast<size_t>(yy) * span + b.x - lo) * 3
                                    : tmp + c.tmp_off + (static_cast<size_t>(b.x - lo) * S + xx) * 3;
    const size_t step = vfirst ? 3 : static_cast<size_t>(S) * 3;
    int s0 = 1 << 21, s1 = 1 << 21, s2 = 1 << 21;
    for (int y = 0; y < b.y; ++y) {
      const int w = k[y];
      const unsigned char* q = p + y * step;
      s0 += q[0] * w;
      s1 += q[1] * w;
      s2 += q[2] * w;
    }
    o[0] = clip8(s0); o[1] = clip8(s1); o[2] = clip8(s2);
  }
}

// ------------------------------------------------------------------------------------------------ color jitter (PIL)
// Image.blend(d, s, f): float32 d + f * (s - d), truncated, clipped (the in-range branch never leaves [0, 255])
__device__ __forceinline__ unsigned char pil_blend(int d, int s, float f) {
  const float t = __fadd_rn(static_cast<float>(d), __fmul_rn(f, static_cast<float>(s - d)));
  if (t <= 0.f) return 0;
  if (t >= 255.f) return 255;
  return static_cast<unsigned char>(t);
}
__device__ __forceinline__ int pil_luma(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

__device__ __forceinline__ int clip_u8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

// Pillow's rgb2hsv (uint8 HSV; float / double mixed exactly as its C source evaluates)
__device__ __forceinline__ void pil_rgb2hsv(int r, int g, int b, int& uh, int& us, int& uv) {
  const int maxc = max(r, max(g, b)), minc = min(r, min(g, b));
  uv = maxc;
  if (minc == maxc) { uh = 0; us = 0; return; }
  const float cr = static_cast<float>(maxc - minc);
  const float s = __fdiv_rn(cr, static_cast<float>(maxc));
  const float rc = __fdiv_rn(static_cast<float>(maxc - r), cr);
  const float gc = __fdiv_rn(static_cast<float>(maxc - g), cr);
  const float bc = __fdiv_rn(static_cast<float>(maxc - b), cr);
  float h;
  if (r == maxc) h = __fsub_rn(bc, gc);
  else if (g == maxc) h = __double2float_rn(__dsub_rn(__dadd_rn(2.0, static_cast<double>(rc)), static_cast<double>(bc)));
  else h = __double2float_rn(__dsub_rn(__dadd_rn(4.0, static_cast<double>(gc)), static_cast<double>(rc)));
  h = __double2float_rn(fmod(__dadd_rn(__ddiv_rn(static_cast<double>(h), 6.0), 1.0), 1.0));
  uh = clip_u8(static_cast<int>(__dmul_rn(static_cast<double>(h), 255.0)));
  us = clip_u8(static_cast<int>(__dmul_rn(static_cast<double>(s), 255.0)));
}

// Pillow's hsv2rgb; C round() is half away from zero
__device__ __forceinline__ void pil_hsv2rgb(int h, int s, int v, int& r, int& g, int& b) {
  if (s == 0) { r = g = b = v; return; }
  const double h6 = __ddiv_rn(__dmul_rn(static_cast<double>(static_cast<float>(h)), 6.0), 255.0);
  const int i = static_cast<int>(floor(h6));
  const float f = __double2float_rn(__dsub_rn(h6, static_cast<double>(static_cast<float>(i))));
  const float fs = __double2float_rn(__ddiv_rn(static_cast<double>(s), 255.0));
  const double vd = static_cast<double>(v);
  const int p = clip_u8(static_cast<int>(round(__dmul_rn(vd, __dsub_rn(1.0, static_cast<double>(fs))))));
  const int q = clip_u8(static_cast<int>(round(__dmul_rn(vd, __dsub_rn(1.0, static_cast<double>(__fmul_rn(fs, f)))))));
  const int t = clip_u8(static_cast<int>(round(__dmul_rn(
      vd, __dsub_rn(1.0, __dmul_rn(static_cast<double>(fs), __dsub_rn(1.0, static_cast<double>(f))))))));
  switch (i % 6) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// one jitter op on one pixel; `mean` is the contrast op's grey level
__device__ __forceinline__ void jitter_op(int op, const float* fac, int hue_shift, int mean, int& r, int& g, int& b) {
  if (op == PK_JIT_BRIGHTNESS) {
    r = pil_blend(0, r, fac[0]); g = pil_blend(0, g, fac[0]); b = pil_blend(0, b, fac[0]);
  } else if (op == PK_JIT_CONTRAST) {
    r = pil_blend(mean, r, fac[1]); g = pil_blend(mean, g, fac[1]); b = pil_blend(mean, b, fac[1]);
  } else if (op == PK_JIT_SATURATION) {
    const int l = pil_luma(r, g, b);
    r = pil_blend(l, r, fac[2]); g = pil_blend(l, g, fac[2]); b = pil_blend(l, b, fac[2]);
  } else if (op == PK_JIT_HUE) {
    int h, s, v;
    pil_rgb2hsv(r, g, b, h, s, v);
    pil_hsv2rgb((h + hue_shift) & 255, s, v, r, g, b);
  }
}

// One CTA per image, in place.  Pass 1 applies the ops before contrast and sums L of its result; pass 2 (only when
// contrast is drawn) applies contrast around int(sum / n + 0.5) and the ops after it.  Every thread touches the same
// pixels in both passes, so the block reduction is the only synchronisation.
__global__ void __launch_bounds__(1024)
jitter_kernel(unsigned char* __restrict__ imgs, const int* __restrict__ jobs, long long npix) {
  const int* jb = jobs + blockIdx.x * PK_AUG_JIT_FIELDS;
  unsigned char* img = imgs + static_cast<size_t>(jb[0]) * npix * 3;
  const int ops[4] = {jb[1], jb[2], jb[3], jb[4]};
  const float fac[3] = {__int_as_float(jb[5]), __int_as_float(jb[6]), __int_as_float(jb[7])};
  const int hue_shift = jb[8] & 255;
  int cpos = 4;
  for (int k = 0; k < 4; ++k)
    if (ops[k] == PK_JIT_CONTRAST) { cpos = k; break; }
  unsigned long long lsum = 0;
  for (long long i = threadIdx.x; i < npix; i += blockDim.x) {
    unsigned char* p = img + i * 3;
    int r = p[0], g = p[1], b = p[2];
    for (int k = 0; k < cpos; ++k) jitter_op(ops[k], fac, hue_shift, 0, r, g, b);
    if (cpos < 4) lsum += pil_luma(r, g, b);
    p[0] = r; p[1] = g; p[2] = b;
  }
  if (cpos == 4) return;
  __shared__ unsigned long long part[32];
  for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = lsum;
  __syncthreads();
  unsigned long long tot = 0;
  for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) tot += part[w];
  // ImageStat mean of the L image: sum / count in double, + 0.5, truncated
  const int mean = static_cast<int>(__dadd_rn(__ddiv_rn(static_cast<double>(tot), static_cast<double>(npix)), 0.5));
  for (long long i = threadIdx.x; i < npix; i += blockDim.x) {
    unsigned char* p = img + i * 3;
    int r = p[0], g = p[1], b = p[2];
    for (int k = cpos; k < 4; ++k) jitter_op(ops[k], fac, hue_shift, mean, r, g, b);
    p[0] = r; p[1] = g; p[2] = b;
  }
}

// ------------------------------------------------------------------------------------------------ ToTensor + Normalize
// slot j = (b * P + p) * 2 + t  (t = 0 image, 1 target) -> canvas_t[b, :, p * S : (p + 1) * S, :]
__global__ void __launch_bounds__(256)
normalize_kernel(const unsigned char* __restrict__ slots, int P, int S, float* __restrict__ img,
                 float* __restrict__ tgt) {
  const int j = blockIdx.y;
  const int t = j & 1, p = (j >> 1) % P, b = (j >> 1) / P;
  const float mean[3] = {0.485f, 0.456f, 0.406f};
  const float stdv[3] = {0.229f, 0.224f, 0.225f};
  const unsigned char* in = slots + static_cast<size_t>(j) * S * S * 3;
  float* out = (t ? tgt : img) + static_cast<size_t>(b) * 3 * P * S * S + static_cast<size_t>(p) * S * S;
  const int n = S * S;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    for (int c = 0; c < 3; ++c) {
      const float x = __fdiv_rn(static_cast<float>(in[static_cast<size_t>(i) * 3 + c]), 255.f);
      out[static_cast<size_t>(c) * P * S * S + i] = __fdiv_rn(__fsub_rn(x, mean[c]), stdv[c]);
    }
}

// ------------------------------------------------------------------------------------------------ second crop (torch)
// torch-CPU's antialiased cubic filter; the build it runs contracts both polynomials to FMA
__device__ __forceinline__ float aa_cubic(float x) {
  x = fabsf(x);
  if (x < 1.f) return __fmaf_rn(__fmul_rn(__fmaf_rn(1.5f, x, -2.5f), x), x, 1.f);
  if (x < 2.f) return __fmaf_rn(__fmaf_rn(__fmaf_rn(-0.5f, x, 2.5f), x, -4.f), x, 2.f);
  return 0.f;
}

// one thread per (sample x {image, target}, axis, output index): float weights (AA bicubic) or the source index
__global__ void __launch_bounds__(128)
sec_coeffs_kernel(const int* __restrict__ jobs, int OH, int OW, float* __restrict__ wts, int2* __restrict__ bounds) {
  const int axis = blockIdx.y;                // 0: x, out = OW; 1: y, out = OH
  const int out = axis == 0 ? OW : OH;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int j = blockIdx.z;
  if (i >= out) return;
  const int* jb = jobs + j * PK_AUG_SEC_FIELDS;
  const int in = axis == 0 ? jb[3] : jb[2];
  const size_t row = (static_cast<size_t>(j) * 2 + axis) * OH + i;
  const float scale = __fdiv_rn(static_cast<float>(in), static_cast<float>(out));
  if (jb[4] == 1) {   // upsample_nearest2d: min(floor(i * scale), in - 1)
    const int s = static_cast<int>(floorf(__fmul_rn(static_cast<float>(i), scale)));
    bounds[row] = make_int2(s < in - 1 ? s : in - 1, 1);
    return;
  }
  const float support = scale >= 1.f ? __fmul_rn(2.f, scale) : 2.f;
  const float invscale = scale >= 1.f ? __double2float_rn(__ddiv_rn(1.0, static_cast<double>(scale))) : 1.f;
  const float center = __double2float_rn(__dmul_rn(static_cast<double>(scale), static_cast<double>(i) + 0.5));
  int xmin = static_cast<int>(__dadd_rn(static_cast<double>(__fsub_rn(center, support)), 0.5));
  if (xmin < 0) xmin = 0;
  int xsize = static_cast<int>(__dadd_rn(static_cast<double>(__fadd_rn(center, support)), 0.5));
  if (xsize > in) xsize = in;
  xsize -= xmin;
  if (xsize > PK_AUG_AA_TAPS) xsize = PK_AUG_AA_TAPS;
  if (xsize < 0) xsize = 0;
  float w[PK_AUG_AA_TAPS];
  float tot = 0.f;
#pragma unroll
  for (int k = 0; k < PK_AUG_AA_TAPS; ++k) {
    w[k] = 0.f;
    if (k < xsize) {
      const float d = __fsub_rn(static_cast<float>(k + xmin), center);
      w[k] = aa_cubic(__double2float_rn(__dmul_rn(__dadd_rn(static_cast<double>(d), 0.5), static_cast<double>(invscale))));
      tot = __fadd_rn(tot, w[k]);
    }
  }
  float* o = wts + row * PK_AUG_AA_TAPS;
#pragma unroll
  for (int k = 0; k < PK_AUG_AA_TAPS; ++k) o[k] = (k < xsize && tot != 0.f) ? __fdiv_rn(w[k], tot) : w[k];
  bounds[row] = make_int2(xmin, xsize);
}

__device__ __forceinline__ float aa_dot(const float* p, long long stride, const float* w, int n) {
  float acc = __fmul_rn(p[0], w[0]);
  for (int k = 1; k < n; ++k) acc = __fmaf_rn(p[k * stride], w[k], acc);
  return acc;
}

// horizontal pass over rows [top, top + h) of the crop: [3, h, w] -> tmp [3, h, OW]
__global__ void __launch_bounds__(256)
sec_hpass_kernel(const float* __restrict__ img, const float* __restrict__ tgt, const int* __restrict__ jobs, int OH,
                 int OW, const float* __restrict__ wts, const int2* __restrict__ bounds, float* __restrict__ tmp) {
  const int j = blockIdx.z;
  const int* jb = jobs + j * PK_AUG_SEC_FIELDS;
  const int top = jb[0], left = jb[1], h = jb[2];
  const float* src = ((j & 1) ? tgt : img) + static_cast<size_t>(j >> 1) * 3 * OH * OW;
  float* out = tmp + static_cast<size_t>(j) * 3 * OH * OW;
  const int2* bx = bounds + static_cast<size_t>(j) * 2 * OH;
  const float* wx = wts + static_cast<size_t>(j) * 2 * OH * PK_AUG_AA_TAPS;
  const int n = 3 * h * OW;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int xx = i % OW, cy = i / OW, y = cy % h, c = cy / h;
    const int2 b = bx[xx];
    const float* p = src + (static_cast<size_t>(c) * OH + top + y) * OW + left + b.x;
    out[i] = jb[4] == 1 ? p[0] : aa_dot(p, 1, wx + static_cast<size_t>(xx) * PK_AUG_AA_TAPS, b.y);
  }
}

// vertical pass: tmp [3, h, OW] -> out [3, OH, OW]
__global__ void __launch_bounds__(256)
sec_vpass_kernel(const float* __restrict__ tmp, const int* __restrict__ jobs, int OH, int OW,
                 const float* __restrict__ wts, const int2* __restrict__ bounds, float* __restrict__ img_out,
                 float* __restrict__ tgt_out) {
  const int j = blockIdx.z;
  const int* jb = jobs + j * PK_AUG_SEC_FIELDS;
  const int h = jb[2];
  const float* in = tmp + static_cast<size_t>(j) * 3 * OH * OW;
  float* out = ((j & 1) ? tgt_out : img_out) + static_cast<size_t>(j >> 1) * 3 * OH * OW;
  const int2* by = bounds + (static_cast<size_t>(j) * 2 + 1) * OH;
  const float* wy = wts + (static_cast<size_t>(j) * 2 + 1) * OH * PK_AUG_AA_TAPS;
  const int n = 3 * OH * OW;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int xx = i % OW, cy = i / OW, yy = cy % OH, c = cy / OH;
    const int2 b = by[yy];
    const float* p = in + (static_cast<size_t>(c) * h + b.x) * OW + xx;
    out[i] = jb[4] == 1 ? p[0] : aa_dot(p, OW, wy + static_cast<size_t>(yy) * PK_AUG_AA_TAPS, b.y);
  }
}

}  // namespace pk

using namespace pk;

static int grid_for(long long n, int per_job) {
  long long g = (n + 255) / 256;
  const long long cap = (static_cast<long long>(sm_count()) * 8 + per_job - 1) / per_job;
  if (g > cap) g = cap;
  return static_cast<int>(g < 1 ? 1 : g);
}

extern "C" int pk_aug_resized_crop(const uint8_t* src, const int* jobs, int J, int S, int KP, int max_rows,
                                   int* coef, int* bounds, uint8_t* tmp, uint8_t* dst, void* stream) {
  PK_CHECK(src && jobs && coef && bounds && tmp && dst && J > 0 && S > 0 && KP > 0 && max_rows > 0,
           "pk_aug_resized_crop: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int2* b2 = reinterpret_cast<int2*>(bounds);
  crop_coeffs_kernel<<<dim3((S + 127) / 128, 2, J), 128, 0, st>>>(jobs, S, KP, coef, b2);
  PK_LAUNCH_CHECK("pk_aug_resized_crop(coeffs)");
  crop_pass1_kernel<<<dim3(grid_for(static_cast<long long>(max_rows) * S, J), 1, J), 256, 0, st>>>(
      src, jobs, S, KP, coef, b2, tmp);
  PK_LAUNCH_CHECK("pk_aug_resized_crop(first pass)");
  crop_pass2_kernel<<<dim3(grid_for(static_cast<long long>(S) * S, J), 1, J), 256, 0, st>>>(
      src, jobs, S, KP, coef, b2, tmp, dst);
  PK_LAUNCH_CHECK("pk_aug_resized_crop(second pass)");
  return 0;
}

extern "C" int pk_aug_color_jitter(uint8_t* imgs, const int* jobs, int n, long long npix, void* stream) {
  PK_CHECK(imgs && jobs && n >= 0 && npix > 0, "pk_aug_color_jitter: bad arguments");
  if (n == 0) return 0;
  jitter_kernel<<<n, 1024, 0, static_cast<cudaStream_t>(stream)>>>(imgs, jobs, npix);
  PK_LAUNCH_CHECK("pk_aug_color_jitter");
  return 0;
}

extern "C" int pk_aug_normalize(const uint8_t* slots, int B, int P, int S, float* img, float* tgt, void* stream) {
  PK_CHECK(slots && img && tgt && B > 0 && P > 0 && S > 0, "pk_aug_normalize: bad arguments");
  normalize_kernel<<<dim3(grid_for(static_cast<long long>(S) * S, 2 * B * P), 2 * B * P), 256, 0,
                     static_cast<cudaStream_t>(stream)>>>(slots, P, S, img, tgt);
  PK_LAUNCH_CHECK("pk_aug_normalize");
  return 0;
}

extern "C" int pk_aug_second_crop(const float* img, const float* tgt, const int* jobs, int B, int OH, int OW,
                                  float* wts, int* bounds, float* tmp, float* img_out, float* tgt_out, void* stream) {
  PK_CHECK(img && tgt && jobs && wts && bounds && tmp && img_out && tgt_out && B > 0 && OH >= OW && OW > 0,
           "pk_aug_second_crop: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int2* b2 = reinterpret_cast<int2*>(bounds);
  sec_coeffs_kernel<<<dim3((OH + 127) / 128, 2, 2 * B), 128, 0, st>>>(jobs, OH, OW, wts, b2);
  PK_LAUNCH_CHECK("pk_aug_second_crop(coeffs)");
  const long long n = 3LL * OH * OW;
  sec_hpass_kernel<<<dim3(grid_for(n, 2 * B), 1, 2 * B), 256, 0, st>>>(img, tgt, jobs, OH, OW, wts, b2, tmp);
  PK_LAUNCH_CHECK("pk_aug_second_crop(horizontal)");
  sec_vpass_kernel<<<dim3(grid_for(n, 2 * B), 1, 2 * B), 256, 0, st>>>(tmp, jobs, OH, OW, wts, b2, img_out, tgt_out);
  PK_LAUNCH_CHECK("pk_aug_second_crop(vertical)");
  return 0;
}
