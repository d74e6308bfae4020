// painter_b200 — COCO panoptic post-processing on the device (painter_b200/panoptic.py): the instance decoding, matrix
// NMS, class vote and panoptic merge of Painter/eval/coco_panoptic, computed from run_batch's device outputs.
//
//  pk_pano_candidates / _select   COCOCAInstSegEvaluatorCustom.py:252-325 (post_process_segm_output_by_threshold: one
//                                 candidate mask per (palette colour, threshold), maskness, the first sort, top 2000)
//  pk_pano_pack / _gram / _nms    util/matrix_nms.py:43-121 (mask_matrix_nms: the intersection matrix, the gaussian
//                                 decay, the second sort, top max_num)
//  pk_pano_minmax*                COCOCAInstSegEvaluatorCustom.py:172-250 (post_process_segm_output_by_minmax)
//  pk_pano_vote                   COCOPanoEvaluatorCustom.py:259-276 / COCOInstSegEvaluatorCustom.py:169-194
//                                 (merge_inst_semseg_result_to_instseg, dist_type 'abs')
//  pk_pano_merge                  COCOPanoEvaluatorCustom.py:47-134 (combine_semantic_and_instance_outputs_custom)
//
// Candidate masks are implicit: candidate (t, c) is {p : dist(p, c) < thr_t} with dist = fp32(L1(pix_p, P_c)) / 3 as
// torch computes it on the device (the L1 sum times the fp32 reciprocal of 3).  dist depends on the integer L1 sum s
// (0..765) alone and is monotone in it, so the mask is {p : s < bound_t}, with bound_t the count of s whose dist is
// below thr_t (computed on the host).  Every dist is a multiple of 2^-25 below 256: the maskness sums are int64
// fixed-point, exact and independent of order.  Kept masks are materialised once as bit rows (bit p of row i: pixel p
// in mask i, rows padded with zeros to a multiple of 1024 bits); intersection counts are AND-popcount products of
// those rows on the tensor cores (mma.sync b1), exact.  Matrix NMS restates the reference's fp32 expressions with
// explicitly rounded operations and the same expf.  The class vote sums 1 - d / max d (an fp32 value, a multiple of
// 2^-24 in [0, 1]) as int64 fixed-point, exact.  Every sort is stable on explicit keys.  Results are bitwise
// reproducible; no kernel synchronises with the host.
#include <climits>

#include <cub/device/device_segmented_radix_sort.cuh>

#include "common.cuh"
#include "host_common.h"
#include "../../include/painter_b200.h"

namespace pk {

constexpr int kPanoMaxPalette = PK_PANO_MAX_PALETTE;   // 6400 instance colours
constexpr int kPanoMaxThr = PK_PANO_MAX_THR;
constexpr int kSemMax = 200;
constexpr int kVoteClasses = 80;                       // the vote reads the first 80 (thing) colours
constexpr float kFx25 = 33554432.0f;                   // 2^25
constexpr float kFx24 = 16777216.0f;                   // 2^24

struct PanoItem {
  const uint8_t* px;
  long long aux;
  int H, W;
};
__device__ __forceinline__ PanoItem pano_item(const long long* items, const uint8_t* base, int i) {
  const long long* r = items + static_cast<size_t>(i) * PK_PANO_FIELDS;
  PanoItem it;
  it.px = r[1] == 1 ? base + r[0] : reinterpret_cast<const uint8_t*>(r[0]);
  it.aux = r[1];
  it.H = static_cast<int>(r[2]);
  it.W = static_cast<int>(r[3]);
  return it;
}

__device__ __forceinline__ uint32_t rgb_at(const uint8_t* px, long long p) {
  return static_cast<uint32_t>(px[3 * p]) | (static_cast<uint32_t>(px[3 * p + 1]) << 8) |
         (static_cast<uint32_t>(px[3 * p + 2]) << 16);
}

__device__ __forceinline__ void stage_colours(const uint8_t* palette, int P, uint32_t* pal) {
  for (int k = threadIdx.x; k < P; k += blockDim.x)
    pal[k] = static_cast<uint32_t>(palette[3 * k]) | (static_cast<uint32_t>(palette[3 * k + 1]) << 8) |
             (static_cast<uint32_t>(palette[3 * k + 2]) << 16);
}

// torch's CUDA `fp32 tensor / 3.` multiplies by the fp32 reciprocal; as an int64 multiple of 2^-25
__device__ __forceinline__ float sad_dist(int s) { return __fmul_rn(static_cast<float>(s), 1.0f / 3.0f); }
__device__ __forceinline__ long long sad_fx(int s) { return __float2ll_rn(__fmul_rn(sad_dist(s), kFx25)); }

__device__ __forceinline__ long long warp_sum_ll(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct Bounds {
  int b[kPanoMaxThr];
  // constant indices only: a dynamic index would place the struct in local memory
  __device__ __forceinline__ int at(int t) const { return t == 0 ? b[0] : t == 1 ? b[1] : t == 2 ? b[2] : b[3]; }
};

// ------------------------------------------------------------------------------------------------------------------
// Candidate statistics.  CTA (x, image) takes a grid-stride share of the pixels; every lane compares its pixel with
// every palette colour (shared memory).  Iterations where a lane of the warp is within the largest bound are rare:
// the warp then sums, per threshold, its hit count and fixed-point dist and one lane adds them to area / sumfx.
constexpr int kCandThreads = 256;
__global__ void __launch_bounds__(kCandThreads)
pano_candidates_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base,
                       const uint8_t* __restrict__ palette, int P, Bounds bounds, int T, int* __restrict__ area,
                       unsigned long long* __restrict__ sumfx) {
  __shared__ uint32_t pal[kPanoMaxPalette];
  __shared__ int bnd[kPanoMaxThr];
  const PanoItem it = pano_item(items, base, blockIdx.y);
  const long long npix = static_cast<long long>(it.H) * it.W;
  const long long first = static_cast<long long>(blockIdx.x) * kCandThreads;
  if (first >= npix) return;
  stage_colours(palette, P, pal);
  if (threadIdx.x < kPanoMaxThr) bnd[threadIdx.x] = bounds.at(threadIdx.x);
  __syncthreads();
  int smax = 0;
  for (int t = 0; t < T; ++t) smax = max(smax, bnd[t]);
  int* ar = area + static_cast<size_t>(blockIdx.y) * T * P;
  unsigned long long* sm = sumfx + static_cast<size_t>(blockIdx.y) * T * P;
  const int lane = threadIdx.x & 31;
  const long long stride = static_cast<long long>(gridDim.x) * kCandThreads;
  for (long long b0 = first; b0 < npix; b0 += stride) {          // b0 is warp-uniform: every lane takes part
    const long long p = b0 + threadIdx.x;
    const bool valid = p < npix;
    const uint32_t c = valid ? rgb_at(it.px, p) : 0u;
    const int lim = valid ? smax : 0;
#pragma unroll 4
    for (int k = 0; k < P; ++k) {
      const int s = static_cast<int>(__vsadu4(c, pal[k]));
      const unsigned m = __ballot_sync(0xffffffffu, s < lim);
      if (m) {
        const long long fx = sad_fx(s);
        for (int t = 0; t < T; ++t) {
          const bool h = valid && s < bnd[t];
          const unsigned mh = __ballot_sync(0xffffffffu, h);
          if (!mh) continue;
          const long long v = warp_sum_ll(h ? fx : 0ll);
          if (lane == 0) {
            atomicAdd(&ar[t * P + k], __popc(mh));
            atomicAdd(&sm[t * P + k], static_cast<unsigned long long>(v));
          }
        }
      }
    }
  }
}

__device__ __forceinline__ float maskness(long long fx, int area) {
  return __fdiv_rn(__fmul_rn(__ll2float_rn(fx), 1.0f / kFx25), static_cast<float>(area));
}

// Sort keys: (maskness bits, candidate index) for non-empty candidates (maskness >= 0: its bits order as the value),
// all ones for empty ones.  Candidate index = t * P + c (threshold-major, palette order).
__global__ void pano_keys_kernel(const int* __restrict__ area, const unsigned long long* __restrict__ sumfx, int n,
                                 int NC, unsigned long long* __restrict__ keys, int* __restrict__ offsets) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i <= n && i < static_cast<long long>(n) * NC + 1 && i <= n) offsets[i] = static_cast<int>(i * NC);
  if (i >= static_cast<long long>(n) * NC) return;
  const int a = area[i];
  unsigned long long key = ~0ull;
  if (a > 0) {
    const float m = maskness(static_cast<long long>(sumfx[i]), a);
    key = (static_cast<unsigned long long>(__float_as_uint(m)) << 32) | static_cast<unsigned>(i % NC);
  }
  keys[i] = key;
}

// One CTA per image: the first `keep` non-empty sorted keys become the kept candidates, with
// score = 1 - m / max(max m, 1) (the largest kept m is the last one).
__global__ void __launch_bounds__(256)
pano_select_kernel(const unsigned long long* __restrict__ sorted, int NC, int keep, int ncap, int* __restrict__ count,
                   int* __restrict__ cand, float* __restrict__ scores) {
  __shared__ int s_n;
  const unsigned long long* k = sorted + static_cast<size_t>(blockIdx.x) * NC;
  if (threadIdx.x == 0) s_n = 0;
  __syncthreads();
  // keys are ascending with the empty ones last: the kept count is the first empty position, capped at keep
  const int lim = min(keep, NC);
  for (int i = threadIdx.x; i < lim; i += blockDim.x) {
    const bool full = k[i] != ~0ull;
    const bool next_empty = i + 1 == lim || k[i + 1] == ~0ull;
    if (full && next_empty) s_n = i + 1;
  }
  __syncthreads();
  const int n = s_n;
  const float mmax = n ? __uint_as_float(static_cast<unsigned>(k[n - 1] >> 32)) : 0.0f;
  const float den = fmaxf(mmax, 1.0f);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float m = __uint_as_float(static_cast<unsigned>(k[i] >> 32));
    cand[static_cast<size_t>(blockIdx.x) * ncap + i] = static_cast<int>(k[i] & 0xffffffffu);
    scores[static_cast<size_t>(blockIdx.x) * ncap + i] = __fsub_rn(1.0f, __fdiv_rn(m, den));
  }
  if (threadIdx.x == 0) count[blockIdx.x] = n;
}

// ------------------------------------------------------------------------------------------------------------------
// Bit rows.  Warp w of a CTA builds 32 consecutive words (1024 pixels): in step j its lanes test pixels 32 j + lane
// and the ballot is word j.  Rows of images smaller than the row width are padded with zeros.
constexpr int kPackThreads = 256;
__global__ void __launch_bounds__(kPackThreads)
pano_pack_candidates_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base,
                            const uint8_t* __restrict__ palette, int P, Bounds bounds, const int* __restrict__ cand,
                            const int* __restrict__ count, int ncap, int words, uint32_t* __restrict__ bits) {
  const int row = blockIdx.y, img = blockIdx.z;
  if (row >= count[img]) return;
  const PanoItem it = pano_item(items, base, img);
  const long long npix = static_cast<long long>(it.H) * it.W;
  const int ci = cand[static_cast<size_t>(img) * ncap + row];
  const int t = ci / P, c = ci % P;
  const uint32_t col = static_cast<uint32_t>(palette[3 * c]) | (static_cast<uint32_t>(palette[3 * c + 1]) << 8) |
                       (static_cast<uint32_t>(palette[3 * c + 2]) << 16);
  const int bound = bounds.at(t);
  const int lane = threadIdx.x & 31;
  const long long w0 = (static_cast<long long>(blockIdx.x) * (kPackThreads / 32) + (threadIdx.x >> 5)) * 32;
  if (w0 >= words) return;
  uint32_t mine = 0;
#pragma unroll 4
  for (int j = 0; j < 32; ++j) {
    const long long p = (w0 + j) * 32 + lane;
    const bool in = p < npix && static_cast<int>(__vsadu4(rgb_at(it.px, p), col)) < bound;
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if (lane == j) mine = b;
  }
  bits[(static_cast<size_t>(img) * ncap + row) * words + w0 + lane] = mine;
}

// Bit rows of explicit masks: items rows [bool [n, H, W] address, n, H, W]; aux rows [fp32 scores [n] address, int64
// classes [n] address or 0], gathered into scores / classes [images, ncap].
__global__ void __launch_bounds__(kPackThreads)
pano_pack_masks_kernel(const long long* __restrict__ items, int ncap, int words, uint32_t* __restrict__ bits,
                       const long long* __restrict__ aux, float* __restrict__ scores, long long* __restrict__ classes) {
  const long long* r = items + static_cast<size_t>(blockIdx.z) * PK_PANO_FIELDS;
  const int row = blockIdx.y;
  if (row >= r[1]) return;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const long long* a = aux + static_cast<size_t>(blockIdx.z) * 2;
    const size_t o = static_cast<size_t>(blockIdx.z) * ncap + row;
    scores[o] = reinterpret_cast<const float*>(a[0])[row];
    if (classes && a[1]) classes[o] = reinterpret_cast<const long long*>(a[1])[row];
  }
  const long long npix = r[2] * r[3];
  const uint8_t* m = reinterpret_cast<const uint8_t*>(r[0]) + static_cast<size_t>(row) * npix;
  const int lane = threadIdx.x & 31;
  const long long w0 = (static_cast<long long>(blockIdx.x) * (kPackThreads / 32) + (threadIdx.x >> 5)) * 32;
  if (w0 >= words) return;
  uint32_t mine = 0;
#pragma unroll 4
  for (int j = 0; j < 32; ++j) {
    const long long p = (w0 + j) * 32 + lane;
    const unsigned b = __ballot_sync(0xffffffffu, p < npix && m[p] != 0);
    if (lane == j) mine = b;
  }
  bits[(static_cast<size_t>(blockIdx.z) * ncap + row) * words + w0 + lane] = mine;
}

// ------------------------------------------------------------------------------------------------------------------
// Intersection Gram matrix: gram[i][j] = popc(row_i AND row_j) for the tiles of 128 x 128 on or above the diagonal of
// every image's count x count matrix.  mma.sync m16n8k256 b1 AND-popc, s32 accumulators; a three-stage cp.async ring
// of 1024-bit K slices (128 rows x 32 words per operand, row stride 36 words: fragment loads are conflict-free).
// 8 warps as 2 x 4, a 64 x 32 warp tile of 4 x 4 mma tiles.
constexpr int kGramTile = 128;
constexpr int kGramKW = 32;                 // words per stage
constexpr int kGramLd = 36;
constexpr int kGramStages = 3;
constexpr int kGramThreads = 256;
constexpr size_t kGramSmem = static_cast<size_t>(kGramStages) * 2 * kGramTile * kGramLd * 4;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const unsigned s = static_cast<unsigned>(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void mma_b1(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k256.row.col.s32.b1.b1.s32.and.popc {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
      "{%0,%1,%2,%3};\n"
      : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(kGramThreads)
pano_gram_kernel(const uint32_t* __restrict__ bits, int ncap, int words, const int* __restrict__ count,
                 int* __restrict__ gram) {
  extern __shared__ __align__(16) uint32_t gsm[];
  const int tiles = ncap / kGramTile;
  int t = blockIdx.x, ti = 0;
  while (t >= tiles - ti) {
    t -= tiles - ti;
    ++ti;
  }
  const int tj = ti + t;
  const int img = blockIdx.y;
  const int n = count[img];
  if (tj * kGramTile >= n) return;                       // tj >= ti: the whole tile is past the last row or column
  const uint32_t* A = bits + (static_cast<size_t>(img) * ncap + ti * kGramTile) * words;
  const uint32_t* B = bits + (static_cast<size_t>(img) * ncap + tj * kGramTile) * words;
  const int ksteps = words / kGramKW;
  auto load = [&](int ks, int stage) {
    uint32_t* sa = gsm + stage * 2 * kGramTile * kGramLd;
    uint32_t* sb = sa + kGramTile * kGramLd;
#pragma unroll
    for (int q = 0; q < 4; ++q) {                         // 128 rows x 8 chunks of 16 bytes, per operand
      const int idx = threadIdx.x + q * kGramThreads;
      const int r = idx >> 3, ch = idx & 7;
      cp_async16(sa + r * kGramLd + ch * 4, A + static_cast<size_t>(r) * words + ks * kGramKW + ch * 4);
      cp_async16(sb + r * kGramLd + ch * 4, B + static_cast<size_t>(r) * words + ks * kGramKW + ch * 4);
    }
  };
#pragma unroll
  for (int s = 0; s < kGramStages - 1; ++s) {
    if (s < ksteps) load(s, s);
    cp_async_commit();
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, q = lane & 3;
  const int wm = (warp >> 2) * 64, wn = (warp & 3) * 32;
  int acc[4][4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0;
  for (int ks = 0; ks < ksteps; ++ks) {
    cp_async_wait<kGramStages - 2>();
    __syncthreads();
    const int nxt = ks + kGramStages - 1;
    if (nxt < ksteps) load(nxt, nxt % kGramStages);
    cp_async_commit();
    const uint32_t* sa = gsm + (ks % kGramStages) * 2 * kGramTile * kGramLd;
    const uint32_t* sb = sa + kGramTile * kGramLd;
#pragma unroll
    for (int kk = 0; kk < kGramKW; kk += 8) {            // 256 bits per mma
      uint32_t a[4][4], b[4][2];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t* r0 = sa + (wm + i * 16 + g) * kGramLd + kk + q;
        a[i][0] = r0[0];
        a[i][1] = r0[8 * kGramLd];
        a[i][2] = r0[4];
        a[i][3] = r0[8 * kGramLd + 4];
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t* r0 = sb + (wn + j * 8 + g) * kGramLd + kk + q;
        b[j][0] = r0[0];
        b[j][1] = r0[4];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) mma_b1(acc[i][j], a[i], b[j][0], b[j][1]);
    }
  }
  cp_async_wait<0>();
  int* G = gram + static_cast<size_t>(img) * ncap * ncap;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = ti * kGramTile + wm + i * 16 + g;
      const int c = tj * kGramTile + wn + j * 8 + 2 * q;
      *reinterpret_cast<int2*>(G + static_cast<size_t>(r) * ncap + c) = make_int2(acc[i][j][0], acc[i][j][1]);
      *reinterpret_cast<int2*>(G + static_cast<size_t>(r + 8) * ncap + c) = make_int2(acc[i][j][2], acc[i][j][3]);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Matrix NMS (one thread per sorted column j, CTA (x, image)).  Ranks: a stable descending order of fp32 scores.
constexpr int kNmsThreads = 256;
__global__ void __launch_bounds__(kNmsThreads)
pano_rank_kernel(const float* __restrict__ keys, const int* __restrict__ count, int ncap, int* __restrict__ perm) {
  extern __shared__ float rk[];
  const int img = blockIdx.y, n = count[img];
  if (blockIdx.x * kNmsThreads >= n) return;
  const float* k = keys + static_cast<size_t>(img) * ncap;
  for (int i = threadIdx.x; i < n; i += kNmsThreads) rk[i] = k[i];
  __syncthreads();
  const int j = blockIdx.x * kNmsThreads + threadIdx.x;
  if (j >= n) return;
  const float v = rk[j];
  int r = 0;
  for (int i = 0; i < n; ++i) r += rk[i] > v || (rk[i] == v && i < j);
  perm[static_cast<size_t>(img) * ncap + r] = j;
}

__device__ __forceinline__ float pair_iou(const int* G, int ncap, int a, int b) {
  const int lo = min(a, b), hi = max(a, b);
  const float inter = static_cast<float>(G[static_cast<size_t>(lo) * ncap + hi]);
  const float ai = static_cast<float>(G[static_cast<size_t>(a) * ncap + a]);
  const float bj = static_cast<float>(G[static_cast<size_t>(b) * ncap + b]);
  // (area[j] + area[i]) - inter, then the division, as the reference's fp32 tensor expression
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(bj, ai), inter));
}

// comp[j] = max over sorted rows i < j with the same label of iou(i, j) (0 when there is none)
__global__ void __launch_bounds__(kNmsThreads)
pano_nms_comp_kernel(const int* __restrict__ gram, const long long* __restrict__ labels, const int* __restrict__ count,
                     int ncap, const int* __restrict__ perm, float* __restrict__ comp) {
  const int img = blockIdx.y, n = count[img];
  const int j = blockIdx.x * kNmsThreads + threadIdx.x;
  if (j >= n) return;
  const int* G = gram + static_cast<size_t>(img) * ncap * ncap;
  const int* pm = perm + static_cast<size_t>(img) * ncap;
  const long long* lb = labels ? labels + static_cast<size_t>(img) * ncap : nullptr;
  const int oj = pm[j];
  float c = 0.0f;
#pragma unroll 1
  for (int i = 0; i < j; ++i) {
    const int oi = pm[i];
    if (lb && lb[oi] != lb[oj]) continue;
    c = fmaxf(c, pair_iou(G, ncap, oi, oj));
  }
  comp[static_cast<size_t>(img) * ncap + j] = c;
}

// decayed[j] = score(j) * min over every sorted row i of exp(-sigma iou(i, j)^2) / exp(-sigma comp[i]^2), with
// iou(i, j) = 0 for i >= j or different labels (the zero entries of the reference's triangle)
__global__ void __launch_bounds__(kNmsThreads)
pano_nms_decay_kernel(const int* __restrict__ gram, const long long* __restrict__ labels,
                      const int* __restrict__ count, int ncap, const int* __restrict__ perm,
                      const float* __restrict__ comp, const float* __restrict__ scores, float neg_sigma,
                      float* __restrict__ decayed) {
  const int img = blockIdx.y, n = count[img];
  const int j = blockIdx.x * kNmsThreads + threadIdx.x;
  if (j >= n) return;
  const int* G = gram + static_cast<size_t>(img) * ncap * ncap;
  const int* pm = perm + static_cast<size_t>(img) * ncap;
  const float* cp = comp + static_cast<size_t>(img) * ncap;
  const long long* lb = labels ? labels + static_cast<size_t>(img) * ncap : nullptr;
  const int oj = pm[j];
  float coef = INFINITY;
  for (int i = 0; i < n; ++i) {
    float d = 0.0f;
    if (i < j) {
      const int oi = pm[i];
      if (!lb || lb[oi] == lb[oj]) d = pair_iou(G, ncap, oi, oj);
    }
    const float ci = cp[i];
    const float r = __fdiv_rn(expf(__fmul_rn(neg_sigma, __fmul_rn(d, d))), expf(__fmul_rn(neg_sigma, __fmul_rn(ci, ci))));
    coef = fminf(coef, r);
  }
  decayed[static_cast<size_t>(img) * ncap + j] = __fmul_rn(scores[static_cast<size_t>(img) * ncap + oj], coef);
}

// The final order: rows[r] = the input index of the r-th largest decayed score (stable), r < max_num; an image with
// no candidate gets the one empty row (-1, score 0, label 0) when empty_one != 0.
__global__ void __launch_bounds__(kNmsThreads)
pano_nms_out_kernel(const float* __restrict__ decayed, const int* __restrict__ count, int ncap,
                    const int* __restrict__ perm, const int* __restrict__ perm2, int max_num, int empty_one,
                    const long long* __restrict__ labels, int* __restrict__ rows, float* __restrict__ out_scores,
                    int* __restrict__ out_count, long long* __restrict__ out_labels) {
  const int img = blockIdx.y, n = count[img];
  const int r = blockIdx.x * kNmsThreads + threadIdx.x;
  const size_t o = static_cast<size_t>(img) * max_num;
  if (r == 0) out_count[img] = n ? min(n, max_num) : (empty_one ? 1 : 0);
  if (n == 0 && r == 0 && empty_one) {
    rows[o] = -1;
    out_scores[o] = 0.0f;
    if (out_labels) out_labels[o] = 0;
  }
  if (r >= min(n, max_num)) return;
  const int j = perm2[static_cast<size_t>(img) * ncap + r];
  const int row = perm ? perm[static_cast<size_t>(img) * ncap + j] : j;
  rows[o + r] = row;
  out_scores[o + r] = decayed[static_cast<size_t>(img) * ncap + j];
  // labels[row], or 1 (the class-agnostic decoding's label) without labels
  if (out_labels) out_labels[o + r] = labels ? labels[static_cast<size_t>(img) * ncap + row] : 1;
}

// ------------------------------------------------------------------------------------------------------------------
// Masks out: out[i][p] = bit p of row rows[i] (all zeros for row -1).  outs rows: [bool [n, H, W] address, n, H, W].
__global__ void __launch_bounds__(256)
pano_unpack_kernel(const uint32_t* __restrict__ bits, int ncap, int words, const int* __restrict__ rows, int rows_ld,
                   const long long* __restrict__ outs) {
  const long long* r = outs + static_cast<size_t>(blockIdx.z) * PK_PANO_FIELDS;
  const int i = blockIdx.y;
  if (i >= r[1]) return;
  const long long npix = r[2] * r[3];
  const int row = rows[static_cast<size_t>(blockIdx.z) * rows_ld + i];
  uint8_t* out = reinterpret_cast<uint8_t*>(r[0]) + static_cast<size_t>(i) * npix;
  const uint32_t* src = bits + (static_cast<size_t>(blockIdx.z) * ncap + (row < 0 ? 0 : row)) * words;
  for (long long p = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; p < npix;
       p += static_cast<long long>(gridDim.x) * 256)
    out[p] = row < 0 ? 0 : static_cast<uint8_t>((src[p >> 5] >> (p & 31)) & 1u);
}

// ------------------------------------------------------------------------------------------------------------------
// Minmax: per pixel the first nearest of the P colours and black (index P) by L1; per colour its pixel count and
// integer L1 sum.
__global__ void __launch_bounds__(kCandThreads)
pano_minmax_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base,
                   const uint8_t* __restrict__ palette, int P, long long max_pix, short* __restrict__ pred,
                   int* __restrict__ cnt, unsigned long long* __restrict__ sum) {
  __shared__ uint32_t pal[kPanoMaxPalette + 1];
  const PanoItem it = pano_item(items, base, blockIdx.y);
  const long long npix = static_cast<long long>(it.H) * it.W;
  const long long first = static_cast<long long>(blockIdx.x) * kCandThreads;
  if (first >= npix) return;
  stage_colours(palette, P, pal);
  if (threadIdx.x == 0) pal[P] = 0u;
  __syncthreads();
  int* cn = cnt + static_cast<size_t>(blockIdx.y) * (P + 1);
  unsigned long long* sm = sum + static_cast<size_t>(blockIdx.y) * (P + 1);
  for (long long p = first + threadIdx.x; p < npix; p += static_cast<long long>(gridDim.x) * kCandThreads) {
    const uint32_t c = rgb_at(it.px, p);
    int best = INT_MAX, idx = 0;
#pragma unroll 4
    for (int k = 0; k <= P; ++k) {
      const int s = static_cast<int>(__vsadu4(c, pal[k]));
      if (s < best) {
        best = s;
        idx = k;
      }
    }
    pred[static_cast<size_t>(blockIdx.y) * max_pix + p] = static_cast<short>(idx);
    atomicAdd(&cn[idx], 1);
    atomicAdd(&sm[idx], static_cast<unsigned long long>(best));
  }
}

// One CTA per image: the colours present, in index order; score = 1 - mean / max(max mean, 1); class 0 for black.
__global__ void __launch_bounds__(1024)
pano_minmax_select_kernel(const int* __restrict__ cnt, const unsigned long long* __restrict__ sum, int P1,
                          int* __restrict__ cols, float* __restrict__ scores, long long* __restrict__ classes,
                          int* __restrict__ count) {
  __shared__ int wsum[32];
  __shared__ float wmax[32];
  __shared__ int s_base;
  __shared__ float s_max;
  const int img = blockIdx.x;
  const int* cn = cnt + static_cast<size_t>(img) * P1;
  const unsigned long long* sm = sum + static_cast<size_t>(img) * P1;
  const size_t o = static_cast<size_t>(img) * P1;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float mx = 0.0f;
  for (int k = threadIdx.x; k < P1; k += 1024)
    if (cn[k]) mx = fmaxf(mx, __fdiv_rn(__ull2float_rn(sm[k]), static_cast<float>(cn[k])));
  for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
  if (lane == 0) wmax[warp] = mx;
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = 0.0f;
    for (int w = 0; w < 32; ++w) m = fmaxf(m, wmax[w]);
    s_max = fmaxf(m, 1.0f);
  }
  __syncthreads();
  for (int k0 = 0; k0 < P1; k0 += 1024) {
    const int k = k0 + threadIdx.x;
    const bool present = k < P1 && cn[k] > 0;
    const unsigned b = __ballot_sync(0xffffffffu, present);
    if (lane == 0) wsum[warp] = __popc(b);
    __syncthreads();
    int before = s_base;
    for (int w = 0; w < warp; ++w) before += wsum[w];
    before += __popc(b & ((1u << lane) - 1u));
    if (present) {
      const float m = __fdiv_rn(__ull2float_rn(sm[k]), static_cast<float>(cn[k]));
      cols[o + before] = k;
      scores[o + before] = __fsub_rn(1.0f, __fdiv_rn(m, s_max));
      classes[o + before] = k == P1 - 1 ? 0 : 1;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int w = 0; w < 32; ++w) tot += wsum[w];
      s_base += tot;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) count[img] = s_base;
}

__global__ void __launch_bounds__(256)
pano_minmax_masks_kernel(const short* __restrict__ pred, long long max_pix, const int* __restrict__ cols, int P1,
                         const long long* __restrict__ outs) {
  const long long* r = outs + static_cast<size_t>(blockIdx.z) * PK_PANO_FIELDS;
  const int i = blockIdx.y;
  if (i >= r[1]) return;
  const long long npix = r[2] * r[3];
  const int col = cols[static_cast<size_t>(blockIdx.z) * P1 + i];
  const short* pm = pred + static_cast<size_t>(blockIdx.z) * max_pix;
  uint8_t* out = reinterpret_cast<uint8_t*>(r[0]) + static_cast<size_t>(i) * npix;
  for (long long p = static_cast<long long>(blockIdx.x) * 256 + threadIdx.x; p < npix;
       p += static_cast<long long>(gridDim.x) * 256)
    out[p] = pm[p] == col;
}

// ------------------------------------------------------------------------------------------------------------------
// Class vote.  dmax[img] = max over pixels and the first 80 colours of the L1 distance (zeroed by the caller).
__global__ void __launch_bounds__(256)
pano_sem_dmax_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base,
                     const uint8_t* __restrict__ palette, int* __restrict__ dmax) {
  __shared__ uint32_t pal[kVoteClasses];
  const PanoItem it = pano_item(items, base, blockIdx.y);
  const long long npix = static_cast<long long>(it.H) * it.W;
  const long long first = static_cast<long long>(blockIdx.x) * 256;
  if (first >= npix) return;
  stage_colours(palette, kVoteClasses, pal);
  __syncthreads();
  int mx = 0;
  for (long long p = first + threadIdx.x; p < npix; p += static_cast<long long>(gridDim.x) * 256) {
    const uint32_t c = rgb_at(it.px, p);
    for (int k = 0; k < kVoteClasses; ++k) mx = max(mx, static_cast<int>(__vsadu4(c, pal[k])));
  }
  for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0) atomicMax(&dmax[blockIdx.y], mx);
}

// CTA (instance, image): its warps walk the instance's bit row; for every pixel in the mask, lane l adds the
// fixed-point prob of colours l, l + 32, l + 64 (< 80).  The class is the first maximum of the exact sums.
constexpr int kVoteThreads = 256;
__global__ void __launch_bounds__(kVoteThreads)
pano_vote_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base,
                 const uint8_t* __restrict__ palette, const int* __restrict__ dmax, const uint32_t* __restrict__ bits,
                 int ncap, int words, const int* __restrict__ count, long long* __restrict__ classes) {
  __shared__ uint32_t pal[kVoteClasses];
  __shared__ long long prob[766];
  __shared__ long long part[kVoteThreads / 32][kVoteClasses];
  const int row = blockIdx.x, img = blockIdx.y;
  if (row >= count[img]) return;
  const PanoItem it = pano_item(items, base, img);
  stage_colours(palette, kVoteClasses, pal);
  const float dm = static_cast<float>(dmax[img]);
  for (int s = threadIdx.x; s < 766; s += kVoteThreads)
    prob[s] = __float2ll_rn(__fmul_rn(__fsub_rn(1.0f, __fdiv_rn(static_cast<float>(s), dm)), kFx24));
  __syncthreads();
  const uint32_t* src = bits + (static_cast<size_t>(img) * ncap + row) * words;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long v0 = 0, v1 = 0, v2 = 0;
  const bool has2 = lane + 64 < kVoteClasses;
  for (int w = warp; w < words; w += kVoteThreads / 32) {
    uint32_t word = src[w];
    while (word) {
      const int b = __ffs(word) - 1;
      word &= word - 1;
      const uint32_t c = rgb_at(it.px, static_cast<long long>(w) * 32 + b);
      v0 += prob[__vsadu4(c, pal[lane])];
      v1 += prob[__vsadu4(c, pal[lane + 32])];
      if (has2) v2 += prob[__vsadu4(c, pal[lane + 64])];
    }
  }
  part[warp][lane] = v0;
  part[warp][lane + 32] = v1;
  if (has2) part[warp][lane + 64] = v2;
  __syncthreads();
  if (threadIdx.x < kVoteClasses) {
    long long s = 0;
    for (int w = 0; w < kVoteThreads / 32; ++w) s += part[w][threadIdx.x];
    part[0][threadIdx.x] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int best = 0;
    for (int k = 1; k < kVoteClasses; ++k)
      if (part[0][k] > part[0][best]) best = k;
    classes[static_cast<size_t>(img) * ncap + row] = best;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Panoptic merge, one CTA per image.  labels: the semantic argmin map (uint8 [max_pix] per image).  The pixels
// claimed by instances are a bitmap in shared memory; instances are taken in stable descending score order.
// segs[img][s] = {instance index or -1, category, area (stuff), score bits (things)}; nseg[img] their count.
__global__ void __launch_bounds__(256)
pano_sem_labels_kernel(const long long* __restrict__ items, const uint8_t* __restrict__ base,
                       const uint8_t* __restrict__ palette, int K, long long max_pix, uint8_t* __restrict__ labels) {
  __shared__ uint32_t pal[kSemMax];
  const PanoItem it = pano_item(items, base, blockIdx.y);
  const long long npix = static_cast<long long>(it.H) * it.W;
  const long long first = static_cast<long long>(blockIdx.x) * 256;
  if (first >= npix) return;
  stage_colours(palette, K, pal);
  __syncthreads();
  for (long long p = first + threadIdx.x; p < npix; p += static_cast<long long>(gridDim.x) * 256) {
    const uint32_t c = rgb_at(it.px, p);
    int best = INT_MAX, idx = 0;
    for (int k = 0; k < K; ++k) {
      const int s = static_cast<int>(__vsadu4(c, pal[k]));
      if (s < best) {
        best = s;
        idx = k;
      }
    }
    labels[static_cast<size_t>(blockIdx.y) * max_pix + p] = static_cast<uint8_t>(idx);
  }
}

constexpr int kMergeThreads = 1024;
__device__ __forceinline__ void block_sum2(int& a, int& b, int (*red)[kMergeThreads / 32]) {
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int warp = threadIdx.x >> 5;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) {
    red[0][warp] = a;
    red[1][warp] = b;
  }
  __syncthreads();
  a = b = 0;
  for (int w = 0; w < kMergeThreads / 32; ++w) {
    a += red[0][w];
    b += red[1][w];
  }
}

__global__ void __launch_bounds__(kMergeThreads)
pano_merge_kernel(const long long* __restrict__ maps, const uint8_t* __restrict__ labels, long long max_pix, int K,
                  const uint32_t* __restrict__ bits, int ncap, int words, const float* __restrict__ scores,
                  const long long* __restrict__ classes, const int* __restrict__ count, double overlap,
                  double stuff_area, double score_thresh, int max_seg, long long* __restrict__ segs,
                  int* __restrict__ nseg) {
  extern __shared__ uint32_t claimed[];                 // words
  int* order = reinterpret_cast<int*>(claimed + words); // ncap
  __shared__ int red[2][kMergeThreads / 32];
  __shared__ int bins[kSemMax], present[kSemMax], segid[kSemMax];
  const int img = blockIdx.x, n = count[img];
  const long long* mr = maps + static_cast<size_t>(img) * PK_PANO_FIELDS;
  int* map = reinterpret_cast<int*>(mr[0]);
  const long long npix = mr[2] * mr[3];
  const float* sc = scores + static_cast<size_t>(img) * ncap;
  const long long* cl = classes + static_cast<size_t>(img) * ncap;
  const uint8_t* lab = labels + static_cast<size_t>(img) * max_pix;
  long long* sg = segs + static_cast<size_t>(img) * max_seg * 4;
  for (int w = threadIdx.x; w < words; w += kMergeThreads) claimed[w] = 0u;
  for (int k = threadIdx.x; k < kSemMax; k += kMergeThreads) bins[k] = present[k] = segid[k] = 0;
  for (int j = threadIdx.x; j < n; j += kMergeThreads) {
    const float v = sc[j];
    int r = 0;
    for (int i = 0; i < n; ++i) r += sc[i] > v || (sc[i] == v && i < j);
    order[r] = j;
  }
  __syncthreads();
  int seg = 0;
  for (int r = 0; r < n; ++r) {
    const int i = order[r];
    const float score = sc[i];
    if (static_cast<double>(score) < score_thresh) break;
    const uint32_t* row = bits + (static_cast<size_t>(img) * ncap + i) * words;
    int area = 0, inter = 0;
    for (int w = threadIdx.x; w < words; w += kMergeThreads) {
      const uint32_t m = row[w];
      area += __popc(m);
      inter += __popc(m & claimed[w]);
    }
    block_sum2(area, inter, red);
    if (area == 0) continue;
    if (static_cast<double>(inter) * 1.0 / static_cast<double>(area) > overlap) continue;
    ++seg;
    for (int w = threadIdx.x; w < words; w += kMergeThreads) {
      uint32_t fresh = row[w] & ~claimed[w];
      claimed[w] |= fresh;
      while (fresh) {
        const int b = __ffs(fresh) - 1;
        fresh &= fresh - 1;
        map[static_cast<long long>(w) * 32 + b] = seg;
      }
    }
    if (threadIdx.x == 0) {
      long long* s = sg + static_cast<size_t>(seg - 1) * 4;
      s[0] = i;
      s[1] = cl[i];
      s[2] = area;
      s[3] = __float_as_uint(score);
    }
    __syncthreads();
  }
  // stuff: every semantic label >= 80 present in the map, in ascending order, over the pixels no instance claimed
  for (long long p = threadIdx.x; p < npix; p += kMergeThreads) {
    const int l = lab[p];
    if (l < kVoteClasses) continue;
    atomicOr(&present[l], 1);
    if (!((claimed[p >> 5] >> (p & 31)) & 1u)) atomicAdd(&bins[l], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int l = kVoteClasses; l < K; ++l) {
      if (!present[l] || static_cast<double>(bins[l]) < stuff_area) continue;
      ++seg;
      segid[l] = seg;
      long long* s = sg + static_cast<size_t>(seg - 1) * 4;
      s[0] = -1;
      s[1] = l;
      s[2] = bins[l];
      s[3] = 0;
    }
    nseg[img] = seg;
  }
  __syncthreads();
  for (long long p = threadIdx.x; p < npix; p += kMergeThreads) {
    const int l = lab[p];
    if (l >= kVoteClasses && segid[l] && !((claimed[p >> 5] >> (p & 31)) & 1u)) map[p] = segid[l];
  }
}

}  // namespace pk

using namespace pk;

namespace {
unsigned grid_for(long long max_pix, int threads, int per_thread) {
  const long long per = static_cast<long long>(threads) * per_thread;
  const long long want = (max_pix + per - 1) / per;
  return static_cast<unsigned>(want < 1 ? 1 : want);
}
Bounds to_bounds(const int* b, int T) {
  Bounds r{};
  for (int t = 0; t < T; ++t) r.b[t] = b[t];
  return r;
}
}  // namespace

extern "C" int pk_pano_candidates(const long long* items, const void* base, int n, long long max_pix,
                                  const uint8_t* palette, int P, const int* bounds, int T, int* area, long long* sumfx,
                                  void* stream) {
  PK_CHECK(items && base && palette && bounds && area && sumfx && n >= 1 && n <= 65535 && max_pix > 0,
           "pk_pano_candidates: bad arguments");
  PK_CHECK(P >= 1 && P <= kPanoMaxPalette && T >= 1 && T <= kPanoMaxThr, "pk_pano_candidates: P %d or T %d", P, T);
  const dim3 grid(grid_for(max_pix, kCandThreads, 4), n);
  pano_candidates_kernel<<<grid, kCandThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      items, static_cast<const uint8_t*>(base), palette, P, to_bounds(bounds, T), T, area,
      reinterpret_cast<unsigned long long*>(sumfx));
  PK_LAUNCH_CHECK("pk_pano_candidates");
  return 0;
}

extern "C" long long pk_pano_select_ws_bytes(int n, int NC) {
  if (n < 1 || NC < 1) return 0;
  size_t temp = 0;
  const long long total = static_cast<long long>(n) * NC;
  cub::DeviceSegmentedRadixSort::SortKeys(nullptr, temp, static_cast<const unsigned long long*>(nullptr),
                                          static_cast<unsigned long long*>(nullptr), static_cast<int>(total), n,
                                          static_cast<const int*>(nullptr), static_cast<const int*>(nullptr) + 1);
  const size_t keys = static_cast<size_t>(total) * 8;
  const size_t offs = (static_cast<size_t>(n + 1) * 4 + 255) / 256 * 256;
  return static_cast<long long>(2 * keys + offs + temp);
}

extern "C" int pk_pano_select(const int* area, const long long* sumfx, int n, int NC, int keep, int ncap, void* ws,
                              long long ws_bytes, int* count, int* cand, float* scores, void* stream) {
  PK_CHECK(area && sumfx && ws && count && cand && scores && n >= 1 && NC >= 1 && keep >= 1 && keep <= ncap,
           "pk_pano_select: bad arguments");
  PK_CHECK(ws_bytes >= pk_pano_select_ws_bytes(n, NC), "pk_pano_select: workspace too small");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long total = static_cast<long long>(n) * NC;
  unsigned long long* keys = static_cast<unsigned long long*>(ws);
  unsigned long long* sorted = keys + total;
  int* offs = reinterpret_cast<int*>(sorted + total);
  uint8_t* temp = reinterpret_cast<uint8_t*>(offs) + (static_cast<size_t>(n + 1) * 4 + 255) / 256 * 256;
  size_t temp_bytes = static_cast<size_t>(ws_bytes) - static_cast<size_t>(temp - static_cast<uint8_t*>(ws));
  pano_keys_kernel<<<static_cast<unsigned>((total + 256) / 256), 256, 0, st>>>(
      area, reinterpret_cast<const unsigned long long*>(sumfx), n, NC, keys, offs);
  PK_LAUNCH_CHECK("pano_keys_kernel");
  PK_CHECK(cub::DeviceSegmentedRadixSort::SortKeys(temp, temp_bytes, keys, sorted, static_cast<int>(total), n, offs,
                                                   offs + 1, 0, 64, st) == cudaSuccess,
           "pk_pano_select: segmented sort failed");
  pano_select_kernel<<<n, 256, 0, st>>>(sorted, NC, keep, ncap, count, cand, scores);
  PK_LAUNCH_CHECK("pk_pano_select");
  return 0;
}

extern "C" int pk_pano_pack_candidates(const long long* items, const void* base, int n, const uint8_t* palette, int P,
                                       const int* bounds, int T, const int* cand, const int* count, int ncap,
                                       int words, uint32_t* bits, void* stream) {
  PK_CHECK(items && base && palette && bounds && cand && count && bits && n >= 1 && n <= 65535,
           "pk_pano_pack_candidates: bad arguments");
  PK_CHECK(ncap >= 1 && ncap <= 65535 && words >= 32 && words % 32 == 0 && T >= 1 && T <= kPanoMaxThr,
           "pk_pano_pack_candidates: ncap %d, words %d or T %d", ncap, words, T);
  const dim3 grid((words / 32 + kPackThreads / 32 - 1) / (kPackThreads / 32), ncap, n);
  pano_pack_candidates_kernel<<<grid, kPackThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      items, static_cast<const uint8_t*>(base), palette, P, to_bounds(bounds, T), cand, count, ncap, words, bits);
  PK_LAUNCH_CHECK("pk_pano_pack_candidates");
  return 0;
}

extern "C" int pk_pano_pack_masks(const long long* items, int n, int max_rows, int ncap, int words, uint32_t* bits,
                                  const long long* aux, float* scores, long long* classes, void* stream) {
  PK_CHECK(items && bits && aux && scores && n >= 1 && n <= 65535 && max_rows >= 1 && max_rows <= ncap && ncap <= 65535,
           "pk_pano_pack_masks: bad arguments");
  PK_CHECK(words >= 32 && words % 32 == 0, "pk_pano_pack_masks: words %d", words);
  const dim3 grid((words / 32 + kPackThreads / 32 - 1) / (kPackThreads / 32), max_rows, n);
  pano_pack_masks_kernel<<<grid, kPackThreads, 0, static_cast<cudaStream_t>(stream)>>>(items, ncap, words, bits, aux,
                                                                                      scores, classes);
  PK_LAUNCH_CHECK("pk_pano_pack_masks");
  return 0;
}

extern "C" int pk_pano_gram(const uint32_t* bits, int n, int ncap, int words, const int* count, int* gram,
                            void* stream) {
  PK_CHECK(bits && count && gram && n >= 1 && n <= 65535, "pk_pano_gram: bad arguments");
  PK_CHECK(ncap % kGramTile == 0 && ncap >= kGramTile && words % kGramKW == 0 && words >= kGramKW,
           "pk_pano_gram: ncap %d must be a multiple of %d, words %d of %d", ncap, kGramTile, words, kGramKW);
  static bool attr = false;
  if (!attr) {
    PK_CHECK(cudaFuncSetAttribute(pano_gram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(kGramSmem)) == cudaSuccess,
             "pk_pano_gram: %zu bytes of shared memory not available", kGramSmem);
    attr = true;
  }
  const int tiles = ncap / kGramTile;
  const dim3 grid(static_cast<unsigned>(tiles * (tiles + 1) / 2), n);
  pano_gram_kernel<<<grid, kGramThreads, kGramSmem, static_cast<cudaStream_t>(stream)>>>(bits, ncap, words, count,
                                                                                        gram);
  PK_LAUNCH_CHECK("pk_pano_gram");
  return 0;
}

extern "C" int pk_pano_nms(const int* gram, const long long* labels, const float* scores, const int* count, int n,
                           int ncap, float sigma, int max_num, int empty_one, int* ws, int* rows, float* out_scores,
                           int* out_count, long long* out_labels, void* stream) {
  PK_CHECK(scores && count && ws && rows && out_scores && out_count && n >= 1 && n <= 65535 && max_num >= 1,
           "pk_pano_nms: bad arguments");
  PK_CHECK(ncap >= 1 && ncap <= 8192, "pk_pano_nms: ncap %d outside 1..8192", ncap);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t plane = static_cast<size_t>(n) * ncap;
  int* perm = ws;
  int* perm2 = ws + plane;
  float* comp = reinterpret_cast<float*>(ws + 2 * plane);
  float* decayed = reinterpret_cast<float*>(ws + 3 * plane);
  const dim3 grid((ncap + kNmsThreads - 1) / kNmsThreads, n);
  const size_t rsmem = static_cast<size_t>(ncap) * 4;
  if (gram) {
    pano_rank_kernel<<<grid, kNmsThreads, rsmem, st>>>(scores, count, ncap, perm);
    pano_nms_comp_kernel<<<grid, kNmsThreads, 0, st>>>(gram, labels, count, ncap, perm, comp);
    pano_nms_decay_kernel<<<grid, kNmsThreads, 0, st>>>(gram, labels, count, ncap, perm, comp, scores, -sigma,
                                                        decayed);
    pano_rank_kernel<<<grid, kNmsThreads, rsmem, st>>>(decayed, count, ncap, perm2);
  } else {                                             // no decay: the stable descending order of the scores
    pano_rank_kernel<<<grid, kNmsThreads, rsmem, st>>>(scores, count, ncap, perm2);
  }
  const dim3 ogrid((max_num + kNmsThreads - 1) / kNmsThreads, n);
  pano_nms_out_kernel<<<ogrid, kNmsThreads, 0, st>>>(gram ? decayed : scores, count, ncap, gram ? perm : nullptr,
                                                     perm2, max_num, empty_one, labels, rows, out_scores,
                                                     out_count, out_labels);
  PK_LAUNCH_CHECK("pk_pano_nms");
  return 0;
}

extern "C" int pk_pano_unpack(const uint32_t* bits, int n, int ncap, int words, const int* rows, int rows_ld,
                              int max_rows, long long max_pix, const long long* outs, void* stream) {
  PK_CHECK(bits && rows && outs && n >= 1 && n <= 65535 && max_rows >= 1 && max_rows <= 65535 && max_pix > 0,
           "pk_pano_unpack: bad arguments");
  const dim3 grid(grid_for(max_pix, 256, 16), max_rows, n);
  pano_unpack_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(bits, ncap, words, rows, rows_ld, outs);
  PK_LAUNCH_CHECK("pk_pano_unpack");
  return 0;
}

extern "C" int pk_pano_minmax(const long long* items, const void* base, int n, long long max_pix,
                              const uint8_t* palette, int P, short* pred, int* cnt, long long* sum, int* cols,
                              float* scores, long long* classes, int* count, void* stream) {
  PK_CHECK(items && base && palette && pred && cnt && sum && cols && scores && classes && count && n >= 1 &&
               n <= 65535 && max_pix > 0,
           "pk_pano_minmax: bad arguments");
  PK_CHECK(P >= 1 && P <= kPanoMaxPalette, "pk_pano_minmax: palette size %d outside 1..%d", P, kPanoMaxPalette);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(grid_for(max_pix, kCandThreads, 4), n);
  pano_minmax_kernel<<<grid, kCandThreads, 0, st>>>(items, static_cast<const uint8_t*>(base), palette, P, max_pix,
                                                     pred, cnt, reinterpret_cast<unsigned long long*>(sum));
  pano_minmax_select_kernel<<<n, 1024, 0, st>>>(cnt, reinterpret_cast<const unsigned long long*>(sum), P + 1, cols,
                                                scores, classes, count);
  PK_LAUNCH_CHECK("pk_pano_minmax");
  return 0;
}

extern "C" int pk_pano_minmax_masks(const short* pred, int n, long long max_pix, const int* cols, int P1,
                                    int max_rows, const long long* outs, void* stream) {
  PK_CHECK(pred && cols && outs && n >= 1 && n <= 65535 && max_rows >= 1 && max_rows <= 65535 && max_pix > 0,
           "pk_pano_minmax_masks: bad arguments");
  const dim3 grid(grid_for(max_pix, 256, 16), max_rows, n);
  pano_minmax_masks_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(pred, max_pix, cols, P1, outs);
  PK_LAUNCH_CHECK("pk_pano_minmax_masks");
  return 0;
}

extern "C" int pk_pano_vote(const long long* items, const void* base, int n, long long max_pix,
                            const uint8_t* palette, const uint32_t* bits, int ncap, int words, const int* count,
                            int max_rows, int* dmax_zeroed, long long* classes, void* stream) {
  PK_CHECK(items && base && palette && bits && count && dmax_zeroed && classes && n >= 1 && n <= 65535 &&
               max_pix > 0 && max_rows >= 1 && max_rows <= ncap,
           "pk_pano_vote: bad arguments");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  pano_sem_dmax_kernel<<<dim3(grid_for(max_pix, 256, 16), n), 256, 0, st>>>(
      items, static_cast<const uint8_t*>(base), palette, dmax_zeroed);
  pano_vote_kernel<<<dim3(max_rows, n), kVoteThreads, 0, st>>>(items, static_cast<const uint8_t*>(base), palette,
                                                               dmax_zeroed, bits, ncap, words, count, classes);
  PK_LAUNCH_CHECK("pk_pano_vote");
  return 0;
}

extern "C" long long pk_pano_merge_smem(int words, int ncap) {
  return static_cast<long long>(words) * 4 + static_cast<long long>(ncap) * 4;
}

extern "C" int pk_pano_merge(const long long* sem_items, const void* base, const long long* maps, int n,
                             long long max_pix, const uint8_t* palette, int K, uint8_t* labels, const uint32_t* bits,
                             int ncap, int words, const float* scores, const long long* classes, const int* count,
                             double overlap, double stuff_area, double score_thresh, int max_seg, long long* segs,
                             int* nseg, void* stream) {
  PK_CHECK(sem_items && base && maps && palette && labels && bits && scores && classes && count && segs && nseg &&
               n >= 1 && n <= 65535 && max_pix > 0,
           "pk_pano_merge: bad arguments");
  PK_CHECK(K >= kVoteClasses && K <= kSemMax, "pk_pano_merge: palette size %d outside %d..%d", K, kVoteClasses,
           kSemMax);
  const long long smem = pk_pano_merge_smem(words, ncap);
  PK_CHECK(smem <= 200 * 1024, "pk_pano_merge: image or instance count too large (%lld bytes of shared memory)",
           smem);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  pano_sem_labels_kernel<<<dim3(grid_for(max_pix, 256, 16), n), 256, 0, st>>>(
      sem_items, static_cast<const uint8_t*>(base), palette, K, max_pix, labels);
  PK_CHECK(cudaFuncSetAttribute(pano_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(smem)) == cudaSuccess,
           "pk_pano_merge: %lld bytes of shared memory not available", smem);
  pano_merge_kernel<<<n, kMergeThreads, static_cast<size_t>(smem), st>>>(
      maps, labels, max_pix, K, bits, ncap, words, scores, classes, count, overlap, stuff_area, score_thresh, max_seg,
      segs, nseg);
  PK_LAUNCH_CHECK("pk_pano_merge");
  return 0;
}
