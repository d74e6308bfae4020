// painter_b200 — COCO pose post-processing on the device (painter_b200/pose.py): the heatmap decoding, flip averaging,
// keypoint decoding, rescoring and OKS NMS of Painter/eval/mmpose_custom, computed from run_batch's device outputs.
//
//  pk_pose_decode   model/top_down.py:163-258 (forward_pseudo_test: decode_images_to_heatmaps_minmax, flip_back, the
//                   one-pixel shift, the average) and the head's decode (keypoints_from_heatmaps, post_process
//                   'default', transform_preds) as the offline config runs them
//  pk_pose_nms      data/topdown_coco_dataset.py:266-297 (the rescoring loop and oks_nms per image)
//
// No heatmap is stored.  A pixel p of box i belongs to at most two joints: the class k_h of the painted image at p, and
// swap(k_g) for the class k_g of the flipped image at p' = (y, W - 1 - max(x - 1, 0)) (flip_back, then the shift).  The
// averaged heatmap A_k(p) is therefore known at p for every k from two pixel reads, and the per-(box, joint) argmax is
// an atomicMax over 64-bit keys (value bits << 32 | ~linear index): values are >= 0, so their bits order like the
// values, and the inverted index makes the first maximum win, as np.argmax does.  Zero values never enter: when the
// maximum is 0 the whole heatmap is 0 and np.argmax gives index 0, which is what the finisher returns for a key of 0.
// The last CTA of a box (a per-box counter) re-derives the four neighbours of each winner from the images and applies
// the +-0.25 shift and transform_preds.  Every fp32 / fp64 step is an explicitly rounded intrinsic (no contraction).
#include <climits>

#include "common.cuh"
#include "host_common.h"
#include "../../include/painter_b200.h"

namespace pk {

constexpr int kJ = PK_POSE_JOINTS;                     // 17
constexpr int kPal = PK_POSE_PALETTE;                  // 17 joint colours and the background
constexpr int kPoseRows = 8;                           // image rows per decode CTA
constexpr int kDecodeThreads = 256;
constexpr int kNmsThreads = 256;
constexpr int kRow = PK_POSE_ROW;                      // output row of pk_pose_nms: position, score, 51 keypoint floats

struct PoseConsts {
  int g[kPal], b[kPal];                                // the (G, B) palette
  int swap[kJ];                                        // flip_back's channel swap
};

struct PoseBox {
  const uint8_t* pred;
  const uint8_t* flip;                                 // null without flip test
};
__device__ __forceinline__ PoseBox pose_box(const long long* items, const uint8_t* base, int i) {
  const long long* r = items + static_cast<size_t>(i) * PK_POSE_FIELDS;
  PoseBox b;
  b.pred = r[1] == 1 ? base + r[0] : reinterpret_cast<const uint8_t*>(r[0]);
  b.flip = r[3] == 2 ? nullptr : r[3] == 1 ? base + r[2] : reinterpret_cast<const uint8_t*>(r[2]);
  return b;
}

// argmin_c |G - G_c| + |B - B_c| over the 18 colours, the first on ties (torch.min over the colour dimension); the fp32
// distances of the reference are exact integers
__device__ __forceinline__ int pose_class(const PoseConsts& pc, int G, int B) {
  int best = INT_MAX, cls = 0;
#pragma unroll
  for (int c = 0; c < kPal; ++c) {
    const int d = abs(G - pc.g[c]) + abs(B - pc.b[c]);
    if (d < best) {
      best = d;
      cls = c;
    }
  }
  return cls;
}

// fl32(R / 255.): `heatmaps.cpu().numpy() / 255.` divides the fp32 heatmap by 255 in fp32
__device__ __forceinline__ float pose_value(int R) { return __fdiv_rn(static_cast<float>(R), 255.0f); }

// The heatmap value of joint k at (y, x): the painted image's contribution h, the flipped one's f (g of the swapped
// channel at (y, W - 1 - max(x - 1, 0))), and (h + f) / 2 in fp32 with flip test.
__device__ __forceinline__ float pose_heat(const PoseConsts& pc, const PoseBox& bx, int W, int k, int y, int x) {
  const uint8_t* p = bx.pred + 3 * (static_cast<long long>(y) * W + x);
  const float h = pose_class(pc, p[1], p[2]) == k ? pose_value(p[0]) : 0.0f;
  if (!bx.flip) return h;
  const int xf = W - 1 - max(x - 1, 0);
  const uint8_t* q = bx.flip + 3 * (static_cast<long long>(y) * W + xf);
  const int kg = pose_class(pc, q[1], q[2]);
  const float f = kg < kJ && pc.swap[kg] == k ? pose_value(q[0]) : 0.0f;
  return __fmul_rn(__fadd_rn(h, f), 0.5f);
}

__device__ __forceinline__ void pose_offer(unsigned long long* skey, int k, float v, unsigned idx) {
  if (!(v > 0.0f)) return;
  const unsigned long long key = (static_cast<unsigned long long>(__float_as_uint(v)) << 32) | (~idx & 0xffffffffu);
  if (key > skey[k]) atomicMax(skey + k, key);
}

// grid (ceil(H / kPoseRows), n): each CTA reduces kPoseRows rows of one box into shared keys, merges them into the
// box's global keys, and the box's last CTA finishes its 17 joints.
__global__ void __launch_bounds__(kDecodeThreads) pose_decode_kernel(const long long* items, const uint8_t* base,
                                                                     int H, int W, PoseConsts pc, const float* cs,
                                                                     unsigned long long* keys, unsigned* done,
                                                                     float* out) {
  __shared__ unsigned long long skey[kJ];
  __shared__ bool last;
  const int box = blockIdx.y;
  const PoseBox bx = pose_box(items, base, box);
  if (threadIdx.x < kJ) skey[threadIdx.x] = 0ull;
  __syncthreads();
  const int y0 = blockIdx.x * kPoseRows;
  const int y1 = min(H, y0 + kPoseRows);
  const int npix = (y1 - y0) * W;
  for (int t = threadIdx.x; t < npix; t += kDecodeThreads) {
    const int y = y0 + t / W, x = t % W;
    const unsigned idx = static_cast<unsigned>(y * W + x);
    const uint8_t* p = bx.pred + 3 * static_cast<long long>(idx);
    const int kh = pose_class(pc, p[1], p[2]);
    const float h = kh < kJ ? pose_value(p[0]) : 0.0f;
    if (!bx.flip) {
      if (kh < kJ) pose_offer(skey, kh, h, idx);
      continue;
    }
    const int xf = W - 1 - max(x - 1, 0);
    const uint8_t* q = bx.flip + 3 * (static_cast<long long>(y) * W + xf);
    const int kg = pose_class(pc, q[1], q[2]);
    const int kf = kg < kJ ? pc.swap[kg] : kJ;
    const float f = kg < kJ ? pose_value(q[0]) : 0.0f;
    if (kh == kf) {
      if (kh < kJ) pose_offer(skey, kh, __fmul_rn(__fadd_rn(h, f), 0.5f), idx);
    } else {
      if (kh < kJ) pose_offer(skey, kh, __fmul_rn(h, 0.5f), idx);      // fl32(h + 0) / 2
      if (kf < kJ) pose_offer(skey, kf, __fmul_rn(f, 0.5f), idx);
    }
  }
  __syncthreads();
  if (threadIdx.x < kJ && skey[threadIdx.x]) atomicMax(keys + static_cast<size_t>(box) * kJ + threadIdx.x,
                                                      skey[threadIdx.x]);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(done + box, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last || threadIdx.x >= kJ) return;
  __threadfence();
  const int k = threadIdx.x;
  const unsigned long long key = __ldcg(keys + static_cast<size_t>(box) * kJ + k);
  // _get_max_preds: the first maximum; 0 (no positive value) is index 0 with maxval 0
  const float maxval = key ? __uint_as_float(static_cast<unsigned>(key >> 32)) : 0.0f;
  const int idx = key ? static_cast<int>(~static_cast<unsigned>(key)) : 0;
  const int px = idx % W, py = idx / W;
  float fx = static_cast<float>(px), fy = static_cast<float>(py);
  if (!(maxval > 0.0f)) {
    fx = -1.0f;
    fy = -1.0f;
  } else if (1 < px && px < W - 1 && 1 < py && py < H - 1) {
    // keypoints_from_heatmaps' 'default' post-process: sign(fp32 neighbour difference) * .25
    const float dx = __fsub_rn(pose_heat(pc, bx, W, k, py, px + 1), pose_heat(pc, bx, W, k, py, px - 1));
    const float dy = __fsub_rn(pose_heat(pc, bx, W, k, py + 1, px), pose_heat(pc, bx, W, k, py - 1, px));
    fx = __fadd_rn(fx, dx > 0.0f ? 0.25f : dx < 0.0f ? -0.25f : 0.0f);
    fy = __fadd_rn(fy, dy > 0.0f ? 0.25f : dy < 0.0f ? -0.25f : 0.0f);
  }
  // transform_preds (no UDP), fp32: S = s * 200, x' = (x * S0 / W + c0) - S0 * 0.5
  const float* c = cs + static_cast<size_t>(box) * 4;
  const float S0 = __fmul_rn(c[2], 200.0f), S1 = __fmul_rn(c[3], 200.0f);
  const float sx = __fdiv_rn(S0, static_cast<float>(W)), sy = __fdiv_rn(S1, static_cast<float>(H));
  float* o = out + (static_cast<size_t>(box) * kJ + k) * 3;
  o[0] = __fsub_rn(__fadd_rn(__fmul_rn(fx, sx), c[0]), __fmul_rn(S0, 0.5f));
  o[1] = __fsub_rn(__fadd_rn(__fmul_rn(fy, sy), c[1]), __fmul_rn(S1, 0.5f));
  o[2] = maxval;
}

struct PoseNmsArgs {
  double var[kJ];                                      // (2 sigma)^2, as numpy computes it
  float vis_thr, oks_thr;
};

// oks_iou of boxes a and b (float32 [51] keypoint rows), fp32 area terms: the reference's expression and numpy's
// pairwise summation order for 17 terms
__device__ __forceinline__ float pose_oks(const float* ka, const float* kb, float area_a, float area_b,
                                          const PoseNmsArgs& a) {
  const double den = __dadd_rn(static_cast<double>(__fdiv_rn(__fadd_rn(area_a, area_b), 2.0f)),
                               2.220446049250313e-16);                          // + np.spacing(1)
  double ex[kJ];
#pragma unroll
  for (int j = 0; j < kJ; ++j) {
    const float dx = __fsub_rn(kb[3 * j], ka[3 * j]);
    const float dy = __fsub_rn(kb[3 * j + 1], ka[3 * j + 1]);
    const float d2 = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
    const double e = __ddiv_rn(__ddiv_rn(__ddiv_rn(static_cast<double>(d2), a.var[j]), den), 2.0);
    ex[j] = exp(-e);
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(ex[j], ex[j + 8]);
  double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])),
                       __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  s = __dadd_rn(s, ex[16]);
  return __double2float_rn(__ddiv_rn(s, 17.0));
}

// The order numpy's argsort gives float32 scores, as an unsigned key: -0 and +0 equal, every NaN above +inf
__device__ __forceinline__ unsigned score_key(float v) {
  if (v != v) return 0xffffffffu;
  const unsigned u = v == 0.0f ? 0u : __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// One CTA per image: rescore, rank (score descending, then the later box first), the OKS triangle as suppression bits
// in rank order (row a: bit b set unless oks(a, b) <= oks_thr, b > a), the greedy scan in one warp, and the kept rows.
// images int32 [n_img, 2] (start, count) into pos; shared: bits [count, words] u32, score / order / keep [count].
__global__ void __launch_bounds__(kNmsThreads) pose_nms_kernel(const int* images, const int* pos, const float* kpts,
                                                               const float* box_scores, const float* areas,
                                                               PoseNmsArgs a, int* rows, int* counts) {
  extern __shared__ uint32_t smem[];
  __shared__ int nkeep;
  const int img = blockIdx.x;
  const int start = images[2 * img], cnt = images[2 * img + 1];
  const int words = (cnt + 31) / 32;
  uint32_t* bits = smem;
  float* score = reinterpret_cast<float*>(bits + static_cast<size_t>(cnt) * words);
  int* order = reinterpret_cast<int*>(score + cnt);
  int* keep = order + cnt;
  const int* ipos = pos + start;
  // the rescoring loop: fp32 mean of the joint scores above vis_thr, times the box score (0 * box score without one)
  for (int j = threadIdx.x; j < cnt; j += kNmsThreads) {
    const float* kp = kpts + static_cast<size_t>(ipos[j]) * 3 * kJ;
    float sum = 0.0f;
    int valid = 0;
    for (int t = 0; t < kJ; ++t) {
      const float s = kp[3 * t + 2];
      if (s > a.vis_thr) {
        sum = __fadd_rn(sum, s);
        ++valid;
      }
    }
    const float bs = box_scores[ipos[j]];
    score[j] = valid ? __fmul_rn(__fdiv_rn(sum, static_cast<float>(valid)), bs) : __fmul_rn(0.0f, bs);
  }
  __syncthreads();
  // argsort descending; ties: the larger index (bbox_id) first, as reversing a stable ascending sort orders them.
  // The rank is taken on (score_key, index), a strict total order for any score bits (NaN included), so every slot
  // of order[] is written exactly once.
  for (int j = threadIdx.x; j < cnt; j += kNmsThreads) {
    const unsigned s = score_key(score[j]);
    int r = 0;
    for (int i = 0; i < cnt; ++i) {
      const unsigned t = score_key(score[i]);
      r += (t > s) || (t == s && i > j);
    }
    order[r] = j;
  }
  __syncthreads();
  // the triangle, one warp per rank row, one ballot per 32 columns
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int ra = warp; ra < cnt; ra += kNmsThreads / 32) {
    const int ja = order[ra];
    const float* ka = kpts + static_cast<size_t>(ipos[ja]) * 3 * kJ;
    const float area_a = areas[ipos[ja]];
    uint32_t* row = bits + static_cast<size_t>(ra) * words;
    for (int w = 0; w < words; ++w) {
      const int rb = 32 * w + lane;
      bool sup = false;
      if (rb > ra && rb < cnt) {
        const int jb = order[rb];
        // the reference keeps `oks <= thr` (np.where(oks_ovr <= thr)): a NaN OKS suppresses
        sup = !(pose_oks(ka, kpts + static_cast<size_t>(ipos[jb]) * 3 * kJ, area_a, areas[ipos[jb]], a) <=
                a.oks_thr);
      }
      const uint32_t word = __ballot_sync(0xffffffffu, sup);
      if (lane == 0) row[w] = word;
    }
  }
  __syncthreads();
  // the greedy scan: lane w holds the removed bits of columns 32 w .. 32 w + 31 (cnt <= 1024)
  if (warp == 0) {
    uint32_t removed = 0;
    int k = 0;
    for (int r = 0; r < cnt; ++r) {
      const uint32_t wr = __shfl_sync(0xffffffffu, removed, r >> 5);
      if ((wr >> (r & 31)) & 1u) continue;
      if (lane == 0) keep[k] = r;
      ++k;
      if (lane < words) removed |= bits[static_cast<size_t>(r) * words + lane];
    }
    if (lane == 0) nkeep = k;
  }
  __syncthreads();
  const int nk = nkeep;
  if (threadIdx.x == 0) counts[img] = nk;
  for (int t = threadIdx.x; t < nk * kRow; t += kNmsThreads) {
    const int k = t / kRow, f = t % kRow;
    const int j = order[keep[k]];
    const int p = ipos[j];
    int v;
    if (f == 0) v = p;
    else if (f == 1) v = __float_as_int(score[j]);
    else v = __float_as_int(kpts[static_cast<size_t>(p) * 3 * kJ + f - 2]);
    rows[static_cast<size_t>(start + k) * kRow + f] = v;
  }
}

}  // namespace pk

using namespace pk;

extern "C" int pk_pose_decode(const long long* items, const void* base, int n, int H, int W, const uint8_t* palette,
                              const int* swap, const float* cs, unsigned long long* keys_zeroed,
                              unsigned* done_zeroed, float* out, void* stream) {
  PK_CHECK(items && base && palette && swap && cs && keys_zeroed && done_zeroed && out && n >= 1 && n <= 65535,
           "pk_pose_decode: bad arguments");
  PK_CHECK(H >= 3 && W >= 3 && static_cast<long long>(H) * W < INT_MAX, "pk_pose_decode: image size %d x %d", H, W);
  PoseConsts pc;
  for (int c = 0; c < kPal; ++c) {
    pc.g[c] = palette[2 * c];
    pc.b[c] = palette[2 * c + 1];
  }
  for (int k = 0; k < kJ; ++k) {
    PK_CHECK(swap[k] >= 0 && swap[k] < kJ, "pk_pose_decode: swap[%d] = %d", k, swap[k]);
    pc.swap[k] = swap[k];
  }
  const dim3 grid((H + kPoseRows - 1) / kPoseRows, n);
  pose_decode_kernel<<<grid, kDecodeThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      items, static_cast<const uint8_t*>(base), H, W, pc, cs, keys_zeroed, done_zeroed, out);
  PK_LAUNCH_CHECK("pk_pose_decode");
  return 0;
}

extern "C" long long pk_pose_nms_smem(int max_count) {
  const long long words = (max_count + 31) / 32;
  return static_cast<long long>(max_count) * words * 4 + static_cast<long long>(max_count) * 12;
}

extern "C" int pk_pose_nms(const int* images, int n_img, int max_count, const int* pos, const float* kpts,
                           const float* box_scores, const float* areas, const double* vars, float vis_thr,
                           float oks_thr, int* rows, int* counts, void* stream) {
  PK_CHECK(images && pos && kpts && box_scores && areas && vars && rows && counts && n_img >= 1,
           "pk_pose_nms: bad arguments");
  PK_CHECK(max_count >= 1 && max_count <= PK_POSE_MAX_BOXES, "pk_pose_nms: %d boxes in one image (1..%d)", max_count,
           PK_POSE_MAX_BOXES);
  PoseNmsArgs a;
  for (int j = 0; j < kJ; ++j) a.var[j] = vars[j];
  a.vis_thr = vis_thr;
  a.oks_thr = oks_thr;
  const long long smem = pk_pose_nms_smem(max_count);
  PK_CHECK(cudaFuncSetAttribute(pose_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                static_cast<int>(smem)) == cudaSuccess,
           "pk_pose_nms: %lld bytes of shared memory not available", smem);
  pose_nms_kernel<<<n_img, kNmsThreads, static_cast<size_t>(smem), static_cast<cudaStream_t>(stream)>>>(
      images, pos, kpts, box_scores, areas, a, rows, counts);
  PK_LAUNCH_CHECK("pk_pose_nms");
  return 0;
}
