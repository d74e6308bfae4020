// painter_b200 — pieces of the wgmma GEMM (gemm.cu) shared with its host-side planner: argument structs, the
// work scheduler, the fused epilogues and the decoder-head epilogue.
#pragma once
#include <string.h>

#include "common.cuh"
#include "host_common.h"
#include "../../include/painter_b200.h"

namespace pk {

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_A_BYTES = GEMM_BM * GEMM_BK * 2;  // 16 KiB
constexpr int GEMM_THREADS = 384;   // TMA producer warpgroup + two math warpgroups (64 accumulator rows each)
constexpr int STG_LD = 68;          // floats per row of a math warpgroup's 64 x 64 epilogue staging tile
constexpr int GEMM_STG_BYTES = 2 * 64 * STG_LD * 4;

// internal epilogue kinds (beyond the public PK_EPI_*)
constexpr int EPI_HEAD = 100;    // decoder head fused behind the 3x3 conv (LN2D + GELU + 1x1 conv + loss)
constexpr int EPI_UNSHUF = 101;  // inverse pixel shuffle: pixel rows -> token rows [B*h*w, p*p*c]

// Implicit-GEMM modes for the decoder's 3x3 convolution (models_painter.py:328-333):
//   mode 1: A rows are pixels of an NHWC bf16 image fetched by a 4D TMA box {c, TW, TH, 1}; k-block = tap
//           (OOB box coordinates give the zero padding).                  used by conv fwd and dgrad
//   mode 2: wgrad.  out[(tap, c), o] = sum_pix G[pix + tap, c] * dC1[pix, o]; A (MN-major) = G shifted by
//           the two taps of the m-block, B (MN-major) = dC1; k-blocks run over 64-pixel groups.
struct ConvArgs {
  int mode;
  int H, W, TW, TH, tiles_x, tiles_y;
};
struct HeadArgs {
  const float* tgts;        // [B,3,H,W]
  const uint8_t* mask;      // [maskB, N]
  const float* valid;       // [B,3,H,W]
  __nv_bfloat16* c1_out;    // [B,H,W,64]
  float* patch_out;         // [B, N, p*p*3]
  float* num;               // [B] atomics: sum smoothl1 * mask * valid
  int maskB, p, loss_kind;
  int slot;                 // which copy of the head parameters in constant memory this launch reads
};

// Epilogues whose results leave through TMA stores (gemm.cu): every math warpgroup applies the epilogue to its
// accumulator fragments and writes 64-column bf16 sub-tiles (64 rows x 128 B, 128B-swizzled: one TMA box) into one of
// two staging slots; a slot holds one sub-tile per output (GELU: z and gelu(z)).
__host__ __device__ constexpr bool gemm_tma_epilogue(int kind) { return kind == PK_EPI_BF16 || kind == PK_EPI_GELU; }
constexpr int GEMM_SUB_BYTES = 64 * 128;   // one 64 x 64 bf16 sub-tile
__host__ __device__ constexpr int gemm_slot_bytes(int kind) { return (kind == PK_EPI_GELU ? 2 : 1) * GEMM_SUB_BYTES; }
// staging bytes of a kind: 2 math warpgroups x 2 slots, or the fp32 staging tiles of the other epilogues
__host__ __device__ constexpr int gemm_stg_bytes(int kind) {
  return gemm_tma_epilogue(kind) ? 2 * 2 * gemm_slot_bytes(kind) : GEMM_STG_BYTES;
}

// operand ring depth that fits beside the epilogue staging of `kind`
__host__ inline int gemm_stages_for(int stage_bytes, int kind) {
  const int budget = 227 * 1024 - 1024 - 256 - gemm_stg_bytes(kind);
  int st = budget / stage_bytes;
  return st > 8 ? 8 : st;
}

struct GemmArgs {
  int M, N, K;
  int BN;
  int stages;
  int transA, transB;
  int num_m_tiles, num_n_tiles;
  int splits, kb_per_split;  // split-K (epilogue accumulates with fp32 atomics when splits > 1)
  int streamk_units;         // > 0: stream-K: every CTA owns this many consecutive (tile, k-block) units;
                             // partial tiles are added with fp32 atomics
  int group_m;               // tile rasterisation: groups of group_m row blocks, the column blocks of a group
                             // consecutive (0 = row blocks fastest)
  PkEpilogue epi;
  ConvArgs conv;
  HeadArgs head;
};

// Work iterator shared by the producer and math roles of the persistent kernel: each role walks the same sequence
// of (output tile, k-block range) items.  Classic mode: item = (tile, split) strided over the CTAs; stream-K mode:
// the tiles_mn * num_kb k-block units are cut into consecutive ranges of equal length, one per CTA, so the machine
// is full whatever the tile count (weight-gradient GEMMs have 32..256 tiles for 132 SMs).
struct GemmSched {
  int tiles_mn, num_kb, kbps, total, ncl, cur, end;
  bool sk;
  __host__ __device__ __forceinline__ void init(const GemmArgs& g, int tiles_mn_, int num_kb_, int cid, int ncl_) {
    tiles_mn = tiles_mn_;
    num_kb = num_kb_;
    kbps = g.kb_per_split;
    ncl = ncl_;
    sk = g.streamk_units > 0;
    if (sk) {
      total = tiles_mn * num_kb;
      cur = cid * g.streamk_units;
      end = total < cur + g.streamk_units ? total : cur + g.streamk_units;
    } else {
      total = tiles_mn * g.splits;
      cur = cid;
      end = total;
    }
  }
  __host__ __device__ __forceinline__ bool next(int& mn, int& kb0, int& kb1) {
    if (cur >= end) return false;
    if (sk) {
      mn = cur / num_kb;
      kb0 = cur - mn * num_kb;
      const int len = (num_kb - kb0) < (end - cur) ? (num_kb - kb0) : (end - cur);
      kb1 = kb0 + len;
      cur += len;
    } else {
      mn = cur % tiles_mn;
      const int split = cur / tiles_mn;
      kb0 = split * kbps;
      kb1 = num_kb < kb0 + kbps ? num_kb : kb0 + kbps;
      cur += ncl;
    }
    return true;
  }
};

// Linear tile index -> (row block, column block).  Concurrent CTAs should share operand blocks so that each is
// fetched from HBM once and from L2 otherwise: with group_m = 1 the column blocks of one row block are adjacent
// (A read once; right whenever B - weights, <= 40 MB - stays resident in the 50 MB L2); larger groups bound the B
// re-reads when B does not fit (decoder_embed: 134 MB of weights).
__host__ __device__ __forceinline__ void gemm_tile_coords(const GemmArgs& g, int mn, int& m_blk, int& n_blk) {
  if (g.group_m <= 0) {
    m_blk = mn % g.num_m_tiles;
    n_blk = mn / g.num_m_tiles;
    return;
  }
  const int per_group = g.group_m * g.num_n_tiles;
  const int grp = mn / per_group, r = mn - grp * per_group;
  const int rem = g.num_m_tiles - grp * g.group_m;
  const int gm = g.group_m < rem ? g.group_m : rem;
  m_blk = grp * g.group_m + r % gm;
  n_blk = r / gm;
}

// decoder-head parameters, refreshed per call by async D2D copies:
// [0,64) conv bias | [64,128) LN2D gamma | [128,192) LN2D beta | [192,384) 1x1 weight [3][64] | [384,387) 1x1 bias
// HEAD_SLOTS copies, handed out round-robin per call (HeadArgs::slot): launches on different streams - or queued
// back to back with different parameters - never share a copy unless more than HEAD_SLOTS head launches are in flight
constexpr int HEAD_SLOTS = 8;
static __constant__ float c_head_all[HEAD_SLOTS][392];   // only gemm.cu (EPI_HEAD) writes and reads it

__device__ __forceinline__ float smooth_l1(float d, int kind) {
  const float ad = fabsf(d);
  // smoothl1 beta=0.01 (0.5 d^2 leaves the normal range only for |d| < 2e-19, where the term is immaterial)
  if (kind == 0) return ad < 0.01f ? div_rn_nocall(0.5f * d * d, 0.01f) : ad - 0.005f;
  if (kind == 1) return ad;                                             // l1
  if (kind == 2) return d * d;                                          // l2
  return (ad + d * d) * 0.5f;                                           // l1l2
}

// One pixel (= one accumulator row, 64 conv outputs) of the fused decoder head, models_painter.py:328-333 +
// vitdet_utils.py:204-209 + forward_loss :433-462 + patchify :355-368.
__device__ __forceinline__ void head_epilogue_row(const GemmArgs& g, int b, int y, int x, float (&c)[64]) {
  const HeadArgs& hd = g.head;
  const float* c_head = c_head_all[hd.slot];
  const int H = g.conv.H, W = g.conv.W, p = hd.p;
  // conv bias, round to bf16 (the conv output is what backward re-reads), store NHWC
  float mean = 0.f;
#pragma unroll
  for (int k = 0; k < 64; ++k) {
    c[k] = bf16_round(c[k] + c_head[k]);
    mean += c[k];
  }
  {
    uint4* d = reinterpret_cast<uint4*>(hd.c1_out + ((static_cast<size_t>(b) * H + y) * W + x) * 64);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      uint4 u;
      u.x = pack_bf16x2(c[q * 8 + 0], c[q * 8 + 1]);
      u.y = pack_bf16x2(c[q * 8 + 2], c[q * 8 + 3]);
      u.z = pack_bf16x2(c[q * 8 + 4], c[q * 8 + 5]);
      u.w = pack_bf16x2(c[q * 8 + 6], c[q * 8 + 7]);
      d[q] = u;
    }
  }
  mean *= (1.0f / 64);
  float var = 0.f;
#pragma unroll
  for (int k = 0; k < 64; ++k) {
    const float dlt = c[k] - mean;
    var += dlt * dlt;
  }
  const float rstd = rsqrtf(var * (1.0f / 64) + 1e-6f);
  float p0 = c_head[384], p1 = c_head[385], p2 = c_head[386];
#pragma unroll
  for (int k = 0; k < 64; ++k) {
    const float ln = c_head[64 + k] * ((c[k] - mean) * rstd) + c_head[128 + k];
    const float ge = gelu_erf(ln);
    p0 = fmaf(c_head[192 + k], ge, p0);
    p1 = fmaf(c_head[256 + k], ge, p1);
    p2 = fmaf(c_head[320 + k], ge, p2);
  }
  const int wt = W / p;
  const int tok = (y / p) * wt + x / p;
  const int Ntok = (H / p) * wt;
  const float m = hd.mask[static_cast<size_t>(b % hd.maskB) * Ntok + tok] ? 1.f : 0.f;
  const size_t plane = static_cast<size_t>(H) * W;
  const size_t pix = static_cast<size_t>(b) * 3 * plane + static_cast<size_t>(y) * W + x;
  const float pr[3] = {p0, p1, p2};
  float num = 0.f;
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float d = pr[ch] - hd.tgts[pix + ch * plane];
    num += smooth_l1(d, hd.loss_kind) * (m * hd.valid[pix + ch * plane]);
  }
  float* po = hd.patch_out + (static_cast<size_t>(b) * Ntok + tok) * (p * p * 3) + ((y % p) * p + x % p) * 3;
  po[0] = p0;
  po[1] = p1;
  po[2] = p2;
  num = warp_sum(num);
  if ((threadIdx.x & 31) == 0) atomicAdd(hd.num + b, num);
}

__device__ __forceinline__ void store_bf16x32(__nv_bfloat16* dst, const float (&x)[32]) {
  uint4* d = reinterpret_cast<uint4*>(dst);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint4 u;
    u.x = pack_bf16x2(x[q * 8 + 0], x[q * 8 + 1]);
    u.y = pack_bf16x2(x[q * 8 + 2], x[q * 8 + 3]);
    u.z = pack_bf16x2(x[q * 8 + 4], x[q * 8 + 5]);
    u.w = pack_bf16x2(x[q * 8 + 6], x[q * 8 + 7]);
    d[q] = u;
  }
}

// Generic epilogue for one 32-row x 32-column accumulator chunk of one warp.  `stg` is the warp's 32 x 32 block of
// its warpgroup's staging tile (row stride STG_LD floats: 16-byte aligned, conflict-free for float4 quarter-warps).
// Phase 1 (thread = accumulator row): alpha, bias, per-sample row scale -> back into the staging block.
// Phase 2 (lane = 4 consecutive columns, 8 lanes per row, 4 rows per instruction): every global access of the
// warp covers whole contiguous row segments (128 B fp32 / 64 B bf16) instead of 32 scattered rows.

__device__ __forceinline__ uint2 pack4_bf16(const float4& v) {
  uint2 u;
  u.x = pack_bf16x2(v.x, v.y);
  u.y = pack_bf16x2(v.z, v.w);
  return u;
}
__device__ __forceinline__ float4 unpack4_bf16(const uint2& u) {
  return make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xFFFF0000u), __uint_as_float(u.y << 16),
                     __uint_as_float(u.y & 0xFFFF0000u));
}

// Global reads a chunk's epilogue needs (residual / saved pre-activation / accumulate-into output), in the
// coalesced phase-2 layout.
struct EpiAux {
  float4 f[8];
  uint2 h[8];
};

template <int KIND>
__device__ __forceinline__ void gemm_epilogue_prefetch(const PkEpilogue& e, int row0, int M, int col, EpiAux& a) {
  const int lane = threadIdx.x & 31;
  const int rsub = lane >> 3, cc = col + (lane & 7) * 4;
  if constexpr (KIND == PK_EPI_RESID) {
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = row0 + it * 4 + rsub;
      a.f[it] = row < M ? *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(e.aux) +
                                                           static_cast<size_t>(row) * e.ld_aux + cc)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  } else if constexpr (KIND == PK_EPI_DGELU) {
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = row0 + it * 4 + rsub;
      a.h[it] = row < M ? *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(e.aux) +
                                                          static_cast<size_t>(row) * e.ld_aux + cc)
                        : make_uint2(0u, 0u);
    }
  } else if constexpr (KIND == PK_EPI_F32) {
    if (e.accumulate == 1) {
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int row = row0 + it * 4 + rsub;
        a.f[it] = row < M ? *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(e.out) +
                                                             static_cast<size_t>(row) * e.ldc + cc)
                          : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  }
}

template <int KIND>
__device__ __forceinline__ void gemm_epilogue_chunk(const PkEpilogue& e, float* stg, int row0, int M, int col,
                                                    const uint32_t (&v)[32], const EpiAux& aux) {
  const int lane = threadIdx.x & 31;
  const int rsub = lane >> 3, c4 = (lane & 7) * 4;
  const int cc = col + c4;
  const float4 (&auxf)[8] = aux.f;
  const uint2 (&auxh)[8] = aux.h;
  {
    // ---- phase 1 (thread = accumulator row) ----
    const int row = row0 + lane;
    float sc = e.alpha;
    if (KIND == PK_EPI_RESID && e.rowscale != nullptr && row < M) sc *= __ldg(e.rowscale + row / e.rows_per_group);
    float4* srow = reinterpret_cast<float4*>(stg + lane * STG_LD);
    if (e.bias != nullptr) {
      const float4* b4 = reinterpret_cast<const float4*>(e.bias + col);
      const float bsc = KIND == PK_EPI_RESID ? div_rn_nocall(sc, e.alpha) : 1.0f;  // rowscale also multiplies the bias
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 b = __ldg(b4 + q);
        srow[q] = make_float4(fmaf(__uint_as_float(v[q * 4 + 0]), sc, b.x * bsc),
                              fmaf(__uint_as_float(v[q * 4 + 1]), sc, b.y * bsc),
                              fmaf(__uint_as_float(v[q * 4 + 2]), sc, b.z * bsc),
                              fmaf(__uint_as_float(v[q * 4 + 3]), sc, b.w * bsc));
      }
    } else {
#pragma unroll
      for (int q = 0; q < 8; ++q)
        srow[q] = make_float4(__uint_as_float(v[q * 4 + 0]) * sc, __uint_as_float(v[q * 4 + 1]) * sc,
                              __uint_as_float(v[q * 4 + 2]) * sc, __uint_as_float(v[q * 4 + 3]) * sc);
    }
  }
  __syncwarp();
  // ---- phase 2 (lane = 4 consecutive columns; 8 lanes per row, 4 rows per instruction) ----
  // staged values first, then all the math (32 independent elements per lane -> ILP), then all the stores
  float4 xs[8];
#pragma unroll
  for (int it = 0; it < 8; ++it) xs[it] = *reinterpret_cast<const float4*>(stg + (it * 4 + rsub) * STG_LD + c4);
  __syncwarp();  // the staging tile may be overwritten by the next chunk from here on

  if constexpr (KIND == PK_EPI_BF16 || KIND == PK_EPI_PIXSHUF) {
    uint2 o[8];
#pragma unroll
    for (int it = 0; it < 8; ++it) o[it] = pack4_bf16(xs[it]);
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = row0 + it * 4 + rsub;
      if (row >= M) continue;
      size_t off;
      if constexpr (KIND == PK_EPI_BF16) {
        off = static_cast<size_t>(row) * e.ldc + cc;
      } else {
        const int hw = e.ps_h * e.ps_w;
        const int b = row / hw, t = row - b * hw;
        const int i = t / e.ps_w, j = t - i * e.ps_w;
        const int pc = e.ps_p * e.ps_c;
        const int rr = cc / pc, rem = cc - rr * pc;
        const int ss = rem / e.ps_c, c = rem - ss * e.ps_c;
        off = ((static_cast<size_t>(b) * (e.ps_h * e.ps_p) + i * e.ps_p + rr) * (static_cast<size_t>(e.ps_w) * e.ps_p) +
               j * e.ps_p + ss) * e.ps_c + c;
      }
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(e.out) + off) = o[it];
    }
  } else if constexpr (KIND == PK_EPI_F32 || KIND == PK_EPI_RESID) {
    if (KIND == PK_EPI_RESID || e.accumulate == 1) {
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        xs[it].x += auxf[it].x; xs[it].y += auxf[it].y; xs[it].z += auxf[it].z; xs[it].w += auxf[it].w;
      }
    }
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = row0 + it * 4 + rsub;
      if (row >= M) continue;
      float* d = reinterpret_cast<float*>(e.out) + static_cast<size_t>(row) * e.ldc + cc;
      if (KIND == PK_EPI_F32 && e.accumulate == 2) {  // split-K / stream-K partials
        // one 16-byte vector reduction per thread instead of four scalar ones: the partial tiles of a weight-gradient
        // GEMM are 32 K fp32 per CTA, and at ~1.3 cycles per scalar lane the atomics were ~40 % of those kernels
        asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(d), "f"(xs[it].x),
                     "f"(xs[it].y), "f"(xs[it].z), "f"(xs[it].w)
                     : "memory");
      } else {
        *reinterpret_cast<float4*>(d) = xs[it];
      }
    }
  } else if constexpr (KIND == PK_EPI_GELU) {
    uint2 zb[8], hb[8];
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      zb[it] = pack4_bf16(xs[it]);
      const float4 zr = unpack4_bf16(zb[it]);
      float4 g;
      gelu_fast_pair(zr.x, zr.y, g.x, g.y);
      gelu_fast_pair(zr.z, zr.w, g.z, g.w);
      hb[it] = pack4_bf16(g);
    }
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = row0 + it * 4 + rsub;
      if (row >= M) continue;
      const size_t off = static_cast<size_t>(row) * e.ldc + cc;
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(e.out) + off) = zb[it];
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(e.out2) + off) = hb[it];
    }
  } else if constexpr (KIND == PK_EPI_DGELU) {
    uint2 o[8];
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const float4 z = unpack4_bf16(auxh[it]);
      float4 d;
      gelu_fast_grad_mul_pair(z.x, z.y, xs[it].x, xs[it].y, d.x, d.y);
      gelu_fast_grad_mul_pair(z.z, z.w, xs[it].z, xs[it].w, d.z, d.w);
      o[it] = pack4_bf16(d);
    }
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int row = row0 + it * 4 + rsub;
      if (row >= M) continue;
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(e.out) + static_cast<size_t>(row) * e.ldc + cc) = o[it];
    }
  }
}

}  // namespace pk
