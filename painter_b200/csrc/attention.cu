// painter_b200 — fused attention with decomposed relative-position bias, forward and backward (sm_90a), and the
// fp32-accurate forward of windowed blocks (attn_fwd_split3_kernel, below the bf16 forward).
//
// Replaces models_painter.py:73-86 + util/vitdet_utils.py:63-125 (q*scale @ k^T, add_decomposed_rel_pos, softmax,
// @ v) and autograd's backward through them, without ever materialising the [B*heads, N, N] score tensor.
//
// Every kernel is one warpgroup (4 warps, warp w owns rows [16 w, 16 w + 16)) working on 64-row tiles with
// wgmma.mma_async m64n64k16 (bf16 in, fp32 accumulation in registers).  Operand tiles live in shared memory in the
// 128B-swizzled layout the wgmma descriptors read, filled by cp.async and double-buffered, so the loads of the next
// tile overlap the math of this one.  A tile stored [rows][64] serves both as a K-major operand and, through the
// descriptor's transpose bit, as an MN-major one: no transposed copies are made.  The probabilities P (and dS) stay in
// registers between the two products: their accumulator fragment is the register A operand of the next wgmma.
//   forward   one CTA per 64 queries of one (batch, head): S = Q K^T over 64-key tiles, online softmax in the log2
//             domain, O += P V; writes O and the log-sum-exp.
//   backward  dQ kernel (per 64 queries; also the bias-row gradients and the per-CTA table-gradient partials) and
//             dK/dV kernel (per 64 keys, loops over the query tiles); both recompute P from the log-sum-exp.
// The bias rows rel_h[q, i] = q . T_h[i_q - i + h - 1] and rel_w[q, j] = q . T_w[j_q - j + w - 1] are one product
// R = Q [T_h; T_w]^T per query tile (the tables staged as [rows][64] tiles), scattered from the accumulator into
// log2e-scaled rows in shared memory; the training forward stores them for the backward kernels
// ([B*heads, Np, h] / [B*heads, Np, w]).  The dQ kernel gets the bias-row gradients of each key tile as one more
// product, dS . E with E the tile's one-hot [key][image column | image row] matrix, and its tail runs both table
// terms as products over the Toeplitz matrix G[q, table row] of those gradients: dQ += G [T_h; T_w] and the
// table-gradient partials G^T Q.
#include <type_traits>

#include "common.cuh"
#include "wgmma.cuh"
#include "split3.cuh"
#include "host_common.h"
#include "../../include/painter_b200.h"

namespace pk {

constexpr int AT_BM = 64;                     // rows (queries or keys) per CTA and per loop tile
constexpr int AT_THREADS = 128;               // one warpgroup
constexpr int AT_TILE = AT_BM * 128;          // bytes of one 64 x 64 bf16 operand tile
constexpr float AT_LOG2E = 1.4426950408889634f;

struct AttnArgs {
  const __nv_bfloat16* qkv;   // [B*N, 3C]
  const __nv_bfloat16* th;    // [th_pad, 64]
  const __nv_bfloat16* tw;    // [tw_pad, 64]
  const __nv_bfloat16* O;     // [B*N, C]   (backward)
  const __nv_bfloat16* dO;    // [B*N, C]   (backward)
  __nv_bfloat16* out;         // forward: O [B*N, C]; backward: dqkv [B*N, 3C]
  float* lse;                 // [B*heads, N] (log2 domain: m + log2(l))
  const float* delta;         // [B*heads, N] rowsum(dO * O)
  float* relh;                // [B*heads, Np, h] log2e-scaled rel_h rows (nullable in the forward)
  float* relw;                // [B*heads, Np, w]
  float* dt_ws;               // [dQ CTAs][64][2h-1 + 2w-1] table-gradient partials
  int h, w, N, Np, heads;
  float scale_log2;           // head_dim^-0.5 * log2(e)
};

__device__ __forceinline__ float bf16lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16hi(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }

// Byte offset of 16-byte chunk `ch` of row `row` in a [rows][64] bf16 tile with 128-byte swizzle (8-row atoms of
// 1024 bytes; the tile is 1024-byte aligned), the layout SWIZZLE_128B descriptors expect.
__device__ __forceinline__ uint32_t sw128(int row, int ch) { return row * 128 + ((ch ^ (row & 7)) << 4); }

// cp.async with zero fill: the destination gets `bytes` bytes from src and zeros for the rest of the copy size
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, uint32_t bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t dst, const void* src, uint32_t bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(dst), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Start copying rows [r0, r0 + 64) x columns [c0, c0 + 64) of a bf16 matrix (row stride ld elements, rows >= nrows
// read as zero) into the swizzled tile at shared address s.
__device__ __forceinline__ void load_tile(uint32_t s, const __nv_bfloat16* g, size_t ld, int r0, int nrows, int c0) {
#pragma unroll
  for (int it = 0; it < (AT_BM * 8) / AT_THREADS; ++it) {
    const int idx = it * AT_THREADS + threadIdx.x;
    const int row = idx >> 3, ch = idx & 7, r = r0 + row;
    const __nv_bfloat16* src = g + static_cast<size_t>(min(r, nrows - 1)) * ld + c0 + ch * 8;
    cp_async16(s + sw128(row, ch), src, r < nrows ? 16u : 0u);
  }
}
// The cp.async data of the waited groups becomes visible to every thread's wgmma (async proxy).
template <int PENDING>
__device__ __forceinline__ void tiles_ready() {
  cp_async_wait<PENDING>();
  fence_proxy_async_smem();
  __syncthreads();
}

// d[64 x 64] = A . B^T: A a [64][64] tile (rows = output rows), B a [64][64] tile (rows = output columns), both
// K-major.  Issues the wgmmas only; the caller fences, commits and waits.  acc = 1 adds to d.
__device__ __forceinline__ void mma_ss(float (&d)[32], uint32_t sa, uint32_t sb, uint32_t acc = 0u) {
  const uint64_t da = make_wgmma_desc(sa, 16, 1024), db = make_wgmma_desc(sb, 16, 1024);
#pragma unroll
  for (int k = 0; k < 4; ++k)
    wgmma_m64n64k16<0, 0>(d, wgmma_desc_add(da, k * 32), wgmma_desc_add(db, k * 32), k > 0 ? 1u : acc);
}
// d[64 x 64] (+)= P . B: P as packed register fragments (pack_frag), B a [64][64] tile (rows = the reduction index)
// read MN-major.  acc = 0 overwrites d.
__device__ __forceinline__ void mma_rs(float (&d)[32], const uint32_t (&p)[4][4], uint32_t sb, uint32_t acc = 1u) {
  const uint64_t db = make_wgmma_desc(sb, AT_TILE, 1024);
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_m64n64k16_rs<1>(d, p[k], wgmma_desc_add(db, k * 2048), k > 0 ? 1u : acc);
}
// accumulator fragment -> bf16 A fragments of the next product (wgmma_m64n64k16_rs)
__device__ __forceinline__ void pack_frag(const float (&s)[32], uint32_t (&p)[4][4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      p[k][j] = pack_bf16x2(s[8 * k + 2 * j], s[8 * k + 2 * j + 1]);
      asm volatile("" : "+r"(p[k][j])::"memory");   // written before the wgmma.fence
    }
  }
}
__device__ __forceinline__ void zero32(float (&d)[32]) {
#pragma unroll
  for (int i = 0; i < 32; ++i) d[i] = 0.f;
}

// Staged tables: one swizzled [rows][64] block, T_h in rows [0, tab_h_rows(h)), T_w in the next tab_h_rows(w) rows,
// each zero past its 2h - 1 (2w - 1) real rows, the whole rounded up to 64 rows.  Read K-major in 64-row chunks by the
// bias-row product (table rows = output columns) and MN-major by the dQ tail (table rows = the reduction index).
__host__ __device__ inline int tab_h_rows(int h) { return (2 * h - 1 + 15) / 16 * 16; }
__host__ __device__ inline int tab_rows(int h, int w) { return tab_h_rows(h) + tab_h_rows(w); }
__host__ __device__ inline size_t table_bytes(int h, int w) { return static_cast<size_t>(tab_rows(h, w) + 63) / 64 * AT_TILE; }

// Start copying both tables into the staged block at shared address s.
__device__ __forceinline__ void load_tables(const AttnArgs& a, uint32_t s) {
  const int Lh = 2 * a.h - 1, Lw = 2 * a.w - 1, hp = tab_h_rows(a.h);
  const int rows = static_cast<int>(table_bytes(a.h, a.w) / 128);
  for (int idx = threadIdx.x; idx < rows * 8; idx += AT_THREADS) {
    const int row = idx >> 3, ch = idx & 7;
    const bool hs = row < hp;
    const int tr = hs ? row : row - hp;
    const bool valid = tr < (hs ? Lh : Lw);
    const __nv_bfloat16* src = (hs ? a.th : a.tw) + static_cast<size_t>(valid ? tr : 0) * 64 + ch * 8;
    cp_async16(s + sw128(row, ch), src, valid ? 16u : 0u);
  }
}

// Bias rows of the 64 queries [q0, q0 + 64) of one (batch, head) into relh_s [64][h] / relw_s [64][w] from the query
// tile sQ and the staged tables sT (both visible to wgmma).  R = Q . [T_h; T_w]^T in 64-column chunks; R[q, r] is
// rel_h[q, i_q + h - 1 - r] for the T_h rows and rel_w[q, j_q + w - 1 - r'] for the T_w rows, so each (q, i) and
// (q, j) comes from exactly one accumulator entry.  Queries past N take the image position of query N - 1 (their Q
// rows are zero, so their rows are zero).
//   SPLIT = false: bf16 operands, one product, rows scaled by log2e (the log2-domain softmax of the bf16 kernels).
//   SPLIT = true:  three-term split operands (split3.cuh): sQ's terms AT_TILE bytes apart, sT's `tterm` bytes apart;
//                  the six products in c_termA / c_termB order, rows unscaled.
template <bool SPLIT>
__device__ __forceinline__ void bias_rows_product(int h, int w, int N, uint32_t sQ, uint32_t sT, uint32_t tterm,
                                                  int q0, float* relh_s, float* relw_s) {
  const int hp = tab_h_rows(h), rows = tab_rows(h, w);
  const int lane = threadIdx.x & 31, c2 = 2 * (lane & 3);
  const int rl0 = (threadIdx.x >> 5) * 16 + (lane >> 2);
  int iq[2], jq[2];
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int t = min(q0 + rl0 + 8 * e, N - 1);
    iq[e] = t / w;
    jq[e] = t - iq[e] * w;
  }
  float r[32];
  zero32(r);
  for (int n0 = 0; n0 < rows; n0 += AT_BM) {
    wgmma_fence_operands(r);
    wgmma_fence();
    if constexpr (SPLIT) {
#pragma unroll
      for (int k = 0; k < 6; ++k)
        mma_ss(r, sQ + c_termA[k] * AT_TILE, sT + c_termB[k] * tterm + n0 * 128, k > 0 ? 1u : 0u);
    } else {
      mma_ss(r, sQ, sT + n0 * 128);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(r);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int e = (i >> 1) & 1, q = rl0 + 8 * e, col = n0 + 8 * (i >> 2) + c2 + (i & 1);
      const float v = SPLIT ? r[i] : r[i] * AT_LOG2E;
      if (col < hp) {
        const int k = iq[e] + h - 1 - col;
        if (k >= 0 && k < h) relh_s[q * h + k] = v;
      } else {
        const int k = jq[e] + w - 1 - (col - hp);
        if (k >= 0 && k < w) relw_s[q * w + k] = v;
      }
    }
  }
}

// bf16 bias rows, log2e-scaled, into relh_s / relw_s (and to global when relh_g / relw_g are given).  sQ: the query
// tile (its cp.async group committed); sT: scratch for the staged tables.
__device__ void compute_bias_rows(const AttnArgs& a, uint32_t sQ, uint32_t sT, int q0, float* relh_s, float* relw_s,
                                  float* relh_g, float* relw_g) {
  const int h = a.h, w = a.w;
  load_tables(a, sT);
  cp_async_commit();
  tiles_ready<0>();
  bias_rows_product<false>(h, w, a.N, sQ, sT, 0, q0, relh_s, relw_s);
  if (relh_g) {
    __syncthreads();
    for (int i = threadIdx.x; i < AT_BM * h; i += AT_THREADS) relh_g[static_cast<size_t>(q0) * h + i] = relh_s[i];
    for (int i = threadIdx.x; i < AT_BM * w; i += AT_THREADS) relw_g[static_cast<size_t>(q0) * w + i] = relw_s[i];
  }
}

// Image (row, column) of the 16 key columns nt * 8 + c2 + u (u = 0, 1) a thread holds in every 64-key tile: set for
// the first tile, then moved on by 64 keys per tile, so the score loops divide by w only once.
__device__ __forceinline__ void key_coords_init(int c2, int w, int (&kr)[16], int (&kc)[16]) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int x = (j >> 1) * 8 + c2 + (j & 1);
    kr[j] = x / w;
    kc[j] = x - kr[j] * w;
  }
}
__device__ __forceinline__ void key_coords_next(int dr, int dc, int w, int (&kr)[16], int (&kc)[16]) {
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    kr[j] += dr;
    kc[j] += dc;
    if (kc[j] >= w) {
      kc[j] -= w;
      ++kr[j];
    }
  }
}

// Shared-memory carve-ups (bytes past the 1024-byte aligned base; the launch adds 1024 bytes of alignment slack).
// forward / dQ: 2-stage K | V ring, which also holds the staged tables when no tile is in flight
__host__ __device__ inline size_t kv_ring_bytes(int h, int w) {
  const size_t t = table_bytes(h, w);
  return t > 4 * AT_TILE ? t : 4 * AT_TILE;
}
// dK/dV: one stage = Q | dO | relh rows [64][h] | relw rows [64][w] | lse [64] | delta [64]
__host__ __device__ inline size_t dkv_stage_bytes(int h, int w) {
  return (2 * AT_TILE + static_cast<size_t>(AT_BM) * (h + w) * 4 + 2 * AT_BM * 4 + 1023) / 1024 * 1024;
}

__device__ __forceinline__ uint8_t* aligned_smem(uint8_t* raw, uint32_t& base) {
  const uint32_t r = smem_u32(raw);
  base = (r + 1023u) & ~1023u;
  return raw + (base - r);
}

// ------------------------------------------------------------------------------------------------------------------
// forward.  grid (query tiles, heads, B)
// smem: sQ | K/V ring (tables before the loop) | relh_s [64][h] | relw_s [64][w]
__global__ void __launch_bounds__(AT_THREADS)
attn_fwd_kernel(const AttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint32_t sQ;
  uint8_t* sm = aligned_smem(smem_raw, sQ);
  const uint32_t ring = sQ + AT_TILE;
  const int h = a.h, w = a.w, N = a.N, C = a.heads * 64;
  float* relh_s = reinterpret_cast<float*>(sm + AT_TILE + kv_ring_bytes(h, w));
  float* relw_s = relh_s + AT_BM * h;
  const int q0 = blockIdx.x * AT_BM, head = blockIdx.y, b = blockIdx.z;
  const size_t bh = static_cast<size_t>(b) * a.heads + head;
  const __nv_bfloat16* base = a.qkv + static_cast<size_t>(b) * N * 3 * C;
  pdl_launch_dependents();
  pdl_wait();

  load_tile(sQ, base, 3 * C, q0, N, head * 64);
  cp_async_commit();
  compute_bias_rows(a, sQ, ring, q0, relh_s, relw_s, a.relh ? a.relh + bh * a.Np * h : nullptr,
                    a.relw ? a.relw + bh * a.Np * w : nullptr);
  __syncthreads();   // the tables are dead: the ring takes their place

  const int ntiles = (N + AT_BM - 1) / AT_BM;
  auto issue = [&](int t) {
    if (t < ntiles) {
      const uint32_t st = ring + (t & 1) * 2 * AT_TILE;
      load_tile(st, base, 3 * C, t * AT_BM, N, C + head * 64);
      load_tile(st + AT_TILE, base, 3 * C, t * AT_BM, N, 2 * C + head * 64);
    }
    cp_async_commit();
  };
  issue(0);

  const int lane = threadIdx.x & 31, g = lane >> 2, c2 = 2 * (lane & 3);
  const int rl0 = (threadIdx.x >> 5) * 16 + g;     // local query rows rl0, rl0 + 8
  const float sc = a.scale_log2;
  const int dr = AT_BM / w, dc = AT_BM - dr * w;
  int kr[16], kc[16];
  key_coords_init(c2, w, kr, kc);
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[32], s[32];
  zero32(o);
  zero32(s);
  const float* rh[2] = {relh_s + rl0 * h, relh_s + (rl0 + 8) * h};
  const float* rw[2] = {relw_s + rl0 * w, relw_s + (rl0 + 8) * w};

  // log2-domain scores of one key tile into s and their row maxima into mx.  The bias rows are gathered before the
  // first use.  PARTIAL (the last tile when 64 does not divide N): keys past N score -inf by a select, and their
  // gathers use a clamped image row.
  auto tile_scores = [&](int k0, float (&mx)[2], auto partial) {
    constexpr bool PARTIAL = decltype(partial)::value;
    float bias[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int j = 2 * (i >> 2) + (i & 1), e = (i >> 1) & 1;
      bias[i] = rh[e][PARTIAL ? min(kr[j], h - 1) : kr[j]] + rw[e][kc[j]];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float v = fmaf(s[i], sc, bias[i]);
      s[i] = PARTIAL ? (k0 + 8 * (i >> 2) + c2 + (i & 1) < N ? v : -INFINITY) : v;
      mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
    }
  };

  for (int t = 0; t < ntiles; ++t) {
    issue(t + 1);
    tiles_ready<1>();
    const uint32_t sK = ring + (t & 1) * 2 * AT_TILE, sV = sK + AT_TILE;
    const int k0 = t * AT_BM;
    wgmma_fence_operands(s);
    wgmma_fence();
    mma_ss(s, sQ, sK);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(s);
    float mx[2] = {-INFINITY, -INFINITY};
    if (k0 + AT_BM <= N) tile_scores(k0, mx, std::false_type{});
    else tile_scores(k0, mx, std::true_type{});
    float alpha[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
      const float mn = fmaxf(m[i], mx[i]);
      alpha[i] = fast_exp2(m[i] - mn);   // m = -inf on the first tile: alpha = 0 (nothing accumulated yet)
      m[i] = mn;
      l[i] *= alpha[i];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float p = fast_exp2(s[i] - m[(i >> 1) & 1]);
      s[i] = p;
      l[(i >> 1) & 1] += p;
      o[i] *= alpha[(i >> 1) & 1];
    }
    uint32_t pa[4][4];
    pack_frag(s, pa);
    wgmma_fence_operands(o);
    wgmma_fence();
    mma_rs(o, pa, sV);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(o);
    key_coords_next(dr, dc, w, kr, kc);
    __syncthreads();   // stage t & 1 is free for tile t + 2
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int t = q0 + rl0 + 8 * i;
    if (t >= N) continue;
    const float inv = 1.0f / l[i];
    __nv_bfloat16* orow = a.out + (static_cast<size_t>(b) * N + t) * C + head * 64;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt)
      *reinterpret_cast<uint32_t*>(orow + dt * 8 + c2) =
          pack_bf16x2(o[4 * dt + 2 * i] * inv, o[4 * dt + 2 * i + 1] * inv);
    if (a.lse && (lane & 3) == 0) a.lse[bh * N + t] = m[i] + log2f(l[i]);
  }
}

// bias rows only (pk_attn_bwd without rows kept by the forward).  grid (query tiles, heads, B)
// smem: sQ | tables | relh_s | relw_s
__global__ void __launch_bounds__(AT_THREADS)
attn_bias_rows_kernel(const AttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint32_t sQ;
  uint8_t* sm = aligned_smem(smem_raw, sQ);
  const int h = a.h, w = a.w, N = a.N, C = a.heads * 64;
  float* relh_s = reinterpret_cast<float*>(sm + AT_TILE + table_bytes(h, w));
  float* relw_s = relh_s + AT_BM * h;
  const int q0 = blockIdx.x * AT_BM, head = blockIdx.y, b = blockIdx.z;
  const size_t bh = static_cast<size_t>(b) * a.heads + head;
  pdl_launch_dependents();
  pdl_wait();
  load_tile(sQ, a.qkv + static_cast<size_t>(b) * N * 3 * C, 3 * C, q0, N, head * 64);
  cp_async_commit();
  compute_bias_rows(a, sQ, sQ + AT_TILE, q0, relh_s, relw_s, a.relh + bh * a.Np * h, a.relw + bh * a.Np * w);
}

// ------------------------------------------------------------------------------------------------------------------
// fp32-accurate forward (pk_attn_fwd_split3; the attention of windowed blocks in the fp32 inference mode).
// grid (query tiles, heads, B).  The tiling, key streaming and online softmax of attn_fwd_kernel on fp32 operands:
// every operand tile is staged as the three bf16 terms h, m, l of accurate.cu's split (split3.cuh), and each product is
// the six terms above 2^-24 in c_termA / c_termB order, accumulated in fp32 by wgmma:
//   S = sum_6 q_a k_b^T, R = sum_6 q_a [T_h; T_w]_b^T (bias rows), O += sum_6 p_a v_b (P split in registers).
// S is taken on the unscaled q and multiplied by 0.125 in the softmax (a power of two: exactly the product on the
// scaled q), so one split Q tile serves S and the bias rows, which the reference computes on the unscaled q.  The
// softmax runs in the natural-log domain with expf.  K and V arrive as raw fp32 through cp.async one tile ahead and
// are split in shared memory; Q and the tables are split on their way in.
// smem: sQ (3 terms) | split K (3) | split V (3) | raw K | raw V (two tiles of 64 rows x 32 fp32 each; the split
//       tables take the place of split K / V and raw before the loop) | relh_s [64][h] | relw_s [64][w]
struct SplitAttnArgs {
  const float* qkv;   // [B*N, 3C]
  const float* th;    // [2h-1, 64]
  const float* tw;    // [2w-1, 64]
  float* out;         // [B*N, C]
  int h, w, N, heads;
};

// Split 8 fp32 values into the three bf16 terms and store them as 16-byte chunk `ch` of row `row` of three swizzled
// tiles `tstride` bytes apart (term order h, m, l).
__device__ __forceinline__ void store_split8(uint32_t s, uint32_t tstride, int row, int ch, const float (&x)[8]) {
  uint32_t t[3][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    __nv_bfloat16 a[3], b[3];
    split3(x[2 * j], a);
    split3(x[2 * j + 1], b);
#pragma unroll
    for (int k = 0; k < 3; ++k)
      t[k][j] = static_cast<uint32_t>(__bfloat16_as_ushort(a[k])) |
                static_cast<uint32_t>(__bfloat16_as_ushort(b[k])) << 16;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k)
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(s + k * tstride + sw128(row, ch)), "r"(t[k][0]),
                 "r"(t[k][1]), "r"(t[k][2]), "r"(t[k][3]) : "memory");
}
// 8 fp32 from global (16-byte aligned), zeros when !valid
__device__ __forceinline__ void load8(const float* g, bool valid, float (&x)[8]) {
  float4 u = make_float4(0.f, 0.f, 0.f, 0.f), v = u;
  if (valid) {
    u = reinterpret_cast<const float4*>(g)[0];
    v = reinterpret_cast<const float4*>(g)[1];
  }
  x[0] = u.x; x[1] = u.y; x[2] = u.z; x[3] = u.w;
  x[4] = v.x; x[5] = v.y; x[6] = v.z; x[7] = v.w;
}

__global__ void __launch_bounds__(AT_THREADS)
attn_fwd_split3_kernel(const SplitAttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint32_t sQ;
  uint8_t* sm = aligned_smem(smem_raw, sQ);
  const int h = a.h, w = a.w, N = a.N, C = a.heads * 64;
  const uint32_t sKV = sQ + 3 * AT_TILE, sRaw = sKV + 6 * AT_TILE;
  const size_t tb = table_bytes(h, w), area = 3 * tb > 10 * AT_TILE ? 3 * tb : 10 * AT_TILE;
  float* relh_s = reinterpret_cast<float*>(sm + 3 * AT_TILE + area);
  float* relw_s = relh_s + AT_BM * h;
  const int q0 = blockIdx.x * AT_BM, head = blockIdx.y, b = blockIdx.z;
  const float* base = a.qkv + static_cast<size_t>(b) * N * 3 * C;
  pdl_launch_dependents();
  pdl_wait();

  // split Q tile and split tables (in the K / V area), then the bias rows
#pragma unroll
  for (int it = 0; it < (AT_BM * 8) / AT_THREADS; ++it) {
    const int idx = it * AT_THREADS + threadIdx.x, row = idx >> 3, ch = idx & 7;
    float x[8];
    load8(base + static_cast<size_t>(q0 + row) * 3 * C + head * 64 + ch * 8, q0 + row < N, x);
    store_split8(sQ, AT_TILE, row, ch, x);
  }
  {
    const int Lh = 2 * h - 1, Lw = 2 * w - 1, hp = tab_h_rows(h), rows = static_cast<int>(tb / 128);
    for (int idx = threadIdx.x; idx < rows * 8; idx += AT_THREADS) {
      const int row = idx >> 3, ch = idx & 7;
      const bool hs = row < hp;
      const int tr = hs ? row : row - hp;
      float x[8];
      load8((hs ? a.th : a.tw) + static_cast<size_t>(tr) * 64 + ch * 8, tr < (hs ? Lh : Lw), x);
      store_split8(sKV, static_cast<uint32_t>(tb), row, ch, x);
    }
  }
  fence_proxy_async_smem();
  __syncthreads();
  bias_rows_product<true>(h, w, N, sQ, sKV, static_cast<uint32_t>(tb), q0, relh_s, relw_s);
  __syncthreads();   // the tables are dead: split K / V and the raw tiles take their place

  // raw K / V tile t: each fp32 row of 64 is read as 128 bf16-sized columns, 32 fp32 per swizzled tile
  const int ntiles = (N + AT_BM - 1) / AT_BM;
  const __nv_bfloat16* raw = reinterpret_cast<const __nv_bfloat16*>(base);
  auto issue = [&](int t) {
    if (t < ntiles) {
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int j = 0; j < 2; ++j)
          load_tile(sRaw + (2 * m + j) * AT_TILE, raw, 6 * C, t * AT_BM, N, 2 * ((m + 1) * C + head * 64) + 64 * j);
    }
    cp_async_commit();
  };
  issue(0);

  const int lane = threadIdx.x & 31, g = lane >> 2, c2 = 2 * (lane & 3);
  const int rl0 = (threadIdx.x >> 5) * 16 + g;
  const int dr = AT_BM / w, dc = AT_BM - dr * w;
  int kr[16], kc[16];
  key_coords_init(c2, w, kr, kc);
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[32], s[32], pv[32];
  zero32(o);
  zero32(s);
  zero32(pv);

  for (int t = 0; t < ntiles; ++t) {
    cp_async_wait<0>();
    __syncthreads();   // raw tile t has landed; the products of tile t - 1 are done with split K / V
    // split: output chunk ch of a row covers fp32 columns [8 ch, 8 ch + 8): raw tile ch / 4, raw chunks 2 (ch % 4) (+1)
#pragma unroll
    for (int it = 0; it < (2 * AT_BM * 8) / AT_THREADS; ++it) {
      const int idx = it * AT_THREADS + threadIdx.x, mat = idx >> 9, row = (idx >> 3) & 63, ch = idx & 7;
      const uint32_t src = sRaw + (2 * mat + (ch >> 2)) * AT_TILE;
      float x[8];
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x[0]), "=f"(x[1]), "=f"(x[2]), "=f"(x[3])
                   : "r"(src + sw128(row, 2 * (ch & 3))) : "memory");
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x[4]), "=f"(x[5]), "=f"(x[6]), "=f"(x[7])
                   : "r"(src + sw128(row, 2 * (ch & 3) + 1)) : "memory");
      store_split8(sKV + mat * 3 * AT_TILE, AT_TILE, row, ch, x);
    }
    fence_proxy_async_smem();
    __syncthreads();   // split tiles visible to wgmma; the raw tiles are free
    issue(t + 1);
    const uint32_t sK = sKV, sV = sKV + 3 * AT_TILE;
    const int k0 = t * AT_BM;
    wgmma_fence_operands(s);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 6; ++k) mma_ss(s, sQ + c_termA[k] * AT_TILE, sK + c_termB[k] * AT_TILE, k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(s);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = k0 + nt * 8 + c2 + (e & 1), r = rl0 + 8 * (e >> 1);
        const int j = 2 * nt + (e & 1);
        float v = -INFINITY;
        if (key < N) v = fmaf(s[4 * nt + e], 0.125f, relh_s[r * h + kr[j]] + relw_s[r * w + kc[j]]);
        s[4 * nt + e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
    float alpha[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
      mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
      const float mn = fmaxf(m[i], mx[i]);
      alpha[i] = expf(m[i] - mn);   // m = -inf on the first tile: alpha = 0 (nothing accumulated yet)
      m[i] = mn;
      l[i] *= alpha[i];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float p = expf(s[i] - m[(i >> 1) & 1]);
      s[i] = p;
      l[(i >> 1) & 1] += p;
    }
    // P as three register fragments: h = bf16(p), m = bf16(p - h), l = bf16(p - h - m) (the differences are exact)
    uint32_t pa[3][4][4];
    pack_frag(s, pa[0]);
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] -= bf16_round(s[i]);
    pack_frag(s, pa[1]);
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] -= bf16_round(s[i]);
    pack_frag(s, pa[2]);
    // this tile's P V starts from zero, smallest terms first, and is added to O in fp32: the small terms are never
    // summed into the running O inside the tensor core, which does not round them like an fp32 add
    wgmma_fence_operands(pv);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 6; ++k) mma_rs(pv, pa[c_termA[k]], sV + c_termB[k] * AT_TILE, k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(pv);
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = fmaf(o[i], alpha[(i >> 1) & 1], pv[i]);
    key_coords_next(dr, dc, w, kr, kc);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 1);
    l[i] += __shfl_xor_sync(0xffffffffu, l[i], 2);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int t = q0 + rl0 + 8 * i;
    if (t >= N) continue;
    const float inv = 1.0f / l[i];
    float* orow = a.out + (static_cast<size_t>(b) * N + t) * C + head * 64;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt)
      *reinterpret_cast<float2*>(orow + dt * 8 + c2) = make_float2(o[4 * dt + 2 * i] * inv, o[4 * dt + 2 * i + 1] * inv);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// backward, dQ side.  grid (query tiles, heads, B)
//   dS = P * (dP - delta),  dQ = scale dS K + G [T_h; T_w]
//   dRelh[q, i] = sum of dS over the keys of image row i, dRelw[q, j] over image column j: per key tile the product
//   dS . E with the one-hot E[key x][column] = 1 at column (k0 + x) mod w and at column w + (k0 mod w + x) / w (image
//   row k0 / w + that offset).  w <= 56 (attn_check) keeps w plus the tile's image rows within 64 columns; for w = 1
//   the column part is left out and dRelw is the row sum of dRelh.  Each accumulator entry has one owner thread that
//   adds it up tile after tile: no atomics, a fixed order, reproducible.  Image-column entries are summed in
//   registers and stored to drelw_s after the loop; image-row entries are added into drelh_s.
//   G[q, r] = dRelh[q, i_q + h - 1 - r] for the T_h rows r of the staged tables (zero outside [0, h)), likewise for
//   T_w; the table-gradient partials of the CTA are G^T Q, ws[cta][c][table row].  TGRAD = false (frozen rel-pos
//   tables) leaves those partials out; dQ is computed by the same instructions in the same order either way.
// smem: sQ | sdO | K/V ring (tables after the loop) | E | relh_s | relw_s | drelh_s | drelw_s
template <bool TGRAD>
__global__ void __launch_bounds__(AT_THREADS)
attn_bwd_dq_kernel(const AttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint32_t sQ;
  uint8_t* sm = aligned_smem(smem_raw, sQ);
  const uint32_t sdO = sQ + AT_TILE, ring = sdO + AT_TILE, sE = ring + static_cast<uint32_t>(kv_ring_bytes(a.h, a.w));
  const int h = a.h, w = a.w, N = a.N, C = a.heads * 64, Lh = 2 * h - 1, Lw = 2 * w - 1;
  float* relh_s = reinterpret_cast<float*>(sm + (sE - sQ) + AT_TILE);
  float* relw_s = relh_s + AT_BM * h;
  float* drelh_s = relw_s + AT_BM * w;
  float* drelw_s = drelh_s + AT_BM * h;
  const int q0 = blockIdx.x * AT_BM, head = blockIdx.y, b = blockIdx.z;
  const size_t bh = static_cast<size_t>(b) * a.heads + head;
  const __nv_bfloat16* base = a.qkv + static_cast<size_t>(b) * N * 3 * C;
  pdl_launch_dependents();
  pdl_wait();

  load_tile(sQ, base, 3 * C, q0, N, head * 64);
  load_tile(sdO, a.dO + static_cast<size_t>(b) * N * C, C, q0, N, head * 64);
  cp_async_commit();
  const int ntiles = (N + AT_BM - 1) / AT_BM;
  auto issue = [&](int t) {
    if (t < ntiles) {
      const uint32_t st = ring + (t & 1) * 2 * AT_TILE;
      load_tile(st, base, 3 * C, t * AT_BM, N, C + head * 64);
      load_tile(st + AT_TILE, base, 3 * C, t * AT_BM, N, 2 * C + head * 64);
    }
    cp_async_commit();
  };
  issue(0);
  {
    const float* gh = a.relh + (bh * a.Np + q0) * h;
    const float* gw = a.relw + (bh * a.Np + q0) * w;
    for (int i = threadIdx.x; i < AT_BM * h; i += AT_THREADS) {
      relh_s[i] = gh[i];
      drelh_s[i] = 0.f;
    }
    for (int i = threadIdx.x; i < AT_BM * w; i += AT_THREADS) relw_s[i] = gw[i];
  }

  const int lane = threadIdx.x & 31, g = lane >> 2, c2 = 2 * (lane & 3);
  const int rl0 = (threadIdx.x >> 5) * 16 + g;
  const float sc = a.scale_log2;
  const int dr = AT_BM / w, dc = AT_BM - dr * w;
  const int wcols = w > 1 ? w : 0;   // E columns [0, wcols): image columns; then image rows from k0 / w on
  int kr[16], kc[16];
  key_coords_init(c2, w, kr, kc);
  int kr0 = 0, kc0 = 0;              // k0 / w, k0 mod w
  // image (row, column) of the key k0 + (threadIdx.x >> 3), the first of the four E rows this thread writes; the
  // other three are 16 keys apart
  const int er16 = 16 / w, ec16 = 16 - er16 * w;
  int er = (threadIdx.x >> 3) / w, ec = (threadIdx.x >> 3) - er * w;
  float lse[2], dlt[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int t = min(q0 + rl0 + 8 * i, N - 1);
    lse[i] = a.lse[bh * N + t];
    dlt[i] = a.delta[bh * N + t];
  }
  const float* rh[2] = {relh_s + rl0 * h, relh_s + (rl0 + 8) * h};
  const float* rw[2] = {relw_s + rl0 * w, relw_s + (rl0 + 8) * w};
  float dq[32], s[32], dp[32];
  // dRel_w of the accumulator entries i < 28 (columns below 56 >= w): an image column has the same E column in every
  // tile, so its sum over the key tiles stays in registers
  float dwc[28];
  // the image-row columns [wcols, wcols + 64 / w + 2) lie in the 8-column groups rc_lo .. rc_hi
  const int rc_lo = wcols >> 3, rc_hi = min(7, (wcols + AT_BM / w + 1) >> 3);
  zero32(dq);
  zero32(s);
  zero32(dp);
#pragma unroll
  for (int i = 0; i < 28; ++i) dwc[i] = 0.f;

  // dS of one tile into s.  PARTIAL (the last tile when 64 does not divide N): keys past N get dS = 0 by a select,
  // and their bias gathers use a clamped image row
  auto tile_ds = [&](int k0, auto partial) {
    constexpr bool PARTIAL = decltype(partial)::value;
    float bias[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int j = 2 * (i >> 2) + (i & 1), e = (i >> 1) & 1;
      bias[i] = rh[e][PARTIAL ? min(kr[j], h - 1) : kr[j]] + rw[e][kc[j]];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int e = (i >> 1) & 1;
      const float p = fast_exp2(fmaf(s[i], sc, bias[i]) - lse[e]);
      const float ds = p * (dp[i] - dlt[e]);
      s[i] = PARTIAL ? (k0 + 8 * (i >> 2) + c2 + (i & 1) < N ? ds : 0.f) : ds;
    }
  };

  for (int t = 0; t < ntiles; ++t) {
    issue(t + 1);
    // E of this tile (the previous tile's products that read it have completed)
    {
      int xr = er, xc = ec;
#pragma unroll
      for (int it = 0; it < (AT_BM * 8) / AT_THREADS; ++it) {
        const int x = it * (AT_THREADS / 8) + (threadIdx.x >> 3), ch = threadIdx.x & 7;
        const int ccol = w > 1 ? xc : -1, rcol = wcols + xr - kr0;
        uint32_t v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int c = ch * 8 + 2 * u;
          v[u] = (c == ccol || c == rcol ? 0x3F80u : 0u) | (c + 1 == ccol || c + 1 == rcol ? 0x3F800000u : 0u);
        }
        asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(sE + sw128(x, ch)), "r"(v[0]), "r"(v[1]),
                     "r"(v[2]), "r"(v[3]) : "memory");
        xr += er16;
        xc += ec16;
        if (xc >= w) {
          xc -= w;
          ++xr;
        }
      }
    }
    tiles_ready<1>();
    const uint32_t sK = ring + (t & 1) * 2 * AT_TILE, sV = sK + AT_TILE;
    const int k0 = t * AT_BM;
    wgmma_fence_operands(s);
    wgmma_fence_operands(dp);
    wgmma_fence();
    mma_ss(s, sQ, sK);
    mma_ss(dp, sdO, sV);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(s);
    wgmma_fence_operands(dp);
    if (k0 + AT_BM <= N) tile_ds(k0, std::false_type{});
    else tile_ds(k0, std::true_type{});
    uint32_t da[4][4];
    pack_frag(s, da);
    // dQ += dS . K and, into s, this tile's bias-row gradients dS . E
    wgmma_fence_operands(dq);
    wgmma_fence_operands(s);
    wgmma_fence();
    mma_rs(dq, da, sK);
    mma_rs(s, da, sE, 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(dq);
    wgmma_fence_operands(s);
#pragma unroll
    for (int i = 0; i < 28; ++i) dwc[i] += s[i];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      if (nt < rc_lo || nt > rc_hi) continue;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = 4 * nt + u, r = rl0 + 8 * (u >> 1), col = 8 * nt + c2 + (u & 1), ir = kr0 + col - wcols;
        if (col >= wcols && ir < h) drelh_s[r * h + ir] += s[i];
      }
    }
    key_coords_next(dr, dc, w, kr, kc);
    kr0 += dr;
    kc0 += dc;
    if (kc0 >= w) {
      kc0 -= w;
      ++kr0;
    }
    er += dr;
    ec += dc;
    if (ec >= w) {
      ec -= w;
      ++er;
    }
    __syncthreads();   // stage t & 1 is free for tile t + 2, E for tile t + 1
  }
  load_tables(a, ring);
  cp_async_commit();
#pragma unroll
  for (int i = 0; i < 28; ++i) {
    const int r = rl0 + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + c2 + (i & 1);
    if (col < wcols) drelw_s[r * w + col] = dwc[i];
  }
  if (w == 1 && threadIdx.x < AT_BM) {
    float acc = 0.f;
    for (int k = 0; k < h; ++k) acc += drelh_s[threadIdx.x * h + k];
    drelw_s[threadIdx.x] = acc;
  }
  tiles_ready<0>();   // tables staged, drelh_s / drelw_s complete

  // G[q, r] of the T_h rows (r < hp) and T_w rows of the staged tables; `q` local, `iq` / `jq` its image position
  const int hp = tab_h_rows(h), krows = tab_rows(h, w);
  auto gval = [&](int q, int iq, int jq, int r) -> float {
    if (r < hp) {
      const int k = iq + h - 1 - r;
      return k >= 0 && k < h ? drelh_s[q * h + k] : 0.f;
    }
    const int k = jq + w - 1 - (r - hp);
    return k >= 0 && k < w ? drelw_s[q * w + k] : 0.f;
  };

  // dQ = (dS K + 8 G [T_h; T_w]) / 8, written into the q columns of dqkv (G stored times 8: exact in bf16)
  {
    int iq[2], jq[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int tq = min(q0 + rl0 + 8 * e, N - 1);
      iq[e] = tq / w;
      jq[e] = tq - iq[e] * w;
    }
    const uint64_t dt = make_wgmma_desc(ring, AT_TILE, 1024);
    wgmma_fence_operands(dq);
    // The A fragments are built before the wgmmas that read them are issued, and those complete before the
    // fragments are rebuilt: 64 table rows per round, then 16 at a time.
    auto gfrag = [&](int kk, uint32_t (&ga)[4]) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int e = u & 1, q = rl0 + 8 * e, r = 16 * kk + 8 * (u >> 1) + c2;
        ga[u] = pack_bf16x2(8.f * gval(q, iq[e], jq[e], r), 8.f * gval(q, iq[e], jq[e], r + 1));
        asm volatile("" : "+r"(ga[u])::"memory");
      }
    };
    int kk = 0;
    for (; kk + 4 <= krows / 16; kk += 4) {
      uint32_t ga[4][4];
#pragma unroll
      for (int k = 0; k < 4; ++k) gfrag(kk + k, ga[k]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_m64n64k16_rs<1>(dq, ga[k], wgmma_desc_add(dt, (kk + k) * 2048), 1u);
      wgmma_commit();
      wgmma_wait<0>();
    }
    for (; kk < krows / 16; ++kk) {
      uint32_t ga[4];
      gfrag(kk, ga);
      wgmma_fence();
      wgmma_m64n64k16_rs<1>(dq, ga, wgmma_desc_add(dt, kk * 2048), 1u);
      wgmma_commit();
      wgmma_wait<0>();
    }
    wgmma_fence_operands(dq);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int t = q0 + rl0 + 8 * i;
    if (t < N) {
      __nv_bfloat16* drow = a.out + (static_cast<size_t>(b) * N + t) * 3 * C + head * 64;
#pragma unroll
      for (int dt = 0; dt < 8; ++dt)
        *reinterpret_cast<uint32_t*>(drow + dt * 8 + c2) =
            pack_bf16x2(dq[4 * dt + 2 * i] * 0.125f, dq[4 * dt + 2 * i + 1] * 0.125f);
    }
  }

  if constexpr (!TGRAD) return;
  // table-gradient partials of this CTA, G^T Q in 64-row chunks of the staged table rows (every entry of the slice
  // is written; queries past N contribute nothing)
  const int rows = Lh + Lw;
  float* ws = a.dt_ws + ((bh * gridDim.x) + blockIdx.x) * static_cast<size_t>(rows) * 64;
  int qiq[16], qjq[16];   // image position of the queries 16 kk + 8 v + c2 + u of the A fragments, iq = -h if past N
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int tq = q0 + (j >> 2) * 16 + ((j >> 1) & 1) * 8 + c2 + (j & 1);
    qiq[j] = tq < N ? tq / w : -h;
    qjq[j] = tq < N ? tq - qiq[j] * w : -w;
  }
  const uint64_t dqd = make_wgmma_desc(sQ, AT_TILE, 1024);
  float acc[32];
  zero32(acc);
  for (int m0 = 0; m0 < krows; m0 += AT_BM) {
    uint32_t ga[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = m0 + rl0 + 8 * (u & 1), j = 4 * kk + 2 * (u >> 1), q = j >> 2 << 4 | ((j >> 1) & 1) << 3 | c2;
        ga[kk][u] = pack_bf16x2(gval(q, qiq[j], qjq[j], r), gval(q + 1, qiq[j + 1], qjq[j + 1], r));
        asm volatile("" : "+r"(ga[kk][u])::"memory");
      }
    wgmma_fence_operands(acc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_m64n64k16_rs<1>(acc, ga[kk], wgmma_desc_add(dqd, kk * 2048), kk > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = m0 + rl0 + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + c2 + (i & 1);
      const int wr = r < hp ? (r < Lh ? r : -1) : (r - hp < Lw ? Lh + r - hp : -1);
      if (wr >= 0) ws[static_cast<size_t>(c) * rows + wr] = acc[i];
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// backward, dK / dV side.  grid (key tiles, heads, B); each warp owns 16 keys, the loop runs over the query tiles
//   P^T = exp2(scale K Q^T + bias - lse),  dV += P^T dO,  dS^T = P^T * (V dO^T - delta),  dK += scale dS^T Q
// smem: sK | sV | STAGES x (sQ | sdO | relh rows [64][h] | relw rows [64][w] | lse [64] | delta [64])
// STAGES = 2 overlaps the next query tile's loads with this one's math; 1 keeps two CTAs per SM on large grids.
template <int STAGES>
__global__ void __launch_bounds__(AT_THREADS)
attn_bwd_dkv_kernel(const AttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint32_t sK;
  uint8_t* sm = aligned_smem(smem_raw, sK);
  const uint32_t sV = sK + AT_TILE, ring = sV + AT_TILE;
  const int h = a.h, w = a.w, N = a.N, C = a.heads * 64;
  const uint32_t stage_bytes = static_cast<uint32_t>(dkv_stage_bytes(h, w));
  const int k0 = blockIdx.x * AT_BM, head = blockIdx.y, b = blockIdx.z;
  const size_t bh = static_cast<size_t>(b) * a.heads + head;
  const __nv_bfloat16* base = a.qkv + static_cast<size_t>(b) * N * 3 * C;
  const __nv_bfloat16* dObase = a.dO + static_cast<size_t>(b) * N * C;
  pdl_launch_dependents();
  pdl_wait();

  load_tile(sK, base, 3 * C, k0, N, C + head * 64);
  load_tile(sV, base, 3 * C, k0, N, 2 * C + head * 64);
  cp_async_commit();
  const int ntiles = (N + AT_BM - 1) / AT_BM;
  auto issue = [&](int t) {
    if (t < ntiles) {
      const int q0 = t * AT_BM;
      const uint32_t st = ring + (t % STAGES) * stage_bytes;
      load_tile(st, base, 3 * C, q0, N, head * 64);
      load_tile(st + AT_TILE, dObase, C, q0, N, head * 64);
      const uint32_t srh = st + 2 * AT_TILE, srw = srh + AT_BM * h * 4, sl = srw + AT_BM * w * 4;
      const float* gh = a.relh + (bh * a.Np + q0) * h;   // 64 rows: inside the Np-row buffer
      const float* gw = a.relw + (bh * a.Np + q0) * w;
      for (int i = threadIdx.x; i < AT_BM * h / 4; i += AT_THREADS) cp_async16(srh + 16 * i, gh + 4 * i, 16u);
      for (int i = threadIdx.x; i < AT_BM * w / 4; i += AT_THREADS) cp_async16(srw + 16 * i, gw + 4 * i, 16u);
      const int q = threadIdx.x & (AT_BM - 1), qc = min(q0 + q, N - 1);
      const uint32_t bytes = q0 + q < N ? 4u : 0u;
      if (threadIdx.x < AT_BM) cp_async4(sl + 4 * q, a.lse + bh * N + qc, bytes);
      else cp_async4(sl + AT_BM * 4 + 4 * q, a.delta + bh * N + qc, bytes);
    }
    cp_async_commit();
  };
#pragma unroll
  for (int t = 0; t < STAGES - 1; ++t) issue(t);

  const int lane = threadIdx.x & 31, g = lane >> 2, c2 = 2 * (lane & 3);
  const int kl0 = (threadIdx.x >> 5) * 16 + g;     // local key rows kl0, kl0 + 8
  int kr[2], kc[2];
  bool kvalid[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int key = k0 + kl0 + 8 * i;
    kvalid[i] = key < N;
    kr[i] = min(key, N - 1) / w;
    kc[i] = min(key, N - 1) - kr[i] * w;
  }
  const bool kfull = k0 + AT_BM <= N;
  const float sc = a.scale_log2;
  float dk[32], dv[32], s[32], dp[32];
  zero32(dk);
  zero32(dv);
  zero32(s);
  zero32(dp);

  // P^T into s and dS^T into dp for one query tile.  Every bias row and lse / delta value the thread needs is read
  // before the first use.  PARTIAL (a key or query tile cut by N): P = 0 past N by a select; all reads stay inside
  // the stage (kr / kc are clamped, queries past N read the zero-filled or zero-Q rows of the tile).
  auto tile_p = [&](const float* relh_s, const float* relw_s, const float* lse_s, const float* dlt_s, int q0,
                    auto partial) {
    constexpr bool PARTIAL = decltype(partial)::value;
    float bias[32], lq[16], dq[16];
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int q = 8 * (i >> 2) + c2 + (i & 1), e = (i >> 1) & 1;
      bias[i] = relh_s[q * h + kr[e]] + relw_s[q * w + kc[e]];
    }
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int q = 8 * (j >> 1) + c2 + (j & 1);
      lq[j] = lse_s[q];
      dq[j] = dlt_s[q];
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int j = 2 * (i >> 2) + (i & 1), e = (i >> 1) & 1;
      float p = fast_exp2(fmaf(s[i], sc, bias[i]) - lq[j]);
      if (PARTIAL) p = kvalid[e] && q0 + 8 * (i >> 2) + c2 + (i & 1) < N ? p : 0.f;
      s[i] = p;
      dp[i] = p * (dp[i] - dq[j]);
    }
  };

  for (int t = 0; t < ntiles; ++t) {
    issue(t + STAGES - 1);
    tiles_ready<STAGES - 1>();
    const int q0 = t * AT_BM;
    const uint32_t sQ = ring + (t % STAGES) * stage_bytes, sdO = sQ + AT_TILE;
    const float* relh_s = reinterpret_cast<const float*>(sm + (sQ - sK) + 2 * AT_TILE);
    const float* relw_s = relh_s + AT_BM * h;
    const float* lse_s = relw_s + AT_BM * w;
    const float* dlt_s = lse_s + AT_BM;
    wgmma_fence_operands(s);
    wgmma_fence_operands(dp);
    wgmma_fence();
    mma_ss(s, sK, sQ);
    mma_ss(dp, sV, sdO);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(s);
    wgmma_fence_operands(dp);
    if (kfull && q0 + AT_BM <= N) tile_p(relh_s, relw_s, lse_s, dlt_s, q0, std::false_type{});
    else tile_p(relh_s, relw_s, lse_s, dlt_s, q0, std::true_type{});
    uint32_t pa[4][4], da[4][4];
    pack_frag(s, pa);
    pack_frag(dp, da);
    wgmma_fence_operands(dv);
    wgmma_fence_operands(dk);
    wgmma_fence();
    mma_rs(dv, pa, sdO);
    mma_rs(dk, da, sQ);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_operands(dv);
    wgmma_fence_operands(dk);
    __syncthreads();   // this stage is free for tile t + STAGES
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int key = k0 + kl0 + 8 * i;
    if (key >= N) continue;
    __nv_bfloat16* row = a.out + (static_cast<size_t>(b) * N + key) * 3 * C + head * 64;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      *reinterpret_cast<uint32_t*>(row + C + dt * 8 + c2) =
          pack_bf16x2(dk[4 * dt + 2 * i] * 0.125f, dk[4 * dt + 2 * i + 1] * 0.125f);
      *reinterpret_cast<uint32_t*>(row + 2 * C + dt * 8 + c2) = pack_bf16x2(dv[4 * dt + 2 * i], dv[4 * dt + 2 * i + 1]);
    }
  }
}

// delta[b*heads + head][t] = sum_d O[b, t, head, d] * dO[b, t, head, d]: 8 lanes per (token, head) row of 64 bf16
// (one 16-byte load each from O and dO, fully coalesced), xor-shuffle tree, lane 0 of the group stores.
__global__ void __launch_bounds__(256)
attn_delta_kernel(const __nv_bfloat16* __restrict__ O, const __nv_bfloat16* __restrict__ dO,
                  float* __restrict__ delta, int B, int N, int heads) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t groups = static_cast<size_t>(B) * N * heads;
  const size_t g = idx >> 3;
  float acc = 0.f;
  if (g < groups) {
    const uint4 o = reinterpret_cast<const uint4*>(O)[idx], d = reinterpret_cast<const uint4*>(dO)[idx];
    const uint32_t ow[4] = {o.x, o.y, o.z, o.w}, dw[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      acc += bf16lo(ow[e]) * bf16lo(dw[e]);
      acc += bf16hi(ow[e]) * bf16hi(dw[e]);
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (g < groups && (idx & 7) == 0) {
    const size_t tok = g / heads, head = g - tok * heads;
    const size_t b = tok / N, t = tok - b * N;
    delta[(b * heads + head) * N + t] = acc;
  }
}

// dT[r][c] += sum over CTA slices ws[cta][c][r] (table row innermost).  grid (64 columns, DT_STRIPES, row chunks), block
// (DT_RX, DT_RY): threadIdx.x walks the table rows (coalesced), the slices are strided over blockIdx.y / threadIdx.y
// with four loads in flight per thread, smem tree over threadIdx.y, one atomic per (row, column, stripe).
constexpr int DT_STRIPES = 4;
constexpr int DT_RX = 64, DT_RY = 16;
__global__ void __launch_bounds__(DT_RX * DT_RY)
attn_dt_reduce_kernel(const float* __restrict__ ws, int nctas, int rows, int rows_h, float* __restrict__ dTh,
                      float* __restrict__ dTw) {
  __shared__ float red[DT_RY][DT_RX];
  pdl_launch_dependents();
  pdl_wait();
  const int c = blockIdx.x;
  const size_t slice = static_cast<size_t>(rows) * 64;
  const int step = DT_STRIPES * DT_RY;
  {
    const int r = blockIdx.z * DT_RX + threadIdx.x;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    if (r < rows) {
      const float* p = ws + static_cast<size_t>(c) * rows + r;
      int i = blockIdx.y * DT_RY + threadIdx.y;
      for (; i + 3 * step < nctas; i += 4 * step) {
        s0 += p[static_cast<size_t>(i) * slice];
        s1 += p[static_cast<size_t>(i + step) * slice];
        s2 += p[static_cast<size_t>(i + 2 * step) * slice];
        s3 += p[static_cast<size_t>(i + 3 * step) * slice];
      }
      for (; i < nctas; i += step) s0 += p[static_cast<size_t>(i) * slice];
    }
    red[threadIdx.y][threadIdx.x] = (s0 + s1) + (s2 + s3);
    __syncthreads();
    if (threadIdx.y == 0 && r < rows) {
      float s = 0.f;
#pragma unroll
      for (int y = 0; y < DT_RY; ++y) s += red[y][threadIdx.x];
      float* dst = r < rows_h ? dTh + static_cast<size_t>(r) * 64 + c : dTw + static_cast<size_t>(r - rows_h) * 64 + c;
      atomicAdd(dst, s);
    }
  }
}

static int attn_check(const void* qkv, const void* th, const void* tw, int B, int heads, int h, int w, int th_pad,
                      int tw_pad, const char* who) {
  PK_CHECK(qkv && th && tw, "%s: null pointer", who);
  PK_CHECK(B > 0 && heads > 0 && h > 0 && w > 0, "%s: bad shape", who);
  PK_CHECK(th_pad % 16 == 0 && tw_pad % 16 == 0 && th_pad >= 2 * h - 1 && tw_pad >= 2 * w - 1 && th_pad <= 224 &&
               tw_pad <= 112,
           "%s: bad table padding th_pad=%d tw_pad=%d (h=%d w=%d)", who, th_pad, tw_pad, h, w);
  return 0;
}

static AttnArgs attn_args(const void* qkv, const void* th, const void* tw, int B, int heads, int h, int w) {
  AttnArgs a;
  memset(&a, 0, sizeof(a));
  a.qkv = static_cast<const __nv_bfloat16*>(qkv);
  a.th = static_cast<const __nv_bfloat16*>(th);
  a.tw = static_cast<const __nv_bfloat16*>(tw);
  a.h = h;
  a.w = w;
  a.N = h * w;
  a.Np = (a.N + 127) / 128 * 128;
  a.heads = heads;
  a.scale_log2 = 0.125f * AT_LOG2E;
  return a;
}

template <class Args>
static int launch_attn(void (*kernel)(Args), dim3 grid, size_t smem, cudaStream_t st, const Args& a, const char* who) {
  PK_CHECK(smem <= 227 * 1024, "%s: h=%d w=%d needs %zu B of shared memory", who, a.h, a.w, smem);
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  PK_CHECK(e == cudaSuccess, "%s: cudaFuncSetAttribute: %s", who, cudaGetErrorString(e));
  e = launch_pdl(kernel, grid, dim3(AT_THREADS), smem, st, a);
  PK_CHECK(e == cudaSuccess, "%s: launch: %s", who, cudaGetErrorString(e));
  PK_LAUNCH_CHECK(who);
  return 0;
}

static int attn_fwd_impl(const void* qkv, const void* th, const void* tw, void* out, float* lse, float* relh_out,
                         float* relw_out, int B, int heads, int h, int w, int th_pad, int tw_pad, void* stream) {
  if (attn_check(qkv, th, tw, B, heads, h, w, th_pad, tw_pad, "pk_attn_fwd")) return 1;
  PK_CHECK(out, "pk_attn_fwd: null pointer");
  AttnArgs a = attn_args(qkv, th, tw, B, heads, h, w);
  a.out = static_cast<__nv_bfloat16*>(out);
  a.lse = lse;
  a.relh = relh_out;
  a.relw = relw_out;
  const size_t smem = 1024 + AT_TILE + kv_ring_bytes(h, w) + static_cast<size_t>(AT_BM) * (h + w) * 4;
  dim3 grid((a.N + AT_BM - 1) / AT_BM, heads, B);
  return launch_attn(attn_fwd_kernel, grid, smem, static_cast<cudaStream_t>(stream), a, "pk_attn_fwd");
}

}  // namespace pk

using namespace pk;

// qkv: bf16 [B*N, 3C] (columns (3, head, 64) as produced by the qkv Linear, models_painter.py:76-78)
// th / tw: bf16 rel-pos tables, zero-padded to th_pad / tw_pad rows (multiples of 16), [rows, 64]
extern "C" int pk_attn_fwd(const void* qkv, const void* th, const void* tw, void* out, float* lse, int B,
                           int heads, int h, int w, int th_pad, int tw_pad, void* stream) {
  return attn_fwd_impl(qkv, th, tw, out, lse, nullptr, nullptr, B, heads, h, w, th_pad, tw_pad, stream);
}
// training forward: additionally stores every query's bias rows (relh_g / relw_g: B*heads*Np*h resp. *w floats,
// Np = N rounded up to 128) for pk_attn_bwd_saved
extern "C" int pk_attn_fwd_save(const void* qkv, const void* th, const void* tw, void* out, float* lse, float* relh_g,
                                float* relw_g, int B, int heads, int h, int w, int th_pad, int tw_pad, void* stream) {
  PK_CHECK(lse && relh_g && relw_g, "pk_attn_fwd_save: null pointer");
  return attn_fwd_impl(qkv, th, tw, out, lse, relh_g, relw_g, B, heads, h, w, th_pad, tw_pad, stream);
}

// fp32-accurate forward: qkv fp32 [B*N, 3C] (the qkv GEMM's layout), th / tw the fp32 tables [2h-1, 64] /
// [2w-1, 64], out fp32 [B*N, C] (heads merged, like pk_attn_fwd)
extern "C" int pk_attn_fwd_split3(const float* qkv, const float* th, const float* tw, float* out, int B, int heads,
                                  int h, int w, void* stream) {
  PK_CHECK(qkv && th && tw && out, "pk_attn_fwd_split3: null pointer");
  PK_CHECK(B > 0 && heads > 0 && h > 0 && w > 0 && h <= 112 && w <= 56, "pk_attn_fwd_split3: bad shape h=%d w=%d", h,
           w);
  SplitAttnArgs a{qkv, th, tw, out, h, w, h * w, heads};
  const size_t tb = table_bytes(h, w);
  const size_t smem = 1024 + 3 * AT_TILE + (3 * tb > 10 * AT_TILE ? 3 * tb : 10 * AT_TILE) +
                      static_cast<size_t>(AT_BM) * (h + w) * 4;
  const dim3 grid((a.N + AT_BM - 1) / AT_BM, heads, B);
  return launch_attn(attn_fwd_split3_kernel, grid, smem, static_cast<cudaStream_t>(stream), a, "pk_attn_fwd_split3");
}

// qkv / dqkv: bf16 [B*N, 3C];  O, dO: bf16 [B*N, C];  lse: fp32 [B*heads, N] from pk_attn_fwd
// scratch buffers (caller-allocated): delta [B*heads*N], relh_g [B*heads*Np*h], relw_g [B*heads*Np*w] fp32 with
// Np = N rounded up to a multiple of 128 (query-major rows of bias values)
// dt_ws: pk_attn_bwd_ws_floats(B, heads, h, w) fp32 (per-CTA partial table gradients)
// dTh [2h-1, 64], dTw [2w-1, 64]: fp32, ADDED to (caller zero-initialises or passes a running gradient); both NULL:
// no table gradients (the dQ kernel skips its G^T Q partials, no reduction runs, dt_ws may be NULL), dqkv unchanged
extern "C" long long pk_attn_bwd_ws_floats(int B, int heads, int h, int w) {
  const long long ctas = static_cast<long long>((h * w + AT_BM - 1) / AT_BM) * heads * B;
  return ctas * (2 * h - 1 + 2 * w - 1) * 64;
}

static int attn_bwd_impl(const void* qkv, const void* O, const void* dO, const float* lse, const void* th,
                         const void* tw, void* dqkv, float* dTh, float* dTw, float* delta, float* relh_g,
                         float* relw_g, float* dt_ws, int B, int heads, int h, int w, int th_pad, int tw_pad,
                         int rel_ready, void* stream) {
  if (attn_check(qkv, th, tw, B, heads, h, w, th_pad, tw_pad, "pk_attn_bwd")) return 1;
  PK_CHECK(O && dO && lse && dqkv && delta && relh_g && relw_g, "pk_attn_bwd: null pointer");
  // dTh = dTw = NULL: the tables' gradients are not needed (frozen tables); dt_ws is then unused and may be NULL
  const bool tgrad = dTh != nullptr;
  PK_CHECK((dTw != nullptr) == tgrad, "pk_attn_bwd: dTh and dTw must both be given or both be NULL");
  PK_CHECK(!tgrad || dt_ws, "pk_attn_bwd: null pointer (dt_ws)");
  AttnArgs a = attn_args(qkv, th, tw, B, heads, h, w);
  a.O = static_cast<const __nv_bfloat16*>(O);
  a.dO = static_cast<const __nv_bfloat16*>(dO);
  a.out = static_cast<__nv_bfloat16*>(dqkv);
  a.lse = const_cast<float*>(lse);
  a.delta = delta;
  a.relh = relh_g;
  a.relw = relw_g;
  a.dt_ws = dt_ws;
  const int N = a.N;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid((N + AT_BM - 1) / AT_BM, heads, B);
  const size_t rel_bytes = static_cast<size_t>(AT_BM) * (h + w) * 4;
  if (!rel_ready) {
    if (launch_attn(attn_bias_rows_kernel, grid, 1024 + AT_TILE + table_bytes(h, w) + rel_bytes, st, a,
                    "pk_attn_bwd(bias rows)"))
      return 2;
  }
  {
    const size_t threads = static_cast<size_t>(B) * N * heads * 8;
    launch_pdl(attn_delta_kernel, dim3(static_cast<unsigned>((threads + 255) / 256)), dim3(256), 0, st,
               static_cast<const __nv_bfloat16*>(O), static_cast<const __nv_bfloat16*>(dO), delta, B, N, heads);
    PK_LAUNCH_CHECK("pk_attn_bwd(delta)");
  }
  if (launch_attn(tgrad ? attn_bwd_dq_kernel<true> : attn_bwd_dq_kernel<false>, grid,
                  1024 + 3 * AT_TILE + kv_ring_bytes(h, w) + 2 * rel_bytes, st, a,
                  "pk_attn_bwd(dq)"))
    return 2;
  {
    // two query-tile stages while two CTAs still fit on an SM (228 KB, 1 KB reserved per CTA), else one
    const size_t smem1 = 1024 + 2 * AT_TILE + dkv_stage_bytes(h, w), smem2 = smem1 + dkv_stage_bytes(h, w);
    const bool two = smem2 <= 113 * 1024;
    if (launch_attn(two ? attn_bwd_dkv_kernel<2> : attn_bwd_dkv_kernel<1>, grid, two ? smem2 : smem1, st, a,
                    "pk_attn_bwd(dkv)"))
      return 2;
  }
  if (tgrad) {
    const int rows = 2 * h - 1 + 2 * w - 1;
    const int nctas = static_cast<int>(grid.x * grid.y * grid.z);
    launch_pdl(attn_dt_reduce_kernel, dim3(64, DT_STRIPES, (rows + DT_RX - 1) / DT_RX), dim3(DT_RX, DT_RY), 0, st,
               static_cast<const float*>(dt_ws), nctas, rows, 2 * h - 1, dTh, dTw);
    PK_LAUNCH_CHECK("pk_attn_bwd(dT reduce)");
  }
  return 0;
}

extern "C" int pk_attn_bwd(const void* qkv, const void* O, const void* dO, const float* lse, const void* th,
                           const void* tw, void* dqkv, float* dTh, float* dTw, float* delta, float* relh_g,
                           float* relw_g, float* dt_ws, int B, int heads, int h, int w, int th_pad, int tw_pad,
                           void* stream) {
  return attn_bwd_impl(qkv, O, dO, lse, th, tw, dqkv, dTh, dTw, delta, relh_g, relw_g, dt_ws, B, heads, h, w, th_pad,
                       tw_pad, 0, stream);
}
// relh_g / relw_g are INPUTS here: the bias rows stored by pk_attn_fwd_save on the same qkv / tables
extern "C" int pk_attn_bwd_saved(const void* qkv, const void* O, const void* dO, const float* lse, const void* th,
                                 const void* tw, void* dqkv, float* dTh, float* dTw, float* delta,
                                 const float* relh_g, const float* relw_g, float* dt_ws, int B, int heads, int h, int w,
                                 int th_pad, int tw_pad, void* stream) {
  return attn_bwd_impl(qkv, O, dO, lse, th, tw, dqkv, dTh, dTw, delta, const_cast<float*>(relh_g),
                       const_cast<float*>(relw_g), dt_ws, B, heads, h, w, th_pad, tw_pad, 1, stream);
}

// fp32 table [L, 64] -> bf16 [Lpad, 64], rows >= L zero  (rel_pos_h / rel_pos_w, models_painter.py:66-67)
__global__ void pad_cast_table_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, int L,
                                      int Lpad) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= Lpad * 64) return;
  out[idx] = __float2bfloat16_rn(idx < L * 64 ? in[idx] : 0.f);
}
extern "C" int pk_relpos_table_bf16(const float* table, void* out_bf16, int L, int Lpad, void* stream) {
  PK_CHECK(table && out_bf16 && Lpad >= L, "pk_relpos_table_bf16: bad args");
  pad_cast_table_kernel<<<(Lpad * 64 + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      table, static_cast<__nv_bfloat16*>(out_bf16), L, Lpad);
  PK_LAUNCH_CHECK("pk_relpos_table_bf16");
  return 0;
}
