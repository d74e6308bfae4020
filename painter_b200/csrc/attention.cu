// painter_b200 — fused global attention with decomposed relative-position bias, forward and backward (sm_90a).
//
// Replaces models_painter.py:73-86 + util/vitdet_utils.py:63-125 (q*scale @ k^T, add_decomposed_rel_pos, softmax,
// @ v) and autograd's backward through them, without ever materialising the [B*heads, N, N] score tensor.
//
// Every kernel works on 64-row tiles with 4 warps (16 rows each) and bf16 tensor-core MMAs (mma.sync m16n8k16, fp32
// accumulation); the probabilities P stay in registers between the two products (their accumulator fragment is the
// A-operand fragment of the next MMA), operand tiles are staged in padded shared memory (row stride 72 bf16:
// fragment loads are conflict-free).
//   forward   one CTA per 64 queries of one (batch, head): S = Q K^T over 64-key tiles, online softmax in the log2
//             domain, O += P V; writes O and the log-sum-exp.
//   backward  dQ kernel (per 64 queries; also the bias-row gradients and the per-CTA table-gradient partials) and
//             dK/dV kernel (per 64 keys, loops over the query tiles); both recompute P from the log-sum-exp.
// The bias rows rel_h[q, i] = q . T_h[i_q - i + h - 1] and rel_w[q, j] = q . T_w[j_q - j + w - 1] (h + w dot products
// per query, ~3 % of the attention FLOPs) are computed once per query tile on the FMA pipe and kept, log2e-scaled, in
// shared memory; the training forward stores them for the backward kernels ([B*heads, Np, h] / [B*heads, Np, w]).
#include "common.cuh"
#include "host_common.h"
#include "../../include/painter_b200.h"

namespace pk {

constexpr int AT_BM = 64;          // rows (queries or keys) per CTA and per loop tile
constexpr int AT_THREADS = 128;
constexpr int AT_LDS = 72;         // bf16 per staged row (64 + 8 pad)
constexpr int AT_TILE = AT_BM * AT_LDS;   // bf16 elements of one staged 64 x 64 tile
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

__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t lds32(const __nv_bfloat16* s, int row, int col) {
  return *reinterpret_cast<const uint32_t*>(s + row * AT_LDS + col);
}
__device__ __forceinline__ float bf16lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16hi(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }

// Stage rows [r0, r0 + 64) x columns [c0, c0 + 64) of a bf16 matrix (row stride ld elements, rows >= nrows read as
// zero): row-major into s[row][col] and/or transposed into st[col][row].
__device__ __forceinline__ void stage_tile(const __nv_bfloat16* g, size_t ld, int r0, int nrows, int c0,
                                           __nv_bfloat16* s, __nv_bfloat16* st) {
#pragma unroll
  for (int it = 0; it < (AT_BM * 8) / AT_THREADS; ++it) {
    const int idx = it * AT_THREADS + threadIdx.x;
    const int row = idx >> 3, ch = idx & 7;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r0 + row < nrows) v = *reinterpret_cast<const uint4*>(g + static_cast<size_t>(r0 + row) * ld + c0 + ch * 8);
    if (s != nullptr) *reinterpret_cast<uint4*>(s + row * AT_LDS + ch * 8) = v;
    if (st != nullptr) {
      const __nv_bfloat16* e = reinterpret_cast<const __nv_bfloat16*>(&v);
#pragma unroll
      for (int k = 0; k < 8; ++k) st[(ch * 8 + k) * AT_LDS + row] = e[k];
    }
  }
}

// A-operand fragments of rows [16 warp, 16 warp + 16) x 64 of a staged row-major tile
__device__ __forceinline__ void load_afrag(const __nv_bfloat16* s, uint32_t (&a)[4][4]) {
  const int lane = threadIdx.x & 31, r = (threadIdx.x >> 5) * 16 + (lane >> 2), c = 2 * (lane & 3);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
    a[ks][0] = lds32(s, r, ks * 16 + c);
    a[ks][1] = lds32(s, r + 8, ks * 16 + c);
    a[ks][2] = lds32(s, r, ks * 16 + c + 8);
    a[ks][3] = lds32(s, r + 8, ks * 16 + c + 8);
  }
}
// acc[16 x 64] += A[16 x 64] . B^T, B = 64 rows of a staged row-major tile (rows = output columns)
__device__ __forceinline__ void mma_rows(float (&acc)[8][4], const uint32_t (&a)[4][4], const __nv_bfloat16* sb) {
  const int lane = threadIdx.x & 31, g = lane >> 2, c = 2 * (lane & 3);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
      mma_16816(acc[nt], a[ks], lds32(sb, nt * 8 + g, ks * 16 + c), lds32(sb, nt * 8 + g, ks * 16 + c + 8));
}
// acc[16 x 64] += P[16 x 64] . B, P given as accumulator fragments (bf16-rounded here), B^T staged row-major
__device__ __forceinline__ void mma_p(float (&acc)[8][4], const float (&p)[8][4], const __nv_bfloat16* sbt) {
  const int lane = threadIdx.x & 31, g = lane >> 2, c = 2 * (lane & 3);
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint32_t a[4] = {pack_bf16x2(p[2 * kk][0], p[2 * kk][1]), pack_bf16x2(p[2 * kk][2], p[2 * kk][3]),
                           pack_bf16x2(p[2 * kk + 1][0], p[2 * kk + 1][1]),
                           pack_bf16x2(p[2 * kk + 1][2], p[2 * kk + 1][3])};
#pragma unroll
    for (int dt = 0; dt < 8; ++dt)
      mma_16816(acc[dt], a, lds32(sbt, dt * 8 + g, kk * 16 + c), lds32(sbt, dt * 8 + g, kk * 16 + c + 8));
  }
}

// Bias rows of the 64 queries [q0, q0 + 64) of one (batch, head), log2e-scaled, into relh_s [64][h] / relw_s [64][w]
// (and to global when relh_g / relw_g are given).  sQ: the staged query tile; sT: scratch for both bf16 tables.
__device__ void compute_bias_rows(const AttnArgs& a, const __nv_bfloat16* sQ, __nv_bfloat16* sT, int q0,
                                  float* relh_s, float* relw_s, float* relh_g, float* relw_g) {
  const int h = a.h, w = a.w, Lh = 2 * h - 1, Lw = 2 * w - 1;
  for (int idx = threadIdx.x; idx < (Lh + Lw) * 8; idx += AT_THREADS) {
    const int row = idx >> 3, ch = idx & 7;
    const __nv_bfloat16* src = row < Lh ? a.th + static_cast<size_t>(row) * 64 : a.tw + static_cast<size_t>(row - Lh) * 64;
    *reinterpret_cast<uint4*>(sT + row * AT_LDS + ch * 8) = *reinterpret_cast<const uint4*>(src + ch * 8);
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < AT_BM * (h + w); idx += AT_THREADS) {
    const int q = idx / (h + w), k = idx - q * (h + w);
    const int t = min(q0 + q, a.N - 1);
    const int iq = t / w, jq = t - iq * w;
    const int trow = k < h ? iq - k + h - 1 : Lh + jq - (k - h) + w - 1;
    const uint32_t* qa = reinterpret_cast<const uint32_t*>(sQ + q * AT_LDS);
    const uint32_t* ta = reinterpret_cast<const uint32_t*>(sT + trow * AT_LDS);
    float s0 = 0.f, s1 = 0.f;
#pragma unroll 8
    for (int c = 0; c < 32; ++c) {
      const uint32_t x = qa[c], y = ta[c];
      s0 = fmaf(bf16lo(x), bf16lo(y), s0);
      s1 = fmaf(bf16hi(x), bf16hi(y), s1);
    }
    const float v = (s0 + s1) * AT_LOG2E;
    if (k < h) {
      relh_s[q * h + k] = v;
      if (relh_g) relh_g[static_cast<size_t>(q0 + q) * h + k] = v;
    } else {
      relw_s[q * w + k - h] = v;
      if (relw_g) relw_g[static_cast<size_t>(q0 + q) * w + k - h] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------
// forward.  grid (query tiles, heads, B)
// smem: sQ | sK | sVt | tables (2h-1 + 2w-1 rows) | relh_s [64][h] | relw_s [64][w]
__global__ void __launch_bounds__(AT_THREADS)
attn_fwd_kernel(const AttnArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sK = sQ + AT_TILE;
  __nv_bfloat16* sVt = sK + AT_TILE;
  __nv_bfloat16* sT = sVt + AT_TILE;
  const int h = a.h, w = a.w, N = a.N, C = a.heads * 64;
  float* relh_s = reinterpret_cast<float*>(sT + (2 * h - 1 + 2 * w - 1) * AT_LDS);
  float* relw_s = relh_s + AT_BM * h;
  const int q0 = blockIdx.x * AT_BM, head = blockIdx.y, b = blockIdx.z;
  const size_t bh = static_cast<size_t>(b) * a.heads + head;
  const __nv_bfloat16* base = a.qkv + static_cast<size_t>(b) * N * 3 * C;
  pdl_launch_dependents();
  pdl_wait();

  stage_tile(base, 3 * C, q0, N, head * 64, sQ, nullptr);
  __syncthreads();
  compute_bias_rows(a, sQ, sT, q0, relh_s, relw_s, a.relh ? a.relh + bh * a.Np * h : nullptr,
                    a.relw ? a.relw + bh * a.Np * w : nullptr);
  uint32_t qa[4][4];
  load_afrag(sQ, qa);

  const int lane = threadIdx.x & 31, g = lane >> 2, c2 = 2 * (lane & 3);
  const int rl0 = (threadIdx.x >> 5) * 16 + g;     // local query rows rl0, rl0 + 8
  const float sc = a.scale_log2;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f;

  for (int k0 = 0; k0 < N; k0 += AT_BM) {
    __syncthreads();
    stage_tile(base, 3 * C, k0, N, C + head * 64, sK, nullptr);
    stage_tile(base, 3 * C, k0, N, 2 * C + head * 64, nullptr, sVt);
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
    mma_rows(s, qa, sK);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = k0 + nt * 8 + c2 + (e & 1), r = rl0 + 8 * (e >> 1);
        float v = -INFINITY;
        if (key < N) {
          const int kr = key / w, kc = key - kr * w;
          v = fmaf(s[nt][e], sc, relh_s[r * h + kr] + relw_s[r * w + kc]);
        }
        s[nt][e] = v;
        mx[e >> 1] = fmaxf(mx[e >> 1], v);
      }
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
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float p = fast_exp2(s[nt][e] - m[e >> 1]);
        s[nt][e] = p;
        l[e >> 1] += p;
        o[nt][e] *= alpha[e >> 1];
      }
    mma_p(o, s, sVt);
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
      *reinterpret_cast<uint32_t*>(orow + dt * 8 + c2) = pack_bf16x2(o[dt][2 * i] * inv, o[dt][2 * i + 1] * inv);
    if (a.lse && (lane & 3) == 0) a.lse[bh * N + t] = m[i] + log2f(l[i]);
  }
}

// bias rows only (pk_attn_bwd without rows kept by the forward).  grid (query tiles, heads, B)
__global__ void __launch_bounds__(AT_THREADS)
attn_bias_rows_kernel(const AttnArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sT = sQ + AT_TILE;
  const int h = a.h, w = a.w, N = a.N, C = a.heads * 64;
  float* relh_s = reinterpret_cast<float*>(sT + (2 * h - 1 + 2 * w - 1) * AT_LDS);
  float* relw_s = relh_s + AT_BM * h;
  const int q0 = blockIdx.x * AT_BM, head = blockIdx.y, b = blockIdx.z;
  const size_t bh = static_cast<size_t>(b) * a.heads + head;
  pdl_launch_dependents();
  pdl_wait();
  stage_tile(a.qkv + static_cast<size_t>(b) * N * 3 * C, 3 * C, q0, N, head * 64, sQ, nullptr);
  __syncthreads();
  compute_bias_rows(a, sQ, sT, q0, relh_s, relw_s, a.relh + bh * a.Np * h, a.relw + bh * a.Np * w);
}

// ------------------------------------------------------------------------------------------------------------------
// backward, dQ side.  grid (query tiles, heads, B)
//   dS = P * (dP - delta),  dQ = scale dS K + dRelh . T_h(gathered) + dRelw . T_w(gathered)
//   dRelh[q, i] = sum of dS over the keys of image row i, dRelw[q, j] over image column j (shared-memory atomics)
//   table-gradient partials: ws[cta][c][r] = sum_q dRel[q, .] q[c] over the (q, bias column) pairs hitting table row r
// smem: sQ | sdO | sK | sKt | sV | tables | relh_s | relw_s | drelh_s | drelw_s
__global__ void __launch_bounds__(AT_THREADS)
attn_bwd_dq_kernel(const AttnArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sdO = sQ + AT_TILE;
  __nv_bfloat16* sK = sdO + AT_TILE;
  __nv_bfloat16* sKt = sK + AT_TILE;
  __nv_bfloat16* sV = sKt + AT_TILE;
  __nv_bfloat16* sT = sV + AT_TILE;
  const int h = a.h, w = a.w, N = a.N, C = a.heads * 64, Lh = 2 * h - 1, Lw = 2 * w - 1;
  float* relh_s = reinterpret_cast<float*>(sT + (Lh + Lw) * AT_LDS);
  float* relw_s = relh_s + AT_BM * h;
  float* drelh_s = relw_s + AT_BM * w;
  float* drelw_s = drelh_s + AT_BM * h;
  const int q0 = blockIdx.x * AT_BM, head = blockIdx.y, b = blockIdx.z;
  const size_t bh = static_cast<size_t>(b) * a.heads + head;
  const __nv_bfloat16* base = a.qkv + static_cast<size_t>(b) * N * 3 * C;
  pdl_launch_dependents();
  pdl_wait();

  stage_tile(base, 3 * C, q0, N, head * 64, sQ, nullptr);
  stage_tile(a.dO + static_cast<size_t>(b) * N * C, C, q0, N, head * 64, sdO, nullptr);
  for (int idx = threadIdx.x; idx < (Lh + Lw) * 8; idx += AT_THREADS) {
    const int row = idx >> 3, ch = idx & 7;
    const __nv_bfloat16* src = row < Lh ? a.th + static_cast<size_t>(row) * 64 : a.tw + static_cast<size_t>(row - Lh) * 64;
    *reinterpret_cast<uint4*>(sT + row * AT_LDS + ch * 8) = *reinterpret_cast<const uint4*>(src + ch * 8);
  }
  {
    const float* gh = a.relh + (bh * a.Np + q0) * h;
    const float* gw = a.relw + (bh * a.Np + q0) * w;
    for (int i = threadIdx.x; i < AT_BM * h; i += AT_THREADS) {
      relh_s[i] = gh[i];
      drelh_s[i] = 0.f;
    }
    for (int i = threadIdx.x; i < AT_BM * w; i += AT_THREADS) {
      relw_s[i] = gw[i];
      drelw_s[i] = 0.f;
    }
  }
  __syncthreads();
  uint32_t qa[4][4], da[4][4];
  load_afrag(sQ, qa);
  load_afrag(sdO, da);

  const int lane = threadIdx.x & 31, g = lane >> 2, c2 = 2 * (lane & 3);
  const int rl0 = (threadIdx.x >> 5) * 16 + g;
  const float sc = a.scale_log2;
  float lse[2], dlt[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int t = min(q0 + rl0 + 8 * i, N - 1);
    lse[i] = a.lse[bh * N + t];
    dlt[i] = a.delta[bh * N + t];
  }
  float dq[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) dq[i][0] = dq[i][1] = dq[i][2] = dq[i][3] = 0.f;

  for (int k0 = 0; k0 < N; k0 += AT_BM) {
    __syncthreads();
    stage_tile(base, 3 * C, k0, N, C + head * 64, sK, sKt);
    stage_tile(base, 3 * C, k0, N, 2 * C + head * 64, sV, nullptr);
    __syncthreads();
    float s[8][4], dp[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
    mma_rows(s, qa, sK);
    mma_rows(dp, da, sV);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = k0 + nt * 8 + c2 + (e & 1), r = rl0 + 8 * (e >> 1);
        float ds = 0.f;
        if (key < N) {
          const int kr = key / w, kc = key - kr * w;
          const float p = fast_exp2(fmaf(s[nt][e], sc, relh_s[r * h + kr] + relw_s[r * w + kc]) - lse[e >> 1]);
          ds = p * (dp[nt][e] - dlt[e >> 1]);
          atomicAdd(drelh_s + r * h + kr, ds);
          atomicAdd(drelw_s + r * w + kc, ds);
        }
        s[nt][e] = ds;
      }
    mma_p(dq, s, sKt);
  }
  __syncthreads();   // drelh_s / drelw_s complete

  // dQ = scale dS K + gathered table rows, written into the q columns of dqkv
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = rl0 + 8 * i, t = q0 + r;
    const int tc = min(t, N - 1), iq = tc / w, jq = tc - iq * w;
    float acc[16];
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      acc[2 * dt] = dq[dt][2 * i] * 0.125f;
      acc[2 * dt + 1] = dq[dt][2 * i + 1] * 0.125f;
    }
    for (int k = 0; k < h; ++k) {
      const float d = drelh_s[r * h + k];
      const __nv_bfloat16* trow = sT + (iq - k + h - 1) * AT_LDS + c2;
#pragma unroll
      for (int dt = 0; dt < 8; ++dt) {
        const uint32_t u = *reinterpret_cast<const uint32_t*>(trow + dt * 8);
        acc[2 * dt] = fmaf(d, bf16lo(u), acc[2 * dt]);
        acc[2 * dt + 1] = fmaf(d, bf16hi(u), acc[2 * dt + 1]);
      }
    }
    for (int k = 0; k < w; ++k) {
      const float d = drelw_s[r * w + k];
      const __nv_bfloat16* trow = sT + (Lh + jq - k + w - 1) * AT_LDS + c2;
#pragma unroll
      for (int dt = 0; dt < 8; ++dt) {
        const uint32_t u = *reinterpret_cast<const uint32_t*>(trow + dt * 8);
        acc[2 * dt] = fmaf(d, bf16lo(u), acc[2 * dt]);
        acc[2 * dt + 1] = fmaf(d, bf16hi(u), acc[2 * dt + 1]);
      }
    }
    if (t < N) {
      __nv_bfloat16* drow = a.out + (static_cast<size_t>(b) * N + t) * 3 * C + head * 64;
#pragma unroll
      for (int dt = 0; dt < 8; ++dt)
        *reinterpret_cast<uint32_t*>(drow + dt * 8 + c2) = pack_bf16x2(acc[2 * dt], acc[2 * dt + 1]);
    }
  }

  // table-gradient partials of this CTA (every entry of the slice is written)
  const int rows = Lh + Lw;
  float* ws = a.dt_ws + ((bh * gridDim.x) + blockIdx.x) * static_cast<size_t>(rows) * 64;
  const int qn = min(AT_BM, N - q0);
  for (int idx = threadIdx.x; idx < rows * 64; idx += AT_THREADS) {
    const int c = idx / rows, r = idx - c * rows;
    float acc = 0.f;
    for (int q = 0; q < qn; ++q) {
      const int t = q0 + q, iq = t / w, jq = t - iq * w;
      float d;
      if (r < Lh) {
        const int i = iq + h - 1 - r;
        d = (i >= 0 && i < h) ? drelh_s[q * h + i] : 0.f;
      } else {
        const int j = jq + w - 1 - (r - Lh);
        d = (j >= 0 && j < w) ? drelw_s[q * w + j] : 0.f;
      }
      acc = fmaf(d, __bfloat162float(sQ[q * AT_LDS + c]), acc);
    }
    ws[idx] = acc;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// backward, dK / dV side.  grid (key tiles, heads, B); each warp owns 16 keys, the loop runs over the query tiles
//   P^T = exp2(scale K Q^T + bias - lse),  dV += P^T dO,  dS^T = P^T * (V dO^T - delta),  dK += scale dS^T Q
// smem: sK | sV | sQ | sQt | sdO | sdOt | relh_s [64][h] | relw_s [64][w] | lse_s [64] | dlt_s [64]
__global__ void __launch_bounds__(AT_THREADS)
attn_bwd_dkv_kernel(const AttnArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(smem_raw);
  __nv_bfloat16* sV = sK + AT_TILE;
  __nv_bfloat16* sQ = sV + AT_TILE;
  __nv_bfloat16* sQt = sQ + AT_TILE;
  __nv_bfloat16* sdO = sQt + AT_TILE;
  __nv_bfloat16* sdOt = sdO + AT_TILE;
  const int h = a.h, w = a.w, N = a.N, C = a.heads * 64;
  float* relh_s = reinterpret_cast<float*>(sdOt + AT_TILE);
  float* relw_s = relh_s + AT_BM * h;
  float* lse_s = relw_s + AT_BM * w;
  float* dlt_s = lse_s + AT_BM;
  const int k0 = blockIdx.x * AT_BM, head = blockIdx.y, b = blockIdx.z;
  const size_t bh = static_cast<size_t>(b) * a.heads + head;
  const __nv_bfloat16* base = a.qkv + static_cast<size_t>(b) * N * 3 * C;
  const __nv_bfloat16* dObase = a.dO + static_cast<size_t>(b) * N * C;
  pdl_launch_dependents();
  pdl_wait();

  stage_tile(base, 3 * C, k0, N, C + head * 64, sK, nullptr);
  stage_tile(base, 3 * C, k0, N, 2 * C + head * 64, sV, nullptr);
  __syncthreads();
  uint32_t ka[4][4], va[4][4];
  load_afrag(sK, ka);
  load_afrag(sV, va);

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
  const float sc = a.scale_log2;
  float dk[8][4], dv[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i) dk[i][0] = dk[i][1] = dk[i][2] = dk[i][3] = dv[i][0] = dv[i][1] = dv[i][2] = dv[i][3] = 0.f;

  for (int q0 = 0; q0 < N; q0 += AT_BM) {
    __syncthreads();
    stage_tile(base, 3 * C, q0, N, head * 64, sQ, sQt);
    stage_tile(dObase, C, q0, N, head * 64, sdO, sdOt);
    {
      const int qn = min(AT_BM, N - q0);
      const float* gh = a.relh + (bh * a.Np + q0) * h;
      const float* gw = a.relw + (bh * a.Np + q0) * w;
      for (int i = threadIdx.x; i < qn * h; i += AT_THREADS) relh_s[i] = gh[i];
      for (int i = threadIdx.x; i < qn * w; i += AT_THREADS) relw_s[i] = gw[i];
      for (int i = threadIdx.x; i < AT_BM; i += AT_THREADS) {
        const bool v = i < qn;
        lse_s[i] = v ? a.lse[bh * N + q0 + i] : INFINITY;   // queries past N: p = exp2(-inf) = 0
        dlt_s[i] = v ? a.delta[bh * N + q0 + i] : 0.f;
      }
    }
    __syncthreads();
    float s[8][4], dp[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = dp[i][0] = dp[i][1] = dp[i][2] = dp[i][3] = 0.f;
    mma_rows(s, ka, sQ);
    mma_rows(dp, va, sdO);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int q = nt * 8 + c2 + (e & 1), i = e >> 1;
        float p = 0.f;
        if (kvalid[i] && lse_s[q] != INFINITY)
          p = fast_exp2(fmaf(s[nt][e], sc, relh_s[q * h + kr[i]] + relw_s[q * w + kc[i]]) - lse_s[q]);
        s[nt][e] = p;
        dp[nt][e] = p * (dp[nt][e] - dlt_s[q]);
      }
    mma_p(dv, s, sdOt);
    mma_p(dk, dp, sQt);
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int key = k0 + kl0 + 8 * i;
    if (key >= N) continue;
    __nv_bfloat16* row = a.out + (static_cast<size_t>(b) * N + key) * 3 * C + head * 64;
#pragma unroll
    for (int dt = 0; dt < 8; ++dt) {
      *reinterpret_cast<uint32_t*>(row + C + dt * 8 + c2) =
          pack_bf16x2(dk[dt][2 * i] * 0.125f, dk[dt][2 * i + 1] * 0.125f);
      *reinterpret_cast<uint32_t*>(row + 2 * C + dt * 8 + c2) = pack_bf16x2(dv[dt][2 * i], dv[dt][2 * i + 1]);
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

static size_t table_bytes(int h, int w) { return static_cast<size_t>(2 * h - 1 + 2 * w - 1) * AT_LDS * 2; }

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

static int launch_attn(void (*kernel)(AttnArgs), dim3 grid, size_t smem, cudaStream_t st, const AttnArgs& a,
                       const char* who) {
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
  const size_t smem = 3 * AT_TILE * 2 + table_bytes(h, w) + static_cast<size_t>(AT_BM) * (h + w) * 4;
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

// qkv / dqkv: bf16 [B*N, 3C];  O, dO: bf16 [B*N, C];  lse: fp32 [B*heads, N] from pk_attn_fwd
// scratch buffers (caller-allocated): delta [B*heads*N], relh_g [B*heads*Np*h], relw_g [B*heads*Np*w] fp32 with
// Np = N rounded up to a multiple of 128 (query-major rows of bias values)
// dt_ws: pk_attn_bwd_ws_floats(B, heads, h, w) fp32 (per-CTA partial table gradients)
// dTh [2h-1, 64], dTw [2w-1, 64]: fp32, ADDED to (caller zero-initialises or passes a running gradient)
extern "C" long long pk_attn_bwd_ws_floats(int B, int heads, int h, int w) {
  const long long ctas = static_cast<long long>((h * w + AT_BM - 1) / AT_BM) * heads * B;
  return ctas * (2 * h - 1 + 2 * w - 1) * 64;
}

static int attn_bwd_impl(const void* qkv, const void* O, const void* dO, const float* lse, const void* th,
                         const void* tw, void* dqkv, float* dTh, float* dTw, float* delta, float* relh_g,
                         float* relw_g, float* dt_ws, int B, int heads, int h, int w, int th_pad, int tw_pad,
                         int rel_ready, void* stream) {
  if (attn_check(qkv, th, tw, B, heads, h, w, th_pad, tw_pad, "pk_attn_bwd")) return 1;
  PK_CHECK(O && dO && lse && dqkv && dTh && dTw && delta && relh_g && relw_g && dt_ws, "pk_attn_bwd: null pointer");
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
    if (launch_attn(attn_bias_rows_kernel, grid, AT_TILE * 2 + table_bytes(h, w) + rel_bytes, st, a,
                    "pk_attn_bwd(bias rows)"))
      return 2;
  }
  {
    const size_t threads = static_cast<size_t>(B) * N * heads * 8;
    launch_pdl(attn_delta_kernel, dim3(static_cast<unsigned>((threads + 255) / 256)), dim3(256), 0, st,
               static_cast<const __nv_bfloat16*>(O), static_cast<const __nv_bfloat16*>(dO), delta, B, N, heads);
    PK_LAUNCH_CHECK("pk_attn_bwd(delta)");
  }
  if (launch_attn(attn_bwd_dq_kernel, grid, 5 * AT_TILE * 2 + table_bytes(h, w) + 2 * rel_bytes, st, a,
                  "pk_attn_bwd(dq)"))
    return 2;
  if (launch_attn(attn_bwd_dkv_kernel, grid, 6 * AT_TILE * 2 + rel_bytes + 2 * AT_BM * 4, st, a, "pk_attn_bwd(dkv)"))
    return 2;
  {
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
