// painter_b200 — bandwidth-bound kernels of the hot path (LayerNorm, token assembly, layout/cast
// helpers, reductions).  All are warp-shuffle / 128-bit vectorised HBM streamers; none needs tensor cores.
#include "common.cuh"
#include "host_common.h"
#include "../../include/painter_b200.h"

namespace pk {

// =============================================================================================
// LayerNorm over the channel dim (nn.LayerNorm(eps=1e-6), models_painter.py:193,200,315)
// one warp per row; row kept in registers (C <= 1024, C % 128 == 0); two-pass variance.
// =============================================================================================
constexpr int LN_MAX_V4 = 8;   // C <= 1024

template <typename OutT>
__global__ void __launch_bounds__(256)
ln_fwd_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ gamma,
              const float* __restrict__ beta, float eps, OutT* __restrict__ out, int ldo,
              float* __restrict__ mean_out, float* __restrict__ rstd_out, int M, int C) {
  pdl_launch_dependents();   // programmatic dependent launch (host_common.h)
  pdl_wait();
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const int nv = C / 128;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * ldx);
  float4 v[LN_MAX_V4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_V4; ++i)
    if (i < nv) {
      v[i] = xr[i * 32 + lane];
      s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  const float mean = warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < LN_MAX_V4; ++i)
    if (i < nv) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  const float rstd = rsqrtf(warp_sum(q) / C + eps);
  if (lane == 0) {
    if (mean_out) mean_out[row] = mean;
    if (rstd_out) rstd_out[row] = rstd;
  }
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  OutT* orow = out + static_cast<size_t>(row) * ldo;
#pragma unroll
  for (int i = 0; i < LN_MAX_V4; ++i)
    if (i < nv) {
      const float4 g = __ldg(g4 + i * 32 + lane), b = __ldg(b4 + i * 32 + lane);
      const float y0 = (v[i].x - mean) * rstd * g.x + b.x;
      const float y1 = (v[i].y - mean) * rstd * g.y + b.y;
      const float y2 = (v[i].z - mean) * rstd * g.z + b.z;
      const float y3 = (v[i].w - mean) * rstd * g.w + b.w;
      if constexpr (sizeof(OutT) == 2) {
        uint2 u;
        u.x = pack_bf16x2(y0, y1);
        u.y = pack_bf16x2(y2, y3);
        reinterpret_cast<uint2*>(orow)[i * 32 + lane] = u;
      } else {
        reinterpret_cast<float4*>(orow)[i * 32 + lane] = make_float4(y0, y1, y2, y3);
      }
    }
}

// dx = rstd * (g*dy - mean(g*dy) - xhat * mean(g*dy*xhat)) (+ dres);  dgamma += dy*xhat; dbeta += dy
// One block (C/4 threads, thread = one float4 column) walks groups of LNB_ROWS rows: the 2*LNB_ROWS row sums are
// reduced warp-wise, exchanged through a double-buffered smem slab (one __syncthreads per group), and the
// dgamma/dbeta partials stay in 8 registers per thread - no spills, >= 3 blocks per SM, LNB_ROWS*2 float4 loads
// in flight per thread.  HBM-bound: 4 fp32 streams (dy, x, dres in; dx out).
// FUSE: the caller also needs bf16(rowscale[row / rows_per_group] * dx) (the next GEMM's operand after DropPath) and
// its column sums (that GEMM's bias gradient): emitted here instead of re-reading dx in a second kernel; the
// column sums ride in a third partials block.
constexpr int LNB_ROWS = 4;
// DYB: dy arrives as bf16 (the dgrad GEMM in front writes bf16 - the rounding point of the reference's autocast Linear
// backward - which halves both that GEMM's store traffic and this kernel's dy stream).
template <bool FUSE, bool DYB>
__global__ void __launch_bounds__(256, FUSE ? 2 : 3)
ln_bwd_kernel(const void* __restrict__ dy_, int lddy, const float* __restrict__ x, int ldx,
              const float* __restrict__ mean, const float* __restrict__ rstd,
              const float* __restrict__ gamma, const float* __restrict__ dres, float* __restrict__ dx,
              float* __restrict__ partials /* [gridDim.x][2C or 3C] */, int M, int C,
              const float* __restrict__ rowscale, int rows_per_group, __nv_bfloat16* __restrict__ dx_bf16) {
  __shared__ float4 xch[2][8][2 * LNB_ROWS / 4];  // [buffer][warp][s1[0..R) | s2[0..R)]
  pdl_launch_dependents();   // programmatic dependent launch (host_common.h)
  pdl_wait();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nw = blockDim.x >> 5;
  const float4 gam = reinterpret_cast<const float4*>(gamma)[tid];
  float4 ag = make_float4(0.f, 0.f, 0.f, 0.f), ab = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 acs = make_float4(0.f, 0.f, 0.f, 0.f);
  const float invC = 1.0f / C;
  int it = 0;
  for (int r0 = blockIdx.x * LNB_ROWS; r0 < M; r0 += gridDim.x * LNB_ROWS, ++it) {
    float4 xh[LNB_ROWS], gd[LNB_ROWS], rv[LNB_ROWS];
    float rs[LNB_ROWS], s[2 * LNB_ROWS];
#pragma unroll
    for (int u = 0; u < LNB_ROWS; ++u) {
      const int row = min(r0 + u, M - 1);
      xh[u] = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * ldx)[tid];
      if constexpr (DYB) {
        const uint2 q = reinterpret_cast<const uint2*>(static_cast<const __nv_bfloat16*>(dy_) +
                                                       static_cast<size_t>(row) * lddy)[tid];
        gd[u] = make_float4(__uint_as_float(q.x << 16), __uint_as_float(q.x & 0xFFFF0000u),
                            __uint_as_float(q.y << 16), __uint_as_float(q.y & 0xFFFF0000u));
      } else {
        gd[u] = reinterpret_cast<const float4*>(static_cast<const float*>(dy_) + static_cast<size_t>(row) * lddy)[tid];
      }
      if (dres) rv[u] = reinterpret_cast<const float4*>(dres + static_cast<size_t>(row) * C)[tid];
    }
#pragma unroll
    for (int u = 0; u < LNB_ROWS; ++u) {
      const int row = min(r0 + u, M - 1);
      const float mu = mean[row];
      rs[u] = rstd[row];
      const float4 dv = gd[u];
      xh[u] = make_float4((xh[u].x - mu) * rs[u], (xh[u].y - mu) * rs[u], (xh[u].z - mu) * rs[u],
                          (xh[u].w - mu) * rs[u]);
      gd[u] = make_float4(dv.x * gam.x, dv.y * gam.y, dv.z * gam.z, dv.w * gam.w);
      s[u] = (gd[u].x + gd[u].y) + (gd[u].z + gd[u].w);
      s[LNB_ROWS + u] = (gd[u].x * xh[u].x + gd[u].y * xh[u].y) + (gd[u].z * xh[u].z + gd[u].w * xh[u].w);
      if (r0 + u < M) {
        ag.x += dv.x * xh[u].x; ag.y += dv.y * xh[u].y; ag.z += dv.z * xh[u].z; ag.w += dv.w * xh[u].w;
        ab.x += dv.x; ab.y += dv.y; ab.z += dv.z; ab.w += dv.w;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int k = 0; k < 2 * LNB_ROWS; ++k) s[k] += __shfl_xor_sync(0xffffffffu, s[k], o);
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < 2 * LNB_ROWS / 4; ++k)
        xch[it & 1][warp][k] = make_float4(s[4 * k], s[4 * k + 1], s[4 * k + 2], s[4 * k + 3]);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 2 * LNB_ROWS; ++k) s[k] = 0.f;
    for (int w = 0; w < nw; ++w) {
#pragma unroll
      for (int k = 0; k < 2 * LNB_ROWS / 4; ++k) {
        const float4 t = xch[it & 1][w][k];
        s[4 * k] += t.x; s[4 * k + 1] += t.y; s[4 * k + 2] += t.z; s[4 * k + 3] += t.w;
      }
    }
#pragma unroll
    for (int u = 0; u < LNB_ROWS; ++u) {
      if (r0 + u >= M) break;
      const float c1 = s[u] * invC, c2 = s[LNB_ROWS + u] * invC;
      float4 o = make_float4(rs[u] * (gd[u].x - c1 - xh[u].x * c2), rs[u] * (gd[u].y - c1 - xh[u].y * c2),
                             rs[u] * (gd[u].z - c1 - xh[u].z * c2), rs[u] * (gd[u].w - c1 - xh[u].w * c2));
      if (dres) {
        o.x += rv[u].x; o.y += rv[u].y; o.z += rv[u].z; o.w += rv[u].w;
      }
      reinterpret_cast<float4*>(dx + static_cast<size_t>(r0 + u) * C)[tid] = o;
      if constexpr (FUSE) {
        const float sc = rowscale ? rowscale[(r0 + u) / rows_per_group] : 1.f;
        o.x *= sc; o.y *= sc; o.z *= sc; o.w *= sc;
        acs.x += o.x; acs.y += o.y; acs.z += o.z; acs.w += o.w;
        uint2 pk2;
        pk2.x = pack_bf16x2(o.x, o.y);
        pk2.y = pack_bf16x2(o.z, o.w);
        reinterpret_cast<uint2*>(dx_bf16 + static_cast<size_t>(r0 + u) * C)[tid] = pk2;
      }
    }
  }
  // per-block partials, one row of the workspace per block (no atomics: a second small kernel sums the rows); no
  // workspace when none of the column sums is wanted
  if (partials == nullptr) return;
  constexpr int NP = FUSE ? 3 : 2;
  float4* pg = reinterpret_cast<float4*>(partials + static_cast<size_t>(blockIdx.x) * NP * C);
  pg[tid] = ag;
  pg[C / 4 + tid] = ab;
  if constexpr (FUSE) pg[2 * (C / 4) + tid] = acs;
}

// dgamma[c] += sum_b partials[b][c];  dbeta[c] += sum_b partials[b][C + c].   block (32, 8): 32 columns, the
// rows strided over threadIdx.y, 4 loads in flight per thread.  A block whose target is NULL (a gradient that is not
// needed) does nothing: C % 128 == 0 keeps each block's 32 columns inside one target.
__global__ void __launch_bounds__(256)
ln_bwd_reduce_kernel(const float* __restrict__ partials, int nblocks, float* __restrict__ dgamma,
                     float* __restrict__ dbeta, float* __restrict__ colsum, int C, int np) {
  __shared__ float red[8][33];
  pdl_launch_dependents();   // programmatic dependent launch (host_common.h)
  pdl_wait();
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int seg = blockIdx.x * 32 / C;
  if ((seg == 0 ? dgamma : seg == 1 ? dbeta : colsum) == nullptr) return;
  const size_t ld = static_cast<size_t>(np) * C;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  int b = threadIdx.y;
  for (; b + 24 < nblocks; b += 32) {
    s0 += partials[static_cast<size_t>(b) * ld + c];
    s1 += partials[static_cast<size_t>(b + 8) * ld + c];
    s2 += partials[static_cast<size_t>(b + 16) * ld + c];
    s3 += partials[static_cast<size_t>(b + 24) * ld + c];
  }
  for (; b < nblocks; b += 8) s0 += partials[static_cast<size_t>(b) * ld + c];
  red[threadIdx.y][threadIdx.x] = (s0 + s1) + (s2 + s3);
  __syncthreads();
  if (threadIdx.y == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    if (c < C) dgamma[c] += s;
    else if (c < 2 * C) dbeta[c - C] += s;
    else colsum[c - 2 * C] += s;
  }
}

// =============================================================================================
// PatchEmbed lowering: stride-16 conv == GEMM over (c, r, s)-ordered patch rows
// (vitdet_utils.py:178-186, models_painter.py:387-388).  Both images (imgs | tgts) in one launch.
// out[(img*N + i*w + j), (c*p + r)*p + s] = bf16(src[img][c][i*p + r][j*p + s])
// =============================================================================================
__global__ void __launch_bounds__(256)
im2col_patch_kernel(const float* __restrict__ imgs, const float* __restrict__ tgts,
                    __nv_bfloat16* __restrict__ out, int B, int Cin, int H, int W, int p) {
  const int h = H / p, w = W / p, N = h * w;
  const int kdim = Cin * p * p;
  const int chunks = kdim / 8;
  const size_t total = static_cast<size_t>(2 * B) * N * chunks;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int ch = static_cast<int>(idx % chunks);
    const size_t row = idx / chunks;
    const int img = static_cast<int>(row / N), t = static_cast<int>(row % N);
    const int i = t / w, j = t % w;
    const int k0 = ch * 8;
    const int c = k0 / (p * p), rem = k0 % (p * p), r = rem / p, s0 = rem % p;
    const float* src = (img < B ? imgs + static_cast<size_t>(img) * Cin * H * W
                                : tgts + static_cast<size_t>(img - B) * Cin * H * W) +
                       (static_cast<size_t>(c) * H + i * p + r) * W + j * p + s0;
    const float4 a = *reinterpret_cast<const float4*>(src);
    const float4 b = *reinterpret_cast<const float4*>(src + 4);
    uint4 u;
    u.x = pack_bf16x2(a.x, a.y); u.y = pack_bf16x2(a.z, a.w);
    u.z = pack_bf16x2(b.x, b.y); u.w = pack_bf16x2(b.z, b.w);
    *reinterpret_cast<uint4*>(out + row * kdim + k0) = u;
  }
}

// Input gradient of the PatchEmbed lowering: the exact inverse of im2col_patch_kernel's layout (the patches do not
// overlap, so every image element is one entry of the column matrix).  dcols_x / dcols_y fp32 [B*h*w, Cin*p*p] (the
// x rows and the y rows) -> dimgs / dtgts fp32 NCHW; a NULL half is neither read nor written (img0 / nimg select the
// images).  thread = 4 consecutive pixels of one image row (p % 8 == 0 keeps them inside one patch).
__global__ void __launch_bounds__(256)
col2im_patch_kernel(const float* __restrict__ dcols_x, const float* __restrict__ dcols_y, float* __restrict__ dimgs,
                    float* __restrict__ dtgts, int B, int Cin, int H, int W, int p, int img0, int nimg) {
  const int h = H / p, w = W / p, N = h * w;
  const int kdim = Cin * p * p, w4 = W / 4;
  const size_t per_img = static_cast<size_t>(Cin) * H * w4;
  const size_t total = static_cast<size_t>(nimg) * per_img;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int img = img0 + static_cast<int>(idx / per_img);
    const size_t e = idx % per_img;
    const int x = static_cast<int>(e % w4) * 4;
    const size_t cy = e / w4;
    const int y = static_cast<int>(cy % H), c = static_cast<int>(cy / H);
    const int i = y / p, r = y % p, j = x / p, s = x % p;
    const int b = img < B ? img : img - B;
    const float4 v = *reinterpret_cast<const float4*>((img < B ? dcols_x : dcols_y) +
                                                      (static_cast<size_t>(b) * N + i * w + j) * kdim +
                                                      (c * p + r) * p + s);
    float* dst = (img < B ? dimgs : dtgts) + static_cast<size_t>(b) * Cin * H * W;
    *reinterpret_cast<float4*>(dst + cy * W + x) = v;
  }
}

// =============================================================================================
// Token assembly (models_painter.py:392-409; SegGPT type tokens models_seggpt.py:414-420)
//   x rows: E + seg_x + P (+ type);   y rows: (E*(1-m) + mask_token*m) + seg_y + P (+ type)
// =============================================================================================
__global__ void __launch_bounds__(256)
assemble_kernel(const float* __restrict__ E, const uint8_t* __restrict__ mask, int maskB,
                const float* __restrict__ mask_token, const float* __restrict__ seg_x,
                const float* __restrict__ seg_y, const float* __restrict__ pos,
                const float* __restrict__ type_emb, float* __restrict__ out, int B, int N, int C) {
  const int c4n = C / 4;
  const size_t total = static_cast<size_t>(2 * B) * N * c4n;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c4 = static_cast<int>(idx % c4n);
    const size_t row = idx / c4n;
    const int img = static_cast<int>(row / N), n = static_cast<int>(row % N);
    const bool isY = img >= B;
    const int b = isY ? img - B : img;
    float4 e = reinterpret_cast<const float4*>(E)[idx];
    if (isY) {
      const float m = mask[static_cast<size_t>(b % maskB) * N + n] ? 1.f : 0.f;
      const float4 mt = __ldg(reinterpret_cast<const float4*>(mask_token) + c4);
      e.x = e.x * (1.f - m) + mt.x * m; e.y = e.y * (1.f - m) + mt.y * m;
      e.z = e.z * (1.f - m) + mt.z * m; e.w = e.w * (1.f - m) + mt.w * m;
    }
    const float4 sg = __ldg(reinterpret_cast<const float4*>(isY ? seg_y : seg_x) + c4);
    const float4 ps = __ldg(reinterpret_cast<const float4*>(pos) + static_cast<size_t>(n) * c4n + c4);
    e.x = (e.x + sg.x) + ps.x; e.y = (e.y + sg.y) + ps.y;
    e.z = (e.z + sg.z) + ps.z; e.w = (e.w + sg.w) + ps.w;
    if (type_emb) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(type_emb) + static_cast<size_t>(b) * c4n + c4);
      e.x += t.x; e.y += t.y; e.z += t.z; e.w += t.w;
    }
    reinterpret_cast<float4*>(out)[idx] = e;
  }
}

// backward of the assembly: dE (bf16, y rows gated by 1-m), dpos[N,C], dseg_x, dseg_y, dmask_token and the SegGPT
// type tokens (models_seggpt.py:415-420: sample b's x and y rows feed type_token_cls when seg_type[b] == 0,
// type_token_ins when it is 1, neither otherwise; seg_type is compared as fp32, like the forward's mask arithmetic)
// block = (C/4, TY) threads, one token per threadIdx.y
__global__ void assemble_bwd_kernel(const float* __restrict__ dZ, const uint8_t* __restrict__ mask,
                                    int maskB, __nv_bfloat16* __restrict__ dE, float* __restrict__ dpos,
                                    float* __restrict__ dseg_x, float* __restrict__ dseg_y,
                                    float* __restrict__ dmask_token, const float* __restrict__ seg_type,
                                    float* __restrict__ dtype_cls, float* __restrict__ dtype_ins, int B, int N,
                                    int C) {
  extern __shared__ float4 sred[];  // [3 or 5][TY][C/4]
  const int c4n = C / 4;
  const int c4 = threadIdx.x;
  const int n = blockIdx.x * blockDim.y + threadIdx.y;
  const bool tok = dseg_x != nullptr, typ = dtype_cls != nullptr;
  float4 sx = make_float4(0, 0, 0, 0), sy = sx, sm = sx, tc = sx, ti = sx;
  if (n < N) {
    for (int img = 0; img < 2 * B; ++img) {
      const size_t off = (static_cast<size_t>(img) * N + n) * c4n + c4;
      float4 d = reinterpret_cast<const float4*>(dZ)[off];
      if (typ) {
        const float st = __ldg(seg_type + (img < B ? img : img - B));
        if (st == 0.f) {
          tc.x += d.x; tc.y += d.y; tc.z += d.z; tc.w += d.w;
        } else if (st == 1.f) {
          ti.x += d.x; ti.y += d.y; ti.z += d.z; ti.w += d.w;
        }
      }
      if (img < B) {
        sx.x += d.x; sx.y += d.y; sx.z += d.z; sx.w += d.w;
      } else {
        sy.x += d.x; sy.y += d.y; sy.z += d.z; sy.w += d.w;
        if (mask[static_cast<size_t>((img - B) % maskB) * N + n]) {
          sm.x += d.x; sm.y += d.y; sm.z += d.z; sm.w += d.w;
          d = make_float4(0, 0, 0, 0);
        }
      }
      uint2 u;
      u.x = pack_bf16x2(d.x, d.y);
      u.y = pack_bf16x2(d.z, d.w);
      reinterpret_cast<uint2*>(dE)[off] = u;
    }
    if (dpos)
      reinterpret_cast<float4*>(dpos)[static_cast<size_t>(n) * c4n + c4] =
          make_float4(sx.x + sy.x, sx.y + sy.y, sx.z + sy.z, sx.w + sy.w);
  }
  if (!tok && !typ) return;   // frozen tokens: no reduction
  // slots 0..2: dseg_x, dseg_y, dmask_token (all three or none); slots 3..4: dtype_cls, dtype_ins (both or none)
  const int TY = blockDim.y;
  const size_t slot = static_cast<size_t>(TY) * c4n;
  float4* mine = sred + threadIdx.y * c4n + c4;
  if (tok) {
    mine[0] = sx;
    mine[slot] = sy;
    mine[2 * slot] = sm;
  }
  if (typ) {
    mine[3 * slot] = tc;
    mine[4 * slot] = ti;
  }
  __syncthreads();
  for (int which = tok ? threadIdx.y : threadIdx.y + 3; which < (typ ? 5 : 3); which += TY) {
    float4 s = make_float4(0, 0, 0, 0);
    for (int t = 0; t < TY; ++t) {
      const float4 v = sred[which * slot + t * c4n + c4];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    float* dst = (which == 0 ? dseg_x : which == 1 ? dseg_y : which == 2 ? dmask_token :
                  which == 3 ? dtype_cls : dtype_ins) + c4 * 4;
    atomicAdd(dst + 0, s.x); atomicAdd(dst + 1, s.y); atomicAdd(dst + 2, s.z); atomicAdd(dst + 3, s.w);
  }
}

// =============================================================================================
// Bicubic resize of the absolute position table (get_abs_pos, vitdet_utils.py:141-157):
// F.interpolate(mode="bicubic", align_corners=False), A = -0.75, border-clamped taps.  NHWC [s,s,C]->[h,w,C]
// =============================================================================================
__device__ __forceinline__ void cubic_coeffs(float t, float (&w)[4]) {
  const float A = -0.75f;
  const float x0 = t + 1.f, x1 = t, x2 = 1.f - t, x3 = 2.f - t;
  w[0] = ((A * x0 - 5.f * A) * x0 + 8.f * A) * x0 - 4.f * A;
  w[1] = ((A + 2.f) * x1 - (A + 3.f)) * x1 * x1 + 1.f;
  w[2] = ((A + 2.f) * x2 - (A + 3.f)) * x2 * x2 + 1.f;
  w[3] = ((A * x3 - 5.f * A) * x3 + 8.f * A) * x3 - 4.f * A;
}
template <bool BWD>
__global__ void bicubic_kernel(const float* __restrict__ src, float* __restrict__ dst, int sh, int sw,
                               int h, int w, int C) {
  // FWD: src [sh,sw,C] -> dst [h,w,C].   BWD: src = d(dst) [h,w,C], dst = d(src) [sh,sw,C] (atomic)
  const size_t total = static_cast<size_t>(h) * w * C;
  const float scale_h = static_cast<float>(sh) / h, scale_w = static_cast<float>(sw) / w;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % C);
    const int j = static_cast<int>((idx / C) % w), i = static_cast<int>(idx / (static_cast<size_t>(C) * w));
    const float ry = scale_h * (i + 0.5f) - 0.5f, rx = scale_w * (j + 0.5f) - 0.5f;
    const float fy = floorf(ry), fx = floorf(rx);
    float wy[4], wx[4];
    cubic_coeffs(ry - fy, wy);
    cubic_coeffs(rx - fx, wx);
    const int iy = static_cast<int>(fy), ix = static_cast<int>(fx);
    float acc = 0.f;
    const float g = BWD ? src[idx] : 0.f;
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      const int yy = min(max(iy - 1 + a, 0), sh - 1);
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int xx = min(max(ix - 1 + b, 0), sw - 1);
        const size_t so = (static_cast<size_t>(yy) * sw + xx) * C + c;
        if (BWD) atomicAdd(dst + so, g * wy[a] * wx[b]);
        else acc += src[so] * wy[a] * wx[b];
      }
    }
    if (!BWD) dst[idx] = acc;
  }
}

// =============================================================================================
// Early merge (models_painter.py:414-415): out = 0.5 * (z[:half] + z[half:]);  bwd: both halves = 0.5 * d
// =============================================================================================
__global__ void merge_halves_kernel(const float4* __restrict__ z, float4* __restrict__ out, size_t half4) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < half4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 a = z[i], b = z[i + half4];
    out[i] = make_float4((a.x + b.x) * 0.5f, (a.y + b.y) * 0.5f, (a.z + b.z) * 0.5f, (a.w + b.w) * 0.5f);
  }
}
__global__ void merge_halves_bwd_kernel(const float4* __restrict__ d, float4* __restrict__ out, size_t half4) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < half4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 a = d[i];
    const float4 o = make_float4(a.x * 0.5f, a.y * 0.5f, a.z * 0.5f, a.w * 0.5f);
    out[i] = o;
    out[i + half4] = o;
  }
}

// =============================================================================================
// fp32 -> bf16 cast (weights each step; gradients entering a GEMM), optional per-row-group scale
// (DropPath backward) and optional fused column sum (bias gradient).
// =============================================================================================
__global__ void __launch_bounds__(256)
cast_bf16_kernel(const float4* __restrict__ in, uint2* __restrict__ out, size_t n4) {
  pdl_launch_dependents();   // programmatic dependent launch (host_common.h)
  pdl_wait();
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const float4 v = in[i];
    uint2 u;
    u.x = pack_bf16x2(v.x, v.y);
    u.y = pack_bf16x2(v.z, v.w);
    out[i] = u;
  }
}

// in f32 [M, C] (ld = ldin) -> out bf16 [M, C] scaled by rowscale[row / rows_per_group];
// colsum[c] += sum_rows(scaled value).  block (C/4 <= 256 threads x), rows strided by gridDim.
__global__ void scale_cast_colsum_kernel(const float* __restrict__ in, int ldin,
                                         const float* __restrict__ rowscale, int rows_per_group,
                                         __nv_bfloat16* __restrict__ out, float* __restrict__ colsum,
                                         int M, int C) {
  pdl_launch_dependents();   // programmatic dependent launch (host_common.h)
  pdl_wait();
  const int c4n = C / 4;
  for (int c4 = threadIdx.x; c4 < c4n; c4 += blockDim.x) {
    float4 acc = make_float4(0, 0, 0, 0);
    for (int row0 = blockIdx.x * 4; row0 < M; row0 += gridDim.x * 4) {
      float4 v[4];
      float sc[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {  // four independent rows in flight per thread
        const int row = row0 + r;
        if (row < M) {
          v[r] = reinterpret_cast<const float4*>(in + static_cast<size_t>(row) * ldin)[c4];
          sc[r] = rowscale ? rowscale[row / rows_per_group] : 1.f;
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int row = row0 + r;
        if (row < M) {
          float4 t = v[r];
          t.x *= sc[r]; t.y *= sc[r]; t.z *= sc[r]; t.w *= sc[r];
          acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
          uint2 u;
          u.x = pack_bf16x2(t.x, t.y);
          u.y = pack_bf16x2(t.z, t.w);
          reinterpret_cast<uint2*>(out + static_cast<size_t>(row) * C)[c4] = u;
        }
      }
    }
    if (colsum) {
      atomicAdd(colsum + c4 * 4 + 0, acc.x); atomicAdd(colsum + c4 * 4 + 1, acc.y);
      atomicAdd(colsum + c4 * 4 + 2, acc.z); atomicAdd(colsum + c4 * 4 + 3, acc.w);
    }
  }
}

// colsum[c] += sum_m in[m, c]   (bf16 in, ld = ldin);  grid (ceil(C/256), row chunks)
__global__ void __launch_bounds__(256)
colsum_bf16_kernel(const __nv_bfloat16* __restrict__ in, int ldin, float* __restrict__ colsum, int M,
                   int C, int rows_per_block) {
  __shared__ float red[8][256];
  pdl_launch_dependents();   // programmatic dependent launch (host_common.h)
  pdl_wait();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.x * 256 + lane * 8;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(M, r0 + rows_per_block);
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (c0 < C) {
    for (int row = r0 + warp; row < r1; row += 8) {
      const uint4 u = *reinterpret_cast<const uint4*>(in + static_cast<size_t>(row) * ldin + c0);
      const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        acc[2 * t] += __uint_as_float(w[t] << 16);
        acc[2 * t + 1] += __uint_as_float(w[t] & 0xFFFF0000u);
      }
    }
  }
#pragma unroll
  for (int t = 0; t < 8; ++t) red[warp][lane * 8 + t] = acc[t];
  __syncthreads();
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < C) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][threadIdx.x];
    atomicAdd(colsum + c, s);
  }
}

// =============================================================================================
// SegGPT feature ensemble + residual (models_seggpt.py:220-231 then :233):
//   out = z + (top-half rows: a ; bottom-half rows: mean of a over the members of the prompt group)
// a, z, out: [G*P, N, C] with G groups (2 before the early merge, 1 after)
// =============================================================================================
__global__ void ensemble_resid_kernel(const float4* __restrict__ a, const float4* __restrict__ z,
                                      float4* __restrict__ out, int G, int P, int N, int C4) {
  const size_t per_img = static_cast<size_t>(N) * C4;
  const size_t total = static_cast<size_t>(G) * per_img;
  const float inv = 1.0f / P;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int g = static_cast<int>(idx / per_img);
    const size_t r = idx % per_img;
    const int n = static_cast<int>(r / C4);
    const size_t base = static_cast<size_t>(g) * P * per_img + r;
    if (n < N / 2) {
      for (int p = 0; p < P; ++p) {
        const float4 av = a[base + p * per_img], zv = z[base + p * per_img];
        out[base + p * per_img] = make_float4(zv.x + av.x, zv.y + av.y, zv.z + av.z, zv.w + av.w);
      }
    } else {
      float4 s = make_float4(0, 0, 0, 0);
      for (int p = 0; p < P; ++p) {
        const float4 av = a[base + p * per_img];
        s.x += av.x; s.y += av.y; s.z += av.z; s.w += av.w;
      }
      s.x *= inv; s.y *= inv; s.z *= inv; s.w *= inv;
      for (int p = 0; p < P; ++p) {
        const float4 zv = z[base + p * per_img];
        out[base + p * per_img] = make_float4(zv.x + s.x, zv.y + s.y, zv.z + s.z, zv.w + s.w);
      }
    }
  }
}

static inline int grid_for(size_t work_items, int block) {
  size_t g = (work_items + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count()) * 16;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace pk

using namespace pk;

extern "C" int pk_layernorm_fwd(const float* x, int ldx, const float* gamma, const float* beta, float eps,
                                void* out, int ldo, int out_is_bf16, float* mean, float* rstd, int M,
                                int C, void* stream) {
  PK_CHECK(x && gamma && beta && out, "pk_layernorm_fwd: null pointer");
  PK_CHECK(C % 128 == 0 && C <= 128 * LN_MAX_V4, "pk_layernorm_fwd: C=%d must be a multiple of 128, <= %d", C,
           128 * LN_MAX_V4);
  PK_CHECK(ldx % 4 == 0 && ldo % 4 == 0, "pk_layernorm_fwd: strides must be multiples of 4");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int grid = (M + 7) / 8;
  if (out_is_bf16)
    launch_pdl(ln_fwd_kernel<__nv_bfloat16>, dim3(grid), dim3(256), 0, st, x, ldx, gamma, beta, eps,
               static_cast<__nv_bfloat16*>(out), ldo, mean, rstd, M, C);
  else
    launch_pdl(ln_fwd_kernel<float>, dim3(grid), dim3(256), 0, st, x, ldx, gamma, beta, eps, static_cast<float*>(out),
               ldo, mean, rstd, M, C);
  PK_LAUNCH_CHECK("pk_layernorm_fwd");
  return 0;
}

static int ln_bwd_grid(int M) {
  int grid = sm_count() * 3;
  if (grid > (M + LNB_ROWS - 1) / LNB_ROWS) grid = (M + LNB_ROWS - 1) / LNB_ROWS;
  return grid;
}
// fp32 workspace elements pk_layernorm_bwd needs (per-block partial sums of dgamma / dbeta)
extern "C" long long pk_layernorm_bwd_ws_floats(int M, int C) {
  return static_cast<long long>(ln_bwd_grid(M)) * 3 * C;
}

extern "C" int pk_layernorm_bwd(const void* dy, int dy_is_bf16, int lddy, const float* x, int ldx, const float* mean,
                                const float* rstd, const float* gamma, const float* dres, float* dx,
                                float* dgamma, float* dbeta, float* workspace, int M, int C, void* stream) {
  PK_CHECK(dy && x && mean && rstd && gamma && dx, "pk_layernorm_bwd: null pointer");
  // dgamma = dbeta = NULL: no affine gradients (frozen LayerNorm); no workspace is touched and dx is unchanged
  const bool affine = dgamma || dbeta;
  PK_CHECK(!affine || workspace, "pk_layernorm_bwd: null pointer (workspace)");
  PK_CHECK(C % 128 == 0 && C <= 1024 && lddy % 4 == 0 && ldx % 4 == 0, "pk_layernorm_bwd: bad C=%d", C);
  const int grid = ln_bwd_grid(M);
  if (!affine) workspace = nullptr;
  if (dy_is_bf16)
    launch_pdl(ln_bwd_kernel<false, true>, dim3(grid), dim3(C / 4), 0, static_cast<cudaStream_t>(stream), dy, lddy, x,
               ldx, mean, rstd, gamma, dres, dx, workspace, M, C, static_cast<const float*>(nullptr), 0,
               static_cast<__nv_bfloat16*>(nullptr));
  else
    launch_pdl(ln_bwd_kernel<false, false>, dim3(grid), dim3(C / 4), 0, static_cast<cudaStream_t>(stream), dy, lddy, x,
               ldx, mean, rstd, gamma, dres, dx, workspace, M, C, static_cast<const float*>(nullptr), 0,
               static_cast<__nv_bfloat16*>(nullptr));
  PK_LAUNCH_CHECK("pk_layernorm_bwd");
  if (affine) {
    launch_pdl(ln_bwd_reduce_kernel, dim3(2 * C / 32), dim3(32, 8), 0, static_cast<cudaStream_t>(stream),
               static_cast<const float*>(workspace), grid, dgamma, dbeta, static_cast<float*>(nullptr), C, 2);
    PK_LAUNCH_CHECK("pk_layernorm_bwd(reduce)");
  }
  return 0;
}

// pk_layernorm_bwd + pk_scale_cast_colsum of its result in one pass: additionally writes
// dx_bf16 = bf16(rowscale[row / rows_per_group] * dx) and adds its column sums to colsum[C].
extern "C" int pk_layernorm_bwd_cast(const void* dy, int dy_is_bf16, int lddy, const float* x, int ldx, const float* mean,
                                     const float* rstd, const float* gamma, const float* dres, float* dx,
                                     float* dgamma, float* dbeta, float* workspace, const float* rowscale,
                                     int rows_per_group, void* dx_bf16, float* colsum, int M, int C, void* stream) {
  PK_CHECK(dy && x && mean && rstd && gamma && dx && dx_bf16, "pk_layernorm_bwd_cast: null pointer");
  // dgamma / dbeta / colsum = NULL: that column sum is not needed; with all three NULL no workspace is touched.  dx and
  // dx_bf16 are unchanged either way.
  const bool sums = dgamma || dbeta || colsum;
  PK_CHECK(!sums || workspace, "pk_layernorm_bwd_cast: null pointer (workspace)");
  if (!sums) workspace = nullptr;
  PK_CHECK(C % 128 == 0 && C <= 1024 && lddy % 4 == 0 && ldx % 4 == 0, "pk_layernorm_bwd_cast: bad C=%d", C);
  if (rowscale) PK_CHECK(rows_per_group > 0, "pk_layernorm_bwd_cast: rows_per_group must be > 0");
  int grid = sm_count() * 2;   // the fused variant keeps 2 blocks per SM resident (<= ln_bwd_grid(M): workspace fits)
  if (grid > (M + LNB_ROWS - 1) / LNB_ROWS) grid = (M + LNB_ROWS - 1) / LNB_ROWS;
  if (dy_is_bf16)
    launch_pdl(ln_bwd_kernel<true, true>, dim3(grid), dim3(C / 4), 0, static_cast<cudaStream_t>(stream), dy, lddy, x,
               ldx, mean, rstd, gamma, dres, dx, workspace, M, C, rowscale, rows_per_group,
               static_cast<__nv_bfloat16*>(dx_bf16));
  else
    launch_pdl(ln_bwd_kernel<true, false>, dim3(grid), dim3(C / 4), 0, static_cast<cudaStream_t>(stream), dy, lddy, x,
               ldx, mean, rstd, gamma, dres, dx, workspace, M, C, rowscale, rows_per_group,
               static_cast<__nv_bfloat16*>(dx_bf16));
  PK_LAUNCH_CHECK("pk_layernorm_bwd_cast");
  if (sums) {
    launch_pdl(ln_bwd_reduce_kernel, dim3(3 * C / 32), dim3(32, 8), 0, static_cast<cudaStream_t>(stream),
               static_cast<const float*>(workspace), grid, dgamma, dbeta, colsum, C, 3);
    PK_LAUNCH_CHECK("pk_layernorm_bwd_cast(reduce)");
  }
  return 0;
}

extern "C" int pk_im2col_patch(const float* imgs, const float* tgts, void* out_bf16, int B, int Cin, int H,
                               int W, int p, void* stream) {
  PK_CHECK(imgs && tgts && out_bf16, "pk_im2col_patch: null pointer");
  PK_CHECK(p % 8 == 0 && H % p == 0 && W % p == 0 && W % 4 == 0, "pk_im2col_patch: bad geometry");
  const size_t total = static_cast<size_t>(2 * B) * (H / p) * (W / p) * (Cin * p * p / 8);
  im2col_patch_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      imgs, tgts, static_cast<__nv_bfloat16*>(out_bf16), B, Cin, H, W, p);
  PK_LAUNCH_CHECK("pk_im2col_patch");
  return 0;
}

extern "C" int pk_col2im_patch(const float* dcols_x, const float* dcols_y, float* dimgs, float* dtgts, int B, int Cin,
                               int H, int W, int p, void* stream) {
  PK_CHECK((dcols_x || !dimgs) && (dcols_y || !dtgts), "pk_col2im_patch: null pointer");
  PK_CHECK(p % 8 == 0 && H % p == 0 && W % p == 0 && W % 4 == 0, "pk_col2im_patch: bad geometry");
  const int img0 = dimgs ? 0 : B, nimg = (dimgs ? B : 0) + (dtgts ? B : 0);
  if (nimg == 0) return 0;
  const size_t total = static_cast<size_t>(nimg) * Cin * H * (W / 4);
  col2im_patch_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      dcols_x, dcols_y, dimgs, dtgts, B, Cin, H, W, p, img0, nimg);
  PK_LAUNCH_CHECK("pk_col2im_patch");
  return 0;
}

extern "C" int pk_assemble_tokens(const float* E, const uint8_t* mask, int maskB, const float* mask_token,
                                  const float* seg_x, const float* seg_y, const float* pos,
                                  const float* type_emb, float* out, int B, int N, int C, void* stream) {
  PK_CHECK(E && mask && mask_token && seg_x && seg_y && pos && out, "pk_assemble_tokens: null pointer");
  PK_CHECK(C % 4 == 0 && maskB >= 1, "pk_assemble_tokens: bad shape");
  const size_t total = static_cast<size_t>(2 * B) * N * (C / 4);
  assemble_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      E, mask, maskB, mask_token, seg_x, seg_y, pos, type_emb, out, B, N, C);
  PK_LAUNCH_CHECK("pk_assemble_tokens");
  return 0;
}

extern "C" int pk_assemble_tokens_bwd_typed(const float* dZ, const uint8_t* mask, int maskB, void* dE_bf16,
                                            float* dpos, float* dseg_x, float* dseg_y, float* dmask_token,
                                            const float* seg_type, float* dtype_cls, float* dtype_ins, int B, int N,
                                            int C, void* stream) {
  // dpos = NULL: the position gradient is not needed; dseg_x = dseg_y = dmask_token = NULL: the token gradients are
  // not needed (all three or none); dtype_cls = dtype_ins = NULL: no type-token gradients (both or none, and then
  // seg_type is not read).  dE is unchanged either way.
  PK_CHECK(dZ && mask && dE_bf16, "pk_assemble_tokens_bwd: null pointer");
  PK_CHECK((dseg_x != nullptr) == (dseg_y != nullptr) && (dseg_x != nullptr) == (dmask_token != nullptr),
           "pk_assemble_tokens_bwd: dseg_x, dseg_y and dmask_token must all be given or all be NULL");
  PK_CHECK((dtype_cls != nullptr) == (dtype_ins != nullptr) && (dtype_cls == nullptr || seg_type != nullptr),
           "pk_assemble_tokens_bwd: dtype_cls and dtype_ins must both be given (with seg_type) or both be NULL");
  PK_CHECK(C % 4 == 0 && C / 4 <= 256, "pk_assemble_tokens_bwd: C=%d unsupported", C);
  const int tx = C / 4;
  int ty = 1024 / tx;
  if (ty > 8) ty = 8;
  if (ty < 3) ty = 3;
  PK_CHECK(tx * ty <= 1024, "pk_assemble_tokens_bwd: C too large");
  const int slots = dtype_cls ? 5 : 3;
  const size_t smem = static_cast<size_t>(slots) * ty * tx * sizeof(float4);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(assemble_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 5 * 1024 * 16);
    attr = true;
  }
  assemble_bwd_kernel<<<(N + ty - 1) / ty, dim3(tx, ty), smem, static_cast<cudaStream_t>(stream)>>>(
      dZ, mask, maskB, static_cast<__nv_bfloat16*>(dE_bf16), dpos, dseg_x, dseg_y, dmask_token, seg_type, dtype_cls,
      dtype_ins, B, N, C);
  PK_LAUNCH_CHECK("pk_assemble_tokens_bwd");
  return 0;
}

extern "C" int pk_assemble_tokens_bwd(const float* dZ, const uint8_t* mask, int maskB, void* dE_bf16,
                                      float* dpos, float* dseg_x, float* dseg_y, float* dmask_token, int B,
                                      int N, int C, void* stream) {
  return pk_assemble_tokens_bwd_typed(dZ, mask, maskB, dE_bf16, dpos, dseg_x, dseg_y, dmask_token, nullptr, nullptr,
                                      nullptr, B, N, C, stream);
}

extern "C" int pk_bicubic_fwd(const float* src, float* dst, int sh, int sw, int h, int w, int C, void* stream) {
  PK_CHECK(src && dst, "pk_bicubic_fwd: null pointer");
  bicubic_kernel<false><<<grid_for(static_cast<size_t>(h) * w * C, 256), 256, 0,
                          static_cast<cudaStream_t>(stream)>>>(src, dst, sh, sw, h, w, C);
  PK_LAUNCH_CHECK("pk_bicubic_fwd");
  return 0;
}
extern "C" int pk_bicubic_bwd(const float* ddst, float* dsrc_accum, int sh, int sw, int h, int w, int C,
                              void* stream) {
  PK_CHECK(ddst && dsrc_accum, "pk_bicubic_bwd: null pointer");
  bicubic_kernel<true><<<grid_for(static_cast<size_t>(h) * w * C, 256), 256, 0,
                         static_cast<cudaStream_t>(stream)>>>(ddst, dsrc_accum, sh, sw, h, w, C);
  PK_LAUNCH_CHECK("pk_bicubic_bwd");
  return 0;
}

extern "C" int pk_merge_halves(const float* z, float* out, long long half_elems, void* stream) {
  PK_CHECK(z && out && half_elems % 4 == 0, "pk_merge_halves: bad args");
  merge_halves_kernel<<<grid_for(half_elems / 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(z), reinterpret_cast<float4*>(out), half_elems / 4);
  PK_LAUNCH_CHECK("pk_merge_halves");
  return 0;
}
extern "C" int pk_merge_halves_bwd(const float* d, float* out, long long half_elems, void* stream) {
  PK_CHECK(d && out && half_elems % 4 == 0, "pk_merge_halves_bwd: bad args");
  merge_halves_bwd_kernel<<<grid_for(half_elems / 4, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(d), reinterpret_cast<float4*>(out), half_elems / 4);
  PK_LAUNCH_CHECK("pk_merge_halves_bwd");
  return 0;
}

extern "C" int pk_cast_bf16(const float* in, void* out_bf16, long long n, void* stream) {
  PK_CHECK(in && out_bf16 && n % 4 == 0, "pk_cast_bf16: bad args (n must be a multiple of 4)");
  launch_pdl(cast_bf16_kernel, dim3(grid_for(n / 4, 256)), dim3(256), 0, static_cast<cudaStream_t>(stream),
             reinterpret_cast<const float4*>(in), reinterpret_cast<uint2*>(out_bf16), static_cast<size_t>(n / 4));
  PK_LAUNCH_CHECK("pk_cast_bf16");
  return 0;
}

extern "C" int pk_scale_cast_colsum(const float* in, int ldin, const float* rowscale, int rows_per_group,
                                    void* out_bf16, float* colsum, int M, int C, void* stream) {
  PK_CHECK(in && out_bf16 && C % 4 == 0 && ldin % 4 == 0, "pk_scale_cast_colsum: bad args");
  if (rowscale) PK_CHECK(rows_per_group > 0, "pk_scale_cast_colsum: rows_per_group must be > 0");
  int tx = C / 4;
  if (tx > 256) tx = 256;
  int grid = sm_count() * 4;
  if (grid > (M + 3) / 4) grid = (M + 3) / 4;
  launch_pdl(scale_cast_colsum_kernel, dim3(grid), dim3(tx), 0, static_cast<cudaStream_t>(stream), in, ldin, rowscale,
             rows_per_group, static_cast<__nv_bfloat16*>(out_bf16), colsum, M, C);
  PK_LAUNCH_CHECK("pk_scale_cast_colsum");
  return 0;
}

extern "C" int pk_colsum_bf16(const void* in_bf16, int ldin, float* colsum, int M, int C, void* stream) {
  PK_CHECK(in_bf16 && colsum && C % 8 == 0 && ldin % 8 == 0, "pk_colsum_bf16: bad args");
  const int rpb = 256;
  dim3 grid((C + 255) / 256, (M + rpb - 1) / rpb);
  launch_pdl(colsum_bf16_kernel, grid, dim3(256), 0, static_cast<cudaStream_t>(stream),
             static_cast<const __nv_bfloat16*>(in_bf16), ldin, colsum, M, C, rpb);
  PK_LAUNCH_CHECK("pk_colsum_bf16");
  return 0;
}

extern "C" int pk_ensemble_resid(const float* a, const float* z, float* out, int G, int P, int N, int C,
                                 void* stream) {
  PK_CHECK(a && z && out && C % 4 == 0 && N % 2 == 0, "pk_ensemble_resid: bad args");
  const size_t total = static_cast<size_t>(G) * N * (C / 4);
  ensemble_resid_kernel<<<grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(a), reinterpret_cast<const float4*>(z), reinterpret_cast<float4*>(out),
      G, P, N, C / 4);
  PK_LAUNCH_CHECK("pk_ensemble_resid");
  return 0;
}

// =============================================================================================
// Window attention plumbing (vitdet_utils.py:16-60): zero-padded partition of a [B,H,W,C] token grid into
// [B*nWh*nWw, ws, ws, C] windows and its inverse.  Only reachable through Painter(window_block_indexes=[...]);
// the stock factories build no windowed block (SURVEY.md section 0.1).
// =============================================================================================
namespace pk {

// bf16 partition: 16-byte chunks (8 channels)
__global__ void window_partition_bf16_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int B, int H,
                                             int W, int C8, int ws, int nWh, int nWw) {
  const size_t total = static_cast<size_t>(B) * nWh * nWw * ws * ws * C8;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % C8);
    size_t r = idx / C8;
    const int wx = static_cast<int>(r % ws); r /= ws;
    const int wy = static_cast<int>(r % ws); r /= ws;
    const int ww = static_cast<int>(r % nWw); r /= nWw;
    const int wh = static_cast<int>(r % nWh);
    const int b = static_cast<int>(r / nWh);
    const int y = wh * ws + wy, x = ww * ws + wx;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (y < H && x < W) v = in[((static_cast<size_t>(b) * H + y) * W + x) * C8 + c];
    out[idx] = v;
  }
}

// out[b,y,x,:] = (resid ? resid[b,y,x,:] : 0) + scale_b * win[window(b,y,x), :]   (fp32, float4 chunks)
__global__ void window_unpartition_kernel(const float4* __restrict__ win, const float4* __restrict__ resid,
                                          const float* __restrict__ rowscale, float4* __restrict__ out, int B,
                                          int H, int W, int C4, int ws, int nWh, int nWw) {
  const size_t total = static_cast<size_t>(B) * H * W * C4;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(idx % C4);
    size_t r = idx / C4;
    const int x = static_cast<int>(r % W); r /= W;
    const int y = static_cast<int>(r % H);
    const int b = static_cast<int>(r / H);
    const size_t widx =
        ((((static_cast<size_t>(b) * nWh + y / ws) * nWw + x / ws) * ws + y % ws) * ws + x % ws) * C4 + c;
    const float sc = rowscale ? rowscale[b] : 1.f;
    float4 v = win[widx];
    v.x *= sc; v.y *= sc; v.z *= sc; v.w *= sc;
    if (resid) {
      const float4 rr = resid[idx];
      v.x += rr.x; v.y += rr.y; v.z += rr.z; v.w += rr.w;
    }
    out[idx] = v;
  }
}
}  // namespace pk

extern "C" int pk_window_partition_bf16(const void* in, void* out, int B, int H, int W, int C, int ws,
                                        void* stream) {
  PK_CHECK(in && out && C % 8 == 0 && ws > 0, "pk_window_partition_bf16: bad args");
  const int nWh = (H + ws - 1) / ws, nWw = (W + ws - 1) / ws;
  const size_t total = static_cast<size_t>(B) * nWh * nWw * ws * ws * (C / 8);
  pk::window_partition_bf16_kernel<<<pk::grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(in), static_cast<uint4*>(out), B, H, W, C / 8, ws, nWh, nWw);
  PK_LAUNCH_CHECK("pk_window_partition_bf16");
  return 0;
}

extern "C" int pk_window_unpartition(const float* win, const float* resid, const float* rowscale, float* out,
                                     int B, int H, int W, int C, int ws, void* stream) {
  PK_CHECK(win && out && C % 4 == 0 && ws > 0, "pk_window_unpartition: bad args");
  const int nWh = (H + ws - 1) / ws, nWw = (W + ws - 1) / ws;
  const size_t total = static_cast<size_t>(B) * H * W * (C / 4);
  pk::window_unpartition_kernel<<<pk::grid_for(total, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const float4*>(win), reinterpret_cast<const float4*>(resid), rowscale,
      reinterpret_cast<float4*>(out), B, H, W, C / 4, ws, nWh, nWw);
  PK_LAUNCH_CHECK("pk_window_unpartition");
  return 0;
}
