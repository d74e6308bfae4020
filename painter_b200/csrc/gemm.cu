// painter_b200 — persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   C[M,N] = A[M,K] . B[N,K]^T      bf16 operands, fp32 accumulation in registers
//
// One CTA per SM, 384 threads, 128 x BN output tiles (BN = 64 / 128 / 256), K-blocks of 64:
//   warpgroup 0     TMA producer   (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier tx);
//                                  gives its registers up (setmaxnreg) to the math warpgroups
//   warpgroups 1-2  math           (wgmma.mma_async 64 x BN x 16 from shared memory, 64 accumulator rows each;
//                                  one wgmma group stays in flight while the previous ring slot is released),
//                                  then the fused epilogue: bf16 / GELU outputs in registers -> swizzled smem
//                                  sub-tiles -> asynchronous TMA stores (gemm_tma_epilogue_tile); the other kinds
//                                  accumulators -> smem staging tile (64 x 64 per warpgroup) -> coalesced epilogue
//                                  chunks of 32 x 32 per warp
// The producer runs up to `stages` K-blocks ahead, so the next tile's operands stream in during an epilogue.
// Operands may be K-major (row-major [rows,K]) or MN-major (row-major [K,rows]); the latter is what the backward
// GEMMs (dgrad: B = W[out,in]; wgrad: A = dY[tokens,out], B = X[tokens,in]) need, so no transposed copies of weights
// or activations are ever materialised.  Weight-gradient GEMMs (zero-initialised fp32 output) run stream-K.
//
// Reference call sites replaced: every nn.Linear on the path (models_painter.py:60-61,76,87; timm Mlp
// fc1/fc2 via :201; decoder_embed :327,423) and autograd's mm backward for them.
#include "gemm_common.cuh"
#include "wgmma.cuh"

namespace pk {

// One 64-deep K-block of one math warpgroup: acc[64 x BN] (+)= A[64 x 64] . B[64 x BN]^T (4 wgmma, K = 16 each),
// committed as one wgmma group.  The fence and the commit sit inside the operand-layout branch, next to the wgmmas:
// with a branch between them ptxas cannot prove the accumulators untouched and injects warpgroup.arrive (C7519).
template <int BN, int TA, int TB>
__device__ __forceinline__ void gemm_kblock(float (&acc)[BN / 2], uint32_t a_addr, uint32_t b_addr, bool first) {
  const uint64_t da = TA ? make_wgmma_desc(a_addr, 8192, 1024) : make_wgmma_desc(a_addr, 16, 1024);
  const uint64_t db = TB ? make_wgmma_desc(b_addr, 8192, 1024) : make_wgmma_desc(b_addr, 16, 1024);
  constexpr uint32_t a_step = TA ? 2048u : 32u, b_step = TB ? 2048u : 32u;
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < GEMM_BK / 16; ++k) {
    const uint64_t a = wgmma_desc_add(da, k * a_step), b = wgmma_desc_add(db, k * b_step);
    const uint32_t accf = (first && k == 0) ? 0u : 1u;
    if constexpr (BN == 64) wgmma_m64n64k16<TA, TB>(acc, a, b, accf);
    else if constexpr (BN == 128) wgmma_m64n128k16<TA, TB>(acc, a, b, accf);
    else wgmma_m64n256k16<TA, TB>(acc, a, b, accf);
  }
  wgmma_commit();
}

// Epilogue of the TMA-store kinds (bf16, GELU) for the 64 accumulator rows of one math warpgroup: alpha and bias on
// the fragments in registers, each 64-column sub-tile written in the output's 128B-swizzled layout into one of the
// warpgroup's two staging slots and stored by one thread with cp.async.bulk.tensor.  The warpgroup does not wait for
// the stores: a slot is only waited on (wait_group.read) when it is about to be rewritten, two sub-tiles later.
// Every element goes through the same expressions as the staged epilogue (gemm_epilogue_chunk), so the results are
// bit-identical to it.
template <int KIND, int BN>
__device__ __forceinline__ void gemm_tma_epilogue_tile(const GemmArgs& g, const CUtensorMap* tmC,
                                                       const CUtensorMap* tmC2, const float (&acc)[BN / 2],
                                                       uint32_t stg_wg, uint32_t& slot, int m_blk, int n_blk, int cw,
                                                       int wl, int lane) {
  constexpr uint32_t SLOT = gemm_slot_bytes(KIND);
  const bool issuer = (threadIdx.x & 127) == 0;
  const int r0 = 16 * wl + (lane >> 2);   // fragment rows r0 and r0 + 8; both have (row % 8) = lane / 4
  const uint32_t sw = static_cast<uint32_t>(lane >> 2);
  const uint32_t off0 = r0 * 128u + 4u * (lane & 3), off1 = off0 + 8u * 128u;
  const float sc = g.epi.alpha;
  const float bsc = 1.0f;
  const float* bias = g.epi.bias;
#pragma unroll
  for (int j = 0; j < BN / 64; ++j) {
    if (issuer) tma_store_wait_read<1>();   // the store that last read this slot (two sub-tiles ago) is done
    named_bar_sync(1 + cw, 128);
    const uint32_t buf = stg_wg + slot * SLOT;
    const int col0 = n_blk * BN + 64 * j;
#pragma unroll
    for (int n8 = 0; n8 < 8; ++n8) {
      const int i = 4 * (8 * j + n8);   // acc[i], acc[i + 1]: row r0; acc[i + 2], acc[i + 3]: row r0 + 8
      float v[4];
      if (bias != nullptr) {
        const float2 b = __ldg(reinterpret_cast<const float2*>(bias + col0 + 8 * n8 + 2 * (lane & 3)));
        v[0] = fmaf(acc[i], sc, b.x * bsc);
        v[1] = fmaf(acc[i + 1], sc, b.y * bsc);
        v[2] = fmaf(acc[i + 2], sc, b.x * bsc);
        v[3] = fmaf(acc[i + 3], sc, b.y * bsc);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = acc[i + q] * sc;
      }
      const uint32_t chunk = ((static_cast<uint32_t>(n8) ^ sw) << 4);
      const uint32_t z0 = pack_bf16x2(v[0], v[1]), z1 = pack_bf16x2(v[2], v[3]);
      st_shared_u32(buf + off0 + chunk, z0);
      st_shared_u32(buf + off1 + chunk, z1);
      if constexpr (KIND == PK_EPI_GELU) {
        float h[4];
        gelu_fast_pair(__uint_as_float(z0 << 16), __uint_as_float(z0 & 0xFFFF0000u), h[0], h[1]);
        gelu_fast_pair(__uint_as_float(z1 << 16), __uint_as_float(z1 & 0xFFFF0000u), h[2], h[3]);
        st_shared_u32(buf + GEMM_SUB_BYTES + off0 + chunk, pack_bf16x2(h[0], h[1]));
        st_shared_u32(buf + GEMM_SUB_BYTES + off1 + chunk, pack_bf16x2(h[2], h[3]));
      }
    }
    fence_proxy_async_smem();   // the generic-proxy writes above become visible to the bulk copy
    named_bar_sync(1 + cw, 128);
    if (issuer) {
      const int row0 = m_blk * GEMM_BM + 64 * cw;   // rows past M are clipped by the tensor map
      tma_store_2d(tmC, buf, col0, row0);
      if constexpr (KIND == PK_EPI_GELU) tma_store_2d(tmC2, buf + GEMM_SUB_BYTES, col0, row0);
      tma_store_commit();
    }
    slot ^= 1u;
  }
}

template <int KIND, int BN>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmC2,
                 const GemmArgs g) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_base = smem_u32(smem_raw);
  const uint32_t base = (raw_base + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (base - raw_base);

  constexpr bool TMA_EPI = gemm_tma_epilogue(KIND);
  constexpr uint32_t B_BYTES = static_cast<uint32_t>(BN) * 128u;
  const int stages = g.stages;
  const uint32_t sA = base;
  const uint32_t sB = base + stages * GEMM_A_BYTES;
  const uint32_t sStg = sB + stages * B_BYTES;   // 1024-aligned (swizzled TMA boxes)
  const uint32_t bar_base = sStg + gemm_stg_bytes(KIND);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (stages + s); };

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;
  const int num_kb = (g.K + GEMM_BK - 1) / GEMM_BK;
  const int tiles_mn = g.num_m_tiles * g.num_n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if constexpr (TMA_EPI) tma_prefetch_desc(&tmC);
    if constexpr (KIND == PK_EPI_GELU) tma_prefetch_desc(&tmC2);
    for (int s = 0; s < stages; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), 256);   // every math thread releases the slot after its wgmma retired
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_launch_dependents();   // programmatic dependent launch (host_common.h): the prologue above overlaps the
  pdl_wait();                // previous kernel's tail; nothing before this line touches global memory

  GemmSched sch;
  sch.init(g, tiles_mn, num_kb, blockIdx.x, gridDim.x);
  int mn, kb0, kb1;

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      // ------------------------------ TMA producer ------------------------------
      uint32_t s = 0, ph = 0;
      while (sch.next(mn, kb0, kb1)) {
        int m_blk, n_blk;
        gemm_tile_coords(g, mn, m_blk, n_blk);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty_bar(s), ph ^ 1u);
          mbar_expect_tx(full_bar(s), GEMM_A_BYTES + B_BYTES);
          const uint32_t a_dst = sA + s * GEMM_A_BYTES;
          const uint32_t b_dst = sB + s * B_BYTES;
          if (g.conv.mode == 1) {
            const int tx = m_blk % g.conv.tiles_x, r1 = m_blk / g.conv.tiles_x;
            const int ty = r1 % g.conv.tiles_y, bi = r1 / g.conv.tiles_y;
            const int dy = kb / 3, dx = kb - dy * 3;
            tma_load_4d(a_dst, &tmA, full_bar(s), 0, tx * g.conv.TW + dx - 1, ty * g.conv.TH + dy - 1, bi);
            tma_load_2d(b_dst, &tmB, full_bar(s), kb * GEMM_BK, n_blk * BN);
          } else if (g.conv.mode == 2) {
            const int tx = kb % g.conv.tiles_x, r1 = kb / g.conv.tiles_x;
            const int ty = r1 % g.conv.tiles_y, bi = r1 / g.conv.tiles_y;
#pragma unroll
            for (int gi = 0; gi < 2; ++gi) {
              const int tap = m_blk * 2 + gi;
              const int dy = tap / 3, dx = tap - dy * 3;
              // tap 9 does not exist: a far out-of-bounds box yields the zero rows of the last m-block
              const int yy = tap < 9 ? ty * g.conv.TH + dy - 1 : -(1 << 20);
              tma_load_4d(a_dst + gi * 8192, &tmA, full_bar(s), 0, tx * g.conv.TW + dx - 1, yy, bi);
            }
            tma_load_4d(b_dst, &tmB, full_bar(s), 0, tx * g.conv.TW, ty * g.conv.TH, bi);
          } else {
            if (!g.transA) {
              tma_load_2d(a_dst, &tmA, full_bar(s), kb * GEMM_BK, m_blk * GEMM_BM);
            } else {
              tma_load_2d(a_dst, &tmA, full_bar(s), m_blk * GEMM_BM, kb * GEMM_BK);
              tma_load_2d(a_dst + 8192, &tmA, full_bar(s), m_blk * GEMM_BM + 64, kb * GEMM_BK);
            }
            if (!g.transB) {
              tma_load_2d(b_dst, &tmB, full_bar(s), kb * GEMM_BK, n_blk * BN);
            } else {
              for (int gi = 0; gi < BN / 64; ++gi)
                tma_load_2d(b_dst + gi * 8192, &tmB, full_bar(s), n_blk * BN + gi * 64, kb * GEMM_BK);
            }
          }
          if (++s == static_cast<uint32_t>(stages)) {
            s = 0;
            ph ^= 1u;
          }
        }
      }
    }
    return;
  }

  // ------------------------------------ math warpgroups ------------------------------------
  setmaxnreg_inc<232>();
  const int cw = wg - 1;                // accumulator rows [64 cw, 64 cw + 64) of the tile
  const int wl = warp & 3;              // warp within the warpgroup
  float* stg = reinterpret_cast<float*>(smem_gen + (sStg - base)) + cw * 64 * STG_LD;
  const int frag_r = 16 * wl + (lane >> 2), frag_c = 2 * (lane & 3);
  const uint32_t stg_wg = sStg + cw * 2u * gemm_slot_bytes(KIND);   // TMA-store kinds: this warpgroup's two slots
  uint32_t slot = 0;
  uint32_t s = 0, ph = 0;
  float acc[BN / 2];
  while (sch.next(mn, kb0, kb1)) {
    int m_blk, n_blk;
    gemm_tile_coords(g, mn, m_blk, n_blk);
    int prev = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(full_bar(s), ph);
      const uint32_t a_addr = sA + s * GEMM_A_BYTES + cw * 8192;   // 64 K-major rows / one 64-wide MN group
      const uint32_t b_addr = sB + s * B_BYTES;
      if (g.transA) {
        if (g.transB) gemm_kblock<BN, 1, 1>(acc, a_addr, b_addr, kb == kb0);
        else gemm_kblock<BN, 1, 0>(acc, a_addr, b_addr, kb == kb0);
      } else {
        if (g.transB) gemm_kblock<BN, 0, 1>(acc, a_addr, b_addr, kb == kb0);
        else gemm_kblock<BN, 0, 0>(acc, a_addr, b_addr, kb == kb0);
      }
      wgmma_fence_operands(acc);
      wgmma_wait<1>();
      wgmma_fence_operands(acc);
      if (prev >= 0) mbar_arrive(empty_bar(prev));
      prev = static_cast<int>(s);
      if (++s == static_cast<uint32_t>(stages)) {
        s = 0;
        ph ^= 1u;
      }
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    mbar_arrive(empty_bar(prev));

    // --------------------------------- epilogue ---------------------------------
    if constexpr (TMA_EPI) {
      gemm_tma_epilogue_tile<KIND, BN>(g, &tmC, &tmC2, acc, stg_wg, slot, m_blk, n_blk, cw, wl, lane);
      continue;
    }
#pragma unroll
    for (int c0 = 0; c0 < BN; c0 += 64) {
      named_bar_sync(1 + cw, 128);     // the previous chunk's readers are done with the staging tile
#pragma unroll
      for (int i = 0; i < BN / 2; i += 2) {
        const int cb = 8 * (i / 4);
        if (cb >= c0 && cb < c0 + 64) {
          const int r = frag_r + 8 * ((i / 2) & 1);
          *reinterpret_cast<float2*>(stg + r * STG_LD + cb - c0 + frag_c) = make_float2(acc[i], acc[i + 1]);
        }
      }
      named_bar_sync(1 + cw, 128);
      if constexpr (KIND == EPI_HEAD || KIND == EPI_UNSHUF) {
        // pixel-row tile (BN = 64, one chunk): warps 0-1 of the warpgroup own one accumulator row per thread
        if (wl < 2) {
          const int rloc = cw * 64 + wl * 32 + lane;
          const float* srow = stg + (wl * 32 + lane) * STG_LD;
          const int tx = m_blk % g.conv.tiles_x, r1 = m_blk / g.conv.tiles_x;
          const int ty = r1 % g.conv.tiles_y, bi = r1 / g.conv.tiles_y;
          const int y = ty * g.conv.TH + rloc / g.conv.TW, x = tx * g.conv.TW + rloc % g.conv.TW;
          float c[64];
#pragma unroll
          for (int q = 0; q < 16; ++q) {
            const float4 v4 = reinterpret_cast<const float4*>(srow)[q];
            c[4 * q] = v4.x; c[4 * q + 1] = v4.y; c[4 * q + 2] = v4.z; c[4 * q + 3] = v4.w;
          }
          if constexpr (KIND == EPI_HEAD) {
            head_epilogue_row(g, bi, y, x, c);
          } else {  // EPI_UNSHUF: token row m = (b, y/p, x/p), columns ((y%p)*p + x%p)*64 + c
            const int p = g.epi.ps_p;
            const size_t mtok = (static_cast<size_t>(bi) * (g.conv.H / p) + y / p) * (g.conv.W / p) + x / p;
            __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(g.epi.out) + mtok * g.epi.ldc +
                                 ((y % p) * p + x % p) * 64 + n_blk * BN;
            store_bf16x32(dst, reinterpret_cast<const float(&)[32]>(c[0]));
            store_bf16x32(dst + 32, reinterpret_cast<const float(&)[32]>(c[32]));
          }
        }
      } else {
        const int rb = (wl & 1) * 32, cb = (wl >> 1) * 32;
        float* blk = stg + rb * STG_LD + cb;
        const int row0 = m_blk * GEMM_BM + cw * 64 + rb;
        const int col = n_blk * BN + c0 + cb;
        EpiAux aux;
        gemm_epilogue_prefetch<KIND>(g.epi, row0, g.M, col, aux);
        uint32_t v[32];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 v4 = reinterpret_cast<const float4*>(blk + lane * STG_LD)[q];
          v[4 * q] = __float_as_uint(v4.x); v[4 * q + 1] = __float_as_uint(v4.y);
          v[4 * q + 2] = __float_as_uint(v4.z); v[4 * q + 3] = __float_as_uint(v4.w);
        }
        gemm_epilogue_chunk<KIND>(g.epi, blk, row0, g.M, col, v, aux);
      }
    }
  }
  // the bulk stores read shared memory and must have written their results before the CTA exits: shared memory is
  // released then, and a dependent launch (PDL) only waits for this grid to complete
  if constexpr (TMA_EPI) {
    if ((threadIdx.x & 127) == 0) tma_store_wait_all();
  }
}

int g_force_bn = 0;
int g_force_splits = 0;

static size_t gemm_smem_bytes(const GemmArgs& g) {
  return 1024 + static_cast<size_t>(g.stages) * (GEMM_A_BYTES + g.BN * 128) + gemm_stg_bytes(g.epi.kind) + 256;
}

// persistent CTAs a call runs: one per stream-K range, otherwise one per work item up to the SM count
static int gemm_workers(const GemmArgs& g) {
  const int num_kb = (g.K + GEMM_BK - 1) / GEMM_BK;
  const long long tiles = static_cast<long long>(g.num_m_tiles) * g.num_n_tiles;
  if (g.streamk_units > 0) return static_cast<int>((tiles * num_kb + g.streamk_units - 1) / g.streamk_units);
  const long long items = tiles * g.splits;
  return items < sm_count() ? static_cast<int>(items) : sm_count();
}

// The output tensor maps of the TMA-store epilogues (tmC: out, tmC2: GELU's out2); other kinds pass unused maps.
struct GemmOutMaps {
  CUtensorMap c, c2;
};

template <int KK, int BN>
static cudaError_t launch_gemm_kernel(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmOutMaps& tmo,
                                      const GemmArgs& g, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_bf16_kernel<KK, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         227 * 1024);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  return launch_pdl(gemm_bf16_kernel<KK, BN>, dim3(gemm_workers(g)), dim3(GEMM_THREADS), gemm_smem_bytes(g), st,
                    tmA, tmB, tmo.c, tmo.c2, g);
}

template <int KK>
static cudaError_t launch_gemm_bn(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmOutMaps& tmo,
                                  const GemmArgs& g, cudaStream_t st) {
  if (g.BN == 256) return launch_gemm_kernel<KK, 256>(tmA, tmB, tmo, g, st);
  if (g.BN == 128) return launch_gemm_kernel<KK, 128>(tmA, tmB, tmo, g, st);
  return launch_gemm_kernel<KK, 64>(tmA, tmB, tmo, g, st);
}

static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmOutMaps& tmo, GemmArgs& g,
                       cudaStream_t st, const char* who) {
  PK_CHECK(gemm_smem_bytes(g) <= 227 * 1024 && g.stages >= 2, "%s: BN=%d does not fit shared memory", who, g.BN);
  cudaError_t e = cudaSuccess;
  switch (g.epi.kind) {
    case PK_EPI_BF16: e = launch_gemm_bn<PK_EPI_BF16>(tmA, tmB, tmo, g, st); break;
    case PK_EPI_F32: e = launch_gemm_bn<PK_EPI_F32>(tmA, tmB, tmo, g, st); break;
    case PK_EPI_GELU: e = launch_gemm_bn<PK_EPI_GELU>(tmA, tmB, tmo, g, st); break;
    case PK_EPI_RESID: e = launch_gemm_bn<PK_EPI_RESID>(tmA, tmB, tmo, g, st); break;
    case PK_EPI_DGELU: e = launch_gemm_bn<PK_EPI_DGELU>(tmA, tmB, tmo, g, st); break;
    case PK_EPI_PIXSHUF: e = launch_gemm_bn<PK_EPI_PIXSHUF>(tmA, tmB, tmo, g, st); break;
    case EPI_HEAD: e = launch_gemm_kernel<EPI_HEAD, 64>(tmA, tmB, tmo, g, st); break;
    case EPI_UNSHUF: e = launch_gemm_kernel<EPI_UNSHUF, 64>(tmA, tmB, tmo, g, st); break;
    default:
      PK_CHECK(false, "%s: bad epilogue kind %d", who, g.epi.kind);
  }
  PK_CHECK(e == cudaSuccess, "%s: launch: %s", who, cudaGetErrorString(e));
  PK_LAUNCH_CHECK(who);
  return 0;
}

static bool conv_tile_geometry(int H, int W, int pixels, int* TW, int* TH) {
  int tw = W < 64 ? W : 64;
  if (W % tw != 0 || pixels % tw != 0) return false;
  int th = pixels / tw;
  if (H % th != 0) return false;
  *TW = tw;
  *TH = th;
  return true;
}

}  // namespace pk

// test hooks: force the N tile (64/128/256) / the split-K factor; 0 restores the heuristics
extern "C" void pk_gemm_force_bn(int bn) { pk::g_force_bn = bn; }
extern "C" void pk_gemm_force_splits(int s) { pk::g_force_splits = s; }

// Tiling / scheduling decisions of one pk_gemm_bf16 call (host only; also reachable through pk_gemm_plan for the
// CPU-side schedule tests).
static void plan_gemm(int M, int N, int K, int transA, int transB, const PkEpilogue* epi, pk::GemmArgs& g) {
  using namespace pk;
  memset(&g, 0, sizeof(g));
  g.M = M;
  g.N = N;
  g.K = K;
  g.transA = transA ? 1 : 0;
  g.transB = transB ? 1 : 0;
  g.epi = *epi;
  if (g.epi.alpha == 0.0f) g.epi.alpha = 1.0f;
  const int sms = sm_count();
  const int mt = (M + GEMM_BM - 1) / GEMM_BM;
  const bool zero_init_f32 = epi->kind == PK_EPI_F32 && epi->accumulate == 2;
  // 128 x 128 tiles where the shape allows, 128 x 256 for the bf16 and GELU epilogues when that still gives every
  // SM a tile: 8-13 % faster than BN = 128 at the ViT-L block shapes on H100 (qkv / fc1 forward, fc1 / qkv dgrad).
  // At BN = 256 the math warpgroups hold 128 accumulator registers per thread; the kernels with the fp32, residual
  // and GELU' epilogues spill 8-16 bytes there (ptxas -v), so those keep BN = 128.
  int BN = 64;
  if (zero_init_f32) {
    // weight-gradient GEMMs (K = tokens): take the wide tile and fill the machine with stream-K instead of
    // shrinking the tile
    if (N % 128 == 0) BN = 128;
  } else if ((epi->kind == PK_EPI_BF16 || epi->kind == PK_EPI_GELU) && N % 256 == 0 &&
             static_cast<long long>(mt) * (N / 256) >= sms) {
    BN = 256;
  } else if (N % 128 == 0 && static_cast<long long>(mt) * (N / 128) >= sms / 2) {
    BN = 128;
  }
  if (g_force_bn > 0 && N % g_force_bn == 0) BN = g_force_bn;
  g.BN = BN;
  g.stages = gemm_stages_for(GEMM_A_BYTES + BN * 128, epi->kind);
  g.num_m_tiles = mt;
  g.num_n_tiles = N / BN;
  const int num_kb = (K + GEMM_BK - 1) / GEMM_BK;
  g.splits = 1;
  g.kb_per_split = num_kb;
  if (zero_init_f32) {
    // zero-initialised fp32 output (weight gradients): stream-K.  The tiles_mn * num_kb k-block units are cut into
    // consecutive ranges of streamk_units, one per CTA; a tile that straddles ranges is finished with fp32 atomics.
    const int tiles = g.num_m_tiles * g.num_n_tiles;
    const long long units = static_cast<long long>(tiles) * num_kb;
    if (g_force_splits > 0) {
      const int want = g_force_splits < num_kb ? g_force_splits : num_kb;
      g.kb_per_split = (num_kb + want - 1) / want;
      g.splits = (num_kb + g.kb_per_split - 1) / g.kb_per_split;
      if (g.splits == 1) g.epi.accumulate = 1;
    } else if (tiles % sms == 0 || units < 4ll * sms) {
      g.epi.accumulate = 1;   // already balanced (or too small to matter): plain data-parallel tiles
    } else {
      // Range length: a whole number of K-phases (num_kb / q, q <= 8) where that costs at most ~10 % over the equal
      // cut.  Every range then starts at one of q K-offsets, so the CTAs running together read the same few K-slices
      // of both operands and share them in L2; with the equal cut the starting K-blocks of the 132 ranges are spread
      // over all of K and nearly every operand block comes from HBM once per CTA that reads it (fc1 weight gradient
      // at B = 8: 2 whole tiles per CTA on 128 CTAs instead of 381 of 196 K-blocks each).
      const int equal = static_cast<int>((units + sms - 1) / sms);
      int per = equal;
      for (int q = 1; q <= 8; q *= 2) {
        if (num_kb % q != 0) continue;
        const int seg = num_kb / q;
        const int k = static_cast<int>((units + static_cast<long long>(sms) * seg - 1) / (static_cast<long long>(sms) * seg));
        if (static_cast<long long>(k) * seg * 10 <= static_cast<long long>(equal) * 11) {
          per = k * seg;
          break;
        }
      }
      if (per < 4) per = 4;
      g.streamk_units = per;
    }
  }
  // rasterisation: keep B L2-resident when it fits, otherwise sweep the columns inside groups of 8 row blocks
  // (stream-K calls keep the row-fastest order)
  g.group_m = (static_cast<long long>(N) * K * 2 <= (40ll << 20)) ? 1 : (g.streamk_units > 0 ? 0 : 8);
}

// Host-side views of the scheduler (no device work): the plan of a call, and the (row block, column block, k-block
// range) items one CTA walks - the same GemmSched / gemm_tile_coords code the kernel runs.
extern "C" int pk_gemm_plan(int M, int N, int K, int kind, int accumulate, int* out9) {
  using namespace pk;
  PK_CHECK(out9 && M > 0 && N > 0 && K > 0 && N % 64 == 0, "pk_gemm_plan: bad arguments");
  PkEpilogue e;
  memset(&e, 0, sizeof(e));
  e.kind = kind;
  e.accumulate = accumulate;
  GemmArgs g;
  plan_gemm(M, N, K, 0, 0, &e, g);
  const int vals[9] = {0, g.BN, g.num_m_tiles, g.num_n_tiles, g.splits, g.kb_per_split, g.streamk_units,
                       g.group_m, gemm_workers(g)};
  for (int i = 0; i < 9; ++i) out9[i] = vals[i];
  return 0;
}

extern "C" int pk_gemm_plan_walk(int M, int N, int K, int kind, int accumulate, int worker, int* out4, int max_items) {
  using namespace pk;
  PK_CHECK(out4 && max_items > 0, "pk_gemm_plan_walk: bad arguments");
  PK_CHECK(M > 0 && N > 0 && K > 0 && N % 64 == 0, "pk_gemm_plan_walk: bad arguments");
  PkEpilogue e;
  memset(&e, 0, sizeof(e));
  e.kind = kind;
  e.accumulate = accumulate;
  GemmArgs g;
  plan_gemm(M, N, K, 0, 0, &e, g);
  const int num_kb = (K + GEMM_BK - 1) / GEMM_BK;
  GemmSched sch;
  sch.init(g, g.num_m_tiles * g.num_n_tiles, num_kb, worker, gemm_workers(g));
  int n = 0, mn, kb0, kb1;
  while (n < max_items && sch.next(mn, kb0, kb1)) {
    int mb, nb;
    gemm_tile_coords(g, mn, mb, nb);
    out4[4 * n] = mb; out4[4 * n + 1] = nb; out4[4 * n + 2] = kb0; out4[4 * n + 3] = kb1;
    ++n;
  }
  return -n;   // number of items, negated (0 and positive values are the usual status codes)
}

extern "C" int pk_gemm_bf16(const void* A, const void* B, int M, int N, int K, int lda, int ldb,
                            int transA, int transB, const PkEpilogue* epi, void* stream) {
  using namespace pk;
  PK_CHECK(A && B && epi && epi->out, "pk_gemm_bf16: null pointer");
  PK_CHECK(M > 0 && N > 0 && K > 0, "pk_gemm_bf16: bad shape M=%d N=%d K=%d", M, N, K);
  PK_CHECK(N % 64 == 0, "pk_gemm_bf16: N=%d must be a multiple of 64", N);
  PK_CHECK(lda % 8 == 0 && ldb % 8 == 0, "pk_gemm_bf16: lda/ldb must be multiples of 8 (16 B)");
  PK_CHECK((reinterpret_cast<uintptr_t>(A) & 15) == 0 && (reinterpret_cast<uintptr_t>(B) & 15) == 0,
           "pk_gemm_bf16: operands must be 16-byte aligned");
  PK_CHECK(epi->kind >= PK_EPI_BF16 && epi->kind <= PK_EPI_PIXSHUF, "pk_gemm_bf16: bad epilogue %d",
           epi->kind);
  if (epi->kind != PK_EPI_PIXSHUF)
    PK_CHECK(epi->ldc % 8 == 0 && epi->ldc >= N, "pk_gemm_bf16: bad ldc %d", epi->ldc);
  if (epi->kind == PK_EPI_RESID || epi->kind == PK_EPI_DGELU)
    PK_CHECK(epi->aux && epi->ld_aux % 8 == 0, "pk_gemm_bf16: epilogue %d needs aux", epi->kind);
  if (epi->kind == PK_EPI_GELU) PK_CHECK(epi->out2, "pk_gemm_bf16: GELU epilogue needs out2");
  if (epi->kind == PK_EPI_RESID && epi->rowscale)
    PK_CHECK(epi->rows_per_group > 0, "pk_gemm_bf16: rows_per_group must be > 0");
  if (epi->kind == PK_EPI_PIXSHUF)
    PK_CHECK(epi->ps_c % 32 == 0 && epi->ps_h * epi->ps_w > 0 && M % (epi->ps_h * epi->ps_w) == 0 &&
                 N == epi->ps_p * epi->ps_p * epi->ps_c,
             "pk_gemm_bf16: bad pixel-shuffle geometry");

  GemmArgs g;
  plan_gemm(M, N, K, transA, transB, epi, g);

  CUtensorMap tmA, tmB;
  {
    uint64_t dims[2], strides[1];
    uint32_t box[2];
    if (!g.transA) {
      dims[0] = K; dims[1] = M; box[0] = 64; box[1] = GEMM_BM;
    } else {
      dims[0] = M; dims[1] = K; box[0] = 64; box[1] = 64;
    }
    strides[0] = static_cast<uint64_t>(lda) * 2;
    if (!make_tmap_bf16(&tmA, A, 2, dims, strides, box)) return 3;
    if (!g.transB) {
      dims[0] = K; dims[1] = N; box[0] = 64; box[1] = static_cast<uint32_t>(g.BN);
    } else {
      dims[0] = N; dims[1] = K; box[0] = 64; box[1] = 64;
    }
    strides[0] = static_cast<uint64_t>(ldb) * 2;
    if (!make_tmap_bf16(&tmB, B, 2, dims, strides, box)) return 3;
  }
  GemmOutMaps tmo;
  memset(&tmo, 0, sizeof(tmo));
  if (gemm_tma_epilogue(epi->kind)) {
    // [M, N] bf16 outputs with row stride ldc, stored in 64 x 64 boxes; rows past M are clipped
    PK_CHECK((reinterpret_cast<uintptr_t>(epi->out) & 15) == 0 &&
                 (epi->kind != PK_EPI_GELU || (reinterpret_cast<uintptr_t>(epi->out2) & 15) == 0),
             "pk_gemm_bf16: outputs must be 16-byte aligned");
    const uint64_t dims[2] = {static_cast<uint64_t>(N), static_cast<uint64_t>(M)};
    const uint64_t strides[1] = {static_cast<uint64_t>(epi->ldc) * 2};
    const uint32_t box[2] = {64, 64};
    if (!make_tmap_bf16(&tmo.c, epi->out, 2, dims, strides, box)) return 3;
    if (epi->kind == PK_EPI_GELU && !make_tmap_bf16(&tmo.c2, epi->out2, 2, dims, strides, box)) return 3;
  }
  return launch_gemm(tmA, tmB, tmo, g, static_cast<cudaStream_t>(stream), "pk_gemm_bf16");
}

// ------------------------------------------------------------------------------------------------
// Decoder 3x3 convolution (64 -> 64, pad 1) as implicit GEMM over NHWC bf16 (models_painter.py:328-333)
// ------------------------------------------------------------------------------------------------
static int conv_common(const void* img_nhwc, const void* wmat, int B, int H, int W, pk::GemmArgs& g,
                       void* stream, const char* who) {
  using namespace pk;
  int TW, TH;
  PK_CHECK(conv_tile_geometry(H, W, 128, &TW, &TH), "%s: unsupported image size %dx%d", who, H, W);
  g.M = B * H * W;
  g.N = 64;
  g.K = 576;
  g.BN = 64;
  g.stages = gemm_stages_for(GEMM_A_BYTES + 64 * 128, g.epi.kind);
  g.transA = g.transB = 0;
  g.splits = 1;
  g.kb_per_split = 9;
  g.conv.mode = 1;
  g.conv.H = H; g.conv.W = W; g.conv.TW = TW; g.conv.TH = TH;
  g.conv.tiles_x = W / TW; g.conv.tiles_y = H / TH;
  g.num_m_tiles = B * g.conv.tiles_x * g.conv.tiles_y;
  g.num_n_tiles = 1;
  CUtensorMap tmA, tmB;
  uint64_t dims[4] = {64, static_cast<uint64_t>(W), static_cast<uint64_t>(H), static_cast<uint64_t>(B)};
  uint64_t strides[3] = {128, static_cast<uint64_t>(W) * 128, static_cast<uint64_t>(H) * W * 128};
  uint32_t box[4] = {64, static_cast<uint32_t>(TW), static_cast<uint32_t>(TH), 1};
  if (!make_tmap_bf16(&tmA, img_nhwc, 4, dims, strides, box)) return 3;
  uint64_t d2[2] = {576, 64};
  uint64_t s2[1] = {576 * 2};
  uint32_t b2[2] = {64, 64};
  if (!make_tmap_bf16(&tmB, wmat, 2, d2, s2, b2)) return 3;
  GemmOutMaps tmo;
  memset(&tmo, 0, sizeof(tmo));
  return launch_gemm(tmA, tmB, tmo, g, static_cast<cudaStream_t>(stream), who);
}

extern "C" int pk_decoder_head_fwd(const void* g_nhwc, const void* wmat, const float* head_params,
                                   const float* tgts, const uint8_t* mask, int maskB, const float* valid,
                                   void* c1_out, float* patch_out, float* num, int B, int H, int W, int p,
                                   int loss_kind, void* stream) {
  using namespace pk;
  PK_CHECK(g_nhwc && wmat && head_params && tgts && mask && valid && c1_out && patch_out && num,
           "pk_decoder_head_fwd: null pointer");
  PK_CHECK(H % p == 0 && W % p == 0 && maskB >= 1, "pk_decoder_head_fwd: bad geometry");
  // the head parameters ride in constant memory (operands of the epilogue's FFMAs): every call takes the next of
  // HEAD_SLOTS copies, uploaded on the call's stream just ahead of its kernel
  static std::atomic<unsigned> next_slot{0};
  const int slot = static_cast<int>(next_slot.fetch_add(1, std::memory_order_relaxed) % HEAD_SLOTS);
  cudaError_t e = cudaMemcpyToSymbolAsync(c_head_all, head_params, 387 * sizeof(float), slot * 392 * sizeof(float),
                                          cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream));
  PK_CHECK(e == cudaSuccess, "pk_decoder_head_fwd: constant upload: %s", cudaGetErrorString(e));
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.head.slot = slot;
  g.epi.kind = EPI_HEAD;
  g.epi.alpha = 1.0f;
  g.head.tgts = tgts; g.head.mask = mask; g.head.valid = valid; g.head.maskB = maskB;
  g.head.c1_out = static_cast<__nv_bfloat16*>(c1_out);
  g.head.patch_out = patch_out; g.head.num = num; g.head.p = p; g.head.loss_kind = loss_kind;
  return conv_common(g_nhwc, wmat, B, H, W, g, stream, "pk_decoder_head_fwd");
}

// dG (inverse pixel shuffle) [B*h*w, p*p*64] = conv3x3^T(dC1); wmat_t = dgrad weight matrix (flipped taps)
extern "C" int pk_conv3x3_dgrad_unshuffle(const void* dc1_nhwc, const void* wmat_t, void* out_tok, int B, int H,
                                          int W, int p, void* stream) {
  using namespace pk;
  PK_CHECK(dc1_nhwc && wmat_t && out_tok && H % p == 0 && W % p == 0, "pk_conv3x3_dgrad_unshuffle: bad args");
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.epi.kind = EPI_UNSHUF;
  g.epi.alpha = 1.0f;
  g.epi.out = out_tok;
  g.epi.ldc = p * p * 64;
  g.epi.ps_p = p;
  return conv_common(dc1_nhwc, wmat_t, B, H, W, g, stream, "pk_conv3x3_dgrad_unshuffle");
}

// wgrad: out[(tap*64 + c), o] += sum_pix G[pix + tap, c] * dC1[pix, o]   (out fp32 [576(+pad to 640), 64], zeroed)
extern "C" int pk_conv3x3_wgrad(const void* g_nhwc, const void* dc1_nhwc, float* out, int B, int H, int W,
                                void* stream) {
  using namespace pk;
  PK_CHECK(g_nhwc && dc1_nhwc && out, "pk_conv3x3_wgrad: null pointer");
  int TW, TH;
  PK_CHECK(conv_tile_geometry(H, W, 64, &TW, &TH), "pk_conv3x3_wgrad: unsupported image size %dx%d", H, W);
  GemmArgs g;
  memset(&g, 0, sizeof(g));
  g.M = 576; g.N = 64; g.K = B * H * W;
  g.BN = 64; g.stages = gemm_stages_for(GEMM_A_BYTES + 64 * 128, PK_EPI_F32);
  g.transA = g.transB = 1;
  g.conv.mode = 2;
  g.conv.H = H; g.conv.W = W; g.conv.TW = TW; g.conv.TH = TH;
  g.conv.tiles_x = W / TW; g.conv.tiles_y = H / TH;
  g.num_m_tiles = 5; g.num_n_tiles = 1;
  const int num_kb = B * g.conv.tiles_x * g.conv.tiles_y;
  int splits = sm_count() / 5;
  if (splits > num_kb) splits = num_kb;
  if (splits < 1) splits = 1;
  g.kb_per_split = (num_kb + splits - 1) / splits;
  g.splits = (num_kb + g.kb_per_split - 1) / g.kb_per_split;
  g.epi.kind = PK_EPI_F32;
  g.epi.out = out;
  g.epi.ldc = 64;
  g.epi.alpha = 1.0f;
  g.epi.accumulate = 2;
  CUtensorMap tmA, tmB;
  uint64_t dims[4] = {64, static_cast<uint64_t>(W), static_cast<uint64_t>(H), static_cast<uint64_t>(B)};
  uint64_t strides[3] = {128, static_cast<uint64_t>(W) * 128, static_cast<uint64_t>(H) * W * 128};
  uint32_t box[4] = {64, static_cast<uint32_t>(TW), static_cast<uint32_t>(TH), 1};
  if (!make_tmap_bf16(&tmA, g_nhwc, 4, dims, strides, box)) return 3;
  if (!make_tmap_bf16(&tmB, dc1_nhwc, 4, dims, strides, box)) return 3;
  GemmOutMaps tmo;
  memset(&tmo, 0, sizeof(tmo));
  return launch_gemm(tmA, tmB, tmo, g, static_cast<cudaStream_t>(stream), "pk_conv3x3_wgrad");
}
