// painter_b200 — pieces shared by the task-metric kernels (metrics.cu, restoration_matlab.cu): the per-image row of the
// descriptor table and a fixed-order CTA sum.
#pragma once
#include "common.cuh"
#include "../../include/painter_b200.h"

namespace pk {

// One image of a metric launch: a row of PK_METRIC_FIELDS int64 of the descriptor table.
struct MetricItem {
  const void* pred;
  const void* gt;
  int H, W;
};
__device__ __forceinline__ MetricItem metric_item(const long long* items, const uint8_t* base, int i) {
  const long long* r = items + static_cast<size_t>(i) * PK_METRIC_FIELDS;
  MetricItem it;
  it.pred = r[1] ? static_cast<const void*>(base + r[0]) : reinterpret_cast<const void*>(r[0]);
  it.gt = base + r[2];
  it.H = static_cast<int>(r[3]);
  it.W = static_cast<int>(r[4]);
  return it;
}

// Fixed-order CTA sum of NV doubles per thread (warp shuffle tree, then the warps' partials in warp order); the
// result is valid in thread 0.
template <int NV, int THREADS>
__device__ __forceinline__ void block_sum(double (&v)[NV], double (*red)[THREADS / 32]) {
#pragma unroll
  for (int j = 0; j < NV; ++j) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[j] += __shfl_down_sync(0xffffffffu, v[j], o);
  }
  const int warp = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int j = 0; j < NV; ++j) red[j][warp] = v[j];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      double s = red[j][0];
      for (int w = 1; w < THREADS / 32; ++w) s += red[j][w];
      v[j] = s;
    }
  }
}

}  // namespace pk
