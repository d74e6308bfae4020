// painter_b200 — the three-term bf16 split of fp32 operands, shared by the fp32-accurate kernels (accurate.cu and the
// split attention forward in attention.cu), so that both evaluate the same six cross products in the same order.
#pragma once
#include <cuda_bf16.h>

namespace pk {

// term index of K-block t (0..5) for an A-side / B-side operand: 0 = h, 1 = m, 2 = l
__device__ constexpr int c_termA[6] = {2, 1, 0, 1, 0, 0};
__device__ constexpr int c_termB[6] = {0, 1, 2, 0, 1, 0};

__device__ __forceinline__ void split3(float x, __nv_bfloat16 (&t)[3]) {
  t[0] = __float2bfloat16_rn(x);
  const float r1 = x - __bfloat162float(t[0]);
  t[1] = __float2bfloat16_rn(r1);
  const float r2 = r1 - __bfloat162float(t[1]);
  t[2] = __float2bfloat16_rn(r2);
}

}  // namespace pk
