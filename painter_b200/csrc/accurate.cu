// painter_b200 — kernels of the fp32-ACCURATE forward mode (north star: outputs within 1e-5 of the reference's fp32
// forward, which is how seggpt_engine.run_one_image calls the model: `.float()`, no autocast, seggpt_engine.py:47).
//
// The tensor cores stay the compute engine.  Every fp32 operand x is split into three bf16 terms
//     h = bf16(x),  m = bf16(x - h),  l = bf16(x - h - m)          (x = h + m + l up to 2^-24 |x|)
// and a product a.b is evaluated as  a_l b_h + a_m b_m + a_h b_l + a_m b_h + a_h b_m + a_h b_h  (the six terms above
// 2^-24; smallest first) by CONCATENATING the terms along K:  A' = [l | m | h | m | h | h],  B' = [h | m | l | h | m | h],
// K' = 6 K - ONE ordinary wgmma GEMM (pk_gemm_bf16) with fp32 accumulation in registers.  The kernels here produce
// those split operands (fused with the elementwise step in front of the GEMM: GELU, softmax, im2col) and the few fp32
// elementwise stages the bf16 path had fused into GEMM epilogues.  All are HBM-bound streaming kernels.  The split
// itself and the term order (split3.cuh) are shared with the fused split attention forward of windowed blocks
// (pk_attn_fwd_split3, attention.cu), which splits its tiles in shared memory instead of writing 6x-wide operands.
#include "common.cuh"
#include "split3.cuh"
#include "host_common.h"
#include "../../include/painter_b200.h"

namespace pk {

__device__ __forceinline__ float gelu_exact(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }

static inline int stream_grid2(size_t total, int block = 256) {
  size_t g = (total + block - 1) / block;
  const size_t cap = static_cast<size_t>(sm_count()) * 32;
  return static_cast<int>(g < 1 ? 1 : (g > cap ? cap : g));
}

// out[r, t*K + k] = term_{side}(t)(f(x[r, k])),  f = identity or exact-erf GELU
template <bool GELU>
__global__ void __launch_bounds__(256)
split3_kernel(const float* __restrict__ x, int ldx, __nv_bfloat16* __restrict__ out, int M, int K, int side_b) {
  const size_t total = static_cast<size_t>(M) * K;
  const size_t ldo = static_cast<size_t>(6) * K;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t r = i / K;
    const int k = static_cast<int>(i - r * K);
    float v = x[r * ldx + k];
    if (GELU) v = gelu_exact(v);
    __nv_bfloat16 t[3];
    split3(v, t);
    __nv_bfloat16* o = out + r * ldo + k;
#pragma unroll
    for (int b = 0; b < 6; ++b) o[static_cast<size_t>(b) * K] = t[side_b ? c_termB[b] : c_termA[b]];
  }
}

// qkv fp32 [B*N, 3C] (columns (3, head, 64)) -> per-(b, head) split operands of the attention GEMMs:
//   which = 0 (q): out [B*heads, N, 6*64]       A-side, rows = queries
//   which = 1 (k): out [B*heads, Npad, 6*64]    B-side, rows = keys (rows >= N stay zero: caller zero-fills)
//   which = 2 (v): out [B*heads, 6*Npad, 64]    B-side stacked along K' = (term block, key) for an MN-major B operand
__global__ void __launch_bounds__(256)
split3_heads_kernel(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int B, int heads, int N, int Npad,
                    int which) {
  const int C = heads * 64;
  const size_t total = static_cast<size_t>(B) * N * C;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int d = static_cast<int>(i & 63);
    size_t r = i >> 6;
    const int hd = static_cast<int>(r % heads);
    r /= heads;
    const int t = static_cast<int>(r % N), b = static_cast<int>(r / N);
    const float v = qkv[(static_cast<size_t>(b) * N + t) * (3 * C) + which * C + hd * 64 + d];
    __nv_bfloat16 s[3];
    split3(v, s);
    const size_t bh = static_cast<size_t>(b) * heads + hd;
    if (which == 0) {
      __nv_bfloat16* o = out + (bh * N + t) * 384 + d;
#pragma unroll
      for (int k = 0; k < 6; ++k) o[k * 64] = s[c_termA[k]];
    } else if (which == 1) {
      __nv_bfloat16* o = out + (bh * Npad + t) * 384 + d;
#pragma unroll
      for (int k = 0; k < 6; ++k) o[k * 64] = s[c_termB[k]];
    } else {
      __nv_bfloat16* o = out + (bh * 6 * Npad + t) * 64 + d;
#pragma unroll
      for (int k = 0; k < 6; ++k) o[static_cast<size_t>(k) * Npad * 64] = s[c_termB[k]];
    }
  }
}

// One block per (b*head, query row): s[u] = scale * S[u] + Gh[i_t - i_u + h - 1] + Gw[j_t - j_u + w - 1],
// p = softmax(s) in fp32 (models_painter.py:80-86, vitdet_utils.py:113-123), written as A-side split operand
// P' [N, 6*Npad] (columns >= N of every term block stay zero: caller zero-fills once).
__global__ void __launch_bounds__(256)
softmax_relpos_split3_kernel(const float* __restrict__ S, const float* __restrict__ Gh, int ldgh,
                             const float* __restrict__ Gw, int ldgw, __nv_bfloat16* __restrict__ P, int N, int Npad,
                             int h, int w, float scale) {
  extern __shared__ float row[];   // N scores
  __shared__ float red[8];
  const size_t bh = blockIdx.y;
  const int t = blockIdx.x;
  const int i_t = t / w, j_t = t - i_t * w;
  const float* s_in = S + (bh * N + t) * static_cast<size_t>(Npad);
  const float* gh = Gh + (bh * N + t) * static_cast<size_t>(ldgh) + (i_t + h - 1);
  const float* gw = Gw + (bh * N + t) * static_cast<size_t>(ldgw) + (j_t + w - 1);
  float mx = -INFINITY;
  for (int u = threadIdx.x; u < N; u += 256) {
    const int i_u = u / w, j_u = u - i_u * w;
    const float v = s_in[u] * scale + gh[-i_u] + gw[-j_u];
    row[u] = v;
    mx = fmaxf(mx, v);
  }
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int k = 1; k < 8; ++k) mx = fmaxf(mx, red[k]);
  __syncthreads();
  float sum = 0.f;
  for (int u = threadIdx.x; u < N; u += 256) {
    const float e = expf(row[u] - mx);
    row[u] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  sum = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) sum += red[k];
  const float inv = 1.0f / sum;
  __nv_bfloat16* o = P + (bh * N + t) * static_cast<size_t>(6) * Npad;
  for (int u = threadIdx.x; u < N; u += 256) {
    __nv_bfloat16 sp[3];
    split3(row[u] * inv, sp);
#pragma unroll
    for (int k = 0; k < 6; ++k) o[static_cast<size_t>(k) * Npad + u] = sp[c_termA[k]];
  }
}

// PatchEmbed im2col (vitdet_utils.py:178-186; K order (c, pr, pc)) of imgs and tgts, A-side split:
// out [2*B*h*w, 6*Cin*p*p]
__global__ void __launch_bounds__(256)
im2col_patch_split3_kernel(const float* __restrict__ imgs, const float* __restrict__ tgts,
                           __nv_bfloat16* __restrict__ out, int B, int Cin, int H, int W, int p) {
  const int h = H / p, w = W / p, K = Cin * p * p;
  const size_t total = static_cast<size_t>(2) * B * h * w * K;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % K);
    const size_t r = i / K;
    const int tj = static_cast<int>(r % w);
    size_t q = r / w;
    const int ti = static_cast<int>(q % h);
    const int bb = static_cast<int>(q / h);
    const int pc = k % p, pr = (k / p) % p, c = k / (p * p);
    const float* src = bb < B ? imgs : tgts;
    const int b = bb < B ? bb : bb - B;
    const float v = src[((static_cast<size_t>(b) * Cin + c) * H + ti * p + pr) * W + tj * p + pc];
    __nv_bfloat16 s[3];
    split3(v, s);
    __nv_bfloat16* o = out + r * static_cast<size_t>(6) * K + k;
#pragma unroll
    for (int t = 0; t < 6; ++t) o[static_cast<size_t>(t) * K] = s[c_termA[t]];
  }
}

// im2col of the pixel-shuffled decoder feature map for the 3x3 convolution (models_painter.py:424-430):
// D fp32 [B*h*w, p*p*dd] (token-major, columns (r, s, c))  ->  out [B*H*W, 6 * 9*dd] A-side split, column
// (ky*3 + kx)*dd + c of a term block = G[b, c, y+ky-1, x+kx-1] (zero outside the image).
__global__ void __launch_bounds__(256)
dec_im2col_split3_kernel(const float* __restrict__ D, __nv_bfloat16* __restrict__ out, int B, int h, int w, int p,
                         int dd) {
  const int H = h * p, W = w * p, K = 9 * dd;
  const size_t total = static_cast<size_t>(B) * H * W * K;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % K);
    const size_t pix = i / K;
    const int x = static_cast<int>(pix % W);
    const size_t q = pix / W;
    const int y = static_cast<int>(q % H), b = static_cast<int>(q / H);
    const int c = k % dd, tap = k / dd, ky = tap / 3, kx = tap - ky * 3;
    const int yy = y + ky - 1, xx = x + kx - 1;
    float v = 0.f;
    if (yy >= 0 && yy < H && xx >= 0 && xx < W) {
      const size_t tok = (static_cast<size_t>(b) * h + yy / p) * w + xx / p;
      v = D[tok * (static_cast<size_t>(p) * p * dd) + ((yy % p) * p + (xx % p)) * dd + c];
    }
    __nv_bfloat16 s[3];
    split3(v, s);
    __nv_bfloat16* o = out + pix * static_cast<size_t>(6) * K + k;
#pragma unroll
    for (int t = 0; t < 6; ++t) o[static_cast<size_t>(t) * K] = s[c_termA[t]];
  }
}

// Decoder head in fp32, one thread per pixel (vitdet_utils.py:204-209 LayerNorm2D, nn.GELU exact, conv1x1) + the
// masked loss terms and the patchified store (models_painter.py:355-368,433-462).  c1: fp32 [B*H*W, 64] (conv3x3
// output incl. bias); hp: [c3_b 64 (unused here) | ln_w 64 | ln_b 64 | w1 3x64 | b1 3]; num[b] += sum of loss terms.
__global__ void __launch_bounds__(128)
head_f32_kernel(const float* __restrict__ c1, const float* __restrict__ hp, const float* __restrict__ tgts,
                const uint8_t* __restrict__ mask, int maskB, const float* __restrict__ valid,
                float* __restrict__ patch, double* __restrict__ num, int B, int H, int W, int p, int loss_kind) {
  const size_t npix = static_cast<size_t>(B) * H * W;
  const size_t pix = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  float lsum = 0.f;
  int b = 0;
  if (pix < npix) {
    const int x = static_cast<int>(pix % W);
    const size_t q = pix / W;
    const int y = static_cast<int>(q % H);
    b = static_cast<int>(q / H);
    float v[64];
    const float4* src = reinterpret_cast<const float4*>(c1 + pix * 64);
    float mean = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const float4 t = src[k];
      v[4 * k] = t.x; v[4 * k + 1] = t.y; v[4 * k + 2] = t.z; v[4 * k + 3] = t.w;
      mean += (t.x + t.y) + (t.z + t.w);
    }
    mean *= (1.f / 64);
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < 64; ++k) {
      v[k] -= mean;
      var += v[k] * v[k];
    }
    const float rstd = 1.0f / sqrtf(var * (1.f / 64) + 1e-6f);
    float pr[3] = {hp[384], hp[385], hp[386]};
#pragma unroll
    for (int k = 0; k < 64; ++k) {
      const float g = gelu_exact(hp[64 + k] * (v[k] * rstd) + hp[128 + k]);
      pr[0] += hp[192 + k] * g;
      pr[1] += hp[256 + k] * g;
      pr[2] += hp[320 + k] * g;
    }
    const int wt = W / p, ti = y / p, tj = x / p;
    const int ntok = (H / p) * wt;
    const float mk = mask[static_cast<size_t>(b % maskB) * ntok + ti * wt + tj] ? 1.f : 0.f;
    float* po = patch + ((static_cast<size_t>(b) * ntok + ti * wt + tj) * (p * p) + (y % p) * p + (x % p)) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      po[c] = pr[c];
      const size_t o = (static_cast<size_t>(b) * 3 + c) * H * W + static_cast<size_t>(y) * W + x;
      const float d = pr[c] - tgts[o];
      const float ad = fabsf(d);
      float l;
      if (loss_kind == 0) l = ad < 0.01f ? 0.5f * d * d / 0.01f : ad - 0.005f;
      else if (loss_kind == 1) l = ad;
      else if (loss_kind == 2) l = d * d;
      else l = 0.5f * (ad + d * d);
      lsum += l * mk * valid[o];
    }
  }
  // a block never straddles two samples when H*W % 128 == 0 (checked on the host): one fp64 atomic per warp (the
  // 1e-5 loss bar leaves no room for a 10^4-term fp32 accumulation chain)
  lsum = warp_sum(lsum);
  if ((threadIdx.x & 31) == 0 && pix < npix) atomicAdd(num + b, static_cast<double>(lsum));
}

__global__ void f64_to_f32_kernel(const double* __restrict__ in, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = static_cast<float>(in[i]);
}

}  // namespace pk

using namespace pk;

extern "C" int pk_split3(const float* x, int ldx, void* out_bf16, int M, int K, int side_b, int gelu, void* stream) {
  PK_CHECK(x && out_bf16 && M > 0 && K > 0 && ldx >= K, "pk_split3: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t total = static_cast<size_t>(M) * K;
  if (gelu)
    split3_kernel<true><<<stream_grid2(total), 256, 0, st>>>(x, ldx, static_cast<__nv_bfloat16*>(out_bf16), M, K, side_b);
  else
    split3_kernel<false><<<stream_grid2(total), 256, 0, st>>>(x, ldx, static_cast<__nv_bfloat16*>(out_bf16), M, K, side_b);
  PK_LAUNCH_CHECK("pk_split3");
  return 0;
}

extern "C" int pk_split3_heads(const float* qkv, void* out_bf16, int B, int heads, int N, int Npad, int which,
                               void* stream) {
  PK_CHECK(qkv && out_bf16 && B > 0 && heads > 0 && N > 0 && Npad >= N && which >= 0 && which <= 2,
           "pk_split3_heads: bad arguments");
  const size_t total = static_cast<size_t>(B) * N * heads * 64;
  split3_heads_kernel<<<stream_grid2(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      qkv, static_cast<__nv_bfloat16*>(out_bf16), B, heads, N, Npad, which);
  PK_LAUNCH_CHECK("pk_split3_heads");
  return 0;
}

extern "C" int pk_softmax_relpos_split3(const float* S, const float* Gh, int ldgh, const float* Gw, int ldgw,
                                        void* P_bf16, int BH, int N, int Npad, int h, int w, float scale,
                                        void* stream) {
  PK_CHECK(S && Gh && Gw && P_bf16 && BH > 0 && N == h * w && Npad >= N && ldgh >= 2 * h - 1 && ldgw >= 2 * w - 1,
           "pk_softmax_relpos_split3: bad arguments");
  const size_t smem = static_cast<size_t>(N) * sizeof(float);
  PK_CHECK(smem <= 200 * 1024, "pk_softmax_relpos_split3: N=%d too large", N);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(softmax_relpos_split3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    attr = true;
  }
  softmax_relpos_split3_kernel<<<dim3(N, BH), 256, smem, static_cast<cudaStream_t>(stream)>>>(
      S, Gh, ldgh, Gw, ldgw, static_cast<__nv_bfloat16*>(P_bf16), N, Npad, h, w, scale);
  PK_LAUNCH_CHECK("pk_softmax_relpos_split3");
  return 0;
}

extern "C" int pk_im2col_patch_split3(const float* imgs, const float* tgts, void* out_bf16, int B, int Cin, int H,
                                      int W, int p, void* stream) {
  PK_CHECK(imgs && tgts && out_bf16 && H % p == 0 && W % p == 0, "pk_im2col_patch_split3: bad arguments");
  const size_t total = static_cast<size_t>(2) * B * (H / p) * (W / p) * Cin * p * p;
  im2col_patch_split3_kernel<<<stream_grid2(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      imgs, tgts, static_cast<__nv_bfloat16*>(out_bf16), B, Cin, H, W, p);
  PK_LAUNCH_CHECK("pk_im2col_patch_split3");
  return 0;
}

extern "C" int pk_dec_im2col_split3(const float* D, void* out_bf16, int B, int h, int w, int p, int dd,
                                    void* stream) {
  PK_CHECK(D && out_bf16 && B > 0 && h > 0 && w > 0 && p > 0 && dd > 0, "pk_dec_im2col_split3: bad arguments");
  const size_t total = static_cast<size_t>(B) * h * p * w * p * 9 * dd;
  dec_im2col_split3_kernel<<<stream_grid2(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      D, static_cast<__nv_bfloat16*>(out_bf16), B, h, w, p, dd);
  PK_LAUNCH_CHECK("pk_dec_im2col_split3");
  return 0;
}

extern "C" int pk_head_f32(const float* c1, const float* head_params, const float* tgts, const uint8_t* mask,
                           int maskB, const float* valid, float* patch, double* num_zeroed, float* num_out, int B,
                           int H, int W, int p, int loss_kind, void* stream) {
  PK_CHECK(c1 && head_params && tgts && mask && valid && patch && num_zeroed && num_out, "pk_head_f32: null pointer");
  PK_CHECK((static_cast<long long>(H) * W) % 128 == 0 && H % p == 0 && W % p == 0, "pk_head_f32: bad image size");
  const size_t npix = static_cast<size_t>(B) * H * W;
  head_f32_kernel<<<static_cast<unsigned>((npix + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      c1, head_params, tgts, mask, maskB, valid, patch, num_zeroed, B, H, W, p, loss_kind);
  PK_LAUNCH_CHECK("pk_head_f32");
  f64_to_f32_kernel<<<(B + 63) / 64, 64, 0, static_cast<cudaStream_t>(stream)>>>(num_zeroed, num_out, B);
  PK_LAUNCH_CHECK("pk_head_f32(num)");
  return 0;
}
