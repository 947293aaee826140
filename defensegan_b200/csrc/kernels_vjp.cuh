// Cotangent entry of dgan_vjp: a caller's dL/dy enters the generator's backward in place of the projection's (y - x).
//
//   d(pre) = dy * act'(y)        act' = y(1-y) (sigmoid) | 1 - y^2 (tanh), from the same fp32 y the epilogues use
//
// fp32 path: d(pre) goes to the [n_pad][H*W*C] buffer the last layer's backward reads.
// fp16 path: it goes to the last layer's 4x4 block tensor [n_blocks][n_pad][16*C_out] (column (li*4+lj)*C_out + co), scaled
// per row by a power of two s_n chosen so that the row's largest |d(pre)| * s_n lies in [8, 16) - the ceiling the
// MNIST MSE cotangent reaches with the projection's fixed scale.  Being powers of two, the scales are exact: undoing
// them after the backward (scale_copy_kernel) makes the result independent of |dy| up to the fp32/fp16 range limits.
// With batch-statistics BatchNorm the backward mixes rows, so every row gets the same scale (see cotangent_scale_kernel).
// Plain launches (no PDL): each kernel starts after its predecessor has completed.
#pragma once
#include "common.cuh"

namespace dgan {

template <int ACT>
__device__ __forceinline__ float cotangent_pre(float y, float dy) {
  const float dact = (ACT == ACT_SIGMOID) ? y * (1.f - y) : 1.f - y * y;
  return dy * dact;
}

// rowmax[n] = max_i |d(pre)[n][i]|.  One block per row.
template <int ACT>
__global__ void __launch_bounds__(256)
cotangent_rowmax_kernel(const float* __restrict__ y, const float* __restrict__ dy, int hwc, float* __restrict__ rowmax) {
  __shared__ float red[8];
  const size_t base = (size_t)blockIdx.x * hwc;
  float m = 0.f;
  for (int i = threadIdx.x; i < hwc; i += 256) m = fmaxf(m, fabsf(cotangent_pre<ACT>(y[base + i], dy[base + i])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) m = fmaxf(m, red[k]);
    rowmax[blockIdx.x] = m;
  }
}

// 2^e with m * 2^e in [8, 16); 1 when m is 0 (a row with dy == 0) or not finite.  e is clamped so that both 2^e and
// 2^-e are normal fp32 numbers.
__device__ __forceinline__ float pow2_scale(float m) {
  if (!(m > 0.f) || isinf(m)) return 1.f;
  int ex;
  frexpf(m, &ex);                                  // m = f * 2^ex, f in [0.5, 1)
  return ldexpf(1.f, min(max(4 - ex, -126), 126));
}

// In place: row maxima -> row scales.  `shared` (BatchNorm): one scale for the call, the one of the largest row maximum,
// i.e. the smallest per-row scale among the rows whose cotangent is not zero (rows with dy == 0 do not pin it to 1,
// which would make the result depend on |dy|).  One block.
__global__ void __launch_bounds__(1024) cotangent_scale_kernel(float* __restrict__ scale, int n_rows, int shared) {
  __shared__ float red[32];
  if (!shared) {
    for (int n = threadIdx.x; n < n_rows; n += 1024) scale[n] = pow2_scale(scale[n]);
    return;
  }
  float m = 0.f;
  for (int n = threadIdx.x; n < n_rows; n += 1024) m = fmaxf(m, scale[n]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int k = 1; k < 32; ++k) m = fmaxf(m, red[k]);
  const float s = pow2_scale(m);
  for (int n = threadIdx.x; n < n_rows; n += 1024) scale[n] = s;
}

// One thread per element of y [n_rows][w_out][w_out][CO].  BLOCKS (fp16 path): dblk[blk][n][(li*4+lj)*CO + co] =
// fp16(d(pre) * scale[n]) for pixel (4*by+li, 4*bx+lj), blk = by * (w_out/4) + bx.  Otherwise dpre[n][i] = d(pre)
// (rows share y's layout).
template <int ACT, int CO, bool BLOCKS>
__global__ void __launch_bounds__(256)
cotangent_kernel(const float* __restrict__ y, const float* __restrict__ dy, int n_rows, int w_out,
                 const float* __restrict__ scale, float* __restrict__ dpre, __half* __restrict__ dblk, int n_pad) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int hwc = w_out * w_out * CO;
  if (i >= (size_t)n_rows * hwc) return;
  const float d = cotangent_pre<ACT>(y[i], dy[i]);
  if (!BLOCKS) { dpre[i] = d; return; }
  const int n = (int)(i / hwc), r = (int)(i % hwc);
  const int pix = r / CO, co = r % CO, row = pix / w_out, col = pix % w_out;
  const int blk = (row >> 2) * (w_out >> 2) + (col >> 2);
  const int k = ((row & 3) * 4 + (col & 3)) * CO + co;
  dblk[((size_t)blk * n_pad + n) * (16 * CO) + k] = __float2half_rn(d * scale[n]);
}

}  // namespace dgan
