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
//
// Tangent entry and exit of dgan_jvp, the same scheme run forwards: a caller's tangent t of z enters the tangent pass
// (tangent_in_kernel; on the fp16 path scaled per row so that max_k |t[n][k]| * s_n lies in [0.25, 0.5), the magnitude of
// the primal z the fp16 path serves), and the tangent of the last layer's pre-activation leaves it as
//
//   ty = t(pre) * act'(y) / s_n                               (tangent_out_kernel)
//
// read from the fp32 block tensor [n_blocks][n_pad][16*C_out] (fp16 path) or [n_pad][H*W*C] (fp32 path, s_n = 1).
// Plain launches (no PDL): each kernel starts after its predecessor has completed.
#pragma once
#include "common.cuh"

namespace dgan {

// ACT_NONE: dy itself (the row maxima of a tangent of z)
template <int ACT>
__device__ __forceinline__ float cotangent_pre(float y, float dy) {
  if (ACT == ACT_NONE) return dy;
  const float dact = (ACT == ACT_SIGMOID) ? y * (1.f - y) : 1.f - y * y;
  return dy * dact;
}

// rowmax[n] = max_i |d(pre)[n][i]| over rows of hwc values (ACT_NONE: max_i |dy[n][i]|, y is not read).  One block per row.
template <int ACT>
__global__ void __launch_bounds__(256)
cotangent_rowmax_kernel(const float* __restrict__ y, const float* __restrict__ dy, int hwc, float* __restrict__ rowmax) {
  __shared__ float red[8];
  const size_t base = (size_t)blockIdx.x * hwc;
  float m = 0.f;
  for (int i = threadIdx.x; i < hwc; i += 256) m = fmaxf(m, fabsf(cotangent_pre<ACT>(ACT == ACT_NONE ? 0.f : y[base + i], dy[base + i])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) m = fmaxf(m, red[k]);
    rowmax[blockIdx.x] = m;
  }
}

// 2^e with m * 2^e in [2^(top-1), 2^top) (the cotangent: top = 4, [8, 16); the tangent: top = -1, [0.25, 0.5)); 1 when
// m is 0 (a row with dy == 0) or not finite.  e is clamped so that both 2^e and 2^-e are normal fp32 numbers.
__device__ __forceinline__ float pow2_scale(float m, int top) {
  if (!(m > 0.f) || isinf(m)) return 1.f;
  int ex;
  frexpf(m, &ex);                                  // m = f * 2^ex, f in [0.5, 1)
  return ldexpf(1.f, min(max(top - ex, -126), 126));
}

// In place: row maxima -> row scales pow2_scale(., top).  `shared` (BatchNorm): one scale for the call, the one of the
// largest row maximum,
// i.e. the smallest per-row scale among the rows whose cotangent is not zero (rows with dy == 0 do not pin it to 1,
// which would make the result depend on |dy|).  One block.
__global__ void __launch_bounds__(1024) cotangent_scale_kernel(float* __restrict__ scale, int n_rows, int shared, int top) {
  __shared__ float red[32];
  if (!shared) {
    for (int n = threadIdx.x; n < n_rows; n += 1024) scale[n] = pow2_scale(scale[n], top);
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
  const float s = pow2_scale(m, top);
  for (int n = threadIdx.x; n < n_rows; n += 1024) scale[n] = s;
}

// Index in the last layer's block tensor [n_blocks][n_pad][16 * CO] of element r of row n of y [n_rows][w_out][w_out][CO]:
// pixel (4*by+li, 4*bx+lj) is block by * (w_out/4) + bx, column (li*4+lj)*CO + co.
template <int CO>
__device__ __forceinline__ size_t block_index(int n, int r, int w_out, int n_pad) {
  const int pix = r / CO, co = r % CO, row = pix / w_out, col = pix % w_out;
  const int blk = (row >> 2) * (w_out >> 2) + (col >> 2);
  const int k = ((row & 3) * 4 + (col & 3)) * CO + co;
  return ((size_t)blk * n_pad + n) * (16 * CO) + k;
}

// One thread per element of y [n_rows][w_out][w_out][CO].  BLOCKS (fp16 path): dblk[block_index] = fp16(d(pre) *
// scale[n]).  Otherwise dpre[n][i] = d(pre) (rows share y's layout).
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
  dblk[block_index<CO>(n, r, w_out, n_pad)] = __float2half_rn(d * scale[n]);
}

// z's tangent at the padded latent width ld: out[n][k] = t[n][k] * scale[n] (scale NULL: 1) for the real rows and
// columns, 0 elsewhere; fp32 into out (fp32 path) or fp16 into out_h (fp16 path).
__global__ void tangent_in_kernel(const float* __restrict__ t, const float* __restrict__ scale, int n_rows, int n_pad,
                                  int latent, int ld, float* __restrict__ out, __half* __restrict__ out_h) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n_pad * ld) return;
  const int row = (int)(i / ld), col = (int)(i % ld);
  float v = 0.f;
  if (row < n_rows && col < latent) v = t[(size_t)row * latent + col] * (scale != nullptr ? scale[row] : 1.f);
  if (out != nullptr) out[i] = v;
  if (out_h != nullptr) out_h[i] = __float2half_rn(v);
}

// One thread per element of ty [n_rows][w_out][w_out][CO] = t(pre) * act'(y) / scale[n], t(pre) from the fp32 block
// tensor (BLOCKS, fp16 path) or from [n_pad][H*W*C] (scale NULL).  The scales are powers of two: the division is exact.
template <int ACT, int CO, bool BLOCKS>
__global__ void __launch_bounds__(256)
tangent_out_kernel(const float* __restrict__ y, const float* __restrict__ tpre, int n_rows, int w_out,
                   const float* __restrict__ scale, int n_pad, float* __restrict__ ty) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int hwc = w_out * w_out * CO;
  if (i >= (size_t)n_rows * hwc) return;
  const int n = (int)(i / hwc), r = (int)(i % hwc);
  const float t = BLOCKS ? tpre[block_index<CO>(n, r, w_out, n_pad)] : tpre[i];
  float v = cotangent_pre<ACT>(y[i], t);
  if (scale != nullptr) v /= scale[n];
  ty[i] = v;
}

}  // namespace dgan
