// The Adam update of the latent rows (dgan_reconstruct_adam and its measured and pruned forms): the alternative to the
// momentum update of tf.train.MomentumOptimizer that every projection entry point can run instead.  Per coordinate and
// per row, so rows stay independent and restart pruning keeps its guarantees without BatchNorm.
#pragma once
#include "common.cuh"

namespace dgan {

// Adam (Kingma & Ba 2015) on z, iteration k = t + 1 of the loop:
//   g  = gm * (sum of the n_parts split-K partials, fixed order 0, 1, 2, ...)
//        gm = gmul / row_scale[row] on the real rows when row_scale is not NULL (the measured loop's power-of-two
//        cotangent scales, so the division is exact), gmul otherwise - the g of momentum_kernel / momentum_rows_kernel
//   m  = fmaf(b1, m, (1 - b1) * g)
//   s  = fmaf(b2, s, (1 - b2) * (g * g))
//   z  = z - (c1 * m) / fmaf(sqrtf(s), c2, eps)        c1 = lr_t / (1 - b1^k), c2 = 1 / sqrt(1 - b2^k)
// in fp32 with IEEE sqrtf and division (the library is built without fast-math), c1 and c2 rounded to fp32 from double
// on the host.  eps > 0: a coordinate whose gradient is 0 on every step (padded latent columns, an image whose pixel
// weights are all 0) keeps m = s = 0 and moves by 0 / eps = 0.  Optionally refreshes the fp16 copy of z
// that feeds the tensor-core Linear.
// PRIOR (adam_prior_kernel, the prior entries): g = fmaf(two_lambda, z, g) on the pre-update z, the gradient of
// J = D + lambda ||z||^2; the rest is unchanged.
template <bool PRIOR>
__device__ __forceinline__ void adam_body(float* __restrict__ z, float* __restrict__ m, float* __restrict__ s,
                                          const float* __restrict__ g, int n_parts, float gmul,
                                          const float* __restrict__ row_scale, int ld, int n_rows, float b1, float b2,
                                          float eps, float c1, float c2, size_t count, __half* __restrict__ z_h,
                                          float two_lambda) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float gs = g[i];
  for (int p = 1; p < n_parts; ++p) gs += g[i + (size_t)p * count];   // split-K partials, fixed order
  const size_t row = i / ld;
  const float gm = row_scale != nullptr && row < (size_t)n_rows ? gmul / row_scale[row] : gmul;
  float gg = gm * gs;
  if (PRIOR) gg = fmaf(two_lambda, z[i], gg);
  const float mm = fmaf(b1, m[i], (1.f - b1) * gg);
  const float ss = fmaf(b2, s[i], (1.f - b2) * (gg * gg));
  const float zz = z[i] - (c1 * mm) / fmaf(sqrtf(ss), c2, eps);
  m[i] = mm;
  s[i] = ss;
  z[i] = zz;
  if (z_h != nullptr) z_h[i] = __float2half_rn(zz);
}

__global__ void adam_kernel(float* __restrict__ z, float* __restrict__ m, float* __restrict__ s, const float* __restrict__ g,
                            int n_parts, float gmul, const float* __restrict__ row_scale, int ld, int n_rows, float b1,
                            float b2, float eps, float c1, float c2, size_t count, __half* __restrict__ z_h) {
  adam_body<false>(z, m, s, g, n_parts, gmul, row_scale, ld, n_rows, b1, b2, eps, c1, c2, count, z_h, 0.f);
}

__global__ void adam_prior_kernel(float* __restrict__ z, float* __restrict__ m, float* __restrict__ s,
                                  const float* __restrict__ g, int n_parts, float gmul, const float* __restrict__ row_scale,
                                  int ld, int n_rows, float b1, float b2, float eps, float c1, float c2, size_t count,
                                  __half* __restrict__ z_h, float two_lambda) {
  adam_body<true>(z, m, s, g, n_parts, gmul, row_scale, ld, n_rows, b1, b2, eps, c1, c2, count, z_h, two_lambda);
}

// prune_gather_kernel with Adam's second state: the survivors' z, m (in v), s and (fp16 path, z_h != NULL) z_h into the
// next region, row r from row src[r] of the current region; the tile-padding rows n_rows .. n_pad - 1 are zeroed.  One
// launch, as the momentum call's gather.
__global__ void prune_gather_adam_kernel(const float* __restrict__ z, const float* __restrict__ v, const float* __restrict__ s,
                                         const __half* __restrict__ z_h, const int* __restrict__ src, int n_rows, int n_pad,
                                         int ld, float* __restrict__ z_out, float* __restrict__ v_out,
                                         float* __restrict__ s_out, __half* __restrict__ z_h_out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n_pad * ld) return;
  const int row = (int)(i / ld), col = (int)(i % ld);
  float zz = 0.f, vv = 0.f, ss = 0.f;
  __half hh = __float2half_rn(0.f);
  if (row < n_rows) {
    const size_t j = (size_t)src[row] * ld + col;
    zz = z[j];
    vv = v[j];
    ss = s[j];
    if (z_h != nullptr) hh = z_h[j];
  }
  z_out[i] = zz;
  v_out[i] = vv;
  s_out[i] = ss;
  if (z_h_out != nullptr) z_h_out[i] = hh;
}

}  // namespace dgan
