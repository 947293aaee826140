// Sparse deviations (the *_sparse_dev entries; Sparse-Gen, Dhar, Grover & Ermon 2018): each restart row fits
// u = G(z) + nu with an l1 penalty on nu.  The measured loop runs unchanged around four kernels:
//
//   sdev_update_kernel        after each forward: nu <- S_tau(fmaf(-eta, g, nu)) from the previous step's g (t > 0), or
//                             nu = +0 (t = 0); then u = y + nu.  The measurement product (or sdev_image_resid_kernel)
//                             reads u in place of y.
//   sdev_image_resid_kernel   the image loss's data term on u as the identity operator: the loss parts of the CSR
//                             measurement product and g = dy of its adjoint product, on the identity CSR (m = H*W*C).
//   sdev_term_kernel          J = loss + l1 * sum |nu| per row, after the loss finish (iteration L - 1, prune points).
//   sdev_gather_kernel        a prune point's survivors' nu and g into the next region.
//   sdev_select_kernel        dev_out: the nu row of each image's arg-min restart (select_kernel's rule).
//
// g is the fp32 dy = dD/du the measured loop builds before the cotangent entry (w.dym); nothing else reads or writes
// nu or u.  Every kernel works on the real rows only (rows < n_rows) and in fp32 on both precisions.
#pragma once
#include "common.cuh"
#include "kernels_measured.cuh"

namespace dgan {

// One thread per 4 consecutive elements of the real rows' [n_rows][hwc] (hwc % 4 == 0):
//   apply: a = fmaf(-eta, g, nu); nu = |a| > tau ? a - copysignf(tau, a) : +0       (the ISTA step, S_tau soft threshold)
//   else:  nu = +0                                                                   (iteration 0)
//   u = y + nu                                                                       (one fp32 add)
__global__ void __launch_bounds__(256)
sdev_update_kernel(const float* __restrict__ y, const float* __restrict__ g, float* __restrict__ nu,
                   float* __restrict__ u, size_t n4, int apply, float eta, float tau) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n4) return;
  const float4 yy = reinterpret_cast<const float4*>(y)[i];
  float4 vv = make_float4(0.f, 0.f, 0.f, 0.f);
  if (apply) {
    const float4 gg = reinterpret_cast<const float4*>(g)[i];
    const float4 nn = reinterpret_cast<const float4*>(nu)[i];
    auto shrink = [&](float gi, float ni) -> float {
      const float a = fmaf(-eta, gi, ni);
      return fabsf(a) > tau ? __fsub_rn(a, copysignf(tau, a)) : 0.f;
    };
    vv = make_float4(shrink(gg.x, nn.x), shrink(gg.y, nn.y), shrink(gg.z, nn.z), shrink(gg.w, nn.w));
  }
  reinterpret_cast<float4*>(nu)[i] = vv;
  reinterpret_cast<float4*>(u)[i] = make_float4(__fadd_rn(yy.x, vv.x), __fadd_rn(yy.y, vv.y), __fadd_rn(yy.z, vv.z),
                                                __fadd_rn(yy.w, vv.w));
}

// The image data term on u [n_rows][hwc] against x [batch][hwc] (row n's image n / R), optional weights w [batch][hwc]
// (NULL: unweighted), as the identity operator with m = hwc measurements zero-padded to m_ld (a multiple of 64) columns:
// grid (n_rows, ceil(m_ld / 4 / 256)), 256 threads, thread q owns columns 4q .. 4q + 3 of row blockIdx.x.  Per column p:
//   a = u + 0; r = a - x; c = r (HUBER: |r| > delta ? copysignf(delta, r) : r); columns >= hwc have r = 0
//   loss term fmaf(w c, c, .) (HUBER: fmaf(w c, 2 r - c, .)), w c = c when unweighted
//   g[n][p] = (w c + 0) * s,  s = 2 / m
// The loss parts are the CSR measurement product's: per quad an fmaf chain from +0 in column order, then a butterfly over
// the 16 quads of a 64-column tile at offsets 1, 2, 4, 8 into loss_part[tile * loss_ld + n].  The "+ 0" adds are the
// identity CSR's fmaf(v, 1, +0) chains, so unweighted calls are bit-identical to the CSR entry on the identity matrix.
template <bool HUBER, bool WEIGHTED>
__global__ void __launch_bounds__(256)
sdev_image_resid_kernel(const float* __restrict__ u, const float* __restrict__ x, const float* __restrict__ w, int hwc,
                        int m_ld, int R, float delta, float s, float* __restrict__ g, float* __restrict__ loss_part,
                        int loss_ld) {
  const int n = blockIdx.x;
  const int q = blockIdx.y * blockDim.x + threadIdx.x;
  const bool active = q < m_ld / 4;          // m_ld / 4 is a multiple of 16: a 16-lane group is all in or all out
  float rsum = 0.f;
  if (active && 4 * q < hwc) {
    const size_t off = (size_t)n * hwc + 4 * q, xoff = (size_t)(n / R) * hwc + 4 * q;
    const float4 uu = *reinterpret_cast<const float4*>(u + off);
    const float4 xx = *reinterpret_cast<const float4*>(x + xoff);
    float4 ww = make_float4(1.f, 1.f, 1.f, 1.f);
    if (WEIGHTED) ww = *reinterpret_cast<const float4*>(w + xoff);
    const float ua[4] = {uu.x, uu.y, uu.z, uu.w}, xa[4] = {xx.x, xx.y, xx.z, xx.w}, wa[4] = {ww.x, ww.y, ww.z, ww.w};
    float ga[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float r = __fsub_rn(__fadd_rn(ua[j], 0.f), xa[j]);
      const float c = HUBER ? (fabsf(r) > delta ? copysignf(delta, r) : r) : r;
      const float wc = WEIGHTED ? __fmul_rn(wa[j], c) : c;
      rsum = HUBER ? fmaf(wc, 2.f * r - c, rsum) : fmaf(wc, c, rsum);
      ga[j] = __fmul_rn(__fadd_rn(wc, 0.f), s);
    }
    *reinterpret_cast<float4*>(g + off) = make_float4(ga[0], ga[1], ga[2], ga[3]);
  }
#pragma unroll
  for (int o = 1; o < 16; o <<= 1) rsum += __shfl_xor_sync(0xffffffffu, rsum, o);
  if (active && (q & 15) == 0) loss_part[(size_t)(q / 16) * loss_ld + n] = rsum;
}

// J per real row: loss[n] = loss[n] + l1 * S with S = sum_p |nu[n][p]| over p < hwc, one warp per row: lane l adds
// |nu[n][l]|, |nu[n][l + 32]|, ... in ascending p from +0, then a butterfly over the 32 lanes at offsets 16, 8, 4, 2, 1.
// Launched after the loss finish, so J = (D [+ p_z]) + p_nu.  256 threads: 8 rows per block.
__global__ void __launch_bounds__(256)
sdev_term_kernel(const float* __restrict__ nu, int hwc, int n_rows, float l1, float* __restrict__ loss) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= n_rows) return;                   // uniform per warp
  const float* row = nu + (size_t)n * hwc;
  float acc = 0.f;
  for (int p = lane; p < hwc; p += 32) acc = __fadd_rn(acc, fabsf(row[p]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = __fadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
  if (lane == 0) loss[n] = __fadd_rn(loss[n], __fmul_rn(l1, acc));
}

// A prune point's survivors: row r of nu_out and g_out [n_rows][hwc] from row src[r] of nu and g, 4 floats per thread
// (hwc % 4 == 0).  g is the pending update's gradient: the next region's first step applies it.
__global__ void __launch_bounds__(256)
sdev_gather_kernel(const float* __restrict__ nu, const float* __restrict__ g, const int* __restrict__ src, int n_rows,
                   int hwc, float* __restrict__ nu_out, float* __restrict__ g_out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int q4 = hwc / 4;
  if (i >= (size_t)n_rows * q4) return;
  const size_t r = i / q4, c = i % q4;
  const size_t from = (size_t)src[r] * q4 + c;
  reinterpret_cast<float4*>(nu_out)[i] = reinterpret_cast<const float4*>(nu)[from];
  reinterpret_cast<float4*>(g_out)[i] = reinterpret_cast<const float4*>(g)[from];
}

// dev_out [batch][hwc] (16-byte aligned): the nu row of each image's arg-min restart among its R rows of loss, chosen by
// select_kernel's rule (strictly lower loss wins, so the lowest index wins ties).  One block per image.
__global__ void __launch_bounds__(256)
sdev_select_kernel(const float* __restrict__ loss, const float* __restrict__ nu, int R, int hwc, float* __restrict__ out) {
  const int img = blockIdx.x;
  __shared__ int best_s;
  if (threadIdx.x == 0) {
    int best = 0;
    float bl = loss[(size_t)img * R];
    for (int r = 1; r < R; ++r) {
      const float l = loss[(size_t)img * R + r];
      if (l < bl) { bl = l; best = r; }
    }
    best_s = best;
  }
  __syncthreads();
  const float* src = nu + ((size_t)img * R + best_s) * hwc;
  float* dst = out + (size_t)img * hwc;
  for (int e = threadIdx.x * 4; e < hwc; e += blockDim.x * 4)
    *reinterpret_cast<float4*>(dst + e) = *reinterpret_cast<const float4*>(src + e);
}

}  // namespace dgan
