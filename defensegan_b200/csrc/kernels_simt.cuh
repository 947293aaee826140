// fp32 CUDA-core kernels of the projection loop (DGAN_PREC_FP32) plus the small kernels both
// precisions share (final C_out<=3 layer + loss, momentum update, z init, arg-min select).
#pragma once
#include "common.cuh"

namespace dgan {

// ------------------------------------------------------------------------------------------
// Pixel-graph GEMM, fp32:  out[q][n][co] = epi( sum_{(p,t)} sum_ci in[p][n][ci] * W_t[ci][co] )
//   in  : [P_in ][n_pad][C_in ] fp32        out : [P_out][n_pad][C_out] fp32
//   W_t : wt + t*tile_stride, row ci at stride ldw, C_out contiguous
// Block = 128 rows x 64 channels of one output pixel; 256 threads, 8x4 register tile each;
// K is walked in 16-wide slices over every (pair, ci-slice), double-buffered through shared
// memory with the next slice prefetched into registers while the current one is multiplied.
// Replaces tf.matmul (tflib/ops/linear.py:129-133), tf.nn.conv2d_transpose
// (tflib/ops/deconv2d.py:104-110) and their tf.gradients-generated input gradients.
// ------------------------------------------------------------------------------------------
template <int EPI>
__global__ void __launch_bounds__(256)
bsgemm_f32_kernel(const float* __restrict__ in, int C_in, int n_pad, const float* __restrict__ wt,
                  int tile_stride, int ldw, const int* __restrict__ pair_off,
                  const int2* __restrict__ pairs, float* __restrict__ out, int C_out,
                  const float* __restrict__ bias, int bias_pstride, const float* __restrict__ mask_src) {
  __shared__ __align__(16) float As[2][16][132];
  __shared__ __align__(16) float Bs[2][16][64];

  const int tid = threadIdx.x;
  const int n0 = blockIdx.x * kRowTile;
  const int q = blockIdx.y;
  const int co0 = blockIdx.z * 64;
  const int pbeg = pair_off[q];
  const int kch = C_in >> 4;
  const int T = (pair_off[q + 1] - pbeg) * kch;

  const int ar = tid >> 2, ac = (tid & 3) << 2;   // A slice: rows ar, ar+64; 4 consecutive ci
  const int br = tid >> 4, bc = (tid & 15) << 2;  // B slice: row br; 4 consecutive co
  const int ty = tid >> 4, tx = tid & 15;

  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  float4 ra0, ra1, rb;
  auto gload = [&](int it) {
    const int2 pr = pairs[pbeg + it / kch];
    const int k0 = (it % kch) << 4;
    const float* ap = in + ((size_t)pr.x * n_pad + n0 + ar) * C_in + k0 + ac;
    ra0 = *reinterpret_cast<const float4*>(ap);
    ra1 = *reinterpret_cast<const float4*>(ap + (size_t)64 * C_in);
    rb = *reinterpret_cast<const float4*>(wt + (size_t)pr.y * tile_stride + (size_t)(k0 + br) * ldw + co0 + bc);
  };
  auto sstore = [&](int buf) {
    As[buf][ac + 0][ar] = ra0.x; As[buf][ac + 1][ar] = ra0.y;
    As[buf][ac + 2][ar] = ra0.z; As[buf][ac + 3][ar] = ra0.w;
    As[buf][ac + 0][ar + 64] = ra1.x; As[buf][ac + 1][ar + 64] = ra1.y;
    As[buf][ac + 2][ar + 64] = ra1.z; As[buf][ac + 3][ar + 64] = ra1.w;
    *reinterpret_cast<float4*>(&Bs[buf][br][bc]) = rb;
  };

  if (T > 0) { gload(0); sstore(0); }
  __syncthreads();
  for (int it = 0; it < T; ++it) {
    const int buf = it & 1;
    if (it + 1 < T) gload(it + 1);
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const float4 a_lo = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 8]);
      const float4 a_hi = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 8 + 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
      const float a[8] = {a_lo.x, a_lo.y, a_lo.z, a_lo.w, a_hi.x, a_hi.y, a_hi.z, a_hi.w};
      const float bb[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
    }
    if (it + 1 < T) sstore(buf ^ 1);
    __syncthreads();
  }

  float4 bv = make_float4(0.f, 0.f, 0.f, 0.f);
  if (EPI == EPI_BIAS_RELU || EPI == EPI_BIAS) bv = *reinterpret_cast<const float4*>(bias + (size_t)q * bias_pstride + co0 + tx * 4);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const size_t o = ((size_t)q * n_pad + n0 + ty * 8 + i) * C_out + co0 + tx * 4;
    float4 v = make_float4(acc[i][0] + bv.x, acc[i][1] + bv.y, acc[i][2] + bv.z, acc[i][3] + bv.w);
    if (EPI == EPI_BIAS_RELU) {
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    }
    if (EPI == EPI_MASK) {  // tf.nn.relu gradient: pass where the forward output was > 0
      const float4 m = *reinterpret_cast<const float4*>(mask_src + o);
      v.x = m.x > 0.f ? v.x : 0.f; v.y = m.y > 0.f ? v.y : 0.f;
      v.z = m.z > 0.f ? v.z : 0.f; v.w = m.w > 0.f ? v.w : 0.f;
    }
    *reinterpret_cast<float4*>(out + o) = v;
  }
}

// ------------------------------------------------------------------------------------------
// Final layer forward (5x5/stride-2 transposed conv to C_OUT <= 3 channels) fused with the
// output non-linearity, the per-row squared error and dL/d(pre-activation):
//   pre = b + deconv(h);  y = sigmoid|tanh(pre);  loss_part = sum (y - x)^2 over the band;
//   dpre = (y - x) * act'(pre)        (the 2/(HWC) factor is applied in the z update)
// models/dataset_models.py:68-69,161-163; models/gan.py:411-414.
// Block = (band of 4 output rows, one latent row); the <=4 input rows it needs are staged in
// shared memory (row stride C_in+4 words: conflict-free 16-byte reads), threads are ordered by
// sub-pixel phase so that filter reads are (nearly) warp-uniform broadcasts.
// TIN = float (fp32 path) or __half (tensor-core path activations).  ACT_NONE (dgan_jvp, fp32 path): y = the deconv alone,
// without bias - the tangent of the pre-activation, from the tangent of the input.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 load4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float4 load4(const __half* p) {
  const uint2 u = *reinterpret_cast<const uint2*>(p);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
  const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void store4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void store4(__half* p, float4 v) {
  __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<uint32_t*>(&a);
  u.y = *reinterpret_cast<uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}

constexpr int kBandRows = 4;

// WEIGHTED (dgan_reconstruct_weighted): xw [B][P_out*C_OUT] weights each pixel's squared error, e = xw (y - x): the loss
// takes e (y - x) and dpre = e act'(y).  With xw = 1, e == y - x, so every output is the unweighted kernel's.
// HUBER (dgan_reconstruct_huber; x not null): the Huber loss at delta = huber > 0 instead of the squared error.  With
// d = y - x and c = |d| > delta ? copysign(delta, d) : d, e = xw c (e = c unweighted): the loss takes e (2 d - c) and
// dpre = e act'(y).  When no |d| exceeds delta, c == d and 2 d - c == d, so every output is the squared-error kernel's.
template <typename TIN, int C_OUT, int ACT, bool WEIGHTED, bool HUBER>
__device__ __forceinline__ void
final_fwd_loss_body(const TIN* __restrict__ hin, int n_pad, int h_in, int w_in, int C_in, const float* __restrict__ w,
                    const float* __restrict__ bias, const float* __restrict__ x, int R, int B, float* __restrict__ y,
                    float* __restrict__ dpre, float* __restrict__ loss_part, const float* __restrict__ xw, float huber) {
  extern __shared__ __align__(16) float smem_f[];
  const int ldh = C_in + 4;
  float* ws = smem_f;                                  // [25*C_OUT][C_in]
  float* hs = smem_f + kTaps * C_OUT * C_in;           // [rows*w_in][ldh]
  __shared__ float red[4];

  const int band = blockIdx.y, n = blockIdx.x, tid = threadIdx.x;   // rows on grid.x: no 65535 limit
  const int w_out = 2 * w_in, h_out = 2 * h_in;
  const int i0 = band * kBandRows;
  const int o_lo = max(0, (i0 - 2) >> 1);
  const int o_hi = min(h_in - 1, (i0 + kBandRows) >> 1);
  const int c4n = C_in >> 2;

  for (int e = tid; e < kTaps * C_OUT * c4n; e += 128) store4(ws + e * 4, load4(w + e * 4));
  const int n_pix = (o_hi - o_lo + 1) * w_in;
  for (int e = tid; e < n_pix * c4n; e += 128) {
    const int pix = e / c4n, c4 = e % c4n;
    const size_t g = ((size_t)(o_lo * w_in + pix) * n_pad + n) * C_in + c4 * 4;
    store4(hs + pix * ldh + c4 * 4, load4(hin + g));
  }
  __syncthreads();

  const int half_w = w_in;                 // w_out / 2 columns per phase
  const int items = 4 * 2 * half_w;        // 4 phases x (2 rows x w_out/2 cols)
  const int img = min(n / R, B - 1);
  const int px_per_row = w_out * C_OUT;
  float lsum = 0.f;
  for (int item = tid; item < items; item += 128) {
    const int phase = item / (2 * half_w), k = item % (2 * half_w);
    const int py = phase >> 1, px = phase & 1;
    const int i = i0 + 2 * (k / half_w) + py, j = 2 * (k % half_w) + px;
    if (i >= h_out) continue;
    float acc[C_OUT];
#pragma unroll
    for (int co = 0; co < C_OUT; ++co) acc[co] = ACT == ACT_NONE ? 0.f : bias[co];
    // i = 2o + ka - 1  =>  ka has the parity of i+1
    for (int ka = (i + 1) & 1; ka < 5; ka += 2) {
      const int o = (i + 1 - ka) >> 1;
      if (o < 0 || o >= h_in) continue;
      for (int kb = (j + 1) & 1; kb < 5; kb += 2) {
        const int p = (j + 1 - kb) >> 1;
        if (p < 0 || p >= w_in) continue;
        const float* hp = hs + ((o - o_lo) * w_in + p) * ldh;
        const float* wp = ws + (ka * 5 + kb) * C_OUT * C_in;
        for (int c4 = 0; c4 < c4n; ++c4) {
          const float4 hv = *reinterpret_cast<const float4*>(hp + c4 * 4);
#pragma unroll
          for (int co = 0; co < C_OUT; ++co) {
            const float4 wv = *reinterpret_cast<const float4*>(wp + co * C_in + c4 * 4);
            acc[co] = fmaf(hv.x, wv.x, acc[co]); acc[co] = fmaf(hv.y, wv.y, acc[co]);
            acc[co] = fmaf(hv.z, wv.z, acc[co]); acc[co] = fmaf(hv.w, wv.w, acc[co]);
          }
        }
      }
    }
    const size_t ob = (size_t)n * h_out * px_per_row + (size_t)i * px_per_row + j * C_OUT;
#pragma unroll
    for (int co = 0; co < C_OUT; ++co) {
      float yv, dact;
      if (ACT == ACT_SIGMOID) { yv = 1.f / (1.f + expf(-acc[co])); dact = yv * (1.f - yv); }
      else if (ACT == ACT_TANH) { yv = tanhf(acc[co]); dact = 1.f - yv * yv; }
      else { yv = acc[co]; dact = 1.f; }
      y[ob + co] = yv;
      if (HUBER) {
        const size_t xi = (size_t)img * h_out * px_per_row + (size_t)i * px_per_row + j * C_OUT + co;
        const float d = yv - x[xi];
        const float c = fabsf(d) > huber ? copysignf(huber, d) : d;
        const float e = WEIGHTED ? xw[xi] * c : c;
        lsum = fmaf(e, 2.f * d - c, lsum);
        dpre[ob + co] = e * dact;
      } else if (WEIGHTED) {
        const size_t xi = (size_t)img * h_out * px_per_row + (size_t)i * px_per_row + j * C_OUT + co;
        const float d = yv - x[xi];
        const float e = xw[xi] * d;
        lsum = fmaf(e, d, lsum);
        dpre[ob + co] = e * dact;
      } else if (x != nullptr) {
        const float d = yv - x[(size_t)img * h_out * px_per_row + (size_t)i * px_per_row + j * C_OUT + co];
        lsum = fmaf(d, d, lsum);
        dpre[ob + co] = d * dact;
      }
    }
  }
  if (loss_part != nullptr) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, s);
    if ((tid & 31) == 0) red[tid >> 5] = lsum;
    __syncthreads();
    if (tid == 0) loss_part[(size_t)n * gridDim.y + band] = (red[0] + red[1]) + (red[2] + red[3]);
  }
}

template <typename TIN, int C_OUT, int ACT, bool WEIGHTED = false>
__global__ void __launch_bounds__(128)
final_fwd_loss_kernel(const TIN* __restrict__ hin, int n_pad, int h_in, int w_in, int C_in,
                      const float* __restrict__ w /*[25][C_OUT][C_in]*/, const float* __restrict__ bias,
                      const float* __restrict__ x /*[B][P_out*C_OUT] or null*/, int R, int B,
                      float* __restrict__ y /*[n_pad][P_out*C_OUT]*/,
                      float* __restrict__ dpre /*[n_pad][P_out*C_OUT] or null*/,
                      float* __restrict__ loss_part /*[n_pad][n_bands] or null*/,
                      const float* __restrict__ xw = nullptr /*[B][P_out*C_OUT], WEIGHTED only*/) {
  final_fwd_loss_body<TIN, C_OUT, ACT, WEIGHTED, false>(hin, n_pad, h_in, w_in, C_in, w, bias, x, R, B, y, dpre, loss_part,
                                                        xw, 0.f);
}

// The Huber loss of final_fwd_loss_kernel (x, dpre and loss_part not null; xw too when WEIGHTED)
template <typename TIN, int C_OUT, int ACT, bool WEIGHTED>
__global__ void __launch_bounds__(128)
final_fwd_huber_kernel(const TIN* __restrict__ hin, int n_pad, int h_in, int w_in, int C_in, const float* __restrict__ w,
                       const float* __restrict__ bias, const float* __restrict__ x, int R, int B, float* __restrict__ y,
                       float* __restrict__ dpre, float* __restrict__ loss_part, const float* __restrict__ xw, float huber) {
  final_fwd_loss_body<TIN, C_OUT, ACT, WEIGHTED, true>(hin, n_pad, h_in, w_in, C_in, w, bias, x, R, B, y, dpre, loss_part,
                                                       xw, huber);
}

// ------------------------------------------------------------------------------------------
// Final layer backward-to-input (+ ReLU mask of the layer below):
//   din[p][n][ci] = mask * sum_{ka,kb,co} dpre[n][(2o+ka-1, 2p+kb-1), co] * F[ka,kb,co,ci]
// Thread = (pixel p, latent row n, 4 input channels).  TOUT = float | __half (scaled by gscale).
// ------------------------------------------------------------------------------------------
template <typename TOUT, int C_OUT>
__global__ void __launch_bounds__(256)
final_bwd_kernel(const float* __restrict__ dpre /*[n_pad][P_out*C_OUT]*/, int n_pad, int h_in, int w_in,
                 int C_in, const float* __restrict__ w /*[25][C_OUT][C_in]*/,
                 const TOUT* __restrict__ mask_src /*[P_in][n_pad][C_in] or null*/, float gscale,
                 TOUT* __restrict__ din /*[P_in][n_pad][C_in]*/) {
  extern __shared__ __align__(16) float smem_f[];
  float* ws = smem_f;  // [25*C_OUT][C_in]
  const int tid = threadIdx.x;
  const int c4n = C_in >> 2;
  for (int e = tid; e < kTaps * C_OUT * c4n; e += 256) store4(ws + e * 4, load4(w + e * 4));
  __syncthreads();

  const size_t widx = (size_t)blockIdx.x * 256 + tid;
  const int c4 = (int)(widx % c4n);
  const size_t np = widx / c4n;
  const int n = (int)(np % n_pad);
  const int p_lin = (int)(np / n_pad);
  if (p_lin >= h_in * w_in) return;
  const int o = p_lin / w_in, p = p_lin % w_in;
  const int w_out = 2 * w_in, h_out = 2 * h_in;
  const float* dp = dpre + (size_t)n * h_out * w_out * C_OUT;

  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int ka = 0; ka < 5; ++ka) {
    const int i = 2 * o + ka - 1;
    if (i < 0 || i >= h_out) continue;
#pragma unroll
    for (int kb = 0; kb < 5; ++kb) {
      const int j = 2 * p + kb - 1;
      if (j < 0 || j >= w_out) continue;
#pragma unroll
      for (int co = 0; co < C_OUT; ++co) {
        const float d = dp[(i * w_out + j) * C_OUT + co];
        const float4 wv = *reinterpret_cast<const float4*>(ws + ((ka * 5 + kb) * C_OUT + co) * C_in + c4 * 4);
        acc.x = fmaf(d, wv.x, acc.x); acc.y = fmaf(d, wv.y, acc.y);
        acc.z = fmaf(d, wv.z, acc.z); acc.w = fmaf(d, wv.w, acc.w);
      }
    }
  }
  const size_t g = ((size_t)p_lin * n_pad + n) * C_in + c4 * 4;
  if (mask_src != nullptr) {
    const float4 m = load4(mask_src + g);
    acc.x = m.x > 0.f ? acc.x : 0.f; acc.y = m.y > 0.f ? acc.y : 0.f;
    acc.z = m.z > 0.f ? acc.z : 0.f; acc.w = m.w > 0.f ? acc.w : 0.f;
  }
  acc.x *= gscale; acc.y *= gscale; acc.z *= gscale; acc.w *= gscale;
  store4(din + g, acc);
}

// ------------------------------------------------------------------------------------------
// tf.train.MomentumOptimizer(lr, 0.7), non-Nesterov (models/gan.py:389-391):
//   v <- mu*v + g ;  z <- z - lr*v,   g = gmul * (accumulated J^T dpre)
// gmul carries the 2/(HWC) of the mean (gan.py:411-413) and undoes any fp16 gradient scaling.
// Optionally refreshes the fp16 copy of z that feeds the tensor-core Linear.
// PRIOR (momentum_prior_kernel, the prior entries): the gradient of J = D + lambda ||z||^2, g = fmaf(two_lambda, z, g)
// on the pre-update z, with two_lambda = 2 lambda rounded on the host.
// ------------------------------------------------------------------------------------------
template <bool PRIOR>
__device__ __forceinline__ void momentum_body(float* __restrict__ z, float* __restrict__ v, const float* __restrict__ g,
                                              int n_parts, float gmul, float lr, float mu, size_t count,
                                              __half* __restrict__ z_h, float two_lambda) {
  pdl_launch_dependents();
  pdl_wait();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float gs = g[i];
  for (int p = 1; p < n_parts; ++p) gs += g[i + (size_t)p * count];   // split-K partials, fixed order
  float gg = gmul * gs;
  if (PRIOR) gg = fmaf(two_lambda, z[i], gg);
  const float vv = fmaf(mu, v[i], gg);
  const float zz = z[i] - lr * vv;
  v[i] = vv;
  z[i] = zz;
  if (z_h != nullptr) z_h[i] = __float2half_rn(zz);
}

__global__ void momentum_kernel(float* __restrict__ z, float* __restrict__ v, const float* __restrict__ g, int n_parts,
                                float gmul, float lr, float mu, size_t count, __half* __restrict__ z_h) {
  momentum_body<false>(z, v, g, n_parts, gmul, lr, mu, count, z_h, 0.f);
}

__global__ void momentum_prior_kernel(float* __restrict__ z, float* __restrict__ v, const float* __restrict__ g,
                                      int n_parts, float gmul, float lr, float mu, size_t count, __half* __restrict__ z_h,
                                      float two_lambda) {
  momentum_body<true>(z, v, g, n_parts, gmul, lr, mu, count, z_h, two_lambda);
}

// Philox4x32-10 counter-based generator (public algorithm, Salmon et al. 2011) + Box-Muller.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, ctr.x), lo0 = 0xD2511F53u * ctr.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, ctr.z), lo1 = 0xCD9E8D57u * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += 0x9E3779B9u;
    key.y += 0xBB67AE85u;
  }
  return ctr;
}

// z_hat / momentum-slot initialisation = tf.local_variables_initializer() per batch
// (utils/gan_defense.py:119; models/gan.py:370-377,424-428): z ~ N(0, 1/latent) or z0, v = 0.
// z is [n_pad][ld] with ld >= latent (the padded latent width); rows >= n_rows (tile padding) and columns >= latent are
// zeroed.  Element (row, col) of the draw is value e % 4 of Philox block e / 4 with e = elem_offset + row * latent + col,
// the index of the real [rows][latent] array: the draw does not depend on the padding or on how the batch is chained.
__global__ void init_z_kernel(float* __restrict__ z, float* __restrict__ v, __half* __restrict__ z_h,
                              const float* __restrict__ z0, int n_rows, int n_pad, int latent, int ld,
                              uint64_t seed, float stddev, size_t elem_offset) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n_pad * ld) return;
  const int row = (int)(i / ld), col = (int)(i % ld);
  float val = 0.f;
  if (row < n_rows && col < latent) {
    const size_t e = (size_t)row * latent + col;
    if (z0 != nullptr) {
      val = z0[e];
    } else {
      const size_t g = e + elem_offset, gq = g / 4;
      const int lane = (int)(g % 4);
      const uint4 r = philox4x32_10(make_uint4((uint32_t)gq, (uint32_t)(gq >> 32), 0u, 0u),
                                    make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
      // Box-Muller on (u0, u1) -> values 0, 1 and on (u2, u3) -> values 2, 3
      const uint32_t ra = lane < 2 ? r.x : r.z, rb = lane < 2 ? r.y : r.w;
      const float ua = ((float)ra + 0.5f) * 2.3283064365386963e-10f;
      const float ub = ((float)rb + 0.5f) * 2.3283064365386963e-10f;
      const float m = sqrtf(-2.f * logf(ua)) * stddev;
      float sn, cs;
      sincosf(6.283185307179586f * ub, &sn, &cs);
      val = (lane & 1) ? m * sn : m * cs;
    }
  }
  z[i] = val;
  if (v != nullptr) v[i] = 0.f;
  if (z_h != nullptr) z_h[i] = __float2half_rn(val);
}

// loss[n] = (sum of band partials, fixed order) / (H*W*C)            (models/gan.py:411-413)
// PRIOR (loss_finish_prior_kernel): loss[n] holds the row's prior term p (prior_term_kernel) on entry and receives
// J = D + p, one fp32 add after the rounded D.
template <bool PRIOR>
__device__ __forceinline__ void loss_finish_body(const float* __restrict__ loss_part, int n_bands, size_t stride_n,
                                                 size_t stride_b, float inv_hwc, int n_rows, float* __restrict__ loss) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_rows) return;
  float s = 0.f;
  for (int b = 0; b < n_bands; ++b) s += loss_part[(size_t)n * stride_n + (size_t)b * stride_b];
  if (PRIOR) loss[n] = __fadd_rn(__fmul_rn(s, inv_hwc), loss[n]);
  else loss[n] = s * inv_hwc;
}

__global__ void loss_finish_kernel(const float* __restrict__ loss_part, int n_bands, size_t stride_n, size_t stride_b,
                                   float inv_hwc, int n_rows, float* __restrict__ loss) {
  loss_finish_body<false>(loss_part, n_bands, stride_n, stride_b, inv_hwc, n_rows, loss);
}

__global__ void loss_finish_prior_kernel(const float* __restrict__ loss_part, int n_bands, size_t stride_n,
                                         size_t stride_b, float inv_hwc, int n_rows, float* __restrict__ loss) {
  loss_finish_body<true>(loss_part, n_bands, stride_n, stride_b, inv_hwc, n_rows, loss);
}

// The latent prior's term of each real row (the prior entries): p[n] = lambda * sum_{j < latent} z[n][j]^2, the sum one
// fmaf chain from +0 in ascending column j over the real latent columns (z is [n_pad][ld]).  Launched on the z the data
// term of the same evaluation is computed on; p lands in the workspace's per-row loss, which loss_finish_prior_kernel
// then completes.
__global__ void prior_term_kernel(const float* __restrict__ z, int ld, int latent, int n_rows, float lambda,
                                  float* __restrict__ p) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= n_rows) return;
  const float* zr = z + (size_t)n * ld;
  float acc = 0.f;
  for (int j = 0; j < latent; ++j) acc = fmaf(zr[j], zr[j], acc);
  p[n] = lambda * acc;
}

// Arg-min restart per image and gather (models/gan.py:438-449): lowest index wins ties
// (tf.argmin).  One block per image; the reconstruction row is copied straight into the
// caller's [B, H*W*C] buffer (for multi-GPU runs that is this rank's slot of the all-gather
// buffer, so the collective needs no staging copy).
__global__ void select_kernel(const float* __restrict__ loss, const float* __restrict__ y, int R, int hwc,
                              float* __restrict__ rec, float* __restrict__ loss_min, int32_t* __restrict__ idx) {
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
    if (loss_min != nullptr) loss_min[img] = bl;
    if (idx != nullptr) idx[img] = best;
  }
  __syncthreads();
  const float* src = y + ((size_t)img * R + best_s) * hwc;
  float* dst = rec + (size_t)img * hwc;
  for (int e = threadIdx.x * 4; e < hwc; e += blockDim.x * 4)
    *reinterpret_cast<float4*>(dst + e) = *reinterpret_cast<const float4*>(src + e);
}

}  // namespace dgan

// ==========================================================================================
// Batch-statistics BatchNorm of the generator (opt-in, use_bn=True): tflib/ops/batchnorm.py:80-93
// - the generator always takes the non-fused branch, so BATCH statistics are used even at test
// time (SURVEY F2): mean/var = tf.nn.moments (biased variance) over axes [0] (Linear output: one
// group per flat feature (pixel, channel)) or [0,1,2] (deconv outputs: one group per channel),
// y = (x - mean) * rsqrt(var + 1e-5) * scale + offset, then ReLU.  All latent rows of a call are
// coupled; tile-padding rows (n >= n_rows) are excluded.  Reductions are two-level with a fixed
// order (deterministic).  Activations are [P][n_pad][C]; group index = per_pixel ? p*C + c : c.
// ==========================================================================================
namespace dgan {

constexpr int kBnSplits = 16;

// The BN kernels run on the fp32 path's activations (float) and on the tensor-core path's: pre-activations TP = float
// (written by the GEMM's float epilogue: normalising a value that was first rounded to fp16 would amplify the rounding
// by |pre| / sigma), activations and gradients T = fp16 storage with fp32 arithmetic.
__device__ __forceinline__ float bn_ld(const float* p, size_t i) { return p[i]; }
__device__ __forceinline__ float bn_ld(const __half* p, size_t i) { return __half2float(p[i]); }
__device__ __forceinline__ void bn_st(float* p, size_t i, float v) { p[i] = v; }
__device__ __forceinline__ void bn_st(__half* p, size_t i, float v) {   // saturating, as the tensor-core epilogues
  p[i] = __float2half_rn(fminf(fmaxf(v, -65504.f), 65504.f));
}

// MODE 0: sum x            MODE 1: sum (x - mean)^2
// MODE 2: S1 = sum dy, S2 = sum dy * xhat with dy = dact * (act > 0), xhat = (pre - mean) * inv
// MODE 3: as MODE 2 with dy = dact, unmasked (dgan_jvp: dact holds the tangent of pre)
template <int MODE, typename TP, typename T>
__global__ void __launch_bounds__(256)
bn_reduce_kernel(const TP* __restrict__ x, const T* __restrict__ act, const T* __restrict__ dact,
                 const float* __restrict__ mean_part /*[splits][G]*/, const float* __restrict__ var_part, int P, int n_rows,
                 int n_pad, int C, int per_pixel, float* __restrict__ out0 /*[splits][G]*/, float* __restrict__ out1) {
  __shared__ float red0[8][33], red1[8][33];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int G = per_pixel ? P * C : C;
  const int g = blockIdx.x * 32 + tx;            // C % 32 == 0, so a block never straddles pixels
  const int split = blockIdx.y;
  const long long M = per_pixel ? n_rows : (long long)P * n_rows;
  float mean = 0.f, inv = 0.f;
  if (MODE >= 1) {
    float s = 0.f;
    for (int k = 0; k < kBnSplits; ++k) s += mean_part[(size_t)k * G + g];
    mean = s / (float)M;
  }
  if (MODE >= 2) {
    float s = 0.f;
    for (int k = 0; k < kBnSplits; ++k) s += var_part[(size_t)k * G + g];
    inv = rsqrtf(s / (float)M + 1e-5f);
  }
  const int c = per_pixel ? g % C : g;
  const int p_fixed = per_pixel ? g / C : 0;
  float a0 = 0.f, a1 = 0.f;
  for (long long s = (long long)split * 8 + ty; s < M; s += (long long)kBnSplits * 8) {
    const int p = per_pixel ? p_fixed : (int)(s / n_rows);
    const int n = per_pixel ? (int)s : (int)(s % n_rows);
    const size_t idx = ((size_t)p * n_pad + n) * C + c;
    if (MODE == 0) a0 += bn_ld(x, idx);
    if (MODE == 1) { const float d = bn_ld(x, idx) - mean; a0 = fmaf(d, d, a0); }
    if (MODE >= 2) {
      const float dy = (MODE == 3 || bn_ld(act, idx) > 0.f) ? bn_ld(dact, idx) : 0.f;
      a0 += dy;
      a1 = fmaf(dy, (bn_ld(x, idx) - mean) * inv, a1);
    }
  }
  red0[ty][tx] = a0; red1[ty][tx] = a1;
  __syncthreads();
  if (ty == 0) {
    float s0 = 0.f, s1 = 0.f;
    for (int k = 0; k < 8; ++k) { s0 += red0[k][tx]; s1 += red1[k][tx]; }
    out0[(size_t)split * G + g] = s0;
    if (MODE >= 2) out1[(size_t)split * G + g] = s1;
  }
}

// forward: act = relu((pre - mean) * inv * scale + offset), evaluated the way TF's batch_normalization does:
// x * (inv*scale) + (offset - mean*inv*scale)
template <typename TP, typename T>
__global__ void bn_apply_fwd_kernel(const TP* __restrict__ pre, const float* __restrict__ mean_part,
                                    const float* __restrict__ var_part, const float* __restrict__ scale,
                                    const float* __restrict__ offset, int P, int n_rows, int n_pad, int C, int per_pixel,
                                    T* __restrict__ act) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)P * n_pad * C;
  if (i >= total) return;
  const int c = (int)(i % C);
  const int n = (int)((i / C) % n_pad);
  const int p = (int)(i / ((size_t)C * n_pad));
  if (n >= n_rows) { bn_st(act, i, 0.f); return; }
  const int G = per_pixel ? P * C : C, g = per_pixel ? p * C + c : c;
  const float M = per_pixel ? (float)n_rows : (float)P * (float)n_rows;
  float sm = 0.f, sv = 0.f;
  for (int k = 0; k < kBnSplits; ++k) { sm += mean_part[(size_t)k * G + g]; sv += var_part[(size_t)k * G + g]; }
  const float mean = sm / M, inv = rsqrtf(sv / M + 1e-5f) * scale[g];
  bn_st(act, i, fmaxf(fmaf(bn_ld(pre, i), inv, offset[g] - mean * inv), 0.f));
}

// backward through ReLU + BN:  dpre = scale*inv * (dy - S1/M - xhat * S2/M),  dy = dact * (act > 0)
template <typename TP, typename T>
__global__ void bn_apply_bwd_kernel(const TP* __restrict__ pre, const T* __restrict__ act,
                                    const float* __restrict__ mean_part, const float* __restrict__ var_part,
                                    const float* __restrict__ s1_part, const float* __restrict__ s2_part,
                                    const float* __restrict__ scale, int P, int n_rows, int n_pad, int C, int per_pixel,
                                    T* __restrict__ dact /*in: d(act), out: d(pre)*/) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)P * n_pad * C;
  if (i >= total) return;
  const int c = (int)(i % C);
  const int n = (int)((i / C) % n_pad);
  const int p = (int)(i / ((size_t)C * n_pad));
  if (n >= n_rows) { bn_st(dact, i, 0.f); return; }
  const int G = per_pixel ? P * C : C, g = per_pixel ? p * C + c : c;
  const float M = per_pixel ? (float)n_rows : (float)P * (float)n_rows;
  float sm = 0.f, sv = 0.f, s1 = 0.f, s2 = 0.f;
  for (int k = 0; k < kBnSplits; ++k) {
    sm += mean_part[(size_t)k * G + g]; sv += var_part[(size_t)k * G + g];
    s1 += s1_part[(size_t)k * G + g]; s2 += s2_part[(size_t)k * G + g];
  }
  const float mean = sm / M, inv = rsqrtf(sv / M + 1e-5f);
  const float xhat = (bn_ld(pre, i) - mean) * inv;
  const float dy = bn_ld(act, i) > 0.f ? bn_ld(dact, i) : 0.f;
  bn_st(dact, i, scale[g] * inv * (dy - s1 / M - xhat * (s2 / M)));
}

// tangent through BN + ReLU (dgan_jvp), in place:  t = [act > 0] * scale*inv * (t - S1/M - xhat * S2/M) with S1 = sum t,
// S2 = sum t * xhat over the same rows (and pixels) as the forward statistics (bn_reduce_kernel MODE 3)
template <typename TP, typename T>
__global__ void bn_apply_jvp_kernel(const TP* __restrict__ pre, const T* __restrict__ act,
                                    const float* __restrict__ mean_part, const float* __restrict__ var_part,
                                    const float* __restrict__ s1_part, const float* __restrict__ s2_part,
                                    const float* __restrict__ scale, int P, int n_rows, int n_pad, int C, int per_pixel,
                                    T* __restrict__ t /*in: tangent of pre, out: tangent of act*/) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)P * n_pad * C;
  if (i >= total) return;
  const int c = (int)(i % C);
  const int n = (int)((i / C) % n_pad);
  const int p = (int)(i / ((size_t)C * n_pad));
  if (n >= n_rows || !(bn_ld(act, i) > 0.f)) { bn_st(t, i, 0.f); return; }
  const int G = per_pixel ? P * C : C, g = per_pixel ? p * C + c : c;
  const float M = per_pixel ? (float)n_rows : (float)P * (float)n_rows;
  float sm = 0.f, sv = 0.f, s1 = 0.f, s2 = 0.f;
  for (int k = 0; k < kBnSplits; ++k) {
    sm += mean_part[(size_t)k * G + g]; sv += var_part[(size_t)k * G + g];
    s1 += s1_part[(size_t)k * G + g]; s2 += s2_part[(size_t)k * G + g];
  }
  const float mean = sm / M, inv = rsqrtf(sv / M + 1e-5f);
  const float xhat = (bn_ld(pre, i) - mean) * inv;
  bn_st(t, i, scale[g] * inv * (bn_ld(t, i) - s1 / M - xhat * (s2 / M)));
}

}  // namespace dgan
