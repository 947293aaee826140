// The two measurement products of dgan_reconstruct_measured, the projection onto the generator's range from linear
// measurements y = A x (loss_n = (1/m) ||A G(z_n) - y[n / R]||^2):
//
//   measurement product   r[n][j]  = sum_k G[n][k] A[j][k] - y[n / R][j]      (MEAS_RESID: the per-row sum of r^2 too)
//   adjoint product       dy[n][p] = (2/m) sum_j r[n][j] At[p][j]             (MEAS_SCALE)
//
// Both are C[M][N] = s * sum_k X[m][k] W[n][k] with both operands K-major (row stride ldx, ldw), so one kernel serves them:
// M = the latent rows, N = m or H*W*C, K = H*W*C or m.  The call stores A as [m_ld][H*W*C] and its transpose At as
// [H*W*C][m_ld], and y as [batch][m_ld], with m_ld = m rounded up to the N tile and the padding exact zeros: padded rows
// of A give r = 0 - 0 = 0 exactly, and padded columns of r meet zero columns of At, so no padding is ever observed.
//
// TC (fp16 path): TF32 mma.sync m16n8k8 on the tensor cores, fp32 accumulate.  TF32 keeps fp32's range, so neither A nor
// r needs a scale; operands are rounded to TF32 (cvt.rna) as they are staged.  Not TC (fp32 path): fp32 FFMA on the CUDA
// cores, the reference's arithmetic.  (bsgemm_f32_kernel cannot serve the adjoint product: its C_out must be a multiple
// of 64, and H*W*C = 784 on MNIST is not.)
// Block: 128 rows x 64 columns, K in slices of 16 (K % 16 == 0: H*W*C and m_ld are), staged through double-buffered
// shared memory with the next slice prefetched into registers.  Rows >= M and columns >= N of either operand read as 0
// and are not stored.  The row sums of r^2 are reduced in a fixed order (one partial per N tile, loss_part
// [N / 64][loss_ld]), so every bit is reproducible.  Plain launches (no PDL).
#pragma once
#include "common.cuh"

namespace dgan {

constexpr int kMeasTileM = 128, kMeasTileN = 64, kMeasTileK = 16;
// MEAS_RESID_HUBER (dgan_reconstruct_measured_huber): the Huber loss at delta = s > 0 instead of the squared error, see
// meas_huber.
enum MeasEpi : int { MEAS_RESID = 0, MEAS_SCALE = 1, MEAS_RESID_HUBER = 2 };

// The Huber residual of r at delta: r is replaced by c = |r| > delta ? copysign(delta, r) : r (what the adjoint product
// reads) and its loss term c (2 r - c) returned.  When |r| <= delta, c == r and the term is r * r to the bit.
__device__ __forceinline__ float meas_huber(float& r, float delta) {
  const float c = fabsf(r) > delta ? copysignf(delta, r) : r;
  const float t = 2.f * r - c;
  r = c;
  return c * t;
}

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}

__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// MEAS_RESID: out = acc - ym[row / R][col] (ym at row stride ldo), loss_part[blockIdx.y * loss_ld + row] = the block's
// sum of out^2 over its columns.  MEAS_RESID_HUBER: the same with out and its square replaced by meas_huber's c and term
// at delta = s (measured_gemm_huber_kernel).  MEAS_SCALE: out = s * acc.
template <bool TC, int EPI>
__device__ __forceinline__ void
measured_gemm_body(const float* __restrict__ X, int ldx, int M, const float* __restrict__ W, int ldw, int N, int K,
                   float* __restrict__ out, int ldo, const float* __restrict__ ym, int R, float s,
                   float* __restrict__ loss_part, int loss_ld) {
  // TC: [buf][row][k] at stride 20 (conflict-free fragment reads); not TC: [buf][k][row] at strides 132 and 68
  constexpr int kLd = kMeasTileK + 4;
  constexpr int kStage = TC ? (kMeasTileM + kMeasTileN) * kLd : kMeasTileK * (kMeasTileM + 4 + kMeasTileN + 4);
  __shared__ __align__(16) float sm[2 * kStage];
  __shared__ float red[2][kMeasTileM];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * kMeasTileM, n0 = blockIdx.y * kMeasTileN;
  const int lr = tid >> 2, lk = (tid & 3) * 4;     // loads: rows lr, lr + 64 of X, row lr of W; 4 consecutive k
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 rx0, rx1, rw;
  auto gload = [&](int k0) {
    rx0 = m0 + lr < M ? *reinterpret_cast<const float4*>(X + (size_t)(m0 + lr) * ldx + k0 + lk) : zero4;
    rx1 = m0 + lr + 64 < M ? *reinterpret_cast<const float4*>(X + (size_t)(m0 + lr + 64) * ldx + k0 + lk) : zero4;
    rw = n0 + lr < N ? *reinterpret_cast<const float4*>(W + (size_t)(n0 + lr) * ldw + k0 + lk) : zero4;
  };
  auto sstore = [&](int buf) {
    float* st = sm + buf * kStage;
    if (TC) {
      uint32_t* xs = reinterpret_cast<uint32_t*>(st);
      uint32_t* ws = xs + kMeasTileM * kLd;
      *reinterpret_cast<uint4*>(xs + lr * kLd + lk) = make_uint4(to_tf32(rx0.x), to_tf32(rx0.y), to_tf32(rx0.z), to_tf32(rx0.w));
      *reinterpret_cast<uint4*>(xs + (lr + 64) * kLd + lk) = make_uint4(to_tf32(rx1.x), to_tf32(rx1.y), to_tf32(rx1.z), to_tf32(rx1.w));
      *reinterpret_cast<uint4*>(ws + lr * kLd + lk) = make_uint4(to_tf32(rw.x), to_tf32(rw.y), to_tf32(rw.z), to_tf32(rw.w));
    } else {
      float* xs = st;                                  // [k][132]
      float* ws = st + kMeasTileK * (kMeasTileM + 4);  // [k][68]
      const float a0[4] = {rx0.x, rx0.y, rx0.z, rx0.w}, a1[4] = {rx1.x, rx1.y, rx1.z, rx1.w}, b[4] = {rw.x, rw.y, rw.z, rw.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        xs[(lk + j) * (kMeasTileM + 4) + lr] = a0[j];
        xs[(lk + j) * (kMeasTileM + 4) + lr + 64] = a1[j];
        ws[(lk + j) * (kMeasTileN + 4) + lr] = b[j];
      }
    }
  };

  // TC: warp (wm, wn) holds rows wm*32 .. +32 and columns wn*32 .. +32 as 2 x 4 m16n8 tiles.
  // Not TC: thread (ty, tx) holds rows ty*8 .. +8 and columns tx*4 .. +4.
  const int lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int wm = warp & 3, wn = warp >> 2;
  const int ty = tid >> 4, tx = tid & 15;
  float acc[32];                                     // TC: [mi][ni][4] fragments; not TC: [i][j]
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;

  const int T = K / kMeasTileK;
  if (T > 0) { gload(0); sstore(0); }
  __syncthreads();
  for (int it = 0; it < T; ++it) {
    const int buf = it & 1;
    if (it + 1 < T) gload((it + 1) * kMeasTileK);
    const float* st = sm + buf * kStage;
    if (TC) {
      const uint32_t* xs = reinterpret_cast<const uint32_t*>(st);
      const uint32_t* ws = xs + kMeasTileM * kLd;
#pragma unroll
      for (int k8 = 0; k8 < kMeasTileK; k8 += 8) {
        uint32_t a[2][4];
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
          const uint32_t* p = xs + (wm * 32 + mi * 16 + g) * kLd + k8 + t;
          a[mi][0] = p[0]; a[mi][1] = p[8 * kLd]; a[mi][2] = p[4]; a[mi][3] = p[8 * kLd + 4];
        }
#pragma unroll
        for (int ni = 0; ni < 4; ++ni) {
          const uint32_t* q = ws + (wn * 32 + ni * 8 + g) * kLd + k8 + t;
          const uint32_t b0 = q[0], b1 = q[4];
#pragma unroll
          for (int mi = 0; mi < 2; ++mi) mma_tf32(*reinterpret_cast<float(*)[4]>(&acc[(mi * 4 + ni) * 4]), a[mi], b0, b1);
        }
      }
    } else {
      const float* xs = st;
      const float* ws = st + kMeasTileK * (kMeasTileM + 4);
#pragma unroll
      for (int kk = 0; kk < kMeasTileK; ++kk) {
        const float4 a_lo = *reinterpret_cast<const float4*>(xs + kk * (kMeasTileM + 4) + ty * 8);
        const float4 a_hi = *reinterpret_cast<const float4*>(xs + kk * (kMeasTileM + 4) + ty * 8 + 4);
        const float4 b = *reinterpret_cast<const float4*>(ws + kk * (kMeasTileN + 4) + tx * 4);
        const float av[8] = {a_lo.x, a_lo.y, a_lo.z, a_lo.w, a_hi.x, a_hi.y, a_hi.z, a_hi.w};
        const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i * 4 + j] = fmaf(av[i], bv[j], acc[i * 4 + j]);
      }
    }
    if (it + 1 < T) sstore(buf ^ 1);
    __syncthreads();
  }

  // epilogue on column pairs (TC) or quads (not TC); N is even (m_ld, H*W*C), so a pair is in range when its first is
  auto epi = [&](int row, int col, float& v) -> float {
    if (EPI == MEAS_RESID) {
      v -= ym[(size_t)(row / R) * ldo + col];
      return v * v;
    }
    if (EPI == MEAS_RESID_HUBER) {
      v -= ym[(size_t)(row / R) * ldo + col];
      return meas_huber(v, s);
    }
    v *= s;
    return 0.f;
  };
  if (TC) {
    float rs[2][2] = {{0.f, 0.f}, {0.f, 0.f}};     // [mi][half]: the thread's part of rows wm*32 + mi*16 + g + 8*half
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 4; ++ni)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = m0 + wm * 32 + mi * 16 + g + 8 * h, col = n0 + wn * 32 + ni * 8 + 2 * t;
          float* c = &acc[(mi * 4 + ni) * 4 + 2 * h];
          if (row >= M || col >= N) continue;
          float v0 = c[0], v1 = c[1];
          rs[mi][h] += epi(row, col, v0) + epi(row, col + 1, v1);
          *reinterpret_cast<float2*>(out + (size_t)row * ldo + col) = make_float2(v0, v1);
        }
    if (EPI != MEAS_SCALE) {
#pragma unroll
      for (int mi = 0; mi < 2; ++mi)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v = rs[mi][h];
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          if (t == 0) red[wn][wm * 32 + mi * 16 + g + 8 * h] = v;
        }
      __syncthreads();
      if (tid < kMeasTileM && m0 + tid < M) loss_part[(size_t)blockIdx.y * loss_ld + m0 + tid] = red[0][tid] + red[1][tid];
    }
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int row = m0 + ty * 8 + i, col = n0 + tx * 4;
      float rsum = 0.f;
      if (row < M && col < N) {
        float v[4] = {acc[i * 4], acc[i * 4 + 1], acc[i * 4 + 2], acc[i * 4 + 3]};
#pragma unroll
        for (int j = 0; j < 4; ++j) rsum += epi(row, col + j, v[j]);
        *reinterpret_cast<float4*>(out + (size_t)row * ldo + col) = make_float4(v[0], v[1], v[2], v[3]);
      }
      if (EPI != MEAS_SCALE) {
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) rsum += __shfl_xor_sync(0xffffffffu, rsum, o);
        if (tx == 0 && row < M) loss_part[(size_t)blockIdx.y * loss_ld + row] = rsum;
      }
    }
  }
}

template <bool TC, int EPI>
__global__ void __launch_bounds__(256)
measured_gemm_kernel(const float* __restrict__ X, int ldx, int M, const float* __restrict__ W, int ldw, int N, int K,
                     float* __restrict__ out, int ldo, const float* __restrict__ ym, int R, float s,
                     float* __restrict__ loss_part, int loss_ld) {
  measured_gemm_body<TC, EPI>(X, ldx, M, W, ldw, N, K, out, ldo, ym, R, s, loss_part, loss_ld);
}

// The measurement product with the Huber residual (MEAS_RESID_HUBER) at delta = s
template <bool TC>
__global__ void __launch_bounds__(256)
measured_gemm_huber_kernel(const float* __restrict__ X, int ldx, int M, const float* __restrict__ W, int ldw, int N, int K,
                           float* __restrict__ out, int ldo, const float* __restrict__ ym, int R, float s,
                           float* __restrict__ loss_part, int loss_ld) {
  measured_gemm_body<TC, MEAS_RESID_HUBER>(X, ldx, M, W, ldw, N, K, out, ldo, ym, R, s, loss_part, loss_ld);
}

// The momentum update of tf.train.MomentumOptimizer (as momentum_kernel) with a multiplier per latent row: the gradient of
// row i / ld is g / row_scale[row] (the fp16 path's power-of-two cotangent scales, so the division is exact), or g itself
// when row_scale is NULL (the fp32 path) and on the tile-padding rows (>= n_rows: no scale, and a gradient of 0).  The
// measured loop's d(pre) already carries the 2/m of its loss.  PRIOR (momentum_rows_prior_kernel, the prior entries): the
// gradient of J = D + lambda ||z||^2, g = fmaf(two_lambda, z, g) on the pre-update z after the scale is divided out.
template <bool PRIOR>
__device__ __forceinline__ void momentum_rows_body(float* __restrict__ z, float* __restrict__ v, const float* __restrict__ g,
                                                   int n_parts, const float* __restrict__ row_scale, int ld, int n_rows,
                                                   float lr, float mu, size_t count, __half* __restrict__ z_h,
                                                   float two_lambda) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float gs = g[i];
  for (int p = 1; p < n_parts; ++p) gs += g[i + (size_t)p * count];   // split-K partials, fixed order
  const size_t row = i / ld;
  const float gmul = row_scale != nullptr && row < (size_t)n_rows ? 1.f / row_scale[row] : 1.f;
  const float vv = fmaf(mu, v[i], PRIOR ? fmaf(two_lambda, z[i], gmul * gs) : gmul * gs);
  const float zz = z[i] - lr * vv;
  v[i] = vv;
  z[i] = zz;
  if (z_h != nullptr) z_h[i] = __float2half_rn(zz);
}

__global__ void momentum_rows_kernel(float* __restrict__ z, float* __restrict__ v, const float* __restrict__ g, int n_parts,
                                     const float* __restrict__ row_scale, int ld, int n_rows, float lr, float mu,
                                     size_t count, __half* __restrict__ z_h) {
  momentum_rows_body<false>(z, v, g, n_parts, row_scale, ld, n_rows, lr, mu, count, z_h, 0.f);
}

__global__ void momentum_rows_prior_kernel(float* __restrict__ z, float* __restrict__ v, const float* __restrict__ g,
                                           int n_parts, const float* __restrict__ row_scale, int ld, int n_rows, float lr,
                                           float mu, size_t count, __half* __restrict__ z_h, float two_lambda) {
  momentum_rows_body<true>(z, v, g, n_parts, row_scale, ld, n_rows, lr, mu, count, z_h, two_lambda);
}

}  // namespace dgan
