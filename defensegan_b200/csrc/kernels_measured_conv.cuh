// The measured loss with a convolution operator (dgan_reconstruct_measured_conv): for an image x [H][W][C] (NHWC) and a
// kernel k [kh][kw] per image, stride s and zero padding (ph, pw), the per-channel cross-correlation
//
//   (A x)[(u Wo + v) C + c] = sum over in-bounds (a, b) of k[a][b] x[s u + a - ph][s v + b - pw][c]
//
// with Ho = (H + 2 ph - kh) / s + 1, Wo = (W + 2 pw - kw) / s + 1 and m = Ho Wo C.  The same two products as
// kernels_measured.cuh and the same outputs, with no matrix: each reads its operand (G or r) once and writes its result
// once.
//
//   measurement product   r[n][j]  = (A_{n / R} G[n])_j - y[n / R][j]                 (MEAS_RESID[_HUBER]: loss parts)
//   adjoint product       dy[n][p] = (2/m) sum_j A_{n / R}[j][p] r[n][j]               (MEAS_SCALE)
//
// Arithmetic: fp32 FFMA on the CUDA cores on both precisions, in the order of the CSR products (kernels_measured_csr.cuh)
// on the matrix the stencil represents, so the two calls are bit-identical:
//   - measurement output j: one fmaf chain from +0 over the in-bounds taps in ascending (a, b) - ascending input column,
//     the CSR row's order - then measured_csr_body's epilogue;
//   - loss parts: per 4 consecutive columns fmaf(v, v, sum) in order from +0, then a butterfly over the 16 quads of each
//     64-column tile at offsets 1, 2, 4, 8; padded columns j >= m give r = 0;
//   - adjoint output p = (i, j, c): one chain from +0 over the output pixels (u, v) whose window covers (i, j), in
//     ascending order - the staged transpose's ascending row-of-A order - then the multiply by 2/m.
// A tap whose value is 0 adds a term where the CSR has none: the chains start at +0 and never hold -0, and G and r are
// finite, so no bit changes.
//
// Work: one CTA of 256 threads per (latent row, chunk of kConvCols consecutive outputs).  The CTA stages the image's
// kernel and the rows of the operand its chunk reads - output bands with their input halo - in dynamic shared memory
// (conv_meas_span / conv_adj_span: a few KB for a blur, at most one operand row), so several CTAs share an SM.
//
// Staging (once per call, outside the captured loop; conv_stage_kernel): the kernels [batch][kh][kw] and the
// measurements, ym [batch][m_ld] = y [batch][m] with zero columns.
#pragma once
#include "common.cuh"
#include "kernels_measured.cuh"

namespace dgan {

constexpr int kConvThreads = 256;
constexpr int kConvCols = 2048;      // outputs per CTA of the products (a multiple of the loss tile, 64)

// The image and the operator: H, W, C of the handle, the kernel's kh x kw, padding, stride and the output size.
struct ConvGeom {
  int H, W, C, kh, kw, ph, pw, s, Ho, Wo;
};

// Floats of shared memory before the staged operand rows: the kernel's taps, rounded up to 16 bytes.
__host__ __device__ inline int conv_taps_ld(const ConvGeom& g) { return (g.kh * g.kw + 3) & ~3; }

// The input rows [*lo, *hi] the measurement outputs [j0, j1) read (j0 < j1 <= m); empty (*hi < *lo) when j0 >= j1.
__host__ __device__ inline void conv_meas_span(const ConvGeom& g, int j0, int j1, int* lo, int* hi) {
  *lo = 0; *hi = -1;
  if (j0 >= j1) return;
  const int woc = g.Wo * g.C;
  *lo = max(0, g.s * (j0 / woc) - g.ph);
  *hi = min(g.H - 1, g.s * ((j1 - 1) / woc) - g.ph + g.kh - 1);
}

// The output rows u in [*lo, *hi] whose windows cover input row i (empty when *hi < *lo).
__host__ __device__ inline void conv_rows_covering(const ConvGeom& g, int i, int* lo, int* hi) {
  const int x = i + g.ph - g.kh + 1;
  *lo = x > 0 ? (x + g.s - 1) / g.s : 0;
  *hi = min(g.Ho - 1, (i + g.ph) / g.s);
}

// The output rows [*lo, *hi] the adjoint outputs [p0, p1) read (p0 < p1 <= H*W*C); possibly empty.
__host__ __device__ inline void conv_adj_span(const ConvGeom& g, int p0, int p1, int* lo, int* hi) {
  const int wc = g.W * g.C;
  int l2, h1;
  conv_rows_covering(g, p0 / wc, lo, &h1);
  conv_rows_covering(g, (p1 - 1) / wc, &l2, hi);
}

// dst[0..n) = src[0..n), 16 bytes at a time when both are 16-byte aligned
__device__ __forceinline__ void conv_stage_span(float* __restrict__ dst, const float* __restrict__ src, int n) {
  const int tid = threadIdx.x;
  if ((((uintptr_t)src | (uintptr_t)dst) & 15) == 0) {
    const int nq = n / 4;
    for (int i = tid; i < nq; i += kConvThreads)
      reinterpret_cast<float4*>(dst)[i] = reinterpret_cast<const float4*>(src)[i];
    for (int i = 4 * nq + tid; i < n; i += kConvThreads) dst[i] = src[i];
  } else {
#pragma unroll 4
    for (int i = tid; i < n; i += kConvThreads) dst[i] = src[i];
  }
}

// The measurement product of M latent rows of G (X, row stride ldx = H*W*C) through image n / R's kernel (ck
// [batch][kh][kw]): out [M][ldo] over N = m_ld columns (m real), ym at row stride ldo, loss_part[(col / 64) * loss_ld +
// row] the 64-column tile's sum of out^2 (MEAS_RESID) or of meas_huber's term at delta = s (MEAS_RESID_HUBER, out = c).
// Grid: M * ceil(N / kConvCols) CTAs, row-major over (row, chunk).
template <int EPI>
__device__ __forceinline__ void
measured_conv_body(const float* __restrict__ X, int ldx, ConvGeom g, const float* __restrict__ ck, int N, int m,
                   float* __restrict__ out, int ldo, const float* __restrict__ ym, int R, float s,
                   float* __restrict__ loss_part, int loss_ld) {
  extern __shared__ __align__(16) float csm[];
  const int tid = threadIdx.x;
  const int n_chunks = (N + kConvCols - 1) / kConvCols;
  const int row = blockIdx.x / n_chunks, chunk = blockIdx.x % n_chunks;
  const int j0 = chunk * kConvCols, j1 = min(N, j0 + kConvCols);
  const int taps = g.kh * g.kw, wc = g.W * g.C, woc = g.Wo * g.C;
  int lo, hi;
  conv_meas_span(g, j0, min(j1, m), &lo, &hi);
  float* kt = csm;
  float* xs = csm + conv_taps_ld(g);
  const float* kg = ck + (size_t)(row / R) * taps;
  for (int t = tid; t < taps; t += kConvThreads) kt[t] = kg[t];
  if (hi >= lo) conv_stage_span(xs, X + (size_t)row * ldx + (size_t)lo * wc, (hi - lo + 1) * wc);
  __syncthreads();

  const int nq = (j1 - j0) / 4;
  // every thread runs every round, so the loss butterfly's shuffles see full warps (nq % 16 == 0)
  for (int qb = 0; qb < nq; qb += kConvThreads) {
    const int q = j0 / 4 + qb + tid;
    const bool active = qb + tid < nq;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    if (active) {
      // the four outputs' window origins and in-bounds tap ranges; the tap loop is shared, each output adds only its
      // in-bounds taps, in ascending (a, b)
      int ib[4], jb[4], cc[4];
      bool real[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * q + e;
        real[e] = j < m;
        const int u = j / woc, rem = j - u * woc, v = rem / g.C;
        cc[e] = rem - v * g.C;
        ib[e] = g.s * u - g.ph;
        jb[e] = g.s * v - g.pw;
      }
      for (int a = 0; a < g.kh; ++a) {
        bool row_in[4];
        int base[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int i = ib[e] + a;
          row_in[e] = real[e] && i >= 0 && i < g.H;
          base[e] = (i - lo) * wc + cc[e];
        }
        for (int b = 0; b < g.kw; ++b) {
          const float k = kt[a * g.kw + b];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int jj = jb[e] + b;
            if (row_in[e] && jj >= 0 && jj < g.W) acc[e] = fmaf(xs[base[e] + jj * g.C], k, acc[e]);
          }
        }
      }
    }
    float rsum = 0.f;
    if (active) {
      const int col = 4 * q;
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (EPI == MEAS_RESID) {
          v[e] = acc[e] - ym[(size_t)(row / R) * ldo + col + e];
          rsum = fmaf(v[e], v[e], rsum);
        } else {
          const float rj = acc[e] - ym[(size_t)(row / R) * ldo + col + e];
          v[e] = fabsf(rj) > s ? copysignf(s, rj) : rj;
          rsum = fmaf(v[e], 2.f * rj - v[e], rsum);
        }
      }
      *reinterpret_cast<float4*>(out + (size_t)row * ldo + col) = make_float4(v[0], v[1], v[2], v[3]);
    }
#pragma unroll
    for (int o = 1; o < 16; o <<= 1) rsum += __shfl_xor_sync(0xffffffffu, rsum, o);
    if (active && (q & 15) == 0) loss_part[(size_t)(q / 16) * loss_ld + row] = rsum;
  }
}

__global__ void __launch_bounds__(kConvThreads)
measured_conv_kernel(const float* __restrict__ X, int ldx, ConvGeom g, const float* __restrict__ ck, int N, int m,
                     float* __restrict__ out, int ldo, const float* __restrict__ ym, int R, float s,
                     float* __restrict__ loss_part, int loss_ld) {
  measured_conv_body<MEAS_RESID>(X, ldx, g, ck, N, m, out, ldo, ym, R, s, loss_part, loss_ld);
}

// The measurement product with the Huber residual (MEAS_RESID_HUBER) at delta = s
__global__ void __launch_bounds__(kConvThreads)
measured_conv_huber_kernel(const float* __restrict__ X, int ldx, ConvGeom g, const float* __restrict__ ck, int N, int m,
                           float* __restrict__ out, int ldo, const float* __restrict__ ym, int R, float s,
                           float* __restrict__ loss_part, int loss_ld) {
  measured_conv_body<MEAS_RESID_HUBER>(X, ldx, g, ck, N, m, out, ldo, ym, R, s, loss_part, loss_ld);
}

// The adjoint product of M latent rows of r (X, row stride ldx = m_ld) through image n / R's kernel: out [M][ldo] over
// the N = H*W*C pixels, out = s * acc.  Grid: M * ceil(N / kConvCols) CTAs, row-major over (row, chunk).
__global__ void __launch_bounds__(kConvThreads)
measured_conv_adjoint_kernel(const float* __restrict__ X, int ldx, ConvGeom g, const float* __restrict__ ck, int N,
                             float* __restrict__ out, int ldo, int R, float s) {
  extern __shared__ __align__(16) float csm[];
  const int tid = threadIdx.x;
  const int n_chunks = (N + kConvCols - 1) / kConvCols;
  const int row = blockIdx.x / n_chunks, chunk = blockIdx.x % n_chunks;
  const int p0 = chunk * kConvCols, p1 = min(N, p0 + kConvCols);
  const int taps = g.kh * g.kw, wc = g.W * g.C, woc = g.Wo * g.C;
  int lo, hi;
  conv_adj_span(g, p0, p1, &lo, &hi);
  float* kt = csm;
  float* rs = csm + conv_taps_ld(g);
  const float* kg = ck + (size_t)(row / R) * taps;
  for (int t = tid; t < taps; t += kConvThreads) kt[t] = kg[t];
  if (hi >= lo) conv_stage_span(rs, X + (size_t)row * ldx + (size_t)lo * woc, (hi - lo + 1) * woc);
  __syncthreads();

  const int nq = (p1 - p0) / 4;
  for (int qi = tid; qi < nq; qi += kConvThreads) {
    const int q = p0 / 4 + qi;
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int p = 4 * q + e;
      const int i = p / wc, rem = p - i * wc, j = rem / g.C, c = rem - j * g.C;
      int u0, u1, v0, v1;
      conv_rows_covering(g, i, &u0, &u1);
      {
        const int x = j + g.pw - g.kw + 1;
        v0 = x > 0 ? (x + g.s - 1) / g.s : 0;
        v1 = min(g.Wo - 1, (j + g.pw) / g.s);
      }
      float acc = 0.f;
      for (int u = u0; u <= u1; ++u) {
        const float* rr = rs + (u - lo) * woc + c;
        const float* kr = kt + (i + g.ph - g.s * u) * g.kw + j + g.pw;
        for (int vv = v0; vv <= v1; ++vv) acc = fmaf(rr[vv * g.C], kr[-g.s * vv], acc);
      }
      v[e] = acc * s;
    }
    *reinterpret_cast<float4*>(out + (size_t)row * ldo + 4 * q) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// One grid over two index ranges: ck [batch][taps] = k, and ym [batch][m_ld] = y [batch][m] with zero columns.
__global__ void conv_stage_kernel(const float* __restrict__ k, const float* __restrict__ y, int batch, int taps, int m,
                                  int m_ld, float* __restrict__ ck, float* __restrict__ ym) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (size_t)batch * taps) ck[i] = k[i];
  if (i < (size_t)batch * m_ld) {
    const int b = (int)(i / m_ld), j = (int)(i % m_ld);
    ym[i] = j < m ? y[(size_t)b * m + j] : 0.f;
  }
}

}  // namespace dgan
