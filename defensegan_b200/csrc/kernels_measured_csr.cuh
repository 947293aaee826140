// The measured loss with a sparse operator (dgan_reconstruct_measured_csr): A [m][H*W*C] and its transpose At in CSR, the
// same two products as kernels_measured.cuh and the same outputs, at a cost set by the non-zeros:
//
//   measurement product   r[n][j]  = sum_{e in row j of A} val[e] G[n][col[e]] - y[n / R][j]   (MEAS_RESID: loss parts)
//   adjoint product       dy[n][p] = (2/m) sum_{e in row p of At} r[n][col[e]] At_val[e]           (MEAS_SCALE)
//
// Arithmetic: fp32 FFMA on the CUDA cores on both precisions.  Each output is one fmaf chain from +0 in ascending column
// order, then the epilogue of measured_gemm_kernel<false, EPI>; the dense fp32 kernel's chain runs over every k, and a
// skipped exact zero changes no bit (the accumulator starts at +0 and so is never -0; G and r are finite).  The loss
// parts are the dense epilogue's tree: per 4 consecutive columns fmaf(v, v, sum) in order from +0 (what ptxas makes of
// the dense kernel's quad sum), then a butterfly over the 16 quads of a 64-column tile at offsets 1, 2, 4, 8.  So on the
// fp32 path every output is bit-identical to the dense call's on the same matrix.
//
// Block: 256 threads, kCsrRows latent rows.  The CTA stages its rows of X (G or r) in dynamic shared memory with
// coalesced loads, so X is read from memory once per product; thread t then computes the output quads t, t + 256, ...
// of those rows from shared-memory gathers.  Rows >= M are neither read nor stored.
//
// Staging (once per call, outside the captured loop; no host synchronisation, no allocation): the caller's CSR is
// validated - row_ptr starts at 0, ends at nnz and never decreases, the columns of each row are strictly ascending and
// in [0, H*W*C) - reading only row_ptr[0..m] and col_idx / val[0..nnz).  A valid operator is copied with m_ld - m empty
// rows appended and transposed (within each row of At the entries in ascending row-of-A order, deterministically); an
// invalid one is staged as the empty operator, with NaN measurements, so the call returns NaN instead of reading out of
// bounds.  The products read only the staged buffers.
#pragma once
#include "common.cuh"
#include "kernels_measured.cuh"

namespace dgan {

constexpr int kCsrRows = 4;          // latent rows per CTA of the products
constexpr int kCsrThreads = 256;

// EPI(X A^T) of kCsrRows rows of X [M][K] (row stride ldx) through a CSR operator (rp [N + 1], ci / val) with N output
// columns: out [M][ldo].  MEAS_RESID: out = acc - ym[row / R][col] (ym at row stride ldo) and
// loss_part[(col / 64) * loss_ld + row] = the 64-column tile's sum of out^2 (N % 64 == 0).  MEAS_RESID_HUBER: the same
// with out and its square replaced by meas_huber's c and term at delta = s, as the dense kernel's
// (measured_csr_huber_kernel).  MEAS_SCALE:
// out = s * acc.
// K % 4 == 0, N % 4 == 0, ldx % 4 == 0.  Dynamic shared memory: kCsrRows * K floats.
template <int EPI>
__device__ __forceinline__ void
measured_csr_body(const float* __restrict__ X, int ldx, int M, int K, const int* __restrict__ rp,
                  const int* __restrict__ ci, const float* __restrict__ val, int N, float* __restrict__ out, int ldo,
                  const float* __restrict__ ym, int R, float s, float* __restrict__ loss_part, int loss_ld) {
  extern __shared__ __align__(16) float xs[];        // [kCsrRows][K]
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * kCsrRows;
  const int kq = K / 4;
#pragma unroll
  for (int r = 0; r < kCsrRows; ++r) {
    if (m0 + r >= M) continue;
    const float4* src = reinterpret_cast<const float4*>(X + (size_t)(m0 + r) * ldx);
    float4* dst = reinterpret_cast<float4*>(xs + (size_t)r * K);
    for (int i = tid; i < kq; i += kCsrThreads) dst[i] = src[i];
  }
  __syncthreads();

  const int nq = N / 4;
  // every thread runs every round, so the loss butterfly's shuffles see full warps (nq % 16 == 0 where they run)
  for (int qb = 0; qb < nq; qb += kCsrThreads) {
    const int q = qb + tid;
    const bool active = q < nq;
    float acc[kCsrRows][4];
#pragma unroll
    for (int r = 0; r < kCsrRows; ++r)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[r][j] = 0.f;
    if (active) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e1 = rp[4 * q + j + 1];
        for (int e = rp[4 * q + j]; e < e1; ++e) {
          const int c = ci[e];
          const float a = val[e];
#pragma unroll
          for (int r = 0; r < kCsrRows; ++r) acc[r][j] = fmaf(xs[r * K + c], a, acc[r][j]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < kCsrRows; ++r) {
      const int row = m0 + r;
      if (row >= M) continue;                        // uniform across the CTA
      float rsum = 0.f;
      if (active) {
        const int col = 4 * q;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (EPI == MEAS_RESID) {
            v[j] = acc[r][j] - ym[(size_t)(row / R) * ldo + col + j];
            rsum = fmaf(v[j], v[j], rsum);
          } else if (EPI == MEAS_RESID_HUBER) {
            const float rj = acc[r][j] - ym[(size_t)(row / R) * ldo + col + j];
            v[j] = fabsf(rj) > s ? copysignf(s, rj) : rj;
            rsum = fmaf(v[j], 2.f * rj - v[j], rsum);
          } else {
            v[j] = acc[r][j] * s;
          }
        }
        *reinterpret_cast<float4*>(out + (size_t)row * ldo + col) = make_float4(v[0], v[1], v[2], v[3]);
      }
      if (EPI != MEAS_SCALE) {
#pragma unroll
        for (int o = 1; o < 16; o <<= 1) rsum += __shfl_xor_sync(0xffffffffu, rsum, o);
        if (active && (q & 15) == 0) loss_part[(size_t)(q / 16) * loss_ld + row] = rsum;
      }
    }
  }
}

template <int EPI>
__global__ void __launch_bounds__(kCsrThreads)
measured_csr_kernel(const float* __restrict__ X, int ldx, int M, int K, const int* __restrict__ rp,
                    const int* __restrict__ ci, const float* __restrict__ val, int N, float* __restrict__ out, int ldo,
                    const float* __restrict__ ym, int R, float s, float* __restrict__ loss_part, int loss_ld) {
  measured_csr_body<EPI>(X, ldx, M, K, rp, ci, val, N, out, ldo, ym, R, s, loss_part, loss_ld);
}

// The measurement product with the Huber residual (MEAS_RESID_HUBER) at delta = s
__global__ void __launch_bounds__(kCsrThreads)
measured_csr_huber_kernel(const float* __restrict__ X, int ldx, int M, int K, const int* __restrict__ rp,
                          const int* __restrict__ ci, const float* __restrict__ val, int N, float* __restrict__ out,
                          int ldo, const float* __restrict__ ym, int R, float s, float* __restrict__ loss_part,
                          int loss_ld) {
  measured_csr_body<MEAS_RESID_HUBER>(X, ldx, M, K, rp, ci, val, N, out, ldo, ym, R, s, loss_part, loss_ld);
}

// ---- staging ---------------------------------------------------------------------------------------------------------

// bad[i] = 1 when row i of the caller's CSR breaks the format (see the top of the file), else 0; i < m
__global__ void csr_validate_kernel(const int* __restrict__ row_ptr, const int* __restrict__ col_idx, int m, int nnz,
                                    int n_cols, int* __restrict__ bad) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int lo = row_ptr[i], hi = row_ptr[i + 1];
  int b = lo < 0 || hi < lo || hi > nnz || (i == 0 && lo != 0) || (i == m - 1 && hi != nnz);
  if (!b) {
    int prev = -1;
    for (int e = lo; e < hi && !b; ++e) {
      const int c = col_idx[e];
      b = c <= prev || c >= n_cols;
      prev = c;
    }
  }
  bad[i] = b;
}

// One CTA of 1024 threads: valid[0] = no row is bad; the staged row pointers a_rp [m_ld + 1]: the caller's, with m_ld - m
// empty rows appended, or all 0 (the empty operator) when the CSR is invalid.
__global__ void __launch_bounds__(1024) csr_stage_rows_kernel(const int* __restrict__ row_ptr, const int* __restrict__ bad,
                                                              int m, int m_ld, int nnz, int* __restrict__ valid,
                                                              int* __restrict__ a_rp) {
  int b = 0;
  for (int i = threadIdx.x; i < m; i += blockDim.x) b |= bad[i];
  const int ok = !__syncthreads_or(b);
  if (threadIdx.x == 0) valid[0] = ok;
  for (int i = threadIdx.x; i <= m_ld; i += blockDim.x) a_rp[i] = ok ? (i <= m ? row_ptr[i] : nnz) : 0;
}

// One grid over three index ranges:
//   i < nnz:          the entries, a_ci / a_v[i] = col_idx / val[i];
//   i < batch * m_ld: the measurements, ym [batch][m_ld] = y [batch][m] with zero columns, all NaN for an invalid CSR;
//   i < n_cols:       cnt[i] = the non-zeros of column i (rows of the staged a_rp holding it, by binary search in the
//                     caller's sorted columns: a_rp is all 0 for an invalid CSR, so nothing is read).
__global__ void csr_stage_entries_kernel(const int* __restrict__ col_idx, const float* __restrict__ val, int nnz,
                                         const float* __restrict__ y, int batch, int m, int m_ld,
                                         const int* __restrict__ a_rp, const int* __restrict__ valid, int n_cols,
                                         int* __restrict__ a_ci, float* __restrict__ a_v, float* __restrict__ ym,
                                         int* __restrict__ cnt) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (size_t)nnz) {
    a_ci[i] = col_idx[i];
    a_v[i] = val[i];
  }
  if (i < (size_t)batch * m_ld) {
    const int b = (int)(i / m_ld), j = (int)(i % m_ld);
    ym[i] = valid[0] ? (j < m ? y[(size_t)b * m + j] : 0.f) : __int_as_float(0x7fffffff);
  }
  if (i < (size_t)n_cols) {
    const int c = (int)i;
    int n = 0;
    for (int r = 0; r < m; ++r) {
      int lo = a_rp[r], hi = a_rp[r + 1];
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (col_idx[mid] < c) lo = mid + 1; else hi = mid;
      }
      n += lo < a_rp[r + 1] && col_idx[lo] == c;
    }
    cnt[c] = n;
  }
}

// One CTA of 1024 threads: at_rp [n + 1] = the exclusive prefix sum of the counts it holds in at_rp[0..n), in place.
__global__ void __launch_bounds__(1024) csr_scan_kernel(int* __restrict__ at_rp, int n) {
  __shared__ int part[1024];
  const int t = threadIdx.x, per = (n + 1023) / 1024;
  const int lo = min(n, t * per), hi = min(n, lo + per);
  int sum = 0;
  for (int i = lo; i < hi; ++i) sum += at_rp[i];
  part[t] = sum;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {               // inclusive scan of the per-thread sums
    const int v = t >= o ? part[t - o] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  int run = t > 0 ? part[t - 1] : 0;
  for (int i = lo; i < hi; ++i) {
    const int c = at_rp[i];
    at_rp[i] = run;
    run += c;
  }
  if (t == 1023) at_rp[n] = part[1023];
}

// Thread c fills row c of At (at_rp from csr_scan_kernel) from the staged A, visiting the rows of A in ascending order:
// at_ci = the row of A, at_v = its value.
__global__ void csr_fill_transpose_kernel(const int* __restrict__ a_rp, const int* __restrict__ a_ci,
                                          const float* __restrict__ a_v, int m, int n_cols, const int* __restrict__ at_rp,
                                          int* __restrict__ at_ci, float* __restrict__ at_v) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cols) return;
  int pos = at_rp[c];
  for (int r = 0; r < m; ++r) {
    int lo = a_rp[r], hi = a_rp[r + 1];
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (a_ci[mid] < c) lo = mid + 1; else hi = mid;
    }
    if (lo < a_rp[r + 1] && a_ci[lo] == c) {
      at_ci[pos] = r;
      at_v[pos] = a_v[lo];
      ++pos;
    }
  }
}

}  // namespace dgan
