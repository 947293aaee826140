// Restart pruning (dgan_reconstruct_pruned): at a prune point every image keeps its `keep` best restarts, and the rest of
// the loop runs on the survivors only, in the next workspace region.  Rows of a region are image-major: row
// img * per_image + j is the j-th surviving restart of image img, survivors in ascending original restart index.
#pragma once
#include "common.cuh"

namespace dgan {

// The most restarts an image may have in a pruned call: prune_select_kernel keeps one flag byte per restart of an image in
// (static) shared memory.
constexpr int kPruneMaxRestarts = 32768;

// Does restart (la, oa) rank before (lb, ob)?  Lower loss first, ties by the lower original index; a NaN loss ranks after
// every number, NaNs among themselves by index.
__device__ __forceinline__ bool prune_before(float la, int oa, float lb, int ob) {
  const bool na = isnan(la), nb = isnan(lb);
  if (na || nb) return na ? (nb && oa < ob) : true;
  return la < lb || (la == lb && oa < ob);
}

// One CTA per image.  loss [batch * n_prev]: the per-row loss of the current region; orig [batch * n_prev]: each row's
// original restart index (NULL: the first region, where row j of an image is restart j).  Keeps each image's `keep`
// first-ranked rows and writes the next region's maps: src [batch * keep] (the row of the current region each row comes
// from) and orig_out [batch * keep].  The ranks of one image are distinct (the original indices are), so exactly `keep`
// rows survive, and they stay in the order of the current region: ascending original index.
__global__ void __launch_bounds__(256)
prune_select_kernel(const float* __restrict__ loss, const int* __restrict__ orig, int n_prev, int keep,
                    int* __restrict__ src, int* __restrict__ orig_out) {
  __shared__ unsigned char kept[kPruneMaxRestarts];
  const int img = blockIdx.x;
  const float* l = loss + (size_t)img * n_prev;
  const int* o = orig != nullptr ? orig + (size_t)img * n_prev : nullptr;
  for (int j = threadIdx.x; j < n_prev; j += blockDim.x) {
    const float lj = l[j];
    const int oj = o != nullptr ? o[j] : j;
    int rank = 0;
    for (int i = 0; i < n_prev; ++i) rank += prune_before(l[i], o != nullptr ? o[i] : i, lj, oj) ? 1 : 0;
    kept[j] = rank < keep ? 1 : 0;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < n_prev; j += blockDim.x) {
    if (!kept[j]) continue;
    int pos = 0;
    for (int i = 0; i < j; ++i) pos += kept[i];
    const size_t dst = (size_t)img * keep + pos;
    src[dst] = img * n_prev + j;
    orig_out[dst] = o != nullptr ? o[j] : j;
  }
}

// The survivors' optimiser state into the next region: z, v and (fp16 path, z_h != NULL) z_h, rows of `ld` values (the
// padded latent width), row r from row src[r] of the current region; the tile-padding rows n_rows .. n_pad - 1 are zeroed,
// as init_z_kernel leaves them in a fresh workspace.
__global__ void prune_gather_kernel(const float* __restrict__ z, const float* __restrict__ v, const __half* __restrict__ z_h,
                                    const int* __restrict__ src, int n_rows, int n_pad, int ld, float* __restrict__ z_out,
                                    float* __restrict__ v_out, __half* __restrict__ z_h_out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n_pad * ld) return;
  const int row = (int)(i / ld), col = (int)(i % ld);
  float zz = 0.f, vv = 0.f;
  __half hh = __float2half_rn(0.f);
  if (row < n_rows) {
    const size_t s = (size_t)src[row] * ld + col;
    zz = z[s];
    vv = v[s];
    if (z_h != nullptr) hh = z_h[s];
  }
  z_out[i] = zz;
  v_out[i] = vv;
  if (z_h_out != nullptr) z_h_out[i] = hh;
}

// idx[img] = the original restart index of the survivor select_kernel chose (sel [batch], an index among the image's
// `per_image` survivors); nothing when idx is NULL.
__global__ void prune_idx_kernel(const int* __restrict__ sel, const int* __restrict__ orig, int per_image, int batch,
                                 int32_t* __restrict__ idx) {
  const int img = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx == nullptr || img >= batch) return;
  idx[img] = orig[(size_t)img * per_image + sel[img]];
}

}  // namespace dgan
