// Shared declarations for the Defense-GAN projection-loop kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <string>
#include <vector>
#include <numeric>

#include "../../include/defensegan_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "defensegan_b200 kernels are written for sm_90a only"
#endif

namespace dgan {

void set_error(const std::string& msg);

#define DGAN_CUDA_CHECK(expr)                                                              \
  do {                                                                                     \
    cudaError_t _e = (expr);                                                               \
    if (_e != cudaSuccess) {                                                               \
      ::dgan::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));               \
      return DGAN_ERR_CUDA;                                                                \
    }                                                                                      \
  } while (0)

// Programmatic dependent launch: kernels of the L-step loop are launched with
// cudaLaunchAttributeProgrammaticStreamSerialization; each calls pdl_launch_dependents() at its start
// (the next kernel's CTAs may be scheduled on SMs as they free up and run their prologue) and
// pdl_wait() before touching memory written by its predecessors (waits for their full completion).
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

constexpr int kRowTile = 128;   // latent rows per tile: the MMA M dimension / SIMT block tile
constexpr int kTaps = 25;       // 5x5 filter

enum Epilogue : int {
  EPI_BIAS_RELU = 0,  // out = relu(acc + bias[co])                      (forward, ReLU layers)
  EPI_BIAS = 1,       // out = acc + bias[co]                            (CelebA Generator.5: no activation)
  EPI_MASK = 2,       // out = acc * (mask_src > 0)                      (backward into a ReLU output)
  EPI_NONE = 3        // out = acc                                       (backward into a linear output / dz)
};

// ACT_NONE: the last layer's linear part alone, no bias (dgan_jvp's tangent of the pre-activation)
enum FinalAct : int { ACT_SIGMOID = 0, ACT_TANH = 1, ACT_NONE = 2 };

// One (input pixel, weight tile) contribution to an output pixel.  Every layer of the generator -
// Linear, 5x5/stride-2 transposed conv forward, and their backward-to-input - is expressed as
//   out[q][n][:] = epi( sum_{(p,t) in pairs(q)} in[p][n][:] x W_t )
// over activations stored pixel-major [P][N][C]; only in-bounds taps are listed, so the kernels
// issue exactly the algorithmic MACs (SURVEY section 8d) and never touch zero padding.
struct PairTable {
  std::vector<int> off;     // size P_out + 1
  std::vector<int2> pairs;  // (in pixel, weight tile)
  int max_per_pixel() const {
    int m = 0;
    for (size_t i = 0; i + 1 < off.size(); ++i) m = (off[i + 1] - off[i] > m) ? off[i + 1] - off[i] : m;
    return m;
  }
};

// TF conv2d_transpose(k=5, stride 2, SAME): out[i] += in[o] * w[k], i = 2o + k - 1
// (tflib/ops/deconv2d.py:100-110; SURVEY F7).  h_used/w_used = the output rows/cols that are
// kept (MNIST crops 8x8 -> 7x7 after Generator.2, models/dataset_models.py:59).
// `in_raster` (>= w_in): the input buffer is an in_raster x in_raster pixel raster of which only the
// top-left h_in x w_in pixels are consumed (MNIST + BatchNorm: Generator.2 keeps its full 8x8 output
// because the batch statistics cover the pixels that are cropped afterwards).
PairTable deconv_fwd_pairs(int h_in, int w_in, int h_used, int w_used, int in_raster = 0);
PairTable deconv_bwd_pairs(int h_in, int w_in, int h_used, int w_used, int in_raster = 0);
// Linear [latent] -> [16 pixels x C]: column f = (h*4 + w)*C + c (SURVEY F8b)
PairTable linear_fwd_pairs(int n_pix);
PairTable linear_bwd_pairs(int n_pix);

}  // namespace dgan
