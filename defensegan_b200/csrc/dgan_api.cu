// C-ABI of the H100-native Defense-GAN projection loop (see include/defensegan_b200.h).
// Host side: generator plan (pixel-graph tables), weight re-layout, workspace carving and the
// on-device L-step driver.  Everything is enqueued on the caller's stream; nothing here
// synchronises the host.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <new>

#include "common.cuh"
#include "kernels_simt.cuh"
#include "kernels_tc.cuh"
#include "kernels_tc2.cuh"
#include "kernels_vjp.cuh"

namespace dgan {

static thread_local std::string g_last_error;
void set_error(const std::string& msg) { g_last_error = msg; }

// ---------------------------------------------------------------------------------------
// geometry tables
// ---------------------------------------------------------------------------------------
PairTable deconv_fwd_pairs(int h_in, int w_in, int h_used, int w_used, int in_raster) {
  if (in_raster <= 0) in_raster = w_in;
  PairTable t;
  t.off.push_back(0);
  for (int i = 0; i < h_used; ++i)
    for (int j = 0; j < w_used; ++j) {
      for (int ka = 0; ka < 5; ++ka) {
        const int oo = i + 1 - ka;
        if (oo < 0 || (oo & 1) || (oo >> 1) >= h_in) continue;
        for (int kb = 0; kb < 5; ++kb) {
          const int pp = j + 1 - kb;
          if (pp < 0 || (pp & 1) || (pp >> 1) >= w_in) continue;
          t.pairs.push_back(make_int2((oo >> 1) * in_raster + (pp >> 1), ka * 5 + kb));
        }
      }
      t.off.push_back((int)t.pairs.size());
    }
  return t;
}

PairTable deconv_bwd_pairs(int h_in, int w_in, int h_used, int w_used, int in_raster) {
  if (in_raster <= 0) in_raster = w_in;
  PairTable t;
  t.off.push_back(0);
  for (int o = 0; o < in_raster; ++o)
    for (int p = 0; p < in_raster; ++p) {
      // raster pixels outside the consumed h_in x w_in window receive no gradient (empty list -> zeros)
      for (int ka = 0; ka < 5 && o < h_in && p < w_in; ++ka) {
        const int i = 2 * o + ka - 1;
        if (i < 0 || i >= h_used) continue;
        for (int kb = 0; kb < 5; ++kb) {
          const int j = 2 * p + kb - 1;
          if (j < 0 || j >= w_used) continue;
          t.pairs.push_back(make_int2(i * w_used + j, ka * 5 + kb));
        }
      }
      t.off.push_back((int)t.pairs.size());
    }
  return t;
}

PairTable linear_fwd_pairs(int n_pix) {
  PairTable t;
  t.off.push_back(0);
  for (int q = 0; q < n_pix; ++q) {
    t.pairs.push_back(make_int2(0, q));
    t.off.push_back((int)t.pairs.size());
  }
  return t;
}

PairTable linear_bwd_pairs(int n_pix) {
  PairTable t;
  t.off.push_back(0);
  for (int q = 0; q < n_pix; ++q) t.pairs.push_back(make_int2(q, q));
  t.off.push_back((int)t.pairs.size());
  return t;
}

// ---------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------
struct DevTable {
  int* off = nullptr;
  int2* pairs = nullptr;
  int n_out = 0;
  int n_pairs = 0;
};

struct GemmLayer {
  // forward: [P_in][N][C_in] -> [P_out][N][C_out]
  int P_in, C_in, P_out, C_out;
  int h_in, w_in, h_used, w_used;  // spatial geometry (Linear: 1x1 -> 4x4)
  bool relu;                       // ReLU after bias (false: CelebA Generator.5)
  DevTable fwd, bwd;
  PairTable fwd_host, bwd_host;
  // fp32 weight tiles.  forward tile t: rows = C_in (K), cols = C_out; backward: rows = C_out, cols = C_in
  const float* wf = nullptr; int wf_tile_stride = 0, wf_ld = 0;
  const float* wb = nullptr; int wb_tile_stride = 0, wb_ld = 0;
  const float* bias = nullptr;
  int bias_pstride = 0;            // Linear: bias is per flat feature f = pixel*C_out + c
  const float* bn_offset = nullptr;   // use_bn: Generator.BN{1,2,3}.offset / .scale (else null)
  const float* bn_scale = nullptr;
  int bn_per_pixel = 0;               // BN1 normalises each flat feature (axes [0]); BN2/3 each channel (axes [0,1,2])
  // fp16 K-major tiles for the tensor-core path (kernels_tc.cuh): [tile][N rows][K cols]
  TcWeights tc_f, tc_b;
  TcWeights2 tc2_f, tc2_b;
};

struct FinalLayer {
  int h_in, w_in, C_in, C_out, act;
  const float* w = nullptr;  // [25][C_out][C_in] == the TF filter layout
  const float* bias = nullptr;
  int n_bands = 0;
  size_t fwd_smem = 0, bwd_smem = 0;
};

}  // namespace dgan

using namespace dgan;

struct dgan_ctx {
  dgan_desc desc;
  int H = 0, W = 0, C = 0, hwc = 0;
  std::vector<GemmLayer> layers;
  FinalLayer fin;
  std::vector<void*> allocs;
  int64_t macs_per_row = 0;
  int64_t last_launches = 0;
  int64_t launches = 0;
  TcState tc;
  TcFinal tc_fin;
  TcWeights2 tc2_fin_f, tc2_fin_b;
  // optional per-launch CUDA-event timing (dgan_profile_*): serialises nothing by itself but
  // adds two event records per launch, so it is never enabled in a timed benchmark pass
  bool profile = false;
  int n_rows_cur = 0;
  // The L-step loop of a projection as a CUDA graph: captured once per (workspace, batch, R, L, lr, momentum, decay) on a
  // private stream, replayed with one cudaGraphLaunch per call.
  struct LoopGraph {
    const void* ws; int batch, rec_rr, rec_iters, decay_lr; float rec_lr, momentum;
    cudaGraphExec_t exec; int64_t kernels;
  };
  std::vector<LoopGraph> graphs;
  cudaStream_t cap_stream = nullptr;
  int64_t last_enqueues = 0;
  struct ProfRec { int kind; cudaEvent_t a, b; };
  std::vector<ProfRec> prof;
  std::vector<std::string> kind_names;
  std::vector<double> kind_macs_per_row;
};

namespace dgan {

struct ProfScope {
  dgan_ctx* c; cudaStream_t s; bool on; dgan_ctx::ProfRec r;
  ProfScope(dgan_ctx* c_, int kind, cudaStream_t s_) : c(c_), s(s_), on(c_->profile) {
    if (!on) return;
    r.kind = kind;
    cudaEventCreate(&r.a); cudaEventCreate(&r.b);
    cudaEventRecord(r.a, s);
  }
  ~ProfScope() {
    if (!on) return;
    cudaEventRecord(r.b, s);
    c->prof.push_back(r);
  }
};

static int dev_alloc(dgan_ctx* c, void** p, size_t bytes) {
  DGAN_CUDA_CHECK(cudaMalloc(p, bytes));
  c->allocs.push_back(*p);
  return 0;
}

static int upload_table(dgan_ctx* c, const PairTable& t, DevTable* d, cudaStream_t s) {
  d->n_out = (int)t.off.size() - 1;
  d->n_pairs = (int)t.pairs.size();
  int rc;
  if ((rc = dev_alloc(c, (void**)&d->off, t.off.size() * sizeof(int)))) return rc;
  if ((rc = dev_alloc(c, (void**)&d->pairs, t.pairs.size() * sizeof(int2)))) return rc;
  // pageable-source async copies are staged by the runtime before returning
  DGAN_CUDA_CHECK(cudaMemcpyAsync(d->off, t.off.data(), t.off.size() * sizeof(int), cudaMemcpyHostToDevice, s));
  DGAN_CUDA_CHECK(cudaMemcpyAsync(d->pairs, t.pairs.data(), t.pairs.size() * sizeof(int2), cudaMemcpyHostToDevice, s));
  return 0;
}

// out[t][c][r] = in[t][r][c]   (per-tile transpose; rows x cols -> cols x rows)
__global__ void transpose_tiles_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols,
                                       size_t total) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const size_t per = (size_t)rows * cols;
  const size_t t = i / per, rem = i % per;
  const int r = (int)(rem / cols), cc = (int)(rem % cols);
  out[t * per + (size_t)cc * rows + r] = in[i];
}

// out = s * (sum of the n_parts partial sums, fixed order); with row_scale, row r (row_len values) is also divided by
// row_scale[r] (dgan_vjp: its power-of-two cotangent scales, so the division is exact)
__global__ void scale_copy_kernel(const float* __restrict__ in, int n_parts, size_t part_stride,
                                  float* __restrict__ out, float s, size_t n,
                                  const float* __restrict__ row_scale, int row_len) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float g = in[i];
  for (int p = 1; p < n_parts; ++p) g += in[i + (size_t)p * part_stride];
  float m = s;
  if (row_scale != nullptr) m /= row_scale[i / row_len];
  out[i] = g * m;
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---------------------------------------------------------------------------------------
// workspace
// ---------------------------------------------------------------------------------------
struct Workspace {
  int n_rows = 0, n_pad = 0;
  float *z = nullptr, *v = nullptr, *g = nullptr;
  std::vector<float*> act, dact;     // fp32 path: per hidden layer output [P][n_pad][C]
  std::vector<float*> pre;           // use_bn: pre-normalisation outputs (null otherwise)
  std::vector<float*> bn_part;       // use_bn: [4][kBnSplits][G] partial sums (mean, var, S1, S2)
  std::vector<__half*> act_h, dact_h;  // fp16 path
  std::vector<float*> pre_h;           // fp16 path, use_bn: pre-normalisation outputs, fp32 (null otherwise)
  __half* z_h = nullptr;
  std::vector<unsigned long long*> maskbits;   // fp16 path: 1-bit ReLU masks per hidden layer output
  // fp16 CTA-pair path: TMA descriptors of every launch site, encoded once per workspace
  // index 2l = forward of layer l (in, out), 2l+1 = backward of layer l; 2nl = last-layer forward, 2nl+1 = its backward
  std::vector<CUtensorMap> map_in, map_out;
  bool have_maps = false;
  unsigned* mom_counter = nullptr;     // fp16 path: [n_pad / 128] tickets of the split-K Linear backward's momentum tail
  __half* dblk = nullptr;              // fp16 path: [n_blocks][n_pad][16 * C_out] scaled dL/dpre of the last layer
  int n_loss_parts = 0, n_g_parts = 1;
  size_t loss_stride_n = 1, loss_stride_b = 1;   // loss_part index = n * stride_n + part * stride_b
  float *y = nullptr, *dpre = nullptr, *loss_part = nullptr;
  float* loss = nullptr;               // [n_pad] per-row loss; dgan_vjp (which computes no loss) keeps its row scales here
  float* x = nullptr;                  // [batch][H*W*C] copy of the call's images (the captured loop reads them from here)
  size_t bytes = 0;
};

static Workspace carve(const dgan_ctx* c, int n_rows, void* base) {
  Workspace w;
  w.n_rows = n_rows;
  w.n_pad = (int)align_up((size_t)std::max(n_rows, 1), c->desc.precision == DGAN_PREC_FP16 ? 2 * kRowTile : kRowTile);
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t bytes) -> void* {
    void* p = b ? (void*)(b + off) : nullptr;
    off += align_up(bytes, 1024);
    return p;
  };
  const size_t np = (size_t)w.n_pad;
  const int latent = c->desc.latent_dim;
  w.z = (float*)take(np * latent * 4);
  w.v = (float*)take(np * latent * 4);
  const bool tc = c->desc.precision == DGAN_PREC_FP16;
  w.n_g_parts = tc ? TC_LINEAR_SPLIT : 1;
  w.g = (float*)take(np * latent * 4 * w.n_g_parts);
  if (tc) w.z_h = (__half*)take(np * latent * 2);
  if (tc) w.mom_counter = (unsigned*)take(np / kRowTile * sizeof(unsigned));
  if (tc) w.dblk = (__half*)take((size_t)c->tc_fin.n_blocks * np * 16 * c->tc_fin.C_out * 2);
  w.n_loss_parts = tc ? c->tc_fin.n_blocks : c->fin.n_bands;
  w.loss_stride_n = tc ? 1 : (size_t)w.n_loss_parts;          // fp16 path: [block][n_pad] (coalesced epilogue stores)
  w.loss_stride_b = tc ? (size_t)np : 1;
  for (const GemmLayer& l : c->layers) {
    const size_t elems = (size_t)l.P_out * np * l.C_out;
    if (tc) {
      w.act_h.push_back((__half*)take(elems * 2));
      w.dact_h.push_back((__half*)take(elems * 2));
      w.maskbits.push_back((unsigned long long*)take(elems / 8));
      if (l.bn_scale != nullptr) {
        const size_t G = l.bn_per_pixel ? (size_t)l.P_out * l.C_out : (size_t)l.C_out;
        w.pre_h.push_back((float*)take(elems * 4));
        w.bn_part.push_back((float*)take((size_t)4 * kBnSplits * G * 4));
      } else {
        w.pre_h.push_back(nullptr);
        w.bn_part.push_back(nullptr);
      }
    } else {
      w.act.push_back((float*)take(elems * 4));
      w.dact.push_back((float*)take(elems * 4));
      if (l.bn_scale != nullptr) {
        const size_t G = l.bn_per_pixel ? (size_t)l.P_out * l.C_out : (size_t)l.C_out;
        w.pre.push_back((float*)take(elems * 4));
        w.bn_part.push_back((float*)take((size_t)4 * kBnSplits * G * 4));
      } else {
        w.pre.push_back(nullptr);
        w.bn_part.push_back(nullptr);
      }
    }
  }
  w.x = (float*)take(np * c->hwc * 4);     // batch <= n_pad
  w.y = (float*)take(np * c->hwc * 4);
  w.dpre = (float*)take(np * c->hwc * 4);
  w.loss_part = (float*)take(np * w.n_loss_parts * 4);
  w.loss = (float*)take(np * 4);
  w.bytes = off;
  return w;
}

// ---------------------------------------------------------------------------------------
// launches
// ---------------------------------------------------------------------------------------
#define DGAN_LAUNCH_CHECK(c)                                                     \
  do {                                                                           \
    (c)->launches++;                                                             \
    cudaError_t _e = cudaGetLastError();                                         \
    if (_e != cudaSuccess) {                                                     \
      set_error(std::string("kernel launch: ") + cudaGetErrorString(_e));        \
      return DGAN_ERR_CUDA;                                                      \
    }                                                                            \
  } while (0)

static int launch_bsgemm_f32(dgan_ctx* c, int epi, const float* in, int C_in, int n_pad, const float* wt,
                             int tile_stride, int ldw, const DevTable& tab, float* out, int C_out,
                             const float* bias, int bias_pstride, const float* mask_src, cudaStream_t s) {
  dim3 grid(n_pad / kRowTile, tab.n_out, C_out / 64), block(256);
  switch (epi) {
    case EPI_BIAS_RELU:
      bsgemm_f32_kernel<EPI_BIAS_RELU><<<grid, block, 0, s>>>(in, C_in, n_pad, wt, tile_stride, ldw, tab.off,
                                                              tab.pairs, out, C_out, bias, bias_pstride, mask_src);
      break;
    case EPI_BIAS:
      bsgemm_f32_kernel<EPI_BIAS><<<grid, block, 0, s>>>(in, C_in, n_pad, wt, tile_stride, ldw, tab.off, tab.pairs,
                                                         out, C_out, bias, bias_pstride, mask_src);
      break;
    case EPI_MASK:
      bsgemm_f32_kernel<EPI_MASK><<<grid, block, 0, s>>>(in, C_in, n_pad, wt, tile_stride, ldw, tab.off, tab.pairs,
                                                         out, C_out, bias, bias_pstride, mask_src);
      break;
    default:
      bsgemm_f32_kernel<EPI_NONE><<<grid, block, 0, s>>>(in, C_in, n_pad, wt, tile_stride, ldw, tab.off, tab.pairs,
                                                         out, C_out, bias, bias_pstride, mask_src);
      break;
  }
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

template <typename TIN>
static int launch_final_fwd(dgan_ctx* c, const TIN* hin, const Workspace& w, const float* x, int R, int B,
                            bool want_grad, cudaStream_t s) {
  const FinalLayer& f = c->fin;
  dim3 grid(w.n_rows, f.n_bands), block(128);
  const size_t smem = f.fwd_smem;
  float* dpre = want_grad ? w.dpre : nullptr;
  float* lp = x ? w.loss_part : nullptr;
#define FF(CO, ACT)                                                                                         \
  final_fwd_loss_kernel<TIN, CO, ACT><<<grid, block, smem, s>>>(hin, w.n_pad, f.h_in, f.w_in, f.C_in, f.w, \
                                                                f.bias, x, R, B, w.y, dpre ? dpre : w.dpre, lp)
  if (f.C_out == 1 && f.act == ACT_SIGMOID) FF(1, ACT_SIGMOID);
  else if (f.C_out == 3 && f.act == ACT_TANH) FF(3, ACT_TANH);
  else { set_error("unsupported final layer"); return DGAN_ERR_UNSUPPORTED; }
#undef FF
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

template <typename TOUT>
static int launch_final_bwd(dgan_ctx* c, const Workspace& w, const TOUT* mask_src, float gscale, TOUT* din,
                            cudaStream_t s) {
  const FinalLayer& f = c->fin;
  const size_t work = (size_t)f.h_in * f.w_in * w.n_pad * (f.C_in / 4);
  dim3 grid((unsigned)((work + 255) / 256)), block(256);
  if (f.C_out == 1)
    final_bwd_kernel<TOUT, 1><<<grid, block, f.bwd_smem, s>>>(w.dpre, w.n_pad, f.h_in, f.w_in, f.C_in, f.w, mask_src,
                                                              gscale, din);
  else
    final_bwd_kernel<TOUT, 3><<<grid, block, f.bwd_smem, s>>>(w.dpre, w.n_pad, f.h_in, f.w_in, f.C_in, f.w, mask_src,
                                                              gscale, din);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

static int tcx_launch(dgan_ctx* c, const TcWeights& w1, const TcWeights2& w2, const __half* in, __half* out, int n_pad,
                      int epi, const float* bias, cudaStream_t s,
                      unsigned long long* mb_out = nullptr, const unsigned long long* mb_in = nullptr,
                      const CUtensorMap* pre_a = nullptr, const CUtensorMap* pre_out = nullptr);

// Encode the TMA descriptors of all launch sites for this workspace (once per call instead of per launch).
static int build_maps(dgan_ctx* c, Workspace& w) {
  if (c->desc.precision != DGAN_PREC_FP16) return 0;
  const int nl = (int)c->layers.size();
  w.map_in.assign((size_t)2 * nl + 2, CUtensorMap{});
  w.map_out.assign((size_t)2 * nl + 2, CUtensorMap{});
  int rc;
  auto mk = [&](CUtensorMap* m, const void* base, int K, int P, uint32_t box_rows = 128) {
    return tc_make_map(c->tc, m, base, (uint64_t)K, (uint64_t)w.n_pad, (uint64_t)P, box_rows, tc2_box_k(K));
  };
  for (int l = 0; l < nl; ++l) {
    const GemmLayer& L = c->layers[l];
    const void* fin = (l == 0) ? (const void*)w.z_h : (const void*)w.act_h[l - 1];
    if ((rc = mk(&w.map_in[2 * l], fin, L.C_in, L.P_in))) return rc;
    if ((rc = mk(&w.map_out[2 * l], w.act_h[l], L.C_out, L.P_out, TC2_STORE_ROWS))) return rc;   // unused by BN layers (float epilogue)
    if ((rc = mk(&w.map_in[2 * l + 1], w.dact_h[l], L.C_out, L.P_out))) return rc;
    if (l >= 1 && (rc = mk(&w.map_out[2 * l + 1], w.dact_h[l - 1], L.C_in, L.P_in, TC2_STORE_ROWS))) return rc;
  }
  const GemmLayer& last = c->layers[nl - 1];
  if ((rc = mk(&w.map_in[2 * nl], w.act_h[nl - 1], c->fin.C_in, last.P_out))) return rc;
  if ((rc = mk(&w.map_in[2 * nl + 1], w.dblk, 16 * c->tc_fin.C_out, c->tc_fin.n_blocks))) return rc;   // 16-channel boxes
  if ((rc = mk(&w.map_out[2 * nl + 1], w.dact_h[nl - 1], last.C_out, last.P_out, TC2_STORE_ROWS))) return rc;
  w.have_maps = true;
  return 0;
}

// ---- batch-statistics BatchNorm of layer l on either path's activations (tflib/ops/batchnorm.py:80-93) ----
// forward: act = relu(BN(pre)); backward: d(act) -> d(pre) through the ReLU and the batch statistics, in place in dact
template <typename TP, typename T>
static int bn_forward_t(dgan_ctx* c, const Workspace& w, int l, const TP* pre, T* act, cudaStream_t s) {
  const GemmLayer& L = c->layers[l];
  const int G = L.bn_per_pixel ? L.P_out * L.C_out : L.C_out;
  float* part = w.bn_part[l];
  float *mean_p = part, *var_p = part + (size_t)kBnSplits * G;
  dim3 rgrid(G / 32, kBnSplits);
  bn_reduce_kernel<0, TP, T><<<rgrid, 256, 0, s>>>(pre, nullptr, nullptr, nullptr, nullptr, L.P_out, w.n_rows, w.n_pad, L.C_out,
                                               L.bn_per_pixel, mean_p, nullptr);
  DGAN_LAUNCH_CHECK(c);
  bn_reduce_kernel<1, TP, T><<<rgrid, 256, 0, s>>>(pre, nullptr, nullptr, mean_p, nullptr, L.P_out, w.n_rows, w.n_pad, L.C_out,
                                               L.bn_per_pixel, var_p, nullptr);
  DGAN_LAUNCH_CHECK(c);
  const size_t total = (size_t)L.P_out * w.n_pad * L.C_out;
  bn_apply_fwd_kernel<TP, T><<<(unsigned)((total + 255) / 256), 256, 0, s>>>(pre, mean_p, var_p, L.bn_scale, L.bn_offset, L.P_out,
                                                                          w.n_rows, w.n_pad, L.C_out, L.bn_per_pixel, act);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}
template <typename TP, typename T>
static int bn_backward_t(dgan_ctx* c, const Workspace& w, int l, const TP* pre, const T* act, T* dact, cudaStream_t s) {
  const GemmLayer& L = c->layers[l];
  const int G = L.bn_per_pixel ? L.P_out * L.C_out : L.C_out;
  float* part = w.bn_part[l];
  float *mean_p = part, *var_p = part + (size_t)kBnSplits * G, *s1_p = part + (size_t)2 * kBnSplits * G,
        *s2_p = part + (size_t)3 * kBnSplits * G;
  dim3 rgrid(G / 32, kBnSplits);
  bn_reduce_kernel<2, TP, T><<<rgrid, 256, 0, s>>>(pre, act, dact, mean_p, var_p, L.P_out, w.n_rows, w.n_pad, L.C_out,
                                               L.bn_per_pixel, s1_p, s2_p);
  DGAN_LAUNCH_CHECK(c);
  const size_t total = (size_t)L.P_out * w.n_pad * L.C_out;
  bn_apply_bwd_kernel<TP, T><<<(unsigned)((total + 255) / 256), 256, 0, s>>>(pre, act, mean_p, var_p, s1_p, s2_p, L.bn_scale, L.P_out,
                                                                          w.n_rows, w.n_pad, L.C_out, L.bn_per_pixel, dact);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// ---- one generator forward (+ loss and dL/dpre when x != null) ---------------------------
static int run_forward(dgan_ctx* c, const Workspace& w, const float* x, int R, int B, bool want_grad,
                       cudaStream_t s, bool want_y = true) {
  int rc;
  const int nl = (int)c->layers.size();
  if (c->desc.precision == DGAN_PREC_FP16) {
    const __half* in = w.z_h;
    for (int l = 0; l < nl; ++l) {
      const GemmLayer& L = c->layers[l];
      ProfScope ps(c, 2 * l, s);
      if (L.bn_scale != nullptr) {               // pre = GEMM + bias (fp32 out);  act = relu(BN_batchstat(pre)) (fp16)
        TcFinalArgs fa{};
        if ((rc = tc2_launch_impl<float>(c->tc, &c->launches, L.tc_f, L.tc2_f, in, w.pre_h[l], w.n_pad, EPI_BIAS, L.bias, s, &fa,
                                         w.have_maps ? &w.map_in[2 * l] : nullptr, nullptr)))
          return rc;
        if ((rc = bn_forward_t<float, __half>(c, w, l, w.pre_h[l], w.act_h[l], s))) return rc;
      } else if ((rc = tcx_launch(c, L.tc_f, L.tc2_f, in, w.act_h[l], w.n_pad, L.relu ? EPI_BIAS_RELU : EPI_BIAS, L.bias, s,
                                  (L.relu && want_grad) ? w.maskbits[l] : nullptr, nullptr,
                                  w.have_maps ? &w.map_in[2 * l] : nullptr, w.have_maps ? &w.map_out[2 * l] : nullptr))) {
        return rc;
      }
      in = w.act_h[l];
    }
    ProfScope ps(c, 2 * nl, s);
    TcFinalArgs fa{};
    fa.x = x; fa.y = w.y; fa.loss_part = w.loss_part; fa.R = R; fa.B = B; fa.n_rows = w.n_rows;
    fa.nbx = c->tc_fin.nbx; fa.w_out = c->tc_fin.w_out; fa.gscale = c->tc.grad_scale; fa.write_y = want_y ? 1 : 0;
    return tc2_launch_impl<__half>(c->tc, &c->launches, c->tc_fin.f, c->tc2_fin_f, in, w.dblk, w.n_pad,
                                   c->tc_fin.C_out == 1 ? EPI_FINAL_SIGMOID1 : EPI_FINAL_TANH3, c->fin.bias, s, &fa,
                                   w.have_maps ? &w.map_in[2 * nl] : nullptr, nullptr);
  }
  const float* in = w.z;
  for (int l = 0; l < nl; ++l) {
    const GemmLayer& L = c->layers[l];
    ProfScope ps(c, 2 * l, s);
    if (L.bn_scale != nullptr) {
      // pre = GEMM + bias;  act = relu(BN_batchstat(pre))
      if ((rc = launch_bsgemm_f32(c, EPI_BIAS, in, L.C_in, w.n_pad, L.wf, L.wf_tile_stride, L.wf_ld, L.fwd, w.pre[l], L.C_out,
                                  L.bias, L.bias_pstride, nullptr, s)))
        return rc;
      if ((rc = bn_forward_t<float, float>(c, w, l, w.pre[l], w.act[l], s))) return rc;
    } else if ((rc = launch_bsgemm_f32(c, L.relu ? EPI_BIAS_RELU : EPI_BIAS, in, L.C_in, w.n_pad, L.wf, L.wf_tile_stride,
                                       L.wf_ld, L.fwd, w.act[l], L.C_out, L.bias, L.bias_pstride, nullptr, s))) {
      return rc;
    }
    in = w.act[l];
  }
  ProfScope ps(c, 2 * nl, s);
  return launch_final_fwd<float>(c, in, w, x, R, B, want_grad, s);
}

// ---- backward-to-z: w.g = J^T dpre (unscaled by 2/HWC; fp16 path additionally x gscale) -----
struct MomentumArgs { bool tail = false; float lr = 0.f, mu = 0.f; };   // tail: update z in the Linear backward's tail

static float grad_multiplier(const dgan_ctx* c);

static int run_backward(dgan_ctx* c, const Workspace& w, cudaStream_t s, MomentumArgs mom = MomentumArgs()) {
  int rc;
  const int nl = (int)c->layers.size();
  if (c->desc.precision == DGAN_PREC_FP16) {
    const GemmLayer& last = c->layers[nl - 1];
    // with BatchNorm after layer j the GEMM writes d(act_j) unmasked and the BN backward turns it into d(pre_j) in place
    auto bn_backward_h = [&](int j) -> int { return bn_backward_t<float, __half>(c, w, j, w.pre_h[j], w.act_h[j], w.dact_h[j], s); };
    {
      ProfScope ps(c, 2 * nl + 1, s);
      const bool bn = last.bn_scale != nullptr, mask = last.relu && !bn;
      if ((rc = tcx_launch(c, c->tc_fin.b, c->tc2_fin_b, w.dblk, w.dact_h[nl - 1], w.n_pad, mask ? EPI_MASK : EPI_NONE,
                           nullptr, s, nullptr, mask ? w.maskbits[nl - 1] : nullptr,
                           w.have_maps ? &w.map_in[2 * nl + 1] : nullptr, w.have_maps ? &w.map_out[2 * nl + 1] : nullptr)))
        return rc;
      if (bn && (rc = bn_backward_h(nl - 1))) return rc;
    }
    for (int l = nl - 1; l >= 1; --l) {
      const GemmLayer& L = c->layers[l];
      const bool bn = c->layers[l - 1].bn_scale != nullptr, mask = c->layers[l - 1].relu && !bn;
      ProfScope ps(c, 2 * l + 1, s);
      if ((rc = tcx_launch(c, L.tc_b, L.tc2_b, w.dact_h[l], w.dact_h[l - 1], w.n_pad, mask ? EPI_MASK : EPI_NONE, nullptr,
                           s, nullptr, mask ? w.maskbits[l - 1] : nullptr,
                           w.have_maps ? &w.map_in[2 * l + 1] : nullptr, w.have_maps ? &w.map_out[2 * l + 1] : nullptr)))
        return rc;
      if (bn && (rc = bn_backward_h(l - 1))) return rc;
    }
    const GemmLayer& L0 = c->layers[0];
    ProfScope ps(c, 1, s);
    TcFinalArgs fa{};
    if (mom.tail) {      // the CTA that completes a row tile's partial sums applies the momentum update
      fa.mz = w.z; fa.mv = w.v; fa.mz_h = w.z_h; fa.m_gmul = grad_multiplier(c); fa.m_lr = mom.lr; fa.m_mu = mom.mu;
      fa.m_counter = w.mom_counter; fa.m_nparts = w.n_g_parts; fa.m_count = (size_t)w.n_pad * c->desc.latent_dim;
    }
    return tc2_launch_impl<float>(c->tc, &c->launches, L0.tc_b, L0.tc2_b, w.dact_h[0], w.g, w.n_pad, EPI_NONE, nullptr, s,
                                  &fa, w.have_maps ? &w.map_in[1] : nullptr, nullptr);
  }
  auto bn_backward = [&](int l) -> int { return bn_backward_t<float, float>(c, w, l, w.pre[l], w.act[l], w.dact[l], s); };
  const GemmLayer& last = c->layers[nl - 1];
  {
    ProfScope ps(c, 2 * nl + 1, s);
    const bool bn = last.bn_scale != nullptr;
    if ((rc = launch_final_bwd<float>(c, w, (last.relu && !bn) ? w.act[nl - 1] : nullptr, 1.f, w.dact[nl - 1], s))) return rc;
    if (bn && (rc = bn_backward(nl - 1))) return rc;
  }
  for (int l = nl - 1; l >= 1; --l) {
    const GemmLayer& L = c->layers[l];
    const bool bn = c->layers[l - 1].bn_scale != nullptr;
    const bool mask = c->layers[l - 1].relu && !bn;
    ProfScope ps(c, 2 * l + 1, s);
    if ((rc = launch_bsgemm_f32(c, mask ? EPI_MASK : EPI_NONE, w.dact[l], L.C_out, w.n_pad, L.wb, L.wb_tile_stride,
                                L.wb_ld, L.bwd, w.dact[l - 1], L.C_in, nullptr, 0, mask ? w.act[l - 1] : nullptr, s)))
      return rc;
    if (bn && (rc = bn_backward(l - 1))) return rc;
  }
  const GemmLayer& L0 = c->layers[0];
  ProfScope ps(c, 1, s);
  return launch_bsgemm_f32(c, EPI_NONE, w.dact[0], L0.C_out, w.n_pad, L0.wb, L0.wb_tile_stride, L0.wb_ld, L0.bwd, w.g,
                           L0.C_in, nullptr, 0, nullptr, s);
}

static int run_init_z(dgan_ctx* c, const Workspace& w, const float* z0, uint64_t seed, cudaStream_t s, size_t row_offset = 0) {
  const int latent = c->desc.latent_dim;
  const size_t total4 = (size_t)w.n_pad * latent / 4;
  if (w.mom_counter != nullptr) DGAN_CUDA_CHECK(cudaMemsetAsync(w.mom_counter, 0, (size_t)w.n_pad / kRowTile * sizeof(unsigned), s));
  // fp32 path: the last layer's forward writes dL/dpre for the real rows only while its backward walks all n_pad rows;
  // the tile-padding rows are never observed, but they must not be read uninitialised
  if (w.dblk == nullptr && w.n_pad > w.n_rows)
    DGAN_CUDA_CHECK(cudaMemsetAsync(w.dpre + (size_t)w.n_rows * c->hwc, 0, (size_t)(w.n_pad - w.n_rows) * c->hwc * sizeof(float), s));
  init_z_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, s>>>(w.z, w.v, w.z_h, z0, w.n_rows, w.n_pad, latent, seed,
                                                                 sqrtf(1.0f / (float)latent), row_offset * latent);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// ---- a caller's cotangent dy [n_rows][H*W*C] -> the last layer's d(pre), after a forward that wrote w.y ----------
// fp16 path: per-row power-of-two scales (one shared scale with BatchNorm) in w.loss, d(pre) * scale in w.dblk;
// fp32 path: d(pre) unscaled in w.dpre.  See kernels_vjp.cuh.
static int launch_cotangent(dgan_ctx* c, const Workspace& w, const float* dy, cudaStream_t s) {
  const FinalLayer& f = c->fin;
  const bool tc = c->desc.precision == DGAN_PREC_FP16;
  const bool sigmoid = f.C_out == 1 && f.act == ACT_SIGMOID;
  if (!sigmoid && !(f.C_out == 3 && f.act == ACT_TANH)) { set_error("unsupported final layer"); return DGAN_ERR_UNSUPPORTED; }
  if (tc) {
    if (sigmoid) cotangent_rowmax_kernel<ACT_SIGMOID><<<w.n_rows, 256, 0, s>>>(w.y, dy, c->hwc, w.loss);
    else cotangent_rowmax_kernel<ACT_TANH><<<w.n_rows, 256, 0, s>>>(w.y, dy, c->hwc, w.loss);
    DGAN_LAUNCH_CHECK(c);
    cotangent_scale_kernel<<<1, 1024, 0, s>>>(w.loss, w.n_rows, c->desc.use_bn ? 1 : 0);
    DGAN_LAUNCH_CHECK(c);
  }
  if (tc && w.n_pad > w.n_rows) {
    // the cotangent covers the real rows; the block tensor's tile-padding rows get zeros (the last layer's backward
    // reads all n_pad rows)
    const size_t row_b = (size_t)16 * f.C_out * sizeof(__half);
    DGAN_CUDA_CHECK(cudaMemset2DAsync(w.dblk + (size_t)w.n_rows * 16 * f.C_out, (size_t)w.n_pad * row_b, 0,
                                      (size_t)(w.n_pad - w.n_rows) * row_b, (size_t)c->tc_fin.n_blocks, s));
  }
  const size_t total = (size_t)w.n_rows * c->hwc;
  const unsigned grid = (unsigned)((total + 255) / 256);
  const int w_out = 2 * f.w_in;
#define CT(ACT, CO, BLK) cotangent_kernel<ACT, CO, BLK><<<grid, 256, 0, s>>>(w.y, dy, w.n_rows, w_out, w.loss, w.dpre, w.dblk, w.n_pad)
  if (sigmoid) { if (tc) CT(ACT_SIGMOID, 1, true); else CT(ACT_SIGMOID, 1, false); }
  else { if (tc) CT(ACT_TANH, 3, true); else CT(ACT_TANH, 3, false); }
#undef CT
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

static int check_ws(const dgan_ctx* c, int n_rows, void* ws, size_t ws_bytes, Workspace* out) {
  if (ws == nullptr) { set_error("workspace is NULL"); return DGAN_ERR_WORKSPACE; }
  if (((uintptr_t)ws & 1023) != 0) { set_error("workspace must be 1024-byte aligned"); return DGAN_ERR_WORKSPACE; }
  *out = carve(c, n_rows, ws);
  if (out->bytes > ws_bytes) {
    set_error("workspace too small: need " + std::to_string(out->bytes) + " bytes, got " + std::to_string(ws_bytes));
    return DGAN_ERR_WORKSPACE;
  }
  return 0;
}

// one hidden layer-direction on the tensor cores
static int tcx_launch(dgan_ctx* c, const TcWeights& w1, const TcWeights2& w2, const __half* in, __half* out, int n_pad,
                      int epi, const float* bias, cudaStream_t s, unsigned long long* mb_out,
                      const unsigned long long* mb_in, const CUtensorMap* pre_a, const CUtensorMap* pre_out) {
  TcFinalArgs fa{};
  fa.mb_out = mb_out; fa.mb_in = mb_in;
  return tc2_launch_impl<__half>(c->tc, &c->launches, w1, w2, in, out, n_pad, epi, bias, s, &fa, pre_a, pre_out);
}

// element counts of the weight tensors in creation order (include/defensegan_b200.h, dgan_num_weights)
static std::vector<size_t> weight_counts(const dgan_desc* d) {
  const size_t nd = (size_t)d->net_dim, latent = (size_t)d->latent_dim, feat = 16 * 4 * nd;
  std::vector<size_t> n = {latent * feat, feat};
  if (d->use_bn) { n.push_back(feat); n.push_back(feat); }
  std::vector<std::pair<size_t, size_t>> dc = {{4 * nd, 2 * nd}, {2 * nd, nd}};
  if (d->arch == DGAN_ARCH_CELEBA) { dc.push_back({nd, nd}); dc.push_back({nd, 3}); } else dc.push_back({nd, 1});
  for (size_t i = 0; i < dc.size(); ++i) {
    n.push_back(25 * dc[i].first * dc[i].second); n.push_back(dc[i].second);
    if (d->use_bn && i < 2) { n.push_back(dc[i].second); n.push_back(dc[i].second); }
  }
  return n;
}

static float grad_multiplier(const dgan_ctx* c) {
  float m = 2.0f / (float)c->hwc;  // d/dy mean_{HWC}(y-x)^2
  if (c->desc.precision == DGAN_PREC_FP16) m /= c->tc.grad_scale;
  return m;
}

}  // namespace dgan

// =========================================================================================
// C ABI
// =========================================================================================
namespace {
struct PlanDir { std::string name; int N, K; dgan::PairTable tab; int h, w, force_acc, epi, out_bytes; };
// every tensor-core layer-direction of the fp16 path, as create_impl sets it up (host only)
std::vector<PlanDir> plan_dirs(const dgan_desc* d) {
  using namespace dgan;
  typedef PlanDir Dir;
  const bool celeba = d->arch == DGAN_ARCH_CELEBA;
  const int nd = d->net_dim, latent = d->latent_dim;
  std::vector<Dir> dirs;
  dirs.push_back({"Linear.fwd", 4 * nd, latent, linear_fwd_pairs(16), 4, 4, 0, EPI_BIAS_RELU, 2});
  dirs.push_back({"Linear.bwd", latent, 4 * nd, linear_split_pairs(16), 1, TC_LINEAR_SPLIT, 1, EPI_NONE, 4});
  struct DSpec { int c_in, c_out, h_in, h_used, in_raster; bool relu; };
  std::vector<DSpec> specs;
  if (celeba) specs = {{4 * nd, 2 * nd, 4, 8, 4, true}, {2 * nd, nd, 8, 16, 8, true}, {nd, nd, 16, 32, 16, false}};
  else if (d->use_bn) specs = {{4 * nd, 2 * nd, 4, 8, 4, true}, {2 * nd, nd, 7, 14, 8, true}};   // BN2 sees the 8x8 raster (create_impl)
  else specs = {{4 * nd, 2 * nd, 4, 7, 4, true}, {2 * nd, nd, 7, 14, 7, true}};
  int li = 2;
  for (const DSpec& sp : specs) {
    const std::string nm = "Generator." + std::to_string(li == 4 ? 5 : li);
    const bool bn = d->use_bn && li <= 3;          // a BN layer's GEMMs neither apply the ReLU nor its mask
    dirs.push_back({nm + ".fwd", sp.c_out, sp.c_in, tc_with_zero_tile(deconv_fwd_pairs(sp.h_in, sp.h_in, sp.h_used, sp.h_used, sp.in_raster), kTaps),
                    sp.h_used, sp.h_used, 0, (sp.relu && !bn) ? EPI_BIAS_RELU : EPI_BIAS, 2});
    dirs.push_back({nm + ".bwd", sp.c_in, sp.c_out, tc_with_zero_tile(deconv_bwd_pairs(sp.h_in, sp.h_in, sp.h_used, sp.h_used, sp.in_raster), kTaps),
                    sp.in_raster, sp.in_raster, 0, d->use_bn ? EPI_NONE : EPI_MASK, 2});
    ++li;
  }
  const int fh = celeba ? 32 : 14, c_img = celeba ? 3 : 1;
  dirs.push_back({"last.fwd", 16 * c_img, nd, final_block_fwd_pairs(fh, fh), fh / 2, fh / 2, 0, celeba ? EPI_FINAL_TANH3 : EPI_FINAL_SIGMOID1, 2});
  dirs.push_back({"last.bwd", nd, 16 * c_img, final_block_bwd_pairs(fh, fh), fh, fh, 0, celeba ? EPI_NONE : EPI_MASK, 2});
  return dirs;
}
}  // namespace

extern "C" {

int dgan_abi_version(void) { return DGAN_ABI_VERSION; }
const char* dgan_last_error(void) { return g_last_error.c_str(); }

int dgan_num_weights(const dgan_desc* d) {
  if (d == nullptr) return DGAN_ERR_INVALID_ARG;
  const int n_deconv = d->arch == DGAN_ARCH_CELEBA ? 4 : 3;
  return 2 + 2 * n_deconv + (d->use_bn ? 6 : 0);
}

static int create_impl(dgan_ctx* c, const dgan_desc* d, const float* const* weights_in, cudaStream_t s) {
  c->desc = *d;
  const bool celeba = d->arch == DGAN_ARCH_CELEBA;
  const int nd = d->net_dim, latent = d->latent_dim;
  c->H = celeba ? 64 : 28; c->W = c->H; c->C = celeba ? 3 : 1;
  c->hwc = c->H * c->W * c->C;
  int rc = 0;
  auto fail = [](int code) { return code; };   // the caller destroys the half-built handle
  // The handle owns copies of every weight tensor: the caller may free or reuse `weights_dev` as soon as the
  // copies enqueued here have run (i.e. after synchronising `stream`).
  std::vector<const float*> wown;
  {
    const std::vector<size_t> counts = weight_counts(d);
    size_t total = 0;
    for (size_t n : counts) total += align_up(n * sizeof(float), 256);
    char* base = nullptr;
    if ((rc = dev_alloc(c, (void**)&base, total))) return fail(rc);
    size_t off = 0;
    for (size_t i = 0; i < counts.size(); ++i) {
      cudaError_t e = cudaMemcpyAsync(base + off, weights_in[i], counts[i] * sizeof(float), cudaMemcpyDeviceToDevice, s);
      if (e != cudaSuccess) { set_error(std::string("weight copy: ") + cudaGetErrorString(e)); return fail(DGAN_ERR_CUDA); }
      wown.push_back((const float*)(base + off));
      off += align_up(counts[i] * sizeof(float), 256);
    }
  }
  const float* const* weights = wown.data();

  // ---- Linear (Generator.Input): [1][N][latent] -> [16][N][4*nd]
  {
    GemmLayer L{};
    L.P_in = 1; L.C_in = latent; L.P_out = 16; L.C_out = 4 * nd; L.h_in = 1; L.w_in = 1; L.h_used = 4; L.w_used = 4;
    L.relu = true;
    L.fwd_host = linear_fwd_pairs(16); L.bwd_host = linear_bwd_pairs(16);
    const float* W = weights[0];             // (latent, 16*4nd), column f = pixel*4nd + c
    L.wf = W; L.wf_tile_stride = L.C_out; L.wf_ld = 16 * L.C_out;
    float* Wt = nullptr;                     // [16*4nd][latent]: backward tile q rows = c, cols = latent
    if ((rc = dev_alloc(c, (void**)&Wt, (size_t)latent * 16 * L.C_out * 4))) return fail(rc);
    const size_t total = (size_t)latent * 16 * L.C_out;
    transpose_tiles_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(W, Wt, latent, 16 * L.C_out, total);
    L.wb = Wt; L.wb_tile_stride = L.C_out * latent; L.wb_ld = latent;
    L.bias = weights[1]; L.bias_pstride = L.C_out;   // bias index f = pixel*C_out + c
    if (d->use_bn) { L.bn_offset = weights[2]; L.bn_scale = weights[3]; L.bn_per_pixel = 1; }   // Generator.BN1, axes [0]
    c->layers.push_back(L);
  }
  // ---- hidden deconvs
  struct DSpec { int c_in, c_out, h_in, h_used; bool relu; int in_raster; };
  std::vector<DSpec> specs;
  if (celeba) specs = {{4 * nd, 2 * nd, 4, 8, true, 4}, {2 * nd, nd, 8, 16, true, 8}, {nd, nd, 16, 32, false, 16}};
  else if (d->use_bn)   // BN2's batch statistics cover all 8x8 outputs of Generator.2; the 7x7 crop comes after BN+ReLU
    specs = {{4 * nd, 2 * nd, 4, 8, true, 4}, {2 * nd, nd, 7, 14, true, 8}};
  else specs = {{4 * nd, 2 * nd, 4, 7, true, 4}, {2 * nd, nd, 7, 14, true, 7}};
  int wi = d->use_bn ? 4 : 2;
  int di = 0;
  for (const DSpec& sp : specs) {
    GemmLayer L{};
    L.P_in = sp.in_raster * sp.in_raster; L.C_in = sp.c_in; L.P_out = sp.h_used * sp.h_used; L.C_out = sp.c_out;
    L.h_in = L.w_in = sp.in_raster; L.h_used = L.w_used = sp.h_used; L.relu = sp.relu;
    L.fwd_host = deconv_fwd_pairs(sp.h_in, sp.h_in, sp.h_used, sp.h_used, sp.in_raster);
    L.bwd_host = deconv_bwd_pairs(sp.h_in, sp.h_in, sp.h_used, sp.h_used, sp.in_raster);
    const float* F = weights[wi];            // (5,5,C_out,C_in)
    float* Ff = nullptr;                     // [25][C_in][C_out]
    const size_t total = (size_t)kTaps * sp.c_out * sp.c_in;
    if ((rc = dev_alloc(c, (void**)&Ff, total * 4))) return fail(rc);
    transpose_tiles_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(F, Ff, sp.c_out, sp.c_in, total);
    L.wf = Ff; L.wf_tile_stride = sp.c_in * sp.c_out; L.wf_ld = sp.c_out;
    L.wb = F;  L.wb_tile_stride = sp.c_in * sp.c_out; L.wb_ld = sp.c_in;
    L.bias = weights[wi + 1];
    wi += 2;
    if (d->use_bn && di < 2) {               // Generator.BN2 / BN3 follow Generator.2 / Generator.3 (axes [0,1,2])
      L.bn_offset = weights[wi]; L.bn_scale = weights[wi + 1]; L.bn_per_pixel = 0;
      wi += 2;
    }
    ++di;
    c->layers.push_back(L);
  }
  // ---- final layer
  {
    FinalLayer& f = c->fin;
    f.h_in = f.w_in = celeba ? 32 : 14; f.C_in = nd; f.C_out = c->C; f.act = celeba ? ACT_TANH : ACT_SIGMOID;
    f.w = weights[wi]; f.bias = weights[wi + 1];
    f.n_bands = (2 * f.h_in + kBandRows - 1) / kBandRows;
    f.fwd_smem = ((size_t)kTaps * f.C_out * f.C_in + (size_t)(kBandRows / 2 + 2) * f.w_in * (f.C_in + 4)) * 4;
    f.bwd_smem = (size_t)kTaps * f.C_out * f.C_in * 4;
  }
  // exact in-bounds MACs per latent row (SURVEY 8d / Appendix B)
  c->macs_per_row = 0;
  for (const GemmLayer& L : c->layers) c->macs_per_row += (int64_t)L.fwd_host.pairs.size() * L.C_in * L.C_out;
  {
    PairTable ft = deconv_fwd_pairs(c->fin.h_in, c->fin.w_in, 2 * c->fin.h_in, 2 * c->fin.w_in);
    c->macs_per_row += (int64_t)ft.pairs.size() * c->fin.C_in * c->fin.C_out;
  }
  for (GemmLayer& L : c->layers) {
    if ((rc = upload_table(c, L.fwd_host, &L.fwd, s))) return fail(rc);
    if ((rc = upload_table(c, L.bwd_host, &L.bwd, s))) return fail(rc);
  }
  // opt in to > 48 KB dynamic shared memory where needed
#define OPTIN(K, BYTES) DGAN_CUDA_CHECK(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(BYTES)))
  OPTIN((final_fwd_loss_kernel<float, 1, ACT_SIGMOID>), 100 * 1024);
  OPTIN((final_fwd_loss_kernel<float, 3, ACT_TANH>), 100 * 1024);
  OPTIN((final_fwd_loss_kernel<__half, 1, ACT_SIGMOID>), 100 * 1024);
  OPTIN((final_fwd_loss_kernel<__half, 3, ACT_TANH>), 100 * 1024);
#undef OPTIN
  if (d->precision == DGAN_PREC_FP16) {
    std::vector<TcLayerSpec> tspecs;
    for (GemmLayer& L : c->layers) {
      TcLayerSpec t{};
      t.P_in = L.P_in; t.C_in = L.C_in; t.P_out = L.P_out; t.C_out = L.C_out;
      t.h_in = L.h_in; t.w_in = L.w_in; t.h_used = L.h_used; t.w_used = L.w_used;
      t.fwd = &L.fwd_host; t.bwd = &L.bwd_host;
      t.w_fwd_kmajor_src = (&L == &c->layers[0]) ? nullptr : L.wb;  // F[t][co][ci]: rows co (N), cols ci (K)
      t.w_bwd_kmajor_src = (&L == &c->layers[0]) ? nullptr : L.wf;  // Ff[t][ci][co]: rows ci (N), cols co (K)
      t.linear_W = (&L == &c->layers[0]) ? weights[0] : nullptr;
      t.linear_Wt = (&L == &c->layers[0]) ? L.wb : nullptr;
      t.out_f = &L.tc_f; t.out_b = &L.tc_b; t.bias_pstride = L.bias_pstride;
      tspecs.push_back(t);
    }
    if ((rc = tc_build(c->tc, tspecs, latent, &c->allocs, s))) return fail(rc);
    if ((rc = tc_build_final(c->tc, &c->tc_fin, c->fin.w, c->fin.h_in, c->fin.w_in, c->fin.C_in, c->fin.C_out,
                             c->fin.act, &c->allocs, s)))
      return fail(rc);
    c->tc.allocs = &c->allocs;
    {
      if ((rc = tc2_optin_all())) return fail(rc);
      for (size_t l = 0; l < c->layers.size(); ++l) {
        GemmLayer& L = c->layers[l];
        if ((rc = tc2_build_direction(c->tc, L.tc_f, &L.tc2_f, tc_with_zero_tile(L.fwd_host, L.tc_f.n_tiles - 1), L.h_used, L.w_used, 0, &c->allocs, s))) return fail(rc);
        if (l == 0) {
          const PairTable split = linear_split_pairs(L.P_out);
          if ((rc = tc2_build_direction(c->tc, L.tc_b, &L.tc2_b, split, 1, TC_LINEAR_SPLIT, 1, &c->allocs, s))) return fail(rc);
        } else if ((rc = tc2_build_direction(c->tc, L.tc_b, &L.tc2_b, tc_with_zero_tile(L.bwd_host, L.tc_b.n_tiles - 1), L.h_in, L.w_in, 0, &c->allocs, s))) {
          return fail(rc);
        }
      }
      const PairTable ft = final_block_fwd_pairs(c->fin.h_in, c->fin.w_in), bt = final_block_bwd_pairs(c->fin.h_in, c->fin.w_in);
      if ((rc = tc2_build_direction(c->tc, c->tc_fin.f, &c->tc2_fin_f, ft, c->fin.h_in / 2, c->fin.w_in / 2, 0, &c->allocs, s))) return fail(rc);
      if ((rc = tc2_build_direction(c->tc, c->tc_fin.b, &c->tc2_fin_b, bt, c->fin.h_in, c->fin.w_in, 0, &c->allocs, s))) return fail(rc);
    }
  }
  {
    static const char* lname_m[] = {"Linear", "Generator.2", "Generator.3"};
    static const char* lname_c[] = {"Linear", "Generator.2", "Generator.3", "Generator.5"};
    for (size_t l = 0; l < c->layers.size(); ++l) {
      const std::string nm = celeba ? lname_c[l] : lname_m[l];
      const double macs = (double)c->layers[l].fwd_host.pairs.size() * c->layers[l].C_in * c->layers[l].C_out;
      c->kind_names.push_back(nm + ".fwd"); c->kind_macs_per_row.push_back(macs);
      c->kind_names.push_back(nm + ".bwd"); c->kind_macs_per_row.push_back(macs);
    }
    double fmacs = 0;
    for (const GemmLayer& L : c->layers) fmacs += (double)L.fwd_host.pairs.size() * L.C_in * L.C_out;
    fmacs = (double)c->macs_per_row - fmacs;
    const std::string fn = celeba ? "Generator.6" : "Generator.5";
    c->kind_names.push_back(fn + "+loss.fwd"); c->kind_macs_per_row.push_back(fmacs);
    c->kind_names.push_back(fn + ".bwd"); c->kind_macs_per_row.push_back(fmacs);
    c->kind_names.push_back("momentum"); c->kind_macs_per_row.push_back(0.0);
  }
  DGAN_CUDA_CHECK(cudaStreamCreateWithFlags(&c->cap_stream, cudaStreamNonBlocking));
  DGAN_CUDA_CHECK(cudaGetLastError());
  return DGAN_OK;
}


int dgan_create(dgan_handle* out, const dgan_desc* d, const float* const* weights, int n_weights, void* stream) {
  if (out == nullptr || d == nullptr || weights == nullptr) { set_error("NULL argument"); return DGAN_ERR_INVALID_ARG; }
  *out = nullptr;
  if (d->abi_version != DGAN_ABI_VERSION) { set_error("ABI version mismatch"); return DGAN_ERR_INVALID_ARG; }
  if (d->arch != DGAN_ARCH_MNIST && d->arch != DGAN_ARCH_CELEBA) { set_error("unknown arch"); return DGAN_ERR_INVALID_ARG; }
  if (d->precision != DGAN_PREC_FP32 && d->precision != DGAN_PREC_FP16) { set_error("unknown precision"); return DGAN_ERR_INVALID_ARG; }
  if (d->net_dim <= 0 || d->net_dim % 64 != 0) { set_error("net_dim must be a positive multiple of 64"); return DGAN_ERR_UNSUPPORTED; }
  if (d->latent_dim <= 0 || d->latent_dim % 64 != 0) { set_error("latent_dim must be a positive multiple of 64"); return DGAN_ERR_UNSUPPORTED; }
  if (n_weights != dgan_num_weights(d)) { set_error("wrong number of weight tensors"); return DGAN_ERR_INVALID_ARG; }
  for (int i = 0; i < n_weights; ++i)
    if (weights[i] == nullptr) { set_error("NULL weight pointer"); return DGAN_ERR_INVALID_ARG; }
  int dev_major = 0, dev = 0;
  DGAN_CUDA_CHECK(cudaGetDevice(&dev));
  DGAN_CUDA_CHECK(cudaDeviceGetAttribute(&dev_major, cudaDevAttrComputeCapabilityMajor, dev));
  if (dev_major != 9) { set_error("defensegan_b200 requires an sm_90 (H100) device"); return DGAN_ERR_UNSUPPORTED; }

  dgan_ctx* c = new (std::nothrow) dgan_ctx();
  if (c == nullptr) { set_error("out of host memory"); return DGAN_ERR_INVALID_ARG; }
  const int rc = create_impl(c, d, weights, (cudaStream_t)stream);
  if (rc != DGAN_OK) { dgan_destroy(c); return rc; }   // every failure path frees device memory, streams and events
  *out = c;
  return DGAN_OK;
}

int dgan_destroy(dgan_handle h) {
  if (h == nullptr) return DGAN_OK;
  for (auto& r : h->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  for (void* p : h->allocs) cudaFree(p);
  delete h;
  return DGAN_OK;
}

// fp16 path: plan and upload the schedules of every layer-direction for this many latent rows (cached in the handle).
// Planning allocates and synchronises; it happens here - a caller needs the workspace size before its first
// dgan_reconstruct of a batch size anyway - so that dgan_reconstruct itself only enqueues kernels.
struct TcDir { const TcWeights* w1; TcWeights2* w2; int epi, out_bytes; };
// The tensor-core layer-directions of the fp16 path with the epilogue and output type they launch with, in the order of
// plan_dirs: layer l forward, layer l backward, ..., last layer forward, last layer backward.
static std::vector<TcDir> tc_dirs(dgan_ctx* c) {
  std::vector<TcDir> dirs;
  const int nl = (int)c->layers.size();
  for (int l = 0; l < nl; ++l) {
    GemmLayer& L = c->layers[(size_t)l];
    const bool bn = L.bn_scale != nullptr;        // BN layers: float epilogue (fp32 pre-activations), see run_forward
    dirs.push_back({&L.tc_f, &L.tc2_f, (L.relu && !bn) ? EPI_BIAS_RELU : EPI_BIAS, bn ? 4 : 2});
    if (l == 0) dirs.push_back({&L.tc_b, &L.tc2_b, EPI_NONE, 4});
    else dirs.push_back({&L.tc_b, &L.tc2_b, c->layers[(size_t)l - 1].relu ? EPI_MASK : EPI_NONE, 2});
  }
  dirs.push_back({&c->tc_fin.f, &c->tc2_fin_f, c->tc_fin.C_out == 1 ? EPI_FINAL_SIGMOID1 : EPI_FINAL_TANH3, 2});
  dirs.push_back({&c->tc_fin.b, &c->tc2_fin_b, c->layers[(size_t)nl - 1].relu ? EPI_MASK : EPI_NONE, 2});
  return dirs;
}

static int plan_all(dgan_ctx* c, int n_rows) {
  if (c->desc.precision != DGAN_PREC_FP16) return 0;
  const int n_pad = (int)align_up((size_t)std::max(n_rows, 1), 2 * kRowTile), n_mpairs = n_pad / (2 * kRowTile);
  const int n_pairs = c->tc.num_sms / 2;
  const Tc2Schedule* sc = nullptr;
  int rc;
  for (const TcDir& d : tc_dirs(c))
    if ((rc = tc2_get_schedule(c->tc, *d.w1, *d.w2, n_mpairs, n_pairs, d.epi, d.out_bytes, c->tc.allocs, (cudaStream_t)0, &sc))) return rc;
  return 0;
}

size_t dgan_workspace_bytes(dgan_handle h, int batch, int rec_rr) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0) return 0;
  if (plan_all(h, batch * rec_rr) != 0) return 0;
  return carve(h, batch * rec_rr, nullptr).bytes;
}

int64_t dgan_last_launch_count(dgan_handle h) { return h ? h->last_launches : 0; }
int64_t dgan_last_enqueue_count(dgan_handle h) { return h ? h->last_enqueues : 0; }
int64_t dgan_macs_per_row(dgan_handle h) { return h ? h->macs_per_row : 0; }

int dgan_forward(dgan_handle h, const float* z_dev, int n_rows, float* y_dev, void* ws, size_t ws_bytes, void* stream) {
  if (h == nullptr || z_dev == nullptr || y_dev == nullptr || n_rows <= 0) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  cudaStream_t s = (cudaStream_t)stream;
  Workspace w;
  int rc;
  if ((rc = check_ws(h, n_rows, ws, ws_bytes, &w))) return rc;
  if ((rc = run_init_z(h, w, z_dev, 0, s))) return rc;
  if ((rc = run_forward(h, w, nullptr, 1, 1, false, s))) return rc;
  DGAN_CUDA_CHECK(cudaMemcpyAsync(y_dev, w.y, (size_t)n_rows * h->hwc * 4, cudaMemcpyDeviceToDevice, s));
  return DGAN_OK;
}

int dgan_loss_grad(dgan_handle h, const float* x_dev, int batch, int rec_rr, const float* z_dev, float* y_dev,
                   float* loss_dev, float* grad_dev, void* ws, size_t ws_bytes, void* stream) {
  if (h == nullptr || x_dev == nullptr || z_dev == nullptr || batch <= 0 || rec_rr <= 0) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  cudaStream_t s = (cudaStream_t)stream;
  const int n_rows = batch * rec_rr;
  Workspace w;
  int rc;
  if ((rc = check_ws(h, n_rows, ws, ws_bytes, &w))) return rc;
  if ((rc = run_init_z(h, w, z_dev, 0, s))) return rc;
  if ((rc = run_forward(h, w, x_dev, rec_rr, batch, true, s))) return rc;
  if ((rc = run_backward(h, w, s))) return rc;
  loss_finish_kernel<<<(n_rows + 255) / 256, 256, 0, s>>>(w.loss_part, w.n_loss_parts, w.loss_stride_n, w.loss_stride_b, 1.0f / (float)h->hwc, n_rows, w.loss);
  DGAN_LAUNCH_CHECK(h);
  if (y_dev) DGAN_CUDA_CHECK(cudaMemcpyAsync(y_dev, w.y, (size_t)n_rows * h->hwc * 4, cudaMemcpyDeviceToDevice, s));
  if (loss_dev) DGAN_CUDA_CHECK(cudaMemcpyAsync(loss_dev, w.loss, (size_t)n_rows * 4, cudaMemcpyDeviceToDevice, s));
  if (grad_dev) {
    const size_t n = (size_t)n_rows * h->desc.latent_dim;
    scale_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.g, w.n_g_parts, (size_t)w.n_pad * h->desc.latent_dim,
                                                                  grad_dev, grad_multiplier(h), n, nullptr, 1);
    DGAN_LAUNCH_CHECK(h);
  }
  return DGAN_OK;
}

int dgan_vjp(dgan_handle h, const float* z_dev, int n_rows, const float* dy_dev, float* y_dev, float* dz_dev, void* ws,
             size_t ws_bytes, void* stream) {
  if (h == nullptr || z_dev == nullptr || dy_dev == nullptr || dz_dev == nullptr || n_rows <= 0) {
    set_error("invalid argument");
    return DGAN_ERR_INVALID_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  Workspace w;
  int rc;
  if ((rc = check_ws(h, n_rows, ws, ws_bytes, &w))) return rc;
  h->n_rows_cur = n_rows;     // the FLOPs dgan_profile_read reports refer to this call
  // the forward of dgan_forward, keeping the ReLU masks; the cotangent replaces the loss's (y - x) in the last layer
  if ((rc = run_init_z(h, w, z_dev, 0, s))) return rc;
  if ((rc = run_forward(h, w, nullptr, 1, 1, true, s))) return rc;
  if ((rc = launch_cotangent(h, w, dy_dev, s))) return rc;
  if ((rc = run_backward(h, w, s))) return rc;
  const size_t n = (size_t)n_rows * h->desc.latent_dim;
  const bool tc = h->desc.precision == DGAN_PREC_FP16;
  scale_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.g, w.n_g_parts, (size_t)w.n_pad * h->desc.latent_dim, dz_dev,
                                                                1.f, n, tc ? w.loss : nullptr, h->desc.latent_dim);
  DGAN_LAUNCH_CHECK(h);
  if (y_dev) DGAN_CUDA_CHECK(cudaMemcpyAsync(y_dev, w.y, (size_t)n_rows * h->hwc * 4, cudaMemcpyDeviceToDevice, s));
  return DGAN_OK;
}

int dgan_sample_z0(dgan_handle h, uint64_t seed, uint64_t z_row_offset, int n_rows, float* z_dev, void* stream) {
  if (h == nullptr || z_dev == nullptr || n_rows <= 0) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  const int latent = h->desc.latent_dim;
  const size_t total4 = (size_t)n_rows * latent / 4;
  init_z_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(z_dev, nullptr, nullptr, nullptr, n_rows, n_rows, latent, seed,
                                                                                      sqrtf(1.0f / (float)latent), (size_t)z_row_offset * latent);
  DGAN_LAUNCH_CHECK(h);
  return DGAN_OK;
}

int dgan_reconstruct(dgan_handle h, const dgan_rec_params* prm, const float* x_dev, const float* z0_dev, float* rec_dev,
                     float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  if (h == nullptr || prm == nullptr || x_dev == nullptr || rec_dev == nullptr) { set_error("NULL argument"); return DGAN_ERR_INVALID_ARG; }
  const int batch = prm->batch, rec_rr = prm->rec_rr, rec_iters = prm->rec_iters, decay_lr = prm->decay_lr;
  const float rec_lr = prm->rec_lr, momentum = prm->momentum;
  const uint64_t seed = prm->seed;
  if (batch <= 0 || rec_rr <= 0 || rec_iters <= 0) { set_error("batch, rec_rr and rec_iters must be positive"); return DGAN_ERR_INVALID_ARG; }
  if (ws == nullptr) { set_error("workspace is NULL"); return DGAN_ERR_WORKSPACE; }
  if (((uintptr_t)ws & 1023) != 0) { set_error("workspace must be 1024-byte aligned"); return DGAN_ERR_WORKSPACE; }
  if (dgan_workspace_bytes(h, batch, rec_rr) > ws_bytes) {
    set_error("workspace too small: need " + std::to_string(dgan_workspace_bytes(h, batch, rec_rr)) + " bytes, got " + std::to_string(ws_bytes));
    return DGAN_ERR_WORKSPACE;
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int latent = h->desc.latent_dim;
  Workspace w = carve(h, batch * rec_rr, ws);
  int rc;
  if ((rc = build_maps(h, w))) return rc;
  const int64_t launches0 = h->launches;
  int64_t enqueues = 0;
  h->n_rows_cur = batch * rec_rr;
  if ((rc = run_init_z(h, w, z0_dev, seed, s, (size_t)prm->z_row_offset))) return rc;
  DGAN_CUDA_CHECK(cudaMemcpyAsync(w.x, x_dev, (size_t)batch * h->hwc * sizeof(float), cudaMemcpyDeviceToDevice, s));
  enqueues += (h->launches - launches0) + 1;
  // The L-step loop (a function of the workspace and the hyper-parameters only): everything it reads or writes lives in
  // the workspace, so it can be captured once and replayed.
  auto enqueue_loop = [&](cudaStream_t ls) -> int {
    const int decay_iter = (int)std::ceil(rec_iters * 0.8);
    // fp16: the momentum update (tf.train.MomentumOptimizer, models/gan.py:389-391) runs in the tail of the split-K Linear
    // backward - the CTA that completes a 128-row tile's partial sums applies it - so an L-step is 8 launches; bit-identical
    // to the separate kernel the fp32 path uses (same arithmetic, parts summed in the same order)
    const bool tail = h->desc.precision == DGAN_PREC_FP16;
    for (int t = 0; t < rec_iters; ++t) {
      const bool last = (t == rec_iters - 1);
      float lr = rec_lr;
      if (decay_lr) lr = rec_lr * std::pow(0.1f, (float)(t / decay_iter));
      // The loop returns the pre-update forward of iteration L-1 (models/gan.py:419-421, SURVEY F4):
      // the L-th update is never observed, so its backward pass is not run.
      int r2;
      if ((r2 = run_forward(h, w, w.x, rec_rr, batch, !last, ls, /*want_y=*/last))) return r2;
      if (last) continue;
      MomentumArgs mom;
      mom.lr = lr; mom.mu = momentum; mom.tail = tail;
      if ((r2 = run_backward(h, w, ls, mom))) return r2;
      if (!tail) {
        const size_t zcount = (size_t)w.n_pad * latent;
        ProfScope ps(h, 2 * (int)h->layers.size() + 2, ls);
        DGAN_CUDA_CHECK(launch_pdl(momentum_kernel, dim3((unsigned)((zcount + 255) / 256)), dim3(256), 0, ls, w.z, w.v,
                                   (const float*)w.g, w.n_g_parts, grad_multiplier(h), lr, momentum, zcount, w.z_h));
        DGAN_LAUNCH_CHECK(h);
      }
    }
    return 0;
  };
  bool replayed = false;
  if (!h->profile && h->cap_stream != nullptr) {      // per-kernel event timing needs the plain launches
    dgan_ctx::LoopGraph* g = nullptr;
    for (auto& e : h->graphs)
      if (e.ws == ws && e.batch == batch && e.rec_rr == rec_rr && e.rec_iters == rec_iters && e.decay_lr == decay_lr &&
          e.rec_lr == rec_lr && e.momentum == momentum) { g = &e; break; }
    if (g == nullptr) {
      const int64_t k0 = h->launches;
      cudaGraph_t graph = nullptr;
      if (cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
        const int crc = enqueue_loop(h->cap_stream);
        const cudaError_t ce = cudaStreamEndCapture(h->cap_stream, &graph);
        cudaGraphExec_t exec = nullptr;
        if (crc == 0 && ce == cudaSuccess && graph != nullptr && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) {
          if (h->graphs.size() >= 8) { cudaGraphExecDestroy(h->graphs.front().exec); h->graphs.erase(h->graphs.begin()); }
          h->graphs.push_back({ws, batch, rec_rr, rec_iters, decay_lr, rec_lr, momentum, exec, h->launches - k0});
          g = &h->graphs.back();
        }
        if (graph) cudaGraphDestroy(graph);
      }
      cudaGetLastError();                     // a failed capture falls back to plain launches below
      h->launches = k0;                       // captured nodes are counted when they run
    }
    if (g != nullptr) {
      DGAN_CUDA_CHECK(cudaGraphLaunch(g->exec, s));
      h->launches += g->kernels;
      enqueues += 1;
      replayed = true;
    }
  }
  if (!replayed) {
    const int64_t k0 = h->launches;
    if ((rc = enqueue_loop(s))) return rc;
    enqueues += h->launches - k0;
  }
  {
    const int n_rows = batch * rec_rr;
    loss_finish_kernel<<<(n_rows + 255) / 256, 256, 0, s>>>(w.loss_part, w.n_loss_parts, w.loss_stride_n, w.loss_stride_b, 1.0f / (float)h->hwc, n_rows, w.loss);
    DGAN_LAUNCH_CHECK(h);
    select_kernel<<<batch, 256, 0, s>>>(w.loss, w.y, rec_rr, h->hwc, rec_dev, loss_dev, idx_dev);
    DGAN_LAUNCH_CHECK(h);
    enqueues += 2;
  }
  h->last_enqueues = enqueues;
  h->last_launches = h->launches - launches0;
  return DGAN_OK;
}

int dgan_profile_enable(dgan_handle h, int enable) {
  if (h == nullptr) return DGAN_ERR_INVALID_ARG;
  for (auto& r : h->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  h->prof.clear();
  h->profile = enable != 0;
  return DGAN_OK;
}

int dgan_profile_num_kinds(dgan_handle h) { return h ? (int)h->kind_names.size() : 0; }

const char* dgan_profile_kind_name(dgan_handle h, int kind) {
  if (h == nullptr || kind < 0 || kind >= (int)h->kind_names.size()) return "";
  return h->kind_names[kind].c_str();
}

int dgan_profile_read(dgan_handle h, int max_kinds, double* ms_out, int64_t* launches_out, double* flops_per_launch_out) {
  if (h == nullptr || ms_out == nullptr || launches_out == nullptr || flops_per_launch_out == nullptr) return DGAN_ERR_INVALID_ARG;
  const int nk = std::min(max_kinds, (int)h->kind_names.size());
  for (int k = 0; k < nk; ++k) {
    ms_out[k] = 0.0; launches_out[k] = 0;
    flops_per_launch_out[k] = 2.0 * h->kind_macs_per_row[k] * (double)h->n_rows_cur;
  }
  for (auto& r : h->prof) {
    DGAN_CUDA_CHECK(cudaEventSynchronize(r.b));
    float ms = 0.f;
    DGAN_CUDA_CHECK(cudaEventElapsedTime(&ms, r.a, r.b));
    if (r.kind >= 0 && r.kind < nk) { ms_out[r.kind] += ms; launches_out[r.kind]++; }
    cudaEventDestroy(r.a); cudaEventDestroy(r.b);
  }
  h->prof.clear();
  return DGAN_OK;
}

// Host-only developer/test aid (not in the public header): plan every tensor-core layer-direction of the fp16 path for
// `n_rows` latent rows on `n_pairs` CTA pairs exactly as dgan_create/dgan_reconstruct would, and validate each plan
// with tc2_check_plan.  Needs no GPU.  Returns 0, or an error code with the failing direction in dgan_last_error().
int dgan_debug_check_plans(const dgan_desc* d, int n_rows, int n_pairs, int mutate) {
  using namespace dgan;
  if (d == nullptr || n_rows <= 0 || n_pairs <= 0) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  const int n_pad = ((n_rows + 2 * kRowTile - 1) / (2 * kRowTile)) * 2 * kRowTile, n_mpairs = n_pad / (2 * kRowTile);
  typedef PlanDir Dir;
  const std::vector<Dir> dirs = plan_dirs(d);
  for (const Dir& dr : dirs) {
    if (dr.N != 16 && dr.N != 48 && dr.N != 64 && dr.N != 128 && dr.N != 256) { set_error(dr.name + ": unsupported N"); return DGAN_ERR_UNSUPPORTED; }
    int max_acc = tc2_maxb(dr.N);
    if (dr.force_acc > 0) max_acc = std::min(max_acc, dr.force_acc);
    Tc2Plan plan;
    int rc = tc2_plan(dr.N, dr.K, dr.tab, dr.h, dr.w, max_acc, 0, dr.epi, dr.out_bytes, n_mpairs, n_pairs, &plan);
    if (rc) { set_error(dr.name + ": " + dgan_last_error()); return rc; }
    // self-test of the validator: damage one plan in one specific way - faults 1-11 that of Generator.3 fwd, faults 12-13
    // (specific to narrow ops) that of the last layer's backward; the check must then fail
    if (mutate >= 12 && dr.name == "last.bwd" && plan.stream_m.size() > 40) {
      switch (mutate) {
        case 12: for (TcRec& r : plan.stream_m) r.w[1] = (r.w[1] & 0xFFu) | ((uint32_t)(plan.ksub == 1 ? 2 : 1) << 8); break;   // k16 per op
        case 13: plan.stream_p[20].w[0] |= 1u << 8; break;                 // a k-chunk >= 1 (a narrow K has one)
        default: break;
      }
    }
    if (mutate != 0 && mutate < 12 && dr.name == "Generator.3.fwd" && plan.stream_m.size() > 40) {
      TcRec& m = plan.stream_m[20];
      TcRec* pp = &plan.stream_p[20];
      switch (mutate) {
        case 1: m.w[2] ^= 1u << 6; break;                                   // first-MMA flag of an op
        case 2: {                                                           // accumulator of an op: swap two ops of round 0
                  const int nb = (int)m.w[1];
                  for (int j = 1; j < nb; ++j) {
                    const uint32_t b0 = m.w[2] & 0xFFu, bj = (m.w[2 + j / 4] >> (8 * (j & 3))) & 0xFFu;
                    if (bj == b0) continue;
                    m.w[2] = (m.w[2] & ~0xFFu) | bj;
                    m.w[2 + j / 4] = (m.w[2 + j / 4] & ~(0xFFu << (8 * (j & 3)))) | (b0 << (8 * (j & 3)));
                    break;
                  }
                  break;
                }
        case 3: pp->w[4] ^= 0x01; break;                                    // weight tile of a B slot
        case 4: pp->w[2] ^= 0x01; break;                                    // input pixel of an A tile
        case 5: pp->w[0] = (pp->w[0] & ~(0xFu << 8)) | ((((pp->w[0] >> 8) & 0xF) ^ 1u) << 8); break;   // k-chunk
        case 6: plan.eitems[0] = -1; break;                                 // epilogue list loses an item
        case 7: for (size_t i = 0; i < plan.stream_m.size(); ++i)           // every dep -> 8: ring hazards
                  plan.stream_p[i].w[0] = (plan.stream_p[i].w[0] & ~(0xFu << 19)) | (8u << 19);
                break;
        case 8: pp->w[0] = (pp->w[0] & ~0xFFu) | 0xBFu; break;              // region past the ring
        case 9: std::swap(plan.stream_m[20], plan.stream_m[21]);            // two steps out of order
                std::swap(plan.stream_p[20], plan.stream_p[21]);
                break;
        case 10: plan.maxb = 3;                                              // slots per round without an instantiation
                 for (TcRec& r : plan.stream_m) r.w[1] = 3;
                 break;
        case 11: for (TcRec& r : plan.stream_m) r.w[1] = 2;                 // records disagree with the plan's slots
                 break;
        default: break;
      }
    }
    std::string err;
    if ((rc = tc2_check_plan(dr.N, dr.K, dr.tab, n_mpairs, dr.epi, dr.out_bytes, plan, &err))) { set_error(dr.name + ": " + err); return rc; }
    if (mutate != 0) continue;
    // the plans dgan_debug_force_slots can select: every other slot count this direction has an instantiation for
    for (const Tc2Kind& k : kTc2Kinds) {
      if (k.n != dr.N || k.ksub != plan.ksub || k.epi != dr.epi || k.out_bytes != dr.out_bytes || k.maxb == plan.maxb) continue;
      Tc2Plan forced;
      if ((rc = tc2_plan(dr.N, dr.K, dr.tab, dr.h, dr.w, max_acc, k.maxb, dr.epi, dr.out_bytes, n_mpairs, n_pairs, &forced))) {
        set_error(dr.name + " (" + std::to_string(k.maxb) + " slots): " + dgan_last_error());
        return rc;
      }
      if ((rc = tc2_check_plan(dr.N, dr.K, dr.tab, n_mpairs, dr.epi, dr.out_bytes, forced, &err))) {
        set_error(dr.name + " (" + std::to_string(k.maxb) + " slots): " + err);
        return rc;
      }
    }
  }
  return 0;
}


// Host-side test aid (not in the public header): plan layer-direction `dir` (plan_dirs order) of an fp16 handle with
// exactly `maxb` accumulator slots per round from now on (0: the planner chooses again).  Schedules and captured loops
// are re-made on the next call, so any instantiation of TC2_KINDS can be run at any batch size; the results must not
// change, because every accumulator keeps its summation order.
int dgan_debug_force_slots(dgan_handle h, int dir, int maxb) {
  if (h == nullptr || h->desc.precision != DGAN_PREC_FP16 || maxb < 0) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  const std::vector<TcDir> dirs = tc_dirs(h);
  if (dir < 0 || dir >= (int)dirs.size()) { set_error("layer-direction out of range"); return DGAN_ERR_INVALID_ARG; }
  const TcDir& d = dirs[(size_t)dir];
  if (maxb > 0 && !tc2_has_kind(d.w1->N, maxb, tc2_ksub(d.w1->K), d.epi, d.out_bytes)) {
    set_error("no kernel instantiation with " + std::to_string(maxb) + " accumulator slots per round for this layer-direction");
    return DGAN_ERR_UNSUPPORTED;
  }
  d.w2->force_maxb = maxb;
  d.w2->by_mpairs.clear();                  // the uploaded tables stay in h->allocs until dgan_destroy
  for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
  h->graphs.clear();
  return DGAN_OK;
}

// Host-side test aid: the accumulator slots per round the instantiations of TC2_KINDS offer for layer-direction `dir`,
// written to out[0 .. n).  Returns n, or -1.
int dgan_debug_slot_choices(dgan_handle h, int dir, int* out, int max_n) {
  if (h == nullptr || h->desc.precision != DGAN_PREC_FP16 || out == nullptr) return -1;
  const std::vector<TcDir> dirs = tc_dirs(h);
  if (dir < 0 || dir >= (int)dirs.size()) return -1;
  const TcDir& d = dirs[(size_t)dir];
  int n = 0;
  for (const Tc2Kind& k : kTc2Kinds)
    if (k.n == d.w1->N && k.ksub == tc2_ksub(d.w1->K) && k.epi == d.epi && k.out_bytes == d.out_bytes && n < max_n) out[n++] = k.maxb;
  return n;
}

#ifdef DGAN_PROBE
// Developer build only: copy (and clear) the per-CTA cycle counters of the tensor-core kernels.  out: [48][160][8] u64.
int dgan_debug_probe_read(unsigned long long* out) {
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(out, dgan::g_tc2_probe, sizeof(dgan::g_tc2_probe)) != cudaSuccess) return -1;
  static unsigned long long zeros[48 * 160 * 8];
  if (cudaMemcpyToSymbol(dgan::g_tc2_probe, zeros, sizeof(zeros)) != cudaSuccess) return -1;
  return 0;
}
#endif

// Host-only developer aid (not in the public header): the plan of every layer-direction in numbers - window shape, items,
// steps, MMAs (ops of KSUB k16 each, and k16 MMAs), operand bytes staged from L2 into shared memory (both CTAs of every
// pair), accumulator slots per round - as text.  Layer-direction `force_dir` (plan_dirs order; -1: none) is planned
// with exactly `force_maxb` slots per round, as dgan_debug_force_slots would, and, when force_shape is not NULL, with
// exactly that window shape {wh, ww, sy, sx}.  Returns the length.
static int plan_stats_impl(const dgan_desc* d, int n_rows, int n_pairs, int force_dir, int force_maxb, const int* force_shape,
                           char* buf, int buf_len) {
  using namespace dgan;
  if (d == nullptr || n_rows <= 0 || n_pairs <= 0 || buf == nullptr || buf_len <= 0) { set_error("invalid argument"); return -1; }
  const int n_pad = ((n_rows + 2 * kRowTile - 1) / (2 * kRowTile)) * 2 * kRowTile, n_mpairs = n_pad / (2 * kRowTile);
  std::string out = "direction | N | K | window (h x w, stride) | items | slots | steps | MMAs | staged MB | busiest pair / mean load"
                    " | zero-tile MMA % | MMAs per round | busiest pair: est. tensor us | busiest pair: est. us | k16 MMAs\n";
  double total = 0.0;
  const std::vector<PlanDir> dirs = plan_dirs(d);
  for (size_t di = 0; di < dirs.size(); ++di) {
    const PlanDir& dr = dirs[di];
    int max_acc = tc2_maxb(dr.N);
    if (dr.force_acc > 0) max_acc = std::min(max_acc, dr.force_acc);
    Tc2Plan plan;
    const bool forced = (int)di == force_dir;
    const int rc = tc2_plan(dr.N, dr.K, dr.tab, dr.h, dr.w, max_acc, forced ? force_maxb : 0, dr.epi, dr.out_bytes,
                            n_mpairs, n_pairs, &plan, forced ? force_shape : nullptr);
    if (rc) return -1;
    char line[256];
    const double mb = (double)plan.n_bytes / 1e6;
    total += mb;
    snprintf(line, sizeof line, "%s | %d | %d | %dx%d, %dx%d | %zu | %d | %lld | %lld | %.1f | %.3f | %.1f | %d | %.1f | %.1f | %lld\n", dr.name.c_str(),
             dr.N, dr.K, plan.shape[0], plan.shape[1], plan.shape[2], plan.shape[3], plan.hdrs.size() * (size_t)n_mpairs, plan.n_slots,
             plan.n_steps, plan.n_mma, mb, plan.load_max / std::max(plan.load_mean, 1.0),
             100.0 * (double)plan.n_pad / (double)std::max(plan.n_mma, 1LL), plan.maxb, plan.op_ns_max / 1e3,
             plan.load_max / 1e3, plan.n_mma * plan.ksub);
    out += line;
  }
  char line[64];
  snprintf(line, sizeof line, "total staged MB per L-step | %.1f\n", total);
  out += line;
  const int n = (int)std::min(out.size(), (size_t)buf_len - 1);
  memcpy(buf, out.data(), (size_t)n);
  buf[n] = 0;
  return n;
}

int dgan_debug_plan_stats_slots(const dgan_desc* d, int n_rows, int n_pairs, int force_dir, int force_maxb, char* buf, int buf_len) {
  return plan_stats_impl(d, n_rows, n_pairs, force_dir, force_maxb, nullptr, buf, buf_len);
}

// As dgan_debug_plan_stats_slots, with layer-direction `force_dir` also planned on exactly the window shape wh x ww with
// strides (sy, sx) (force_maxb = 0: any slot count that fits it): plans of two builds compared at the same window.
int dgan_debug_plan_stats_window(const dgan_desc* d, int n_rows, int n_pairs, int force_dir, int force_maxb, int wh, int ww,
                                 int sy, int sx, char* buf, int buf_len) {
  const int shape[4] = {wh, ww, sy, sx};
  return plan_stats_impl(d, n_rows, n_pairs, force_dir, force_maxb, shape, buf, buf_len);
}

int dgan_debug_plan_stats(const dgan_desc* d, int n_rows, int n_pairs, char* buf, int buf_len) {
  return dgan_debug_plan_stats_slots(d, n_rows, n_pairs, -1, 0, buf, buf_len);
}

}  // extern "C"
