// C-ABI of the H100-native Defense-GAN projection loop (see include/defensegan_b200.h).
// Host side: generator plan (pixel-graph tables), weight re-layout, workspace carving and the
// on-device L-step driver.  Everything is enqueued on the caller's stream; nothing here
// synchronises the host.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <memory>
#include <new>

#include "common.cuh"
#include "kernels_simt.cuh"
#include "kernels_tc.cuh"
#include "kernels_tc2.cuh"
#include "kernels_vjp.cuh"
#include "kernels_measured.cuh"
#include "kernels_measured_csr.cuh"
#include "kernels_measured_conv.cuh"
#include "kernels_prune.cuh"
#include "kernels_adam.cuh"
#include "kernels_sparse_dev.cuh"

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

// The generator's channel widths: the latent and the outputs of the Linear (4 * net_dim), of Generator.2 (2 * net_dim)
// and of the later layers (net_dim).
struct Widths { int latent, c4, c2, c1; };
static Widths real_widths(const dgan_desc* d) { return {d->latent_dim, 4 * d->net_dim, 2 * d->net_dim, d->net_dim}; }

// Shared memory of the fp32 last layer's forward (final_fwd_loss_kernel): all 25 taps of the filter and the input rows of
// one band of output rows.
static size_t final_fwd_smem(int c_in, int c_out, int w_in) {
  return ((size_t)kTaps * c_out * c_in + (size_t)(kBandRows / 2 + 2) * w_in * (c_in + 4)) * 4;
}
// dynamic shared memory the fp32 last layer opts in to: the 227 KB a block may have on an H100, less 1 KB for the
// kernels' static shared memory, which counts against the same limit
constexpr int kFinalSmemMax = TC2_SMEM_MAX - 1024;

// The width rule: every channel width a handle stores, padded with exact zeros (weight rows and columns, biases, BN
// offset and scale), so that the padded activations and gradients are exactly 0 and every real output is the unpadded
// sum with zero terms appended - its bits do not change.
//   fp32 path: the next multiple of 64, the output tile of bsgemm_f32_kernel (a width it served before is not padded).
//   fp16 path: the smallest of 64, 128 and 256 that holds the width, the N of a tensor-core instantiation; above 256, the
//              next multiple of 256, computed in column blocks of 256 (tc_directions).  The Linear's output is at least
//              256 wide: its per-pixel bias is served by the N = 256 instantiations only (tc_dir_supported).
//              latent_dim <= 256 and net_dim <= 128 keep every K within 512 channels, 8 k-chunks (tc_records.cuh).
// Returns 0 with the padded widths, or DGAN_ERR_UNSUPPORTED naming the limit.  Creation, tc_directions, carve (through
// the handle) and the plan validator all take their widths from here.
static int padded_widths(const dgan_desc* d, Widths* out) {
  if (d->latent_dim <= 0 || d->net_dim <= 0) { set_error("unsupported widths: latent_dim and net_dim must be positive"); return DGAN_ERR_UNSUPPORTED; }
  const Widths r = real_widths(d);
  if (d->precision == DGAN_PREC_FP16) {
    if (d->latent_dim > 256) { set_error("unsupported latent_dim " + std::to_string(d->latent_dim) + ": the fp16 path takes latent_dim <= 256"); return DGAN_ERR_UNSUPPORTED; }
    if (d->net_dim > 128) { set_error("unsupported net_dim " + std::to_string(d->net_dim) + ": the fp16 path takes net_dim <= 128 (K <= 512 channels)"); return DGAN_ERR_UNSUPPORTED; }
    auto pad = [](int w) { return w <= 64 ? 64 : w <= 128 ? 128 : (w + 255) / 256 * 256; };
    *out = {pad(r.latent), std::max(256, pad(r.c4)), pad(r.c2), pad(r.c1)};
    return 0;
  }
  auto pad = [](int w) { return (w + 63) / 64 * 64; };
  *out = {pad(r.latent), pad(r.c4), pad(r.c2), pad(r.c1)};
  const bool celeba = d->arch == DGAN_ARCH_CELEBA;
  const int c_img = celeba ? 3 : 1, w_in = celeba ? 32 : 14;
  if (final_fwd_smem(out->c1, c_img, w_in) > (size_t)kFinalSmemMax) {
    int max_nd = 64;
    while (final_fwd_smem(max_nd + 64, c_img, w_in) <= (size_t)kFinalSmemMax) max_nd += 64;
    set_error("unsupported net_dim " + std::to_string(d->net_dim) + ": the fp32 last layer holds its filter and input rows in "
              "shared memory, which allows net_dim <= " + std::to_string(max_nd) + (celeba ? " on CelebA" : " on MNIST"));
    return DGAN_ERR_UNSUPPORTED;
  }
  return 0;
}

// The generator's transposed convs between the Linear (4x4 pixels of c4 channels) and the last layer, whose
// input is the last one's output: channels in and out, valid input rows, output rows, input raster, ReLU after the bias.
struct DeconvSpec { int c_in, c_out, h_in, h_used, in_raster; bool relu; };
static std::vector<DeconvSpec> deconv_specs(const dgan_desc* d, const Widths& w) {
  if (d->arch == DGAN_ARCH_CELEBA) return {{w.c4, w.c2, 4, 8, 4, true}, {w.c2, w.c1, 8, 16, 8, true}, {w.c1, w.c1, 16, 32, 16, false}};
  if (d->use_bn)   // BN2's batch statistics cover all 8x8 outputs of Generator.2; the 7x7 crop comes after BN+ReLU
    return {{w.c4, w.c2, 4, 8, 4, true}, {w.c2, w.c1, 7, 14, 8, true}};
  return {{w.c4, w.c2, 4, 7, 4, true}, {w.c2, w.c1, 7, 14, 7, true}};
}

// Every layer-direction of the fp16 path, in launch-site and profile-kind order: layer l forward, layer l backward, ...,
// last layer forward, last layer backward.  A function of the desc alone: the CPU tests plan without a GPU.
// With BatchNorm after a layer (use_bn: the Linear, Generator.2 and Generator.3) its forward writes fp32 pre-activations
// without the ReLU, and the backward into its output applies no mask (the BN backward does both).
// Widths are the padded ones of padded_widths(); a desc it refuses has no directions.  A layer-direction with more than
// 256 output channels becomes one entry per column block of 256, named and profiled as e.g. "Linear.fwd[256:512]".
// tangent: dgan_jvp's pass instead - each layer's forward becomes its tangent direction "<layer>.jvp" (same geometry,
// pair table and weight tiles, no bias, the tangent epilogue: the ReLU mask of the primal forward, none before a
// BatchNorm or without an activation, fp32 for the last layer), and the backward directions are left out (their logical
// indices stay reserved, so an entry's ld names the same layer-direction in both lists).
// weighted: dgan_reconstruct_weighted's pass - the last layer's forward alone, "last.fwd.w", with the weighted final
// epilogue (per-pixel weights of the squared error); its ld and geometry are those of last.fwd.
enum TcPass { TC_PASS_PROJ, TC_PASS_TANGENT, TC_PASS_WEIGHTED };
static std::vector<TcDir> tc_directions(const dgan_desc* d, TcPass pass = TC_PASS_PROJ) {
  const bool tangent = pass == TC_PASS_TANGENT;
  const bool celeba = d->arch == DGAN_ARCH_CELEBA;
  const int c_img = celeba ? 3 : 1;
  std::vector<TcDir> dirs;
  Widths wd;
  if (padded_widths(d, &wd) != 0) return dirs;
  const Widths rw = real_widths(d);
  int ld = 0;
  // n_real: the real output channels of the layer-direction
  auto add = [&](const std::string& name, const std::string& kind, int N, int K, int P_in, int P_out, int n_tiles,
                 PairTable tab, int h_grid, int w_grid, int epi, int out_bytes, int n_real) {
    for (int col0 = 0; col0 < N; col0 += 256) {
      const int nb = std::min(256, N - col0);
      const std::string blk = nb == N ? "" : "[" + std::to_string(col0) + ":" + std::to_string(col0 + nb) + "]";
      TcDir t;
      t.name = name + blk; t.kind = kind + blk; t.base_kind = kind; t.N = nb; t.K = K; t.P_in = P_in; t.P_out = P_out;
      t.n_tiles = n_tiles; t.tab = tab; t.h_grid = h_grid; t.w_grid = w_grid; t.max_acc = tc2_maxb(nb);
      t.epi = epi; t.out_bytes = out_bytes; t.ld = ld; t.col0 = col0; t.out_ld = N; t.n_real = n_real;
      dirs.push_back(std::move(t));
    }
    ++ld;
  };
  // a forward of the projection, or its tangent direction t_name with epilogue t_epi and output type t_bytes
  auto fwd = [&](const std::string& name, const std::string& kind, const std::string& t_name, int N, int K, int P_in,
                 int P_out, int n_tiles, PairTable tab, int h_grid, int w_grid, int epi, int out_bytes, int t_epi, int t_bytes,
                 int n_real) {
    if (tangent) add(t_name, t_name, N, K, P_in, P_out, n_tiles, std::move(tab), h_grid, w_grid, t_epi, t_bytes, n_real);
    else add(name, kind, N, K, P_in, P_out, n_tiles, std::move(tab), h_grid, w_grid, epi, out_bytes, n_real);
  };
  // a GEMM layer's directions have one weight tile more than their pairs use: the all-zero tile of tc_with_zero_tile()
  const bool bn0 = d->use_bn != 0;
  fwd("Linear.fwd", "Linear.fwd", "Linear.jvp", wd.c4, wd.latent, 1, 16, 17, tc_with_zero_tile(linear_fwd_pairs(16), 16), 4, 4,
      bn0 ? EPI_BIAS : EPI_BIAS_RELU, bn0 ? 4 : 2, bn0 ? EPI_NONE : EPI_MASK, 2, rw.c4);
  if (!tangent)
    for (TcDir& t : dirs) t.bias_pstride = wd.c4;   // bias index f = pixel * C_out + c
  // dz as TC_LINEAR_SPLIT partial sums over the 16 pixels, one accumulator per window
  if (tangent) {
    ++ld;
  } else {
    add("Linear.bwd", "Linear.bwd", wd.latent, wd.c4, 16, TC_LINEAR_SPLIT, 17, linear_split_pairs(16), 1, TC_LINEAR_SPLIT,
        EPI_NONE, 4, rw.latent);
    dirs.back().max_acc = 1;
  }
  bool mask_in = !bn0;                               // the backward into the previous layer's output applies its ReLU mask
  const std::vector<DeconvSpec> specs = deconv_specs(d, wd), real_specs = deconv_specs(d, rw);
  int li = 2;
  for (const DeconvSpec& sp : specs) {
    const std::string nm = "Generator." + std::to_string(li == 4 ? 5 : li);
    const bool bn = d->use_bn && li <= 3;
    const DeconvSpec& rs = real_specs[(size_t)(li - 2)];
    fwd(nm + ".fwd", nm + ".fwd", nm + ".jvp", sp.c_out, sp.c_in, sp.in_raster * sp.in_raster, sp.h_used * sp.h_used, kTaps + 1,
        tc_with_zero_tile(deconv_fwd_pairs(sp.h_in, sp.h_in, sp.h_used, sp.h_used, sp.in_raster), kTaps), sp.h_used, sp.h_used,
        (sp.relu && !bn) ? EPI_BIAS_RELU : EPI_BIAS, bn ? 4 : 2, (sp.relu && !bn) ? EPI_MASK : EPI_NONE, 2, rs.c_out);
    if (tangent) ++ld;
    else add(nm + ".bwd", nm + ".bwd", sp.c_in, sp.c_out, sp.h_used * sp.h_used, sp.in_raster * sp.in_raster, kTaps + 1,
        tc_with_zero_tile(deconv_bwd_pairs(sp.h_in, sp.h_in, sp.h_used, sp.h_used, sp.in_raster), kTaps), sp.in_raster,
        sp.in_raster, mask_in ? EPI_MASK : EPI_NONE, 2, rs.c_in);
    mask_in = sp.relu && !bn;
    ++li;
  }
  // the last layer on 4x4 blocks of image pixels (16 weight tiles per direction); its forward computes the loss
  const int fh = specs.back().h_used, n_blocks = (fh / 2) * (fh / 2);
  const std::string fn = celeba ? "Generator.6" : "Generator.5";
  // its tangent: the fp32 tangent of the pre-activation as a block tensor (dgan_jvp applies act'(y))
  fwd("last.fwd", fn + "+loss.fwd", "last.jvp", 16 * c_img, wd.c1, fh * fh, n_blocks, 16, final_block_fwd_pairs(fh, fh), fh / 2,
      fh / 2, celeba ? EPI_FINAL_TANH3 : EPI_FINAL_SIGMOID1, 2, EPI_NONE, 4, 16 * c_img);
  if (tangent) return dirs;
  if (pass == TC_PASS_WEIGHTED) {      // last.fwd is never split (N = 16 * C_out): one entry
    TcDir t = dirs.back();
    t.name = "last.fwd.w"; t.kind = t.base_kind = fn + "+wloss.fwd";
    t.epi = celeba ? EPI_FINAL_TANH3_W : EPI_FINAL_SIGMOID1_W;
    return {t};
  }
  // K: the 16 * C_out real channels of d(pre), no padding (narrow k16 sub-tiles, see Tc2Cfg)
  add("last.bwd", fn + ".bwd", wd.c1, 16 * c_img, n_blocks, fh * fh, 16, final_block_bwd_pairs(fh, fh), fh, fh,
      mask_in ? EPI_MASK : EPI_NONE, 2, rw.c1);
  return dirs;
}

// Can the tensor-core path run layer-direction t?  One check for dgan_create and the plan validator: an instantiation of
// TC2_KINDS has its N, k16 MMAs per op, epilogue and output type; K is whole 64-channel k-chunks, at most 512 channels
// (the 4-bit k-chunk field of the producer record is not checked at run time, tc_records.cuh), or a narrow operand of
// 16-channel sub-tiles; and the planner's tables hold its tiles and pixels.
static int tc_dir_supported(const TcDir& t) {
  const int ksub = tc2_ksub(t.K);
  bool kind = false;
  for (const Tc2Kind& k : kTc2Kinds) kind = kind || (k.n == t.N && k.ksub == ksub && k.epi == t.epi && k.out_bytes == t.out_bytes);
  if (!kind) {
    set_error(t.name + ": unsupported N = " + std::to_string(t.N) + ", K = " + std::to_string(t.K) + ": no tensor-core instantiation");
    return DGAN_ERR_UNSUPPORTED;
  }
  if (t.K <= 0 || t.K > 512 || (t.K % 64 != 0 && (t.K > 48 || t.K % 16 != 0))) {
    set_error(t.name + ": unsupported K = " + std::to_string(t.K) + ": the tensor-core path takes multiples of 64 up to 512 input channels, or 16 / 32 / 48");
    return DGAN_ERR_UNSUPPORTED;
  }
  if (t.n_tiles > 32 || t.P_in > 65535 || t.P_out > 65535) { set_error(t.name + ": unsupported geometry: tensor-core schedule limits exceeded"); return DGAN_ERR_UNSUPPORTED; }
  if (t.bias_pstride != 0 && t.N != 256) { set_error(t.name + ": unsupported N = " + std::to_string(t.N) + ": a per-pixel bias needs N = 256"); return DGAN_ERR_UNSUPPORTED; }
  return 0;
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
  int64_t macs = 0;                   // algorithmic MACs per latent row, at the real widths (padding is not work)
};

struct FinalLayer {
  int h_in, w_in, C_in, C_out, act;
  const float* w = nullptr;  // [25][C_out][C_in] == the TF filter layout
  const float* bias = nullptr;
  int n_bands = 0;
  int n_blocks = 0;          // fp16 path: the 4x4 blocks of image pixels its GEMMs treat as pixels
  size_t fwd_smem = 0, bwd_smem = 0;
};

}  // namespace dgan

using namespace dgan;

struct dgan_ctx {
  dgan_desc desc;
  Widths wd{};                         // the padded widths the handle stores (padded_widths)
  int H = 0, W = 0, C = 0, hwc = 0;
  std::vector<GemmLayer> layers;
  FinalLayer fin;
  std::vector<void*> allocs;
  int64_t macs_per_row = 0;
  int64_t last_launches = 0;
  int64_t launches = 0;
  TcState tc;
  std::vector<TcDir> tc_dirs;          // fp16 path: tc_directions() with weight tiles and schedules
  // fp16 path: dgan_jvp's tangent directions (tc_directions(desc, TC_PASS_TANGENT)) on tc_dirs' weight tiles; made on the
  // first jvp
  std::vector<TcDir> tc_jvp_dirs;
  // fp16 path: the weighted last-layer forward (tc_directions(desc, TC_PASS_WEIGHTED)) on last.fwd's weight tiles; made on
  // the first weighted call
  std::vector<TcDir> tc_w_dirs;
  int tc_order = TC2_ORDER_BAND;       // item order of every fp16 plan (Tc2Order; dgan_debug_force_order)
  // optional per-launch CUDA-event timing (dgan_profile_*): serialises nothing by itself but
  // adds two event records per launch, so it is never enabled in a timed benchmark pass
  bool profile = false;
  int n_rows_cur = 0;
  // The L-step loop of a projection as a CUDA graph: captured once per (workspace, batch, R, L, lr, momentum, decay,
  // weighted, measured: the m of a measured call, 0 otherwise, csr_nnz: the non-zeros of a CSR operator, -1 otherwise,
  // prune: the prune points of a pruned call as iter, keep, iter, keep, ..., empty otherwise; adam: 1 for the Adam
  // update with beta1, beta2 and eps, 0 for momentum; huber: the Huber entries' delta, 0 for the squared error; conv:
  // a convolution operator's kh, kw, ph, pw and stride, empty otherwise - not its kernel values, which are staged outside
  // the graph; prior: 1 for the latent prior with its lambda z_prior, 0 otherwise; sdev: 1 for sparse deviations with
  // their l1 and step, 0 otherwise) on a private stream, replayed with one cudaGraphLaunch per call.
  struct LoopGraph {
    const void* ws; int batch, rec_rr, rec_iters, decay_lr, weighted, measured, csr_nnz; float rec_lr, momentum;
    std::vector<int> prune;
    cudaGraphExec_t exec; int64_t kernels;
    int adam = 0; float beta1 = 0.f, beta2 = 0.f, eps = 0.f;
    float huber = 0.f;
    std::vector<int> conv;
    int prior = 0; float z_prior = 0.f;
    int sdev = 0; float sdev_l1 = 0.f, sdev_step = 0.f;
    bool same_key(const LoopGraph& o) const {
      return ws == o.ws && batch == o.batch && rec_rr == o.rec_rr && rec_iters == o.rec_iters && decay_lr == o.decay_lr &&
             weighted == o.weighted && measured == o.measured && csr_nnz == o.csr_nnz && rec_lr == o.rec_lr &&
             momentum == o.momentum && prune == o.prune && adam == o.adam && beta1 == o.beta1 && beta2 == o.beta2 &&
             eps == o.eps && huber == o.huber && conv == o.conv && prior == o.prior && z_prior == o.z_prior &&
             sdev == o.sdev && sdev_l1 == o.sdev_l1 && sdev_step == o.sdev_step;
    }
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
  ProfScope(dgan_ctx* c_, int kind, cudaStream_t s_) : c(c_), s(s_), on(c_->profile && kind >= 0) {
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

// out[r][c] = s * (sum of the n_parts partial sums of in[r][c], fixed order) for rows of row_len values, read at the
// row stride in_ld (the padded latent width); with row_scale, row r is also divided by row_scale[r] (dgan_vjp: its
// power-of-two cotangent scales, so the division is exact)
__global__ void scale_copy_kernel(const float* __restrict__ in, int n_parts, size_t part_stride,
                                  float* __restrict__ out, float s, size_t n,
                                  const float* __restrict__ row_scale, int row_len, int in_ld) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t r = i / row_len, j = r * in_ld + i % row_len;
  float g = in[j];
  for (int p = 1; p < n_parts; ++p) g += in[j + (size_t)p * part_stride];
  float m = s;
  if (row_scale != nullptr) m /= row_scale[r];
  out[i] = g * m;
}

// The width rule on a weight tensor: dst [A_p][B_p][C_p] = src [A][B][C] where every index is in range, 0 elsewhere.
__global__ void pad_copy_kernel(const float* __restrict__ src, float* __restrict__ dst, int A, int B, int C, int Ap, int Bp,
                                int Cp) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)Ap * Bp * Cp) return;
  const int c = (int)(i % Cp), b = (int)((i / Cp) % Bp), a = (int)(i / ((size_t)Cp * Bp));
  dst[i] = (a < A && b < B && c < C) ? src[((size_t)a * B + b) * C + c] : 0.f;
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
  // fp16 path: the TMA descriptors of each layer-direction's input and output, indexed as tc_dirs (build_maps)
  std::vector<CUtensorMap> map_in, map_out;
  std::vector<CUtensorMap> jmap_in, jmap_out;   // the same for the tangent directions (tc_jvp_dirs), dgan_jvp only
  std::vector<CUtensorMap> wmap_in, wmap_out;   // the same for the weighted last-layer forward (tc_w_dirs), weighted calls only
  unsigned* mom_counter = nullptr;     // fp16 path: [n_pad / 128] tickets of the split-K Linear backward's momentum tail
  __half* dblk = nullptr;              // fp16 path: [n_blocks][n_pad][16 * C_out] scaled dL/dpre of the last layer
  int n_loss_parts = 0, n_g_parts = 1;
  size_t loss_stride_n = 1, loss_stride_b = 1;   // loss_part index = n * stride_n + part * stride_b
  float *y = nullptr, *dpre = nullptr, *loss_part = nullptr;
  float* loss = nullptr;               // [n_pad] per-row loss; dgan_vjp (which computes no loss) keeps its row scales here
  float* x = nullptr;                  // [batch][H*W*C] copy of the call's images (the captured loop reads them from here)
  float* xw = nullptr;                 // weighted workspaces: [batch][H*W*C] copy of the call's per-pixel weights
  // measured workspaces (m > 0; kernels_measured.cuh): the call's operator A [m_ld][H*W*C], its transpose At [H*W*C][m_ld]
  // and measurements y [batch][m_ld], zero-padded to m_ld columns; the residuals r [n_pad][m_ld], dy = (2/m) At r
  // [n_pad][H*W*C], the measured loss's parts [m_ld / 64][n_pad] and the cotangent's row scales [n_pad] (fp16 path)
  int m = 0, m_ld = 0;
  float *am = nullptr, *amt = nullptr, *ym = nullptr, *r = nullptr, *dym = nullptr, *mloss_part = nullptr, *mscale = nullptr;
  // CSR-measured workspaces (csr; kernels_measured_csr.cuh): no am / amt; the staged operator A (a_rp [m_ld + 1], a_ci /
  // a_v [nnz]) and its transpose At (at_rp [H*W*C + 1], at_ci / at_v [nnz]), the rows the validation found bad [m_ld]
  // and the validity flag [1], after all the buffers above
  bool csr = false;
  int nnz = 0;
  int *a_rp = nullptr, *a_ci = nullptr, *at_rp = nullptr, *at_ci = nullptr, *csr_bad = nullptr, *csr_valid = nullptr;
  float *a_v = nullptr, *at_v = nullptr;
  // convolution-measured workspaces (conv; kernels_measured_conv.cuh): no am / amt and no CSR; the geometry and the staged
  // kernels ck [batch][kh][kw], after all the buffers above
  bool conv = false;
  ConvGeom cg{};
  float* ck = nullptr;
  // the regions of a pruned workspace (prune_maps; kernels_prune.cuh), after all the buffers above: each row's original
  // restart index [n_pad] (written by the prune point that fills the region; the first region's rows are restarts
  // 0 .. R-1 of each image and leave it unwritten), the row of the previous region each row was gathered from [n_pad],
  // and select_kernel's choice per image among its survivors [n_pad] (the last region's only)
  int *orig = nullptr, *src = nullptr, *sel = nullptr;
  // Adam workspaces (kernels_adam.cuh), after all the buffers above: the second moment s [n_pad][latent_pad]; the first
  // moment lives in v, the momentum buffer
  float* s = nullptr;
  size_t bytes = 0;
  // The data term of the call the workspace serves: the Huber loss at this delta (> 0, +inf allowed; the Huber entries),
  // or 0 for the squared error.  Set by the call, not carved: a Huber call's workspace is its counterpart's.
  float huber = 0.f;
  // The latent prior of the call (the prior entries): each row's objective is J = D + z_prior ||z||^2 with z_prior >= 0.
  // Set by the call, not carved: the prior term lives in `loss` between its evaluation and the loss's finish.
  bool prior = false;
  float z_prior = 0.f;
  // Sparse deviations (the *_sparse_dev entries; kernels_sparse_dev.cuh), after all the buffers above: each row's
  // deviation nu [n_pad][H*W*C] and u = G(z) + nu [n_pad][H*W*C], which the data term reads in place of y.  ident: the
  // image loss run through the measured loop as the identity operator (m = H*W*C), with the measured row buffers dym,
  // mloss_part and mscale carved before nu.  eta, tau and l1 are set by the call.
  float *nu = nullptr, *u = nullptr;
  bool ident = false;
  float sdev_eta = 0.f, sdev_tau = 0.f, sdev_l1 = 0.f;
};

// The padded measurement count of a measured workspace: m rounded up to the measurement products' N tile.
static int measured_ld(int m) { return (int)align_up((size_t)m, kMeasTileN); }

// The next buffer of a workspace being carved from b (NULL: sizes only) at *off: the dims' product of elements of type
// `type`, one of the element types below, 1024-byte aligned.  layout (not NULL) receives its line: name, element type,
// byte offset and dims in storage order (outermost first).
static void* carve_take(char* b, size_t* off, std::string* layout, const std::string& name, const char* type,
                        std::initializer_list<size_t> dims) {
  struct ElemType { const char* name; size_t bytes; };
  static const ElemType kTypes[] = {{"f32", 4}, {"f16", 2}, {"u64", 8}, {"u32", 4}, {"i32", 4}};
  size_t bytes = 0;
  for (const ElemType& t : kTypes)
    if (strcmp(t.name, type) == 0) bytes = t.bytes;
  for (size_t d : dims) bytes *= d;
  if (layout != nullptr) {
    *layout += name + " " + type + " " + std::to_string(*off);
    for (size_t d : dims) *layout += " " + std::to_string(d);
    *layout += "\n";
  }
  void* p = b ? (void*)(b + *off) : nullptr;
  *off += align_up(bytes, 1024);
  return p;
}

// The staged CSR operator of a workspace w whose m_ld is set, for nnz non-zeros: a_rp [m_ld + 1], a_ci / a_v [nnz], the
// transpose's at_rp [H*W*C + 1], at_ci / at_v [nnz], csr_bad [m_ld] and csr_valid [1] (carve_take's arguments).
static void carve_csr(const dgan_ctx* c, Workspace* w, int nnz_, char* b, size_t* off, std::string* layout) {
  const size_t mld = (size_t)w->m_ld, hwc = (size_t)c->hwc, nnz = (size_t)nnz_;
  w->nnz = nnz_;
  w->a_rp = (int*)carve_take(b, off, layout, "a_rp", "i32", {mld + 1});
  w->a_ci = (int*)carve_take(b, off, layout, "a_ci", "i32", {nnz});
  w->a_v = (float*)carve_take(b, off, layout, "a_v", "f32", {nnz});
  w->at_rp = (int*)carve_take(b, off, layout, "at_rp", "i32", {hwc + 1});
  w->at_ci = (int*)carve_take(b, off, layout, "at_ci", "i32", {nnz});
  w->at_v = (float*)carve_take(b, off, layout, "at_v", "f32", {nnz});
  w->csr_bad = (int*)carve_take(b, off, layout, "csr_bad", "i32", {mld});
  w->csr_valid = (int*)carve_take(b, off, layout, "csr_valid", "i32", {1});
}

// What a projection's workspace holds beyond the generator's buffers, and how it is split into stages (carve,
// plan_workspace).  weighted: the image loss's per-pixel weights.  m > 0: a measured loss for m measurements; nnz >= 0 a
// CSR operator with nnz non-zeros, conv (not NULL, nnz -1) a convolution, neither a dense operator.  adam: Adam's second
// moment.  sdev: the sparse deviations.  n_points > 0: a pruned projection with the prune points sched, one region per
// stage; 0: unpruned, one workspace.
struct WsShape {
  bool weighted = false;
  int m = 0, nnz = -1;
  const ConvGeom* conv = nullptr;
  bool adam = false, sdev = false;
  const dgan_prune_point* sched = nullptr;
  int n_points = 0;
};

// The workspace's buffers, in carve() order: layout (not NULL) receives one line per buffer (carve_take) for
// dgan_debug_workspace_layout.  sh.weighted: the workspace of the weighted entries, the same buffers at the same offsets
// and the weights "xw" after all of them.  sh.m > 0: the workspace of the measured entries for m measurements, the same
// buffers at the same offsets and the measured ones after all of them.  sh.nnz >= 0: the CSR-measured workspace, the
// measured buffers without am / amt and the CSR ones after all of them.  sh.conv: the convolution-measured workspace, the
// measured buffers without am / amt and the staged kernels "ck" after all of them.  sh.n_points > 0: one region of a
// pruned workspace (plan_workspace), the maps "orig", "src" and "sel" after all the other buffers.  op (not NULL, with
// m > 0): a region of a pruned measured workspace, whose operator - am / amt, the CSR buffers or ck - and ym live in the
// operator block op (carve_operator): only the row-sized measured buffers are carved, the others are op's.  sh.adam: the
// workspace of the Adam entries, the same buffers at the same offsets and the second moment "s" after all of them.
// sh.sdev: the workspace of the sparse-deviation entries, the same buffers at the same offsets and then - for the image
// loss (m = 0), which runs the measured loop as the identity operator - "dym", "mloss_part" and "mscale" as a measured
// workspace for m = H*W*C carves them, then "nu" and "u" [n_pad][H*W*C].
static Workspace carve(const dgan_ctx* c, int n_rows, void* base, std::string* layout, const WsShape& sh,
                       const Workspace* op = nullptr) {
  Workspace w;
  w.n_rows = n_rows;
  w.n_pad = (int)align_up((size_t)std::max(n_rows, 1), c->desc.precision == DGAN_PREC_FP16 ? 2 * kRowTile : kRowTile);
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](const std::string& name, const char* type, std::initializer_list<size_t> dims) -> void* {
    return carve_take(b, &off, layout, name, type, dims);
  };
  const size_t np = (size_t)w.n_pad;
  const size_t latent = (size_t)c->wd.latent;      // z, v, g and z_h are stored at the padded latent width
  const bool tc = c->desc.precision == DGAN_PREC_FP16;
  w.n_g_parts = tc ? TC_LINEAR_SPLIT : 1;
  w.n_loss_parts = tc ? c->fin.n_blocks : c->fin.n_bands;
  if (layout != nullptr) {
    *layout += "n_rows " + std::to_string(n_rows) + "\nn_pad " + std::to_string(np) + "\nwidths " +
               std::to_string(c->wd.latent) + " " + std::to_string(c->wd.c4) + " " + std::to_string(c->wd.c2) + " " +
               std::to_string(c->wd.c1) + "\ng_parts " + std::to_string(w.n_g_parts) + "\n";
  }
  w.z = (float*)take("z", "f32", {np, latent});
  w.v = (float*)take("v", "f32", {np, latent});
  w.g = (float*)take("g", "f32", {(size_t)w.n_g_parts, np, latent});
  if (tc) w.z_h = (__half*)take("z_h", "f16", {np, latent});
  if (tc) w.mom_counter = (unsigned*)take("mom_counter", "u32", {np / kRowTile});
  if (tc) w.dblk = (__half*)take("dblk", "f16", {(size_t)c->fin.n_blocks, np, (size_t)16 * c->fin.C_out});
  w.loss_stride_n = tc ? 1 : (size_t)w.n_loss_parts;          // fp16 path: [block][n_pad] (coalesced epilogue stores)
  w.loss_stride_b = tc ? (size_t)np : 1;
  for (size_t i = 0; i < c->layers.size(); ++i) {
    const GemmLayer& l = c->layers[i];
    const std::string li = "." + std::to_string(i);
    const size_t P = (size_t)l.P_out, C = (size_t)l.C_out;
    const size_t G = l.bn_per_pixel ? P * C : C;
    if (tc) {
      w.act_h.push_back((__half*)take("act_h" + li, "f16", {P, np, C}));
      w.dact_h.push_back((__half*)take("dact_h" + li, "f16", {P, np, C}));
      w.maskbits.push_back((unsigned long long*)take("mask" + li, "u64", {P, np, C / 64}));
      if (l.bn_scale != nullptr) {
        w.pre_h.push_back((float*)take("pre_h" + li, "f32", {P, np, C}));
        w.bn_part.push_back((float*)take("bn_part" + li, "f32", {4, (size_t)kBnSplits, G}));
      } else {
        w.pre_h.push_back(nullptr);
        w.bn_part.push_back(nullptr);
      }
    } else {
      w.act.push_back((float*)take("act" + li, "f32", {P, np, C}));
      w.dact.push_back((float*)take("dact" + li, "f32", {P, np, C}));
      if (l.bn_scale != nullptr) {
        w.pre.push_back((float*)take("pre" + li, "f32", {P, np, C}));
        w.bn_part.push_back((float*)take("bn_part" + li, "f32", {4, (size_t)kBnSplits, G}));
      } else {
        w.pre.push_back(nullptr);
        w.bn_part.push_back(nullptr);
      }
    }
  }
  const size_t hwc = (size_t)c->hwc;
  w.x = (float*)take("x", "f32", {np, hwc});     // batch <= n_pad
  w.y = (float*)take("y", "f32", {np, hwc});
  w.dpre = (float*)take("dpre", "f32", {np, hwc});
  if (tc) w.loss_part = (float*)take("loss_part", "f32", {(size_t)w.n_loss_parts, np});
  else w.loss_part = (float*)take("loss_part", "f32", {np, (size_t)w.n_loss_parts});
  w.loss = (float*)take("loss", "f32", {np});
  if (sh.weighted) w.xw = (float*)take("xw", "f32", {np, hwc});   // batch <= n_pad
  if (sh.m > 0) {
    w.m = sh.m;
    w.m_ld = measured_ld(sh.m);
    const size_t mld = (size_t)w.m_ld;
    w.csr = sh.nnz >= 0;
    w.conv = sh.conv != nullptr;
    if (!w.csr && !w.conv && op == nullptr) {
      w.am = (float*)take("am", "f32", {mld, hwc});
      w.amt = (float*)take("amt", "f32", {hwc, mld});
    }
    if (op == nullptr) w.ym = (float*)take("ym", "f32", {np, mld});            // batch <= n_pad
    w.r = (float*)take("r", "f32", {np, mld});
    w.dym = (float*)take("dym", "f32", {np, hwc});
    w.mloss_part = (float*)take("mloss_part", "f32", {mld / kMeasTileN, np});
    w.mscale = (float*)take("mscale", "f32", {np});
    if (op != nullptr) {
      w.am = op->am; w.amt = op->amt; w.ym = op->ym;
      w.nnz = op->nnz;
      w.a_rp = op->a_rp; w.a_ci = op->a_ci; w.a_v = op->a_v;
      w.at_rp = op->at_rp; w.at_ci = op->at_ci; w.at_v = op->at_v;
      w.csr_bad = op->csr_bad; w.csr_valid = op->csr_valid;
      w.cg = op->cg; w.ck = op->ck;
    } else if (w.csr) {
      carve_csr(c, &w, sh.nnz, b, &off, layout);
    } else if (w.conv) {
      w.cg = *sh.conv;
      w.ck = (float*)take("ck", "f32", {np, (size_t)sh.conv->kh * sh.conv->kw});      // batch <= n_pad
    }
  }
  if (sh.n_points > 0) {
    w.orig = (int*)take("orig", "i32", {np});
    w.src = (int*)take("src", "i32", {np});
    w.sel = (int*)take("sel", "i32", {np});     // batch <= n_pad
  }
  if (sh.adam) w.s = (float*)take("s", "f32", {np, latent});
  if (sh.sdev && sh.m == 0) {
    w.ident = true;
    w.m = c->hwc;
    w.m_ld = measured_ld(c->hwc);
    w.dym = (float*)take("dym", "f32", {np, hwc});
    w.mloss_part = (float*)take("mloss_part", "f32", {(size_t)w.m_ld / kMeasTileN, np});
    w.mscale = (float*)take("mscale", "f32", {np});
  }
  if (sh.sdev) {
    w.nu = (float*)take("nu", "f32", {np, hwc});
    w.u = (float*)take("u", "f32", {np, hwc});
  }
  w.bytes = off;
  return w;
}

// The operator block of a pruned measured workspace, shared by all its regions: the staged operator - "am" / "amt" as in
// carve, or (sh.nnz >= 0) carve's CSR buffers, or (sh.conv) the kernels "ck" [batch][kh][kw] - then the measurements
// "ym" [batch][m_ld].  Only the operator's buffers, m, m_ld, csr, nnz, conv and cg are set.
static Workspace carve_operator(const dgan_ctx* c, int batch, const WsShape& sh, void* base, std::string* layout) {
  Workspace w;
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](const std::string& name, const char* type, std::initializer_list<size_t> dims) -> void* {
    return carve_take(b, &off, layout, name, type, dims);
  };
  const size_t hwc = (size_t)c->hwc;
  w.m = sh.m;
  w.m_ld = measured_ld(sh.m);
  const size_t mld = (size_t)w.m_ld;
  w.csr = sh.nnz >= 0;
  w.conv = sh.conv != nullptr;
  if (w.csr) {
    carve_csr(c, &w, sh.nnz, b, &off, layout);
  } else if (w.conv) {
    w.cg = *sh.conv;
    w.ck = (float*)take("ck", "f32", {(size_t)batch, (size_t)sh.conv->kh * sh.conv->kw});
  } else {
    w.am = (float*)take("am", "f32", {mld, hwc});
    w.amt = (float*)take("amt", "f32", {hwc, mld});
  }
  w.ym = (float*)take("ym", "f32", {(size_t)batch, mld});
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

// xw (not NULL, with x): the per-pixel weights of the squared error (the WEIGHTED instantiations).  w.huber > 0 (with x):
// the Huber loss (final_fwd_huber_kernel) instead of the squared error.
template <typename TIN>
static int launch_final_fwd(dgan_ctx* c, const TIN* hin, const Workspace& w, const float* x, int R, int B,
                            bool want_grad, cudaStream_t s, const float* xw = nullptr) {
  const FinalLayer& f = c->fin;
  dim3 grid(w.n_rows, f.n_bands), block(128);
  const size_t smem = f.fwd_smem;
  float* dpre = want_grad ? w.dpre : nullptr;
  float* lp = x ? w.loss_part : nullptr;
#define FF(CO, ACT, WT)                                                                                         \
  final_fwd_loss_kernel<TIN, CO, ACT, WT><<<grid, block, smem, s>>>(hin, w.n_pad, f.h_in, f.w_in, f.C_in, f.w, \
                                                                    f.bias, x, R, B, w.y, dpre ? dpre : w.dpre, lp, xw)
#define FH(CO, ACT, WT)                                                                                          \
  final_fwd_huber_kernel<TIN, CO, ACT, WT><<<grid, block, smem, s>>>(hin, w.n_pad, f.h_in, f.w_in, f.C_in, f.w, f.bias, x, R, \
                                                                     B, w.y, dpre ? dpre : w.dpre, lp, xw, w.huber)
  const bool wt = xw != nullptr && x != nullptr;
  const bool hub = w.huber > 0.f && x != nullptr;
  if (f.C_out == 1 && f.act == ACT_SIGMOID) {
    if (hub) { if (wt) FH(1, ACT_SIGMOID, true); else FH(1, ACT_SIGMOID, false); }
    else if (wt) FF(1, ACT_SIGMOID, true); else FF(1, ACT_SIGMOID, false);
  } else if (f.C_out == 3 && f.act == ACT_TANH) {
    if (hub) { if (wt) FH(3, ACT_TANH, true); else FH(3, ACT_TANH, false); }
    else if (wt) FF(3, ACT_TANH, true); else FF(3, ACT_TANH, false);
  } else { set_error("unsupported final layer"); return DGAN_ERR_UNSUPPORTED; }
#undef FF
#undef FH
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

// What logical layer-direction i of the fp16 path (TcDir::ld) reads and writes in workspace w, at full width.  mask: the
// 1-bit ReLU masks of the activation it writes (forward) or whose gradient it writes (backward); bias: its epilogue's.
struct TcIo { const void* in; void* out; unsigned long long* mask; const float* bias; };
// tangent (dgan_jvp, forward slots only): the tangent of z (in z_h) and of each layer's output (in dact_h), the last
// layer's into w.dpre; masks are the primal forward's.  The weighted pass reads and writes what the projection's does.
static TcIo tc_io(const dgan_ctx* c, const Workspace& w, int i, TcPass pass = TC_PASS_PROJ) {
  const int nl = (int)c->layers.size(), l = i / 2;
  if (pass == TC_PASS_TANGENT)
    return i == 2 * nl ? TcIo{w.dact_h[nl - 1], w.dpre, nullptr, nullptr}
                       : TcIo{l == 0 ? (const void*)w.z_h : w.dact_h[l - 1], w.dact_h[l], w.maskbits[l], nullptr};
  if (i == 2 * nl) return {w.act_h[nl - 1], w.dblk, nullptr, c->fin.bias};
  if (i % 2 == 0)       // a BatchNorm layer's GEMM writes its fp32 pre-activations
    return {l == 0 ? (const void*)w.z_h : w.act_h[l - 1], w.pre_h[l] ? (void*)w.pre_h[l] : w.act_h[l], w.maskbits[l],
            c->layers[l].bias};
  if (l == 0) return {w.dact_h[0], w.g, nullptr, nullptr};
  return {l == nl ? w.dblk : w.dact_h[l], w.dact_h[l - 1], w.maskbits[l - 1], nullptr};
}

// The layer-directions of a pass and the workspace's tensor maps of them.
static const std::vector<TcDir>& pass_dirs(const dgan_ctx* c, TcPass pass) {
  return pass == TC_PASS_TANGENT ? c->tc_jvp_dirs : pass == TC_PASS_WEIGHTED ? c->tc_w_dirs : c->tc_dirs;
}
template <typename WS>   // Workspace or const Workspace
static auto& pass_maps_in(WS& w, TcPass pass) {
  return pass == TC_PASS_TANGENT ? w.jmap_in : pass == TC_PASS_WEIGHTED ? w.wmap_in : w.map_in;
}
template <typename WS>
static auto& pass_maps_out(WS& w, TcPass pass) {
  return pass == TC_PASS_TANGENT ? w.jmap_out : pass == TC_PASS_WEIGHTED ? w.wmap_out : w.map_out;
}

// Encode the TMA descriptors of every layer-direction's input and output for this workspace (of the pass's directions).
static int build_maps(dgan_ctx* c, Workspace& w, TcPass pass = TC_PASS_PROJ) {
  if (c->desc.precision != DGAN_PREC_FP16) return 0;
  const std::vector<TcDir>& dirs = pass_dirs(c, pass);
  std::vector<CUtensorMap>& map_in = pass_maps_in(w, pass);
  std::vector<CUtensorMap>& map_out = pass_maps_out(w, pass);
  map_in.assign(dirs.size(), CUtensorMap{});
  map_out.assign(dirs.size(), CUtensorMap{});
  int rc;
  for (size_t i = 0; i < dirs.size(); ++i) {
    const TcDir& t = dirs[i];
    const TcIo io = tc_io(c, w, t.ld, pass);
    if ((rc = tc_make_map(c->tc, &map_in[i], io.in, (uint64_t)t.K, (uint64_t)w.n_pad, (uint64_t)t.P_in, 128, tc2_box_k(t.K))))
      return rc;
    map_out[i] = map_in[i];          // a placeholder where the epilogue does not store through TMA
    // the full-width output: a column block stores at its channel offset (TcFinalArgs::col0)
    if (tc2_tma_epilogue(t.N, t.epi, t.out_bytes) &&
        (rc = tc_make_map(c->tc, &map_out[i], io.out, (uint64_t)t.out_ld, (uint64_t)w.n_pad, (uint64_t)t.P_out, TC2_STORE_ROWS)))
      return rc;
  }
  return 0;
}

// Logical layer-direction ld of the fp16 path on workspace w: every column block of it, with the epilogue, output type
// and masks its table entries imply.  want_mask: a forward with the ReLU also stores its masks.  fa: the last layer's and
// the momentum tail's arguments.  Each block of a split layer-direction is profiled as its own kind (its tc_dirs index);
// an unsplit one is profiled by the caller, together with the BatchNorm kernels that follow it.  pass: the tangent
// direction of ld (dgan_jvp; not profiled) or its weighted one (the last layer's forward; profiled by the caller).
static int tc_launch(dgan_ctx* c, const Workspace& w, int ld, cudaStream_t s, bool want_mask = false, TcFinalArgs fa = TcFinalArgs{},
                     TcPass pass = TC_PASS_PROJ) {
  const TcIo io = tc_io(c, w, ld, pass);
  const std::vector<TcDir>& dirs = pass_dirs(c, pass);
  const std::vector<CUtensorMap>& maps_in = pass_maps_in(w, pass);
  const std::vector<CUtensorMap>& maps_out = pass_maps_out(w, pass);
  for (size_t i = 0; i < dirs.size(); ++i) {
    const TcDir& t = dirs[i];
    if (t.ld != ld) continue;
    ProfScope ps(c, t.N == t.out_ld || pass != TC_PASS_PROJ ? -1 : (int)i, s);
    TcFinalArgs f = fa;
    const size_t words = (size_t)t.col0 / 64;          // mask words before the block's channels
    if (t.epi == EPI_BIAS_RELU && want_mask) f.mb_out = io.mask + words;
    if (t.epi == EPI_MASK) f.mb_in = io.mask + words;
    f.out_ld = t.out_ld;
    f.col0 = t.col0;
    void* out = t.out_bytes == 4 ? (void*)((float*)io.out + t.col0) : (void*)((__half*)io.out + t.col0);
    const float* bias = io.bias != nullptr ? io.bias + t.col0 : nullptr;
    if (int rc = tc2_launch(&c->launches, t, maps_in[i], maps_out[i], out, w.n_pad, bias, s, f)) return rc;
  }
  return 0;
}

// The profile kind of logical layer-direction ld when it is one launch (-1 when it is split into column blocks: those
// are profiled by tc_launch).  fp16 kinds are the tc_dirs entries, fp32 kinds the logical layer-directions.
static int prof_kind(const dgan_ctx* c, int ld) {
  if (c->desc.precision != DGAN_PREC_FP16) return ld;
  for (size_t i = 0; i < c->tc_dirs.size(); ++i)
    if (c->tc_dirs[i].ld == ld) return c->tc_dirs[i].N == c->tc_dirs[i].out_ld ? (int)i : -1;
  return -1;
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
// tangent (dgan_jvp): dact holds the tangent of pre and becomes the tangent of act, in place (bn_apply_jvp_kernel)
template <typename TP, typename T>
static int bn_backward_t(dgan_ctx* c, const Workspace& w, int l, const TP* pre, const T* act, T* dact, cudaStream_t s,
                         bool tangent = false) {
  const GemmLayer& L = c->layers[l];
  const int G = L.bn_per_pixel ? L.P_out * L.C_out : L.C_out;
  float* part = w.bn_part[l];
  float *mean_p = part, *var_p = part + (size_t)kBnSplits * G, *s1_p = part + (size_t)2 * kBnSplits * G,
        *s2_p = part + (size_t)3 * kBnSplits * G;
  dim3 rgrid(G / 32, kBnSplits);
  const size_t total = (size_t)L.P_out * w.n_pad * L.C_out;
  const unsigned grid = (unsigned)((total + 255) / 256);
  if (tangent) {
    bn_reduce_kernel<3, TP, T><<<rgrid, 256, 0, s>>>(pre, act, dact, mean_p, var_p, L.P_out, w.n_rows, w.n_pad, L.C_out,
                                                 L.bn_per_pixel, s1_p, s2_p);
    DGAN_LAUNCH_CHECK(c);
    bn_apply_jvp_kernel<TP, T><<<grid, 256, 0, s>>>(pre, act, mean_p, var_p, s1_p, s2_p, L.bn_scale, L.P_out, w.n_rows, w.n_pad,
                                                   L.C_out, L.bn_per_pixel, dact);
    DGAN_LAUNCH_CHECK(c);
    return 0;
  }
  bn_reduce_kernel<2, TP, T><<<rgrid, 256, 0, s>>>(pre, act, dact, mean_p, var_p, L.P_out, w.n_rows, w.n_pad, L.C_out,
                                               L.bn_per_pixel, s1_p, s2_p);
  DGAN_LAUNCH_CHECK(c);
  bn_apply_bwd_kernel<TP, T><<<grid, 256, 0, s>>>(pre, act, mean_p, var_p, s1_p, s2_p, L.bn_scale, L.P_out,
                                                 w.n_rows, w.n_pad, L.C_out, L.bn_per_pixel, dact);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// ---- one generator forward (+ loss and dL/dpre when x != null; weighted per pixel by xw when that is not null too) ----
static int run_forward(dgan_ctx* c, const Workspace& w, const float* x, int R, int B, bool want_grad,
                       cudaStream_t s, bool want_y = true, const float* xw = nullptr) {
  int rc;
  const int nl = (int)c->layers.size();
  if (c->desc.precision == DGAN_PREC_FP16) {
    for (int l = 0; l < nl; ++l) {
      ProfScope ps(c, prof_kind(c, 2 * l), s);
      if ((rc = tc_launch(c, w, 2 * l, s, want_grad))) return rc;
      // with BatchNorm the GEMM wrote pre = GEMM + bias (fp32):  act = relu(BN_batchstat(pre)) (fp16)
      if (c->layers[l].bn_scale != nullptr && (rc = bn_forward_t<float, __half>(c, w, l, w.pre_h[l], w.act_h[l], s))) return rc;
    }
    ProfScope ps(c, prof_kind(c, 2 * nl), s);
    TcFinalArgs fa{};
    fa.x = x; fa.y = w.y; fa.loss_part = w.loss_part; fa.R = R; fa.B = B; fa.n_rows = w.n_rows;
    fa.nbx = c->fin.w_in / 2; fa.w_out = 2 * c->fin.w_in; fa.gscale = c->tc.grad_scale; fa.write_y = want_y ? 1 : 0;
    const bool weighted = x != nullptr && xw != nullptr;
    fa.xw = weighted ? xw : nullptr;
    fa.huber = x != nullptr ? w.huber : 0.f;      // > 0: tc2_launch runs the Huber kind of the direction's final kind
    return tc_launch(c, w, 2 * nl, s, false, fa, weighted ? TC_PASS_WEIGHTED : TC_PASS_PROJ);
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
  return launch_final_fwd<float>(c, in, w, x, R, B, want_grad, s, xw);
}

// ---- backward-to-z: w.g = J^T dpre (unscaled by 2/HWC; fp16 path additionally x gscale) -----
struct MomentumArgs { bool tail = false; float lr = 0.f, mu = 0.f; };   // tail: update z in the Linear backward's tail

static float grad_multiplier(const dgan_ctx* c);

static int run_backward(dgan_ctx* c, const Workspace& w, cudaStream_t s, MomentumArgs mom = MomentumArgs()) {
  int rc;
  const int nl = (int)c->layers.size();
  if (c->desc.precision == DGAN_PREC_FP16) {
    // with BatchNorm after layer j the GEMM writes d(act_j) unmasked and the BN backward turns it into d(pre_j) in place
    for (int l = nl; l >= 1; --l) {       // l = nl: the last layer
      ProfScope ps(c, prof_kind(c, 2 * l + 1), s);
      if ((rc = tc_launch(c, w, 2 * l + 1, s))) return rc;
      const int j = l - 1;
      if (c->layers[j].bn_scale != nullptr &&
          (rc = bn_backward_t<float, __half>(c, w, j, w.pre_h[j], w.act_h[j], w.dact_h[j], s)))
        return rc;
    }
    ProfScope ps(c, prof_kind(c, 1), s);
    TcFinalArgs fa{};
    if (mom.tail) {      // the CTA that completes a row tile's partial sums applies the momentum update
      fa.mz = w.z; fa.mv = w.v; fa.mz_h = w.z_h; fa.m_gmul = grad_multiplier(c); fa.m_lr = mom.lr; fa.m_mu = mom.mu;
      fa.m_counter = w.mom_counter; fa.m_nparts = w.n_g_parts; fa.m_count = (size_t)w.n_pad * c->wd.latent;
    }
    return tc_launch(c, w, 1, s, false, fa);
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

// ---- dgan_jvp's tangent pass, after a forward that kept its ReLU masks (run_forward with want_grad): the tangent of z
// (fp32 path: w.v; fp16 path: z_h, scaled per row) through every layer's forward weights without bias, masked by the
// primal forward (BatchNorm: bn_backward_t's tangent mode), into the tangent of the last layer's pre-activation in w.dpre
// (fp32 path: [n_pad][H*W*C]; fp16 path: the fp32 block tensor [n_blocks][n_pad][16 * C_out]).  The hidden layers'
// tangents live in the gradient buffers (dact, dact_h), which a jvp does not otherwise use.
static int run_tangent(dgan_ctx* c, const Workspace& w, cudaStream_t s) {
  int rc;
  const int nl = (int)c->layers.size();
  if (c->desc.precision == DGAN_PREC_FP16) {
    for (int l = 0; l < nl; ++l) {
      if ((rc = tc_launch(c, w, 2 * l, s, false, TcFinalArgs{}, TC_PASS_TANGENT))) return rc;
      if (c->layers[l].bn_scale != nullptr &&
          (rc = bn_backward_t<float, __half>(c, w, l, w.pre_h[l], w.act_h[l], w.dact_h[l], s, true)))
        return rc;
    }
    return tc_launch(c, w, 2 * nl, s, false, TcFinalArgs{}, TC_PASS_TANGENT);
  }
  const float* in = w.v;
  for (int l = 0; l < nl; ++l) {
    const GemmLayer& L = c->layers[l];
    const bool bn = L.bn_scale != nullptr, mask = L.relu && !bn;
    if ((rc = launch_bsgemm_f32(c, mask ? EPI_MASK : EPI_NONE, in, L.C_in, w.n_pad, L.wf, L.wf_tile_stride, L.wf_ld, L.fwd,
                                w.dact[l], L.C_out, nullptr, 0, mask ? w.act[l] : nullptr, s)))
      return rc;
    if (bn && (rc = bn_backward_t<float, float>(c, w, l, w.pre[l], w.act[l], w.dact[l], s, true))) return rc;
    in = w.dact[l];
  }
  // the last layer's linear part (ACT_NONE: no bias, no activation) writes t(pre) where its forward writes y
  const FinalLayer& f = c->fin;
  dim3 grid(w.n_rows, f.n_bands), block(128);
  if (f.C_out == 1)
    final_fwd_loss_kernel<float, 1, ACT_NONE><<<grid, block, f.fwd_smem, s>>>(in, w.n_pad, f.h_in, f.w_in, f.C_in, f.w, f.bias,
                                                                             nullptr, 1, 1, w.dpre, nullptr, nullptr);
  else
    final_fwd_loss_kernel<float, 3, ACT_NONE><<<grid, block, f.fwd_smem, s>>>(in, w.n_pad, f.h_in, f.w_in, f.C_in, f.w, f.bias,
                                                                             nullptr, 1, 1, w.dpre, nullptr, nullptr);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// The state a fresh workspace needs besides z and v: zeroed momentum tickets (fp16 path), zeroed tile-padding rows of
// d(pre) (fp32 path) and, in an Adam workspace, a zeroed second moment.  Memsets only.
static int clear_start_state(dgan_ctx* c, const Workspace& w, cudaStream_t s) {
  if (w.s != nullptr) DGAN_CUDA_CHECK(cudaMemsetAsync(w.s, 0, (size_t)w.n_pad * c->wd.latent * sizeof(float), s));
  if (w.mom_counter != nullptr) DGAN_CUDA_CHECK(cudaMemsetAsync(w.mom_counter, 0, (size_t)w.n_pad / kRowTile * sizeof(unsigned), s));
  // fp32 path: the last layer's forward writes dL/dpre for the real rows only while its backward walks all n_pad rows;
  // the tile-padding rows are never observed, but they must not be read uninitialised
  if (w.dblk == nullptr && w.n_pad > w.n_rows)
    DGAN_CUDA_CHECK(cudaMemsetAsync(w.dpre + (size_t)w.n_rows * c->hwc, 0, (size_t)(w.n_pad - w.n_rows) * c->hwc * sizeof(float), s));
  return 0;
}

// z (at the padded latent width) from the caller's z0 [n_rows][latent_dim] or the Philox stream, v = 0
static int run_init_z(dgan_ctx* c, const Workspace& w, const float* z0, uint64_t seed, cudaStream_t s, size_t row_offset = 0) {
  const int latent = c->desc.latent_dim, ld = c->wd.latent;
  const size_t total = (size_t)w.n_pad * ld;
  if (int rc = clear_start_state(c, w, s)) return rc;
  init_z_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(w.z, w.v, w.z_h, z0, w.n_rows, w.n_pad, latent, ld, seed,
                                                                sqrtf(1.0f / (float)latent), row_offset * latent);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// ---- a caller's cotangent dy [n_rows][H*W*C] -> the last layer's d(pre), after a forward that wrote w.y ----------
// fp16 path: per-row power-of-two scales (one shared scale with BatchNorm) in w.loss, d(pre) * scale in w.dblk;
// fp32 path: d(pre) unscaled in w.dpre.  See kernels_vjp.cuh.  scale: where the fp16 path keeps the row scales (NULL:
// w.loss).
static int launch_cotangent(dgan_ctx* c, const Workspace& w, const float* dy, cudaStream_t s, float* scale = nullptr) {
  if (scale == nullptr) scale = w.loss;
  const FinalLayer& f = c->fin;
  const bool tc = c->desc.precision == DGAN_PREC_FP16;
  const bool sigmoid = f.C_out == 1 && f.act == ACT_SIGMOID;
  if (!sigmoid && !(f.C_out == 3 && f.act == ACT_TANH)) { set_error("unsupported final layer"); return DGAN_ERR_UNSUPPORTED; }
  if (tc) {
    if (sigmoid) cotangent_rowmax_kernel<ACT_SIGMOID><<<w.n_rows, 256, 0, s>>>(w.y, dy, c->hwc, scale);
    else cotangent_rowmax_kernel<ACT_TANH><<<w.n_rows, 256, 0, s>>>(w.y, dy, c->hwc, scale);
    DGAN_LAUNCH_CHECK(c);
    cotangent_scale_kernel<<<1, 1024, 0, s>>>(scale, w.n_rows, c->desc.use_bn ? 1 : 0, 4);
    DGAN_LAUNCH_CHECK(c);
  }
  if (tc && w.n_pad > w.n_rows) {
    // the cotangent covers the real rows; the block tensor's tile-padding rows get zeros (the last layer's backward
    // reads all n_pad rows)
    const size_t row_b = (size_t)16 * f.C_out * sizeof(__half);
    DGAN_CUDA_CHECK(cudaMemset2DAsync(w.dblk + (size_t)w.n_rows * 16 * f.C_out, (size_t)w.n_pad * row_b, 0,
                                      (size_t)(w.n_pad - w.n_rows) * row_b, (size_t)f.n_blocks, s));
  }
  const size_t total = (size_t)w.n_rows * c->hwc;
  const unsigned grid = (unsigned)((total + 255) / 256);
  const int w_out = 2 * f.w_in;
#define CT(ACT, CO, BLK) cotangent_kernel<ACT, CO, BLK><<<grid, 256, 0, s>>>(w.y, dy, w.n_rows, w_out, scale, w.dpre, w.dblk, w.n_pad)
  if (sigmoid) { if (tc) CT(ACT_SIGMOID, 1, true); else CT(ACT_SIGMOID, 1, false); }
  else { if (tc) CT(ACT_TANH, 3, true); else CT(ACT_TANH, 3, false); }
#undef CT
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// ---- the measured loss (dgan_reconstruct_measured; kernels_measured.cuh) ----------------------------------------------
// Copy a call's operator a [m][H*W*C] and measurements y [batch][m] into the measured workspace w: A with m_ld - m zero
// rows, its transpose, y with m_ld - m zero columns.  The measured loop then reads only the workspace.
static int stage_measured(dgan_ctx* c, const Workspace& w, const float* a, const float* y, int batch, cudaStream_t s) {
  const int hwc = c->hwc;
  const size_t na = (size_t)w.m_ld * hwc, ny = (size_t)batch * w.m_ld;
  pad_copy_kernel<<<(unsigned)((na + 255) / 256), 256, 0, s>>>(a, w.am, w.m, 1, hwc, w.m_ld, 1, hwc);
  DGAN_LAUNCH_CHECK(c);
  transpose_tiles_kernel<<<(unsigned)((na + 255) / 256), 256, 0, s>>>(w.am, w.amt, w.m_ld, hwc, na);
  DGAN_LAUNCH_CHECK(c);
  pad_copy_kernel<<<(unsigned)((ny + 255) / 256), 256, 0, s>>>(y, w.ym, batch, 1, w.m, batch, 1, w.m_ld);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// out = EPI(s_ * X W^T) over the real latent rows: TF32 tensor cores on the fp16 path, fp32 FFMA on the fp32 path
template <int EPI>
static int launch_measured_gemm(dgan_ctx* c, const Workspace& w, const float* X, int ldx, const float* W, int ldw, int N,
                                int K, float* out, int ldo, const float* ym, int R, float s_, float* loss_part, cudaStream_t s) {
  const dim3 grid((unsigned)((w.n_rows + kMeasTileM - 1) / kMeasTileM), (unsigned)((N + kMeasTileN - 1) / kMeasTileN));
  if constexpr (EPI == MEAS_RESID_HUBER) {
    if (c->desc.precision == DGAN_PREC_FP16)
      measured_gemm_huber_kernel<true><<<grid, 256, 0, s>>>(X, ldx, w.n_rows, W, ldw, N, K, out, ldo, ym, R, s_, loss_part, w.n_pad);
    else
      measured_gemm_huber_kernel<false><<<grid, 256, 0, s>>>(X, ldx, w.n_rows, W, ldw, N, K, out, ldo, ym, R, s_, loss_part, w.n_pad);
  } else if (c->desc.precision == DGAN_PREC_FP16)
    measured_gemm_kernel<true, EPI><<<grid, 256, 0, s>>>(X, ldx, w.n_rows, W, ldw, N, K, out, ldo, ym, R, s_, loss_part, w.n_pad);
  else
    measured_gemm_kernel<false, EPI><<<grid, 256, 0, s>>>(X, ldx, w.n_rows, W, ldw, N, K, out, ldo, ym, R, s_, loss_part, w.n_pad);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// Copy a call's CSR operator (row_ptr [m + 1], col_idx / val [nnz]) and measurements y [batch][m] into the CSR-measured
// workspace w, validated, with its transpose built and y padded as stage_measured does (kernels_measured_csr.cuh): five
// kernels.  An invalid CSR is staged as the empty operator with NaN measurements.
static int stage_measured_csr(dgan_ctx* c, const Workspace& w, const int* row_ptr, const int* col_idx, const float* val,
                              const float* y, int batch, cudaStream_t s) {
  const int hwc = c->hwc, m = w.m;
  // the products stage kCsrRows rows of H*W*C (measurement) or m_ld (adjoint) floats; the opt-in limit is per kernel, not
  // per handle, so it is only ever raised
  const int smem = kCsrRows * std::max(hwc, w.m_ld) * (int)sizeof(float);
  cudaFuncAttributes fa;
  DGAN_CUDA_CHECK(cudaFuncGetAttributes(&fa, measured_csr_kernel<MEAS_RESID>));
  if (fa.maxDynamicSharedSizeBytes < smem)
    DGAN_CUDA_CHECK(cudaFuncSetAttribute(measured_csr_kernel<MEAS_RESID>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  DGAN_CUDA_CHECK(cudaFuncGetAttributes(&fa, measured_csr_kernel<MEAS_SCALE>));
  if (fa.maxDynamicSharedSizeBytes < smem)
    DGAN_CUDA_CHECK(cudaFuncSetAttribute(measured_csr_kernel<MEAS_SCALE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  DGAN_CUDA_CHECK(cudaFuncGetAttributes(&fa, measured_csr_huber_kernel));
  if (fa.maxDynamicSharedSizeBytes < smem)
    DGAN_CUDA_CHECK(cudaFuncSetAttribute(measured_csr_huber_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  csr_validate_kernel<<<(m + 255) / 256, 256, 0, s>>>(row_ptr, col_idx, m, w.nnz, hwc, w.csr_bad);
  DGAN_LAUNCH_CHECK(c);
  csr_stage_rows_kernel<<<1, 1024, 0, s>>>(row_ptr, w.csr_bad, m, w.m_ld, w.nnz, w.csr_valid, w.a_rp);
  DGAN_LAUNCH_CHECK(c);
  const size_t n = std::max({(size_t)w.nnz, (size_t)batch * w.m_ld, (size_t)hwc});
  csr_stage_entries_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(col_idx, val, w.nnz, y, batch, m, w.m_ld, w.a_rp,
                                                                       w.csr_valid, hwc, w.a_ci, w.a_v, w.ym, w.at_rp);
  DGAN_LAUNCH_CHECK(c);
  csr_scan_kernel<<<1, 1024, 0, s>>>(w.at_rp, hwc);
  DGAN_LAUNCH_CHECK(c);
  csr_fill_transpose_kernel<<<(hwc + 127) / 128, 128, 0, s>>>(w.a_rp, w.a_ci, w.a_v, m, hwc, w.at_rp, w.at_ci, w.at_v);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// out = EPI(s_ * X A^T) over the real latent rows through a staged CSR operator (rp, ci, val; N output columns): fp32
// FFMA on both precisions.  X rows of K floats at stride ldx are staged in shared memory.
template <int EPI>
static int launch_measured_csr(dgan_ctx* c, const Workspace& w, const float* X, int ldx, int K, const int* rp,
                               const int* ci, const float* val, int N, float* out, int ldo, const float* ym, int R,
                               float s_, float* loss_part, cudaStream_t s) {
  const unsigned grid = (unsigned)((w.n_rows + kCsrRows - 1) / kCsrRows);
  if constexpr (EPI == MEAS_RESID_HUBER)
    measured_csr_huber_kernel<<<grid, kCsrThreads, kCsrRows * K * sizeof(float), s>>>(X, ldx, w.n_rows, K, rp, ci, val, N,
                                                                                      out, ldo, ym, R, s_, loss_part, w.n_pad);
  else
    measured_csr_kernel<EPI><<<grid, kCsrThreads, kCsrRows * K * sizeof(float), s>>>(X, ldx, w.n_rows, K, rp, ci, val, N,
                                                                                      out, ldo, ym, R, s_, loss_part, w.n_pad);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// Dynamic shared memory of a convolution product over the workspace's operator: the kernel's taps and the most operand
// rows any chunk stages (kernels_measured_conv.cuh).  adjoint: the adjoint product's, else the measurement product's.
static size_t conv_smem(const dgan_ctx* c, const Workspace& w, bool adjoint) {
  const ConvGeom& g = w.cg;
  const int n = adjoint ? c->hwc : w.m_ld, row = adjoint ? g.Wo * g.C : g.W * g.C;
  int most = 0;
  for (int x0 = 0; x0 < n; x0 += kConvCols) {
    int lo, hi;
    if (adjoint) conv_adj_span(g, x0, std::min(n, x0 + kConvCols), &lo, &hi);
    else conv_meas_span(g, x0, std::min(std::min(n, x0 + kConvCols), w.m), &lo, &hi);
    most = std::max(most, hi - lo + 1);
  }
  return ((size_t)conv_taps_ld(g) + (size_t)most * row) * sizeof(float);
}

// Copy a call's kernels k [batch][kh][kw] and measurements y [batch][m] into the convolution-measured workspace w, y
// padded as stage_measured does: one kernel.  Raises the products' shared-memory limit where a geometry needs more than
// the default (never lowered: the opt-in limit is per kernel, not per handle).
static int stage_measured_conv(dgan_ctx* c, const Workspace& w, const float* k, const float* y, int batch, cudaStream_t s) {
  const size_t meas = conv_smem(c, w, false), adj = conv_smem(c, w, true);
  cudaFuncAttributes fa;
  DGAN_CUDA_CHECK(cudaFuncGetAttributes(&fa, measured_conv_kernel));
  if ((size_t)fa.maxDynamicSharedSizeBytes < meas)
    DGAN_CUDA_CHECK(cudaFuncSetAttribute(measured_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)meas));
  DGAN_CUDA_CHECK(cudaFuncGetAttributes(&fa, measured_conv_huber_kernel));
  if ((size_t)fa.maxDynamicSharedSizeBytes < meas)
    DGAN_CUDA_CHECK(cudaFuncSetAttribute(measured_conv_huber_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)meas));
  DGAN_CUDA_CHECK(cudaFuncGetAttributes(&fa, measured_conv_adjoint_kernel));
  if ((size_t)fa.maxDynamicSharedSizeBytes < adj)
    DGAN_CUDA_CHECK(cudaFuncSetAttribute(measured_conv_adjoint_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)adj));
  const int taps = w.cg.kh * w.cg.kw;
  const size_t n = std::max((size_t)batch * taps, (size_t)batch * w.m_ld);
  conv_stage_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(k, y, batch, taps, w.m, w.m_ld, w.ck, w.ym);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// The measurement product through the staged convolution operator: r = A_{n / R} G(z) - y[n / R] and the loss parts
// (huber: MEAS_RESID_HUBER at delta = w.huber)
static int launch_measured_conv(dgan_ctx* c, const Workspace& w, const float* in, int R, cudaStream_t s) {
  const unsigned grid = (unsigned)((size_t)w.n_rows * ((w.m_ld + kConvCols - 1) / kConvCols));
  const size_t smem = conv_smem(c, w, false);
  if (w.huber > 0.f)
    measured_conv_huber_kernel<<<grid, kConvThreads, smem, s>>>(in, c->hwc, w.cg, w.ck, w.m_ld, w.m, w.r, w.m_ld, w.ym, R,
                                                                w.huber, w.mloss_part, w.n_pad);
  else
    measured_conv_kernel<<<grid, kConvThreads, smem, s>>>(in, c->hwc, w.cg, w.ck, w.m_ld, w.m, w.r, w.m_ld, w.ym, R, 1.f,
                                                          w.mloss_part, w.n_pad);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// The image loss of a sparse-deviation call (w.ident) on u: the loss parts and dy = (2 / H*W*C) w c of the identity
// operator in one kernel (sdev_image_resid_kernel), against the images in w.x and the weights in w.xw (NULL: unweighted)
static int launch_image_resid(dgan_ctx* c, const Workspace& w, int R, cudaStream_t s) {
  const dim3 grid((unsigned)w.n_rows, (unsigned)((w.m_ld / 4 + 255) / 256));
  const float s_ = 2.f / (float)w.m;
#define IR(HU, WE) sdev_image_resid_kernel<HU, WE><<<grid, 256, 0, s>>>(w.u, w.x, w.xw, c->hwc, w.m_ld, R, w.huber, s_, \
                                                                        w.dym, w.mloss_part, w.n_pad)
  if (w.huber > 0.f) { if (w.xw != nullptr) IR(true, true); else IR(true, false); }
  else { if (w.xw != nullptr) IR(false, true); else IR(false, false); }
#undef IR
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// The measurement product after a forward that wrote w.y: r = A G(z) - y[n / R] and the measured loss's parts.  w.huber > 0:
// the Huber residual psi(r) and the Huber loss's parts (MEAS_RESID_HUBER, delta passed as the scale).  With sparse
// deviations (w.u) the product reads u = G(z) + nu in place of G(z); the image loss's (w.ident) is launch_image_resid.
static int launch_measure(dgan_ctx* c, const Workspace& w, int R, cudaStream_t s) {
  if (w.ident) return launch_image_resid(c, w, R, s);
  const float* in = w.u != nullptr ? w.u : w.y;
  if (w.conv) return launch_measured_conv(c, w, in, R, s);
  if (w.huber > 0.f) {
    if (w.csr)
      return launch_measured_csr<MEAS_RESID_HUBER>(c, w, in, c->hwc, c->hwc, w.a_rp, w.a_ci, w.a_v, w.m_ld, w.r, w.m_ld,
                                                   w.ym, R, w.huber, w.mloss_part, s);
    return launch_measured_gemm<MEAS_RESID_HUBER>(c, w, in, c->hwc, w.am, c->hwc, w.m_ld, c->hwc, w.r, w.m_ld, w.ym, R,
                                                  w.huber, w.mloss_part, s);
  }
  if (w.csr)
    return launch_measured_csr<MEAS_RESID>(c, w, in, c->hwc, c->hwc, w.a_rp, w.a_ci, w.a_v, w.m_ld, w.r, w.m_ld, w.ym, R,
                                           1.f, w.mloss_part, s);
  return launch_measured_gemm<MEAS_RESID>(c, w, in, c->hwc, w.am, c->hwc, w.m_ld, c->hwc, w.r, w.m_ld, w.ym, R, 1.f,
                                          w.mloss_part, s);
}

// Sparse deviations, iteration t of the loop, after its forward: nu from the previous iteration's dy (t > 0; +0 at
// t = 0) and u = y + nu (sdev_update_kernel)
static int launch_sdev_update(dgan_ctx* c, const Workspace& w, int t, cudaStream_t s) {
  const size_t n4 = (size_t)w.n_rows * c->hwc / 4;
  sdev_update_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, s>>>(w.y, w.dym, w.nu, w.u, n4, t > 0 ? 1 : 0, w.sdev_eta,
                                                                  w.sdev_tau);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// The rest of a measured step's gradient after launch_measure: dy = (2/m) At r, then the cotangent entry of dgan_vjp (its
// fp16 row scales in w.mscale: w.loss carries the loss to the select) and the backward-to-z into w.g.  R: the rows per
// image, which pick a convolution operator's kernel.  The image loss of a sparse-deviation call (w.ident) has its dy from launch_image_resid already.
static int measured_backward(dgan_ctx* c, const Workspace& w, int R, cudaStream_t s) {
  int rc;
  if (w.ident) {
    rc = 0;
  } else if (w.conv) {
    const unsigned grid = (unsigned)((size_t)w.n_rows * ((c->hwc + kConvCols - 1) / kConvCols));
    measured_conv_adjoint_kernel<<<grid, kConvThreads, conv_smem(c, w, true), s>>>(w.r, w.m_ld, w.cg, w.ck, c->hwc, w.dym,
                                                                                 c->hwc, R, 2.f / (float)w.m);
    DGAN_LAUNCH_CHECK(c);
    rc = 0;
  } else if (w.csr) rc = launch_measured_csr<MEAS_SCALE>(c, w, w.r, w.m_ld, w.m_ld, w.at_rp, w.at_ci, w.at_v, c->hwc, w.dym,
                                                  c->hwc, nullptr, 1, 2.f / (float)w.m, nullptr, s);
  else rc = launch_measured_gemm<MEAS_SCALE>(c, w, w.r, w.m_ld, w.amt, w.m_ld, c->hwc, w.m_ld, w.dym, c->hwc, nullptr, 1,
                                             2.f / (float)w.m, nullptr, s);
  if (rc) return rc;
  if ((rc = launch_cotangent(c, w, w.dym, s, w.mscale))) return rc;
  return run_backward(c, w, s);
}

// w.loss[n] = inv * (the row's n_parts loss parts at part index n * stride_n + part * stride_b, fixed order); with the
// latent prior (w.prior) the prior term prior_term_kernel left in w.loss is added (loss_finish_prior_kernel)
static int loss_finish(dgan_ctx* c, const Workspace& w, const float* parts, int n_parts, size_t stride_n,
                       size_t stride_b, float inv, cudaStream_t s) {
  const unsigned grid = (unsigned)((w.n_rows + 255) / 256);
  if (w.prior)
    loss_finish_prior_kernel<<<grid, 256, 0, s>>>(parts, n_parts, stride_n, stride_b, inv, w.n_rows, w.loss);
  else
    loss_finish_kernel<<<grid, 256, 0, s>>>(parts, n_parts, stride_n, stride_b, inv, w.n_rows, w.loss);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// loss[n] = (1/m) sum_j r[n][j]^2, from the measurement product's parts (fixed order)
static int measured_loss_finish(dgan_ctx* c, const Workspace& w, cudaStream_t s) {
  return loss_finish(c, w, w.mloss_part, w.m_ld / kMeasTileN, 1, (size_t)w.n_pad, 1.0f / (float)w.m, s);
}

// loss[n] = (1/HWC) (sum of the image loss's parts), as the last forward left them
static int image_loss_finish(dgan_ctx* c, const Workspace& w, cudaStream_t s) {
  return loss_finish(c, w, w.loss_part, w.n_loss_parts, w.loss_stride_n, w.loss_stride_b, 1.0f / (float)c->hwc, s);
}

// fp16 path: plan and upload the schedules of every layer-direction for this many latent rows (cached in the handle).
// Planning allocates and synchronises, so it happens before any kernel of a call is enqueued (and never while the L-step
// loop is captured); a caller that sized its workspace with dgan_workspace_bytes has had it done there.
static int plan_all(dgan_ctx* c, int n_rows) {
  if (c->desc.precision != DGAN_PREC_FP16) return 0;
  const int n_mpairs = (int)align_up((size_t)std::max(n_rows, 1), 2 * kRowTile) / (2 * kRowTile);
  int rc;
  for (TcDir& t : c->tc_dirs)
    if ((rc = tc2_get_schedule(t, n_mpairs, c->tc.num_sms / 2, &c->allocs))) return rc;
  return 0;
}

// fp16 path: the directions of dgan_jvp's tangent pass or of the weighted last-layer forward, made on the first call that
// needs them from tc_directions(desc, pass) with the projection's weight tiles (same layer-direction and column block),
// then planned for this many latent rows like plan_all.  A handle that never runs such a call plans nothing for them and
// holds no schedule.
static int plan_pass(dgan_ctx* c, int n_rows, TcPass pass) {
  if (c->desc.precision != DGAN_PREC_FP16) return 0;
  int rc;
  std::vector<TcDir>& have = pass == TC_PASS_TANGENT ? c->tc_jvp_dirs : c->tc_w_dirs;
  if (have.empty()) {
    std::vector<TcDir> dirs = tc_directions(&c->desc, pass);
    for (TcDir& t : dirs) {
      if ((rc = tc_dir_supported(t))) return rc;
      for (const TcDir& p : c->tc_dirs)
        if (p.ld == t.ld && p.col0 == t.col0) { t.w = p.w; t.tm_b = p.tm_b; }
      t.order = c->tc_order;
    }
    have = std::move(dirs);
  }
  const int n_mpairs = (int)align_up((size_t)std::max(n_rows, 1), 2 * kRowTile) / (2 * kRowTile);
  for (TcDir& t : have)
    if ((rc = tc2_get_schedule(t, n_mpairs, c->tc.num_sms / 2, &c->allocs))) return rc;
  return 0;
}

// A projection's workspace for batch images of rec_rr restarts, at base (NULL: sizes only): every stage's row count
// planned (with the weighted last-layer forward when the image loss is weighted without sparse deviations, which run it
// in the measured loop), then carved.  Unpruned (sh.n_points 0): one carve of batch * rec_rr rows, the operator of a
// measured loss inside it.  Pruned: a measured loss's operator block first (carve_operator; layout: a line
// "operator 0 batch", then its lines), staged once for every stage, then region k for batch * keep_k rows (region 0:
// batch * rec_rr), each a carve with the prune maps and the operator block's pointers, one after the other (every carve
// is a multiple of 1024 bytes); layout: per region a line "region k byte_offset n_rows", then carve's lines with offsets
// relative to the region.  The schedule has passed check_schedule.  *bytes: the total; regs (not NULL): the carves.
// 0, or the planner's error code.
static int plan_workspace(dgan_ctx* c, int batch, int rec_rr, const WsShape& sh, void* base, std::string* layout,
                          std::vector<Workspace>* regs, size_t* bytes) {
  auto stage_rows = [&](int k) { return batch * (k == 0 ? rec_rr : sh.sched[k - 1].keep); };
  int rc;
  for (int k = 0; k <= sh.n_points; ++k) {
    if ((rc = plan_all(c, stage_rows(k)))) return rc;
    if (sh.weighted && !sh.sdev && (rc = plan_pass(c, stage_rows(k), TC_PASS_WEIGHTED))) return rc;
  }
  size_t off = 0;
  Workspace op;
  const bool op_block = sh.n_points > 0 && sh.m > 0;
  if (op_block) {
    if (layout != nullptr) *layout += "operator 0 " + std::to_string(batch) + "\n";
    op = carve_operator(c, batch, sh, base, layout);
    off = op.bytes;
  }
  for (int k = 0; k <= sh.n_points; ++k) {
    if (layout != nullptr && sh.n_points > 0)
      *layout += "region " + std::to_string(k) + " " + std::to_string(off) + " " + std::to_string(stage_rows(k)) + "\n";
    Workspace w = carve(c, stage_rows(k), base ? (void*)((char*)base + off) : nullptr, layout, sh, op_block ? &op : nullptr);
    off += w.bytes;
    if (regs != nullptr) regs->push_back(std::move(w));
  }
  *bytes = off;
  return 0;
}

// The sizer that returns a projection's workspace bytes, as the "workspace too small" message names it (none for
// dgan_workspace_bytes)
static std::string sizer_name(const WsShape& sh) {
  const bool measured = sh.m > 0;
  if (sh.sdev) return measured ? "dgan_workspace_bytes_measured_sparse_dev" : "dgan_workspace_bytes_sparse_dev";
  if (sh.conv != nullptr) return "dgan_workspace_bytes_measured_conv";
  if (sh.adam) return measured ? "dgan_workspace_bytes_measured_adam" : "dgan_workspace_bytes_adam";
  if (sh.n_points > 0) return measured ? "dgan_workspace_bytes_measured_pruned" : "dgan_workspace_bytes_pruned";
  if (sh.weighted) return "dgan_workspace_bytes_weighted";
  if (sh.nnz >= 0) return "dgan_workspace_bytes_measured_csr";
  return measured ? "dgan_workspace_bytes_measured" : "";
}

// Check the caller's workspace and plan and carve it (plan_workspace) into *regs, one per stage; on the fp16 path also
// encode each region's tensor maps, and those of the weighted last-layer forward when it was planned.
static int check_ws(dgan_ctx* c, int batch, int rec_rr, const WsShape& sh, void* ws, size_t ws_bytes,
                    std::vector<Workspace>* regs) {
  if (ws == nullptr) { set_error("workspace is NULL"); return DGAN_ERR_WORKSPACE; }
  if (((uintptr_t)ws & 1023) != 0) { set_error("workspace must be 1024-byte aligned"); return DGAN_ERR_WORKSPACE; }
  int rc;
  size_t need = 0;
  if ((rc = plan_workspace(c, batch, rec_rr, sh, ws, nullptr, regs, &need))) return rc;
  if (need > ws_bytes) {
    const std::string sizer = sizer_name(sh);
    set_error("workspace too small: need " + std::to_string(need) + " bytes, got " + std::to_string(ws_bytes) +
              (sizer.empty() ? "" : " (" + sizer + ")"));
    return DGAN_ERR_WORKSPACE;
  }
  for (Workspace& w : *regs) {
    if ((rc = build_maps(c, w))) return rc;
    if (sh.weighted && !sh.sdev && (rc = build_maps(c, w, TC_PASS_WEIGHTED))) return rc;
  }
  return 0;
}

// The bytes of a projection's workspace (plan_workspace), or 0 when planning fails
static size_t workspace_bytes(dgan_ctx* c, int batch, int rec_rr, const WsShape& sh) {
  size_t bytes = 0;
  return plan_workspace(c, batch, rec_rr, sh, nullptr, nullptr, nullptr, &bytes) ? 0 : bytes;
}

// The weight tensors in creation order (include/defensegan_b200.h, dgan_num_weights) as 3-D arrays: the caller's shape
// [a][b][c] at the real widths and the handle's [ap][bp][cp] at the padded ones.
struct WeightShape { int a, b, c, ap, bp, cp; };
static std::vector<WeightShape> weight_shapes(const dgan_desc* d, const Widths& p) {
  const Widths r = real_widths(d);
  std::vector<WeightShape> n = {{r.latent, 16, r.c4, p.latent, 16, p.c4}, {1, 16, r.c4, 1, 16, p.c4}};   // W [latent][pixel][c]
  if (d->use_bn) { n.push_back(n.back()); n.push_back(n.back()); }
  const int c_img = d->arch == DGAN_ARCH_CELEBA ? 3 : 1;
  std::vector<std::pair<int, int>> dc = {{r.c4, r.c2}, {r.c2, r.c1}}, dp = {{p.c4, p.c2}, {p.c2, p.c1}};   // (C_in, C_out)
  if (d->arch == DGAN_ARCH_CELEBA) { dc.push_back({r.c1, r.c1}); dp.push_back({p.c1, p.c1}); }
  dc.push_back({r.c1, c_img}); dp.push_back({p.c1, c_img});
  for (size_t i = 0; i < dc.size(); ++i) {
    n.push_back({kTaps, dc[i].second, dc[i].first, kTaps, dp[i].second, dp[i].first});   // filters (5,5,C_out,C_in)
    n.push_back({1, 1, dc[i].second, 1, 1, dp[i].second});
    if (d->use_bn && i < 2) { n.push_back(n.back()); n.push_back(n.back()); }
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
  int rc = 0;
  if ((rc = padded_widths(d, &c->wd))) return rc;
  const Widths real = real_widths(d);
  const int latent = c->wd.latent;
  c->H = celeba ? 64 : 28; c->W = c->H; c->C = celeba ? 3 : 1;
  c->hwc = c->H * c->W * c->C;
  auto fail = [](int code) { return code; };   // the caller destroys the half-built handle
  // The handle owns copies of every weight tensor, at the padded widths: the caller may free or reuse `weights_dev` as
  // soon as the copies enqueued here have run (i.e. after synchronising `stream`).
  std::vector<const float*> wown;
  {
    const std::vector<WeightShape> shapes = weight_shapes(d, c->wd);
    size_t total = 0;
    for (const WeightShape& w : shapes) total += align_up((size_t)w.ap * w.bp * w.cp * sizeof(float), 256);
    char* base = nullptr;
    if ((rc = dev_alloc(c, (void**)&base, total))) return fail(rc);
    size_t off = 0;
    for (size_t i = 0; i < shapes.size(); ++i) {
      const WeightShape& w = shapes[i];
      const size_t n = (size_t)w.ap * w.bp * w.cp;
      float* dst = (float*)(base + off);
      if (w.a == w.ap && w.b == w.bp && w.c == w.cp) {
        cudaError_t e = cudaMemcpyAsync(dst, weights_in[i], n * sizeof(float), cudaMemcpyDeviceToDevice, s);
        if (e != cudaSuccess) { set_error(std::string("weight copy: ") + cudaGetErrorString(e)); return fail(DGAN_ERR_CUDA); }
      } else {
        pad_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(weights_in[i], dst, w.a, w.b, w.c, w.ap, w.bp, w.cp);
        DGAN_CUDA_CHECK(cudaGetLastError());
      }
      wown.push_back(dst);
      off += align_up(n * sizeof(float), 256);
    }
  }
  const float* const* weights = wown.data();

  // ---- Linear (Generator.Input): [1][N][latent] -> [16][N][c4]
  {
    GemmLayer L{};
    L.P_in = 1; L.C_in = latent; L.P_out = 16; L.C_out = c->wd.c4;
    L.relu = true;
    L.fwd_host = linear_fwd_pairs(16); L.bwd_host = linear_bwd_pairs(16);
    L.macs = (int64_t)16 * real.latent * real.c4;
    const float* W = weights[0];             // (latent, 16*c4), column f = pixel*c4 + c
    L.wf = W; L.wf_tile_stride = L.C_out; L.wf_ld = 16 * L.C_out;
    float* Wt = nullptr;                     // [16*c4][latent]: backward tile q rows = c, cols = latent
    if ((rc = dev_alloc(c, (void**)&Wt, (size_t)latent * 16 * L.C_out * 4))) return fail(rc);
    const size_t total = (size_t)latent * 16 * L.C_out;
    transpose_tiles_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(W, Wt, latent, 16 * L.C_out, total);
    L.wb = Wt; L.wb_tile_stride = L.C_out * latent; L.wb_ld = latent;
    L.bias = weights[1]; L.bias_pstride = L.C_out;   // bias index f = pixel*C_out + c
    if (d->use_bn) { L.bn_offset = weights[2]; L.bn_scale = weights[3]; L.bn_per_pixel = 1; }   // Generator.BN1, axes [0]
    c->layers.push_back(L);
  }
  // ---- hidden deconvs
  const std::vector<DeconvSpec> specs = deconv_specs(d, c->wd), real_specs = deconv_specs(d, real);
  int wi = d->use_bn ? 4 : 2;
  int di = 0;
  for (const DeconvSpec& sp : specs) {
    GemmLayer L{};
    L.P_in = sp.in_raster * sp.in_raster; L.C_in = sp.c_in; L.P_out = sp.h_used * sp.h_used; L.C_out = sp.c_out;
    L.relu = sp.relu;
    L.fwd_host = deconv_fwd_pairs(sp.h_in, sp.h_in, sp.h_used, sp.h_used, sp.in_raster);
    L.bwd_host = deconv_bwd_pairs(sp.h_in, sp.h_in, sp.h_used, sp.h_used, sp.in_raster);
    L.macs = (int64_t)L.fwd_host.pairs.size() * real_specs[(size_t)di].c_in * real_specs[(size_t)di].c_out;
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
    f.h_in = f.w_in = specs.back().h_used; f.C_in = c->wd.c1; f.C_out = c->C; f.act = celeba ? ACT_TANH : ACT_SIGMOID;
    f.w = weights[wi]; f.bias = weights[wi + 1];
    f.n_bands = (2 * f.h_in + kBandRows - 1) / kBandRows;
    f.n_blocks = (f.h_in / 2) * (f.w_in / 2);
    f.fwd_smem = final_fwd_smem(f.C_in, f.C_out, f.w_in);     // <= kFinalSmemMax: padded_widths refuses more
    f.bwd_smem = (size_t)kTaps * f.C_out * f.C_in * 4;
  }
  // exact in-bounds MACs per latent row at the real widths (SURVEY 8d / Appendix B)
  c->macs_per_row = 0;
  for (const GemmLayer& L : c->layers) c->macs_per_row += L.macs;
  {
    PairTable ft = deconv_fwd_pairs(c->fin.h_in, c->fin.w_in, 2 * c->fin.h_in, 2 * c->fin.w_in);
    c->macs_per_row += (int64_t)ft.pairs.size() * real.c1 * c->fin.C_out;
  }
  for (GemmLayer& L : c->layers) {
    if ((rc = upload_table(c, L.fwd_host, &L.fwd, s))) return fail(rc);
    if ((rc = upload_table(c, L.bwd_host, &L.bwd, s))) return fail(rc);
  }
  // opt in to > 48 KB dynamic shared memory where needed: the fp32 last layer's footprint grows with net_dim, up to what
  // an H100 block can have (padded_widths refuses wider generators)
#define OPTIN(K, BYTES) DGAN_CUDA_CHECK(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(BYTES)))
  OPTIN((final_fwd_loss_kernel<float, 1, ACT_SIGMOID>), kFinalSmemMax);
  OPTIN((final_fwd_loss_kernel<float, 3, ACT_TANH>), kFinalSmemMax);
  OPTIN((final_fwd_loss_kernel<float, 1, ACT_SIGMOID, true>), kFinalSmemMax);   // the weighted loss
  OPTIN((final_fwd_loss_kernel<float, 3, ACT_TANH, true>), kFinalSmemMax);
  OPTIN((final_fwd_huber_kernel<float, 1, ACT_SIGMOID, false>), kFinalSmemMax);   // the Huber loss
  OPTIN((final_fwd_huber_kernel<float, 3, ACT_TANH, false>), kFinalSmemMax);
  OPTIN((final_fwd_huber_kernel<float, 1, ACT_SIGMOID, true>), kFinalSmemMax);
  OPTIN((final_fwd_huber_kernel<float, 3, ACT_TANH, true>), kFinalSmemMax);
  OPTIN((final_fwd_loss_kernel<float, 1, ACT_NONE>), kFinalSmemMax);    // dgan_jvp's tangent of the last layer
  OPTIN((final_fwd_loss_kernel<float, 3, ACT_NONE>), kFinalSmemMax);
  OPTIN((final_fwd_loss_kernel<__half, 1, ACT_SIGMOID>), 100 * 1024);
  OPTIN((final_fwd_loss_kernel<__half, 3, ACT_TANH>), 100 * 1024);
  OPTIN((final_bwd_kernel<float, 1>), kFinalSmemMax);
  OPTIN((final_bwd_kernel<float, 3>), kFinalSmemMax);
#undef OPTIN
  if (d->precision == DGAN_PREC_FP16) {
    if ((rc = tc_init(c->tc))) return fail(rc);
    if ((rc = tc2_optin_all())) return fail(rc);
    c->tc_dirs = tc_directions(d);
    const int nl = (int)c->layers.size();
    for (size_t i = 0; i < c->tc_dirs.size(); ++i) {
      TcDir& t = c->tc_dirs[i];
      if ((rc = tc_dir_supported(t))) return fail(rc);
      // fp16 K-major weight tiles [n_tiles][N rows][K cols]
      const size_t tile = (size_t)t.N * t.K;
      if ((rc = dev_alloc(c, (void**)&t.w, (size_t)t.n_tiles * tile * 2))) return fail(rc);
      if (t.ld < 2 * nl) {       // a GEMM layer: its tiles (rows col0 .. col0 + N), then the all-zero tile of tc_with_zero_tile()
        const GemmLayer& L = c->layers[(size_t)(t.ld / 2)];
        const size_t elems = (size_t)(t.n_tiles - 1) * tile;
        const unsigned blocks = (unsigned)((elems + 255) / 256);
        DGAN_CUDA_CHECK(cudaMemsetAsync(t.w + elems, 0, tile * 2, s));
        if (t.ld % 2 == 0)         // F[t][co][ci]; Linear: Wt[q*C + c][k]
          tc_convert_kernel<<<blocks, 256, 0, s>>>(L.wb, t.w, elems, L.C_out, t.col0, t.N, t.K);
        else if (t.ld == 1)        // W[k][q*C + c]
          tc_linear_bwd_tiles_kernel<<<blocks, 256, 0, s>>>(weights[0], t.w, latent, L.C_out, L.P_out);
        else                       // Ff[t][ci][co]
          tc_convert_kernel<<<blocks, 256, 0, s>>>(L.wf, t.w, elems, L.C_in, t.col0, t.N, t.K);
        DGAN_CUDA_CHECK(cudaGetLastError());
      }
      if ((rc = tc_make_map(c->tc, &t.tm_b, t.w, (uint64_t)t.K, (uint64_t)t.N, (uint64_t)t.n_tiles, (uint32_t)(t.N / 2), tc2_box_k(t.K))))
        return fail(rc);
    }
    // the last layer's two directions (never split: N <= 128) are the table's last two entries
    const size_t nd = c->tc_dirs.size();
    tc_final_tiles_kernel<<<16, 256, 0, s>>>(c->fin.w, c->fin.C_out, c->fin.C_in, c->tc_dirs[nd - 2].w, c->tc_dirs[nd - 1].w);
    DGAN_CUDA_CHECK(cudaGetLastError());
  }
  // profile kinds, then the momentum update: fp16, the tc_directions() entries (a column block of a split layer-direction
  // is a kind of its own, with the share of the MACs that falls on its real channels); fp32, the layer-directions
  std::vector<double> lmacs;        // per logical layer-direction
  double fmacs = (double)c->macs_per_row;
  for (const GemmLayer& L : c->layers) {
    lmacs.insert(lmacs.end(), 2, (double)L.macs);      // forward, backward
    fmacs -= (double)L.macs;
  }
  lmacs.insert(lmacs.end(), 2, fmacs);                 // the last layer's forward, backward
  for (const TcDir& t : tc_directions(d)) {
    if (d->precision == DGAN_PREC_FP16) {
      const int real_in_block = std::max(0, std::min(t.N, t.n_real - t.col0));
      c->kind_names.push_back(t.kind);
      c->kind_macs_per_row.push_back(lmacs[(size_t)t.ld] * real_in_block / t.n_real);
    } else if (t.col0 == 0) {
      c->kind_names.push_back(t.base_kind);
      c->kind_macs_per_row.push_back(lmacs[(size_t)t.ld]);
    }
  }
  c->kind_names.push_back("momentum");
  c->kind_macs_per_row.push_back(0.0);
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
  Widths wd;
  if (const int rc = padded_widths(d, &wd)) return rc;
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

size_t dgan_workspace_bytes(dgan_handle h, int batch, int rec_rr) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0) return 0;
  return workspace_bytes(h, batch, rec_rr, WsShape());
}

size_t dgan_workspace_bytes_weighted(dgan_handle h, int batch, int rec_rr) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0) return 0;
  WsShape sh;
  sh.weighted = true;
  return workspace_bytes(h, batch, rec_rr, sh);
}

size_t dgan_workspace_bytes_measured(dgan_handle h, int batch, int rec_rr, int m) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0 || m <= 0 || m > h->hwc) return 0;
  WsShape sh;
  sh.m = m;
  return workspace_bytes(h, batch, rec_rr, sh);
}

// nnz within 0 .. m * H*W*C (the non-zeros an m-row operator can hold)
static bool csr_nnz_ok(dgan_handle h, int m, int nnz) { return nnz >= 0 && (int64_t)nnz <= (int64_t)m * h->hwc; }

size_t dgan_workspace_bytes_measured_csr(dgan_handle h, int batch, int rec_rr, int m, int nnz) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0 || m <= 0 || m > h->hwc || !csr_nnz_ok(h, m, nnz)) return 0;
  WsShape sh;
  sh.m = m;
  sh.nnz = nnz;
  return workspace_bytes(h, batch, rec_rr, sh);
}

int64_t dgan_last_launch_count(dgan_handle h) { return h ? h->last_launches : 0; }
int64_t dgan_last_enqueue_count(dgan_handle h) { return h ? h->last_enqueues : 0; }
int64_t dgan_macs_per_row(dgan_handle h) { return h ? h->macs_per_row : 0; }

int dgan_forward(dgan_handle h, const float* z_dev, int n_rows, float* y_dev, void* ws, size_t ws_bytes, void* stream) {
  if (h == nullptr || z_dev == nullptr || y_dev == nullptr || n_rows <= 0) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<Workspace> regs;
  int rc;
  if ((rc = check_ws(h, n_rows, 1, WsShape(), ws, ws_bytes, &regs))) return rc;
  const Workspace& w = regs[0];
  if ((rc = run_init_z(h, w, z_dev, 0, s))) return rc;
  if ((rc = run_forward(h, w, nullptr, 1, 1, false, s))) return rc;
  DGAN_CUDA_CHECK(cudaMemcpyAsync(y_dev, w.y, (size_t)n_rows * h->hwc * 4, cudaMemcpyDeviceToDevice, s));
  return DGAN_OK;
}

// The operator and measurements of a measured call (m = 0: not a measured call): dense a, or (nnz >= 0) the CSR rp, ci, val,
// or (conv not NULL) a convolution's geometry and kernels k [batch][kh][kw].
struct MeasuredArgs {
  const float* a = nullptr; const float* y = nullptr; int m = 0;
  const int* rp = nullptr; const int* ci = nullptr; const float* val = nullptr; int nnz = -1;
  const ConvGeom* conv = nullptr; const float* k = nullptr;
};

// m within 1 .. H*W*C and the operator and measurements given; 0 (*meas filled in), or DGAN_ERR_INVALID_ARG naming the
// bad argument
static int check_measured(dgan_handle h, const float* a_dev, int m, const float* y_dev, MeasuredArgs* meas) {
  if (m <= 0 || m > h->hwc) {
    set_error("m = " + std::to_string(m) + " is out of range: 1 <= m <= H*W*C = " + std::to_string(h->hwc));
    return DGAN_ERR_INVALID_ARG;
  }
  if (a_dev == nullptr) { set_error("NULL operator a_dev"); return DGAN_ERR_INVALID_ARG; }
  if (y_dev == nullptr) { set_error("NULL measurements y_dev"); return DGAN_ERR_INVALID_ARG; }
  meas->a = a_dev; meas->y = y_dev; meas->m = m;
  return 0;
}

// The same for a CSR operator: nnz within 0 .. m * H*W*C, row_ptr given, col_idx and val given unless nnz == 0.  The
// contents are validated on the device while they are staged (stage_measured_csr).
static int check_measured_csr(dgan_handle h, const int32_t* row_ptr, const int32_t* col_idx, const float* val, int m,
                              int nnz, const float* y_dev, MeasuredArgs* meas) {
  if (m <= 0 || m > h->hwc) {
    set_error("m = " + std::to_string(m) + " is out of range: 1 <= m <= H*W*C = " + std::to_string(h->hwc));
    return DGAN_ERR_INVALID_ARG;
  }
  if (!csr_nnz_ok(h, m, nnz)) {
    set_error("nnz = " + std::to_string(nnz) + " is out of range: 0 <= nnz <= m * H*W*C");
    return DGAN_ERR_INVALID_ARG;
  }
  if (row_ptr == nullptr) { set_error("NULL row_ptr"); return DGAN_ERR_INVALID_ARG; }
  if (nnz > 0 && (col_idx == nullptr || val == nullptr)) { set_error("NULL col_idx or val with nnz > 0"); return DGAN_ERR_INVALID_ARG; }
  if (y_dev == nullptr) { set_error("NULL measurements y_dev"); return DGAN_ERR_INVALID_ARG; }
  meas->y = y_dev; meas->m = m; meas->rp = row_ptr; meas->ci = col_idx; meas->val = val; meas->nnz = nnz;
  return 0;
}

// Stage a measured call's operator and measurements: dense, CSR or convolution
static int stage_meas(dgan_ctx* c, const Workspace& w, const MeasuredArgs& meas, int batch, cudaStream_t s) {
  if (w.conv) return stage_measured_conv(c, w, meas.k, meas.y, batch, s);
  if (w.csr) return stage_measured_csr(c, w, meas.rp, meas.ci, meas.val, meas.y, batch, s);
  return stage_measured(c, w, meas.a, meas.y, batch, s);
}

// The Huber entries' delta: > 0, +inf allowed (NaN, 0 and negative values are refused).  huber NULL: a squared-error
// call, nothing to check.  0, or DGAN_ERR_INVALID_ARG naming the bad value; the callers check it after every other
// argument and before anything is enqueued.
static int check_huber(const float* huber) {
  if (huber == nullptr || *huber > 0.f) return 0;
  set_error("invalid Huber delta = " + std::to_string(*huber) + ": it must be > 0 (+inf allowed)");
  return DGAN_ERR_INVALID_ARG;
}

// The prior entries' lambda: finite, >= 0, and 2 lambda finite (the gradient's coefficient, rounded on the host).
// z_prior NULL: a call without the prior, nothing to check.  0, or DGAN_ERR_INVALID_ARG naming the bad value; the callers
// check it after every other argument and before anything is enqueued.
static int check_z_prior(const float* z_prior) {
  if (z_prior == nullptr) return 0;
  const float l = *z_prior;
  if (std::isfinite(l) && l >= 0.f && std::isfinite(2.f * l)) return 0;
  set_error("invalid latent prior z_prior = " + std::to_string(l) + ": it must be finite and >= 0, with 2 z_prior finite");
  return DGAN_ERR_INVALID_ARG;
}

// The latent prior's part of a call's workspace and graph-cache key (z_prior not NULL, checked by check_z_prior).
static void set_prior(Workspace* w, dgan_ctx::LoopGraph* key, const float* z_prior) {
  if (z_prior == nullptr) return;
  if (w != nullptr) { w->prior = true; w->z_prior = *z_prior; }
  if (key != nullptr) { key->prior = 1; key->z_prior = *z_prior; }
}

// A call's sparse deviations (on: a *_sparse_dev entry, whose sd must not be NULL; dev_out NULL: nu is not returned)
struct SdevArgs { bool on = false; const dgan_sparse_dev* sd = nullptr; float* dev_out = nullptr; };

// The sparse-deviation entries' l1 and step: finite and >= 0, with eta = step n / 2 and tau = eta l1 (n: H*W*C, or the
// m of a measured call; both in double, rounded to fp32) finite in fp32, and dev_out 16-byte aligned (sdev_select_kernel
// stores 16 bytes at a time).  0 (*eta and *tau set), or DGAN_ERR_INVALID_ARG naming the bad value; the callers check it
// after every other argument and before anything is enqueued.
static int check_sparse_dev(const SdevArgs& a, int n, float* eta, float* tau) {
  if (!a.on) return 0;
  if (a.sd == nullptr) { set_error("NULL sparse_dev"); return DGAN_ERR_INVALID_ARG; }
  const float l1 = a.sd->l1, step = a.sd->step;
  std::string bad;
  if (!(std::isfinite(l1) && l1 >= 0.f)) bad = "l1 = " + std::to_string(l1) + " must be finite and >= 0";
  else if (!(std::isfinite(step) && step >= 0.f)) bad = "step = " + std::to_string(step) + " must be finite and >= 0";
  if (bad.empty()) {
    const double e = (double)step * (double)n / 2.0, t = e * (double)l1;
    *eta = (float)e;
    *tau = (float)t;
    if (!std::isfinite(*eta)) bad = "eta = step * n / 2 = " + std::to_string(e) + " overflows fp32";
    else if (!std::isfinite(*tau)) bad = "tau = eta * l1 = " + std::to_string(t) + " overflows fp32";
  }
  if (bad.empty() && ((uintptr_t)a.dev_out & 15) != 0) bad = "dev_out must be 16-byte aligned";
  if (bad.empty()) return 0;
  set_error("invalid sparse deviations: " + bad);
  return DGAN_ERR_INVALID_ARG;
}

// The sparse deviations' part of a call's workspace and graph-cache key (a.on, checked by check_sparse_dev)
static void set_sdev(Workspace* w, dgan_ctx::LoopGraph* key, const SdevArgs& a, float eta, float tau) {
  if (!a.on) return;
  if (w != nullptr) { w->sdev_eta = eta; w->sdev_tau = tau; w->sdev_l1 = a.sd->l1; }
  if (key != nullptr) { key->sdev = 1; key->sdev_l1 = a.sd->l1; key->sdev_step = a.sd->step; }
}

// After a loss finish of a sparse-deviation workspace (w.nu): J = loss + l1 sum |nu| per row (sdev_term_kernel)
static int sdev_term(dgan_ctx* c, const Workspace& w, cudaStream_t s) {
  if (w.nu == nullptr) return 0;
  sdev_term_kernel<<<(unsigned)((w.n_rows + 7) / 8), 256, 0, s>>>(w.nu, c->hwc, w.n_rows, w.sdev_l1, w.loss);
  DGAN_LAUNCH_CHECK(c);
  return 0;
}

// One projection's options, filled in by its entry after that entry's own argument checks.  The loss: the images x, with
// the per-pixel weights w (NULL: unweighted), or a measured loss (meas.m > 0, x and w NULL).  adam NULL: the momentum
// update; huber NULL: the squared error; z_prior NULL: no latent prior; sdev.on: sparse deviations.  pruned: the prune
// points sched (check_schedule); not pruned: one stage of rec_iters iterations.
struct Projection {
  const float* x = nullptr;
  const float* w = nullptr;
  MeasuredArgs meas;
  const dgan_adam_params* adam = nullptr;
  const float* huber = nullptr;
  const float* z_prior = nullptr;
  SdevArgs sdev;
  bool pruned = false;
  const dgan_prune_point* sched = nullptr;
  int n_points = 0;

  WsShape shape() const {
    WsShape sh;
    sh.weighted = w != nullptr;
    sh.m = meas.m; sh.nnz = meas.nnz; sh.conv = meas.conv;
    sh.adam = adam != nullptr;
    sh.sdev = sdev.on;
    if (pruned) { sh.sched = sched; sh.n_points = n_points; }
    return sh;
  }
};

// dgan_loss_grad (w_dev NULL) and dgan_loss_grad_weighted: the weighted forward reads the caller's weights in place.
// huber (not NULL): dgan_loss_grad_huber, the Huber loss at *huber.
static int loss_grad_impl(dgan_handle h, const float* x_dev, const float* w_dev, int batch, int rec_rr, const float* z_dev,
                          float* y_dev, float* loss_dev, float* grad_dev, void* ws, size_t ws_bytes, void* stream,
                          const float* huber = nullptr) {
  if (h == nullptr || x_dev == nullptr || z_dev == nullptr || batch <= 0 || rec_rr <= 0) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  cudaStream_t s = (cudaStream_t)stream;
  const int n_rows = batch * rec_rr;
  WsShape sh;
  sh.weighted = w_dev != nullptr;
  std::vector<Workspace> regs;
  int rc;
  if ((rc = check_ws(h, batch, rec_rr, sh, ws, ws_bytes, &regs))) return rc;
  Workspace& w = regs[0];
  if ((rc = check_huber(huber))) return rc;
  if (huber != nullptr) w.huber = *huber;
  if ((rc = run_init_z(h, w, z_dev, 0, s))) return rc;
  if ((rc = run_forward(h, w, x_dev, rec_rr, batch, true, s, true, w_dev))) return rc;
  if ((rc = run_backward(h, w, s))) return rc;
  loss_finish_kernel<<<(n_rows + 255) / 256, 256, 0, s>>>(w.loss_part, w.n_loss_parts, w.loss_stride_n, w.loss_stride_b, 1.0f / (float)h->hwc, n_rows, w.loss);
  DGAN_LAUNCH_CHECK(h);
  if (y_dev) DGAN_CUDA_CHECK(cudaMemcpyAsync(y_dev, w.y, (size_t)n_rows * h->hwc * 4, cudaMemcpyDeviceToDevice, s));
  if (loss_dev) DGAN_CUDA_CHECK(cudaMemcpyAsync(loss_dev, w.loss, (size_t)n_rows * 4, cudaMemcpyDeviceToDevice, s));
  if (grad_dev) {
    const size_t n = (size_t)n_rows * h->desc.latent_dim;
    scale_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.g, w.n_g_parts, (size_t)w.n_pad * h->wd.latent,
                                                                  grad_dev, grad_multiplier(h), n, nullptr, h->desc.latent_dim,
                                                                  h->wd.latent);
    DGAN_LAUNCH_CHECK(h);
  }
  return DGAN_OK;
}

int dgan_loss_grad(dgan_handle h, const float* x_dev, int batch, int rec_rr, const float* z_dev, float* y_dev,
                   float* loss_dev, float* grad_dev, void* ws, size_t ws_bytes, void* stream) {
  return loss_grad_impl(h, x_dev, nullptr, batch, rec_rr, z_dev, y_dev, loss_dev, grad_dev, ws, ws_bytes, stream);
}

int dgan_loss_grad_weighted(dgan_handle h, const float* x_dev, const float* w_dev, int batch, int rec_rr, const float* z_dev,
                            float* y_dev, float* loss_dev, float* grad_dev, void* ws, size_t ws_bytes, void* stream) {
  if (w_dev == nullptr) { set_error("NULL weights"); return DGAN_ERR_INVALID_ARG; }
  return loss_grad_impl(h, x_dev, w_dev, batch, rec_rr, z_dev, y_dev, loss_dev, grad_dev, ws, ws_bytes, stream);
}

// The measured loss_grad entries after their operator checks (p.meas); p.huber (not NULL): their Huber entries, the
// Huber loss at *p.huber
static int loss_grad_measured_impl(dgan_handle h, const Projection& p, int batch, int rec_rr, const float* z_dev,
                                   float* g_dev, float* loss_dev, float* grad_dev, void* ws, size_t ws_bytes, void* stream) {
  int rc;
  cudaStream_t s = (cudaStream_t)stream;
  const int n_rows = batch * rec_rr;
  std::vector<Workspace> regs;
  if ((rc = check_ws(h, batch, rec_rr, p.shape(), ws, ws_bytes, &regs))) return rc;
  Workspace& w = regs[0];
  if ((rc = check_huber(p.huber))) return rc;
  if (p.huber != nullptr) w.huber = *p.huber;
  h->n_rows_cur = n_rows;
  if ((rc = run_init_z(h, w, z_dev, 0, s)) || (rc = stage_meas(h, w, p.meas, batch, s))) return rc;
  if ((rc = run_forward(h, w, nullptr, 1, 1, true, s)) || (rc = launch_measure(h, w, rec_rr, s))) return rc;
  if ((rc = measured_backward(h, w, rec_rr, s)) || (rc = measured_loss_finish(h, w, s))) return rc;
  if (g_dev) DGAN_CUDA_CHECK(cudaMemcpyAsync(g_dev, w.y, (size_t)n_rows * h->hwc * 4, cudaMemcpyDeviceToDevice, s));
  DGAN_CUDA_CHECK(cudaMemcpyAsync(loss_dev, w.loss, (size_t)n_rows * 4, cudaMemcpyDeviceToDevice, s));
  const size_t n = (size_t)n_rows * h->desc.latent_dim;
  const bool tc = h->desc.precision == DGAN_PREC_FP16;
  scale_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.g, w.n_g_parts, (size_t)w.n_pad * h->wd.latent, grad_dev,
                                                                1.f, n, tc ? w.mscale : nullptr, h->desc.latent_dim,
                                                                h->wd.latent);
  DGAN_LAUNCH_CHECK(h);
  return DGAN_OK;
}

static bool loss_grad_args_ok(dgan_handle h, const float* z_dev, float* loss_dev, float* grad_dev, int batch, int rec_rr) {
  if (h == nullptr || z_dev == nullptr || loss_dev == nullptr || grad_dev == nullptr || batch <= 0 || rec_rr <= 0) {
    set_error("invalid argument");
    return false;
  }
  return true;
}

int dgan_loss_grad_measured(dgan_handle h, const float* a_dev, int m, const float* y_dev, int batch, int rec_rr,
                            const float* z_dev, float* g_dev, float* loss_dev, float* grad_dev, void* ws, size_t ws_bytes,
                            void* stream) {
  if (!loss_grad_args_ok(h, z_dev, loss_dev, grad_dev, batch, rec_rr)) return DGAN_ERR_INVALID_ARG;
  Projection p;
  if (int rc = check_measured(h, a_dev, m, y_dev, &p.meas)) return rc;
  return loss_grad_measured_impl(h, p, batch, rec_rr, z_dev, g_dev, loss_dev, grad_dev, ws, ws_bytes, stream);
}

int dgan_loss_grad_measured_csr(dgan_handle h, const int32_t* row_ptr, const int32_t* col_idx, const float* val, int m,
                                int nnz, const float* y_dev, int batch, int rec_rr, const float* z_dev, float* g_dev,
                                float* loss_dev, float* grad_dev, void* ws, size_t ws_bytes, void* stream) {
  if (!loss_grad_args_ok(h, z_dev, loss_dev, grad_dev, batch, rec_rr)) return DGAN_ERR_INVALID_ARG;
  Projection p;
  if (int rc = check_measured_csr(h, row_ptr, col_idx, val, m, nnz, y_dev, &p.meas)) return rc;
  return loss_grad_measured_impl(h, p, batch, rec_rr, z_dev, g_dev, loss_dev, grad_dev, ws, ws_bytes, stream);
}

int dgan_vjp(dgan_handle h, const float* z_dev, int n_rows, const float* dy_dev, float* y_dev, float* dz_dev, void* ws,
             size_t ws_bytes, void* stream) {
  if (h == nullptr || z_dev == nullptr || dy_dev == nullptr || dz_dev == nullptr || n_rows <= 0) {
    set_error("invalid argument");
    return DGAN_ERR_INVALID_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<Workspace> regs;
  int rc;
  if ((rc = check_ws(h, n_rows, 1, WsShape(), ws, ws_bytes, &regs))) return rc;
  Workspace& w = regs[0];
  h->n_rows_cur = n_rows;     // the FLOPs dgan_profile_read reports refer to this call
  // the forward of dgan_forward, keeping the ReLU masks; the cotangent replaces the loss's (y - x) in the last layer
  if ((rc = run_init_z(h, w, z_dev, 0, s))) return rc;
  if ((rc = run_forward(h, w, nullptr, 1, 1, true, s))) return rc;
  if ((rc = launch_cotangent(h, w, dy_dev, s))) return rc;
  if ((rc = run_backward(h, w, s))) return rc;
  const size_t n = (size_t)n_rows * h->desc.latent_dim;
  const bool tc = h->desc.precision == DGAN_PREC_FP16;
  scale_copy_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(w.g, w.n_g_parts, (size_t)w.n_pad * h->wd.latent, dz_dev,
                                                                1.f, n, tc ? w.loss : nullptr, h->desc.latent_dim, h->wd.latent);
  DGAN_LAUNCH_CHECK(h);
  if (y_dev) DGAN_CUDA_CHECK(cudaMemcpyAsync(y_dev, w.y, (size_t)n_rows * h->hwc * 4, cudaMemcpyDeviceToDevice, s));
  return DGAN_OK;
}

int dgan_jvp(dgan_handle h, const float* z_dev, int n_rows, const float* t_dev, float* y_dev, float* ty_dev, void* ws,
             size_t ws_bytes, void* stream) {
  if (h == nullptr || z_dev == nullptr || t_dev == nullptr || ty_dev == nullptr || n_rows <= 0) {
    set_error("invalid argument");
    return DGAN_ERR_INVALID_ARG;
  }
  cudaStream_t s = (cudaStream_t)stream;
  std::vector<Workspace> regs;
  int rc;
  if ((rc = check_ws(h, n_rows, 1, WsShape(), ws, ws_bytes, &regs))) return rc;
  Workspace& w = regs[0];
  if ((rc = plan_pass(h, n_rows, TC_PASS_TANGENT)) || (rc = build_maps(h, w, TC_PASS_TANGENT))) return rc;
  h->n_rows_cur = n_rows;
  const FinalLayer& f = h->fin;
  const bool tc = h->desc.precision == DGAN_PREC_FP16;
  const bool sigmoid = f.C_out == 1 && f.act == ACT_SIGMOID;
  if (!sigmoid && !(f.C_out == 3 && f.act == ACT_TANH)) { set_error("unsupported final layer"); return DGAN_ERR_UNSUPPORTED; }
  // the forward of dgan_forward, keeping the ReLU masks the tangent pass reads
  if ((rc = run_init_z(h, w, z_dev, 0, s))) return rc;
  if ((rc = run_forward(h, w, nullptr, 1, 1, true, s))) return rc;
  // the tangent of z, now that the primal Linear has read z_h: fp16 path, row n scaled by 2^e_n with its largest
  // |t| * 2^e_n in [0.25, 0.5) (one scale for the call with BatchNorm), the scales in w.loss
  const int latent = h->desc.latent_dim, ld = h->wd.latent;
  if (tc) {
    cotangent_rowmax_kernel<ACT_NONE><<<n_rows, 256, 0, s>>>(nullptr, t_dev, latent, w.loss);
    DGAN_LAUNCH_CHECK(h);
    cotangent_scale_kernel<<<1, 1024, 0, s>>>(w.loss, n_rows, h->desc.use_bn ? 1 : 0, -1);
    DGAN_LAUNCH_CHECK(h);
  }
  const size_t n_in = (size_t)w.n_pad * ld;
  tangent_in_kernel<<<(unsigned)((n_in + 255) / 256), 256, 0, s>>>(t_dev, tc ? w.loss : nullptr, n_rows, w.n_pad, latent, ld,
                                                                   tc ? nullptr : w.v, tc ? w.z_h : nullptr);
  DGAN_LAUNCH_CHECK(h);
  if ((rc = run_tangent(h, w, s))) return rc;
  // ty = t(pre) * act'(y) / scale
  const size_t total = (size_t)n_rows * h->hwc;
  const unsigned grid = (unsigned)((total + 255) / 256);
  const int w_out = 2 * f.w_in;
#define TO(ACT, CO, BLK) tangent_out_kernel<ACT, CO, BLK><<<grid, 256, 0, s>>>(w.y, w.dpre, n_rows, w_out, BLK ? w.loss : nullptr, w.n_pad, ty_dev)
  if (sigmoid) { if (tc) TO(ACT_SIGMOID, 1, true); else TO(ACT_SIGMOID, 1, false); }
  else { if (tc) TO(ACT_TANH, 3, true); else TO(ACT_TANH, 3, false); }
#undef TO
  DGAN_LAUNCH_CHECK(h);
  if (y_dev) DGAN_CUDA_CHECK(cudaMemcpyAsync(y_dev, w.y, (size_t)n_rows * h->hwc * 4, cudaMemcpyDeviceToDevice, s));
  return DGAN_OK;
}

int dgan_sample_z0(dgan_handle h, uint64_t seed, uint64_t z_row_offset, int n_rows, float* z_dev, void* stream) {
  if (h == nullptr || z_dev == nullptr || n_rows <= 0) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  const int latent = h->desc.latent_dim;
  const size_t total = (size_t)n_rows * latent;
  init_z_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(z_dev, nullptr, nullptr, nullptr, n_rows, n_rows, latent,
                                                                                   latent, seed, sqrtf(1.0f / (float)latent),
                                                                                   (size_t)z_row_offset * latent);
  DGAN_LAUNCH_CHECK(h);
  return DGAN_OK;
}

// Iterations t0 .. t1 - 1 of the L-step loop (models/gan.py:409-421) on workspace w, whose rows are `per_image` restarts
// of each of p.batch images.  Everything it reads or writes lives in the workspace, so it can be captured and replayed.
// The learning rate follows the global iteration t (decay from ceil(0.8 L) of the full L); iteration L-1, when it is in
// the range, is its forward alone.  loss_at_end: the forward of iteration t1 - 1 leaves its per-row loss parts in
// w.loss_part, as the forward of iteration L-1 does (the fp16 path's last-layer forward writes them, and y, only when it
// is asked for y).  adam (not NULL): the Adam update (adam_kernel, with m in w.v and s in w.s) instead of the momentum
// update; on the fp16 image loss the Linear backward then runs without its momentum tail and adam_kernel follows it.
// w.prior (the prior entries): iteration t1 - 1 first leaves each row's prior term on its z in w.loss (prior_term_kernel)
// for the loss finish that follows the range, and every update is the prior form of its kernel (the fp16 image loss's
// momentum runs as on the Adam path: the Linear backward without its tail, then momentum_prior_kernel).
// w.nu (the sparse-deviation entries, measured loop only): after each forward, nu's update from the previous iteration's
// dy and u = G(z) + nu (launch_sdev_update), which the data term reads.
static int enqueue_steps(dgan_ctx* h, const Workspace& w, const dgan_rec_params& p, int per_image, int t0, int t1,
                         bool measured, cudaStream_t ls, bool loss_at_end = false, const dgan_adam_params* adam = nullptr) {
  const int latent = h->wd.latent;
  const float two_lambda = 2.f * w.z_prior;     // finite: check_z_prior
  // Adam at iteration t (k = t + 1): c1 = lr_t / (1 - beta1^k) and c2 = 1 / sqrt(1 - beta2^k), in double, rounded to fp32
  auto launch_adam = [&](int t, float lr, float gmul, const float* row_scale) -> int {
    const double k = (double)t + 1.0;
    const float c1 = (float)((double)lr / (1.0 - std::pow((double)adam->beta1, k)));
    const float c2 = (float)(1.0 / std::sqrt(1.0 - std::pow((double)adam->beta2, k)));
    const size_t zcount = (size_t)w.n_pad * latent;
    ProfScope ps(h, 2 * (int)h->layers.size() + 2, ls);     // the profile kind of the latent update
    if (w.prior)
      DGAN_CUDA_CHECK(launch_pdl(adam_prior_kernel, dim3((unsigned)((zcount + 255) / 256)), dim3(256), 0, ls, w.z, w.v, w.s,
                                 (const float*)w.g, w.n_g_parts, gmul, row_scale, latent, w.n_rows, adam->beta1,
                                 adam->beta2, adam->eps, c1, c2, zcount, w.z_h, two_lambda));
    else
      DGAN_CUDA_CHECK(launch_pdl(adam_kernel, dim3((unsigned)((zcount + 255) / 256)), dim3(256), 0, ls, w.z, w.v, w.s,
                                 (const float*)w.g, w.n_g_parts, gmul, row_scale, latent, w.n_rows, adam->beta1,
                                 adam->beta2, adam->eps, c1, c2, zcount, w.z_h));
    DGAN_LAUNCH_CHECK(h);
    return 0;
  };
  const int decay_iter = (int)std::ceil(p.rec_iters * 0.8);
  // fp16: the momentum update (tf.train.MomentumOptimizer, models/gan.py:389-391) runs in the tail of the split-K Linear
  // backward - the CTA that completes a 128-row tile's partial sums applies it - so an L-step is 8 launches; bit-identical
  // to the separate kernel the fp32 path uses (same arithmetic, parts summed in the same order)
  const bool tail = h->desc.precision == DGAN_PREC_FP16 && !w.prior;
  for (int t = t0; t < t1; ++t) {
    const bool last = (t == p.rec_iters - 1);
    float lr = p.rec_lr;
    if (p.decay_lr) lr = p.rec_lr * std::pow(0.1f, (float)(t / decay_iter));
    if (w.prior && t == t1 - 1) {      // the z of the range's last iteration, before that iteration's update
      prior_term_kernel<<<(w.n_rows + 255) / 256, 256, 0, ls>>>(w.z, latent, h->desc.latent_dim, w.n_rows, w.z_prior,
                                                                 w.loss);
      DGAN_LAUNCH_CHECK(h);
    }
    // The loop returns the pre-update forward of iteration L-1 (models/gan.py:419-421, SURVEY F4):
    // the L-th update is never observed, so its backward pass is not run.
    int r2;
    if (measured) {
      // the forward of dgan_vjp (ReLU masks kept, y written every step: the measurement product reads it), then the
      // measured loss's gradient and the momentum update with the cotangent's row scales divided out
      if ((r2 = run_forward(h, w, nullptr, 1, 1, !last, ls))) return r2;
      if (w.nu != nullptr && (r2 = launch_sdev_update(h, w, t, ls))) return r2;
      if ((r2 = launch_measure(h, w, per_image, ls))) return r2;
      if (last) continue;
      if ((r2 = measured_backward(h, w, per_image, ls))) return r2;
      if (adam != nullptr) {
        if ((r2 = launch_adam(t, lr, 1.f, h->desc.precision == DGAN_PREC_FP16 ? w.mscale : nullptr))) return r2;
        continue;
      }
      const size_t zcount = (size_t)w.n_pad * latent;
      const float* row_scale = h->desc.precision == DGAN_PREC_FP16 ? w.mscale : nullptr;
      if (w.prior)
        momentum_rows_prior_kernel<<<(unsigned)((zcount + 255) / 256), 256, 0, ls>>>(
            w.z, w.v, w.g, w.n_g_parts, row_scale, latent, w.n_rows, lr, p.momentum, zcount, w.z_h, two_lambda);
      else
        momentum_rows_kernel<<<(unsigned)((zcount + 255) / 256), 256, 0, ls>>>(
            w.z, w.v, w.g, w.n_g_parts, row_scale, latent, w.n_rows, lr, p.momentum, zcount, w.z_h);
      DGAN_LAUNCH_CHECK(h);
      continue;
    }
    const bool want_y = last || (loss_at_end && t == t1 - 1);
    if ((r2 = run_forward(h, w, w.x, per_image, p.batch, !last, ls, want_y, w.xw))) return r2;
    if (last) continue;
    if (adam != nullptr) {
      if ((r2 = run_backward(h, w, ls)) || (r2 = launch_adam(t, lr, grad_multiplier(h), nullptr))) return r2;
      continue;
    }
    MomentumArgs mom;
    mom.lr = lr; mom.mu = p.momentum; mom.tail = tail;
    if ((r2 = run_backward(h, w, ls, mom))) return r2;
    if (!tail) {
      const size_t zcount = (size_t)w.n_pad * latent;
      ProfScope ps(h, 2 * (int)h->layers.size() + 2, ls);
      if (w.prior)
        DGAN_CUDA_CHECK(launch_pdl(momentum_prior_kernel, dim3((unsigned)((zcount + 255) / 256)), dim3(256), 0, ls, w.z,
                                   w.v, (const float*)w.g, w.n_g_parts, grad_multiplier(h), lr, p.momentum, zcount, w.z_h,
                                   two_lambda));
      else
        DGAN_CUDA_CHECK(launch_pdl(momentum_kernel, dim3((unsigned)((zcount + 255) / 256)), dim3(256), 0, ls, w.z, w.v,
                                   (const float*)w.g, w.n_g_parts, grad_multiplier(h), lr, p.momentum, zcount, w.z_h));
      DGAN_LAUNCH_CHECK(h);
    }
  }
  return 0;
}

// Run a call's loop, enqueue_loop(stream), on s: captured into a CUDA graph the first time `key` (exec and kernels unset)
// is seen and replayed with one cudaGraphLaunch afterwards, or launched plainly when per-kernel profiling is on or the
// capture fails.  Adds the stream operations the host issued to *enqueues.
static int run_loop(dgan_ctx* h, const dgan_ctx::LoopGraph& key, const std::function<int(cudaStream_t)>& enqueue_loop,
                    cudaStream_t s, int64_t* enqueues) {
  if (!h->profile && h->cap_stream != nullptr) {      // per-kernel event timing needs the plain launches
    dgan_ctx::LoopGraph* g = nullptr;
    for (auto& e : h->graphs)
      if (e.same_key(key)) { g = &e; break; }
    if (g == nullptr) {
      const int64_t k0 = h->launches;
      cudaGraph_t graph = nullptr;
      if (cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal) == cudaSuccess) {
        const int crc = enqueue_loop(h->cap_stream);
        const cudaError_t ce = cudaStreamEndCapture(h->cap_stream, &graph);
        cudaGraphExec_t exec = nullptr;
        if (crc == 0 && ce == cudaSuccess && graph != nullptr && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess) {
          if (h->graphs.size() >= 8) { cudaGraphExecDestroy(h->graphs.front().exec); h->graphs.erase(h->graphs.begin()); }
          h->graphs.push_back(key);
          h->graphs.back().exec = exec;
          h->graphs.back().kernels = h->launches - k0;
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
      *enqueues += 1;
      return 0;
    }
  }
  const int64_t k0 = h->launches;
  if (int rc = enqueue_loop(s)) return rc;
  *enqueues += h->launches - k0;
  return 0;
}

// The optimiser part of a loop's graph-cache key: the Adam hyper-parameters, or none for the momentum update.
static void set_optimizer_key(dgan_ctx::LoopGraph* key, const dgan_adam_params* adam) {
  if (adam == nullptr) return;
  key->adam = 1; key->beta1 = adam->beta1; key->beta2 = adam->beta2; key->eps = adam->eps;
}

// The operator part of a loop's graph-cache key: a convolution's geometry (its kernels are staged outside the graph).
static void set_conv_key(dgan_ctx::LoopGraph* key, const ConvGeom* g) {
  if (g != nullptr) key->conv = {g->kh, g->kw, g->ph, g->pw, g->s};
}

// Adam's hyper-parameters: 0 <= beta1 < 1, 0 <= beta2 < 1 and a finite eps > 0; 0, or DGAN_ERR_INVALID_ARG naming the bad
// value.
static int check_adam(const dgan_adam_params* a) {
  if (a == nullptr) { set_error("NULL Adam parameters"); return DGAN_ERR_INVALID_ARG; }
  std::string bad;
  if (!(a->beta1 >= 0.f && a->beta1 < 1.f)) bad = "beta1 = " + std::to_string(a->beta1) + " must be in [0, 1)";
  else if (!(a->beta2 >= 0.f && a->beta2 < 1.f)) bad = "beta2 = " + std::to_string(a->beta2) + " must be in [0, 1)";
  else if (!(a->eps > 0.f && std::isfinite(a->eps))) bad = "eps = " + std::to_string(a->eps) + " must be finite and > 0";
  if (bad.empty()) return 0;
  set_error("invalid Adam parameters: " + bad);
  return DGAN_ERR_INVALID_ARG;
}

// ---- restart pruning (dgan_reconstruct_pruned; kernels_prune.cuh) ------------------------------------------------------
// A schedule of n_points prune points: 1 <= iter_1 < iter_2 < ... (<= L - 1 when rec_iters > 0: the sizer does not know L)
// and rec_rr >= keep_1 >= keep_2 >= ... >= 1.  0, or DGAN_ERR_INVALID_ARG naming the bad point.
static int check_schedule(const dgan_prune_point* sched, int n_points, int rec_rr, int rec_iters) {
  if (sched == nullptr || n_points < 1) { set_error("a prune schedule needs at least one point (sched NULL or n_points < 1)"); return DGAN_ERR_INVALID_ARG; }
  if (rec_rr > kPruneMaxRestarts) {
    set_error("rec_rr = " + std::to_string(rec_rr) + ": a pruned call takes at most " + std::to_string(kPruneMaxRestarts) + " restarts");
    return DGAN_ERR_INVALID_ARG;
  }
  for (int k = 0; k < n_points; ++k) {
    const int it = sched[k].iter, keep = sched[k].keep;
    const int prev_it = k == 0 ? 0 : sched[k - 1].iter, prev_keep = k == 0 ? rec_rr : sched[k - 1].keep;
    std::string bad;
    if (it <= prev_it) bad = k == 0 ? "iter must be >= 1" : "iter must exceed the previous point's";
    else if (rec_iters > 0 && it > rec_iters - 1) bad = "iter must be <= rec_iters - 1 = " + std::to_string(rec_iters - 1);
    else if (keep < 1) bad = "keep must be >= 1";
    else if (keep > prev_keep) bad = k == 0 ? "keep must be <= rec_rr = " + std::to_string(rec_rr) : "keep must not exceed the previous point's";
    if (!bad.empty()) {
      set_error("prune point " + std::to_string(k) + " (iter " + std::to_string(it) + ", keep " + std::to_string(keep) + "): " + bad);
      return DGAN_ERR_INVALID_ARG;
    }
  }
  return 0;
}

// Every projection after its entry's checks.  The images and weights, or the operator and measurements, are staged into
// the workspace, so the captured loop reads the workspace only.  The loop runs n_points + 1 stages, stage k on region k
// of the workspace (plan_workspace): rec_rr restarts per image from z0 in the first, the survivors of prune point k in
// the others, whose z and v (and z_h, Adam's s, and the sparse deviations' nu and dy) the prune point gathers from the
// previous region; an unpruned projection is the one stage.  A measured loss (and every sparse-deviation loss, the image
// loss as the identity operator) runs the measured loop, whose forward leaves each iteration's loss parts in
// mloss_part, so a prune point sums them as the image loop's do loss_part.  p.adam: the Adam update.  p.huber: the
// Huber loss at *p.huber.  p.z_prior: J = D + *p.z_prior ||z||^2, a prune point's prior term on the z of iteration
// iter_k - 1 (before that iteration's update, as its D).  p.sdev.on: every loss J + l1 ||nu||_1, for the ranking and
// the arg-min.
static int project(dgan_handle h, const dgan_rec_params* prm, const Projection& p, const float* z0_dev, float* rec_dev,
                   float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  const bool measured = p.meas.m > 0, weighted = p.w != nullptr;
  if (h == nullptr || prm == nullptr || (p.x == nullptr && !measured) || rec_dev == nullptr) { set_error("NULL argument"); return DGAN_ERR_INVALID_ARG; }
  // the arg-min select stores the reconstructions 16 bytes at a time (select_kernel).  Checked before the
  // hyper-parameters, so that a call with batch = 0 tells whether a library refuses a misaligned rec_dev, running nothing
  if (((uintptr_t)rec_dev & 15) != 0) { set_error("rec_dev must be 16-byte aligned"); return DGAN_ERR_INVALID_ARG; }
  const int batch = prm->batch, rec_rr = prm->rec_rr, rec_iters = prm->rec_iters;
  if (batch <= 0 || rec_rr <= 0 || rec_iters <= 0) { set_error("batch, rec_rr and rec_iters must be positive"); return DGAN_ERR_INVALID_ARG; }
  int rc;
  if (p.pruned) {
    if ((rc = check_schedule(p.sched, p.n_points, rec_rr, rec_iters))) return rc;
    if (h->desc.use_bn) {
      set_error("restart pruning is not supported with use_bn: the batch statistics couple the rows, so dropping restarts "
                "would change the survivors' trajectories");
      return DGAN_ERR_UNSUPPORTED;
    }
  }
  const WsShape sh = p.shape();
  const int n_points = sh.n_points;
  std::vector<Workspace> regs;
  if ((rc = check_ws(h, batch, rec_rr, sh, ws, ws_bytes, &regs))) return rc;
  float eta = 0.f, tau = 0.f;
  if ((rc = check_huber(p.huber)) || (rc = check_z_prior(p.z_prior)) ||
      (rc = check_sparse_dev(p.sdev, measured ? p.meas.m : h->hwc, &eta, &tau)))
    return rc;
  for (Workspace& w : regs) {
    if (p.huber != nullptr) w.huber = *p.huber;
    set_prior(&w, nullptr, p.z_prior);
    set_sdev(&w, nullptr, p.sdev, eta, tau);
  }
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t launches0 = h->launches;
  int64_t enqueues = 0;
  // every region starts as a fresh workspace would: region 0 from z0, the others' z and v come from the prune points
  for (int k = 0; k <= n_points; ++k) {
    const Workspace& w = regs[(size_t)k];
    const int64_t l0 = h->launches;
    if (k == 0) {
      if ((rc = run_init_z(h, w, z0_dev, prm->seed, s, (size_t)prm->z_row_offset))) return rc;
    } else if ((rc = clear_start_state(h, w, s))) {
      return rc;
    }
    if (measured) {              // the operator, once for every region
      if (k == 0 && (rc = stage_meas(h, w, p.meas, batch, s))) return rc;
      enqueues += h->launches - l0;
      continue;
    }
    DGAN_CUDA_CHECK(cudaMemcpyAsync(w.x, p.x, (size_t)batch * h->hwc * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if (weighted) DGAN_CUDA_CHECK(cudaMemcpyAsync(w.xw, p.w, (size_t)batch * h->hwc * sizeof(float), cudaMemcpyDeviceToDevice, s));
    enqueues += (h->launches - l0) + 1 + (weighted ? 1 : 0);
  }
  // The loop (a function of the workspace and the hyper-parameters only)
  dgan_ctx::LoopGraph key{ws, batch, rec_rr, rec_iters, prm->decay_lr, (int)weighted, p.meas.m, p.meas.nnz, prm->rec_lr,
                          prm->momentum, {}, nullptr, 0};
  for (int k = 0; k < n_points; ++k) { key.prune.push_back(sh.sched[k].iter); key.prune.push_back(sh.sched[k].keep); }
  set_optimizer_key(&key, p.adam);
  key.huber = p.huber != nullptr ? *p.huber : 0.f;
  set_conv_key(&key, p.meas.conv);
  set_prior(nullptr, &key, p.z_prior);
  set_sdev(nullptr, &key, p.sdev, eta, tau);
  // the per-row loss of region w's last iteration, from the parts its last forward (image loss) or measurement product
  // (measured, and every sparse-deviation loss) left, with the deviations' term
  auto finish = [&](const Workspace& w, cudaStream_t ls) -> int {
    const int r2 = w.m > 0 ? measured_loss_finish(h, w, ls) : image_loss_finish(h, w, ls);
    return r2 ? r2 : sdev_term(h, w, ls);
  };
  // the stages and, between them, the prune points: the loss of iteration iter_k - 1 per row (its parts are still in
  // loss_part or mloss_part after that iteration's update), the survivors' maps and the gather of their z, v (and z_h)
  // into the next region
  auto enqueue_loop = [&](cudaStream_t ls) -> int {
    int r2;
    for (int k = 0; k <= n_points; ++k) {
      const Workspace& w = regs[(size_t)k];
      const int per = k == 0 ? rec_rr : sh.sched[k - 1].keep;
      const int t0 = k == 0 ? 0 : sh.sched[k - 1].iter, t1 = k == n_points ? rec_iters : sh.sched[k].iter;
      h->n_rows_cur = w.n_rows;
      if ((r2 = enqueue_steps(h, w, *prm, per, t0, t1, measured || p.sdev.on, ls, k < n_points, p.adam))) return r2;
      if (k == n_points) break;
      const Workspace& nx = regs[(size_t)k + 1];
      if ((r2 = finish(w, ls))) return r2;
      prune_select_kernel<<<batch, 256, 0, ls>>>(w.loss, k == 0 ? nullptr : w.orig, per, sh.sched[k].keep, nx.src, nx.orig);
      DGAN_LAUNCH_CHECK(h);
      const size_t total = (size_t)nx.n_pad * h->wd.latent;
      if (p.adam != nullptr)
        prune_gather_adam_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ls>>>(w.z, w.v, w.s, w.z_h, nx.src, nx.n_rows,
                                                                                 nx.n_pad, h->wd.latent, nx.z, nx.v, nx.s,
                                                                                 nx.z_h);
      else
        prune_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ls>>>(w.z, w.v, w.z_h, nx.src, nx.n_rows, nx.n_pad,
                                                                            h->wd.latent, nx.z, nx.v, nx.z_h);
      DGAN_LAUNCH_CHECK(h);
      if (p.sdev.on) {
        const size_t n4 = (size_t)nx.n_rows * h->hwc / 4;
        sdev_gather_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, ls>>>(w.nu, w.dym, nx.src, nx.n_rows, h->hwc, nx.nu,
                                                                         nx.dym);
        DGAN_LAUNCH_CHECK(h);
      }
    }
    return 0;
  };
  if ((rc = run_loop(h, key, enqueue_loop, s, &enqueues))) return rc;
  // the arg-min of the last stage; a pruned call maps each image's choice among its survivors to the original restart
  const Workspace& w = regs.back();
  const int per = n_points == 0 ? rec_rr : sh.sched[n_points - 1].keep;
  h->n_rows_cur = w.n_rows;
  const int64_t l0 = h->launches;
  if ((rc = finish(w, s))) return rc;
  select_kernel<<<batch, 256, 0, s>>>(w.loss, w.y, per, h->hwc, rec_dev, loss_dev, n_points == 0 ? idx_dev : w.sel);
  DGAN_LAUNCH_CHECK(h);
  if (n_points > 0) {
    prune_idx_kernel<<<(batch + 255) / 256, 256, 0, s>>>(w.sel, w.orig, per, batch, idx_dev);
    DGAN_LAUNCH_CHECK(h);
  }
  if (p.sdev.dev_out != nullptr) {
    sdev_select_kernel<<<batch, 256, 0, s>>>(w.loss, w.nu, per, h->hwc, p.sdev.dev_out);
    DGAN_LAUNCH_CHECK(h);
  }
  enqueues += h->launches - l0;
  h->last_enqueues = enqueues;
  h->last_launches = h->launches - launches0;
  return DGAN_OK;
}

// sched NULL with n_points 0: unpruned; anything else is a schedule under the rules of dgan_reconstruct_pruned
static bool unpruned(const dgan_prune_point* sched, int n_points) { return sched == nullptr && n_points == 0; }

// A sizer's schedule: unpruned, or one check_schedule accepts on a handle without use_bn
static bool sizer_sched_ok(dgan_handle h, int rec_rr, const dgan_prune_point* sched, int n_points) {
  return unpruned(sched, n_points) || (!h->desc.use_bn && check_schedule(sched, n_points, rec_rr, 0) == 0);
}

// The first checks of the entries that take Adam's parameters, in their order: adam's (always for the Adam entries,
// need_adam; otherwise when given), then the handle.
static int check_entry(dgan_handle h, const dgan_adam_params* adam, bool need_adam = false) {
  if (adam != nullptr || need_adam)
    if (int rc = check_adam(adam)) return rc;
  if (h == nullptr) { set_error("NULL argument"); return DGAN_ERR_INVALID_ARG; }
  return 0;
}

// The options an entry passes on besides its loss: adam (NULL: momentum), huber (NULL: squared error), z_prior (NULL: no
// prior) and the schedule (unpruned: sched NULL with n_points 0)
static Projection options(const dgan_adam_params* adam, const float* huber, const float* z_prior,
                          const dgan_prune_point* sched, int n_points) {
  Projection p;
  p.adam = adam; p.huber = huber; p.z_prior = z_prior;
  p.pruned = !unpruned(sched, n_points); p.sched = sched; p.n_points = n_points;
  return p;
}

size_t dgan_workspace_bytes_pruned(dgan_handle h, int batch, int rec_rr, const dgan_prune_point* sched, int n_points,
                                   int weighted) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0 || h->desc.use_bn || check_schedule(sched, n_points, rec_rr, 0) != 0) return 0;
  WsShape sh;
  sh.weighted = weighted != 0;
  sh.sched = sched; sh.n_points = n_points;
  return workspace_bytes(h, batch, rec_rr, sh);
}

int dgan_reconstruct_pruned(dgan_handle h, const dgan_rec_params* prm, const dgan_prune_point* sched, int n_points,
                            const float* x_dev, const float* w_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                            int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  Projection p = options(nullptr, nullptr, nullptr, sched, n_points);
  p.pruned = true;
  p.x = x_dev; p.w = w_dev;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

// m within 1 .. H*W*C and nnz -1 (a dense operator) or within 0 .. m * H*W*C (a CSR one)
static bool measured_pruned_args_ok(dgan_handle h, int m, int nnz) {
  return m > 0 && m <= h->hwc && (nnz == -1 || csr_nnz_ok(h, m, nnz));
}

size_t dgan_workspace_bytes_measured_pruned(dgan_handle h, int batch, int rec_rr, int m, int nnz,
                                            const dgan_prune_point* sched, int n_points) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0 || h->desc.use_bn || !measured_pruned_args_ok(h, m, nnz) ||
      check_schedule(sched, n_points, rec_rr, 0) != 0)
    return 0;
  WsShape sh;
  sh.m = m; sh.nnz = nnz;
  sh.sched = sched; sh.n_points = n_points;
  return workspace_bytes(h, batch, rec_rr, sh);
}

int dgan_reconstruct_measured_pruned(dgan_handle h, const dgan_rec_params* prm, const dgan_prune_point* sched, int n_points,
                                     const float* a_dev, int m, const float* y_dev, const float* z0_dev, float* rec_dev,
                                     float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, nullptr)) return rc;
  Projection p = options(nullptr, nullptr, nullptr, sched, n_points);
  p.pruned = true;
  if (int rc = check_measured(h, a_dev, m, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_csr_pruned(dgan_handle h, const dgan_rec_params* prm, const dgan_prune_point* sched,
                                         int n_points, const int32_t* row_ptr, const int32_t* col_idx, const float* val,
                                         int m, int nnz, const float* y_dev, const float* z0_dev, float* rec_dev,
                                         float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, nullptr)) return rc;
  Projection p = options(nullptr, nullptr, nullptr, sched, n_points);
  p.pruned = true;
  if (int rc = check_measured_csr(h, row_ptr, col_idx, val, m, nnz, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct(dgan_handle h, const dgan_rec_params* prm, const float* x_dev, const float* z0_dev, float* rec_dev,
                     float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  Projection p;
  p.x = x_dev;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_weighted(dgan_handle h, const dgan_rec_params* prm, const float* x_dev, const float* w_dev,
                              const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws,
                              size_t ws_bytes, void* stream) {
  if (w_dev == nullptr) { set_error("NULL weights"); return DGAN_ERR_INVALID_ARG; }
  Projection p;
  p.x = x_dev; p.w = w_dev;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured(dgan_handle h, const dgan_rec_params* prm, const float* a_dev, int m, const float* y_dev,
                              const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws,
                              size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, nullptr)) return rc;
  Projection p;
  if (int rc = check_measured(h, a_dev, m, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_csr(dgan_handle h, const dgan_rec_params* prm, const int32_t* row_ptr, const int32_t* col_idx,
                                  const float* val, int m, int nnz, const float* y_dev, const float* z0_dev, float* rec_dev,
                                  float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, nullptr)) return rc;
  Projection p;
  if (int rc = check_measured_csr(h, row_ptr, col_idx, val, m, nnz, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

// ---- Adam (kernels_adam.cuh): each entry is its momentum counterpart's code path with the Adam update -----------------
size_t dgan_workspace_bytes_adam(dgan_handle h, int batch, int rec_rr, int weighted, const dgan_prune_point* sched,
                                 int n_points) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0 || !sizer_sched_ok(h, rec_rr, sched, n_points)) return 0;
  WsShape sh;
  sh.weighted = weighted != 0; sh.adam = true;
  sh.sched = sched; sh.n_points = n_points;
  return workspace_bytes(h, batch, rec_rr, sh);
}

size_t dgan_workspace_bytes_measured_adam(dgan_handle h, int batch, int rec_rr, int m, int nnz, const dgan_prune_point* sched,
                                          int n_points) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0 || !measured_pruned_args_ok(h, m, nnz) ||
      !sizer_sched_ok(h, rec_rr, sched, n_points))
    return 0;
  WsShape sh;
  sh.m = m; sh.nnz = nnz; sh.adam = true;
  sh.sched = sched; sh.n_points = n_points;
  return workspace_bytes(h, batch, rec_rr, sh);
}

int dgan_reconstruct_adam(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                          const dgan_prune_point* sched, int n_points, const float* x_dev, const float* w_dev,
                          const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes,
                          void* stream) {
  if (int rc = check_entry(h, adam, true)) return rc;
  Projection p = options(adam, nullptr, nullptr, sched, n_points);
  p.x = x_dev; p.w = w_dev;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_adam(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                   const dgan_prune_point* sched, int n_points, const float* a_dev, int m, const float* y_dev,
                                   const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws,
                                   size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam, true)) return rc;
  Projection p = options(adam, nullptr, nullptr, sched, n_points);
  if (int rc = check_measured(h, a_dev, m, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_csr_adam(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                       const dgan_prune_point* sched, int n_points, const int32_t* row_ptr,
                                       const int32_t* col_idx, const float* val, int m, int nnz, const float* y_dev,
                                       const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws,
                                       size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam, true)) return rc;
  Projection p = options(adam, nullptr, nullptr, sched, n_points);
  if (int rc = check_measured_csr(h, row_ptr, col_idx, val, m, nnz, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

// ---- the Huber loss: each entry is its squared-error counterpart's code path with delta -------------------------------
// adam NULL: the momentum counterpart; sched NULL with n_points 0: the unpruned one.  The counterpart's checks come first.
int dgan_reconstruct_huber(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam, float huber_delta,
                           const dgan_prune_point* sched, int n_points, const float* x_dev, const float* w_dev,
                           const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes,
                           void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, &huber_delta, nullptr, sched, n_points);
  p.x = x_dev; p.w = w_dev;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_huber(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                    float huber_delta, const dgan_prune_point* sched, int n_points, const float* a_dev, int m,
                                    const float* y_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                                    int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, &huber_delta, nullptr, sched, n_points);
  if (int rc = check_measured(h, a_dev, m, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_csr_huber(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                        float huber_delta, const dgan_prune_point* sched, int n_points,
                                        const int32_t* row_ptr, const int32_t* col_idx, const float* val, int m, int nnz,
                                        const float* y_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                                        int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, &huber_delta, nullptr, sched, n_points);
  if (int rc = check_measured_csr(h, row_ptr, col_idx, val, m, nnz, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_loss_grad_huber(dgan_handle h, float huber_delta, const float* x_dev, const float* w_dev, int batch, int rec_rr,
                         const float* z_dev, float* y_dev, float* loss_dev, float* grad_dev, void* ws, size_t ws_bytes,
                         void* stream) {
  return loss_grad_impl(h, x_dev, w_dev, batch, rec_rr, z_dev, y_dev, loss_dev, grad_dev, ws, ws_bytes, stream, &huber_delta);
}

int dgan_loss_grad_measured_huber(dgan_handle h, float huber_delta, const float* a_dev, int m, const float* y_dev, int batch,
                                  int rec_rr, const float* z_dev, float* g_dev, float* loss_dev, float* grad_dev, void* ws,
                                  size_t ws_bytes, void* stream) {
  if (!loss_grad_args_ok(h, z_dev, loss_dev, grad_dev, batch, rec_rr)) return DGAN_ERR_INVALID_ARG;
  Projection p;
  p.huber = &huber_delta;
  if (int rc = check_measured(h, a_dev, m, y_dev, &p.meas)) return rc;
  return loss_grad_measured_impl(h, p, batch, rec_rr, z_dev, g_dev, loss_dev, grad_dev, ws, ws_bytes, stream);
}

int dgan_loss_grad_measured_csr_huber(dgan_handle h, float huber_delta, const int32_t* row_ptr, const int32_t* col_idx,
                                      const float* val, int m, int nnz, const float* y_dev, int batch, int rec_rr,
                                      const float* z_dev, float* g_dev, float* loss_dev, float* grad_dev, void* ws,
                                      size_t ws_bytes, void* stream) {
  if (!loss_grad_args_ok(h, z_dev, loss_dev, grad_dev, batch, rec_rr)) return DGAN_ERR_INVALID_ARG;
  Projection p;
  p.huber = &huber_delta;
  if (int rc = check_measured_csr(h, row_ptr, col_idx, val, m, nnz, y_dev, &p.meas)) return rc;
  return loss_grad_measured_impl(h, p, batch, rec_rr, z_dev, g_dev, loss_dev, grad_dev, ws, ws_bytes, stream);
}

// ---- convolution operators (kernels_measured_conv.cuh): a third operator kind through the measured drivers ----------
// The geometry of op on h's image: 1 <= kh <= min(H, 32), 1 <= kw <= min(W, 32), 0 <= 2 ph <= kh - 1,
// 0 <= 2 pw <= kw - 1, 1 <= stride <= 16.  false (with *why naming the bad value) outside that range.
static bool conv_geom(const dgan_ctx* h, const dgan_conv_op* op, ConvGeom* g, std::string* why = nullptr) {
  std::string bad;
  if (op->kh < 1 || op->kh > std::min(h->H, 32)) bad = "kh = " + std::to_string(op->kh) + " must be in [1, " + std::to_string(std::min(h->H, 32)) + "]";
  else if (op->kw < 1 || op->kw > std::min(h->W, 32)) bad = "kw = " + std::to_string(op->kw) + " must be in [1, " + std::to_string(std::min(h->W, 32)) + "]";
  else if (op->pad_h < 0 || 2 * op->pad_h > op->kh - 1) bad = "pad_h = " + std::to_string(op->pad_h) + " must satisfy 0 <= 2 pad_h <= kh - 1";
  else if (op->pad_w < 0 || 2 * op->pad_w > op->kw - 1) bad = "pad_w = " + std::to_string(op->pad_w) + " must satisfy 0 <= 2 pad_w <= kw - 1";
  else if (op->stride < 1 || op->stride > 16) bad = "stride = " + std::to_string(op->stride) + " must be in [1, 16]";
  if (!bad.empty()) {
    if (why != nullptr) *why = "invalid convolution operator: " + bad;
    return false;
  }
  *g = ConvGeom{h->H, h->W, h->C, op->kh, op->kw, op->pad_h, op->pad_w, op->stride,
                (h->H + 2 * op->pad_h - op->kh) / op->stride + 1, (h->W + 2 * op->pad_w - op->kw) / op->stride + 1};
  return true;
}

// A convolution call's operator arguments: op given with a geometry in range, k_dev and y_dev given.  0 (meas filled in,
// its conv pointing at *g), or DGAN_ERR_INVALID_ARG naming the bad argument.
static int check_measured_conv(dgan_handle h, const dgan_conv_op* op, const float* k_dev, const float* y_dev, ConvGeom* g,
                               MeasuredArgs* meas) {
  if (op == nullptr) { set_error("NULL convolution operator op"); return DGAN_ERR_INVALID_ARG; }
  std::string why;
  if (!conv_geom(h, op, g, &why)) { set_error(why); return DGAN_ERR_INVALID_ARG; }
  if (k_dev == nullptr) { set_error("NULL kernels k_dev"); return DGAN_ERR_INVALID_ARG; }
  if (y_dev == nullptr) { set_error("NULL measurements y_dev"); return DGAN_ERR_INVALID_ARG; }
  meas->y = y_dev; meas->m = g->Ho * g->Wo * g->C; meas->k = k_dev; meas->conv = g;
  return 0;
}

int dgan_conv_op_m(dgan_handle h, const dgan_conv_op* op) {
  ConvGeom g;
  if (h == nullptr || op == nullptr || !conv_geom(h, op, &g)) return 0;
  return g.Ho * g.Wo * g.C;
}

size_t dgan_workspace_bytes_measured_conv(dgan_handle h, int batch, int rec_rr, const dgan_conv_op* op,
                                          const dgan_prune_point* sched, int n_points, int adam) {
  ConvGeom g;
  if (h == nullptr || op == nullptr || batch <= 0 || rec_rr <= 0 || !conv_geom(h, op, &g) ||
      !sizer_sched_ok(h, rec_rr, sched, n_points))
    return 0;
  WsShape sh;
  sh.m = g.Ho * g.Wo * g.C; sh.conv = &g; sh.adam = adam != 0;
  sh.sched = sched; sh.n_points = n_points;
  return workspace_bytes(h, batch, rec_rr, sh);
}

int dgan_reconstruct_measured_conv(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                   const float* huber_delta, const dgan_prune_point* sched, int n_points,
                                   const dgan_conv_op* op, const float* k_dev, const float* y_dev, const float* z0_dev,
                                   float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes,
                                   void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, huber_delta, nullptr, sched, n_points);
  ConvGeom g;
  if (int rc = check_measured_conv(h, op, k_dev, y_dev, &g, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

// ---- the latent prior: each entry is its counterpart's code path with lambda = z_prior -------------------------------
// adam NULL: momentum; huber_delta NULL: the squared error; sched NULL with n_points 0: unpruned.  The counterpart's checks
// come first, then lambda's (check_z_prior), before anything is enqueued.
int dgan_reconstruct_prior(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam, const float* huber_delta,
                           float z_prior, const dgan_prune_point* sched, int n_points, const float* x_dev, const float* w_dev,
                           const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes,
                           void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, huber_delta, &z_prior, sched, n_points);
  p.x = x_dev; p.w = w_dev;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_prior(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                    const float* huber_delta, float z_prior, const dgan_prune_point* sched, int n_points,
                                    const float* a_dev, int m, const float* y_dev, const float* z0_dev, float* rec_dev,
                                    float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, huber_delta, &z_prior, sched, n_points);
  if (int rc = check_measured(h, a_dev, m, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_csr_prior(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                        const float* huber_delta, float z_prior, const dgan_prune_point* sched, int n_points,
                                        const int32_t* row_ptr, const int32_t* col_idx, const float* val, int m, int nnz,
                                        const float* y_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                                        int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, huber_delta, &z_prior, sched, n_points);
  if (int rc = check_measured_csr(h, row_ptr, col_idx, val, m, nnz, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_conv_prior(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                         const float* huber_delta, float z_prior, const dgan_prune_point* sched,
                                         int n_points, const dgan_conv_op* op, const float* k_dev, const float* y_dev,
                                         const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws,
                                         size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, huber_delta, &z_prior, sched, n_points);
  ConvGeom g;
  if (int rc = check_measured_conv(h, op, k_dev, y_dev, &g, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_loss_grad_measured_conv(dgan_handle h, const float* huber_delta, const dgan_conv_op* op, const float* k_dev,
                                 const float* y_dev, int batch, int rec_rr, const float* z_dev, float* g_dev,
                                 float* loss_dev, float* grad_dev, void* ws, size_t ws_bytes, void* stream) {
  if (!loss_grad_args_ok(h, z_dev, loss_dev, grad_dev, batch, rec_rr)) return DGAN_ERR_INVALID_ARG;
  Projection p;
  p.huber = huber_delta;
  ConvGeom g;
  if (int rc = check_measured_conv(h, op, k_dev, y_dev, &g, &p.meas)) return rc;
  return loss_grad_measured_impl(h, p, batch, rec_rr, z_dev, g_dev, loss_dev, grad_dev, ws, ws_bytes, stream);
}

// ---- sparse deviations (kernels_sparse_dev.cuh): each entry is its prior entry's code path on the measured loop --------
// with u = G(z) + nu in place of G(z).  adam NULL: momentum; huber_delta NULL: the squared error; z_prior NULL: no prior;
// sched NULL with n_points 0: unpruned.  The counterpart's checks come first, then check_sparse_dev's, before anything
// is enqueued.

// The sparse-deviation sizers' and layout's screening of their arguments (m 0: the image loss, weighted or not; m > 0:
// measured, nnz -1 dense or the CSR non-zeros, conv not NULL a convolution whose m was checked by the caller)
static bool sdev_args_ok(dgan_handle h, int batch, int rec_rr, bool weighted, int m, int nnz, const ConvGeom* conv,
                         const dgan_prune_point* sched, int n_points) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0) return false;
  if (m != 0 && (weighted || (conv == nullptr && !measured_pruned_args_ok(h, m, nnz)))) return false;
  return sizer_sched_ok(h, rec_rr, sched, n_points);
}

size_t dgan_workspace_bytes_sparse_dev(dgan_handle h, int batch, int rec_rr, int weighted, int adam,
                                       const dgan_prune_point* sched, int n_points) {
  if (!sdev_args_ok(h, batch, rec_rr, weighted != 0, 0, -1, nullptr, sched, n_points)) return 0;
  WsShape sh;
  sh.weighted = weighted != 0; sh.adam = adam != 0; sh.sdev = true;
  sh.sched = sched; sh.n_points = n_points;
  return workspace_bytes(h, batch, rec_rr, sh);
}

size_t dgan_workspace_bytes_measured_sparse_dev(dgan_handle h, int batch, int rec_rr, int m, int nnz, const dgan_conv_op* op,
                                                int adam, const dgan_prune_point* sched, int n_points) {
  ConvGeom g;
  if (op != nullptr) {
    if (h == nullptr || !conv_geom(h, op, &g) || m != g.Ho * g.Wo * g.C) return 0;
  } else if (m <= 0) {
    return 0;
  }
  const ConvGeom* conv = op != nullptr ? &g : nullptr;
  if (!sdev_args_ok(h, batch, rec_rr, false, m, nnz, conv, sched, n_points)) return 0;
  WsShape sh;
  sh.m = m; sh.nnz = conv != nullptr ? -1 : nnz; sh.conv = conv; sh.adam = adam != 0; sh.sdev = true;
  sh.sched = sched; sh.n_points = n_points;
  return workspace_bytes(h, batch, rec_rr, sh);
}

int dgan_reconstruct_sparse_dev(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                const float* huber_delta, const float* z_prior, const dgan_prune_point* sched, int n_points,
                                const dgan_sparse_dev* sparse_dev, float* dev_out, const float* x_dev, const float* w_dev,
                                const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws,
                                size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, huber_delta, z_prior, sched, n_points);
  p.sdev = SdevArgs{true, sparse_dev, dev_out};
  p.x = x_dev; p.w = w_dev;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_sparse_dev(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                         const float* huber_delta, const float* z_prior, const dgan_prune_point* sched,
                                         int n_points, const dgan_sparse_dev* sparse_dev, float* dev_out, const float* a_dev,
                                         int m, const float* y_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                                         int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, huber_delta, z_prior, sched, n_points);
  p.sdev = SdevArgs{true, sparse_dev, dev_out};
  if (int rc = check_measured(h, a_dev, m, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_csr_sparse_dev(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                             const float* huber_delta, const float* z_prior, const dgan_prune_point* sched,
                                             int n_points, const dgan_sparse_dev* sparse_dev, float* dev_out,
                                             const int32_t* row_ptr, const int32_t* col_idx, const float* val, int m, int nnz,
                                             const float* y_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                                             int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, huber_delta, z_prior, sched, n_points);
  p.sdev = SdevArgs{true, sparse_dev, dev_out};
  if (int rc = check_measured_csr(h, row_ptr, col_idx, val, m, nnz, y_dev, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
}

int dgan_reconstruct_measured_conv_sparse_dev(dgan_handle h, const dgan_rec_params* prm, const dgan_adam_params* adam,
                                              const float* huber_delta, const float* z_prior, const dgan_prune_point* sched,
                                              int n_points, const dgan_sparse_dev* sparse_dev, float* dev_out,
                                              const dgan_conv_op* op, const float* k_dev, const float* y_dev,
                                              const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev,
                                              void* ws, size_t ws_bytes, void* stream) {
  if (int rc = check_entry(h, adam)) return rc;
  Projection p = options(adam, huber_delta, z_prior, sched, n_points);
  p.sdev = SdevArgs{true, sparse_dev, dev_out};
  ConvGeom g;
  if (int rc = check_measured_conv(h, op, k_dev, y_dev, &g, &p.meas)) return rc;
  return project(h, prm, p, z0_dev, rec_dev, loss_dev, idx_dev, ws, ws_bytes, stream);
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
static int check_plans_impl(const dgan_desc* d, int n_rows, int n_pairs, int mutate, TcPass pass) {
  using namespace dgan;
  if (d == nullptr || n_rows <= 0 || n_pairs <= 0) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  const int n_pad = ((n_rows + 2 * kRowTile - 1) / (2 * kRowTile)) * 2 * kRowTile, n_mpairs = n_pad / (2 * kRowTile);
  Widths wd;
  if (int rc = padded_widths(d, &wd)) return rc;
  const std::string wide_target = pass == TC_PASS_TANGENT ? "Generator.3.jvp" : pass == TC_PASS_WEIGHTED ? "last.fwd.w" : "Generator.3.fwd";
  for (const TcDir& dr : tc_directions(d, pass)) {
    if (int rc = tc_dir_supported(dr)) return rc;
    Tc2Plan plan;
    const bool rev = tc2_band_reverse(dr.ld);
    int rc = tc2_plan(dr.N, dr.K, dr.tab, dr.h_grid, dr.w_grid, dr.max_acc, 0, dr.epi, dr.out_bytes, n_mpairs, n_pairs,
                      dr.order, rev, &plan);
    if (rc) { set_error(dr.name + ": " + dgan_last_error()); return rc; }
    // self-test of the validator: damage one plan in one specific way - faults 1-11 and 14-15 that of Generator.3 fwd (of
    // its tangent direction Generator.3.jvp for the tangent pass), faults 12-13 (specific to narrow ops) that of the last
    // layer's backward; the check must then fail.  Each fault but 6 and 9 decodes records, changes one field and encodes
    // them again.
    const bool narrow = (mutate == 12 || mutate == 13) && dr.name == "last.bwd";
    const bool wide = mutate != 0 && mutate != 12 && mutate != 13 && dr.name == wide_target;
    if ((narrow || wide) && plan.stream_m.size() > 40) {
      auto mma = [&](size_t i, auto f) { TcMmaRec m = TcMmaRec::decode(plan.stream_m[i]); f(m); plan.stream_m[i] = m.encode(); };
      auto producer = [&](size_t i, auto f) { TcProducerRec p = TcProducerRec::decode(plan.stream_p[i]); f(p); plan.stream_p[i] = p.encode(); };
      auto every_mma = [&](auto f) { for (size_t i = 0; i < plan.stream_m.size(); ++i) mma(i, f); };
      switch (mutate) {
        case 1: mma(20, [](TcMmaRec& m) {                                    // first-MMA flag of an op
                  TcOp op = TcOp::decode(m.ops[0]);
                  op.first ^= 1u;
                  m.ops[0] = op.encode();
                });
                break;
        case 2: mma(20, [](TcMmaRec& m) {                                    // accumulator of an op: swap two ops of round 0
                  for (uint32_t j = 1; j < m.maxb; ++j)
                    if (m.ops[j] != m.ops[0]) { std::swap(m.ops[0], m.ops[j]); break; }
                });
                break;
        case 3: producer(20, [](TcProducerRec& p) { p.tile[0] ^= 1u; }); break;   // weight tile of a B slot
        case 4: producer(20, [](TcProducerRec& p) { p.pix[0] ^= 1u; }); break;    // input pixel of an A tile
        case 5: producer(20, [](TcProducerRec& p) { p.kc ^= 1u; }); break;        // k-chunk
        case 6: plan.eitems[0] = -1; break;                                       // epilogue list loses an item
        case 7: for (size_t i = 0; i < plan.stream_p.size(); ++i)                 // every dep -> 8: ring hazards
                  producer(i, [](TcProducerRec& p) { p.dep = TC2_NSLOT; });
                break;
        case 8: producer(20, [](TcProducerRec& p) { p.off = 0xBF; }); break;      // region past the ring
        case 9: std::swap(plan.stream_m[20], plan.stream_m[21]);                  // two steps out of order
                std::swap(plan.stream_p[20], plan.stream_p[21]);
                break;
        case 10: plan.maxb = 3;                                                   // slots per round without an instantiation
                 every_mma([](TcMmaRec& m) { m.maxb = 3; });
                 break;
        case 11: every_mma([](TcMmaRec& m) { m.maxb = 2; }); break;               // records disagree with the plan's slots
        case 12: every_mma([&](TcMmaRec& m) { m.ksub = plan.ksub == 1 ? 2 : 1; }); break;   // k16 per op
        case 13: producer(20, [](TcProducerRec& p) { p.kc |= 1u; }); break;      // a k-chunk >= 1 (a narrow K has one)
        case 14: mma(20, [](TcMmaRec& m) {                                   // a round without a real op
                   for (uint32_t j = 0; j < m.maxb; ++j) m.ops[j] = TC2_PAD_OP;
                 });
                 break;
        case 15: {                                                            // a zero-tile op that overwrites
                   bool done = false;
                   for (size_t i = 20; i < plan.stream_m.size() && !done; ++i)
                     mma(i, [&](TcMmaRec& m) {
                       for (uint32_t j = 0; j < m.n_rounds * m.maxb && !done; ++j)
                         if (TcOp::decode(m.ops[j]).slot == (uint32_t)TC2_ZERO_SLOT) {
                           m.ops[j] = (uint8_t)TcOp::First::put(m.ops[j], 1u);
                           done = true;
                         }
                     });
                   break;
                 }
        default: break;
      }
    }
    std::string err;
    if ((rc = tc2_check_plan(dr.N, dr.K, dr.tab, n_mpairs, dr.epi, dr.out_bytes, plan, &err))) { set_error(dr.name + ": " + err); return rc; }
    if (mutate != 0) continue;
    // the plan in the other order (dgan_debug_force_order)
    Tc2Plan lpt;
    if ((rc = tc2_plan(dr.N, dr.K, dr.tab, dr.h_grid, dr.w_grid, dr.max_acc, 0, dr.epi, dr.out_bytes, n_mpairs, n_pairs,
                       TC2_ORDER_LPT, rev, &lpt))) {
      set_error(dr.name + " (LPT order): " + dgan_last_error());
      return rc;
    }
    if ((rc = tc2_check_plan(dr.N, dr.K, dr.tab, n_mpairs, dr.epi, dr.out_bytes, lpt, &err))) {
      set_error(dr.name + " (LPT order): " + err);
      return rc;
    }
    // the plans dgan_debug_force_slots can select: every other slot count this direction has an instantiation for
    for (const Tc2Kind& k : kTc2Kinds) {
      if (k.n != dr.N || k.ksub != plan.ksub || k.epi != dr.epi || k.out_bytes != dr.out_bytes || k.maxb == plan.maxb) continue;
      Tc2Plan forced;
      if ((rc = tc2_plan(dr.N, dr.K, dr.tab, dr.h_grid, dr.w_grid, dr.max_acc, k.maxb, dr.epi, dr.out_bytes, n_mpairs, n_pairs,
                         dr.order, rev, &forced))) {
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

int dgan_debug_check_plans(const dgan_desc* d, int n_rows, int n_pairs, int mutate) {
  return check_plans_impl(d, n_rows, n_pairs, mutate, TC_PASS_PROJ);
}

// The same for dgan_jvp's tangent directions (tc_directions(d, TC_PASS_TANGENT)); faults 1-11 damage Generator.3.jvp.
int dgan_debug_check_tangent_plans(const dgan_desc* d, int n_rows, int n_pairs, int mutate) {
  return check_plans_impl(d, n_rows, n_pairs, mutate, TC_PASS_TANGENT);
}

// The same for the weighted last-layer forward (tc_directions(d, TC_PASS_WEIGHTED)); faults 1-11 damage last.fwd.w.
int dgan_debug_check_weighted_plans(const dgan_desc* d, int n_rows, int n_pairs, int mutate) {
  return check_plans_impl(d, n_rows, n_pairs, mutate, TC_PASS_WEIGHTED);
}


// Host-side test aid (not in the public header): plan layer-direction `dir` (tc_directions order) of an fp16 handle with
// exactly `maxb` accumulator slots per round from now on (0: the planner chooses again).  Schedules and captured loops
// are re-made on the next call, so any instantiation of TC2_KINDS can be run at any batch size; the results must not
// change, because every accumulator keeps its summation order.
int dgan_debug_force_slots(dgan_handle h, int dir, int maxb) {
  if (h == nullptr || h->desc.precision != DGAN_PREC_FP16 || maxb < 0) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  if (dir < 0 || dir >= (int)h->tc_dirs.size()) { set_error("layer-direction out of range"); return DGAN_ERR_INVALID_ARG; }
  TcDir& d = h->tc_dirs[(size_t)dir];
  if (maxb > 0 && !tc2_has_kind(d.N, maxb, tc2_ksub(d.K), d.epi, d.out_bytes)) {
    set_error("no kernel instantiation with " + std::to_string(maxb) + " accumulator slots per round for this layer-direction");
    return DGAN_ERR_UNSUPPORTED;
  }
  d.force_maxb = maxb;
  d.by_mpairs.clear();                      // the uploaded tables stay in h->allocs until dgan_destroy
  for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
  h->graphs.clear();
  return DGAN_OK;
}

// Host-side test aid (not in the public header): plan every layer-direction of an fp16 handle in item order `order`
// (Tc2Order: 0 LPT, 1 banded, the default) from now on.  Schedules and captured loops are re-made on the next call.  The
// results must not change: the order only decides which CTA pair computes an item, and when.
int dgan_debug_force_order(dgan_handle h, int order) {
  if (h == nullptr || h->desc.precision != DGAN_PREC_FP16 || (order != TC2_ORDER_LPT && order != TC2_ORDER_BAND)) {
    set_error("invalid argument");
    return DGAN_ERR_INVALID_ARG;
  }
  h->tc_order = order;
  for (std::vector<TcDir>* dirs : {&h->tc_dirs, &h->tc_jvp_dirs, &h->tc_w_dirs})
    for (TcDir& d : *dirs) {
      d.order = order;
      d.by_mpairs.clear();                    // the uploaded tables stay in h->allocs until dgan_destroy
    }
  for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
  h->graphs.clear();
  return DGAN_OK;
}

// Host-side test aid: the accumulator slots per round the instantiations of TC2_KINDS offer for layer-direction `dir`,
// written to out[0 .. n).  Returns n, or -1.
int dgan_debug_slot_choices(dgan_handle h, int dir, int* out, int max_n) {
  if (h == nullptr || h->desc.precision != DGAN_PREC_FP16 || out == nullptr) return -1;
  if (dir < 0 || dir >= (int)h->tc_dirs.size()) return -1;
  const TcDir& d = h->tc_dirs[(size_t)dir];
  int n = 0;
  for (const Tc2Kind& k : kTc2Kinds)
    if (k.n == d.N && k.ksub == tc2_ksub(d.K) && k.epi == d.epi && k.out_bytes == d.out_bytes && n < max_n) out[n++] = k.maxb;
  return n;
}

#ifdef DGAN_PROBE
// Developer build only: copy (and clear) the per-CTA cycle counters of the tensor-core kernels.
// out: [48][160][TC2_PROBE_WORDS] u64.
int dgan_debug_probe_read(unsigned long long* out) {
  if (cudaDeviceSynchronize() != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(out, dgan::g_tc2_probe, sizeof(dgan::g_tc2_probe)) != cudaSuccess) return -1;
  static unsigned long long zeros[48 * 160 * dgan::TC2_PROBE_WORDS];
  if (cudaMemcpyToSymbol(dgan::g_tc2_probe, zeros, sizeof(zeros)) != cudaSuccess) return -1;
  return 0;
}
#endif

// Host-only developer aid (not in the public header): the plan of every layer-direction in numbers - window shape, items,
// steps, MMAs (ops of KSUB k16 each, and k16 MMAs), operand bytes staged from L2 into shared memory (both CTAs of every
// pair), accumulator slots per round, epilogue and output type - as text.  The MMA columns count every slot of every
// round, as the time model does; what the kernel issues and skips is in dgan_debug_plan_issue_stats.  Layer-direction
// `force_dir` (tc_directions order; -1: none) is planned with exactly `force_maxb` slots per round, as
// dgan_debug_force_slots would, and, when force_shape is not NULL, with exactly that window shape {wh, ww, sy, sx}.
// Returns the length.
static int plan_stats_impl(const dgan_desc* d, int n_rows, int n_pairs, int force_dir, int force_maxb, const int* force_shape,
                           char* buf, int buf_len) {
  using namespace dgan;
  if (d == nullptr || n_rows <= 0 || n_pairs <= 0 || buf == nullptr || buf_len <= 0) { set_error("invalid argument"); return -1; }
  const int n_pad = ((n_rows + 2 * kRowTile - 1) / (2 * kRowTile)) * 2 * kRowTile, n_mpairs = n_pad / (2 * kRowTile);
  Widths wd;
  if (padded_widths(d, &wd) != 0) return -1;
  std::string out = "direction | N | K | window (h x w, stride) | items | slots | steps | MMAs | staged MB | busiest pair / mean load"
                    " | zero-tile MMA % | MMAs per round | busiest pair: est. tensor us | busiest pair: est. us | k16 MMAs"
                    " | epilogue/output\n";
  auto epi_name = [](int epi) {
    switch (epi) {
      case EPI_BIAS_RELU: return "bias_relu";
      case EPI_BIAS: return "bias";
      case EPI_MASK: return "mask";
      case EPI_FINAL_SIGMOID1: return "final_sigmoid";
      case EPI_FINAL_TANH3: return "final_tanh";
      default: return "none";
    }
  };
  double total = 0.0;
  const std::vector<TcDir> dirs = tc_directions(d);
  for (size_t di = 0; di < dirs.size(); ++di) {
    const TcDir& dr = dirs[di];
    Tc2Plan plan;
    const bool forced = (int)di == force_dir;
    const int rc = tc2_plan(dr.N, dr.K, dr.tab, dr.h_grid, dr.w_grid, dr.max_acc, forced ? force_maxb : 0, dr.epi, dr.out_bytes,
                            n_mpairs, n_pairs, dr.order, tc2_band_reverse(dr.ld), &plan, forced ? force_shape : nullptr);
    if (rc) return -1;
    char line[320];
    const double mb = (double)plan.n_bytes / 1e6;
    total += mb;
    snprintf(line, sizeof line, "%s | %d | %d | %dx%d, %dx%d | %zu | %d | %lld | %lld | %.1f | %.3f | %.1f | %d | %.1f | %.1f | %lld | %s/f%d\n",
             dr.name.c_str(), dr.N, dr.K, plan.shape[0], plan.shape[1], plan.shape[2], plan.shape[3],
             plan.hdrs.size() * (size_t)n_mpairs, plan.n_slots, plan.n_steps, plan.n_mma, mb, plan.load_max / std::max(plan.load_mean, 1.0),
             100.0 * (double)plan.n_pad / (double)std::max(plan.n_mma, 1LL), plan.maxb, plan.op_ns_max / 1e3,
             plan.load_max / 1e3, plan.n_mma * plan.ksub, epi_name(dr.epi), 8 * dr.out_bytes);
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

// Host-only developer aid (not in the public header): the item order of every layer-direction's plan in item order
// `order` (Tc2Order) - the order the planner kept (it falls back to LPT when bands would unbalance the pairs), the row
// pairs per band, the busiest CTA pair's load under LPT and under the kept order (cost-model us), the bytes staged into
// shared memory as activation tiles (both CTAs) and as weight tiles, the distinct activation tiles read (the input
// tensor), and the working set: the peak, over the cost model's timeline of every pair, of the bytes of activation tiles
// between their first and last load - as text, one line per layer-direction in the order of dgan_debug_plan_stats.
// Returns the length, or -1.
int dgan_debug_plan_order_stats(const dgan_desc* d, int n_rows, int n_pairs, int order, char* buf, int buf_len) {
  using namespace dgan;
  if (d == nullptr || n_rows <= 0 || n_pairs <= 0 || buf == nullptr || buf_len <= 0 ||
      (order != TC2_ORDER_LPT && order != TC2_ORDER_BAND)) {
    set_error("invalid argument");
    return -1;
  }
  const int n_pad = ((n_rows + 2 * kRowTile - 1) / (2 * kRowTile)) * 2 * kRowTile, n_mpairs = n_pad / (2 * kRowTile);
  Widths wd;
  if (padded_widths(d, &wd) != 0) return -1;
  std::string out = "direction | order | band row pairs | busiest pair: LPT us | busiest pair: order us | staged A MB"
                    " | staged weight MB | unique input MB | working set MB\n";
  for (const TcDir& dr : tc_directions(d)) {
    Tc2Plan plan;
    if (tc2_plan(dr.N, dr.K, dr.tab, dr.h_grid, dr.w_grid, dr.max_acc, 0, dr.epi, dr.out_bytes, n_mpairs, n_pairs, order,
                 tc2_band_reverse(dr.ld), &plan))
      return -1;
    char line[240];
    snprintf(line, sizeof line, "%s | %s | %d | %.1f | %.1f | %.1f | %.1f | %.1f | %.1f\n", dr.name.c_str(),
             plan.order == TC2_ORDER_BAND ? (tc2_band_reverse(dr.ld) ? "band-" : "band+") : "lpt", plan.band_rows,
             plan.load_max / 1e3, plan.load_max_order / 1e3, plan.n_bytes_a / 1e6, plan.n_bytes_b / 1e6,
             plan.uniq_a_bytes / 1e6, plan.ws_a_bytes / 1e6);
    out += line;
  }
  const int n = (int)std::min(out.size(), (size_t)buf_len - 1);
  memcpy(buf, out.data(), (size_t)n);
  buf[n] = 0;
  return n;
}

// Host-only developer aid (not in the public header): what the kernel issues for the plan of every layer-direction -
// the slots per round, the k16 MMAs issued (the real ones, and the zero-tile ones where the round is fixed:
// tc2_issues_zero_ops), the zero-tile k16 MMAs the kernel skips, and the MMA term of the busiest CTA pair's load for the
// MMAs issued (est. tensor us) - as text, one line per layer-direction in the order of dgan_debug_plan_stats.  The plans
// are the ones dgan_debug_plan_stats describes.  Returns the length, or -1.
int dgan_debug_plan_issue_stats(const dgan_desc* d, int n_rows, int n_pairs, char* buf, int buf_len) {
  using namespace dgan;
  if (d == nullptr || n_rows <= 0 || n_pairs <= 0 || buf == nullptr || buf_len <= 0) { set_error("invalid argument"); return -1; }
  const int n_pad = ((n_rows + 2 * kRowTile - 1) / (2 * kRowTile)) * 2 * kRowTile, n_mpairs = n_pad / (2 * kRowTile);
  Widths wd;
  if (padded_widths(d, &wd) != 0) return -1;
  std::string out = "direction | slots | k16 MMAs issued | zero-tile k16 MMAs skipped | busiest pair: est. tensor us, issued\n";
  for (const TcDir& dr : tc_directions(d)) {
    Tc2Plan plan;
    if (tc2_plan(dr.N, dr.K, dr.tab, dr.h_grid, dr.w_grid, dr.max_acc, 0, dr.epi, dr.out_bytes, n_mpairs, n_pairs, dr.order,
                 tc2_band_reverse(dr.ld), &plan))
      return -1;
    char line[200];
    snprintf(line, sizeof line, "%s | %d | %lld | %lld | %.1f\n", dr.name.c_str(), plan.maxb, plan.n_issued * plan.ksub,
             (plan.n_mma - plan.n_issued) * plan.ksub, plan.op_ns_issued_max / 1e3);
    out += line;
  }
  const int n = (int)std::min(out.size(), (size_t)buf_len - 1);
  memcpy(buf, out.data(), (size_t)n);
  buf[n] = 0;
  return n;
}

// Host-only aid (not in the public header): the widths a handle for `d` stores - out[0..4) = latent, 4 * net_dim,
// 2 * net_dim, net_dim, padded by padded_widths().  Returns 0, or its error code with the limit in dgan_last_error().
int dgan_debug_padded_widths(const dgan_desc* d, int* out) {
  using namespace dgan;
  if (d == nullptr || out == nullptr) { set_error("invalid argument"); return DGAN_ERR_INVALID_ARG; }
  Widths w;
  if (int rc = padded_widths(d, &w)) return rc;
  out[0] = w.latent; out[1] = w.c4; out[2] = w.c2; out[3] = w.c1;
  return 0;
}

// Host-only test aid (not in the public header): the workspace of handle h for n_rows latent rows as text, from carve()
// itself - lines "n_rows N", "n_pad N", "widths latent c4 c2 c1" (padded), "g_parts N", then one line per buffer:
// "name type byte_offset dim0 dim1 ..." (type f32, f16, u64 or u32; dims in storage order, outermost first; the mask
// words of layer l are "mask.l" [P_out][n_pad][C_out / 64]).  Returns the length, or -1 when buf is too small.
// Every layout aid plans its workspace as its sizer does (plan_workspace).
static int write_layout(dgan_handle h, int batch, int rec_rr, const WsShape& sh, char* buf, int buf_len) {
  std::string out;
  size_t bytes = 0;
  if (plan_workspace(h, batch, rec_rr, sh, nullptr, &out, nullptr, &bytes)) return -1;
  if (out.size() + 1 > (size_t)buf_len) { set_error("buffer too small"); return -1; }
  memcpy(buf, out.c_str(), out.size() + 1);
  return (int)out.size();
}

static bool layout_args_ok(dgan_handle h, int n_rows, char* buf, int buf_len) {
  if (h == nullptr || n_rows <= 0 || buf == nullptr || buf_len <= 0) { set_error("invalid argument"); return false; }
  return true;
}

int dgan_debug_workspace_layout(dgan_handle h, int n_rows, char* buf, int buf_len) {
  if (!layout_args_ok(h, n_rows, buf, buf_len)) return -1;
  return write_layout(h, n_rows, 1, WsShape(), buf, buf_len);
}

// The same for the workspace of the weighted entries (dgan_workspace_bytes_weighted): the weights are "xw" [n_pad][H*W*C].
int dgan_debug_workspace_layout_weighted(dgan_handle h, int n_rows, char* buf, int buf_len) {
  if (!layout_args_ok(h, n_rows, buf, buf_len)) return -1;
  WsShape sh;
  sh.weighted = true;
  return write_layout(h, n_rows, 1, sh, buf, buf_len);
}

// The same for the workspace of the measured entries for m measurements (dgan_workspace_bytes_measured): after the
// unweighted buffers, "am" [m_ld][H*W*C], "amt" [H*W*C][m_ld], "ym" [n_pad][m_ld], "r" [n_pad][m_ld], "dym"
// [n_pad][H*W*C], "mloss_part" [m_ld / 64][n_pad] and "mscale" [n_pad].
int dgan_debug_workspace_layout_measured(dgan_handle h, int n_rows, int m, char* buf, int buf_len) {
  if (h == nullptr || m <= 0 || m > h->hwc) { set_error("invalid argument"); return -1; }
  if (!layout_args_ok(h, n_rows, buf, buf_len)) return -1;
  WsShape sh;
  sh.m = m;
  return write_layout(h, n_rows, 1, sh, buf, buf_len);
}

// The same for the workspace of the CSR-measured entries for m measurements and nnz non-zeros
// (dgan_workspace_bytes_measured_csr): after the unweighted buffers, the measured ones without "am" and "amt", then the
// staged operator "a_rp" i32 [m_ld + 1], "a_ci" i32 [nnz], "a_v" f32 [nnz], its transpose "at_rp" i32 [H*W*C + 1],
// "at_ci" i32 [nnz], "at_v" f32 [nnz], the bad-row marks "csr_bad" i32 [m_ld] and the validity flag "csr_valid" i32 [1]
// (1: the caller's CSR was valid; 0: it was staged as the empty operator with NaN measurements).
int dgan_debug_workspace_layout_measured_csr(dgan_handle h, int n_rows, int m, int nnz, char* buf, int buf_len) {
  if (h == nullptr || m <= 0 || m > h->hwc || !csr_nnz_ok(h, m, nnz)) { set_error("invalid argument"); return -1; }
  if (!layout_args_ok(h, n_rows, buf, buf_len)) return -1;
  WsShape sh;
  sh.m = m; sh.nnz = nnz;
  return write_layout(h, n_rows, 1, sh, buf, buf_len);
}

// The same for the workspace of dgan_reconstruct_pruned (dgan_workspace_bytes_pruned): per region a line
// "region k byte_offset n_rows" (the offset from the workspace's start), then that region's lines as above - offsets
// relative to the region - ending with the prune maps "orig", "src" and "sel", i32 [n_pad] each.
int dgan_debug_workspace_layout_pruned(dgan_handle h, int batch, int rec_rr, const dgan_prune_point* sched, int n_points,
                                       int weighted, char* buf, int buf_len) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0 || buf == nullptr || buf_len <= 0) { set_error("invalid argument"); return -1; }
  if (check_schedule(sched, n_points, rec_rr, 0) != 0) return -1;
  WsShape sh;
  sh.weighted = weighted != 0;
  sh.sched = sched; sh.n_points = n_points;
  return write_layout(h, batch, rec_rr, sh, buf, buf_len);
}

// The same for the workspace of dgan_reconstruct_measured[_csr]_pruned (dgan_workspace_bytes_measured_pruned; nnz -1 for
// a dense operator): first a line "operator 0 batch" and the operator block's lines - "am" f32 [m_ld][H*W*C] and "amt"
// f32 [H*W*C][m_ld], or the CSR buffers of dgan_debug_workspace_layout_measured_csr, then "ym" f32 [batch][m_ld] - then
// per region a line "region k byte_offset n_rows" and that region's lines: the unweighted buffers, the row-sized measured
// ones "r", "dym", "mloss_part" and "mscale", and the prune maps.
int dgan_debug_workspace_layout_measured_pruned(dgan_handle h, int batch, int rec_rr, int m, int nnz,
                                                const dgan_prune_point* sched, int n_points, char* buf, int buf_len) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0 || buf == nullptr || buf_len <= 0 || !measured_pruned_args_ok(h, m, nnz)) {
    set_error("invalid argument");
    return -1;
  }
  if (check_schedule(sched, n_points, rec_rr, 0) != 0) return -1;
  WsShape sh;
  sh.m = m; sh.nnz = nnz;
  sh.sched = sched; sh.n_points = n_points;
  return write_layout(h, batch, rec_rr, sh, buf, buf_len);
}

// The same for the workspace of the Adam entries (dgan_workspace_bytes_adam with m = 0, dgan_workspace_bytes_measured_adam
// with m > 0; nnz -1 for a dense operator): unpruned (sched NULL, n_points 0), the layout of
// dgan_debug_workspace_layout[_weighted / _measured / _measured_csr] with one line more at its end, the second moment
// "s" f32 [n_pad][latent_pad]; pruned, that of dgan_debug_workspace_layout[_measured]_pruned with "s" at the end of each
// region (so each later region starts that much further on).
int dgan_debug_workspace_layout_adam(dgan_handle h, int batch, int rec_rr, int weighted, int m, int nnz,
                                     const dgan_prune_point* sched, int n_points, char* buf, int buf_len) {
  if (h == nullptr || batch <= 0 || rec_rr <= 0 || buf == nullptr || buf_len <= 0 ||
      (m != 0 && !measured_pruned_args_ok(h, m, nnz)) || (m > 0 && weighted)) {
    set_error("invalid argument");
    return -1;
  }
  if (!unpruned(sched, n_points) && check_schedule(sched, n_points, rec_rr, 0) != 0) return -1;
  WsShape sh;
  sh.weighted = weighted != 0; sh.m = m; sh.nnz = m > 0 ? nnz : -1; sh.adam = true;
  sh.sched = sched; sh.n_points = n_points;
  return write_layout(h, batch, rec_rr, sh, buf, buf_len);
}

// The same for the workspace of the convolution-measured entries (dgan_workspace_bytes_measured_conv, unpruned, without
// Adam): after the unweighted buffers, the measured ones without "am" and "amt" - "ym" [n_pad][m_ld], "r" [n_pad][m_ld],
// "dym" [n_pad][H*W*C], "mloss_part" [m_ld / 64][n_pad], "mscale" [n_pad] - then the staged kernels "ck" f32
// [n_pad][kh * kw] (image b's at row b).
int dgan_debug_workspace_layout_measured_conv(dgan_handle h, int n_rows, const dgan_conv_op* op, char* buf, int buf_len) {
  ConvGeom g;
  if (h == nullptr || op == nullptr || !conv_geom(h, op, &g) || n_rows <= 0 || buf == nullptr || buf_len <= 0) {
    set_error("invalid argument");
    return -1;
  }
  WsShape sh;
  sh.m = g.Ho * g.Wo * g.C; sh.conv = &g;
  return write_layout(h, n_rows, 1, sh, buf, buf_len);
}

// The same for the workspace of the sparse-deviation entries (dgan_workspace_bytes_sparse_dev with m = 0,
// dgan_workspace_bytes_measured_sparse_dev with m > 0; nnz -1 for a dense or convolution operator, op not NULL for a
// convolution): the layout of the counterpart - unpruned or pruned, Adam or not - with, at the end of the workspace or of
// each region, for the image loss "dym" f32 [n_pad][H*W*C], "mloss_part" f32 [m_ld / 64][n_pad] and "mscale" f32 [n_pad]
// (m_ld: H*W*C rounded up to 64), then "nu" and "u", f32 [n_pad][H*W*C] each.
int dgan_debug_workspace_layout_sparse_dev(dgan_handle h, int batch, int rec_rr, int weighted, int m, int nnz,
                                           const dgan_conv_op* op, int adam, const dgan_prune_point* sched, int n_points,
                                           char* buf, int buf_len) {
  ConvGeom g;
  if (h == nullptr || buf == nullptr || buf_len <= 0 || (op != nullptr && (!conv_geom(h, op, &g) || m != g.Ho * g.Wo * g.C))) {
    set_error("invalid argument");
    return -1;
  }
  const ConvGeom* conv = op != nullptr ? &g : nullptr;
  if (!sdev_args_ok(h, batch, rec_rr, weighted != 0, m, nnz, conv, sched, n_points)) {
    set_error("invalid argument");
    return -1;
  }
  WsShape sh;
  sh.weighted = weighted != 0; sh.m = m; sh.nnz = m > 0 && conv == nullptr ? nnz : -1; sh.conv = conv;
  sh.adam = adam != 0; sh.sdev = true;
  sh.sched = sched; sh.n_points = n_points;
  return write_layout(h, batch, rec_rr, sh, buf, buf_len);
}

int dgan_debug_plan_stats(const dgan_desc* d, int n_rows, int n_pairs, char* buf, int buf_len) {
  return dgan_debug_plan_stats_slots(d, n_rows, n_pairs, -1, 0, buf, buf_len);
}

}  // extern "C"
