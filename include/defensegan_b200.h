/*
 * defensegan_b200.h - C ABI of the H100-native Defense-GAN projection loop.
 *
 * The reference (kabkabm/defensegan) has no FFI/plugin interface: the boundary is the Python
 * method DefenseGANBase.reconstruct (models/gan.py:333-449) plus the eval driver
 * utils/gan_defense.py:32-179.  This header is the C-ABI that sits directly underneath that
 * Python surface (SURVEY.md section 8b); each entry point cites the reference lines it replaces.
 * Plain pointers and sizes only - no torch types.  All device pointers are owned by the
 * caller; the handle owns its own copies of the weights (plain and re-laid-out), so the tensors passed
 * to dgan_create may be freed once `stream` has run the copies.  Nothing is freed across the boundary.  No function synchronises the host: work is enqueued on `stream`.
 *
 * Every function returns 0 on success, a negative dgan_status otherwise; the message is
 * available (thread-local) from dgan_last_error().  No C++ exception crosses the boundary.
 */
#ifndef DEFENSEGAN_B200_H_
#define DEFENSEGAN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DGAN_ABI_VERSION 2

typedef struct dgan_ctx* dgan_handle;

enum dgan_status {
  DGAN_OK = 0,
  DGAN_ERR_INVALID_ARG = -1,
  DGAN_ERR_CUDA = -2,
  DGAN_ERR_UNSUPPORTED = -3,
  DGAN_ERR_WORKSPACE = -4
};

/* generator architectures (models/dataset_models.py:36-71 mnist_generator - also used by
 * F-MNIST, models/gan.py:688-698 - and :127-165 celeba_generator) */
enum dgan_arch { DGAN_ARCH_MNIST = 0, DGAN_ARCH_CELEBA = 1 };

/* arithmetic of the contractions.  State (z, momentum, loss, accumulators) is always fp32. */
enum dgan_precision {
  DGAN_PREC_FP32 = 0, /* fp32 operands, CUDA-core FMA: the reference's arithmetic type */
  DGAN_PREC_FP16 = 1  /* fp16 operands, fp32 accumulate, wgmma tensor cores */
};

typedef struct dgan_desc {
  int32_t abi_version; /* DGAN_ABI_VERSION */
  int32_t arch;        /* dgan_arch */
  int32_t latent_dim;  /* LATENT_DIM (experiments/cfgs/gans/default.yml:4) */
  int32_t net_dim;     /* NET_DIM    (default.yml:7)
                        * Accepted widths (others: DGAN_ERR_UNSUPPORTED, the limit named in dgan_last_error):
                        *   DGAN_PREC_FP32: any latent_dim >= 1; net_dim >= 1 up to what the last layer's shared memory
                        *                   holds: 704 (MNIST), 256 (CelebA).
                        *   DGAN_PREC_FP16: 1 <= latent_dim <= 256, 1 <= net_dim <= 128.
                        * Callers always see the real widths (weights, z, gradients); the handle stores each channel width
                        * padded with exact zeros (fp32: to a multiple of 64; fp16: to 64, 128, 256 or 512), which leaves
                        * every result's bits as the unpadded computation would give them. */
  int32_t use_bn;      /* USE_BN     (default.yml:3); batch-statistics BN, tflib/ops/batchnorm.py:80-93 (both precisions; fp16 path: fp32 pre-activations and statistics, fp16 activations) */
  int32_t precision;   /* dgan_precision */
} dgan_desc;

/* Number of weight tensors dgan_create expects for a descriptor, in the reference's variable
 * creation order (tflib/__init__.py:7-33 names):
 *   Generator.Input.W [latent,4096*] , Generator.Input.b,
 *   [BN1.offset, BN1.scale,]
 *   Generator.2.Filters [5,5,Cout,Cin], Generator.2.Biases, [BN2.offset, BN2.scale,]
 *   Generator.3.Filters, Generator.3.Biases, [BN3.offset, BN3.scale,]
 *   Generator.5.Filters, Generator.5.Biases, (celeba: Generator.6.Filters, Generator.6.Biases)
 * All fp32, device memory, TF layouts (Linear W is (in,out), tflib/ops/linear.py:129-133;
 * Deconv filters are (kh,kw,Cout,Cin), tflib/ops/deconv2d.py:67,104-110). */
int dgan_num_weights(const dgan_desc* desc);

/* Replaces DefenseGANBase.load_generator + the tflib.param registry (models/gan.py:80-87,
 * tflib/__init__.py:7-33): copies the device-resident weights into handle-owned memory and builds the
 * re-laid-out forms (per-tap tiles, transposes, fp16 copies) and the launch schedules on `stream`. */
int dgan_create(dgan_handle* out, const dgan_desc* desc, const float* const* weights_dev,
                int n_weights, void* stream);
int dgan_destroy(dgan_handle h);

/* Bytes of caller-owned scratch needed by dgan_reconstruct / dgan_forward / dgan_loss_grad / dgan_vjp
 * for `batch` images x `rec_rr` restarts.  Also plans and uploads the launch schedules for that many latent rows
 * (cached in the handle; this is where the one-time allocation and synchronisation of a batch size happen). */
size_t dgan_workspace_bytes(dgan_handle h, int batch, int rec_rr);

/* Hyper-parameters of one projection call: the attributes DefenseGANBase.reconstruct reads from the model object at
 * call time (models/gan.py:333-349: rec_rr, rec_iters, rec_lr) plus the optimiser constant of gan.py:389-391. */
typedef struct dgan_rec_params {
  int32_t batch;          /* images in x_dev */
  int32_t rec_rr;         /* R: random restarts per image (REC_RR, mnist.yml:7) */
  int32_t rec_iters;      /* L: gradient steps (REC_ITERS, mnist.yml:5) */
  float rec_lr;           /* constant: the reference's decay is dead code (SURVEY F3) */
  float momentum;         /* 0.7 in the reference (gan.py:389-391) */
  int32_t decay_lr;       /* 0 = reference behaviour; 1 = the evidently intended x0.1 from step ceil(0.8 L) */
  uint64_t seed;          /* Philox key of the z0 stream when z0_dev == NULL */
  uint64_t z_row_offset;  /* index of this call's first latent row in that stream: a caller that shards one batch over
                             several GPUs passes (first image of the shard) * rec_rr so that the draw equals the
                             single-GPU draw row for row; 0 otherwise */
} dgan_rec_params;

/* Replaces one sess.run of the op built by DefenseGANBase.reconstruct (models/gan.py:333-449)
 * preceded by tf.local_variables_initializer() (utils/gan_defense.py:119):
 *   x_dev     [batch, H, W, C] fp32 NHWC, already input-transformed
 *   z0_dev    [batch*rec_rr, latent] fp32 (the reference's z_init_val, gan.py:395-397) or NULL:
 *             z0 ~ N(0, 1/latent) from the Philox stream (seed, z_row_offset) (gan.py:370-377)
 *   rec_dev   [batch, H, W, C] fp32: G(z_{L-1}) of the arg-min restart (gan.py:438-449), 16-byte aligned (it is
 *             stored 16 bytes at a time); a misaligned rec_dev: DGAN_ERR_INVALID_ARG, nothing enqueued
 *   loss_dev  [batch] fp32 min per-image MSE, nullable;  idx_dev [batch] int32 chosen restart, nullable
 * The call enqueues the whole L-step loop on `stream` (8 kernels per L-step with DGAN_PREC_FP16) and never
 * synchronises the host; it does not allocate either once dgan_workspace_bytes has been called for this batch x rec_rr. */
int dgan_reconstruct(dgan_handle h, const dgan_rec_params* params, const float* x_dev,
                     const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev,
                     void* workspace, size_t workspace_bytes, void* stream);

/* Projection onto the generator's range with a per-pixel weighted loss (an extension: the reference has no weighting),
 * for partially observed images - occluded or missing pixels, pixels flagged as corrupted, per-channel weighting:
 *   w_dev [batch, H, W, C] fp32, finite, 0 <= w <= 1 (not checked here); the rec_rr restarts of image i share its map.
 *   Row n's loss is (1/HWC) sum_p w[n / rec_rr, p] (G(z_n)_p - x_p)^2: the normaliser stays H*W*C, so rec_lr keeps its
 *   meaning and weights covering a fraction f of the pixels give gradients about f times smaller.  Evaluation order per
 *   pixel: d = y - x, e = w * d, loss += e * d, d(pre) = e * act'(y); with w == 1 every output is bit-identical to
 *   dgan_reconstruct's.  loss_dev and the arg-min select use the weighted loss; an image whose weights are all 0 keeps
 *   z0 (its gradient is 0) and restart 0 is chosen (lowest index on ties).  Weights above 1 could saturate the fp16
 *   path's fixed d(pre) scale, which is sized for |y - x| <= 1.
 * Workspace: dgan_workspace_bytes_weighted.  The weights are copied into it next to the images: one stream operation
 * more than dgan_reconstruct, no host synchronisation, no allocation once the size has been planned. */
int dgan_reconstruct_weighted(dgan_handle h, const dgan_rec_params* params, const float* x_dev, const float* w_dev,
                              const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev,
                              void* workspace, size_t workspace_bytes, void* stream);

/* Bytes of scratch for dgan_reconstruct_weighted / dgan_loss_grad_weighted: dgan_workspace_bytes plus one weight buffer
 * of batch images.  Also plans the weighted last-layer forward for batch x rec_rr latent rows (a handle that never
 * weights plans nothing for it). */
size_t dgan_workspace_bytes_weighted(dgan_handle h, int batch, int rec_rr);

/* Projection onto the generator's range from linear measurements (an extension: the reference has none; it is the loop of
 * compressed sensing with generative models), for observations y = A x of an image x that is not held itself - a
 * low-resolution copy, a blurred copy, a compressed-sensing sketch:
 *   a_dev [m, H*W*C] fp32 row-major, columns in NHWC pixel order, 1 <= m <= H*W*C; one operator for every image and restart.
 *   y_dev [batch, m] fp32; the rec_rr restarts of image i share y[i].
 *   Row n's loss is (1/m) sum_j ((A G(z_n))_j - y[n / rec_rr]_j)^2: the normaliser is m, so A = I (m = H*W*C) is
 *   dgan_reconstruct's loss and rec_lr keeps its meaning.  Its gradient enters the generator's backward as the cotangent
 *   dy_n = (2/m) A^T r_n with r_n = A G(z_n) - y[n / rec_rr], as in dgan_vjp (DGAN_PREC_FP16: a power-of-two scale per
 *   row, one for the call with use_bn, divided out of the gradient).  The z0 stream, momentum, decay_lr, the pre-update
 *   forward of iteration L-1 and the arg-min select (lowest index on ties) are dgan_reconstruct's; with the same seed the
 *   call starts from the same z0.  rec_dev [batch, H, W, C] (16-byte aligned), loss_dev [batch] (the minimum measured
 *   loss, nullable) and idx_dev [batch] (nullable) as in dgan_reconstruct.
 * Both measurement products run on the tensor cores in TF32 with DGAN_PREC_FP16 (fp32 accumulate) and in fp32 on the
 * CUDA cores with DGAN_PREC_FP32.  m <= 0, m > H*W*C or a NULL operator or measurement pointer: DGAN_ERR_INVALID_ARG.
 * Workspace: dgan_workspace_bytes_measured.  A, its transpose and y are copied into it by three kernels (two stream
 * operations more than dgan_reconstruct's image copy); the captured loop reads only the workspace.  No host
 * synchronisation, no allocation once the size has been planned.  Per L-step it runs the kernels of dgan_reconstruct's
 * plus the measurement product, the adjoint product and the cotangent entry (3 kernels with DGAN_PREC_FP16, 1 with fp32)
 * and, on DGAN_PREC_FP16, a separate momentum update (dgan_reconstruct's runs in the Linear backward); the last L-step
 * adds the measurement product.  So dgan_last_launch_count is dgan_reconstruct's + 3 + 6 (L - 1) + 1 with
 * DGAN_PREC_FP16 and + 3 + 3 (L - 1) + 1 with DGAN_PREC_FP32, and dgan_last_enqueue_count is dgan_reconstruct's + 2. */
int dgan_reconstruct_measured(dgan_handle h, const dgan_rec_params* params, const float* a_dev, int m, const float* y_dev,
                              const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev,
                              void* workspace, size_t workspace_bytes, void* stream);

/* Bytes of scratch for dgan_reconstruct_measured / dgan_loss_grad_measured with m measurements: dgan_workspace_bytes plus
 * the copies of A, A^T and y (m padded to a multiple of 64 with zeros), the residuals, the adjoint product and the measured
 * loss.  0 for m <= 0 or m > H*W*C.  A handle that never measures carves nothing for it. */
size_t dgan_workspace_bytes_measured(dgan_handle h, int batch, int rec_rr, int m);

/* One evaluation of dgan_reconstruct_measured's loop body without the update, for known-answer tests: g_dev
 * [batch*rec_rr, H*W*C] = G(z) (nullable), loss_dev [batch*rec_rr] the measured loss, grad_dev [batch*rec_rr, latent] =
 * d(sum loss)/dz.  Workspace: dgan_workspace_bytes_measured(h, batch, rec_rr, m). */
int dgan_loss_grad_measured(dgan_handle h, const float* a_dev, int m, const float* y_dev, int batch, int rec_rr,
                            const float* z_dev, float* g_dev, float* loss_dev, float* grad_dev, void* workspace,
                            size_t workspace_bytes, void* stream);

/* dgan_reconstruct_measured with a sparse operator: A [m, H*W*C] in CSR, row_ptr [m + 1], col_idx [nnz] and val [nnz]
 * (int32, int32, fp32, on the device), the columns of each row strictly ascending.  The semantics are exactly those of
 * dgan_reconstruct_measured for the dense matrix the CSR represents; the two measurement products cost in proportion to
 * the non-zeros instead of m * H*W*C.  They run in fp32 on the CUDA cores on both precisions: with DGAN_PREC_FP32 every
 * output is bit-identical to dgan_reconstruct_measured's on that dense matrix; with DGAN_PREC_FP16 A is applied in fp32,
 * so the result differs from the dense call's (TF32) by the TF32 rounding of A and of the operands.
 * m <= 0, m > H*W*C, nnz < 0, nnz > m * H*W*C, a NULL row_ptr or y_dev, a NULL col_idx or val with nnz > 0, or a
 * rec_dev that is not 16-byte aligned: DGAN_ERR_INVALID_ARG before anything is enqueued.  The CSR's contents are
 * validated on the device while it is staged (row_ptr from 0 to nnz, never decreasing; columns in [0, H*W*C) and
 * strictly ascending within each row); reading only row_ptr[0..m] and col_idx / val[0..nnz).  A CSR that breaks one of
 * them is never used: the call returns DGAN_OK with NaN losses and reconstructions.
 * Workspace: dgan_workspace_bytes_measured_csr.  The operator is validated and copied into it with its transpose, and y
 * with it, by five kernels (four stream operations more than dgan_reconstruct's image copy); the captured loop reads only
 * the workspace.  No host synchronisation, no allocation once the size has been planned.  Per L-step it runs the kernels
 * of dgan_reconstruct_measured (one kernel per product).  So dgan_last_launch_count is dgan_reconstruct's
 * + 5 + 6 (L - 1) + 1 with DGAN_PREC_FP16 and + 5 + 3 (L - 1) + 1 with DGAN_PREC_FP32, and dgan_last_enqueue_count is
 * dgan_reconstruct's + 4. */
int dgan_reconstruct_measured_csr(dgan_handle h, const dgan_rec_params* params, const int32_t* row_ptr,
                                  const int32_t* col_idx, const float* val, int m, int nnz, const float* y_dev,
                                  const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev,
                                  void* workspace, size_t workspace_bytes, void* stream);

/* Bytes of scratch for dgan_reconstruct_measured_csr / dgan_loss_grad_measured_csr with m measurements and nnz
 * non-zeros: dgan_workspace_bytes plus the copies of the CSR and of its transpose, y (m padded to a multiple of 64), the
 * residuals, the adjoint product and the measured loss - no dense copy of A.  0 for m <= 0, m > H*W*C, nnz < 0 or
 * nnz > m * H*W*C.  A handle that never uses a CSR operator carves nothing for it. */
size_t dgan_workspace_bytes_measured_csr(dgan_handle h, int batch, int rec_rr, int m, int nnz);

/* dgan_loss_grad_measured with the CSR operator of dgan_reconstruct_measured_csr.
 * Workspace: dgan_workspace_bytes_measured_csr(h, batch, rec_rr, m, nnz). */
int dgan_loss_grad_measured_csr(dgan_handle h, const int32_t* row_ptr, const int32_t* col_idx, const float* val, int m,
                                int nnz, const float* y_dev, int batch, int rec_rr, const float* z_dev, float* g_dev,
                                float* loss_dev, float* grad_dev, void* workspace, size_t workspace_bytes,
                                void* stream);

/* One prune point of a pruned projection, in host memory. */
typedef struct dgan_prune_point {
  int32_t iter; /* the iteration from which on the image's survivors run alone */
  int32_t keep; /* restarts each image keeps */
} dgan_prune_point;

/* Bytes of scratch for dgan_reconstruct_pruned with this schedule (weighted != 0: with per-pixel weights): one region
 * per stage, one after the other, each the workspace that dgan_workspace_bytes or dgan_workspace_bytes_weighted carves
 * for that stage's rows - batch * rec_rr, then batch * keep_k - plus three int32 maps of its rows.  Also plans every
 * stage's row count.  0 for a handle with use_bn and for a schedule that breaks the rules of dgan_reconstruct_pruned,
 * except iter <= rec_iters - 1, as L is not known here. */
size_t dgan_workspace_bytes_pruned(dgan_handle h, int batch, int rec_rr, const dgan_prune_point* sched, int n_points,
                                   int weighted);

/* dgan_reconstruct with w_dev NULL, dgan_reconstruct_weighted otherwise (w_dev as there), that drops each image's worst restarts
 * partway through the loop (an extension: the reference runs every restart to the end).  sched [n_points] in host
 * memory: 1 <= iter_1 < iter_2 < ... < iter_n <= rec_iters - 1 and rec_rr >= keep_1 >= ... >= keep_n >= 1.
 *   At prune point k, after iteration iter_k - 1 has run with its update: each image's surviving restarts are ranked by
 *   their loss at iteration iter_k - 1 (lower first; ties by the lower original restart index; NaN after every number)
 *   and the first keep_k go on, with their z and momentum unchanged, image-major and in ascending original restart
 *   index.  Iterations iter_k .. run on batch * keep_k rows; the learning rate follows the global iteration (decay_lr
 *   from ceil(0.8 rec_iters)).  The arg-min select of dgan_reconstruct then picks among the last survivors: rec_dev and
 *   loss_dev are that survivor's G(z_{L-1}) and loss, idx_dev its original restart index in [0, rec_rr).
 * Rows are independent without BatchNorm, so each survivor follows exactly its unpruned trajectory: keep_k = rec_rr at
 * every point gives dgan_reconstruct's bits.  use_bn couples the rows: DGAN_ERR_UNSUPPORTED.  A schedule that breaks the
 * rules, NULL arguments or a misaligned rec_dev: DGAN_ERR_INVALID_ARG; a workspace smaller than
 * dgan_workspace_bytes_pruned: DGAN_ERR_WORKSPACE; nothing is enqueued in either case.
 * Before the captured loop the host enqueues the z0 initialiser (into region 0), the zeroing of each later region's
 * momentum tickets or d(pre) padding rows (memsets, not counted, as in dgan_reconstruct) and one image copy per region
 * (with w_dev, one weight copy per region too).  The loop - every stage's L-steps and, at each prune point, the loss sum,
 * prune_select_kernel and prune_gather_kernel - is one CUDA graph per (workspace, hyper-parameters, schedule).  After it:
 * loss sum, arg-min select and the mapping of the chosen survivor to its original index.  So, with P = n_points,
 * dgan_last_launch_count is that of dgan_reconstruct or dgan_reconstruct_weighted with the same rec_iters + 3 P + 1, and
 * dgan_last_enqueue_count is theirs + P (image copies; 2 P with w_dev) + 1. */
int dgan_reconstruct_pruned(dgan_handle h, const dgan_rec_params* params, const dgan_prune_point* sched, int n_points,
                            const float* x_dev, const float* w_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                            int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream);

/* Bytes of scratch for dgan_reconstruct_measured_pruned with nnz = -1, or dgan_reconstruct_measured_csr_pruned with
 * nnz >= 0 non-zeros, for m measurements and this schedule: one operator block - the copies of A and A^T, or of the CSR and its
 * transpose, and y for batch images - shared by every stage, then one region per stage, each the workspace that
 * dgan_workspace_bytes carves for that stage's rows plus the residuals, the adjoint product, the measured loss and three
 * int32 maps of its rows.  Also plans every stage's row count.  0 for a handle with use_bn, for a schedule that breaks the
 * rules of dgan_reconstruct_pruned (except iter <= rec_iters - 1, as L is not known here), for m <= 0 or m > H*W*C and
 * for nnz < -1 or nnz > m * H*W*C. */
size_t dgan_workspace_bytes_measured_pruned(dgan_handle h, int batch, int rec_rr, int m, int nnz,
                                            const dgan_prune_point* sched, int n_points);

/* dgan_reconstruct_measured with the restart pruning of dgan_reconstruct_pruned - a_dev, m and y_dev as in the first,
 * sched and n_points as in the second: at prune point k each image's survivors are ranked by their measured loss (1/m) ||A G(z) - y||^2
 * at iteration iter_k - 1, with the same order, ties and NaN rule, and the arg-min select picks among the last
 * survivors; idx_dev is the original restart index.  Without BatchNorm each survivor follows exactly its unpruned
 * trajectory: keep_k = rec_rr at every point gives dgan_reconstruct_measured's bits, and any schedule gives the result
 * composed from rec_rr = 1 calls.  use_bn: DGAN_ERR_UNSUPPORTED.  The argument checks of dgan_reconstruct_measured and
 * dgan_reconstruct_pruned apply, before anything is enqueued; a workspace smaller than
 * dgan_workspace_bytes_measured_pruned: DGAN_ERR_WORKSPACE.
 * Before the captured loop the host enqueues the z0 initialiser (into region 0), the memsets of each later region and
 * the three kernels that stage A, A^T and y into the operator block, once.  The loop - every stage's measured L-steps on
 * its rows and, at each prune point, the measured loss sum, prune_select_kernel and prune_gather_kernel - is one CUDA
 * graph; after it: measured loss sum, arg-min select and the mapping to the original index.  So, with P = n_points,
 * dgan_last_launch_count is dgan_reconstruct_measured's with the same rec_iters + 3 P + 1, and dgan_last_enqueue_count
 * is dgan_reconstruct_measured's + 1. */
int dgan_reconstruct_measured_pruned(dgan_handle h, const dgan_rec_params* params, const dgan_prune_point* sched,
                                     int n_points, const float* a_dev, int m, const float* y_dev, const float* z0_dev,
                                     float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes,
                                     void* stream);

/* dgan_reconstruct_measured_pruned with the CSR operator of dgan_reconstruct_measured_csr - row_ptr, col_idx, val, m,
 * nnz and their checks as there: it is validated and staged once, by five kernels, into the operator block; a malformed
 * CSR is staged as the empty operator with NaN measurements, so every loss is NaN and each image keeps survivors 0 ..
 * keep - 1 by the NaN rule.  dgan_last_launch_count is dgan_reconstruct_measured_csr's + 3 P + 1, and
 * dgan_last_enqueue_count is dgan_reconstruct_measured_csr's + 1. */
int dgan_reconstruct_measured_csr_pruned(dgan_handle h, const dgan_rec_params* params, const dgan_prune_point* sched,
                                         int n_points, const int32_t* row_ptr, const int32_t* col_idx, const float* val,
                                         int m, int nnz, const float* y_dev, const float* z0_dev, float* rec_dev,
                                         float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream);

/* Hyper-parameters of the Adam update (an extension: the reference optimises z with tf.train.MomentumOptimizer only). */
typedef struct dgan_adam_params {
  float beta1; /* [0, 1): decay of the first moment m */
  float beta2; /* [0, 1): decay of the second moment s */
  float eps;   /* finite, > 0 */
} dgan_adam_params;

/* Bytes of scratch for dgan_reconstruct_adam, with per-pixel weights when weighted != 0.  sched NULL and n_points 0: the
 * workspace of dgan_workspace_bytes or dgan_workspace_bytes_weighted plus Adam's second moment s [n_pad][latent] fp32;
 * a schedule: that of dgan_workspace_bytes_pruned with s in every region.  0 where those sizers return 0. */
size_t dgan_workspace_bytes_adam(dgan_handle h, int batch, int rec_rr, int weighted, const dgan_prune_point* sched,
                                 int n_points);

/* Bytes of scratch for dgan_reconstruct_measured_adam with nnz = -1, or dgan_reconstruct_measured_csr_adam with nnz >= 0
 * non-zeros.  Unpruned (sched NULL, n_points 0), the workspace of dgan_workspace_bytes_measured[_csr] plus s; a schedule:
 * that of dgan_workspace_bytes_measured_pruned with s in every region.  0 where those sizers return 0. */
size_t dgan_workspace_bytes_measured_adam(dgan_handle h, int batch, int rec_rr, int m, int nnz, const dgan_prune_point* sched,
                                          int n_points);

/* dgan_reconstruct (w_dev NULL) or dgan_reconstruct_weighted, with sched NULL and n_points 0, or dgan_reconstruct_pruned
 * with a schedule, that updates z with Adam instead of momentum (an extension: GAN inversion and compressed sensing with
 * generative models commonly use Adam).  For latent row n at iteration t, with k = t + 1 and g the gradient the momentum
 * update uses (the split-K parts summed in order, times the loss's multiplier):
 *   m = beta1 m + (1 - beta1) g;  s = beta2 s + (1 - beta2) g^2;  z = z - c1 m / (sqrt(s) c2 + eps)
 *   c1 = lr_t / (1 - beta1^k), c2 = 1 / sqrt(1 - beta2^k), computed on the host in double and rounded to fp32;
 * lr_t is rec_lr or its decay_lr schedule, as in dgan_reconstruct.  rec_lr is therefore a step in z units: the
 * momentum path's values do not carry over.  params->momentum is ignored.  m and s start at 0 on every call; iteration
 * L-1 runs no update.  The fp32 evaluation order is in kernels_adam.cuh (adam_kernel).  A coordinate whose gradient is
 * always 0 - padded latent columns, an image whose pixel weights are all 0 - keeps its z0.  Loss, select, ties, the NaN rule and the
 * prune ranking are those of the momentum entries; without BatchNorm each pruned survivor follows exactly its unpruned
 * trajectory.  adam NULL, beta1 or beta2 outside [0, 1) or eps not finite and > 0: DGAN_ERR_INVALID_ARG, nothing
 * enqueued; the checks of the momentum counterpart apply too (use_bn with a schedule: DGAN_ERR_UNSUPPORTED).
 * Workspace: dgan_workspace_bytes_adam; s is zeroed by a memset with z0, and a prune point gathers it with z and m.
 * Counts: dgan_last_enqueue_count is the momentum counterpart's; dgan_last_launch_count is the momentum counterpart's
 * with DGAN_PREC_FP32, and L - 1 more with DGAN_PREC_FP16 (the momentum update runs in the Linear backward's tail there,
 * the Adam update in a kernel of its own). */
int dgan_reconstruct_adam(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                          const dgan_prune_point* sched, int n_points, const float* x_dev, const float* w_dev,
                          const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes,
                          void* stream);

/* dgan_reconstruct_measured, or dgan_reconstruct_measured_pruned with a schedule, with the Adam update of
 * dgan_reconstruct_adam; g is the measured loop's gradient with the cotangent's row scales divided out.  Workspace:
 * dgan_workspace_bytes_measured_adam with nnz = -1.  dgan_last_launch_count and dgan_last_enqueue_count equal the momentum
 * counterpart's on both precisions (adam_kernel replaces the measured loop's momentum kernel). */
int dgan_reconstruct_measured_adam(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                   const dgan_prune_point* sched, int n_points, const float* a_dev, int m, const float* y_dev,
                                   const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws,
                                   size_t ws_bytes, void* stream);

/* The same with the CSR operator of dgan_reconstruct_measured_csr (dgan_reconstruct_measured_csr_pruned with a
 * schedule).  Workspace: dgan_workspace_bytes_measured_adam with this nnz; counts as the momentum counterpart's. */
int dgan_reconstruct_measured_csr_adam(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                       const dgan_prune_point* sched, int n_points, const int32_t* row_ptr,
                                       const int32_t* col_idx, const float* val, int m, int nnz, const float* y_dev,
                                       const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws,
                                       size_t ws_bytes, void* stream);

/* The projection with a Huber data term instead of the squared error (an extension: the reference's loss is the squared
 * error only).  A few badly wrong pixels or measurements - impulse noise, dead pixels, occluders whose place is not known,
 * corrupted measurements - then pull G(z) much less far from the point that fits the rest.
 * For a residual d in fp32 (d = y - x per pixel on the image loss, r = (A G(z))_j - y_j per measurement on the measured
 * loss) and huber_delta = delta > 0 (+inf allowed):
 *   c = |d| > delta ? copysign(delta, d) : d      (psi_delta(d); NaN passes through)
 *   e = w c (weighted image loss; e = c without weights)
 *   term = e (2 d - c)                             (= w rho_delta(d): d^2 for |d| <= delta, 2 delta |d| - delta^2 beyond)
 *   d(pre) = e act'(y) on the image loss (times the fp16 path's fixed gradient scale, as in dgan_reconstruct);
 *   the measured loss stores c as the residual, so the adjoint product gives (2/m) A^T psi(r).
 * The row loss is (1/HWC) sum_p w_p rho_delta(d_p) on the image loss and (1/m) sum_j rho_delta(r_j) on the measured loss:
 * the normalisers of the squared error, so rho = 2 torch.nn.functional.huber_loss(..., delta, reduction='none').  When no
 * residual exceeds delta, c == d and 2 d - c == d exactly, so every stored value, and the whole call, has the bits of
 * its squared-error counterpart: always at delta = +inf, and on the image loss at any delta >= 2 when the images lie in
 * the generator's output range (|y - x| < 2).  |c| <= |d|, so the fp16 path's fixed d(pre) scale saturates nowhere it
 * did not before.  The Huber loss is what loss_dev, the arg-min select, ties, the NaN rule and the prune ranking use;
 * z0, the momentum or Adam update, decay_lr, the pre-update forward of iteration L-1 and BatchNorm are unchanged.
 * With momentum the gradient of a clipped residual shrinks with delta, so rec_lr has to grow as delta falls; Adam is
 * invariant to the gradient's scale and needs no re-tuning.
 * Each entry runs its counterpart's code path with delta as one argument more: adam NULL selects the momentum update,
 * otherwise the Adam update of dgan_reconstruct_adam; sched NULL with n_points 0 runs unpruned, any other schedule follows
 * the rules of dgan_reconstruct_pruned (BatchNorm runs unpruned only; with a schedule: DGAN_ERR_UNSUPPORTED).  So
 * dgan_reconstruct_huber's counterpart is dgan_reconstruct (w_dev NULL), dgan_reconstruct_weighted, dgan_reconstruct_pruned
 * or dgan_reconstruct_adam.  Workspace: the counterpart's sizer, unchanged (dgan_workspace_bytes[_weighted | _pruned], or
 * dgan_workspace_bytes_adam when adam is not NULL).  dgan_last_launch_count and dgan_last_enqueue_count equal the
 * counterpart's; the graph cache keys on delta too.  A delta that is NaN, 0 or negative: DGAN_ERR_INVALID_ARG, after
 * the counterpart's other checks and before anything is enqueued. */
int dgan_reconstruct_huber(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam, float huber_delta,
                           const dgan_prune_point* sched, int n_points, const float* x_dev, const float* w_dev,
                           const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes,
                           void* stream);

/* dgan_reconstruct_measured (dgan_reconstruct_measured_pruned with a schedule, dgan_reconstruct_measured_adam with adam)
 * with the Huber loss of dgan_reconstruct_huber on the measurement residuals.  Workspace: the counterpart's
 * (dgan_workspace_bytes_measured[_pruned], or dgan_workspace_bytes_measured_adam with nnz = -1). */
int dgan_reconstruct_measured_huber(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                    float huber_delta, const dgan_prune_point* sched, int n_points, const float* a_dev, int m,
                                    const float* y_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                                    int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream);

/* The same with the CSR operator of dgan_reconstruct_measured_csr.  With DGAN_PREC_FP32 every output is bit-identical to
 * dgan_reconstruct_measured_huber's on the dense matrix the CSR represents.  Workspace: the counterpart's
 * (dgan_workspace_bytes_measured_csr, dgan_workspace_bytes_measured_pruned or dgan_workspace_bytes_measured_adam with this
 * nnz). */
int dgan_reconstruct_measured_csr_huber(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                        float huber_delta, const dgan_prune_point* sched, int n_points,
                                        const int32_t* row_ptr, const int32_t* col_idx, const float* val, int m, int nnz,
                                        const float* y_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                                        int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream);

/* The z_hat initialiser alone (models/gan.py:370-377): z_dev [n_rows, latent] ~ N(0, 1/latent), rows
 * [z_row_offset, z_row_offset + n_rows) of the Philox stream keyed by `seed` - exactly what dgan_reconstruct
 * draws when z0_dev == NULL. */
int dgan_sample_z0(dgan_handle h, uint64_t seed, uint64_t z_row_offset, int n_rows, float* z_dev,
                   void* stream);

/* generator_fn(z) (models/gan.py:657-665,726-735): y_dev [n_rows, H*W*C] fp32. */
int dgan_forward(dgan_handle h, const float* z_dev, int n_rows, float* y_dev, void* workspace,
                 size_t workspace_bytes, void* stream);

/* One evaluation of the loop body (models/gan.py:409-417) without the update, for known-answer
 * tests: y [batch*rec_rr, HWC], loss [batch*rec_rr], grad = d(sum loss)/dz [batch*rec_rr, latent]. */
int dgan_loss_grad(dgan_handle h, const float* x_dev, int batch, int rec_rr, const float* z_dev,
                   float* y_dev, float* loss_dev, float* grad_dev, void* workspace,
                   size_t workspace_bytes, void* stream);

/* dgan_loss_grad with the weighted loss of dgan_reconstruct_weighted (w_dev [batch, H, W, C], read in place).
 * Workspace: dgan_workspace_bytes_weighted(h, batch, rec_rr). */
int dgan_loss_grad_weighted(dgan_handle h, const float* x_dev, const float* w_dev, int batch, int rec_rr,
                            const float* z_dev, float* y_dev, float* loss_dev, float* grad_dev, void* workspace,
                            size_t workspace_bytes, void* stream);

/* dgan_loss_grad (w_dev NULL) or dgan_loss_grad_weighted with the Huber loss of dgan_reconstruct_huber at huber_delta.
 * Workspace: the counterpart's.  A bad delta: DGAN_ERR_INVALID_ARG after the counterpart's other checks. */
int dgan_loss_grad_huber(dgan_handle h, float huber_delta, const float* x_dev, const float* w_dev, int batch, int rec_rr,
                         const float* z_dev, float* y_dev, float* loss_dev, float* grad_dev, void* workspace,
                         size_t workspace_bytes, void* stream);

/* dgan_loss_grad_measured and dgan_loss_grad_measured_csr with the Huber loss of dgan_reconstruct_huber at huber_delta.
 * Workspace: the counterpart's.  A bad delta: DGAN_ERR_INVALID_ARG after the counterpart's other checks. */
int dgan_loss_grad_measured_huber(dgan_handle h, float huber_delta, const float* a_dev, int m, const float* y_dev, int batch,
                                  int rec_rr, const float* z_dev, float* g_dev, float* loss_dev, float* grad_dev,
                                  void* workspace, size_t workspace_bytes, void* stream);
int dgan_loss_grad_measured_csr_huber(dgan_handle h, float huber_delta, const int32_t* row_ptr, const int32_t* col_idx,
                                      const float* val, int m, int nnz, const float* y_dev, int batch, int rec_rr,
                                      const float* z_dev, float* g_dev, float* loss_dev, float* grad_dev, void* workspace,
                                      size_t workspace_bytes, void* stream);

/* A convolution operator: for an image x [H, W, C] (NHWC) and a kernel k [kh, kw] (fp32, one per image, the same for
 * every channel), stride s and zero padding (pad_h, pad_w):
 *   Ho = (H + 2 pad_h - kh) / s + 1,  Wo = (W + 2 pad_w - kw) / s + 1,  m = Ho * Wo * C,
 *   (A x)[(u * Wo + v) * C + c] = sum over a < kh, b < kw with 0 <= i < H, 0 <= j < W of k[a][b] x[i][j][c],
 *                                 i = s u + a - pad_h, j = s v + b - pad_w
 * (a cross-correlation: the kernel is not flipped; torch's conv2d with groups = C and the kernel repeated per channel).
 * A blur is (5, 5, 2, 2, 1), a 2x2 block average (2, 2, 0, 0, 2) with 0.25 everywhere.  Accepted geometry:
 * 1 <= kh <= min(H, 32), 1 <= kw <= min(W, 32), 0 <= 2 pad_h <= kh - 1, 0 <= 2 pad_w <= kw - 1, 1 <= stride <= 16. */
typedef struct dgan_conv_op {
  int32_t kh, kw, pad_h, pad_w, stride;
} dgan_conv_op;

/* m = Ho * Wo * C for this handle's image, or 0 for a geometry outside the accepted range (or a NULL handle or op). */
int dgan_conv_op_m(dgan_handle h, const dgan_conv_op* op);

/* Bytes of scratch for dgan_reconstruct_measured_conv / dgan_loss_grad_measured_conv: unpruned (sched NULL, n_points 0)
 * the workspace of dgan_workspace_bytes_measured without the copies of A and A^T, plus the kernels [batch][kh][kw]; a
 * schedule: that of dgan_workspace_bytes_measured_pruned with this operator block.  adam != 0 adds Adam's s, as
 * dgan_workspace_bytes_measured_adam does.  0 for a geometry outside the accepted range and where those sizers return 0. */
size_t dgan_workspace_bytes_measured_conv(dgan_handle h, int batch, int rec_rr, const dgan_conv_op* op,
                                          const dgan_prune_point* sched, int n_points, int adam);

/* dgan_reconstruct_measured with the convolution operator op: image i's operator A_i uses its own kernel
 * k_dev [batch][kh][kw] (fp32, on the device; a shared kernel is passed as batch copies), y_dev [batch][m].  The loss,
 * its normaliser m, z0, decay_lr, the pre-update forward of iteration L-1 and the select (ties, NaN rule) are those of
 * dgan_reconstruct_measured for A_i; the restarts of image i share k_i and y_i.  adam NULL: the momentum update, else
 * the Adam update of dgan_reconstruct_adam; huber_delta NULL: the squared error, else the Huber loss of
 * dgan_reconstruct_huber at *huber_delta (checked as there); sched NULL with n_points 0: unpruned, else the restart
 * pruning of dgan_reconstruct_measured_pruned (use_bn with a schedule: DGAN_ERR_UNSUPPORTED).
 * Both products run in fp32 on the CUDA cores on both precisions, as a stencil: each reads G or r once and writes r or
 * dy once.  Their evaluation order is the CSR products' on the matrix the stencil represents, so every output is
 * bit-identical to dgan_reconstruct_measured_csr's (and its _adam, _huber and _pruned variants') on that matrix:
 *   measurement output j: one fmaf chain from +0 over the in-bounds taps in ascending (a, b) (ascending input column),
 *     then the residual and loss parts of the CSR product (per quad of columns, then a butterfly over each 64-column
 *     tile; padded columns give r = 0);
 *   adjoint output p = (i, j, c): one chain from +0 over the output pixels (u, v) whose window covers (i, j), in
 *     ascending order (ascending row of A), then the multiply by 2/m.
 * A tap whose value is 0 adds a term the CSR does not hold; the chains start at +0 and G and r are finite, so no bit
 * changes.  The kernels and measurements are not checked for finiteness here.
 * A geometry outside the accepted range, a NULL op, k_dev or y_dev, or a rec_dev that is not 16-byte aligned:
 * DGAN_ERR_INVALID_ARG naming the bad value; a workspace smaller than dgan_workspace_bytes_measured_conv:
 * DGAN_ERR_WORKSPACE; nothing is enqueued in any of these cases.
 * Workspace: dgan_workspace_bytes_measured_conv.  The kernels and y are copied into it by one kernel (no stream
 * operation more than dgan_reconstruct's image copy), outside the captured loop; the graph cache keys on the geometry,
 * not on the kernel values, so new kernels with the same geometry replay the graph.  No host synchronisation, no
 * allocation once the size has been planned.  Per L-step it runs the kernels of dgan_reconstruct_measured (one kernel
 * per product).  So dgan_last_launch_count is dgan_reconstruct's + 1 + 6 (L - 1) + 1 with DGAN_PREC_FP16 and
 * + 1 + 3 (L - 1) + 1 with DGAN_PREC_FP32 (dgan_reconstruct_measured_csr's - 4), plus 3 P + 1 with P prune points and
 * L - 1 nowhere for Adam, as for the other operator kinds; dgan_last_enqueue_count is dgan_reconstruct's, + 1 with a
 * schedule. */
int dgan_reconstruct_measured_conv(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                   const float* huber_delta, const dgan_prune_point* sched, int n_points,
                                   const dgan_conv_op* op, const float* k_dev, const float* y_dev, const float* z0_dev,
                                   float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes,
                                   void* stream);

/* dgan_loss_grad_measured with the convolution operator of dgan_reconstruct_measured_conv (huber_delta NULL: the squared
 * error, else the Huber loss at *huber_delta).  Workspace: dgan_workspace_bytes_measured_conv(h, batch, rec_rr, op,
 * NULL, 0, 0). */
int dgan_loss_grad_measured_conv(dgan_handle h, const float* huber_delta, const dgan_conv_op* op, const float* k_dev,
                                 const float* y_dev, int batch, int rec_rr, const float* z_dev, float* g_dev,
                                 float* loss_dev, float* grad_dev, void* ws, size_t ws_bytes, void* stream);

/* The projection with a Gaussian prior on the latent vector (an extension: the reference has none; compressed sensing with
 * generative models adds it to keep z where the generator was trained).  For lambda = z_prior (fp32, finite, >= 0, and
 * 2 lambda finite) each restart minimises
 *   J(z) = D(z) + lambda ||z||^2
 * where D is the counterpart's data term exactly as it computes it (squared error or Huber, weighted or not, image or
 * measured), with its normaliser 1/(H*W*C) or 1/m: lambda is relative to the normalised data term, so the lambda of a
 * formulation on the unnormalised ||A G(z) - y||^2 does not carry over (divide it by m).
 *   - ||z||^2 runs over the latent_dim real columns in fp32 as one fmaf chain from +0 in ascending column order;
 *     p = lambda * sum, J = D + p as one fp32 add.
 *   - The update takes g' = fmaf(2 lambda, z, g) instead of the counterpart's gradient g (after its multiplier, and with
 *     DGAN_PREC_FP16's measured row scales divided out; split-K parts summed in the same order), on the pre-update z,
 *     with 2 lambda rounded on the host.  The momentum or Adam arithmetic that follows is the counterpart's.  Padded
 *     latent columns stay 0.
 *   - J is evaluated on the z its D is computed on: the z of iteration L-1 for loss_dev and the arg-min select, and at a
 *     prune point the z of iteration iter_k - 1, before that iteration's update.  J is what loss_dev, the select (ties,
 *     NaN rule) and the prune ranking use; rec_dev is G(z) of the chosen restart.
 *   - lambda = 0 gives the counterpart's rec_dev, loss_dev and idx_dev bit for bit.
 *   - use_bn is allowed unpruned (the prior is per row); with a schedule it is refused as by the counterpart.
 * Each entry runs its counterpart's code path with the counterpart's option arguments: adam NULL for momentum, else the
 * Adam update of dgan_reconstruct_adam; huber_delta NULL for the squared error, else the Huber loss of
 * dgan_reconstruct_huber at *huber_delta; sched NULL with n_points 0 unpruned, else the restart pruning of the pruned
 * entries.  Workspace: the counterpart's (dgan_workspace_bytes[_weighted / _pruned / _adam] and their measured forms);
 * the prior needs no buffer of its own.  A lambda that is NaN, infinite or negative, or whose double 2 lambda overflows fp32:
 * DGAN_ERR_INVALID_ARG naming the value, checked after the counterpart's checks and before anything is enqueued.
 * Counts: dgan_last_enqueue_count is the counterpart's.  dgan_last_launch_count is the counterpart's + 1 + P (the prior
 * term, at iteration L-1 and at each of P prune points), + L - 1 on the DGAN_PREC_FP16 image loss with momentum, whose
 * update then runs as a kernel of its own after the Linear backward, as Adam's does.  The graph cache keys on lambda.
 *
 * dgan_reconstruct_prior: the image loss; w_dev NULL for dgan_reconstruct's loss, else dgan_reconstruct_weighted's. */
int dgan_reconstruct_prior(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                           const float* huber_delta, float z_prior, const dgan_prune_point* sched, int n_points,
                           const float* x_dev, const float* w_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                           int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream);

/* dgan_reconstruct_measured (a dense operator) with the latent prior of dgan_reconstruct_prior. */
int dgan_reconstruct_measured_prior(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                    const float* huber_delta, float z_prior, const dgan_prune_point* sched, int n_points,
                                    const float* a_dev, int m, const float* y_dev, const float* z0_dev, float* rec_dev,
                                    float* loss_dev, int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream);

/* dgan_reconstruct_measured_csr with the latent prior of dgan_reconstruct_prior. */
int dgan_reconstruct_measured_csr_prior(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                        const float* huber_delta, float z_prior, const dgan_prune_point* sched, int n_points,
                                        const int32_t* row_ptr, const int32_t* col_idx, const float* val, int m, int nnz,
                                        const float* y_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                                        int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream);

/* dgan_reconstruct_measured_conv with the latent prior of dgan_reconstruct_prior. */
int dgan_reconstruct_measured_conv_prior(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                         const float* huber_delta, float z_prior, const dgan_prune_point* sched,
                                         int n_points, const dgan_conv_op* op, const float* k_dev, const float* y_dev,
                                         const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws,
                                         size_t ws_bytes, void* stream);

/* The projection with sparse deviations (an extension: the reference has none; Sparse-Gen, Dhar, Grover and Ermon, ICML
 * 2018).  Each restart row carries nu in R^{H*W*C}, starting at +0, and fits u = G(z) + nu (one fp32 add per element):
 * the data term D is the counterpart's, computed on u in place of G(z) - the image loss (1/n) sum w l(u - x) with
 * n = H*W*C, or the measured loss (1/m) sum l(A_i u - y_i) - squared error or Huber, weighted or not.  Each restart
 * minimises
 *   J(z, nu) = D(u) + lambda ||z||^2 + l1 ||nu||_1          (the lambda term only with a prior)
 * for l1 >= 0 and step >= 0, both finite.
 *   - p_nu = l1 * S, S = sum |nu_p| over the H*W*C pixels of the row in fp32: lane l of a warp adds |nu_l|, |nu_{l+32}|,
 *     ... in ascending p from +0, then a butterfly over the 32 lanes at offsets 16, 8, 4, 2, 1.  J = ((D + p_z) + p_nu)
 *     as fp32 adds, or D + p_nu without a prior.
 *   - g = dD/du: (2/n) w c for the image loss (c the residual u - x, or for Huber its clip to delta), or the measured
 *     path's fp32 dy = (2/m) A^T c before its cotangent entry.  The generator's backward receives g as the counterpart's
 *     does; the update of z is the counterpart's (momentum or Adam, with or without the prior's term).
 *   - The update of nu is one proximal-gradient (ISTA) step on the same iterate:
 *       nu <- S_tau(fmaf(-eta, g, nu)),  S_tau(a) = |a| > tau ? a - copysign(tau, a) : +0
 *     with eta = step n / 2 (step m / 2 measured) and tau = eta l1, both in double on the host, rounded to fp32.  With
 *     step = 1 on the unweighted squared-error image loss one step is the exact minimiser over nu, S_tau(x - G(z)), and
 *     tau = l1 n / 2 is the residual beyond which a pixel counts as a deviation; Sparse-Gen's unnormalised lambda is n l1.
 *     step = 1 is the 1/Lipschitz step for ||A||_2 <= 1 (the normalised blurs and box averages of a convolution
 *     operator).  nu's step is constant: decay_lr and Adam apply to z only.
 *   - Iteration t computes D, g and J at (z_t, nu_t) and, if t < L - 1, moves both to (z_{t+1}, nu_{t+1}).  loss_dev and
 *     the arg-min use J at iteration L - 1; a prune point iter_k ranks by J at iteration iter_k - 1, before that
 *     iteration's update.  Survivors carry their nu, and each follows its unpruned trajectory exactly.
 *   - rec_dev is G(z) of the chosen restart (the range projection); dev_out [batch, H, W, C] (nullable, 16-byte aligned)
 *     receives that restart's nu.  The full estimate is their sum.
 *   - step = 0 keeps nu and p_nu at +0: every measured entry (dense, CSR, convolution) then gives its counterpart's
 *     rec_dev, loss_dev and idx_dev bit for bit.  The image entry without weights equals the CSR entry on the identity
 *     (m = n) bit for bit at any step on both precisions: its data term is that operator fused (the CSR measurement
 *     product's loss reduction, the adjoint's fmaf chain from +0).  w = 1 everywhere gives the unweighted bits.
 *   - use_bn is allowed unpruned; with a schedule it is refused as by the counterpart.
 * Each entry takes the options of its prior entry - adam NULL for momentum, huber_delta NULL for the squared error,
 * z_prior NULL for no prior (else lambda = *z_prior, checked as dgan_reconstruct_prior checks it), sched NULL with
 * n_points 0 unpruned - then sparse_dev (not NULL) and dev_out.  Every loss, the image loss included, runs the measured
 * loop: the image loss leaves the fused last-layer epilogue of dgan_reconstruct.
 * Workspace: dgan_workspace_bytes_sparse_dev / dgan_workspace_bytes_measured_sparse_dev, the counterpart's layout with nu
 * and u appended (and, for the image loss, the measured row buffers of m = n): 2 * rows * H*W*C * 4 bytes more, where rows
 * is batch * rec_rr rounded up to the row tile, per region when pruned - 126 MB at CelebA batch 128, rec_rr 10.
 * l1 or step NaN, infinite or negative, eta or tau not finite in fp32, a misaligned dev_out or a NULL sparse_dev:
 * DGAN_ERR_INVALID_ARG naming the value, checked after the counterpart's checks and before anything is enqueued.
 * Counts, with L iterations and P prune points, against the counterpart (the same call without sparse deviations):
 * dgan_last_enqueue_count is the counterpart's + 1, + 1 more with dev_out.
 * dgan_last_launch_count is, for a measured entry, the counterpart's + L (the nu update) + 1 + P (p_nu, at
 * iteration L - 1 and at each prune point) + P (the survivors' nu gather), + 1 with dev_out; for the image entry, that of
 * dgan_reconstruct_measured_sparse_dev on a dense operator with m = H*W*C and the same options - 3 (the operator's
 * staging) - (L - 1) (the adjoint products, fused into the image residual).  The graph cache keys on l1 and step. */
typedef struct dgan_sparse_dev {
  float l1;     /* >= 0: the weight of ||nu||_1 in J */
  float step;   /* >= 0: nu's step, in units of 2/n (2/m): step = 1 is eta = n / 2 */
} dgan_sparse_dev;

/* The workspace of dgan_reconstruct_sparse_dev (weighted: with w_dev; adam: with the Adam update; sched / n_points as
 * there).  0 for an invalid argument. */
size_t dgan_workspace_bytes_sparse_dev(dgan_handle h, int batch, int rec_rr, int weighted, int adam,
                                       const dgan_prune_point* sched, int n_points);

/* The workspace of dgan_reconstruct_measured[_csr / _conv]_sparse_dev: nnz -1 for a dense operator, else the CSR
 * non-zeros; op not NULL for a convolution (nnz -1 and m = dgan_conv_op_m(h, op)).  0 for an invalid argument. */
size_t dgan_workspace_bytes_measured_sparse_dev(dgan_handle h, int batch, int rec_rr, int m, int nnz, const dgan_conv_op* op,
                                                int adam, const dgan_prune_point* sched, int n_points);

/* dgan_reconstruct_sparse_dev: the image loss; w_dev NULL for dgan_reconstruct's loss, else dgan_reconstruct_weighted's. */
int dgan_reconstruct_sparse_dev(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                const float* huber_delta, const float* z_prior, const dgan_prune_point* sched, int n_points,
                                const dgan_sparse_dev* sparse_dev, float* dev_out, const float* x_dev, const float* w_dev,
                                const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev, void* ws,
                                size_t ws_bytes, void* stream);

/* dgan_reconstruct_measured (a dense operator) with the sparse deviations of dgan_reconstruct_sparse_dev. */
int dgan_reconstruct_measured_sparse_dev(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                         const float* huber_delta, const float* z_prior, const dgan_prune_point* sched,
                                         int n_points, const dgan_sparse_dev* sparse_dev, float* dev_out, const float* a_dev,
                                         int m, const float* y_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                                         int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream);

/* dgan_reconstruct_measured_csr with the sparse deviations of dgan_reconstruct_sparse_dev. */
int dgan_reconstruct_measured_csr_sparse_dev(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                             const float* huber_delta, const float* z_prior, const dgan_prune_point* sched,
                                             int n_points, const dgan_sparse_dev* sparse_dev, float* dev_out,
                                             const int32_t* row_ptr, const int32_t* col_idx, const float* val, int m, int nnz,
                                             const float* y_dev, const float* z0_dev, float* rec_dev, float* loss_dev,
                                             int32_t* idx_dev, void* ws, size_t ws_bytes, void* stream);

/* dgan_reconstruct_measured_conv with the sparse deviations of dgan_reconstruct_sparse_dev. */
int dgan_reconstruct_measured_conv_sparse_dev(dgan_handle h, const dgan_rec_params* params, const dgan_adam_params* adam,
                                              const float* huber_delta, const float* z_prior, const dgan_prune_point* sched,
                                              int n_points, const dgan_sparse_dev* sparse_dev, float* dev_out,
                                              const dgan_conv_op* op, const float* k_dev, const float* y_dev,
                                              const float* z0_dev, float* rec_dev, float* loss_dev, int32_t* idx_dev,
                                              void* ws, size_t ws_bytes, void* stream);

/* tf.gradients(generator_fn(z), z, grad_ys=dy) (models/gan.py:657-665,726-735 through tflib's ops):
 *   z_dev [n_rows, latent] fp32, dy_dev [n_rows, H*W*C] fp32 -> dz_dev [n_rows, latent] fp32,
 *   y_dev [n_rows, H*W*C] = G(z) (nullable; bit-identical to dgan_forward).  The forward is recomputed.
 *   Workspace: dgan_workspace_bytes(h, n_rows, 1).  With use_bn the batch statistics of the n_rows rows are
 *   differentiated (rows are coupled, as in the reference).  No host synchronisation, no allocation.
 * DGAN_PREC_FP16 scales each row's cotangent by a power of two before its fp16 backward (one scale for the call with
 * use_bn) and divides it out of dz, so dz does not depend on the magnitude of dy beyond the fp32/fp16 range limits. */
int dgan_vjp(dgan_handle h, const float* z_dev, int n_rows, const float* dy_dev, float* y_dev, float* dz_dev,
             void* workspace, size_t workspace_bytes, void* stream);

/* The linearisation of generator_fn at z (models/gan.py:657-665,726-735):
 *   z_dev [n_rows, latent] fp32, t_dev [n_rows, latent] fp32 (tangent) -> ty_dev [n_rows, H*W*C] fp32 = J_G(z) t,
 *   y_dev [n_rows, H*W*C] = G(z) (nullable; bit-identical to dgan_forward).
 *   Workspace: dgan_workspace_bytes(h, n_rows, 1).  With use_bn the batch statistics of the n_rows rows are
 *   differentiated (rows are coupled).  No host synchronisation; no allocation once this row count has been planned
 *   (the first dgan_jvp at a row count plans the tangent pass for it).
 * The forward is recomputed.  DGAN_PREC_FP16 scales each row's tangent by a power of two that puts its largest entry in
 * [0.25, 0.5) (one scale for the call with use_bn) and divides it out of ty, so jvp(z, 2^k t) == 2^k jvp(z, t). */
int dgan_jvp(dgan_handle h, const float* z_dev, int n_rows, const float* t_dev, float* y_dev, float* ty_dev,
             void* workspace, size_t workspace_bytes, void* stream);

/* Kernels run by the most recent dgan_reconstruct on this handle (1 + 8 L - 4 + 2 with DGAN_PREC_FP16 on the MNIST stack
 * without BatchNorm; with net_dim > 64 the Linear's forward and Generator.2's backward each run as two column blocks of
 * 256 channels, 1 + 10 L - 5 + 2).  A dgan_reconstruct_measured call runs 3 + 6 (L - 1) + 1 kernels more with
 * DGAN_PREC_FP16 and 3 + 3 (L - 1) + 1 more with DGAN_PREC_FP32 (see there); a dgan_reconstruct_measured_csr call
 * 5 + 6 (L - 1) + 1 and 5 + 3 (L - 1) + 1 more; a dgan_reconstruct_pruned call with P prune points 3 P + 1 more, and a
 * dgan_reconstruct_measured[_csr]_pruned call 3 P + 1 more than the unpruned measured call with the same operator kind.
 * An Adam call (dgan_reconstruct_adam, dgan_reconstruct_measured[_csr]_adam) runs as many as its momentum counterpart,
 * plus L - 1 on the DGAN_PREC_FP16 image loss, whose Adam update is a kernel of its own.  A Huber call
 * (dgan_reconstruct_huber, dgan_reconstruct_measured[_csr]_huber) runs as many as its squared-error counterpart.  A
 * dgan_reconstruct_measured_conv call runs 4 fewer than the dgan_reconstruct_measured_csr call with the same options.  A
 * prior call (dgan_reconstruct[_measured[_csr / _conv]]_prior) runs its counterpart's + 1 + P with P prune points, + L - 1
 * on the DGAN_PREC_FP16 image loss with momentum.  A sparse-deviation call: see dgan_reconstruct_sparse_dev. */
int64_t dgan_last_launch_count(dgan_handle h);

/* Stream operations the HOST issued for it.  The L-step loop only touches the workspace, so it is captured into a CUDA
 * graph the first time a (workspace, batch, rec_rr, rec_iters, rec_lr, momentum, decay_lr, weighted, m, operator kind,
 * nnz, prune schedule, optimiser: momentum, or Adam with its beta1, beta2 and eps, and data term: the squared error, or
 * the Huber loss with its delta, and latent prior: none, or lambda, and sparse deviations: none, or l1 and step) combination is seen and replayed with one cudaGraphLaunch afterwards: z0 initialiser (+ its memsets), image copy
 * (measured calls: the three kernels that stage A, A^T and y; CSR-measured calls: the five that validate and stage them;
 * convolution-measured calls: the one that stages the kernels and y), graph, loss sum, arg-min select.  A convolution
 * operator's geometry is part of the key; its kernel values are not. */
int64_t dgan_last_enqueue_count(dgan_handle h);

/* Algorithmic multiply-accumulates of one generator forward per latent row (exact in-bounds
 * taps, SURVEY section 8d); backward-to-z has the same count. */
int64_t dgan_macs_per_row(dgan_handle h);

/* Per-kernel device timing for roofline reports (no reference counterpart).  While enabled every
 * kernel launch of dgan_reconstruct is bracketed by CUDA events on the launching stream; never
 * enable it in a timed throughput pass.  dgan_profile_read synchronises on the recorded events
 * and returns, per kernel kind (layer x direction), the summed milliseconds, the launch count and
 * the algorithmic FLOPs of one launch (2 x exact in-bounds MACs x latent rows of the last call). */
int dgan_profile_enable(dgan_handle h, int enable);
int dgan_profile_num_kinds(dgan_handle h);
const char* dgan_profile_kind_name(dgan_handle h, int kind);
int dgan_profile_read(dgan_handle h, int max_kinds, double* ms_out, int64_t* launches_out,
                      double* flops_per_launch_out);

const char* dgan_last_error(void);
int dgan_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* DEFENSEGAN_B200_H_ */
