// Tensor-core path (DGAN_PREC_FP16): shared pieces of the pixel-graph GEMM on Hopper wgmma.
//
//   out[q][n][:] = epi( sum_{(p,t) in pairs(q)} in[p][n][:] x W_t )        fp16 operands, fp32 accumulate
//
// Activations are pixel-major [P][N rows][C] fp16, so one input pixel x 128 latent rows x 64 channels is a dense
// 16 KB box = one TMA box = one 128B-swizzled K-major wgmma operand; weights are stored per tap as [N][K] fp16
// tiles.  The conv geometry is data, not code: only in-bounds (input pixel, tap) pairs are listed, so exactly the
// algorithmic MACs are issued - no zero-insertion, no padding rows, no im2col buffer.
// This header holds the PTX wrappers, the wgmma descriptors, the weight re-layout and the helpers of the epilogue;
// the kernel that uses them and its host-side planning are in kernels_tc2.cuh.
#pragma once
#include <cuda.h>  // CUtensorMap types only; the encoder is fetched through the runtime (no -lcuda)

#include "common.cuh"

namespace dgan {

constexpr int TC_LINEAR_SPLIT = 4;           // partial sums of the Linear backward (dz)

struct TcState {
  float grad_scale = 64.f;      // fp16 gradient scaling (undone in the z update)
  void* encode_fn = nullptr;    // cuTensorMapEncodeTiled
  int num_sms = 132;
};

// ------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------
namespace ptx {
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Keeps the compiler from moving accesses of accumulator registers across wgmma issue / wait.
template <int N>
__device__ __forceinline__ void fence_operands(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T per warpgroup, fp16 x fp16 -> fp32, both operands K-major in shared memory.
// d: the N/2 accumulator registers of this thread (fragment layout of the m64nNk16 f32 accumulator).
template <int N> struct Wgmma;
template <> struct Wgmma<16> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(scale_d));
  }
};
template <> struct Wgmma<48> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
        : "l"(a), "l"(b), "r"(scale_d));
  }
};
template <> struct Wgmma<64> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(scale_d));
  }
};
template <> struct Wgmma<128> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(scale_d));
  }
};
template <> struct Wgmma<192> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
        : "l"(a), "l"(b), "r"(scale_d));
  }
};
template <> struct Wgmma<256> {
  static __device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(a), "l"(b), "r"(scale_d));
  }
};
}  // namespace ptx

// K-major, 128B-swizzled operand tile: rows 128 B apart, 8-row groups 1024 B apart (SBO); wgmma descriptor layout
// type 1 = SWIZZLE_128B (bits 62-63), leading byte offset unused for swizzled K-major operands (1 by convention).
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
// K-major, 32B-swizzled operand sub-tile of 16 channels (one k16): rows 32 B apart, 8-row groups 256 B apart (SBO);
// layout type 3 = SWIZZLE_32B.  The k16 spans the whole 32 B swizzle width, so the leading byte offset is unused.
__device__ __forceinline__ uint64_t make_smem_desc_sw32(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(256 >> 4) << 32) | ((uint64_t)3 << 62);
}

// fp32 pair -> packed fp16, round-to-nearest, saturating to +-65504: a backward activation that exceeds the fp16 range
// (trained filters, |y - x| up to 2 on CelebA) must not become inf and turn z into NaN for the rest of the loop.
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}

// Extra epilogue kinds of the tensor-core path: the generator's last layer (C_out <= 3) is run as
// a pixel-graph GEMM whose "output pixels" are 4x4 blocks of image pixels (N = 16*C_out columns =
// the block's pre-activations), so that the output non-linearity, the squared error, its
// derivative and the per-row loss partial are all computed in the epilogue
// (models/dataset_models.py:68-69,161-163; models/gan.py:411-414).
// The _W kinds weight the squared error per pixel (dgan_reconstruct_weighted): e = w (y - x), loss part += e (y - x),
// d(pre) = e act'(y); with w = 1, e == y - x and every stored value is the unweighted kind's.
// The _H kinds (and _WH, weighted) replace the squared error by the Huber loss at delta = TcFinalArgs::huber
// (dgan_reconstruct_huber): with d = y - x, c = |d| > delta ? copysign(delta, d) : d, e = w c (e = c unweighted), the loss
// part takes e (2 d - c) and d(pre) = e act'(y).  When no |d| exceeds delta, c == d and 2 d - c == d, so every stored
// value is the squared-error kind's.  They run on the plans of the kinds they replace (tc2_launch selects them).
enum TcEpilogue : int { EPI_FINAL_SIGMOID1 = 8, EPI_FINAL_TANH3 = 9, EPI_FINAL_SIGMOID1_W = 10, EPI_FINAL_TANH3_W = 11,
                        EPI_FINAL_SIGMOID1_H = 12, EPI_FINAL_TANH3_H = 13, EPI_FINAL_SIGMOID1_WH = 14, EPI_FINAL_TANH3_WH = 15 };
// The Huber kind that replaces final kind epi (any other epilogue is returned unchanged)
__host__ __device__ constexpr int tc_huber_epi(int epi) {
  return epi == EPI_FINAL_SIGMOID1 ? EPI_FINAL_SIGMOID1_H : epi == EPI_FINAL_TANH3 ? EPI_FINAL_TANH3_H
       : epi == EPI_FINAL_SIGMOID1_W ? EPI_FINAL_SIGMOID1_WH : epi == EPI_FINAL_TANH3_W ? EPI_FINAL_TANH3_WH : epi;
}
__host__ __device__ constexpr bool tc_final_epi(int epi) { return epi >= EPI_FINAL_SIGMOID1 && epi <= EPI_FINAL_TANH3_WH; }

struct TcFinalArgs {
  const float* x;        // [B][H*W*C] target images (NULL: forward only)
  float* y;              // [n_pad][H*W*C] G(z)
  float* loss_part;      // [n_blocks][n_pad] sum over the block of (y-x)^2 (written when write_y)
  int R, B, n_rows;      // restarts per image, images, valid latent rows
  int nbx, w_out;        // blocks per image row, image width
  int write_y;           // store G(z) (only the last iteration / forward-only calls consume it)
  float gscale;          // fp16 gradient scaling applied to dL/dpre
  // 1-bit ReLU masks of the tensor-core path: bit j of word [(q*n_pad + n)*(N/64) + g] <=> out[q][n][g*64+j] > 0.
  // Written by the forward EPI_BIAS_RELU epilogue, read by the backward EPI_MASK epilogue
  // (tf.nn.relu's gradient passes where the forward output was > 0).
  unsigned long long* mb_out;
  const unsigned long long* mb_in;
  // split-K Linear backward with the momentum update (tf.train.MomentumOptimizer, models/gan.py:389-391) in its tail:
  // the CTA whose partial sums complete a 128-row tile (ticket from m_counter[tile]) applies
  // v <- mu v + gmul * sum(parts), z <- z - lr v for that tile
  float* mz; float* mv; __half* mz_h;   // z, velocity [n_pad][latent] fp32, fp16 copy of z
  float m_gmul, m_lr, m_mu;
  unsigned* m_counter;   // [n_pad / 128] arrival tickets, self-resetting; NULL = plain partial sums
  int m_nparts;          // partial sums per row tile
  size_t m_count;        // elements per partial-sum array (n_pad * latent)
  // A column block of a layer-direction wider than one tile (tc_directions): the output's row stride in channels (its
  // full width) and the block's first channel.  The TMA store adds col0 to its channel coordinate; the other outputs,
  // the bias and the ReLU masks are passed already offset to the block.
  int out_ld, col0;
  // The weighted last-layer epilogues: [B][H*W*C] per-pixel weights of the squared error, indexed as x.  Last, so that
  // every other field keeps its offset.
  const float* xw;
  // The Huber final kinds: delta (> 0, +inf allowed); 0 selects the squared-error kinds.  After xw for the same reason.
  float huber;
};

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// fp32 [tiles][rows_full][cols] -> fp16 [tiles][rows][cols]: rows row0 .. row0 + rows of every tile (a column block of a
// layer-direction's weight tiles; rows == rows_full: all of them)
__global__ void tc_convert_kernel(const float* __restrict__ in, __half* __restrict__ out, size_t n, int rows_full, int row0,
                                  int rows, int cols) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const size_t per = (size_t)rows * cols, t = i / per, rem = i % per;
  out[i] = __float2half_rn(in[(t * rows_full + row0) * cols + rem]);
}
// Linear backward tiles: out[q][k][c] = W[k][q*C + c]   (W is (latent, 16*C))
__global__ void tc_linear_bwd_tiles_kernel(const float* __restrict__ W, __half* __restrict__ out, int latent, int C,
                                           int n_pix) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)n_pix * latent * C;
  if (i >= total) return;
  const int c = (int)(i % C);
  const int k = (int)((i / C) % latent);
  const int q = (int)(i / ((size_t)C * latent));
  out[i] = __float2half_rn(W[(size_t)k * n_pix * C + (size_t)q * C + c]);
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 3-D fp16 tensor [d2][d1][d0] (d0 contiguous), box {box0, box1, 1}: box0 = 64 channels with 128B swizzle (the
// 64-channel operand), or 16 channels with 32B swizzle (one 16-channel sub-tile of a narrow operand).
static int tc_make_map(const TcState& st, CUtensorMap* map, const void* base, uint64_t d0, uint64_t d1, uint64_t d2,
                       uint32_t box1, uint32_t box0 = 64) {
  if (st.encode_fn == nullptr) { set_error("cuTensorMapEncodeTiled unavailable"); return DGAN_ERR_CUDA; }
  const cuuint64_t dims[3] = {d0, d1, d2};
  const cuuint64_t strides[2] = {d0 * 2, d0 * d1 * 2};
  if (box0 != 64 && box0 != 16) { set_error("tensor map box must be 64 or 16 channels wide"); return DGAN_ERR_UNSUPPORTED; }
  const cuuint32_t box[3] = {box0, box1, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = ((PFN_encodeTiled)st.encode_fn)(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims,
                                               strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                                               box0 == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_32B,
                                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return DGAN_ERR_CUDA;
  }
  return 0;
}

static int tc_upload(std::vector<void*>* allocs, const void* host, size_t bytes, void** dev, cudaStream_t s) {
  DGAN_CUDA_CHECK(cudaMalloc(dev, bytes));
  allocs->push_back(*dev);
  DGAN_CUDA_CHECK(cudaMemcpyAsync(*dev, host, bytes, cudaMemcpyHostToDevice, s));
  // the host vectors die when the builder returns: make sure the copy has been staged
  DGAN_CUDA_CHECK(cudaStreamSynchronize(s));
  return 0;
}

// The tensor-map encoder and the SM count of the current device.
static int tc_init(TcState& st) {
  cudaDriverEntryPointQueryResult qres;
  void* fn = nullptr;
  DGAN_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (fn == nullptr || qres != cudaDriverEntryPointSuccess) { set_error("cuTensorMapEncodeTiled not found in the driver"); return DGAN_ERR_CUDA; }
  st.encode_fn = fn;
  int dev = 0;
  DGAN_CUDA_CHECK(cudaGetDevice(&dev));
  DGAN_CUDA_CHECK(cudaDeviceGetAttribute(&st.num_sms, cudaDevAttrMultiProcessorCount, dev));
  return 0;
}

// ---- the generator's last layer as block GEMMs ---------------------------------------------
// Image pixels are grouped into 4x4 blocks; block (by,bx) receives from the 4x4 input pixels
// o = 2by-1+ry, p = 2bx-1+rx (ry,rx in 0..3): out row 4by+li = 2o+ka-1  =>  ka = li - 2ry + 3.
// Weight tile (ry,rx), forward:  rows (li*4+lj)*C_out+co, cols ci   = F[ka][kb][co][ci] or 0
//                      backward: rows ci, cols (li*4+lj)*C_out+co
__global__ void tc_final_tiles_kernel(const float* __restrict__ F /*[25][C_out][C_in]*/, int C_out, int C_in,
                                      __half* __restrict__ wf /*[16][16*C_out][C_in]*/,
                                      __half* __restrict__ wb /*[16][C_in][16*C_out]*/) {
  const int tile = blockIdx.x, ry = tile >> 2, rx = tile & 3;
  const int nrow = 16 * C_out;
  for (int e = threadIdx.x; e < nrow * C_in; e += blockDim.x) {
    const int r = e / C_in, ci = e % C_in;
    const int co = r % C_out, l = r / C_out, li = l >> 2, lj = l & 3;
    const int ka = li - 2 * ry + 3, kb = lj - 2 * rx + 3;
    float v = 0.f;
    if (ka >= 0 && ka < 5 && kb >= 0 && kb < 5) v = F[((size_t)(ka * 5 + kb) * C_out + co) * C_in + ci];
    wf[((size_t)tile * nrow + r) * C_in + ci] = __float2half_rn(v);
  }
  for (int e = threadIdx.x; e < C_in * nrow; e += blockDim.x) {
    const int ci = e / nrow, k = e % nrow;
    const int co = k % C_out, l = k / C_out, li = l >> 2, lj = l & 3;
    const int ka = li - 2 * ry + 3, kb = lj - 2 * rx + 3;
    float v = 0.f;
    if (ka >= 0 && ka < 5 && kb >= 0 && kb < 5) v = F[((size_t)(ka * 5 + kb) * C_out + co) * C_in + ci];
    wb[((size_t)tile * C_in + ci) * nrow + k] = __float2half_rn(v);
  }
}

// Pair table of the tensor-core path: an output pixel without contributions (use_bn on MNIST: Generator.3's backward
// over the 8x8 raster of which 7x7 is used - the cropped outputs get no gradient) receives (pixel 0, zero tile).
static PairTable tc_with_zero_tile(const PairTable& t, int zero_tile) {
  PairTable r;
  r.off.push_back(0);
  for (size_t q = 0; q + 1 < t.off.size(); ++q) {
    for (int e = t.off[q]; e < t.off[q + 1]; ++e) r.pairs.push_back(t.pairs[(size_t)e]);
    if (t.off[q] == t.off[q + 1]) r.pairs.push_back(make_int2(0, zero_tile));
    r.off.push_back((int)r.pairs.size());
  }
  return r;
}

// dz = sum over the Linear's 16 output pixels, as TC_LINEAR_SPLIT partial sums
static PairTable linear_split_pairs(int n_pix) {
  PairTable split;
  split.off.push_back(0);
  const int per = n_pix / TC_LINEAR_SPLIT;
  for (int part = 0; part < TC_LINEAR_SPLIT; ++part) {
    for (int q = part * per; q < (part + 1) * per; ++q) split.pairs.push_back(make_int2(q, q));
    split.off.push_back((int)split.pairs.size());
  }
  return split;
}

static PairTable final_block_fwd_pairs(int h_in, int w_in) {
  PairTable t;
  t.off.push_back(0);
  const int nby = h_in / 2, nbx = w_in / 2;   // (2*h_in)/4 blocks per side
  for (int by = 0; by < nby; ++by)
    for (int bx = 0; bx < nbx; ++bx) {
      for (int ry = 0; ry < 4; ++ry)
        for (int rx = 0; rx < 4; ++rx) {
          const int o = 2 * by - 1 + ry, p = 2 * bx - 1 + rx;
          if (o < 0 || o >= h_in || p < 0 || p >= w_in) continue;
          t.pairs.push_back(make_int2(o * w_in + p, ry * 4 + rx));
        }
      t.off.push_back((int)t.pairs.size());
    }
  return t;
}

static PairTable final_block_bwd_pairs(int h_in, int w_in) {
  PairTable t;
  t.off.push_back(0);
  const int nby = h_in / 2, nbx = w_in / 2;
  for (int o = 0; o < h_in; ++o)
    for (int p = 0; p < w_in; ++p) {
      for (int by = 0; by < nby; ++by) {
        const int ry = o - 2 * by + 1;
        if (ry < 0 || ry > 3) continue;
        for (int bx = 0; bx < nbx; ++bx) {
          const int rx = p - 2 * bx + 1;
          if (rx < 0 || rx > 3) continue;
          t.pairs.push_back(make_int2(by * nbx + bx, ry * 4 + rx));
        }
      }
      t.off.push_back((int)t.pairs.size());
    }
  return t;
}

}  // namespace dgan
