// Tensor-core path, version 2: pixel-graph GEMM on Hopper wgmma with a host-planned operand stream.
//
// The CTAs come in clusters of two: CTA rank r of pair `pair` owns the 128-row latent tile 2*mp + r of every item
// (window of 1-8 output pixels x row pair mp) that the host assigned to its pair, so both CTAs walk the same step list
// and need the same weight tiles.  Each CTA loads one half of every weight tile and multicasts it into the shared
// memory of both, so a pair reads each weight tile from L2 once.
//   * operands live in a circular shared-memory ring of variable-size steps planned on the host
//     (tc2_get_schedule): per CTA pair one contiguous stream of step records, LPT-assigned; a ring region is refilled
//     only after the consumers of BOTH CTAs released it (the peer's loads write into it too);
//   * a step's MMA record reaches the consumers as its operands do: the producer copies it into a shared-memory slot,
//     and the copy completes on the step's full barrier, so the consumers' step loop loads nothing from global memory;
//   * roles per CTA: one producer warpgroup (one warp issues the TMA loads) and two consumer warpgroups.  The producer
//     gives up registers (setmaxnreg) so that the consumers can hold accumulators and epilogue without spilling.  Each
//     consumer warpgroup owns 64 of the tile's 128 rows and issues wgmma.mma_async (M = 64, K = 16) into register
//     accumulators - up to 256 columns: the 1-8 accumulators of the item's window.  A step is a run-time number of
//     rounds, and a round is one op per accumulator with something to add, in compile-time order: the consumers branch
//     on the round's active set to a straight-line variant, so the compiler never has to choose an accumulator at run
//     time (the 8-slot and the narrow instantiations issue into every accumulator, and one with nothing to add reads
//     an all-zero weight tile).  One
//     wgmma group is committed per round and one stays in flight, across step boundaries too; a step's ring region is
//     released once the NEXT step's first round is issued and every earlier group has retired; after the item's last
//     step the consumer waits for all MMAs and runs the epilogue straight from the registers.  Each consumer warp
//     stores the 16 rows it holds with its own TMA store.
#pragma once
#include <unordered_map>

#include "kernels_tc.cuh"
#include "tc_records.cuh"

namespace dgan {

constexpr int TC2_SMEM_MAX = 232448;         // 227 KB opt-in limit per CTA
constexpr int TC2_TILE_BYTES = 128 * 128;    // one 128-row x 64-channel fp16 tile (TMA box, 128B swizzle)
constexpr int TC2_BUF_COLS = 256;            // accumulator columns of one item (128 fp32 registers per consumer thread)
constexpr int TC2_CONSUMERS = 256;           // two consumer warpgroups
constexpr int TC2_THREADS = TC2_CONSUMERS + 128;   // + the producer warpgroup
// Register split of the 64K-entry register file (setmaxnreg): 128 x 40 + 256 x 232 = 64512.  Every thread starts at
// the launch's 168.
constexpr int TC2_PRODUCER_REGS = 40, TC2_CONSUMER_REGS = 232;
constexpr int TC2_STORE_ROWS = 16;           // rows per output TMA store: each consumer warp stores the 16 rows it holds

// Where each CTA pair's work starts, passed in the kernel's parameter space (constant bank): the first records are then
// ONE global round trip away from the kernel's entry, and that round trip overlaps the barrier set-up.
constexpr int TC2_MAX_PAIRS = 80;
struct Tc2Heads {
  uint32_t off[TC2_MAX_PAIRS + 1];    // record offsets of the pairs' step streams
};

// A window's output pixels, one per accumulator (the consumers' epilogue reads it).
struct __align__(16) TcItem2 {
  uint16_t q[16];
  uint32_t n_acc;
};
static_assert(sizeof(TcItem2) == 48 && offsetof(TcItem2, n_acc) == 32, "the kernel's item loads");

// Accumulator columns reserved per accumulator of a window.  N <= 32 (MNIST last layer: 16 outputs per block) packs
// 8 accumulators into the 256 columns of an item, so a window can span a whole row of blocks.
__host__ __device__ constexpr int tc2_acc_stride(int n_tile) { return n_tile <= 32 ? 32 : (n_tile < 64 ? 64 : n_tile); }

// Does this instantiation stage its output tiles through shared memory + TMA?
__host__ __device__ constexpr bool tc2_tma_epilogue(int n_tile, int epi, int out_bytes) {
  return out_bytes == 2 && n_tile >= 64 && !tc_final_epi(epi);
}

constexpr int TC2_REC_BATCH = 16;
constexpr int TC2_STAGING_BYTES = TC2_REC_BATCH * (int)sizeof(TcRec);   // producer record ring (records: tc_records.cuh)
// The consumers' MMA records: one slot per barrier slot.  The producer copies a step's record there with the step's
// operands, on the same full barrier.
constexpr int TC2_MREC_BYTES = TC2_NSLOT * (int)sizeof(TcRec);

// Output staging of the TMA-store epilogues: two 16-row x 128 B buffers per consumer warp (the next unit is written
// while the store of the previous one still reads shared memory).
__host__ __device__ constexpr int tc2_epi_tiles(int n_tile, int epi, int out_bytes) {
  return tc2_tma_epilogue(n_tile, epi, out_bytes) ? 2 : 0;
}
// k16 MMAs per op (KSUB) of a direction with K input channels: 4 = a 64-channel k-chunk, one 128B-swizzled operand per
// tile; 1..3 = a narrow operand (the last layer's backward, K = 16 * C_out) of KSUB 16-channel 32B-swizzled sub-tiles.
__host__ __device__ constexpr int tc2_ksub(int K) { return K % 64 == 0 ? 4 : K / 16; }
// Staged bytes of one A tile (128 rows) and one weight tile (N rows) of an op.
__host__ __device__ constexpr int tc2_a_bytes(int ksub) { return 128 * 32 * ksub; }
__host__ __device__ constexpr int tc2_b_bytes(int n_tile, int ksub) { return n_tile * 32 * ksub; }
// Does an instantiation with `maxb` accumulator slots and `ksub` k16 MMAs per op issue zero-tile ops?  With 2 or 4
// slots and 64-channel ops, a round issues only its real ops: the consumers branch on the round's active set to one of
// at most 15 straight-line variants (tc2_mma_round).  The others keep the fixed round, in which an accumulator with
// nothing to add reads the zero tile: the 8-slot instantiations (N = 16), and the narrow ones (the last layer's
// backward, 1 or 3 k16 MMAs per op), where the dispatch measured slower than the zero-tile MMAs it saves.
__host__ __device__ constexpr bool tc2_issues_zero_ops(int maxb, int ksub) { return maxb > 4 || (maxb > 1 && ksub < 4); }
// The all-zero weight tile read by the zero-tile ops of the instantiations that issue them.  It sits right after the
// ring, has the shape of a weight tile and is written once per CTA.  The instantiations that skip zero-tile ops keep
// its space too: the ring size caps the step size (tc2_search), so dropping it would move the plans, and the time
// model's constants were fitted to these rings.
__host__ __device__ constexpr int tc2_zero_bytes(int n_tile, int maxb, int ksub) { return maxb > 1 ? tc2_b_bytes(n_tile, ksub) : 0; }
__host__ __device__ constexpr int tc2_ring_bytes(int n_tile, int maxb, int ksub, int epi, int out_bytes) {
  const int epi_b = tc2_epi_tiles(n_tile, epi, out_bytes) * TC2_TILE_BYTES;
  const int raw = ((TC2_SMEM_MAX - 1024 - 256 - TC2_MREC_BYTES - TC2_STAGING_BYTES - epi_b - tc2_zero_bytes(n_tile, maxb, ksub)) / 1024) * 1024;
  return raw > TC2_RING_MAX_KB * 1024 ? TC2_RING_MAX_KB * 1024 : raw;
}

// MAXB_: accumulator slots of the instantiation = the most ops per round = the most accumulators a window may have.
// With 2 or 4 slots and 64-channel ops a round issues only its real ops.  Where the round is fixed (8 slots, narrow
// ops), fewer slots issue fewer zero-tile MMAs but allow only smaller windows (more staged bytes), and the planner
// weighs the two (tc2_plan).
// KSUB_: k16 MMAs per op (tc2_ksub).  4: A and weight tiles are 64-channel 128B-swizzled boxes and the op's k16 step
// through each 128 B row.  1..3: each tile is KSUB sub-tiles of 16 channels (32 B rows, 32B swizzle), one per k16, so a
// narrow K stages and multiplies only its real channels.
template <int N_TILE, int MAXB_, int KSUB_ = 4, int EPI = EPI_NONE, int OUT_BYTES = 2>
struct Tc2Cfg {
  static_assert(MAXB_ >= 1 && MAXB_ <= TC2_BUF_COLS / tc2_acc_stride(N_TILE), "more accumulator slots than columns");
  static_assert(KSUB_ >= 1 && KSUB_ <= 4, "k16 MMAs per op");
  static constexpr int KSUB = KSUB_;
  static constexpr int A_BYTES = tc2_a_bytes(KSUB);                      // bytes of one staged activation tile
  static constexpr int B_TILE = tc2_b_bytes(N_TILE, KSUB);               // bytes of one staged weight tile
  static constexpr int A_SUB = 128 * 32, B_SUB = N_TILE * 32;            // narrow ops: bytes of one 16-channel sub-tile
  static constexpr int MAXB = MAXB_;
  static constexpr int ACC_REGS = MAXB * N_TILE / 2;                      // accumulator registers per consumer thread
  static constexpr bool TMA_EPI = tc2_tma_epilogue(N_TILE, EPI, OUT_BYTES);
  static constexpr int EPI_TILES = tc2_epi_tiles(N_TILE, EPI, OUT_BYTES);
  static constexpr int EPI_BYTES = EPI_TILES * TC2_TILE_BYTES;
  static constexpr int ZERO_BYTES = tc2_zero_bytes(N_TILE, MAXB, KSUB);
  static constexpr int RING_BYTES = tc2_ring_bytes(N_TILE, MAXB, KSUB, EPI, OUT_BYTES);    // operand ring (offsets are 8-bit KB)
  static constexpr int SMEM_BYTES = RING_BYTES + ZERO_BYTES + EPI_BYTES + TC2_STAGING_BYTES + 1024 + 256 + TC2_MREC_BYTES;
};

// Every instantiation of tc_bsgemm2_kernel: (N, accumulator slots per round, k16 MMAs per op, epilogue, output type).
// tc2_optin_all, the launch dispatch and the planner's candidate set (tc2_plan) all read this list.  For each
// (N, k16 per op, epilogue, output type) it holds the largest slot count, which every window shape can use, and the
// smaller ones the planner picks for the shipped generators.  The narrow kinds (k16 per op < 4) are the last layer's
// backward: K = 16 (MNIST: EPI_MASK, or EPI_NONE with BatchNorm) and K = 48 (CelebA), at N = 64 (net_dim <= 64) and
// N = 128 (64 < net_dim <= 128).  N = 16 / 48 with EPI_NONE and fp32 output: dgan_jvp's tangent of the last layer's
// pre-activation (last.jvp), on the last layer's forward geometry.  The _W final kinds: the weighted last-layer forward
// (last.fwd.w, dgan_reconstruct_weighted), at the N / slots / k16 of the unweighted final kinds.  The _H / _WH kinds: the
// Huber loss of the final kinds (dgan_reconstruct_huber), at the N / slots / k16 of the kinds they replace; tc2_launch runs
// them on those kinds' plans when TcFinalArgs::huber > 0.
#define TC2_KINDS(X)                                                                                                   \
  X(256, 1, 4, EPI_BIAS_RELU, __half) X(256, 1, 4, EPI_BIAS, __half) X(256, 1, 4, EPI_MASK, __half)                    \
  X(256, 1, 4, EPI_NONE, __half) X(256, 1, 4, EPI_NONE, float) X(256, 1, 4, EPI_BIAS, float)                           \
  X(128, 2, 4, EPI_BIAS_RELU, __half) X(128, 2, 4, EPI_BIAS, __half) X(128, 2, 4, EPI_MASK, __half)                    \
  X(128, 2, 4, EPI_NONE, __half) X(128, 2, 4, EPI_NONE, float) X(128, 2, 4, EPI_BIAS, float)                           \
  X(128, 1, 4, EPI_NONE, float)                                                                                        \
  X(64, 4, 4, EPI_BIAS_RELU, __half) X(64, 4, 4, EPI_BIAS, __half) X(64, 4, 4, EPI_MASK, __half)                      \
  X(64, 4, 4, EPI_NONE, __half) X(64, 4, 4, EPI_NONE, float) X(64, 4, 4, EPI_BIAS, float)                              \
  X(64, 4, 1, EPI_MASK, __half) X(64, 4, 1, EPI_NONE, __half) X(64, 4, 3, EPI_NONE, __half)                            \
  X(128, 2, 1, EPI_MASK, __half) X(128, 2, 1, EPI_NONE, __half) X(128, 2, 3, EPI_NONE, __half)                         \
  X(16, 8, 4, EPI_FINAL_SIGMOID1, __half) X(16, 4, 4, EPI_FINAL_SIGMOID1, __half) X(48, 4, 4, EPI_FINAL_TANH3, __half)   \
  X(16, 8, 4, EPI_NONE, float) X(48, 4, 4, EPI_NONE, float)                                                              \
  X(16, 8, 4, EPI_FINAL_SIGMOID1_W, __half) X(16, 4, 4, EPI_FINAL_SIGMOID1_W, __half) X(48, 4, 4, EPI_FINAL_TANH3_W, __half)   \
  X(16, 8, 4, EPI_FINAL_SIGMOID1_H, __half) X(16, 4, 4, EPI_FINAL_SIGMOID1_H, __half) X(48, 4, 4, EPI_FINAL_TANH3_H, __half)   \
  X(16, 8, 4, EPI_FINAL_SIGMOID1_WH, __half) X(16, 4, 4, EPI_FINAL_SIGMOID1_WH, __half) X(48, 4, 4, EPI_FINAL_TANH3_WH, __half)

struct Tc2Kind { int n, maxb, ksub, epi, out_bytes; };
#define TC2_KIND_ROW(NT, MB, KS, EP, T) {NT, MB, KS, EP, (int)sizeof(T)},
static constexpr Tc2Kind kTc2Kinds[] = {TC2_KINDS(TC2_KIND_ROW)};
#undef TC2_KIND_ROW
// The MMA records carry every instantiation's slots per round and k16 MMAs per op.
constexpr bool tc2_kinds_fit_records() {
  for (const Tc2Kind& k : kTc2Kinds)
    if ((uint32_t)k.maxb > TcMmaRec::MaxB::mask || (uint32_t)k.ksub > TcMmaRec::Ksub::mask) return false;
  return true;
}
static_assert(tc2_kinds_fit_records(), "an instantiation's MAXB or KSUB does not fit the MMA record");
// Is there an instantiation with these template arguments?
static inline bool tc2_has_kind(int n, int maxb, int ksub, int epi, int out_bytes) {
  for (const Tc2Kind& k : kTc2Kinds)
    if (k.n == n && k.maxb == maxb && k.ksub == ksub && k.epi == epi && k.out_bytes == out_bytes) return true;
  return false;
}

namespace ptx {
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// Four 8x8 fp16 matrices from the m64nNk16 accumulator fragment into shared memory: lane L names a row of matrix L / 8.
__device__ __forceinline__ void stmatrix_x4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
// prmt.b32 (default mode): selector nibble n picks byte n & 7 of {b, a}; with bit 3 set, that byte's sign fills the byte
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
  return r;
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// TMA load into the same shared-memory offset of both CTAs of the pair; each CTA's barrier at `bar` receives the bytes
// that land in it.
__device__ __forceinline__ void tma_load_3d_mc2(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "h"((uint16_t)3) : "memory");
}
// Arrive on the barrier at `local_bar` in CTA `cta` of the cluster.  Release at CTA scope (the default): the consumers'
// only accesses it orders are their MMAs' shared-memory reads, which wgmma.wait_group has already completed.
// .release.cluster compiles to MEMBAR.ALL.GPU, which also waits for the warp's outstanding global loads (the next
// step's record), once per step.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t local_bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}" ::"r"(local_bar), "r"(cta) : "memory");
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint2 ld_shared_v2(uint32_t addr) {
  uint2 v;
  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
// As ld_shared_v4, but ordered after the barrier wait before it (the data was written by an asynchronous copy that
// completed on that barrier).
__device__ __forceinline__ uint4 ld_shared_v4_ordered(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}
// Copy `bytes` (a multiple of 16) from global memory into this CTA's shared memory; the barrier at `bar` receives them.
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
template <int R> __device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
// true in exactly one lane of a converged warp
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred P1;\n\telect.sync _|P1, 0xffffffff;\n\tselp.u32 %0, 1, 0, P1;\n\t}" : "=r"(pred));
  return pred != 0;
}
}  // namespace ptx

// k-th item word (tc2_item_word) of CTA pair `pair` from the host-computed table [slot][pair] (-1 = no more work).
// The host assigns items largest-first to the least-loaded pair (LPT) with the cost model of tc2_plan.
__device__ __forceinline__ int tc2_item_at(const int* __restrict__ order, int k, int pair, int n_pairs, int n_slots) {
  return k < n_slots ? __ldg(order + (size_t)k * n_pairs + pair) : -1;
}

// The ops of one round into the accumulators of the set MASK (bit a = accumulator a), in compile-time order: for each,
// the KSUB k16 MMAs of one op (a 64-channel k-chunk, or a narrow operand's 16-channel sub-tiles).  Only the operand
// descriptors and the overwrite predicate come from the record byte of (round, a), so the sequence of wgmma
// instructions and the registers they name are fixed.
//   da0 / db0: descriptors of the step's first A tile (this warpgroup's rows) and first B slot; zoff: the zero tile's
//   distance from db0 in 16-byte units (instantiations that issue zero-tile ops).
template <int NT, int MAXB, int KSUB, uint32_t MASK, int NREG>
__device__ __forceinline__ void tc2_mma_ops(float (&acc)[NREG], const uint32_t (&q)[6], uint64_t da0, uint64_t db0, uint32_t zoff) {
  // the next k16: 32 B further along the 128 B row of a 128B-swizzled tile, or the next 16-channel sub-tile
  constexpr uint32_t DA_K = KSUB == 4 ? 2u : (uint32_t)(128 * 32 >> 4), DB_K = KSUB == 4 ? 2u : (uint32_t)(NT * 32 >> 4);
#pragma unroll
  for (int a = 0; a < MAXB; ++a) {
    if (!((MASK >> a) & 1u)) continue;
    const uint32_t e = TcMmaRec::Ops::get(q[a / TcMmaRec::Ops::PER_WORD], a);
    const uint32_t bs = TcOp::Slot::get(e);
    // descriptors differ only in the 14-bit start-address field (smem < 256 KB, no carry)
    const uint64_t da = da0 + (uint64_t)(TcOp::A::get(e) * (uint32_t)(tc2_a_bytes(KSUB) >> 4));
    const uint32_t boff = bs * (uint32_t)(tc2_b_bytes(NT, KSUB) >> 4);
    const uint64_t db = db0 + (uint64_t)(tc2_issues_zero_ops(MAXB, KSUB) && bs == (uint32_t)TC2_ZERO_SLOT ? zoff : boff);
    const uint32_t keep = TcOp::First::get(e) ^ 1u;  // 0: first MMA into the accumulator, overwrite it
#pragma unroll
    for (int k = 0; k < KSUB; ++k) ptx::Wgmma<NT>::mma(acc + a * (NT / 2), da + DA_K * k, db + DB_K * k, k > 0 ? 1u : keep);
  }
  // in the variant itself: a commit where the variants' paths join would close a hardware group of its own, an empty
  // HGMMA
  ptx::wgmma_commit();
}

// One round of a step, committed as one wgmma group.  Where the instantiation issues zero-tile ops
// (tc2_issues_zero_ops): one op into every accumulator (a slot with nothing to add reads the zero tile).  Otherwise only
// the round's real ops.  The round's active set - the accumulators whose op byte names a B slot, not the zero tile - is
// the same in every thread of the warpgroup (it comes from the step's record), and the branch on it leads to a
// straight-line variant per set.  A guard predicate per MMA would instead make ptxas branch around every
// HGMMA and close a hardware wgmma group at each, so that the round's wait_group 1 would drain the pipe.  The plan
// validator rejects a round without a real op (it would commit an empty group).
template <int NT, int MAXB, int KSUB, int NREG>
__device__ __forceinline__ void tc2_mma_round(float (&acc)[NREG], const uint32_t (&q)[6], uint64_t da0, uint64_t db0, uint32_t zoff) {
  if constexpr (tc2_issues_zero_ops(MAXB, KSUB) || MAXB == 1) {
    tc2_mma_ops<NT, MAXB, KSUB, (1u << MAXB) - 1u>(acc, q, da0, db0, zoff);
  } else {
    static_assert(MAXB <= TcMmaRec::Ops::PER_WORD, "a round's op bytes share the queue's first word");
    uint32_t set = 0;
#pragma unroll
    for (int a = 0; a < MAXB; ++a)
      set |= (TcOp::Slot::get(TcMmaRec::Ops::get(q[0], a)) != (uint32_t)TC2_ZERO_SLOT ? 1u : 0u) << a;
    switch (set) {
#define TC2_ROUND_VARIANT(M) \
  case M:                    \
    if constexpr (M < (1u << MAXB)) tc2_mma_ops<NT, MAXB, KSUB, M>(acc, q, da0, db0, zoff); \
    break;
      TC2_ROUND_VARIANT(1u) TC2_ROUND_VARIANT(2u) TC2_ROUND_VARIANT(3u) TC2_ROUND_VARIANT(4u) TC2_ROUND_VARIANT(5u)
      TC2_ROUND_VARIANT(6u) TC2_ROUND_VARIANT(7u) TC2_ROUND_VARIANT(8u) TC2_ROUND_VARIANT(9u) TC2_ROUND_VARIANT(10u)
      TC2_ROUND_VARIANT(11u) TC2_ROUND_VARIANT(12u) TC2_ROUND_VARIANT(13u) TC2_ROUND_VARIANT(14u) TC2_ROUND_VARIANT(15u)
#undef TC2_ROUND_VARIANT
      // an empty set (rejected by the validator) would commit a group without an MMA: ptxas would add an empty HGMMA
      default: __builtin_unreachable();
    }
  }
}

// Drop the op bytes of one round (MAXB of them) from the front of the op queue (the MMA record's words 2..7).
template <int MAXB>
__device__ __forceinline__ void tc2_pop_round(uint32_t (&q)[6]) {
  using Ops = TcMmaRec::Ops;
  static_assert(Ops::WORDS == 6, "the op queue holds every op word");
  if constexpr (MAXB >= Ops::PER_WORD) {
#pragma unroll
    for (int i = 0; i < 6; ++i) q[i] = (i + MAXB / Ops::PER_WORD < 6) ? q[i + MAXB / Ops::PER_WORD] : 0u;
  } else {
#pragma unroll
    for (int i = 0; i < 5; ++i) q[i] = __funnelshift_r(q[i], q[i + 1], Ops::BITS * MAXB);
    q[5] >>= Ops::BITS * MAXB;
  }
}

#ifdef DGAN_PROBE
// Developer build only (-DDGAN_PROBE): per kernel instantiation and CTA, summed over launches: cycles from the PDL wait to
// the end of the CTA's work, launches, cycles from kernel entry to the PDL wait, cycles the first consumer warp waited
// for operands.  [4] cycles of the set-up (kernel entry to the PDL trigger), [5] / [6] %globaltimer (ns) at kernel entry
// / at the end of the CTA's work in the LAST launch, [7] %globaltimer when the CTA's first operands had landed.
// Where the first consumer warp's cycles go, besides the operand wait [3]: [8] issuing a step's MMAs (full barrier
// passed -> last round waited for, minus [9]; the previous step's release included), [9] the wgmma_wait1 after each
// round, [10] the wgmma_wait0 at the end of each item, [11] the item epilogues (registers -> global memory, momentum
// tail included; [8] excludes [12]).  What is left of the warp's cycles after those spans: [12] record wait (full barrier
// passed -> the step's MMA record read from shared memory and first used), [13] item head (end of the previous item's
// epilogue, or the PDL wait, -> the first step's operand wait), [14] end wait (end of the last epilogue -> every warp of
// the CTA has finished, the producer's drain included).  [15] steps the CTA ran.  Inside the epilogues [11]: [16] waiting
// for the epilogue's global inputs (mask words, bias, image and weight pairs: from the point a unit or accumulator needs
// them to their arrival), [17] waiting for a staging buffer of the TMA store (bulk_wait_read1).  Inside the TMA-store
// epilogues, per 64-column unit: [18] the register work (bias, ReLU or mask, fp16 conversion, and in the ReLU kinds the
// mask words: packing, combining across the quad, storing), [19] writing the staging buffer, [20] the
// fence.proxy.async before the TMA store.
constexpr int TC2_PROBE_WORDS = 21;
__device__ unsigned long long g_tc2_probe[48][160][TC2_PROBE_WORDS];
__device__ __forceinline__ unsigned long long probe_gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// clock64() once the load that produces record word 0 `w0` has returned: the clock read is predicated on a bit of the
// word (bit 31, which no record sets), so it cannot be scheduled ahead of the load's arrival.
__device__ __forceinline__ long long probe_clock_after(uint32_t w0) {
  long long t;
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ge.s32 p, %1, 0;\n\tmov.u64 %0, 0;\n\t@p mov.u64 %0, %%clock64;\n\t}" : "=l"(t) : "r"(w0) : "memory");
  return t;
}
// clock64() once `v` has arrived, whatever its bits: both predicated reads depend on it.
__device__ __forceinline__ long long probe_clock_after64(unsigned long long v) {
  long long t;
  asm volatile("{\n\t.reg .pred p;\n\tsetp.eq.u64 p, %1, 0;\n\t@p mov.u64 %0, %%clock64;\n\t@!p mov.u64 %0, %%clock64;\n\t}"
               : "=l"(t) : "l"(v) : "memory");
  return t;
}
__device__ __forceinline__ unsigned long long probe_bits(float2 v) {
  return ((unsigned long long)__float_as_uint(v.y) << 32) | __float_as_uint(v.x);
}
// Keys 0 - 39: (N class) * 8 + epilogue; 40 - 43: the Huber final kinds, one key each (tools/probe_step.py decodes both).
__host__ __device__ constexpr int tc2_probe_key(int n_tile, int epi, int out_bytes) {
  if (epi >= EPI_FINAL_SIGMOID1_H) return 40 + epi - EPI_FINAL_SIGMOID1_H;
  return (n_tile == 256 ? 0 : n_tile == 128 ? 1 : n_tile == 64 ? 2 : n_tile == 48 ? 3 : 4) * 8 + (out_bytes == 4 ? 6 : (epi < 4 ? epi : epi - 4));
}
#endif

template <int N_TILE, int MAXB, int KSUB, int EPI, typename TOUT>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(TC2_THREADS, 1)
tc_bsgemm2_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                  const __grid_constant__ CUtensorMap tm_out,
                  const TcItem2* __restrict__ items, const TcRec* __restrict__ stream_p,
                  const TcRec* __restrict__ stream_m, const __grid_constant__ Tc2Heads heads,
                  const int* __restrict__ eitems, int n_slots,
                  TOUT* __restrict__ out, int n_pad, const float* __restrict__ bias, int bias_pstride, const TcFinalArgs fa) {
  using Cfg = Tc2Cfg<N_TILE, MAXB, KSUB, EPI, (int)sizeof(TOUT)>;
  constexpr bool TMA_EPI = Cfg::TMA_EPI;
  constexpr bool HUBER = (EPI == EPI_FINAL_SIGMOID1_H || EPI == EPI_FINAL_TANH3_H || EPI == EPI_FINAL_SIGMOID1_WH ||
                          EPI == EPI_FINAL_TANH3_WH);
  constexpr bool WEIGHTED = (EPI == EPI_FINAL_SIGMOID1_W || EPI == EPI_FINAL_TANH3_W || EPI == EPI_FINAL_SIGMOID1_WH ||
                             EPI == EPI_FINAL_TANH3_WH);
  constexpr bool FINAL = tc_final_epi(EPI);
  constexpr bool SIGMOID1 = (EPI == EPI_FINAL_SIGMOID1 || EPI == EPI_FINAL_SIGMOID1_W || EPI == EPI_FINAL_SIGMOID1_H ||
                             EPI == EPI_FINAL_SIGMOID1_WH);
  constexpr bool HAS_BIAS = (EPI == EPI_BIAS_RELU || EPI == EPI_BIAS);
  constexpr int B_TILE = Cfg::B_TILE, A_BYTES = Cfg::A_BYTES;
  constexpr int PRODUCER = TC2_CONSUMERS / 32;     // warp index of the TMA producer
  extern __shared__ uint8_t smem_raw[];
#ifdef DGAN_PROBE
  const long long probe_t_start = clock64();
  const unsigned long long probe_g_start = probe_gtime();
  long long probe_wait_full = 0, probe_issue = 0, probe_wait1 = 0, probe_wait0 = 0, probe_epi = 0, probe_in = 0, probe_stage = 0;
  long long probe_regs = 0, probe_sts = 0, probe_fence = 0;
  unsigned probe_rec = 0, probe_head = 0, probe_steps = 0;     // 32-bit cycle counts: a launch is far shorter than 2^32 cycles
#endif
  const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t zero_base = smem_base + Cfg::RING_BYTES;           // the all-zero weight tile
  const uint32_t epi_base = zero_base + Cfg::ZERO_BYTES;            // output staging: 4 KB per consumer warp
  const uint32_t stg_base = epi_base + Cfg::EPI_BYTES;              // producer ring of TcRec
  const uint32_t bar_base = stg_base + TC2_STAGING_BYTES;
  // full[s] @ +8s (s<8), empty[s] @ +64+8s, momentum-tail flag @ +200, MMA record of the step in barrier slot s @ +256+32s
  const uint32_t bar_full = bar_base, bar_empty = bar_base + 64, mrec_base = bar_base + 256;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t rank = ptx::cluster_ctarank();
  const int pair = blockIdx.x >> 1, n_pairs = gridDim.x >> 1;
  const uint32_t rbeg = heads.off[pair], rend = heads.off[pair + 1];

  // The schedule tables are constants: the producer's first records are requested before anything else, so that their
  // latency overlaps the set-up below (and, for CTAs that start early, the previous kernel's tail).
  uint4 mine = make_uint4(0, 0, 0, 0);
  if (warp == PRODUCER) {
    if (2 * rbeg + lane < 2 * rend) mine = __ldg(reinterpret_cast<const uint4*>(stream_p + rbeg) + lane);   // lane = 16-byte half
    if (lane == 0) {
      ptx::prefetch_tmap(&tm_a);
      ptx::prefetch_tmap(&tm_b);
      if (TMA_EPI) ptx::prefetch_tmap(&tm_out);
      for (int s = 0; s < TC2_NSLOT; ++s) {
        ptx::mbar_init(bar_full + 8 * s, 1);                   // producer's arrive.expect_tx
        ptx::mbar_init(bar_empty + 8 * s, 2 * TC2_CONSUMERS / 32);   // one arrive per consumer warp of both CTAs
      }
      ptx::fence_barrier_init();
    }
  }
  if constexpr (Cfg::ZERO_BYTES > 0 && tc2_issues_zero_ops(MAXB, KSUB)) {    // only where zero-tile ops read it
    if (threadIdx.x < TC2_CONSUMERS) {
      for (uint32_t i = threadIdx.x; i < (uint32_t)Cfg::ZERO_BYTES / 16u; i += TC2_CONSUMERS) ptx::st_shared_v4(zero_base + 16u * i, 0u, 0u, 0u, 0u);
      ptx::fence_proxy_async_smem();           // the MMAs read it through the async proxy
    }
  }
  ptx::cluster_sync();                         // barriers of BOTH CTAs initialised before any remote signal
  // everything above overlapped the previous kernel's tail (PDL); from here on we read what it wrote
#ifdef DGAN_PROBE
  const long long probe_t_entry = clock64();
#endif
  pdl_launch_dependents();
  pdl_wait();
#ifdef DGAN_PROBE
  const long long probe_t_go = clock64();
  unsigned probe_h0 = (unsigned)probe_t_go;     // start of the item head
  bool probe_new_item = true;
#endif

  if (warp >= PRODUCER) {
    // ===================== producer warpgroup =====================
    // It hands registers to the consumer warpgroups.  Only its first warp has work; the other three wait at the final
    // cluster barrier.
    ptx::setmaxnreg_dec<TC2_PRODUCER_REGS>();
    if (warp == PRODUCER) {
      // The whole warp walks the step list convergently; every table value is loaded from a warp-uniform address, and
      // one elected lane issues.
      const TcRec* __restrict__ stream = stream_p;
      uint32_t it = 0;
      const uint32_t ring = stg_base;
      for (uint32_t base = rbeg; base < rend; base += TC2_REC_BATCH) {
        ptx::st_shared_v4(ring + lane * 16u, mine.x, mine.y, mine.z, mine.w);
        __syncwarp();
        if (2 * (base + TC2_REC_BATCH) + lane < 2 * rend) mine = __ldg(reinterpret_cast<const uint4*>(stream + base + TC2_REC_BATCH) + lane);
        const uint32_t cnt = min((uint32_t)TC2_REC_BATCH, rend - base);
        for (uint32_t i = 0; i < cnt; ++i, ++it) {
          const uint4 r0 = ptx::ld_shared_v4(ring + i * 32u);
          const uint2 r1 = ptx::ld_shared_v2(ring + i * 32u + 16u);
          const uint32_t slot = it & (TC2_NSLOT - 1);
          using P = TcProducerRec;
          const int kc = P::Kc::get(r0.x), nA = P::NA::get(r0.x), nB = P::NB::get(r0.x);
          // not P::Dep::get(r0.x): the same value, but ptxas then orders this warp's record loads differently
          const uint32_t dep = (r0.x >> P::Dep::shift) & P::Dep::mask;
          const int row0 = (2 * (int)P::Mp::get(r0.y) + (int)rank) * kRowTile;
          if (it >= dep) ptx::mbar_wait(bar_empty + 8 * ((it - dep) & (TC2_NSLOT - 1)), ((it - dep) >> 3) & 1);   // step it-dep consumed
          // implied by the wait above (steps are consumed in order); observing every phase of this slot exactly once
          // before it is re-armed keeps the barrier protocol simple to check
          if (dep != TC2_NSLOT && it >= TC2_NSLOT) ptx::mbar_wait(bar_empty + 8 * slot, ((it - TC2_NSLOT) >> 3) & 1);
          const uint32_t full = bar_full + 8 * slot;
          const uint32_t sa = smem_base + (P::Off::get(r0.x) << 10);
          if (ptx::elect_one()) {
            ptx::mbar_expect_tx(full, (uint32_t)(nA * A_BYTES + nB * B_TILE) + (uint32_t)sizeof(TcRec));
            // the consumers' record of this step (this CTA's own copy, not multicast).  Its slot is free: step it - 8 is
            // consumed (waited for above), and a consumer warp holds a record in registers before it says so
            ptx::bulk_load(mrec_base + slot * (uint32_t)sizeof(TcRec), stream_m + rbeg + it, (uint32_t)sizeof(TcRec), full);
#pragma unroll
            for (int a = 0; a < TC2_MAX_A; ++a) {
              if (a >= nA) break;
              const int p = (int)P::Pix::get(a < P::Pix::PER_WORD ? r0.z : r0.w, a);
              if constexpr (KSUB == 4) {
                ptx::tma_load_3d(sa + a * A_BYTES, &tm_a, full, kc * 64, row0, p);
              } else {
#pragma unroll
                for (int k = 0; k < KSUB; ++k)           // one 16-channel box per sub-tile
                  ptx::tma_load_3d(sa + a * A_BYTES + k * Cfg::A_SUB, &tm_a, full, (kc * KSUB + k) * 16, row0, p);
              }
            }
            const uint32_t sb = sa + nA * A_BYTES;
#pragma unroll
            for (int b = 0; b < TC2_MAX_BSLOTS; ++b) {     // this CTA's half of each weight tile, into both CTAs
              if (b >= nB) break;
              const uint32_t t = P::Tile::get(b < P::Tile::PER_WORD ? r1.x : r1.y, b);
              if constexpr (KSUB == 4) {
                ptx::tma_load_3d_mc2(sb + b * B_TILE + rank * (B_TILE / 2), &tm_b, full, kc * 64, (int)rank * (N_TILE / 2), (int)t);
              } else {
#pragma unroll
                for (int k = 0; k < KSUB; ++k)           // this CTA's half of every sub-tile
                  ptx::tma_load_3d_mc2(sb + b * B_TILE + k * Cfg::B_SUB + rank * (Cfg::B_SUB / 2), &tm_b, full, (kc * KSUB + k) * 16,
                                       (int)rank * (N_TILE / 2), (int)t);
              }
            }
          }
          __syncwarp();
        }
        __syncwarp();
      }
      // drain: the last steps' "consumed" signals are otherwise never observed (nobody leaves while MMAs still read smem)
      for (uint32_t j = it > TC2_NSLOT ? it - TC2_NSLOT : 0; j < it; ++j) ptx::mbar_wait(bar_empty + 8 * (j & (TC2_NSLOT - 1)), (j >> 3) & 1);
    }
  } else {
    // ===================== consumer warpgroups (warps 0..7) =====================
    ptx::setmaxnreg_inc<TC2_CONSUMER_REGS>();
    const int wg = warp >> 2, wl = warp & 3;
    const int r_lo = wg * 64 + wl * 16 + (lane >> 2);      // this thread's rows of the 128-row tile: r_lo and r_lo + 8
    float acc[Cfg::ACC_REGS];
#pragma unroll
    for (int i = 0; i < Cfg::ACC_REGS; ++i) acc[i] = 0.f;
    uint32_t item_count = 0, store_count = 0;
    uint32_t ri = rbeg, it = 0;
    // What the epilogue reads besides the accumulators is requested before the MMAs it follows, so that no global
    // round trip sits between the item's last MMA and its output.  The item descriptors run one item ahead: item i's
    // word, window size and pixels arrive during item i-1, and item i's head requests from them, without waiting, its
    // mask words, its pixel's bias or its image pairs; the epilogue of item i reads registers and shared memory.
    // (Each TMA store is preceded by fence.proxy.async, which waits for ALL of the warp's outstanding loads: what is
    // requested at an item's head has long arrived by its epilogue, nothing is requested later.)
    auto item_desc = [&](int e, int& n, uint32_t& qm) {     // window size and pixels of item word e (-1: none)
      n = 0; qm = 0u;
      if (e < 0) return;
      const TcItem2* ip = items + tc2_item_window(e);
      n = (int)__ldg(&ip->n_acc);
      if (lane < 16) qm = (uint32_t)__ldg(&ip->q[lane]);
    };
    int e_cur = tc2_item_at(eitems, 0, pair, n_pairs, n_slots), e_nx = tc2_item_at(eitems, 1, pair, n_pairs, n_slots), n_acc_cur;
    uint32_t q_cur;
    item_desc(e_cur, n_acc_cur, q_cur);
    // Per-channel bias (the launch validator gives a per-pixel bias only to N = 256): copied once per CTA into the zero
    // tile, which these instantiations keep but never write (tc2_issues_zero_ops), and read from there by the epilogue.
    constexpr bool BIAS_CH = HAS_BIAS && TMA_EPI && N_TILE < 256, BIAS_PX = HAS_BIAS && TMA_EPI && !BIAS_CH;
    static_assert(!BIAS_CH || (Cfg::ZERO_BYTES >= N_TILE * 4 && !tc2_issues_zero_ops(MAXB, KSUB)), "the bias copy's space");
    static_assert(!BIAS_PX || MAXB == 1, "a per-pixel bias is held for one accumulator");
    if constexpr (BIAS_CH) {
      if (threadIdx.x < N_TILE / 2) {     // float2: the epilogue's loads needed 8-byte alignment only
        const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias) + threadIdx.x);
        ptx::st_shared_u32(zero_base + 8u * threadIdx.x, __float_as_uint(b2.x));
        ptx::st_shared_u32(zero_base + 8u * threadIdx.x + 4u, __float_as_uint(b2.y));
      }
      ptx::named_bar_sync(4, TC2_CONSUMERS);
    }
    // final kinds: output channels, the bias of each, pairs per row and accumulator
    constexpr int CO = SIGMOID1 ? 1 : 3, FJ = FINAL ? N_TILE / 8 : 1;
    // CelebA's weighted kind has no registers for a second set of pairs (it would spill): it requests the pairs of a
    // row of an accumulator where it uses them.
    constexpr bool FINAL_PREFETCH = !(WEIGHTED && N_TILE > 32);
    constexpr int FINAL_HELD = FINAL && N_TILE <= 32 && !(WEIGHTED && MAXB > 4) ? MAXB : 1;
    const int hwc = fa.w_out * fa.w_out * CO;
    float bsv[CO];
    if constexpr (FINAL) {
#pragma unroll
      for (int co = 0; co < CO; ++co) bsv[co] = __ldg(bias + co);
    }
    while (ri < rend) {
      const int item_e = e_cur, n_acc = n_acc_cur;
      const uint32_t q_mine = q_cur;
      const int mp = tc2_item_mp(item_e);
      const int tile_row0 = (2 * mp + (int)rank) * kRowTile;
      const size_t n_lo = (size_t)(tile_row0 + r_lo);
      // EPI_MASK: the item's mask words, 8 per quad (the four lanes holding the same two rows): lane k of the quad
      // requests both row words of unit k (accumulator k / G, 64-column group k % G), the epilogue shuffles them.
      constexpr int G_UNITS = TMA_EPI ? N_TILE / 64 : 1;
      static_assert(EPI != EPI_MASK || MAXB * G_UNITS == 4, "one mask unit per lane of a quad");
      unsigned long long mk_pre[2] = {~0ull, ~0ull};
      if constexpr (EPI == EPI_MASK) {
        const int ua = (lane & 3) / G_UNITS, ug = (lane & 3) % G_UNITS;
        const size_t qa = (size_t)__shfl_sync(0xffffffffu, q_mine, ua);
        if (ua < n_acc) {
#pragma unroll
          for (int h = 0; h < 2; ++h) mk_pre[h] = __ldg(fa.mb_in + (qa * n_pad + n_lo + 8 * h) * (size_t)(fa.out_ld >> 6) + ug);
        }
      }
      // N = 256 (one accumulator): the bias of its pixel, which may be per pixel (Linear.fwd).  The lanes with the same
      // lane % 4 need the same columns: lane L requests column pair (g * 8 + L / 4) * 8 + (L % 4) * 2 of every
      // 64-column group g, and the epilogue shuffles them.
      float2 bias_px[BIAS_PX ? G_UNITS : 1];
      if constexpr (BIAS_PX) {
        const size_t q0 = (size_t)__shfl_sync(0xffffffffu, q_mine, 0);
        if (n_acc > 0) {
#pragma unroll
          for (int g = 0; g < G_UNITS; ++g)
            bias_px[g] = __ldg(reinterpret_cast<const float2*>(bias + q0 * bias_pstride + (g * 8 + (lane >> 2)) * 8 + (lane & 3) * 2));
        }
      }
      // Final kinds: the image (and weight) pairs of row r_lo + 8 h of accumulator a.  With N = 16 every accumulator's
      // are requested now (FINAL_HELD = MAXB sets of registers).  Otherwise accumulator 0's are requested now and
      // accumulator a + 1's row h while accumulator a's row h is used: a row of 16 columns is shorter than a round trip.
      auto final_pairs = [&](int a, int h, float2 (&xv)[FJ], float2 (&wv)[FJ]) {
        const int blk = (int)__shfl_sync(0xffffffffu, q_mine, a);
        const int by = blk / fa.nbx, bx = blk % fa.nbx;
        const int img = min((int)((n_lo + 8 * h) / fa.R), fa.B - 1);
#pragma unroll
        for (int j = 0; j < FJ; ++j) {
          const int col = j * 8 + (lane & 3) * 2;     // (li * 4 + lj) * CO + co of the 4x4 block
          const int li = col / (4 * CO), e = col % (4 * CO);
          const size_t off = (size_t)((4 * by + li) * fa.w_out + 4 * bx) * CO + e;
          xv[j] = make_float2(0.f, 0.f);
          if (fa.x != nullptr) xv[j] = __ldg(reinterpret_cast<const float2*>(fa.x + (size_t)img * hwc + off));
          wv[j] = make_float2(1.f, 1.f);      // the weight pair next to the image pair (weighted kinds)
          if (WEIGHTED) wv[j] = __ldg(reinterpret_cast<const float2*>(fa.xw + (size_t)img * hwc + off));
        }
      };
      float2 xp[FINAL_HELD][2][FJ], wp[FINAL_HELD][2][FJ];
      if constexpr (FINAL && FINAL_PREFETCH) {
#pragma unroll
        for (int a = 0; a < FINAL_HELD; ++a) {
          if (a >= n_acc) break;
          final_pairs(a, 0, xp[a][0], wp[a][0]);
          final_pairs(a, 1, xp[a][1], wp[a][1]);
        }
      }
      // the next item's window size and pixels (its word was requested one item earlier), and the word after it
      item_desc(e_nx, n_acc_cur, q_cur);
      e_cur = e_nx;
      e_nx = tc2_item_at(eitems, (int)item_count + 2, pair, n_pairs, n_slots);
      uint32_t flags;
      do {    // the steps of one item
        const uint32_t slot = it & (TC2_NSLOT - 1), phase = (it >> 3) & 1;
#ifdef DGAN_PROBE
        const long long probe_w0 = clock64();
        if (probe_new_item) probe_head += (unsigned)probe_w0 - probe_h0;
        probe_new_item = false;
#endif
        ptx::mbar_wait(bar_full + 8 * slot, phase);
#ifdef DGAN_PROBE
        const long long probe_w1 = clock64();
        probe_wait_full += probe_w1 - probe_w0;
        if (it == 0 && threadIdx.x == 0) g_tc2_probe[tc2_probe_key(N_TILE, EPI, (int)sizeof(TOUT))][blockIdx.x][7] = probe_gtime();
#endif
        // the step's MMA record arrived with its operands, in the barrier slot's record slot: no global load in this loop
        const uint4 r0 = ptx::ld_shared_v4_ordered(mrec_base + slot * (uint32_t)sizeof(TcRec));
        const uint4 r1 = ptx::ld_shared_v4_ordered(mrec_base + slot * (uint32_t)sizeof(TcRec) + 16u);
        flags = TcMmaRec::Flags::get(r0.x);
#ifdef DGAN_PROBE
        const unsigned probe_rec_step = (unsigned)probe_clock_after(r0.x) - (unsigned)probe_w1;
        probe_rec += probe_rec_step;
#endif
        const int nA = TcMmaRec::NA::get(r0.x), n_rounds = TcMmaRec::Rounds::get(r0.x);
        const uint32_t sa = smem_base + (TcMmaRec::Off::get(r0.x) << 10);
        // this warpgroup's 64 rows of the A tiles (of their first sub-tile when narrow)
        const uint64_t da0 = KSUB == 4 ? make_smem_desc_sw128(sa + (uint32_t)wg * 64u * 128u) : make_smem_desc_sw32(sa + (uint32_t)wg * 64u * 32u);
        const uint32_t sb = sa + (uint32_t)nA * A_BYTES;
        const uint64_t db0 = KSUB == 4 ? make_smem_desc_sw128(sb) : make_smem_desc_sw32(sb);
        const uint32_t zoff = (zero_base - sb) >> 4;    // zero tile after the ring: always above the step's B slots
        uint32_t q[6] = {r0.z, r0.w, r1.x, r1.y, r1.z, r1.w};
#ifdef DGAN_PROBE
        long long probe_step_wait = 0;
#endif
        ptx::fence_operands(acc);
        ptx::wgmma_fence();
        // One wgmma group per round, and one group in flight.  ptxas closes a hardware group at the end of every
        // iteration of this run-time loop whatever the commits say, so a single commit per step would make its wait
        // drain the whole step and idle the tensor pipe at every step boundary.
        for (int r = 0; r < n_rounds; ++r) {
          tc2_mma_round<N_TILE, Cfg::MAXB, KSUB>(acc, q, da0, db0, zoff);    // commits the round's group
          tc2_pop_round<Cfg::MAXB>(q);
#ifdef DGAN_PROBE
          const long long probe_c0 = clock64();
#endif
          ptx::wgmma_wait1();           // every group but this round's has retired
#ifdef DGAN_PROBE
          probe_step_wait += clock64() - probe_c0;
#endif
          if (r == 0) {
            __syncwarp();
            // this warp's MMAs no longer read the previous step's region (the previous item's last step was released
            // after its wgmma_wait0 below)
            if (!(flags & TcMmaRec::FIRST) && lane < 2) ptx::mbar_arrive_cluster(bar_empty + 8 * ((it - 1) & (TC2_NSLOT - 1)), (uint32_t)lane);
          }
        }
        ptx::fence_operands(acc);
#ifdef DGAN_PROBE
        probe_wait1 += probe_step_wait;
        probe_issue += clock64() - probe_w1 - probe_step_wait - probe_rec_step;
#endif
        ++ri; ++it;
      } while (!(flags & TcMmaRec::LAST));
      // the epilogue reads the registers: wait for all MMAs, then release the item's last step
#ifdef DGAN_PROBE
      const long long probe_d0 = clock64();
#endif
      ptx::wgmma_wait0();
      ptx::fence_operands(acc);
#ifdef DGAN_PROBE
      const long long probe_e0 = clock64();
      probe_wait0 += probe_e0 - probe_d0;
#endif
      __syncwarp();
      if (lane < 2) ptx::mbar_arrive_cluster(bar_empty + 8 * ((it - 1) & (TC2_NSLOT - 1)), (uint32_t)lane);

      // ---- epilogue of the item: accumulator registers -> (bias | ReLU | mask | last layer) -> global memory.
      //      Register i of accumulator a holds column (i % (N_TILE/2)) / 4 * 8 + (lane % 4) * 2 + (i % 2) of row
      //      r_lo + 8 * ((i / 2) % 2) (the m64nNk16 accumulator fragment).
      auto q_of = [&](int a) { return (int)__shfl_sync(0xffffffffu, q_mine, a); };
      if constexpr (FINAL) {
#pragma unroll
        for (int a = 0; a < Cfg::MAXB; ++a) {
          if (a >= n_acc) break;
          const int blk = q_of(a);
          const int by = blk / fa.nbx, bx = blk % fa.nbx;
#ifdef DGAN_PROBE
          const long long probe_a0 = clock64();
#endif
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float2 xa[FJ], wa[FJ];
            if constexpr (FINAL_PREFETCH) {
#pragma unroll
              for (int j = 0; j < FJ; ++j) { xa[j] = xp[a % FINAL_HELD][h][j]; wa[j] = wp[a % FINAL_HELD][h][j]; }
              if (FINAL_HELD == 1 && a + 1 < Cfg::MAXB && a + 1 < n_acc) final_pairs(a + 1, h, xp[0][h], wp[0][h]);
            } else {
              final_pairs(a, h, xa, wa);
            }
#ifdef DGAN_PROBE
            if (h == 0) probe_in += probe_clock_after64(probe_bits(xa[0]) ^ probe_bits(wa[0])) - probe_a0;
#endif
            const size_t n = n_lo + 8 * h;
            float lsum = 0.f;
#pragma unroll
            for (int j = 0; j < N_TILE / 8; ++j) {
              const int col = j * 8 + (lane & 3) * 2;     // (li * 4 + lj) * CO + co of the 4x4 block
              const int li = col / (4 * CO), e = col % (4 * CO);
              const size_t off = (size_t)((4 * by + li) * fa.w_out + 4 * bx) * CO + e;
              const float2 xv = xa[j], wv = wa[j];
              float yv[2], dv[2];
#pragma unroll
              for (int c = 0; c < 2; ++c) {
                const float pre = acc[a * (N_TILE / 2) + j * 4 + h * 2 + c] + bsv[(e + c) % CO];
                float yy, dact;
                if (SIGMOID1) { yy = __fdividef(1.f, 1.f + __expf(-pre)); dact = yy * (1.f - yy); }
                else { const float t = __expf(-2.f * fabsf(pre)); yy = copysignf(__fdividef(1.f - t, 1.f + t), pre); dact = 1.f - yy * yy; }
                yv[c] = yy;
                float d = 0.f;
                if (HUBER) {              // c = psi_delta(d), e = w c: the loss part takes e (2 d - c), d(pre) e act'(y)
                  d = yy - (c ? xv.y : xv.x);
                  const float cl = fabsf(d) > fa.huber ? copysignf(fa.huber, d) : d;
                  const float ew = WEIGHTED ? (c ? wv.y : wv.x) * cl : cl;
                  lsum = fmaf(ew, 2.f * d - cl, lsum);
                  d = ew;
                } else if (WEIGHTED) {    // e = w d: the loss part takes e d, d(pre) e act'(y)
                  d = yy - (c ? xv.y : xv.x);
                  const float ew = (c ? wv.y : wv.x) * d;
                  lsum = fmaf(ew, d, lsum);
                  d = ew;
                } else if (fa.x != nullptr) { d = yy - (c ? xv.y : xv.x); lsum = fmaf(d, d, lsum); }
                dv[c] = d * dact * fa.gscale;
              }
              if (fa.write_y) *reinterpret_cast<float2*>(fa.y + n * hwc + off) = make_float2(yv[0], yv[1]);
              // d(pre) block tensor [n_blocks][n_pad][16 * CO]: the last layer's backward reads it as its narrow operand
              if (fa.x != nullptr)
                *reinterpret_cast<uint32_t*>(reinterpret_cast<__half*>(out) + ((size_t)blk * n_pad + n) * N_TILE + col) = pack_half2(dv[0], dv[1]);
            }
            lsum += __shfl_xor_sync(0xffffffffu, lsum, 1);
            lsum += __shfl_xor_sync(0xffffffffu, lsum, 2);
            // the loss is consumed after the last forward only
            if (fa.x != nullptr && fa.write_y && (lane & 3) == 0) fa.loss_part[(size_t)blk * n_pad + n] = lsum;
          }
        }
      } else if constexpr (TMA_EPI) {
        // 64-column units: registers -> fp16 -> this warp's 16-row slice of a 128B-swizzled tile -> one TMA store
        constexpr int G = N_TILE / 64;                 // 64-column groups per accumulator
        const int GT = fa.out_ld >> 6;                 // 64-column groups per output row (mask words)
        const int row_w = tile_row0 + wg * 64 + wl * 16;
        const uint32_t s_warp = epi_base + (uint32_t)warp * 4096u;
        const uint32_t l2 = 2u * (uint32_t)(lane & 3);  // this lane's first column in each 8-column chunk
        // stmatrix: lane L gives the address of row L % 8 of 8x8 matrix L / 8, and matrix m of store p is the chunk
        // (row half h = m % 2, column chunk j = 2p + m / 2) of the 128B-swizzled slice, chunk j of row r at (j ^ r) * 16
        const uint32_t sm_row = (uint32_t)(lane & 7) + 8u * (uint32_t)((lane >> 3) & 1);
        const uint32_t sm_x = (((uint32_t)(lane >> 4) ^ (uint32_t)(lane & 7)) << 4);
        // EPI_BIAS_RELU: lane k of a quad ends a unit holding 32-bit half k % 2 of row r_lo + 8 (k / 2)'s mask word; the
        // words are stored after the item's last TMA store, so that no global store precedes a fence.proxy.async.
        uint32_t mw[Cfg::MAXB * G];
#pragma unroll
        for (int a = 0; a < Cfg::MAXB; ++a) {
          if (a >= n_acc) break;
          const int q = q_of(a);
#pragma unroll
          for (int g = 0; g < G; ++g) {
#ifdef DGAN_PROBE
            const long long probe_u0 = clock64(), probe_in0 = probe_in;
#endif
            // EPI_MASK: the unit's bits of this lane, bit 8j + c of row h's word in column 8j + l2 + c, placed as the
            // sign bits of bytes (c = 0: keep7, c = 1: keep6; 32-bit halves lo: j < 4, hi: j >= 4)
            uint32_t keep7[2][2], keep6[2][2];
            if constexpr (EPI == EPI_MASK) {
              unsigned long long mk[2];
#pragma unroll
              for (int h = 0; h < 2; ++h) mk[h] = __shfl_sync(0xffffffffu, mk_pre[h], (lane & ~3) | (a * G + g));
#ifdef DGAN_PROBE
              probe_in += probe_clock_after64(mk[0] ^ mk[1]) - probe_u0;
#endif
#pragma unroll
              for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int hi = 0; hi < 2; ++hi) {
                  const uint32_t w = (uint32_t)(mk[h] >> (32 * hi));
                  keep7[h][hi] = w << (7u - l2);
                  keep6[h][hi] = w << (6u - l2);
                }
            }
            uint32_t pk[2][8];
            uint32_t bits[2][2] = {{0u, 0u}, {0u, 0u}};     // EPI_BIAS_RELU: [row half][32-bit half], lane's bits at 8j + c
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int cl = j * 8 + (lane & 3) * 2;   // column within the 64-column group
              float2 bv = make_float2(0.f, 0.f);
              if constexpr (BIAS_CH) {
                const uint2 b2 = ptx::ld_shared_v2(zero_base + (uint32_t)(g * 64 + cl) * 4u);
                bv = make_float2(__uint_as_float(b2.x), __uint_as_float(b2.y));
              }
              if constexpr (BIAS_PX) {
                bv.x = __shfl_sync(0xffffffffu, bias_px[g].x, j * 4 + (lane & 3));
                bv.y = __shfl_sync(0xffffffffu, bias_px[g].y, j * 4 + (lane & 3));
              }
#ifdef DGAN_PROBE
              if (HAS_BIAS && j == 0) probe_in += probe_clock_after64(probe_bits(bv)) - probe_u0;
#endif
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                float v0 = acc[a * (N_TILE / 2) + (g * 8 + j) * 4 + h * 2];
                float v1 = acc[a * (N_TILE / 2) + (g * 8 + j) * 4 + h * 2 + 1];
                if (HAS_BIAS) { v0 += bv.x; v1 += bv.y; }
                if (EPI == EPI_BIAS_RELU) {
                  // the mask bit is (value after ReLU > 0), i.e. v > 0 (false for NaN and -0, which fmaxf makes 0); a
                  // predicated add of the bit at a compile-time position, shifted to this lane's columns once per unit
                  const uint32_t b = 8u * (uint32_t)(j & 3);
                  if (v0 > 0.f) bits[h][j >> 2] |= 1u << b;
                  if (v1 > 0.f) bits[h][j >> 2] |= 2u << b;
                  v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f);
                }
                pk[h][j] = pack_half2(v0, v1);
                // a masked-out value becomes +0
                if (EPI == EPI_MASK) pk[h][j] &= ptx::prmt(keep7[h][j >> 2], keep6[h][j >> 2], 0xCC88u + 0x1111u * (uint32_t)(j & 3));
              }
            }
            if constexpr (EPI == EPI_BIAS_RELU) {
              // the quad's words: lane k keeps row half k / 2 (exchange with lane k ^ 2), then 32-bit half k % 2 (k ^ 1)
              const bool up = (lane & 2) != 0, odd = (lane & 1) != 0;
              uint32_t k0 = (up ? bits[1][0] : bits[0][0]) << l2, k1 = (up ? bits[1][1] : bits[0][1]) << l2;
              const uint32_t s0 = (up ? bits[0][0] : bits[1][0]) << l2, s1 = (up ? bits[0][1] : bits[1][1]) << l2;
              k0 |= __shfl_xor_sync(0xffffffffu, s0, 2);
              k1 |= __shfl_xor_sync(0xffffffffu, s1, 2);
              mw[a * G + g] = (odd ? k1 : k0) | __shfl_xor_sync(0xffffffffu, odd ? k0 : k1, 1);
            }
            const uint32_t buf = s_warp + (store_count & 1u) * 2048u;
#ifdef DGAN_PROBE
            const long long probe_s0 = probe_clock_after64((((unsigned long long)pk[0][7] << 32) | pk[1][7]) ^
                                                           (EPI == EPI_BIAS_RELU ? mw[a * G + g] : 0u));
            probe_regs += probe_s0 - probe_u0 - (probe_in - probe_in0);
#endif
            if (lane == 0) ptx::bulk_wait_read1();     // the store that used this buffer two units ago has read it
            __syncwarp();
#ifdef DGAN_PROBE
            const long long probe_s1 = clock64();
            probe_stage += probe_s1 - probe_s0;
#endif
#pragma unroll
            for (int p = 0; p < 4; ++p)
              ptx::stmatrix_x4(buf + sm_row * 128u + ((32u * (uint32_t)p) ^ sm_x), pk[0][2 * p], pk[1][2 * p], pk[0][2 * p + 1], pk[1][2 * p + 1]);
#ifdef DGAN_PROBE
            const long long probe_f0 = clock64();
            probe_sts += probe_f0 - probe_s1;
#endif
            ptx::fence_proxy_async_smem();
#ifdef DGAN_PROBE
            probe_fence += clock64() - probe_f0;
#endif
            __syncwarp();
            if (lane == 0) {
              ptx::tma_store_3d(&tm_out, buf, fa.col0 + g * 64, row_w, q);
              ptx::bulk_commit();
            }
            ++store_count;
          }
        }
        if (EPI == EPI_BIAS_RELU && fa.mb_out != nullptr) {
#ifdef DGAN_PROBE
          const long long probe_m0 = clock64();
#endif
          uint32_t* __restrict__ mb32 = reinterpret_cast<uint32_t*>(fa.mb_out);
          const size_t row = n_lo + 8 * ((lane >> 1) & 1);
#pragma unroll
          for (int a = 0; a < Cfg::MAXB; ++a) {
            if (a >= n_acc) break;
            const int q = q_of(a);
#pragma unroll
            for (int g = 0; g < G; ++g) mb32[(((size_t)q * n_pad + row) * GT + g) * 2 + (lane & 1)] = mw[a * G + g];
          }
#ifdef DGAN_PROBE
          probe_regs += clock64() - probe_m0;
#endif
        }
      } else {
        // fp32 outputs (BatchNorm pre-activations, the Linear backward's partial sums): straight from the registers
#pragma unroll
        for (int a = 0; a < Cfg::MAXB; ++a) {
          if (a >= n_acc) break;
          const int q = q_of(a);
#pragma unroll
          for (int j = 0; j < N_TILE / 8; ++j) {
            const int col = j * 8 + (lane & 3) * 2;
            float2 bv = make_float2(0.f, 0.f);
            if (HAS_BIAS) bv = __ldg(reinterpret_cast<const float2*>(bias + (size_t)q * bias_pstride + col));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float v0 = acc[a * (N_TILE / 2) + j * 4 + h * 2] + bv.x, v1 = acc[a * (N_TILE / 2) + j * 4 + h * 2 + 1] + bv.y;
              if (EPI == EPI_BIAS_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
              const size_t o = ((size_t)q * n_pad + n_lo + 8 * h) * fa.out_ld + col;
              if (sizeof(TOUT) == 4) *reinterpret_cast<float2*>(reinterpret_cast<float*>(out) + o) = make_float2(v0, v1);
              else *reinterpret_cast<uint32_t*>(reinterpret_cast<__half*>(out) + o) = pack_half2(v0, v1);
            }
          }
        }
      }
      if (EPI == EPI_NONE && sizeof(TOUT) == 4 && fa.m_counter != nullptr) {
        // ---- momentum in the tail of the split-K Linear backward.  Every consumer thread has stored its share of this
        //      item's partial sums; the CTA that completes the last partial of its 128-row tile applies the update
        //      (same arithmetic and summation order as momentum_kernel: parts 0, 1, 2, ...).
        const uint32_t flag_addr = bar_base + 200;
        const unsigned rt = 2u * (unsigned)mp + rank;
        __threadfence();
        ptx::named_bar_sync(3, TC2_CONSUMERS);
        if (threadIdx.x == 0) {
          const unsigned ticket = atomicAdd(fa.m_counter + rt, 1u);
          ptx::st_shared_u32(flag_addr, ticket == (unsigned)TC_LINEAR_SPLIT - 1u ? 1u : 0u);
        }
        ptx::named_bar_sync(3, TC2_CONSUMERS);
        if (ptx::ld_shared_u32(flag_addr) != 0u) {
          __threadfence();
          const float* __restrict__ gp = reinterpret_cast<const float*>(out);
          const size_t base = (size_t)rt * kRowTile * N_TILE;
          const int tid = threadIdx.x;
          // 4 float4 positions per thread in flight at a time (the loop is latency-bound: 6 L2 reads per position)
          constexpr int STRIDE = 4 * TC2_CONSUMERS, UNR = 4;
          for (int e0 = tid * 4; e0 < kRowTile * N_TILE; e0 += UNR * STRIDE) {
            float4 gs[UNR], vv[UNR], zz[UNR];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
              const size_t i = base + (size_t)(e0 + u * STRIDE);
              gs[u] = __ldcg(reinterpret_cast<const float4*>(gp + i));
              vv[u] = *reinterpret_cast<const float4*>(fa.mv + i);
              zz[u] = *reinterpret_cast<const float4*>(fa.mz + i);
            }
            float4 t[TC_LINEAR_SPLIT - 1][UNR];      // all partial sums of the 4 positions in flight together
#pragma unroll
            for (int pp = 1; pp < TC_LINEAR_SPLIT; ++pp)
#pragma unroll
              for (int u = 0; u < UNR; ++u)
                t[pp - 1][u] = __ldcg(reinterpret_cast<const float4*>(gp + base + (size_t)(e0 + u * STRIDE) + (size_t)pp * fa.m_count));
#pragma unroll
            for (int pp = 1; pp < TC_LINEAR_SPLIT; ++pp)      // fixed order: parts 0, 1, 2, 3 (as momentum_kernel)
#pragma unroll
              for (int u = 0; u < UNR; ++u) { gs[u].x += t[pp - 1][u].x; gs[u].y += t[pp - 1][u].y; gs[u].z += t[pp - 1][u].z; gs[u].w += t[pp - 1][u].w; }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
              const size_t i = base + (size_t)(e0 + u * STRIDE);
              float4 v4 = vv[u], z4 = zz[u];
              v4.x = fmaf(fa.m_mu, v4.x, fa.m_gmul * gs[u].x); v4.y = fmaf(fa.m_mu, v4.y, fa.m_gmul * gs[u].y);
              v4.z = fmaf(fa.m_mu, v4.z, fa.m_gmul * gs[u].z); v4.w = fmaf(fa.m_mu, v4.w, fa.m_gmul * gs[u].w);
              z4.x -= fa.m_lr * v4.x; z4.y -= fa.m_lr * v4.y; z4.z -= fa.m_lr * v4.z; z4.w -= fa.m_lr * v4.w;
              *reinterpret_cast<float4*>(fa.mv + i) = v4;
              *reinterpret_cast<float4*>(fa.mz + i) = z4;
              if (fa.mz_h != nullptr)
                *reinterpret_cast<uint2*>(fa.mz_h + i) = make_uint2(pack_half2(z4.x, z4.y), pack_half2(z4.z, z4.w));
            }
          }
          if (tid == 0) fa.m_counter[rt] = 0u;             // ready for the next launch
        }
      }
#ifdef DGAN_PROBE
      const long long probe_e1 = clock64();
      probe_epi += probe_e1 - probe_e0;
      probe_h0 = (unsigned)probe_e1;
      probe_new_item = true;
      probe_steps = it;
#endif
      ++item_count;
    }
    if (TMA_EPI && lane == 0) ptx::bulk_wait_all0();   // this warp's output stores are complete before the CTA retires
  }

#ifdef DGAN_PROBE
  {
    constexpr int key = tc2_probe_key(N_TILE, EPI, (int)sizeof(TOUT));
    if (threadIdx.x == 0) {
      atomicAdd(&g_tc2_probe[key][blockIdx.x][3], (unsigned long long)probe_wait_full);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][8], (unsigned long long)probe_issue);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][9], (unsigned long long)probe_wait1);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][10], (unsigned long long)probe_wait0);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][11], (unsigned long long)probe_epi);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][16], (unsigned long long)probe_in);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][17], (unsigned long long)probe_stage);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][18], (unsigned long long)probe_regs);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][19], (unsigned long long)probe_sts);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][20], (unsigned long long)probe_fence);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      atomicAdd(&g_tc2_probe[key][blockIdx.x][12], (unsigned long long)probe_rec);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][13], (unsigned long long)probe_head);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][15], (unsigned long long)probe_steps);
      if (probe_steps != 0) atomicAdd(&g_tc2_probe[key][blockIdx.x][14], (unsigned long long)((unsigned)clock64() - probe_h0));
      atomicAdd(&g_tc2_probe[key][blockIdx.x][0], (unsigned long long)(clock64() - probe_t_go));
      atomicAdd(&g_tc2_probe[key][blockIdx.x][1], 1ull);
      atomicAdd(&g_tc2_probe[key][blockIdx.x][2], (unsigned long long)(probe_t_go - probe_t_entry));
      atomicAdd(&g_tc2_probe[key][blockIdx.x][4], (unsigned long long)(probe_t_entry - probe_t_start));
      g_tc2_probe[key][blockIdx.x][5] = probe_g_start;
      g_tc2_probe[key][blockIdx.x][6] = probe_gtime();
    }
  }
#endif
  ptx::cluster_sync();   // the peer's multicasts and barrier arrivals target this CTA's shared memory: nobody leaves early
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
struct Tc2Schedule {           // one window tiling of a layer-direction + its item -> CTA-pair assignment, uploaded
  TcItem2* items = nullptr;
  TcRec* stream_p = nullptr;       // producer records (both ranks of a pair); per CTA pair: its items' steps, concatenated
  TcRec* stream_m = nullptr;       // MMA records, same indexing
  Tc2Heads heads{};                // per pair: record offsets into the streams (kernel parameter)
  int* eitems = nullptr;           // [n_slots][n_pairs] item words (tc2_item_word) for the consumer epilogues, or -1
  int n_slots = 0, n_pairs = 0;
  int maxb = 1;                    // accumulator slots per round: selects the kernel instantiation
};
// 64-channel or 16-channel TMA box for operands of K channels (tc_make_map)
static uint32_t tc2_box_k(int K) { return tc2_ksub(K) == 4 ? 64u : 16u; }
// The order in which the CTA pairs take a layer-direction's items (window, row pair), see tc2_search.  LPT: largest
// first over the whole batch.  BAND: row pairs in bands that every pair walks in the same order, so an activation
// tile's re-reads fall close together in time and hit L2; the default.
enum Tc2Order { TC2_ORDER_LPT = 0, TC2_ORDER_BAND = 1 };
// One layer-direction of the fp16 path: out[P_out][rows][N] = epi(pixel graph `tab` over in[P_in][rows][K] and n_tiles
// [N][K] weight tiles).  dgan_api.cu's tc_directions() fills the description from the generator's desc alone; a handle
// adds the weight tiles, their tensor map and the schedules planned for its row counts.
struct TcDir {
  std::string name, kind;      // plan-statistics row, profile kind
  int N = 0, K = 0, P_in = 0, P_out = 0, n_tiles = 0;
  PairTable tab;               // an output pixel that receives nothing has (pixel 0, zero tile)
  int h_grid = 0, w_grid = 0;  // the output pixels as the grid the planner's windows tile
  int max_acc = 1;             // most accumulators per window
  int epi = EPI_NONE, out_bytes = 2, bias_pstride = 0;
  // The logical layer-direction (layer l forward = 2l, backward = 2l + 1) this entry computes.  A layer-direction with
  // more than 256 output channels is split into column blocks of 256: entry i writes channels [col0, col0 + N) of the
  // one out_ld-wide output tensor that the next layer reads.
  int ld = 0, col0 = 0, out_ld = 0;
  int n_real = 0;              // real (unpadded) output channels of the logical layer-direction
  std::string base_kind;       // profile kind of the logical layer-direction (kind without the block's channel range)
  __half* w = nullptr;         // [n_tiles][N][K] fp16, K contiguous
  CUtensorMap tm_b{};          // box {64 | 16, N/2, 1}: the half of a weight tile (sub-tile) one CTA of the pair loads
  int force_maxb = 0;          // > 0: plan with exactly this many accumulator slots per round (dgan_debug_force_slots)
  int order = TC2_ORDER_BAND;  // item order (Tc2Order; dgan_debug_force_order)
  std::vector<std::pair<int, Tc2Schedule>> by_mpairs;   // uploaded schedule per n_mpairs (tc2_get_schedule)
};

static int tc2_maxb(int N) { return TC2_BUF_COLS / tc2_acc_stride(N); }

// host-side description of one step (same for every row pair; ring offset and dep are filled per CTA-pair stream)
struct Tc2HostStep {
  int kc = 0, nA = 0, nB = 0, n_rounds = 0;
  int a_pix[TC2_MAX_A] = {0, 0, 0, 0};
  uint8_t b_ent[TC2_MAX_BSLOTS] = {0};   // weight tile per B slot
  uint8_t ops[TC2_OP_BYTES] = {0};       // [round][accumulator] op bytes (TcOp)
  int n_real = 0;              // ops that do not read the zero tile (statistics)
  int bytes = 0;               // operand bytes staged per CTA
};
struct Tc2HostItem {
  TcItem2 hdr{};
  std::vector<Tc2HostStep> steps;
  double stage_bytes = 0.0;
  long long n_ops = 0;         // ops of the rounds' slots (rounds x slots, KSUB k16 MMAs each): what the time model charges
  long long n_issued = 0;      // ops the kernel issues: the real ones, and the zero-tile ones where the instantiation
                               // issues them (tc2_issues_zero_ops)
};

// Steps of one window (accumulator a <-> output pixel qs[a]).  Input pixels are taken in ascending order and packed
// greedily into steps of <= max_a A tiles (max_a = 1: one input pixel per step); a weight tile needed by several
// pixels of a step is staged once.  The kernel issues a step as rounds over the max_b accumulator slots of the
// instantiation: an accumulator's r-th contribution in the step (pixel order) goes to round r, and a slot with nothing
// to add in a round - or beyond the window's accumulators - holds a zero-tile op, which only the fixed-round
// instantiations issue (tc2_issues_zero_ops).
static void tc2_build_item(const PairTable& tab, const std::vector<int>& qs, int N, int K, int max_b, int max_a,
                           int step_max_bytes, Tc2HostItem* out) {
  const int ksub = tc2_ksub(K), kch = K / (16 * ksub), a_bytes = tc2_a_bytes(ksub), b_tile = tc2_b_bytes(N, ksub);
  out->hdr = TcItem2{};
  out->hdr.n_acc = (uint32_t)qs.size();
  for (size_t a = 0; a < qs.size(); ++a) out->hdr.q[a] = (uint16_t)qs[a];
  out->steps.clear();
  std::vector<std::pair<int, std::vector<std::pair<int, int>>>> by_p;   // pixel -> (tile, acc), sorted by acc
  for (size_t a = 0; a < qs.size(); ++a)
    for (int e = tab.off[qs[a]]; e < tab.off[qs[a] + 1]; ++e) {
      const int p = tab.pairs[e].x, t = tab.pairs[e].y;
      size_t g = 0;
      for (; g < by_p.size(); ++g)
        if (by_p[g].first == p) break;
      if (g == by_p.size()) by_p.push_back({p, {}});
      by_p[g].second.push_back({t, (int)a});
    }
  std::sort(by_p.begin(), by_p.end(), [](const auto& l, const auto& r) { return l.first < r.first; });
  for (auto& g : by_p)
    std::stable_sort(g.second.begin(), g.second.end(), [](const auto& l, const auto& r) { return l.second < r.second; });
  // a pixel with more entries than one step can hold is split (Linear layers: 16 tiles per input "pixel")
  std::vector<std::pair<int, std::vector<std::pair<int, int>>>> px;
  const int ent_cap = std::min(TC2_MAX_BSLOTS, std::max(1, (step_max_bytes - a_bytes) / b_tile));
  for (auto& g : by_p)
    for (size_t b0 = 0; b0 < g.second.size(); b0 += (size_t)ent_cap)
      px.push_back({g.first, std::vector<std::pair<int, int>>(g.second.begin() + b0,
                                                               g.second.begin() + std::min(g.second.size(), b0 + (size_t)ent_cap))});
  const int max_rounds = TC2_OP_BYTES / max_b;
  // ---- phase 1: greedy groups (each step stages its own weight tiles: re-using the previous step's would save bytes but
  //      hold ring capacity).
  struct Group { size_t i0, i1; };
  std::vector<Group> groups;
  {
    size_t i0 = 0;
    while (i0 < px.size()) {
      size_t i1 = i0;
      std::vector<int> staged;      // tiles this group loads itself
      int cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // contributions per accumulator = rounds it needs
      auto have = [&](int t) { return std::find(staged.begin(), staged.end(), t) != staged.end(); };
      while (i1 < px.size() && (int)(i1 - i0) < max_a) {
        int fresh = 0;
        std::vector<int> fresh_tiles;
        int c2[8];
        std::copy(cnt, cnt + 8, c2);
        int rounds = 0;
        for (auto& ta : px[i1].second) {
          if (!have(ta.first) && std::find(fresh_tiles.begin(), fresh_tiles.end(), ta.first) == fresh_tiles.end()) {
            fresh_tiles.push_back(ta.first); ++fresh;
          }
          ++c2[ta.second];
        }
        for (int a = 0; a < 8; ++a) rounds = std::max(rounds, c2[a]);
        const int nA = (int)(i1 - i0) + 1, nB = (int)staged.size() + fresh;
        const bool dup_pixel = (i1 > i0 && px[i1].first == px[i1 - 1].first);   // split halves of one pixel stay apart
        if (i1 > i0 && (dup_pixel || nB > TC2_MAX_BSLOTS || rounds > max_rounds ||
                        nA * a_bytes + nB * b_tile > step_max_bytes))
          break;
        for (int t : fresh_tiles) staged.push_back(t);
        std::copy(c2, c2 + 8, cnt);
        ++i1;
      }
      groups.push_back({i0, i1});
      i0 = i1;
    }
  }
  // ---- phase 2: B slots + the [round][accumulator] ops
  uint32_t seen = 0;
  for (size_t gi = 0; gi < groups.size(); ++gi) {
    const Group& G = groups[gi];
    Tc2HostStep st;
    st.nA = (int)(G.i1 - G.i0);
    std::fill(st.ops, st.ops + TC2_OP_BYTES, TC2_PAD_OP);
    int slot_of[32], cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int t = 0; t < 32; ++t) slot_of[t] = -1;
    for (size_t i = G.i0; i < G.i1; ++i) {
      st.a_pix[i - G.i0] = px[i].first;
      for (auto& ta : px[i].second) {
        const int t = ta.first, acc = ta.second;
        if (slot_of[t] < 0) {
          slot_of[t] = st.nB;
          st.b_ent[st.nB++] = (uint8_t)t;
        }
        const bool first = !(seen & (1u << acc));
        const int r = cnt[acc]++;
        st.ops[r * max_b + acc] = TcOp{(uint32_t)(i - G.i0), (uint32_t)slot_of[t], first ? 1u : 0u}.encode();
        st.n_rounds = std::max(st.n_rounds, r + 1);
        st.n_real += 1;
        seen |= 1u << acc;
      }
    }
    st.bytes = st.nA * a_bytes + st.nB * b_tile;
    out->steps.push_back(st);
  }
  // k-chunk outermost: every accumulator then sums its (k-chunk, input pixel) contributions in one canonical order
  // - ascending k-chunk, ascending pixel - whatever the window shape and step grouping, so results do not depend
  // on the batch size (the schedule does) and a sharded batch reproduces the unsharded one bit for bit.
  const size_t n_groups = out->steps.size();
  for (int kc = 1; kc < kch; ++kc)
    for (size_t gi = 0; gi < n_groups; ++gi) {
      Tc2HostStep sk = out->steps[gi];
      sk.kc = kc;
      for (int o = 0; o < TC2_OP_BYTES; ++o) sk.ops[o] = (uint8_t)TcOp::First::put(sk.ops[o], 0u);
      out->steps.push_back(sk);
    }
  out->stage_bytes = 0.0;
  out->n_ops = 0;
  out->n_issued = 0;
  for (auto& stp : out->steps) {
    out->stage_bytes += stp.bytes;
    out->n_ops += (long long)stp.n_rounds * max_b;
    out->n_issued += tc2_issues_zero_ops(max_b, ksub) ? (long long)stp.n_rounds * max_b : (long long)stp.n_real;
  }
}

// Windows of wh x ww accumulators with strides (sy, sx) over the output grid.  Stride 2 gathers outputs of equal
// parity of a stride-2 transposed conv: they use the same taps with neighbouring inputs, so weight tiles are shared.
static void tc2_enumerate_windows(int h_grid, int w_grid, int wh, int ww, int sy, int sx, std::vector<std::vector<int>>* wins) {
  wins->clear();
  for (int by = 0; by < h_grid; by += wh * sy)
    for (int bx = 0; bx < w_grid; bx += ww * sx)
      for (int ry = 0; ry < sy; ++ry)
        for (int rx = 0; rx < sx; ++rx) {
          std::vector<int> qs;
          for (int i = 0; i < wh; ++i)
            for (int j = 0; j < ww; ++j) {
              const int y = by + ry + i * sy, x = bx + rx + j * sx;
              if (y < h_grid && x < w_grid) qs.push_back(y * w_grid + x);
            }
          if (!qs.empty()) wins->push_back(qs);
        }
}

#ifndef DGAN_STEP_MAX_KB
#define DGAN_STEP_MAX_KB 48
#endif
#ifndef DGAN_STEP_MAX_KB_N64
#define DGAN_STEP_MAX_KB_N64 64
#endif
#ifndef DGAN_COST_EPI_KB
#define DGAN_COST_EPI_KB 24.0
#endif
#ifndef DGAN_COST_FIXED_KB
#define DGAN_COST_FIXED_KB 48.0
#endif
// Time model of an item (DESIGN.md section 3, least-squares fit to per-kernel times on an H100): NS_PER_KB per KB of
// the cost above (staged bytes + epilogue and fixed charges), OP_NS per 64-channel op (4 k16 MMAs) at N = 64, scaled by
// max(N, OP_MIN_N) / 64 for other widths and by KSUB / 4 for narrow ops, and STEP_NS per step (the consumers' full-barrier wait, wgmma commit and
// wait, region release and record load of a step).
#ifndef DGAN_COST_NS_PER_KB
#define DGAN_COST_NS_PER_KB 6.8
#endif
#ifndef DGAN_COST_OP_NS
#define DGAN_COST_OP_NS 103.0
#endif
#ifndef DGAN_COST_STEP_NS
#define DGAN_COST_STEP_NS 942.0
#endif
#ifndef DGAN_COST_OP_MIN_N
#define DGAN_COST_OP_MIN_N 32
#endif
#ifndef TC2_REFINE_BUDGET
#define TC2_REFINE_BUDGET (1LL << 26)    // candidate evaluations of the assignment refinement per window shape (tc2_search)
#endif
// Banded order (tc2_search): the input and output bytes of one band's row pairs stay within this share of the 50 MB L2,
// and the banded assignment is kept while its makespan is within TC2_BAND_TOLERANCE of LPT's.  On an H100 (DESIGN.md
// section 6) the banded directions ran up to 16 % faster and none slower while their makespans were up to 1.7 % worse.
// A direction whose whole input is smaller than TC2_BAND_MIN_INPUT stays in L2 in any order and keeps LPT: the last
// layer's backward on MNIST (4 and 8 MB of input) ran 5 - 7 % slower in bands, CelebA's Generator.2 forward (10.5 MB)
// 2 - 3 % faster.
#ifndef TC2_BAND_L2_BYTES
#define TC2_BAND_L2_BYTES (16 << 20)
#endif
#ifndef TC2_BAND_TOLERANCE
#define TC2_BAND_TOLERANCE 0.02
#endif
#ifndef TC2_BAND_MIN_INPUT
#define TC2_BAND_MIN_INPUT (9 << 20)
#endif

// The planner.  tc2_search picks the accumulator slots per round and the window tiling for `n_mpairs` row pairs on
// `n_pairs` CTA pairs and assigns the items to the pairs; tc2_encode_streams lays each pair's steps out in its operand
// ring and writes the records; tc2_get_schedule uploads the result.
struct Tc2Plan {               // host result of the planner (what tc2_get_schedule uploads)
  int shape[4] = {1, 1, 1, 1};   // wh, ww, sy, sx
  int n_slots = 0, n_pairs = 0;
  std::vector<TcItem2> hdrs;
  std::vector<TcRec> stream_p, stream_m;
  std::vector<uint32_t> stream_off;
  std::vector<int> eitems;
  // ops of the rounds' slots (rounds x slots, KSUB k16 MMAs each), the zero-tile ones among them, ops issued (the real
  // ones, and the zero-tile ones where the instantiation issues them)
  long long n_mma = 0, n_pad = 0, n_issued = 0, n_steps = 0, n_bytes = 0;
  long long n_bytes_a = 0, n_bytes_b = 0;   // n_bytes split: activation tiles (both CTAs) and weight tiles (multicast)
  long long uniq_a_bytes = 0;  // the distinct activation tiles the plan reads (both CTAs): its input tensor
  // peak, over the cost model's timeline of every pair, of the bytes of activation tiles between their first and last load
  long long ws_a_bytes = 0;
  // cost-model load of the busiest CTA pair / the mean over pairs of the LPT assignment (the window shape's score)
  double load_max = 0.0, load_mean = 0.0;
  double op_ns_max = 0.0;      // the MMA term of that busiest pair's load (estimated tensor time, ns)
  double op_ns_issued_max = 0.0;   // the same term for the ops the kernel issues (n_issued)
  int order = TC2_ORDER_LPT, band_rows = 0;   // the order the plan uses (Tc2Order) and its row pairs per band
  double load_max_order = 0.0;  // the busiest pair's load under that order
  int maxb = 1, ring_bytes = 0;   // accumulator slots per round of the chosen instantiation, its operand ring
  int ksub = 4;                   // k16 MMAs per op of the instantiation (tc2_ksub)
};

static double tc2_op_ns(int N, int ksub) {
  return DGAN_COST_OP_NS * (double)std::max(N, DGAN_COST_OP_MIN_N) / 64.0 * (double)ksub / 4.0;
}

// The time model's cost of one item (ns)
static double tc2_item_cost(const Tc2HostItem& it, int N, double op_ns) {
  return DGAN_COST_NS_PER_KB / 1024.0 *
             (it.stage_bytes + DGAN_COST_EPI_KB * 1024.0 * it.hdr.n_acc * std::max(1, N / 64) + DGAN_COST_FIXED_KB * 1024.0) +
         op_ns * (double)it.n_ops + DGAN_COST_STEP_NS * (double)it.steps.size();
}

// Band of item idx (window * n_mpairs + row pair) in time order: row pairs [b * band_rows, (b + 1) * band_rows) form band
// b, walked from the last band to the first when `reverse`.
static int tc2_band_of(int idx, int n_mpairs, int band_rows, bool reverse) {
  const int b = (idx % n_mpairs) / band_rows, n_bands = (n_mpairs + band_rows - 1) / band_rows;
  return reverse ? n_bands - 1 - b : b;
}

// Assign the items (window w, row pair mp; index w * n_mpairs + mp, cost icost[w]) to the CTA pairs: each in turn to the
// currently least-loaded pair, then refine, then order each pair's list.  band_rows = 0 (LPT): items in index order
// (windows sorted by staged bytes, mp the fast index: cost-descending), each pair's list largest first.  band_rows > 0
// (BAND): items by (band, cost descending), so every pair works through the bands in the same order; the refinement
// swaps items of one band only, and each list is sorted by (band, cost descending).  No pair takes more than max_items
// items (0: no limit).  Returns the makespan.
static double tc2_assign(const std::vector<double>& icost, int n_mpairs, int n_pairs, int band_rows, bool reverse,
                         size_t max_items, std::vector<std::vector<int>>* lists_out, std::vector<double>* load_out) {
  const long long total = (long long)icost.size() * n_mpairs;
  auto cost_of = [&](int idx) { return icost[(size_t)(idx / n_mpairs)]; };
  auto band_of = [&](int idx) { return band_rows > 0 ? tc2_band_of(idx, n_mpairs, band_rows, reverse) : 0; };
  std::vector<int> seq((size_t)total);
  std::iota(seq.begin(), seq.end(), 0);
  if (band_rows > 0)
    std::stable_sort(seq.begin(), seq.end(), [&](int a, int b) {
      return band_of(a) != band_of(b) ? band_of(a) < band_of(b) : cost_of(a) > cost_of(b);
    });
  std::vector<double>& load = *load_out;
  std::vector<std::vector<int>>& lists = *lists_out;
  load.assign((size_t)n_pairs, 0.0);
  lists.assign((size_t)n_pairs, {});
  const size_t cap = max_items > 0 ? max_items : (size_t)total;
  for (int idx : seq) {
    size_t best = (size_t)n_pairs;
    for (size_t pr = 0; pr < (size_t)n_pairs; ++pr)
      if (lists[pr].size() < cap && (best == (size_t)n_pairs || load[pr] < load[best])) best = pr;
    load[best] += cost_of(idx);
    lists[best].push_back(idx);
  }
  // Refinement: while the busiest pair can hand an item to - or swap one with - another pair so that both end
  // up below its load, do the best such move (LPT alone leaves e.g. 35 on a mean of 30.4 for Generator.2 bwd's
  // 160 items of cost 4..25).
  // One pass looks at |P| x (1 + |Q|) candidates for every other pair Q: quadratic in the items per pair.  With many
  // items per pair (large batches: 160 row pairs x 1024 windows) LPT alone is already within one small item of
  // the mean and the search would take minutes, so it runs on a budget of candidate evaluations that the
  // benchmarked sizes (<= 20 row pairs) never reach.
  long long work = 0;
  for (int iter = 0; iter < 4096 && work < TC2_REFINE_BUDGET; ++iter) {
    const size_t P = (size_t)(std::max_element(load.begin(), load.end()) - load.begin());
    double best_peak = load[P];
    size_t bq = P; int bi = -1, bj = -1;
    for (size_t Q = 0; Q < (size_t)n_pairs; ++Q) {
      if (Q == P) continue;
      work += (long long)lists[P].size() * (long long)(1 + lists[Q].size());
      for (size_t i = 0; i < lists[P].size(); ++i) {
        const double ci = cost_of(lists[P][i]);
        double peak = std::max(load[P] - ci, load[Q] + ci);           // move i: P -> Q
        if (lists[Q].size() < cap && peak < best_peak - 1e-9) { best_peak = peak; bq = Q; bi = (int)i; bj = -1; }
        for (size_t j = 0; j < lists[Q].size(); ++j) {                 // swap i <-> j
          const double cj = cost_of(lists[Q][j]);
          if (cj >= ci || band_of(lists[Q][j]) != band_of(lists[P][i])) continue;
          peak = std::max(load[P] - ci + cj, load[Q] + ci - cj);
          if (peak < best_peak - 1e-9) { best_peak = peak; bq = Q; bi = (int)i; bj = (int)j; }
        }
      }
    }
    if (bi < 0) break;
    const int it_i = lists[P][(size_t)bi];
    const double ci = cost_of(it_i);
    if (bj < 0) {
      lists[P].erase(lists[P].begin() + bi);
      lists[bq].push_back(it_i);
      load[P] -= ci; load[bq] += ci;
    } else {
      const int it_j = lists[bq][(size_t)bj];
      const double cj = cost_of(it_j);
      lists[P][(size_t)bi] = it_j; lists[bq][(size_t)bj] = it_i;
      load[P] += cj - ci; load[bq] += ci - cj;
    }
  }
  // biggest first within a band: a pair's last item is its smallest (shortest un-overlapped epilogue)
  for (auto& l : lists)
    std::stable_sort(l.begin(), l.end(), [&](int a, int b) {
      return band_of(a) != band_of(b) ? band_of(a) < band_of(b) : cost_of(a) > cost_of(b);
    });
  return *std::max_element(load.begin(), load.end());
}

// Every candidate - an instantiation of TC2_KINDS for (N, epilogue, output type) and a shape of wh x ww <= its slots
// accumulators, strides 1 or 2 - is scored by an LPT assignment of its items (window, row pair) to the CTA pairs with
// the time model above (operand bytes staged, a per-accumulator epilogue charge, a fixed per-item charge, and the ops
// of the rounds' slots, zero-tile ones included even where the kernel skips them: the constants were fitted to kernels
// that issued them); the smallest makespan wins.  With order BAND the winner's items are then assigned again in bands
// of row pairs (tc2_assign): as few row pairs per band as give every CTA pair about one item, and no more than keep the
// band's input and output within TC2_BAND_L2_BYTES.  Under LPT every pair works on windows of similar cost across all
// row pairs at once, so a tile read by an early (interior) and a late (boundary) window is fetched from L2 twice only if
// the whole input stays there; in bands it is re-read while its band runs.  The banded assignment is kept unless its
// makespan exceeds LPT's by more than TC2_BAND_TOLERANCE.  `reverse` walks the bands from the last row pair down:
// alternated from one layer-direction to the next, a kernel starts on the rows its predecessor wrote last.  Fills the
// plan's shape, slots, ring, order and loads, and returns the winner's items and, per CTA pair, its item indices
// (window * n_mpairs + row pair) in issue order.  force_shape (statistics only): consider only this window shape
// {wh, ww, sy, sx}.
static int tc2_search(int N, int K, const PairTable& tab, int h_grid, int w_grid, int max_acc, int force_maxb, int epi,
                      int out_bytes, int n_mpairs, int n_pairs, int order, bool reverse, const int* force_shape,
                      Tc2Plan* plan, std::vector<Tc2HostItem>* best_items, std::vector<std::vector<int>>* best_lists) {
  const int max_a = TC2_MAX_A;
  // Step size: a step is consumed only once all of it has landed, so big steps cost pipeline depth (4 x 48 KB fit the
  // ring); 48 KB holds one activation tile and one whole N = 256 weight tile.  The N = 64, K = 128 layer (Generator.3
  // forward: 8 KB weight tiles) packs 3 activation tiles and their taps into steps of up to 64 KB.  Three steps always
  // fit the ring, so a step's region never overlaps the previous step's: that one is released only after this step's
  // first round has been issued.
  const int step_kb = (N == 64 && K == 128) ? DGAN_STEP_MAX_KB_N64 : DGAN_STEP_MAX_KB;
  const int ksub = tc2_ksub(K);
  const double op_ns = tc2_op_ns(N, ksub);
  double best_cost = 1e300;
  plan->maxb = 0;
  std::vector<std::vector<int>> wins;
  std::vector<double> best_load;
  for (const Tc2Kind& kind : kTc2Kinds) {
    if (kind.n != N || kind.ksub != ksub || kind.epi != epi || kind.out_bytes != out_bytes) continue;
    if (force_maxb > 0 && kind.maxb != force_maxb) continue;
    const int mb = kind.maxb, ring = tc2_ring_bytes(N, mb, ksub, epi, out_bytes);
    const int step_max = std::min((ring / 3) & ~1023, step_kb * 1024);
    for (int wh = 1; wh <= 2; ++wh)
      for (int ww = 1; ww <= 8; ++ww)
        for (int sy = 1; sy <= (wh > 1 ? 2 : 1); ++sy)
          for (int sx = 1; sx <= (ww > 1 ? 2 : 1); ++sx) {
            if (wh * ww > std::min(max_acc, mb) || wh > h_grid || ww > std::max(w_grid, 1)) continue;
            if (force_shape != nullptr && (wh != force_shape[0] || ww != force_shape[1] || sy != force_shape[2] || sx != force_shape[3])) continue;
            tc2_enumerate_windows(h_grid, std::max(w_grid, 1), wh, ww, sy, sx, &wins);
            std::vector<Tc2HostItem> items(wins.size());
            for (size_t i = 0; i < wins.size(); ++i) tc2_build_item(tab, wins[i], N, K, mb, max_a, step_max, &items[i]);
            std::stable_sort(items.begin(), items.end(), [](const Tc2HostItem& l, const Tc2HostItem& r) { return l.stage_bytes > r.stage_bytes; });
            std::vector<double> icost(items.size());
            for (size_t i = 0; i < items.size(); ++i) icost[i] = tc2_item_cost(items[i], N, op_ns);
            std::vector<std::vector<int>> lists;
            std::vector<double> load;
            const double makespan = tc2_assign(icost, n_mpairs, n_pairs, 0, false, 0, &lists, &load);
            if (makespan < best_cost) {
              best_cost = makespan;
              plan->shape[0] = wh; plan->shape[1] = ww; plan->shape[2] = sy; plan->shape[3] = sx;
              plan->maxb = mb; plan->ring_bytes = ring;
              best_items->swap(items); best_lists->swap(lists); best_load.swap(load);
            }
          }
  }
  if (plan->maxb == 0) { set_error("no tensor-core kernel instantiation for this layer-direction"); return DGAN_ERR_UNSUPPORTED; }
  plan->ksub = ksub;
  const std::vector<Tc2HostItem>& items = *best_items;
  plan->load_max = best_cost;
  plan->load_mean = std::accumulate(best_load.begin(), best_load.end(), 0.0) / (double)n_pairs;
  plan->op_ns_max = 0.0;
  plan->op_ns_issued_max = 0.0;
  for (size_t pr = 0; pr < best_lists->size(); ++pr)
    if (best_load[pr] == best_cost) {
      for (int idx : (*best_lists)[pr]) {
        plan->op_ns_max += op_ns * (double)items[(size_t)(idx / n_mpairs)].n_ops;
        plan->op_ns_issued_max += op_ns * (double)items[(size_t)(idx / n_mpairs)].n_issued;
      }
      break;
    }
  plan->order = TC2_ORDER_LPT;
  plan->band_rows = 0;
  plan->load_max_order = best_cost;
  std::vector<double> icost(items.size());
  for (size_t i = 0; i < items.size(); ++i) icost[i] = tc2_item_cost(items[i], N, op_ns);
  if (order == TC2_ORDER_BAND && n_mpairs > 1) {
    // one row pair's input (the distinct pixels the steps stage, K channels) and output, in bytes
    std::vector<int> pix;
    long long n_out = 0;
    for (const Tc2HostItem& it : items) {
      n_out += it.hdr.n_acc;
      for (const Tc2HostStep& st : it.steps) pix.insert(pix.end(), st.a_pix, st.a_pix + st.nA);
    }
    std::sort(pix.begin(), pix.end());
    const long long n_in = std::unique(pix.begin(), pix.end()) - pix.begin();
    const long long mp_bytes = 2LL * kRowTile * (2LL * K * n_in + (long long)out_bytes * N * n_out);
    const int fill = (n_pairs + (int)items.size() - 1) / (int)items.size();
    const int fit = (int)std::max(1LL, (long long)TC2_BAND_L2_BYTES / std::max(mp_bytes, 1LL));
    const int band_rows = std::min(n_mpairs, std::max(1, std::min(fill, fit)));
    const long long in_bytes = 2LL * kRowTile * n_mpairs * 2LL * K * n_in;
    if (band_rows < n_mpairs && in_bytes >= (long long)TC2_BAND_MIN_INPUT) {
      std::vector<std::vector<int>> lists;
      std::vector<double> load;
      // no pair takes more items than the most LPT gives one: each item is an epilogue and an item head more for its
      // pair, which the time model charges only as a fixed cost, and the epilogue item list keeps LPT's slots
      size_t lpt_items = 0;
      for (const auto& l : *best_lists) lpt_items = std::max(lpt_items, l.size());
      const double makespan = tc2_assign(icost, n_mpairs, n_pairs, band_rows, reverse, lpt_items, &lists, &load);
      if (makespan <= best_cost * (1.0 + TC2_BAND_TOLERANCE)) {
        plan->order = TC2_ORDER_BAND;
        plan->band_rows = band_rows;
        plan->load_max_order = makespan;
        best_lists->swap(lists);
      }
    }
  }
  return 0;
}

// Per CTA pair, its items' steps in issue order: simulate the pair's circular operand ring to give every step its
// region and dependency distance, and encode the producer and MMA records and the epilogue item list.  The only
// writer of the records.
static int tc2_encode_streams(int N, int n_mpairs, int n_pairs, const std::vector<Tc2HostItem>& items,
                              const std::vector<std::vector<int>>& lists, Tc2Plan* plan) {
  const int max_b = plan->maxb, ring_bytes = plan->ring_bytes, ksub = plan->ksub;
  plan->n_pairs = n_pairs;
  size_t n_slots = 0;
  for (auto& l : lists) n_slots = std::max(n_slots, l.size());
  plan->n_slots = (int)n_slots;
  std::vector<int>& eitems = plan->eitems;
  eitems.assign(n_slots * (size_t)n_pairs, -1);
  std::vector<uint32_t>& stream_off = plan->stream_off;
  stream_off.assign((size_t)n_pairs + 1, 0);
  std::vector<TcRec>& stream_p = plan->stream_p;
  std::vector<TcRec>& stream_m = plan->stream_m;
  stream_p.clear(); stream_m.clear();
  long long n_mma = 0, n_pad = 0, n_issued = 0, n_steps = 0, n_bytes_a = 0, n_bytes_b = 0;
  // statistics: per activation tile (row pair, k-chunk, pixel) the first and last time a step loads it, on the time
  // model's timeline of its CTA pair (a step at its share of the item's cost)
  const double op_ns = tc2_op_ns(N, ksub);
  std::unordered_map<long long, std::pair<double, double>> a_span;
  for (size_t pr = 0; pr < lists.size(); ++pr) {
    stream_off[pr] = (uint32_t)stream_m.size();
    double t_item = 0.0;
    // circular operand ring of this CTA pair: sequential allocation, wrap when the step does not fit
    std::vector<std::pair<int, int>> region;     // [begin, end) in KB of every step of this stream
    int cursor = 0;
    for (size_t k = 0; k < lists[pr].size(); ++k) {
      const int win = lists[pr][k] / n_mpairs, mp = lists[pr][k] % n_mpairs;
      if ((uint32_t)win > TcItemWindow::mask || (uint32_t)mp > TcItemMp::mask) { set_error("tensor-core schedule limits exceeded"); return DGAN_ERR_UNSUPPORTED; }
      eitems[k * (size_t)n_pairs + pr] = tc2_item_word(win, mp);
      const Tc2HostItem& itm = items[(size_t)win];
      const double c_item = tc2_item_cost(itm, N, op_ns);
      for (size_t j = 0; j < itm.steps.size(); ++j) {
        const Tc2HostStep& hs = itm.steps[j];
        const double t = t_item + c_item * (double)j / (double)itm.steps.size();
        for (int a = 0; a < hs.nA; ++a) {
          const long long key = ((long long)mp * 16 + hs.kc) * 65536 + hs.a_pix[a];
          auto ins = a_span.insert({key, {t, t}});
          if (!ins.second) ins.first->second.second = t;
        }
        const int kb = (hs.bytes + 1023) / 1024;
        if (kb * 1024 > ring_bytes) { set_error("tensor-core step larger than the operand ring"); return DGAN_ERR_UNSUPPORTED; }
        if (cursor + kb > ring_bytes / 1024) cursor = 0;
        const int beg = cursor, end = cursor + kb;
        cursor = end;
        // The producer may overwrite a region once the step that used it is consumed: dep = distance to the latest
        // earlier step whose region overlaps this one (8 = barrier-slot reuse only).
        int dep = TC2_NSLOT;
        const int kidx = (int)region.size();
        for (int d = 1; d <= TC2_NSLOT && d <= kidx; ++d) {
          const auto& rg = region[(size_t)(kidx - d)];
          if (rg.first < end && beg < rg.second) { dep = d; break; }
        }
        if (dep == 1 && j > 0) { set_error("tensor-core step overlaps the step before it (ring too small)"); return DGAN_ERR_UNSUPPORTED; }
        region.push_back({beg, end});
        TcMmaRec m;
        m.off = (uint32_t)beg; m.nA = (uint32_t)hs.nA; m.n_rounds = (uint32_t)hs.n_rounds; m.maxb = (uint32_t)max_b; m.ksub = (uint32_t)ksub;
        m.flags = (j == 0 ? TcMmaRec::FIRST : 0u) | (j + 1 == itm.steps.size() ? TcMmaRec::LAST : 0u);
        std::copy(hs.ops, hs.ops + hs.n_rounds * max_b, m.ops);    // the op bytes of later rounds stay 0
        stream_m.push_back(m.encode());
        TcProducerRec p;
        p.off = (uint32_t)beg; p.kc = (uint32_t)hs.kc; p.nA = (uint32_t)hs.nA; p.nB = (uint32_t)hs.nB; p.dep = (uint32_t)dep; p.mp = (uint32_t)mp;
        std::copy(hs.a_pix, hs.a_pix + TC2_MAX_A, p.pix);
        std::copy(hs.b_ent, hs.b_ent + TC2_MAX_BSLOTS, p.tile);
        stream_p.push_back(p.encode());
        // bytes read from L2 by the pair: both activation tiles, each weight tile once (multicast)
        n_mma += hs.n_rounds * max_b; n_pad += hs.n_rounds * max_b - hs.n_real;
        n_issued += tc2_issues_zero_ops(max_b, ksub) ? hs.n_rounds * max_b : hs.n_real;
        n_steps += 1; n_bytes_a += 2LL * hs.nA * tc2_a_bytes(ksub); n_bytes_b += (long long)hs.nB * tc2_b_bytes(N, ksub);
      }
      t_item += c_item;
    }
  }
  std::vector<std::pair<double, int>> ev;       // (time, +1 first load / -1 after the last)
  for (const auto& kv : a_span) { ev.push_back({kv.second.first, 1}); ev.push_back({kv.second.second, -1}); }
  std::sort(ev.begin(), ev.end(), [](const auto& l, const auto& r) { return l.first != r.first ? l.first < r.first : l.second > r.second; });
  long long live = 0, peak = 0;
  for (const auto& e : ev) { live += e.second; peak = std::max(peak, live); }
  plan->uniq_a_bytes = 2LL * tc2_a_bytes(ksub) * (long long)a_span.size();
  plan->ws_a_bytes = 2LL * tc2_a_bytes(ksub) * peak;
  stream_off[(size_t)n_pairs] = (uint32_t)stream_m.size();
  plan->hdrs.resize(items.size());
  for (size_t i = 0; i < items.size(); ++i) plan->hdrs[i] = items[i].hdr;
  plan->n_mma = n_mma; plan->n_pad = n_pad; plan->n_issued = n_issued; plan->n_steps = n_steps;
  plan->n_bytes_a = n_bytes_a; plan->n_bytes_b = n_bytes_b; plan->n_bytes = n_bytes_a + n_bytes_b;
  return 0;
}

// Whether layer-direction ld (layer l forward = 2l, backward = 2l + 1) walks its bands in reverse: the directions run
// forward l = 0, 1, .., then backward from the last layer down, so the position in that sequence alternates with
// l + (ld & 1) - also from one L-step's last direction (Linear backward) to the next one's first.
static bool tc2_band_reverse(int ld) { return (((ld >> 1) + (ld & 1)) & 1) != 0; }

// The plan of one layer-direction (tc2_search).  force_shape (statistics only): consider only this window shape
// {wh, ww, sy, sx}.
static int tc2_plan(int N, int K, const PairTable& tab, int h_grid, int w_grid, int max_acc, int force_maxb, int epi,
                    int out_bytes, int n_mpairs, int n_pairs, int order, bool reverse, Tc2Plan* plan,
                    const int* force_shape = nullptr) {
  std::vector<Tc2HostItem> items;
  std::vector<std::vector<int>> lists;
  const int rc = tc2_search(N, K, tab, h_grid, w_grid, max_acc, force_maxb, epi, out_bytes, n_mpairs, n_pairs, order,
                            reverse, force_shape, plan, &items, &lists);
  return rc ? rc : tc2_encode_streams(N, n_mpairs, n_pairs, items, lists, plan);
}

// Independent validation of a plan against the pair table it was built from (host only; used by
// dgan_debug_check_plans and the CPU tests).  Re-derives from the uploaded records alone:
//  * every (output pixel, input pixel, tap, k-chunk) contribution of every item happens exactly once, into the right
//    accumulator, with the weight tiles each CTA stages forming exactly the operand the MMA reads;
//  * the first MMA into an accumulator - and only that one - overwrites it;
//  * every accumulator sums in the canonical order (k-chunk major, input pixel ascending): results then do not
//    depend on the schedule (batch-size / sharding invariance);
//  * an op that reads the zero tile never overwrites its accumulator, and every round has a real op (the kernel
//    commits one wgmma group per round);
//  * ring safety: when a step's loads may start (step k - dep consumed), no earlier step that can still be read
//    overlaps its region, regions stay inside the ring, dep <= number of barrier slots;
//  * progress: a step's region is released only once the next step's first round is issued (unless it ends its item), so
//    no step inside an item may wait for the step right before it (dep >= 2);
//  * every (window, row pair) item is assigned to exactly one CTA pair;
//  * the accumulator slots per round and the k16 MMAs per op name an instantiation of TC2_KINDS, and every MMA record
//    carries the plan's counts (the launch dispatches on them, the kernel decodes the records and stages its operands
//    with them).
static int tc2_check_plan(int N, int K, const PairTable& tab, int n_mpairs, int epi, int out_bytes, const Tc2Plan& pl,
                          std::string* err) {
  auto fail = [&](const std::string& m) { *err = m; return DGAN_ERR_INVALID_ARG; };
  const int ksub = tc2_ksub(K), kch = K / (16 * ksub), a_bytes = tc2_a_bytes(ksub), b_tile = tc2_b_bytes(N, ksub);
  const int max_acc = pl.maxb;
  if (pl.ksub != ksub) return fail("plan's k16 MMAs per op disagree with the direction's channels");
  if (!tc2_has_kind(N, max_acc, ksub, epi, out_bytes)) return fail("no kernel instantiation with these accumulator slots per round");
  const int ring_bytes = tc2_ring_bytes(N, max_acc, ksub, epi, out_bytes);
  const size_t n_pairs = (size_t)pl.n_pairs;
  if (pl.stream_off.size() != n_pairs + 1) return fail("stream_off size");
  if (pl.stream_p.size() != pl.stream_m.size()) return fail("stream sizes differ");
  if (pl.eitems.size() != (size_t)pl.n_slots * n_pairs) return fail("eitems size");
  std::vector<int> assigned(pl.hdrs.size() * (size_t)n_mpairs, 0);
  for (const TcItem2& h : pl.hdrs) {
    if (h.n_acc < 1 || (int)h.n_acc > max_acc) return fail("window with too many accumulators");
    for (uint32_t a = 0; a < h.n_acc; ++a)
      if ((size_t)h.q[a] + 1 >= tab.off.size()) return fail("window pixel out of range");
  }
  struct Step { int beg, end; };
  for (size_t pr = 0; pr < n_pairs; ++pr) {
    const uint32_t r_beg = pl.stream_off[pr], r_end = pl.stream_off[pr + 1];
    if (r_beg > r_end || r_end > pl.stream_m.size()) return fail("stream_off not monotone");
    std::vector<Step> steps;
    int item_k = -1, win = -1, mp = -1;
    bool in_item = false;
    uint32_t seen = 0;
    std::vector<std::pair<int, int>> last_kp;                     // per accumulator: last (kc, p)
    std::vector<std::vector<std::pair<int, int>>> contrib;        // per accumulator: (p * 32 + tile, kc)
    for (uint32_t ri = r_beg; ri < r_end; ++ri) {
      const TcMmaRec m = TcMmaRec::decode(pl.stream_m[ri]);
      const TcProducerRec p0 = TcProducerRec::decode(pl.stream_p[ri]);
      const int k = (int)steps.size();
      const int nA = (int)p0.nA, nB = (int)p0.nB, dep = (int)p0.dep, kc = (int)p0.kc;
      Step st{(int)p0.off, 0};
      if (m.off != p0.off || m.nA != p0.nA) return fail("MMA record disagrees with the producer record");
      if (nA < 1 || nA > TC2_MAX_A || nB > TC2_MAX_BSLOTS || kc >= kch) return fail("step field out of range");
      st.end = st.beg + (nA * a_bytes + nB * b_tile + 1023) / 1024;
      if (st.end * 1024 > ring_bytes) return fail("step region outside the ring");
      if (dep < 1 || dep > TC2_NSLOT) return fail("dep out of range");
      const uint32_t flags = m.flags;
      const int n_rounds = (int)m.n_rounds;
      if ((int)m.maxb != max_acc) return fail("MMA record disagrees with the plan on the accumulator slots per round");
      if ((int)m.ksub != ksub) return fail("MMA record disagrees with the instantiation on the k16 sub-tiles per op");
      if (n_rounds < 1 || n_rounds * max_acc > TC2_OP_BYTES) return fail("round count out of range");
      if (dep == 1 && !(flags & TcMmaRec::FIRST)) return fail("ring deadlock: a step waits for the step before it, which is released only after it");
      if (flags & TcMmaRec::FIRST) {
        if (in_item) return fail("item starts inside an item");
        in_item = true; ++item_k;
        if (item_k >= pl.n_slots) return fail("more items than slots");
        const int e = pl.eitems[(size_t)item_k * n_pairs + pr];
        if (e < 0) return fail("stream has an item the epilogue list lacks");
        win = tc2_item_window(e); mp = tc2_item_mp(e);
        if ((size_t)win >= pl.hdrs.size() || mp >= n_mpairs) return fail("item index out of range");
        if (assigned[(size_t)win * n_mpairs + mp]++) return fail("item assigned twice");
        seen = 0;
        last_kp.assign(pl.hdrs[win].n_acc, {-1, -1});
        contrib.assign(pl.hdrs[win].n_acc, {});
      }
      if (!in_item) return fail("step outside an item");
      if ((int)p0.mp != mp) return fail("row pair of a step differs from its item");
      const TcItem2& hdr = pl.hdrs[win];
      // the kernel issues round by round, accumulator 0 .. max_acc - 1 within a round
      for (int oi = 0; oi < n_rounds * max_acc; ++oi) {
        if (oi % max_acc == 0) {
          int real = 0;
          for (int a = 0; a < max_acc; ++a) real += TcOp::decode(m.ops[oi + a]).slot != (uint32_t)TC2_ZERO_SLOT;
          if (real == 0) return fail("round without a real op (it would commit an empty wgmma group)");
        }
        const TcOp op = TcOp::decode(m.ops[oi]);
        const int a_idx = (int)op.a, slot = (int)op.slot, acc = oi % max_acc;
        const bool first = op.first != 0;
        if (m.ops[oi] & ~TcOp::USED) return fail("op field out of range");
        if (slot == TC2_ZERO_SLOT) {
          // skipped by the instantiations that do not issue zero-tile ops; a zero-tile op never carries First either way
          if (first) return fail("zero-tile op overwrites its accumulator");
          continue;
        }
        if (a_idx >= nA) return fail("op reads an A tile the step does not stage");
        if (acc >= (int)hdr.n_acc) return fail("op writes past the window's accumulators");
        if (slot >= nB) return fail("op reads a B slot the step does not stage");
        if (p0.tile[slot] > TcProducerRec::Tile::mask) return fail("weight tile entry out of range");
        const int p = (int)p0.pix[a_idx];
        const bool unseen = !(seen & (1u << acc));
        if (first != unseen) return fail(first ? "overwrite of a live accumulator" : "accumulate into an uninitialised accumulator");
        const std::pair<int, int> kp{kc, p};
        if (!(last_kp[acc] < kp)) return fail("accumulation order is not canonical (k-chunk major, pixel ascending)");
        last_kp[acc] = kp;
        contrib[acc].push_back({p * 32 + (int)p0.tile[slot], kc});
        seen |= 1u << acc;
      }
      // ring safety
      for (int c = k - 1; c >= 0 && c >= k - 4 * TC2_NSLOT; --c) {
        const Step& o = steps[(size_t)c];
        if (!(o.beg < st.end && st.beg < o.end)) continue;
        if (c > k - dep) return fail("ring hazard: a region may be overwritten while it can still be read");
      }
      steps.push_back(st);
      if (flags & TcMmaRec::LAST) {
        for (uint32_t a = 0; a < hdr.n_acc; ++a) {
          std::vector<std::pair<int, int>> want;
          for (int kc = 0; kc < kch; ++kc)
            for (int e2 = tab.off[hdr.q[a]]; e2 < tab.off[hdr.q[a] + 1]; ++e2) want.push_back({tab.pairs[e2].x * 32 + tab.pairs[e2].y, kc});
          std::vector<std::pair<int, int>> got = contrib[a];
          std::sort(want.begin(), want.end()); std::sort(got.begin(), got.end());
          if (want != got) return fail("an item's MMAs do not cover exactly its pair list");
        }
        in_item = false;
      }
    }
    if (in_item) return fail("stream ends inside an item");
    for (int kk = item_k + 1; kk < pl.n_slots; ++kk)
      if (pl.eitems[(size_t)kk * n_pairs + pr] != -1) return fail("epilogue list has an item the stream lacks");
  }
  for (int v : assigned)
    if (v != 1) return fail("an item is not assigned to any CTA pair");
  return 0;
}

// Plan the schedule of layer-direction d for `n_mpairs` row pairs on `n_pairs` CTA pairs and upload it (allocates and
// synchronises), unless d already has one for that many row pairs.
static int tc2_get_schedule(TcDir& d, int n_mpairs, int n_pairs, std::vector<void*>* allocs) {
  for (auto& kv : d.by_mpairs)
    if (kv.first == n_mpairs) return 0;
  Tc2Plan plan;
  int rc;
  if ((rc = tc2_plan(d.N, d.K, d.tab, d.h_grid, d.w_grid, d.max_acc, d.force_maxb, d.epi, d.out_bytes, n_mpairs, n_pairs,
                     d.order, tc2_band_reverse(d.ld), &plan)))
    return rc;
  const cudaStream_t s = 0;
  Tc2Schedule sc;
  sc.maxb = plan.maxb;
  sc.n_pairs = n_pairs; sc.n_slots = plan.n_slots;
  if ((rc = tc_upload(allocs, plan.hdrs.data(), plan.hdrs.size() * sizeof(TcItem2), (void**)&sc.items, s))) return rc;
  if ((rc = tc_upload(allocs, plan.stream_p.data(), plan.stream_p.size() * sizeof(TcRec), (void**)&sc.stream_p, s))) return rc;
  if ((rc = tc_upload(allocs, plan.stream_m.data(), plan.stream_m.size() * sizeof(TcRec), (void**)&sc.stream_m, s))) return rc;
  if (n_pairs > TC2_MAX_PAIRS) { set_error("more CTA pairs than the kernel's parameter block holds"); return DGAN_ERR_UNSUPPORTED; }
  for (int pr = 0; pr <= n_pairs; ++pr) sc.heads.off[pr] = plan.stream_off[(size_t)pr];
  if ((rc = tc_upload(allocs, plan.eitems.data(), plan.eitems.size() * sizeof(int), (void**)&sc.eitems, s))) return rc;
  d.by_mpairs.push_back({n_mpairs, sc});
  return 0;
}

template <int NT, int MB, int KS, int EP, typename TOUT>
static cudaError_t tc2_optin() {
  return cudaFuncSetAttribute(tc_bsgemm2_kernel<NT, MB, KS, EP, TOUT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              Tc2Cfg<NT, MB, KS, EP, (int)sizeof(TOUT)>::SMEM_BYTES);
}

static int tc2_optin_all() {
#define TC2_OPTIN(NT, MB, KS, EP, T) DGAN_CUDA_CHECK((tc2_optin<NT, MB, KS, EP, T>()));
  TC2_KINDS(TC2_OPTIN)
#undef TC2_OPTIN
  return 0;
}

// Launch layer-direction d on n_pad rows with the schedule tc2_get_schedule made for them.  tm_a, tm_out: the tensor
// maps of its input and output; out: its output, of d.out_bytes per element.  fa.huber > 0: the Huber kind of d's final
// kind (tc_huber_epi), on d's plan.
static int tc2_launch(int64_t* launches, const TcDir& d, const CUtensorMap& tm_a, const CUtensorMap& tm_out, void* out,
                      int n_pad, const float* bias, cudaStream_t s, const TcFinalArgs& fa) {
  if (n_pad % (2 * kRowTile) != 0) { set_error("pair kernel needs n_pad % 256 == 0"); return DGAN_ERR_INVALID_ARG; }
  const int n_mpairs = n_pad / (2 * kRowTile);
  const Tc2Schedule* sc = nullptr;
  for (auto& kv : d.by_mpairs)
    if (kv.first == n_mpairs) sc = &kv.second;
  if (sc == nullptr) { set_error(d.name + ": no schedule planned for " + std::to_string(n_pad) + " rows"); return DGAN_ERR_INVALID_ARG; }
  const int grid = 2 * sc->n_pairs;       // pairs without work find -1 in slot 0 and fall through
  cudaError_t le = cudaSuccess;
  bool found = false;
  const int ksub = tc2_ksub(d.K);
  const int epi = fa.huber > 0.f ? tc_huber_epi(d.epi) : d.epi;
#define TC2_GO(NT, MB, KS, EP, T)                                                                                      \
  if (!found && d.N == NT && sc->maxb == MB && ksub == KS && epi == EP && d.out_bytes == (int)sizeof(T)) {             \
    found = true;                                                                                                     \
    le = launch_pdl(tc_bsgemm2_kernel<NT, MB, KS, EP, T>, dim3(grid), dim3(TC2_THREADS), Tc2Cfg<NT, MB, KS, EP, (int)sizeof(T)>::SMEM_BYTES, s, \
                    tm_a, d.tm_b, tm_out, sc->items, sc->stream_p, sc->stream_m, sc->heads, sc->eitems, sc->n_slots,     \
                    static_cast<T*>(out), n_pad, bias, d.bias_pstride, fa);                                            \
  }
  TC2_KINDS(TC2_GO)
#undef TC2_GO
  if (!found) { set_error("no tensor-core kernel instantiation for this layer-direction"); return DGAN_ERR_UNSUPPORTED; }
  (*launches)++;
  cudaError_t e = (le != cudaSuccess) ? le : cudaGetLastError();
  if (e != cudaSuccess) { set_error(std::string("tc_bsgemm2 launch: ") + cudaGetErrorString(e)); return DGAN_ERR_CUDA; }
  return 0;
}

}  // namespace dgan
