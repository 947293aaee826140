// The schedule records of the tensor-core path: the one definition of their bit layout.  tc2_plan encodes them,
// tc_bsgemm2_kernel reads single fields from the words it loads, tc2_check_plan and the validator's fault injections
// (dgan_debug_check_plans) decode them; nothing else knows a shift or a mask.
//
// One step of a CTA pair's work stream is two 32-byte records, one per role.  The host concatenates, per CTA pair, the
// steps of all the items assigned to it (LPT order), so producer and consumers each read one contiguous array.
//
// A step stages up to 4 input-pixel (A) tiles and up to 8 full weight tiles (B slots) for one k-chunk into a
// variable-size region of a circular shared-memory ring (offset chosen by the host, which simulates the ring), then
// issues rounds of MMAs that combine them.  Several A tiles per step let one weight tile serve several input pixels
// (stride-2 transposed conv: outputs of equal parity use the same tap with neighbouring inputs), which is what the
// L2->SM byte count cares about.
//
// producer record (the same for both ranks of a pair):
//   w[0]: ring offset / 1 KB [0,8) | k-chunk [8,12) | A tiles [12,15) | B slots [15,19) | dep [19,23)
//         dep = D: the region overlaps that of step k-D (or D = 8, barrier-slot reuse): wait until step k-D is consumed
//   w[1]: row pair mp [0,16)
//   w[2..3]: 4 x u16 input pixel of A tile i
//   w[4..5]: 8 x u8 weight tile [0,5) per B slot
// MMA record:
//   w[0]: ring offset / 1 KB [0,8) | A tiles [8,11) | rounds [11,16) | flags [16,18): 1 = first step of an item, 2 = last
//   w[1]: accumulators per round [0,8) (MAXB of the instantiation) | k16 MMAs per op [8,11) (KSUB); checked by the
//         validator only
//   w[2..7]: 24 x u8 op bytes, round-major, one per (round, accumulator): A tile [0,2) | B slot [2,6) | first MMA into
//            the accumulator [6,7).  B slot 15 = the all-zero tile outside the ring (the accumulator has nothing to add
//            in this round; never a first MMA).
// Item word (the consumers' epilogue list): window [16,31) | row pair [0,16); -1 = no item.
//
// The k-chunk needs no run-time check: tc_dir_supported (dgan_api.cu) refuses K > 512, i.e. more than 8 k-chunks.
#pragma once
#include <cstdint>

namespace dgan {

constexpr int TC2_MAX_A = 4, TC2_MAX_BSLOTS = 8, TC2_OP_BYTES = 24, TC2_ZERO_SLOT = 15, TC2_NSLOT = 8;
constexpr int TC2_RING_MAX_KB = 255;   // the operand ring's size cap (tc2_ring_bytes): offsets are 8-bit KB

struct __align__(16) TcRec { uint32_t w[8]; };

// Bits [SHIFT, SHIFT + WIDTH) of record word WORD.
template <int WORD, int SHIFT, int WIDTH>
struct TcField {
  static_assert(WORD >= 0 && WORD < 8 && SHIFT >= 0 && WIDTH >= 1 && WIDTH < 32 && SHIFT + WIDTH <= 32,
                "field outside its 32-bit record word");
  static constexpr int shift = SHIFT;
  static constexpr uint32_t mask = (1u << WIDTH) - 1u, bits = mask << SHIFT;
  __host__ __device__ static constexpr uint32_t get(uint32_t w) { return (w >> SHIFT) & mask; }
  static constexpr uint32_t put(uint32_t w, uint32_t v) { return (w & ~bits) | ((v & mask) << SHIFT); }
  static uint32_t of(const TcRec& r) { return get(r.w[WORD]); }
  static void set(TcRec& r, uint32_t v) { r.w[WORD] = put(r.w[WORD], v); }
  static constexpr uint32_t in_word(int w) { return w == WORD ? bits : 0u; }
};

// COUNT elements of WIDTH bits from record word WORD on, PER_WORD = 32 / WIDTH to a word, the lowest first.  The kernel
// uses the low USE bits of an element (get); the host reads and writes whole elements, so the validator sees the rest.
template <int WORD, int WIDTH, int COUNT, int USE = WIDTH>
struct TcArray {
  static constexpr int BITS = WIDTH, PER_WORD = 32 / WIDTH, WORDS = COUNT / PER_WORD;
  static_assert(32 % WIDTH == 0 && COUNT % PER_WORD == 0 && WORD >= 0 && WORD + WORDS <= 8 && USE <= WIDTH,
                "array outside the record");   // so it fills whole words
  static constexpr uint32_t elem = WIDTH == 32 ? ~0u : (1u << WIDTH) - 1u, mask = USE == 32 ? ~0u : (1u << USE) - 1u;
  // element i from the word that holds it (word WORD + i / PER_WORD)
  __host__ __device__ static constexpr uint32_t get(uint32_t w, int i) { return (w >> (WIDTH * (i & (PER_WORD - 1)))) & mask; }
  static uint32_t of(const TcRec& r, int i) { return (r.w[WORD + i / PER_WORD] >> (WIDTH * (i % PER_WORD))) & elem; }
  static void set(TcRec& r, int i, uint32_t v) {
    uint32_t& w = r.w[WORD + i / PER_WORD];
    const int s = WIDTH * (i % PER_WORD);
    w = (w & ~(elem << s)) | ((v & elem) << s);
  }
  static constexpr uint32_t in_word(int w) { return w >= WORD && w < WORD + WORDS ? ~0u : 0u; }
};

// Do these fields and arrays of one record leave each other's bits alone?
template <class... F>
constexpr bool tc_disjoint() {
  for (int w = 0; w < 8; ++w) {
    uint32_t used = 0;
    bool ok = true;
    ((ok = ok && (used & F::in_word(w)) == 0u, used |= F::in_word(w)), ...);
    if (!ok) return false;
  }
  return true;
}

// Producer record, decoded.
struct TcProducerRec {
  using Off = TcField<0, 0, 8>;     // ring offset / 1 KB
  using Kc = TcField<0, 8, 4>;      // k-chunk
  using NA = TcField<0, 12, 3>;     // A tiles
  using NB = TcField<0, 15, 4>;     // B slots
  using Dep = TcField<0, 19, 4>;    // dependency distance
  using Mp = TcField<1, 0, 16>;     // row pair
  using Pix = TcArray<2, 16, TC2_MAX_A>;               // input pixel of A tile i
  using Tile = TcArray<4, 8, TC2_MAX_BSLOTS, 5>;       // weight tile of B slot i
  uint32_t off = 0, kc = 0, nA = 0, nB = 0, dep = 0, mp = 0;
  uint32_t pix[TC2_MAX_A] = {}, tile[TC2_MAX_BSLOTS] = {};

  TcRec encode() const {
    TcRec r{};
    Off::set(r, off); Kc::set(r, kc); NA::set(r, nA); NB::set(r, nB); Dep::set(r, dep); Mp::set(r, mp);
    for (int i = 0; i < TC2_MAX_A; ++i) Pix::set(r, i, pix[i]);
    for (int i = 0; i < TC2_MAX_BSLOTS; ++i) Tile::set(r, i, tile[i]);
    return r;
  }
  static TcProducerRec decode(const TcRec& r) {
    TcProducerRec p;
    p.off = Off::of(r); p.kc = Kc::of(r); p.nA = NA::of(r); p.nB = NB::of(r); p.dep = Dep::of(r); p.mp = Mp::of(r);
    for (int i = 0; i < TC2_MAX_A; ++i) p.pix[i] = Pix::of(r, i);
    for (int i = 0; i < TC2_MAX_BSLOTS; ++i) p.tile[i] = Tile::of(r, i);
    return p;
  }
};

// MMA record, decoded.
struct TcMmaRec {
  using Off = TcField<0, 0, 8>;     // ring offset / 1 KB
  using NA = TcField<0, 8, 3>;      // A tiles
  using Rounds = TcField<0, 11, 5>;
  using Flags = TcField<0, 16, 2>;  // FIRST | LAST step of an item
  using MaxB = TcField<1, 0, 8>;    // accumulators per round
  using Ksub = TcField<1, 8, 3>;    // k16 MMAs per op
  using Ops = TcArray<2, 8, TC2_OP_BYTES>;             // op bytes (TcOp), [round][accumulator]
  static constexpr uint32_t FIRST = 1u, LAST = 2u;
  uint32_t off = 0, nA = 0, n_rounds = 0, flags = 0, maxb = 0, ksub = 0;
  uint8_t ops[TC2_OP_BYTES] = {};

  TcRec encode() const {
    TcRec r{};
    Off::set(r, off); NA::set(r, nA); Rounds::set(r, n_rounds); Flags::set(r, flags); MaxB::set(r, maxb); Ksub::set(r, ksub);
    for (int i = 0; i < TC2_OP_BYTES; ++i) Ops::set(r, i, ops[i]);
    return r;
  }
  static TcMmaRec decode(const TcRec& r) {
    TcMmaRec m;
    m.off = Off::of(r); m.nA = NA::of(r); m.n_rounds = Rounds::of(r); m.flags = Flags::of(r);
    m.maxb = MaxB::of(r); m.ksub = Ksub::of(r);
    for (int i = 0; i < TC2_OP_BYTES; ++i) m.ops[i] = (uint8_t)Ops::of(r, i);
    return m;
  }
};

// Op byte of an MMA record, decoded.
struct TcOp {
  using A = TcField<0, 0, 2>;       // A tile
  using Slot = TcField<0, 2, 4>;    // B slot, or TC2_ZERO_SLOT
  using First = TcField<0, 6, 1>;   // first MMA into the accumulator: overwrite it
  static constexpr uint32_t USED = A::bits | Slot::bits | First::bits;
  uint32_t a = 0, slot = 0, first = 0;

  uint8_t encode() const { return (uint8_t)First::put(Slot::put(A::put(0u, a), slot), first); }
  static TcOp decode(uint32_t e) { return TcOp{A::get(e), Slot::get(e), First::get(e)}; }
};
constexpr uint8_t TC2_PAD_OP = (uint8_t)TcOp::Slot::put(0u, TC2_ZERO_SLOT);   // A tile 0 x zero tile, accumulate

// Item word: a (window, row pair) item as a non-negative int; -1 = no item.
using TcItemMp = TcField<0, 0, 16>;
using TcItemWindow = TcField<0, 16, 15>;   // bit 31 stays clear
__host__ __device__ constexpr int tc2_item_window(int e) { return e >> TcItemWindow::shift; }
__host__ __device__ constexpr int tc2_item_mp(int e) { return e & (int)TcItemMp::mask; }
constexpr int tc2_item_word(int window, int mp) { return (int)TcItemWindow::put(TcItemMp::put(0u, (uint32_t)mp), (uint32_t)window); }

static_assert(tc_disjoint<TcProducerRec::Off, TcProducerRec::Kc, TcProducerRec::NA, TcProducerRec::NB, TcProducerRec::Dep,
                          TcProducerRec::Mp, TcProducerRec::Pix, TcProducerRec::Tile>(), "producer record fields overlap");
static_assert(tc_disjoint<TcMmaRec::Off, TcMmaRec::NA, TcMmaRec::Rounds, TcMmaRec::Flags, TcMmaRec::MaxB, TcMmaRec::Ksub,
                          TcMmaRec::Ops>(), "MMA record fields overlap");
static_assert(tc_disjoint<TcOp::A, TcOp::Slot, TcOp::First>(), "op byte fields overlap");
static_assert(tc_disjoint<TcItemMp, TcItemWindow>() && TcItemWindow::bits < 0x80000000u, "item word fields overlap");
static_assert(TcProducerRec::Mp::mask >= TcItemMp::mask, "row pair");
static_assert(TcProducerRec::Off::mask >= TC2_RING_MAX_KB - 1 && TcMmaRec::Off::mask >= TC2_RING_MAX_KB - 1, "ring offset");
static_assert(TcProducerRec::NA::mask >= TC2_MAX_A && TcMmaRec::NA::mask >= TC2_MAX_A && TcOp::A::mask >= TC2_MAX_A - 1,
              "A tiles per step");
static_assert(TcProducerRec::NB::mask >= TC2_MAX_BSLOTS, "B slots per step");
static_assert(TcOp::Slot::mask >= TC2_ZERO_SLOT && TC2_ZERO_SLOT >= TC2_MAX_BSLOTS, "B slot of an op");
static_assert(TcProducerRec::Dep::mask >= TC2_NSLOT, "dependency distance");
static_assert(TcMmaRec::Rounds::mask >= TC2_OP_BYTES, "rounds per step (one accumulator per round)");
static_assert(TcMmaRec::Flags::mask >= (TcMmaRec::FIRST | TcMmaRec::LAST), "item flags");
static_assert(TcOp::USED <= TcMmaRec::Ops::mask, "op byte wider than its element");

}  // namespace dgan
