// Negacyclic NTT over Z_q[X]/(X^N + 1) for sm_90a: device code and launch planning,
// shared by ntt.cu (one modulus per launch) and ntt_multi.cu (one modulus per group of
// polynomials inside one launch).
//
// What is computed is exactly the reference's transform
// (hexl/ntt/ntt-radix-2.cpp:17-261 forward, :330-519 inverse; butterflies
// hexl/ntt/ntt-default.hpp:28-42,112-125): Cooley-Tukey forward from natural to
// bit-reversed order, Gentleman-Sande inverse back with N^-1 folded into the
// last stage, Harvey lazy ranges ([0,4q) forward, [0,2q) inverse), Shoup
// twiddles.  HOW it is computed is GPU-shaped:
//
//   * The transform of size N = 2^n is the binary tree of its butterfly groups:
//     node 1 is the stage-0 group, node k has children 2k, 2k+1, and the twiddle
//     of node k is table[k] (for the forward table that IS the reference's
//     bit-reversed power layout).  A sub-transform rooted at node b over a
//     contiguous block of S elements uses node (b << s) + i in its stage s.
//   * "Row" kernel: one CTA owns a contiguous block of C = 2^c <= 8192
//     coefficients (a whole polynomial when N <= C, else one of N/C rows rooted
//     at node N/C + r).  Each thread holds 16 coefficients in registers and runs
//     4 butterfly stages per pass with no data movement; passes are separated by
//     a bank-conflict-free (XOR-swizzled) shared-memory transpose.  Global
//     loads/stores are fully coalesced and touch each coefficient exactly once.
//   * "Column" kernel (N > C only): the top log2(N/C) stages pair coefficients
//     C or more apart.  Each thread owns one column of R <= 32 coefficients
//     (stride S/R), keeps them in registers for log2(R) stages, twiddles staged
//     once per CTA in shared memory (they are the same for every column).
//   * Tiny N (< 16): one radix-2 stage per launch straight on global memory.
//
// No tensor cores: this is 64-bit integer modular arithmetic (IMAD-bound).
#pragma once
#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>

#include "internal.h"

namespace hexl_b200 {
namespace {

// f(Idx<I>{}) for I = BEGIN, ..., END - 1.  Every loop over a register array below is written this way, so each
// index is a compile-time constant by construction: a `#pragma unroll` loop is only unrolled when the compiler
// decides so, and a register array indexed at run time is placed in local memory (the sm_90a front end unrolled
// the stage loops, whose inner trip counts depend on the outer index, only partially).  The body reads the index
// as `constexpr int i = I;`.
template <int I>
struct Idx {
  __host__ __device__ constexpr operator int() const { return I; }
};
template <int BEGIN, int END, typename F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (BEGIN < END) {
    f(Idx<BEGIN>{});
    static_for<BEGIN + 1, END>(f);
  }
}

// ----------------------------------------------------------------- arithmetic
// H100 has no 64-bit integer multiplier; a 64x64 product is built from 32-bit
// IMADs (FMA pipe, full rate) while 64-bit adds/compares/selects cost two
// half-rate ALU-pipe instructions each.  Everything below is therefore written
// as multiply-add chains on 32-bit limbs, with as few compares as possible.
//
// Two arithmetic modes, chosen per modulus at launch time:
//
//  GENERIC (any q < 2^62): Harvey's lazy butterflies exactly as the reference
//    states them (ntt-default.hpp:28-42,112-125): forward values stay in [0,4q),
//    inverse values in [0,2q), one conditional subtraction per butterfly.
//
//  FAST (2^32 <= q < 2^56): the 2^64/q >= 256 of headroom replaces the per-butterfly
//    conditional subtractions.  The Shoup quotient is estimated from three 32x32
//    partial products (no lo*lo term, no carry between the middle terms: low by
//    at most 2), so a twiddle product lands in [0,4q).  Forward: X' = X + T,
//    Y' = X + 4q - T, ranges grow by 4q per stage (<= (4 + 4*20) q = 84q < 2^63)
//    and one Barrett reduction per coefficient at the very end restores [0,q).
//    Inverse: sums are left unreduced inside a register pass; a pass that starts
//    with all values < 8q ends with slot bounds 4*2^(K-1-h) q (h = highest set
//    register bit) or 8*2^K q (all-sum slots), and only slots above 8q are
//    Barrett-reduced at the pass boundary (4 of 16 for a 4-stage pass).  The
//    largest transient is 2 * 8*2^4 * q = 256q < 2^64 for q < 2^56.
//
//  WIDE (2^56 <= q < 2^61): Harvey's butterflies with every lazy range doubled (forward
//    [0,8q), inverse [0,4q); 8q < 2^64), which makes room for FAST's three-product quotient
//    estimate (product in [0,4q)) in place of the exact 64x64 high half: one IMAD.WIDE less
//    per butterfly than GENERIC for the 57..61-bit primes HE parameter sets like best.
//
//  SMALL (q < 2^30): 4q < 2^32, so every lazy value is ONE 32-bit word.  Same Harvey
//    butterflies as GENERIC with beta = 2^32 (twiddle pairs {w, floor(w 2^32/q)}):
//    one IMAD.WIDE + two IMADs per twiddle product instead of 6 + 4, conditional
//    subtraction as min(x, x - 2q).  Registers and shared memory hold 32-bit words
//    (global memory keeps the API's 64-bit coefficients); at ~1/4 of the multiplier
//    work these kernels are HBM-bound.
//  All modes produce the same canonical values; lazy outputs (out_mf 4 / 2)
//  are congruent and inside the advertised range.
enum : int { kGeneric = 0, kFast = 1, kSmall = 2, kWide = 3 };

// element and twiddle types of a mode
template <int MODE>
struct Ar {
  using E = u64;
  using Tw = Twiddle;
};
template <>
struct Ar<kSmall> {
  using E = unsigned;
  using Tw = Twiddle32;
};
constexpr u64 kFastModulusLimit = 1ull << 56;
constexpr u64 kWideModulusLimit = 1ull << 61;
constexpr int kFastProd = 4;   // FAST: a twiddle product is < 4q
constexpr int kFastBound = 8;  // FAST inverse: every value is < 8q at a pass boundary

struct Mod {
  u64 q, two_q, four_q, mu;  // mu = floor(2^64 / q)
  unsigned n0, n1;           // low / high word of 2^64 - q
  unsigned zero;             // 0, unknown to the compiler (add_alu)
};

__device__ __forceinline__ unsigned lo32(u64 x) { return (unsigned)x; }
__device__ __forceinline__ unsigned hi32(u64 x) { return (unsigned)(x >> 32); }
__device__ __forceinline__ u64 join(unsigned lo, unsigned hi) {
  u64 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "r"(lo), "r"(hi));
  return r;
}
__device__ __forceinline__ void split(u64 x, unsigned& lo, unsigned& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=r"(lo), "=r"(hi) : "l"(x));
}
// The multiply primitives are pinned with PTX so that ptxas keeps them on the
// FMA-heavy pipe (IMAD / IMAD.WIDE, one every 2 cycles per scheduler) instead of
// turning accumulations into 64-bit IADD3 pairs plus register-pair moves on the
// ALU pipe, which is the scarcer resource in these kernels (tools/inst_bench.cu;
// IMAD.HI is ~3x slower than IMAD.WIDE and is never used).
__device__ __forceinline__ u64 mul_wide(unsigned a, unsigned b) {
  u64 r;
  asm("mul.wide.u32 %0, %1, %2;" : "=l"(r) : "r"(a), "r"(b));
  return r;
}
__device__ __forceinline__ u64 mad_wide(unsigned a, unsigned b, u64 c) {
  u64 r;
  asm("mad.wide.u32 %0, %1, %2, %3;" : "=l"(r) : "r"(a), "r"(b), "l"(c));
  return r;
}
__device__ __forceinline__ unsigned mad_lo(unsigned a, unsigned b, unsigned c) {
  unsigned r;
  asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
  return r;
}

// a + b with the carry into the high word on the ALU pipe.  ptxas puts the high half of a two-operand 64-bit add on
// the multiplier pipe (IMAD.X) whenever it judges the ALU busier, which in these kernels it always is by that
// measure although the multiplier is the bound.  With a third operand -- m.zero, 0 at run time but a kernel parameter
// the compiler cannot see through -- the low word produces two carries and the high word becomes a three-input
// IADD3.X, which has no IMAD form.  (Checked in SASS: tests/test_pipe_budget.py.)
__device__ __forceinline__ u64 add_alu(u64 a, u64 b, const Mod& m) { return a + b + m.zero; }

__device__ __forceinline__ Twiddle ld_tw(const Twiddle* p) {
  const ulonglong2 v = __ldg(reinterpret_cast<const ulonglong2*>(p));
  Twiddle t;
  t.w = v.x;
  t.wp = v.y;
  return t;
}
__device__ __forceinline__ Twiddle32 ld_tw(const Twiddle32* p) {
  const uint2 v = __ldg(reinterpret_cast<const uint2*>(p));
  Twiddle32 t;
  t.w = v.x;
  t.wp = v.y;
  return t;
}

// floor(a*b / 2^64) - {0,1,2}: a1*b1 + hi32(a1*b0) + hi32(a0*b1).  The two high halves are summed first
// (one IADD3 + IADD3.X pair, a genuine 64-bit value in a register pair) and ride in as the accumulator of
// a1*b1.  Folding them in one at a time -- as multiply-by-one wide mads, or as two 64-bit adds -- makes
// ptxas zero-extend a high half into a fresh register pair (MOV + IMAD.MOV/HFMA2 per butterfly, the latter
// on the multiplier pipe that bounds these kernels).
__device__ __forceinline__ u64 mulhi_approx(u64 a, u64 b) {
  unsigned a0, a1, b0, b1;
  split(a, a0, a1);
  split(b, b0, b1);
  const u64 hs = (u64)hi32(mul_wide(a1, b0)) + (u64)hi32(mul_wide(a0, b1));
  return mad_wide(a1, b1, hs);
}

// low 64 bits of x*w + Q*(2^64 - q): 2 wide and 4 narrow IMADs, no adds
__device__ __forceinline__ u64 mad_chain(u64 x, u64 w, u64 Q, const Mod& m) {
  unsigned x0, x1, w0, w1, q0, q1, t0, t1;
  split(x, x0, x1);
  split(w, w0, w1);
  split(Q, q0, q1);
  split(mad_wide(q0, m.n0, mul_wide(x0, w0)), t0, t1);
  t1 = mad_lo(x0, w1, t1);
  t1 = mad_lo(x1, w0, t1);
  t1 = mad_lo(q0, m.n1, t1);
  t1 = mad_lo(q1, m.n0, t1);
  return join(t0, t1);
}

// x*w mod q, lazily: exact quotient -> [0,2q); approximate quotient -> [0,4q)
template <int MODE>
__device__ __forceinline__ u64 mul_tw(u64 x, const Twiddle w, const Mod& m) {
  const u64 Q = (MODE == kFast || MODE == kWide) ? mulhi_approx(x, w.wp) : mulhi(x, w.wp);
  return mad_chain(x, w.w, Q, m);
}
__device__ __forceinline__ u64 mul_tw_exact(u64 x, const Twiddle w, const Mod& m) {
  return mad_chain(x, w.w, mulhi(x, w.wp), m);
}

// any 64-bit value -> [0,2q):  x - floor(x*mu/2^64)*q, mu = floor(2^64/q)
__device__ __forceinline__ u64 barrett_lazy(u64 x, const Mod& m) {
  unsigned q0, q1, t0, t1;
  split(mulhi(x, m.mu), q0, q1);
  split(mad_wide(q0, m.n0, x), t0, t1);
  t1 = mad_lo(q0, m.n1, t1);
  t1 = mad_lo(q1, m.n0, t1);
  return join(t0, t1);
}
// Same for q >= 2^32, where mu < 2^32 and the quotient is a single 32-bit word:
// Q = floor(x*mu / 2^64) or one less = hi32(x1*mu + hi32(x0*mu)), the carry into the high word taken with
// an explicit add.cc / addc pair (a 64-bit add of the zero-extended high half costs two register moves more).
__device__ __forceinline__ u64 barrett_lazy_bigq(u64 x, const Mod& m) {
  unsigned x0, x1, s0, s1, t0, t1, Q, dummy;
  split(x, x0, x1);
  const unsigned mu0 = lo32(m.mu);
  split(mul_wide(x1, mu0), s0, s1);
  const unsigned h = hi32(mul_wide(x0, mu0));
  asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, %4, 0;" : "=r"(dummy), "=r"(Q) : "r"(s0), "r"(h), "r"(s1));
  split(mad_wide(Q, m.n0, x), t0, t1);
  return join(t0, mad_lo(Q, m.n1, t1));
}
// any 64-bit value -> [0,3q) for q >= 2^32 with one wide product less: Q = hi32(x1*mu) is floor(x*mu/2^64) or
// up to two less.  Enough wherever the result only has to drop below a lazy bound (FAST inverse fix-ups).
// x is added with a three-input IADD3.X rather than as the accumulator of the wide product: the coefficient arrays
// do not keep a value's two words in an aligned register pair, and ptxas then splits the wide mad into a product
// plus a 64-bit add whose high half lands on IMAD.X.
__device__ __forceinline__ u64 barrett_lazy3_bigq(u64 x, const Mod& m) {
  unsigned x0, x1, p0, p1;
  split(x, x0, x1);
  const unsigned Q = hi32(mul_wide(x1, lo32(m.mu)));
  split(mul_wide(Q, m.n0), p0, p1);
  const unsigned qn1 = Q * m.n1;
  const u64 s = x + join(p0, p1);
  return join(lo32(s), hi32(s) + qn1);
}

// any 64-bit value -> [0, q) (Barrett with floor(2^64/q), then one conditional subtraction; q < 2^63)
__device__ __forceinline__ u64 reduce_any(u64 x, const Mod& m) { return csub_s(barrett_lazy(x, m), m.q); }
__device__ __forceinline__ unsigned reduce_any(unsigned x, const Mod& m) { return x % (unsigned)m.q; }

// Second operand of an inverse transform that multiplies on load (NttMulti::mul): row pointer + the generalised-Barrett
// constants of NttDeviceParams.
struct ProdIn {
  const u64* b;
  u64 mu;
  int shift;
};
// x*y mod q for canonical x, y, lazily (eltwise-mult-mod-internal.hpp:52-99 without the final conditional
// subtraction): U = x*y (four wide products, both halves), c1 = floor(U / 2^shift), Q = floor(c1*mu / 2^64),
// U - Q*q.  Exact Q -> [0,2q) (GENERIC inverse inputs); Q low by up to two more (FAST / WIDE) -> [0,4q), inside what
// those modes' first inverse stage accepts.
template <int MODE>
__device__ __forceinline__ u64 prod_lazy(u64 x, u64 y, const Mod& m, u64 pmu, int shift) {
  unsigned x0, x1, y0, y1, q0, q1, t0, t1;
  split(x, x0, x1);
  split(y, y0, y1);
  const u64 t = mul_wide(x0, y0);
  const u64 uu = mad_wide(x0, y1, (u64)hi32(t));
  const u64 vv = mad_wide(x1, y0, (u64)lo32(uu));
  const u64 hi = mad_wide(x1, y1, (u64)hi32(uu) + (u64)hi32(vv));
  const u64 lo = join(lo32(t), lo32(vv));
  const u64 c1 = shift ? ((lo >> shift) | (hi << (64 - shift))) : lo;
  const u64 Q = (MODE == kFast || MODE == kWide) ? mulhi_approx(c1, pmu) : mulhi(c1, pmu);
  split(Q, q0, q1);
  split(mad_wide(q0, m.n0, lo), t0, t1);
  t1 = mad_lo(q0, m.n1, t1);
  t1 = mad_lo(q1, m.n0, t1);
  return join(t0, t1);
}

// ----------------------------------------------------------------- butterflies
template <int MODE, typename TW>
__device__ __forceinline__ void fwd_bfly(u64& X, u64& Y, const TW& w, const Mod& m) {
  if (MODE == kFast) {
    const u64 T = mul_tw<kFast>(Y, w, m);  // [0,4q)
    Y = X + m.four_q - T;
    X = add_alu(X, T, m);
  } else if (MODE == kWide) {
    // (the 64-bit compare form here: with csub_s ptxas moves the high-word adds from IMAD.X to the ALU pipe, which
    // this mode loads as much as the multiplier)
    const u64 tx = csub(X, m.four_q);      // [0,8q) -> [0,4q)
    const u64 T = mul_tw<kWide>(Y, w, m);  // [0,4q)
    X = add_alu(tx, T, m);
    Y = tx + m.four_q - T;
  } else {
    const u64 tx = csub_s(X, m.two_q);
    const u64 T = mul_tw<kGeneric>(Y, w, m);  // [0,2q)
    X = tx + T;
    Y = tx + m.two_q - T;
  }
}

// cq: a multiple of q at least as large as any Y of this stage (FAST only)
template <int MODE, typename TW>
__device__ __forceinline__ void inv_bfly(u64& X, u64& Y, const TW& w, const Mod& m, u64 cq) {
  if (MODE == kFast) {
    const u64 d = X + cq - Y;
    X = add_alu(X, Y, m);
    Y = mul_tw<kFast>(d, w, m);  // [0,4q)
  } else if (MODE == kWide) {
    const u64 s = add_alu(X, Y, m);  // inputs in [0,4q)
    const u64 d = X + m.four_q - Y;
    X = csub_s(s, m.four_q);
    Y = mul_tw<kWide>(d, w, m);  // [0,4q)
  } else {
    const u64 s = X + Y;
    const u64 d = X + m.two_q - Y;
    X = csub_s(s, m.two_q);
    Y = mul_tw<kGeneric>(d, w, m);
  }
}

// Root stage of the inverse with N^-1 folded in (ntt-radix-2.cpp:484-509).  The
// Shoup multiply accepts any 64-bit input, so the sum needs no reduction first.
// FAST / WIDE: the three-product quotient, products in [0,4q) (4q < 2^63 there);
// GENERIC keeps the exact quotient, [0,2q), since 4q may not fit 64 bits.
template <int MODE>
__device__ __forceinline__ void inv_bfly_last(u64& X, u64& Y, const Twiddle inv_n, const Twiddle inv_n_w,
                                              const Mod& m, u64 cq) {
  const u64 s = add_alu(X, Y, m);
  const u64 d = X + cq - Y;
  if (MODE == kFast || MODE == kWide) {
    X = mul_tw<MODE>(s, inv_n, m);    // [0,4q)
    Y = mul_tw<MODE>(d, inv_n_w, m);  // [0,4q)
  } else {
    X = mul_tw_exact(s, inv_n, m);    // [0,2q)
    Y = mul_tw_exact(d, inv_n_w, m);  // [0,2q)
  }
}

// forward output: GENERIC [0,4q) / WIDE [0,8q) / FAST anything  ->  [0,q) (out_mf 1) or < 4q (out_mf 4)
template <int MODE>
__device__ __forceinline__ u64 fwd_out(u64 v, const Mod& m, int out_mf) {
  if (MODE == kFast) v = barrett_lazy3_bigq(v, m);  // [0,3q)
  if (MODE == kWide) v = csub_s(v, m.four_q);       // [0,8q) -> [0,4q)
  return out_mf == 1 ? csub_s(csub_s(v, m.two_q), m.q) : v;
}
// inverse output after the folded root stage: FAST / WIDE [0,4q), GENERIC [0,2q)  ->  [0,2q) (out_mf 2) or
// [0,q) (out_mf 1)
template <int MODE>
__device__ __forceinline__ u64 inv_out(u64 v, const Mod& m, int out_mf) {
  if (MODE == kFast || MODE == kWide) v = csub_s(v, m.two_q);
  return out_mf == 1 ? csub_s(v, m.q) : v;
}

// ---- SMALL mode (q < 2^30): the same butterflies on 32-bit words
__device__ __forceinline__ unsigned csub32(unsigned x, unsigned c) { return min(x, x - c); }  // x < 2c
// x*w mod q in [0,2q) for any 32-bit x:  x*w - hi32(x*wp)*q  (mod 2^32)
__device__ __forceinline__ unsigned mul_tw32(unsigned x, const Twiddle32 w, const Mod& m) {
  const unsigned Q = hi32(mul_wide(x, w.wp));
  return mad_lo(Q, m.n0, x * w.w);  // n0 = low word of 2^64 - q = 2^32 - q
}
template <int MODE, typename TW>
__device__ __forceinline__ void fwd_bfly(unsigned& X, unsigned& Y, const TW& w, const Mod& m) {
  const unsigned two_q = lo32(m.two_q);
  const unsigned tx = csub32(X, two_q);
  const unsigned T = mul_tw32(Y, w, m);
  X = tx + T;
  Y = tx + two_q - T;
}
template <int MODE, typename TW>
__device__ __forceinline__ void inv_bfly(unsigned& X, unsigned& Y, const TW& w, const Mod& m, unsigned) {
  const unsigned two_q = lo32(m.two_q);
  const unsigned s = X + Y;
  const unsigned d = X + two_q - Y;
  X = csub32(s, two_q);
  Y = mul_tw32(d, w, m);
}
template <int MODE>
__device__ __forceinline__ void inv_bfly_last(unsigned& X, unsigned& Y, const Twiddle32 inv_n,
                                              const Twiddle32 inv_n_w, const Mod& m, unsigned) {
  const unsigned s = X + Y;
  const unsigned d = X + lo32(m.two_q) - Y;
  X = mul_tw32(s, inv_n, m);
  Y = mul_tw32(d, inv_n_w, m);
}
template <int MODE>
__device__ __forceinline__ unsigned fwd_out(unsigned v, const Mod& m, int out_mf) {
  return out_mf == 1 ? csub32(csub32(v, lo32(m.two_q)), lo32(m.q)) : v;
}
template <int MODE>
__device__ __forceinline__ unsigned inv_out(unsigned v, const Mod& m, int out_mf) {
  return out_mf == 1 ? csub32(v, lo32(m.q)) : v;
}

// FAST inverse bookkeeping.  After K unreduced GS stages on register bits 0..K-1
// of values that all started below kFastBound*q, the slot whose low K bits are
// `low` is bounded by (in units of q):
__host__ __device__ constexpr int inv_slot_bound(int K, int low) {
  if (low == 0) return kFastBound << K;
  int h = 0;
  for (int b = 0; b < K; ++b)
    if (low & (1 << b)) h = b;
  return kFastProd << (K - 1 - h);
}
// the largest Y entering GS stage s of such a pass (what cq must cover)
__host__ __device__ constexpr int inv_stage_cover(int s) { return kFastBound << s; }
// the multiple of q added before the subtraction of inverse stage `step` of a pass
template <int MODE>
__device__ __forceinline__ typename Ar<MODE>::E stage_cq(int step, const Mod& m) {
  if (MODE == kFast) return (u64)inv_stage_cover(step) * m.q;
  if (MODE == kWide) return m.four_q;
  return (typename Ar<MODE>::E)m.two_q;
}

// Brings every slot of such a pass back below kFastBound*q: a Barrett reduction (< 3q) where the bound exceeds
// kFastFixupCsub*q, else one conditional subtraction per halving (16q -> 8q, 32q -> 16q -> 8q).
constexpr int kFastFixupCsub = 32;
template <int K, int NSLOTS, int E = 0>
__device__ __forceinline__ void inv_pass_fixup(u64* v, const Mod& m) {
  if constexpr (E < NSLOTS) {
    constexpr int bound = inv_slot_bound(K, E & ((1 << K) - 1));
    if constexpr (bound > kFastFixupCsub) {
      v[E] = barrett_lazy3_bigq(v[E], m);
    } else {
      if constexpr (bound > 2 * kFastBound) v[E] = csub_s(v[E], m.four_q << 2);
      if constexpr (bound > kFastBound) v[E] = csub_s(v[E], m.four_q << 1);
    }
    inv_pass_fixup<K, NSLOTS, E + 1>(v, m);
  }
}

// --------------------------------------------------------------- row kernel
// Shared-memory index swizzle for 64-bit elements: XOR the 8-byte-bank index
// (low 4 bits) with the next 4 bits.  Conflict-free (per half-warp) for every
// access pattern of the passes below; a bijection inside each aligned block of
// 16 elements.
// For 32-bit elements (SMALL mode) the same shift with a 5-bit mask spreads the 32
// lanes of a warp over the 32 four-byte banks (tests/test_kernel_model.py checks both).
template <typename E>
__device__ __forceinline__ unsigned swz(unsigned j) {
  return j ^ ((j >> 4) & (sizeof(E) == 8 ? 15u : 31u));
}
// 64-bit rows (round 2) are PADDED instead of swizzled: element j lives at j + (j >> 4), one 8-byte pad per 16
// elements.  Equally conflict-free for every access pattern of the passes (tests/test_kernel_model.py), and -- unlike
// the XOR -- affine in the register slot: for the slot-e element of a thread, pad(U | e << LB) = pad(U) + pad_slot(e)
// with a compile-time pad_slot, so the 16 accesses of an exchange are ONE address plus immediate offsets instead of a
// LOP3/LEA per access (~4 % of the row kernels' instructions).  The 32-bit rows of SMALL mode keep the XOR swizzle.
__host__ __device__ constexpr unsigned pad_slot(int e, int lb) { return ((unsigned)e << lb) + (((unsigned)e << lb) >> 4); }
template <typename E>
__host__ __device__ constexpr unsigned row_elems(int logc) {
  return (1u << logc) + (sizeof(E) == 8 ? (1u << logc) >> 4 : 0u);
}

// Coefficient index held in register slot e of thread u when the 4 register
// bits sit at bit position LB of the row-local index.
template <int LB>
__device__ __forceinline__ unsigned reg_index(unsigned u, int e) {
  return ((u >> LB) << (LB + 4)) | ((unsigned)e << LB) | (u & ((1u << LB) - 1u));
}

// Butterfly stages on row-local index bits HB..LOB (all inside [LB, LB+3]).
// FWD: bits descend (CT).  INV: bits ascend (GS), LOB == LB.
// Sub-tree twiddle tables in shared memory.  A full 4-stage pass whose register
// bits sit at LB runs, for thread u, the radix-16 sub-tree rooted at node
// (base << d) + (u >> LB), d = LOGC - LB - 4.  The first two passes of a row have
// d = 0 (one root) and d = 4 (16 roots): their 17 x 15 twiddles are fetched once
// per row by a cooperative load and then read with LDS (tens of cycles) instead
// of 15 dependent-latency L2 loads per thread per pass.  Layout: 16 entries per
// root, local node l = 2^s + i at slot l; root table 0 first, then the 16 tables
// of depth 4.
constexpr int kRowTwEntries = 17 * 16;
template <int LOGC, int LB, int HB, int LOB>
struct PassTw {
  static constexpr int kDepth = LOGC - LB - 4;
  static constexpr bool kShared = LOGC >= 8 && (HB - LOB) == 3 && (kDepth == 0 || kDepth == 4);
  static constexpr int kOffset = kDepth == 0 ? 0 : 16;
};

template <int LOGC, typename Tw>
__device__ __forceinline__ void load_row_twiddles(Tw* stab, unsigned tid, unsigned nthreads, u64 base,
                                                  const Tw* __restrict__ tw) {
  for (int idx = tid; idx < kRowTwEntries; idx += nthreads) {
    const int l = idx & 15;
    if (l == 0) continue;
    const u64 root = idx < 16 ? base : (base << 4) + ((idx - 16) >> 4);
    const int s = 31 - __clz(l);
    stab[idx] = ld_tw(tw + (root << s) + (l - (1 << s)));
  }
}

// Butterfly stages on row-local index bits HB..LOB (all inside [LB, LB+3]).
// FWD: bits descend (CT).  INV: bits ascend (GS), LOB == LB.
template <int MODE, int LOGC, int LB, int HB, int LOB, bool FWD>
__device__ __forceinline__ void reg_stages(typename Ar<MODE>::E (&v)[16], unsigned u, u64 base,
                                           const typename Ar<MODE>::Tw* __restrict__ tw,
                                           const typename Ar<MODE>::Tw* stab, const Mod& m, bool fold,
                                           typename Ar<MODE>::Tw inv_n, typename Ar<MODE>::Tw inv_n_w) {
  using PT = PassTw<LOGC, LB, HB, LOB>;
  using Tw = typename Ar<MODE>::Tw;
  const Tw* sroot = stab + PT::kOffset + ((u >> LB) << 4);  // this thread's sub-tree table
  static_for<0, HB - LOB + 1>([&](auto STEP) {
    constexpr int step = STEP;
    constexpr int beta = FWD ? HB - step : LOB + step;  // index bit of this stage
    constexpr int eb = beta - LB;                       // register bit
    constexpr int sp = LOGC - 1 - beta;                 // stage number inside the row
    // FAST inverse: multiple of q covering every Y of this stage (GENERIC: 2q)
    const typename Ar<MODE>::E cq = stage_cq<MODE>(step, m);
    auto fetch = [&](int g) {
      if constexpr (PT::kShared)
        return sroot[(8 >> eb) + g];                // local node 2^s' + g, s' = 3 - eb
      else if constexpr (LOGC == 12 && LB == 0)
        // last pass of a 4096-point row: level 3 - beta of the deepest four, stored lane-major (internal.h)
        return ld_tw(tw + (base << (LOGC - 1 - beta)) + lane_major(u, 0, 3 - beta) + (g << 5));
      else
        return ld_tw(tw + (base << (LOGC - 1 - beta)) + ((u64)(u >> LB) << (LB + 3 - beta)) + g);
    };
    auto groups = [&] {
      // Forward stages fetch all their twiddles first.  The inverse fetches each group's twiddle just before its
      // butterflies: its first stage per pass has 8 groups, and 8 twiddles held next to the 16 coefficients push
      // the 64-bit row kernels past their register bound.
      Tw wc[8 >> eb];
      if constexpr (FWD) static_for<0, (8 >> eb)>([&](auto G) { constexpr int g = G; wc[g] = fetch(g); });
      static_for<0, (8 >> eb)>([&](auto G) {
        constexpr int g = G;
        Tw wt;
        if constexpr (FWD)
          wt = wc[g];
        else
          wt = fetch(g);
        static_for<0, (1 << eb)>([&](auto L) {
          constexpr int e = (g << (eb + 1)) | L;
          if constexpr (FWD)
            fwd_bfly<MODE>(v[e], v[e | (1 << eb)], wt, m);
          else
            inv_bfly<MODE>(v[e], v[e | (1 << eb)], wt, m, cq);
        });
      });
    };
    if constexpr (!FWD && sp == 0) {
      if (fold) {
        // root stage of the whole transform: one group, N^-1 folded in
        static_for<0, (1 << eb)>([&](auto L) {
          constexpr int l = L;
          inv_bfly_last<MODE>(v[l], v[l | (1 << eb)], inv_n, inv_n_w, m, cq);
        });
      } else {
        groups();
      }
    } else {
      groups();
    }
  });
  if constexpr (!FWD && MODE == kFast) {
    if (!(fold && LOGC - 1 - HB == 0)) inv_pass_fixup<HB - LOB + 1, 16>(v, m);
  }
}

// Transpose between two register layouts through shared memory.  The exchange
// only permutes thread-id bits [min(LB), max(LB)), so when max(LB) <= 5 every
// value stays inside one warp and __syncwarp() replaces the CTA barrier.  No
// barrier is needed after the reads: the next exchange writes exactly the
// addresses this thread has just read (same layout), which nobody else touches.
template <int LB_FROM, int LB_TO, typename E>
__device__ __forceinline__ void smem_exchange(E (&v)[16], E* srow, unsigned u) {
  constexpr bool kWarpLocal = (LB_FROM > LB_TO ? LB_FROM : LB_TO) <= 5;
  if constexpr (sizeof(E) == 8) {
    const unsigned uf = reg_index<LB_FROM>(u, 0), ut = reg_index<LB_TO>(u, 0);
    E* wr = srow + (uf + (uf >> 4));
    const E* rd = srow + (ut + (ut >> 4));
    static_for<0, 16>([&](auto I) { constexpr int e = I; wr[pad_slot(e, LB_FROM)] = v[e]; });
    if (kWarpLocal)
      __syncwarp();
    else
      __syncthreads();
    static_for<0, 16>([&](auto I) { constexpr int e = I; v[e] = rd[pad_slot(e, LB_TO)]; });
  } else {
    static_for<0, 16>([&](auto I) { constexpr int e = I; srow[swz<E>(reg_index<LB_FROM>(u, e))] = v[e]; });
    if (kWarpLocal)
      __syncwarp();
    else
      __syncthreads();
    static_for<0, 16>([&](auto I) { constexpr int e = I; v[e] = srow[swz<E>(reg_index<LB_TO>(u, e))]; });
  }
}

// Forward passes after pass 0: register bits move down by 4 per pass, clamped at 0.
template <int MODE, int LOGC, int PASS>
__device__ __forceinline__ void fwd_passes(typename Ar<MODE>::E (&v)[16], typename Ar<MODE>::E* srow, unsigned u,
                                           u64 base, const typename Ar<MODE>::Tw* tw,
                                           const typename Ar<MODE>::Tw* stab, const Mod& m) {
  using Tw = typename Ar<MODE>::Tw;
  constexpr int PREV_LB = (LOGC - 4 * PASS) > 0 ? (LOGC - 4 * PASS) : 0;
  constexpr int HB = LOGC - 4 * PASS - 1;  // highest index bit not yet processed
  if constexpr (HB >= 0) {
    constexpr int LB = (HB - 3) > 0 ? (HB - 3) : 0;
    smem_exchange<PREV_LB, LB>(v, srow, u);
    reg_stages<MODE, LOGC, LB, HB, LB, true>(v, u, base, tw, stab, m, false, Tw{}, Tw{});
    fwd_passes<MODE, LOGC, PASS + 1>(v, srow, u, base, tw, stab, m);
  }
}

// Inverse passes: mirror image.  PASS counts down; pass P-1 is done first.
template <int MODE, int LOGC, int PASS>
__device__ __forceinline__ void inv_passes(typename Ar<MODE>::E (&v)[16], typename Ar<MODE>::E* srow, unsigned u,
                                           u64 base, const typename Ar<MODE>::Tw* tw,
                                           const typename Ar<MODE>::Tw* stab, const Mod& m, bool fold,
                                           typename Ar<MODE>::Tw inv_n, typename Ar<MODE>::Tw inv_n_w) {
  // forward pass PASS handled bits HB..LB; the inverse handles the same bits ascending
  constexpr int HB = LOGC - 4 * PASS - 1;
  constexpr int LB = (HB - 3) > 0 ? (HB - 3) : 0;
  reg_stages<MODE, LOGC, LB, HB, LB, false>(v, u, base, tw, stab, m, fold, inv_n, inv_n_w);
  if constexpr (PASS > 0) {
    constexpr int NHB = LOGC - 4 * (PASS - 1) - 1;
    constexpr int NLB = (NHB - 3) > 0 ? (NHB - 3) : 0;
    smem_exchange<LB, NLB>(v, srow, u);
    inv_passes<MODE, LOGC, PASS - 1>(v, srow, u, base, tw, stab, m, fold, inv_n, inv_n_w);
  }
}

// 64-bit row kernels of 256 threads: 3 CTAs per SM (80 registers).  One H100 80GB HBM3 (power limit not recorded), 2^28 coefficients, 55-bit
// q, N = 2^16 (tools/tune_split.py): forward / inverse 3.47 / 3.71 ms, against 3.58 / 3.94 ms with 2 CTAs per SM.
constexpr int kRowMinBlocks = 3;
constexpr int kRowMinBlocks512 = 2;   // rows of 512 threads (C = 8192), both word sizes
constexpr int kRowMinBlocksSmall = 4;  // 32-bit rows of at most 256 threads
template <int LOGC, int MODE = kGeneric>
struct RowCfg {
  using E = typename Ar<MODE>::E;
  using Tw = typename Ar<MODE>::Tw;
  static constexpr int C = 1 << LOGC;
  static constexpr int T = C / 16;                        // threads per row
  static constexpr int ROWS = T >= 256 ? 1 : 256 / T;     // rows per CTA
  static constexpr int THREADS = T * ROWS;
  static constexpr int PASSES = (LOGC + 3) / 4;
  static constexpr bool TW_TABLES = LOGC >= 8;          // sub-tree twiddles staged in shared memory
  static constexpr size_t ROW_BYTES = (size_t)row_elems<E>(LOGC) * sizeof(E) + (TW_TABLES ? kRowTwEntries * sizeof(Tw) : 0);
  static constexpr size_t SMEM = (size_t)ROWS * ROW_BYTES;
  static constexpr int MIN_BLOCKS = THREADS <= 256 ? (MODE == kSmall ? kRowMinBlocksSmall : kRowMinBlocks)
                                                   : (THREADS == 512 ? kRowMinBlocks512 : 1);
};

// Global-memory access policies for coefficients.  Streaming (evict-first) for
// data touched once; L2 variants for the intermediate a fused kernel hands from
// its column phase to its row phase (written by one CTA, read by another).
// kSmemRow: the "global" side is a row of E in shared memory; kSmemRowPad: the same in the padded layout of the 64-bit
// exchanges (element j at j + j / 16), so that the row can double as its own exchange buffer
enum : int { kStream = 0, kViaL2 = 1, kSmemRow = 2, kSmemRowPad = 3 };
template <int POLICY>
__device__ __forceinline__ u64 ld_coef(const u64* p) {
  return POLICY == kViaL2 ? __ldcg(p) : __ldcs(p);
}
template <int POLICY>
__device__ __forceinline__ void st_coef(u64* p, u64 v) {
  if (POLICY == kViaL2)
    __stcg(p, v);
  else
    __stcs(p, v);
}

// coefficient u0 + off of a row whose storage is global u64 (kStream / kViaL2) or a shared-memory row of E.  The
// register slots of a thread are one index u0 = reg_index(u, 0) plus a compile-time offset (slot << LB): in global
// memory the offset is added to the pointer, so the 16 accesses share one 64-bit address and take the offsets as
// immediates instead of widening each 32-bit index (an IADD3 + IMAD.X + LEA pair per access).
template <int POLICY, typename E>
__device__ __forceinline__ E ld_row(const void* base, unsigned u0, unsigned off) {
  const unsigned idx = u0 + off;
  if constexpr (POLICY == kSmemRow)
    return static_cast<const E*>(base)[idx];
  else if constexpr (POLICY == kSmemRowPad)
    return static_cast<const E*>(base)[idx + (idx >> 4)];
  else
    return (E)ld_coef<POLICY>(static_cast<const u64*>(base) + u0 + off);
}
template <int POLICY, typename E>
__device__ __forceinline__ void st_row(void* base, unsigned u0, unsigned off, E v) {
  const unsigned idx = u0 + off;
  if constexpr (POLICY == kSmemRow)
    static_cast<E*>(base)[idx] = v;
  else if constexpr (POLICY == kSmemRowPad)
    static_cast<E*>(base)[idx + (idx >> 4)] = v;
  else
    st_coef<POLICY>(static_cast<u64*>(base) + u0 + off, v);
}

// Extra destinations of a transform's final stores (see NttMulti::mirror): buffer p receives value v at p[i] + off + idx
struct MirrorList {
  u64* const* p;
  unsigned count;
  u64 off;
};

// Forward transform of one row of C = 2^LOGC contiguous coefficients rooted at
// tree node `base`, by the T = C/16 threads whose index in the row is u.
template <int MODE, int LOGC, int LD, int ST>
__device__ __forceinline__ void row_fwd_body(void* out, const void* in, typename Ar<MODE>::E* srow, unsigned u,
                                             u64 base, const typename Ar<MODE>::Tw* __restrict__ tw, const Mod& m,
                                             int out_mf, bool active, typename Ar<MODE>::Tw* cta_stab = nullptr,
                                             bool reduce_in = false) {
  using E = typename Ar<MODE>::E;
  using Tw = typename Ar<MODE>::Tw;
  E v[16];
  constexpr int LB0 = LOGC - 4;  // pass 0: register bits are the top 4 index bits
  // cta_stab: every row of this CTA has the same root (whole polynomials, N == C): one table
  // filled by all threads of the CTA instead of one per row
  Tw* stab = cta_stab ? cta_stab : reinterpret_cast<Tw*>(srow + row_elems<E>(LOGC));
  const unsigned u_in = reg_index<LB0>(u, 0);
  static_for<0, 16>([&](auto I) { constexpr int e = I; v[e] = ld_row<LD, E>(in, u_in, e << LB0); });
  if constexpr (LD < kSmemRow && sizeof(E) == 8) {
    if (reduce_in) {  // NttMulti::gather: the input is a value of ANOTHER modulus
      static_for<0, 16>([&](auto I) { constexpr int e = I; v[e] = reduce_any(v[e], m); });
    }
  }
  if constexpr (RowCfg<LOGC>::TW_TABLES) {
    if (cta_stab)
      load_row_twiddles<LOGC>(stab, threadIdx.x, blockDim.x, base, tw);
    else
      load_row_twiddles<LOGC>(stab, u, (1u << LOGC) / 16, base, tw);
    __syncthreads();
  }
  reg_stages<MODE, LOGC, LB0, LOGC - 1, LB0, true>(v, u, base, tw, stab, m, false, Tw{}, Tw{});
  fwd_passes<MODE, LOGC, 1>(v, srow, u, base, tw, stab, m);
  // registers now hold 16 consecutive coefficients per thread (LB = 0)
  static_for<0, 16>([&](auto I) { constexpr int e = I; v[e] = fwd_out<MODE>(v[e], m, out_mf); });
  // store layout: 16 lanes write one 128-byte line per instruction; reaching it
  // from LB = 0 is a warp-local exchange
  constexpr int LB_OUT = LB0 < 4 ? LB0 : 4;
  if constexpr (LOGC > 4) smem_exchange<0, LB_OUT>(v, srow, u);
  if (active) {
    const unsigned u_out = reg_index<LB_OUT>(u, 0);
    static_for<0, 16>([&](auto I) { constexpr int e = I; st_row<ST, E>(out, u_out, e << LB_OUT, v[e]); });
  }
}

// Inverse transform of one row (the last log2 C ... first stages of the GS order).
template <int MODE, int LOGC, int LD, int ST>
__device__ __forceinline__ void row_inv_body(void* out, const void* in, typename Ar<MODE>::E* srow, unsigned u,
                                             u64 base, const typename Ar<MODE>::Tw* __restrict__ tw, const Mod& m,
                                             int out_mf, bool fold, typename Ar<MODE>::Tw inv_n,
                                             typename Ar<MODE>::Tw inv_n_w, bool active,
                                             typename Ar<MODE>::Tw* cta_stab = nullptr, const MirrorList* mir = nullptr,
                                             const ProdIn* prod = nullptr) {
  using Cfg = RowCfg<LOGC>;
  using E = typename Ar<MODE>::E;
  using Tw = typename Ar<MODE>::Tw;
  E v[16];
  constexpr int LB0 = LOGC - 4;
  constexpr int LB_IN = LB0 < 4 ? LB0 : 4;  // 16 lanes read one 128-byte line per instruction
  Tw* stab = cta_stab ? cta_stab : reinterpret_cast<Tw*>(srow + row_elems<E>(LOGC));
  const unsigned u_in = reg_index<LB_IN>(u, 0);
  static_for<0, 16>([&](auto I) { constexpr int e = I; v[e] = ld_row<LD, E>(in, u_in, e << LB_IN); });
  if constexpr (LD < kSmemRow && sizeof(E) == 8) {
    if (prod) {  // NttMulti::mul: the transform of a point-wise product, multiplied on load
      static_for<0, 16>([&](auto I) {
        constexpr int e = I;
        v[e] = prod_lazy<MODE>(v[e], ld_coef<LD>(prod->b + reg_index<LB_IN>(u, e)), m, prod->mu, prod->shift);
      });
    }
  }
  if constexpr (Cfg::TW_TABLES) {
    if (cta_stab)
      load_row_twiddles<LOGC>(stab, threadIdx.x, blockDim.x, base, tw);
    else
      load_row_twiddles<LOGC>(stab, u, (1u << LOGC) / 16, base, tw);
    __syncthreads();  // tables are filled by other warps than the ones that read them
  }
  // -> 16 consecutive coefficients per thread (warp-local exchange)
  if constexpr (LOGC > 4) smem_exchange<LB_IN, 0>(v, srow, u);
  inv_passes<MODE, LOGC, Cfg::PASSES - 1>(v, srow, u, base, tw, stab, m, fold, inv_n, inv_n_w);
  // last pass left the registers in the coalesced layout (LB = LOGC-4);
  // only the kernel holding the root stage applies the output range
  if (active) {
    static_for<0, 16>([&](auto I) {
      constexpr int e = I;
      st_row<ST, E>(out, reg_index<LB0>(u, 0), e << LB0, fold ? inv_out<MODE>(v[e], m, out_mf) : v[e]);
    });
    if (mir && fold) {
      for (unsigned p = 0; p < mir->count; ++p) {
        static_for<0, 16>([&](auto I) {
          constexpr int e = I;
          mir->p[p][mir->off + reg_index<LB0>(u, e)] = (u64)inv_out<MODE>(v[e], m, out_mf);
        });
      }
    }
  }
}

// One CTA = ROWS rows of C contiguous coefficients.  rows_per_poly = N / C.
template <int MODE, int LOGC>
__global__ void __launch_bounds__(RowCfg<LOGC, MODE>::THREADS, RowCfg<LOGC, MODE>::MIN_BLOCKS)
    ntt_row_fwd(u64* result, const u64* operand, const typename Ar<MODE>::Tw* __restrict__ tw, const Mod m,
                u64 total_rows, unsigned rows_per_poly, int out_mf) {
  using Cfg = RowCfg<LOGC, MODE>;
  extern __shared__ __align__(16) unsigned char smem[];
  const unsigned row_local = threadIdx.x / Cfg::T, u = threadIdx.x % Cfg::T;
  u64 row = (u64)blockIdx.x * Cfg::ROWS + row_local;
  const bool active = row < total_rows;
  if (!active) row = total_rows - 1;  // keep barriers uniform; stores are masked
  const u64 base = (u64)rows_per_poly + (row % rows_per_poly);
  typename Cfg::Tw* cta_stab = nullptr;  // whole polynomials per row: all rows of the CTA share root node 1
  // (SMALL mode only: +5 % there; in the 64-bit modes the run-time table address costs more than the loads save)
  if (MODE == kSmall && Cfg::ROWS > 1 && Cfg::TW_TABLES && rows_per_poly == 1)
    cta_stab = reinterpret_cast<typename Cfg::Tw*>(smem + (size_t)row_elems<typename Cfg::E>(LOGC) * sizeof(typename Cfg::E));
  row_fwd_body<MODE, LOGC, kStream, kStream>(
      result + row * Cfg::C, operand + row * Cfg::C,
      reinterpret_cast<typename Cfg::E*>(smem + (size_t)row_local * Cfg::ROW_BYTES), u, base, tw, m, out_mf, active,
      cta_stab);
}

template <int MODE, int LOGC>
__global__ void __launch_bounds__(RowCfg<LOGC, MODE>::THREADS, RowCfg<LOGC, MODE>::MIN_BLOCKS)
    ntt_row_inv(u64* result, const u64* operand, const typename Ar<MODE>::Tw* __restrict__ tw, const Mod m,
                u64 total_rows, unsigned rows_per_poly, int out_mf, int fold, typename Ar<MODE>::Tw inv_n,
                typename Ar<MODE>::Tw inv_n_w) {
  using Cfg = RowCfg<LOGC, MODE>;
  extern __shared__ __align__(16) unsigned char smem[];
  const unsigned row_local = threadIdx.x / Cfg::T, u = threadIdx.x % Cfg::T;
  u64 row = (u64)blockIdx.x * Cfg::ROWS + row_local;
  const bool active = row < total_rows;
  if (!active) row = total_rows - 1;
  const u64 base = (u64)rows_per_poly + (row % rows_per_poly);
  typename Cfg::Tw* cta_stab = nullptr;
  // (SMALL mode only: +5 % there; in the 64-bit modes the run-time table address costs more than the loads save)
  if (MODE == kSmall && Cfg::ROWS > 1 && Cfg::TW_TABLES && rows_per_poly == 1)
    cta_stab = reinterpret_cast<typename Cfg::Tw*>(smem + (size_t)row_elems<typename Cfg::E>(LOGC) * sizeof(typename Cfg::E));
  row_inv_body<MODE, LOGC, kStream, kStream>(
      result + row * Cfg::C, operand + row * Cfg::C,
      reinterpret_cast<typename Cfg::E*>(smem + (size_t)row_local * Cfg::ROW_BYTES), u, base, tw, m, out_mf,
      fold != 0, inv_n, inv_n_w, active, cta_stab);
}

// ------------------------------------------------------------- column kernel
// One column: R = 2^LOGR coefficients at stride 2^log_stride starting at `off`,
// the first (forward) / last (inverse) LOGR stages of a sub-block whose R-1
// twiddles stw[1..R-1] are laid out as a local tree (node 2^s + i).
// the register work of a column: LOGR stages on R values, twiddles from the local tree stw
template <int MODE, int LOGR, bool FWD>
__device__ __forceinline__ void col_stages(typename Ar<MODE>::E (&v)[1 << LOGR], const typename Ar<MODE>::Tw* stw,
                                           const Mod& m, bool root_fold, typename Ar<MODE>::Tw inv_n,
                                           typename Ar<MODE>::Tw inv_n_w) {
  using E = typename Ar<MODE>::E;
  using Tw = typename Ar<MODE>::Tw;
  constexpr int R = 1 << LOGR;
  static_for<0, LOGR>([&](auto STEP) {
    constexpr int step = STEP;
    constexpr int s = FWD ? step : LOGR - 1 - step;  // stage inside the sub-block
    constexpr int eb = LOGR - 1 - s;                 // register bit
    const E cq = stage_cq<MODE>(step, m);
    auto groups = [&] {
      static_for<0, (1 << s)>([&](auto GI) {
        constexpr int gi = GI;
        const Tw w = stw[(1 << s) + gi];
        static_for<0, (1 << eb)>([&](auto L) {
          constexpr int e = (gi << (eb + 1)) | L;
          if constexpr (FWD)
            fwd_bfly<MODE>(v[e], v[e | (1 << eb)], w, m);
          else
            inv_bfly<MODE>(v[e], v[e | (1 << eb)], w, m, cq);
        });
      });
    };
    if constexpr (!FWD && s == 0) {
      if (root_fold) {
        static_for<0, (1 << eb)>([&](auto L) {
          constexpr int l = L;
          inv_bfly_last<MODE>(v[l], v[l | (1 << eb)], inv_n, inv_n_w, m, cq);
        });
      } else {
        groups();
      }
    } else {
      groups();
    }
  });
  if constexpr (!FWD && MODE == kFast) {
    if (!root_fold) inv_pass_fixup<LOGR, R>(v, m);
  }
}

template <int MODE, int LOGR, bool FWD, int LD, int ST>
__device__ __forceinline__ void col_body(u64* result, const u64* operand, u64 off, int log_stride,
                                         const typename Ar<MODE>::Tw* stw, const Mod& m, int out_mf, bool root_fold,
                                         typename Ar<MODE>::Tw inv_n, typename Ar<MODE>::Tw inv_n_w,
                                         const MirrorList* mir = nullptr, bool reduce_in = false) {
  using E = typename Ar<MODE>::E;
  constexpr int R = 1 << LOGR;
  E v[R];
  static_for<0, R>([&](auto I) {
    constexpr int e = I;
    v[e] = (E)ld_coef<LD>(operand + off + ((u64)e << log_stride));
  });
  if constexpr (FWD && sizeof(E) == 8) {
    if (reduce_in) {
      static_for<0, R>([&](auto I) { constexpr int e = I; v[e] = reduce_any(v[e], m); });
    }
  }
  col_stages<MODE, LOGR, FWD>(v, stw, m, root_fold, inv_n, inv_n_w);
  const bool final_out = !FWD && root_fold;
  static_for<0, R>([&](auto I) {
    constexpr int e = I;
    st_coef<ST>(result + off + ((u64)e << log_stride), final_out ? inv_out<MODE>(v[e], m, out_mf) : v[e]);
  });
  if (mir && final_out) {
    for (unsigned p = 0; p < mir->count; ++p) {
      static_for<0, R>([&](auto I) {
        constexpr int e = I;
        mir->p[p][mir->off + off + ((u64)e << log_stride)] = (u64)inv_out<MODE>(v[e], m, out_mf);
      });
    }
  }
}

// Sub-blocks of S = 2^log_s contiguous coefficients, each rooted at tree node
// (N/S) + block_index.  A thread owns column c of one sub-block: R coefficients
// at stride S/R, and runs the sub-block's first log2(R) stages (forward) or last
// log2(R) stages (inverse) on them in registers.
template <int MODE, int LOGR, bool FWD>
__global__ void __launch_bounds__(256)
    ntt_col(u64* result, const u64* operand, const typename Ar<MODE>::Tw* __restrict__ tw, const Mod m, int log_n,
            int log_s, u64 total_cols, int out_mf, int fold, typename Ar<MODE>::Tw inv_n,
            typename Ar<MODE>::Tw inv_n_w) {
  constexpr int R = 1 << LOGR;
  __shared__ typename Ar<MODE>::Tw stw[R];
  const int log_cols = log_s - LOGR;                 // columns per sub-block (log2)
  const u64 g0 = (u64)blockIdx.x * blockDim.x;       // first column of this CTA
  // blockDim.x divides the columns of a sub-block, so the CTA shares one root node
  const u64 blk = g0 >> log_cols;                    // sub-block index over the whole batch
  const u64 blocks_per_poly = 1ull << (log_n - log_s);
  const u64 base = blocks_per_poly + (blk & (blocks_per_poly - 1));
  for (int l = threadIdx.x; l < R; l += blockDim.x) {
    if (l == 0) continue;                            // local node l = 2^s + i
    const int s = 31 - __clz(l);
    stw[l] = ld_tw(tw + (base << s) + (l - (1 << s)));
  }
  __syncthreads();
  const u64 g = g0 + threadIdx.x;
  if (g >= total_cols) return;
  const u64 c = g & ((1ull << log_cols) - 1);
  col_body<MODE, LOGR, FWD, kStream, kStream>(result, operand, (blk << log_s) + c, log_cols, stw, m, out_mf,
                                              !FWD && fold && log_s == log_n, inv_n, inv_n_w);
}

// ------------------------------------------------------------ fused kernels
// N = R * 4096, R = 2^LOGR in {4, 8, 16, 32}: ONE kernel per transform.  A
// thread-block cluster of K = min(R, 8) CTAs owns one polynomial.  Forward:
// phase 1 runs the top LOGR stages on columns (HBM -> registers -> `result`,
// which stays in the 50 MB L2: at most ~130 clusters x 8N bytes are in flight),
// a cluster barrier (release/acquire) publishes it, phase 2 runs the 4096-point
// row transforms reading the intermediate back from L2.  Inverse: rows first,
// columns second.  HBM sees each coefficient once in and once out (16N bytes),
// half the traffic of the two-kernel path.
__device__ __forceinline__ void cluster_barrier() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// 64-bit words only
template <int LOGR>
struct FusedCfg {
  static constexpr int LOGC = 12, C = 1 << LOGC, R = 1 << LOGR;
  static constexpr int K = R < 8 ? R : 8;            // CTAs per cluster
  static constexpr int THREADS = 256;                // = RowCfg<12>::T
  static constexpr int MIN_BLOCKS = LOGR <= 4 ? kRowMinBlocks : 2;
  static constexpr size_t SMEM = RowCfg<LOGC>::ROW_BYTES;
};

template <int MODE, int LOGR>
__global__ void __launch_bounds__(FusedCfg<LOGR>::THREADS, FusedCfg<LOGR>::MIN_BLOCKS)
    ntt_fused_fwd(u64* result, const u64* operand, const typename Ar<MODE>::Tw* __restrict__ tw, const Mod m,
                  int out_mf) {
  using Cfg = FusedCfg<LOGR>;
  using E = typename Ar<MODE>::E;
  using Tw = typename Ar<MODE>::Tw;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  E* smem = reinterpret_cast<E*>(smem_raw);
  __shared__ Tw stw[Cfg::R];
  const unsigned rank = blockIdx.x % Cfg::K;         // == %cluster_ctarank (1-D clusters)
  const u64 poly_off = (u64)(blockIdx.x / Cfg::K) << (Cfg::LOGC + LOGR);
  for (int l = threadIdx.x; l < Cfg::R; l += Cfg::THREADS)
    if (l) stw[l] = ld_tw(tw + l);                   // root sub-tree: local node == global node
  __syncthreads();
  // phase 1: columns rank*C/K ... of this polynomial
  constexpr int COLS = Cfg::C / Cfg::K;
#pragma unroll 1
  for (int c = threadIdx.x; c < COLS; c += Cfg::THREADS)
    col_body<MODE, LOGR, true, kStream, kViaL2>(result, operand, poly_off + rank * COLS + c, Cfg::LOGC, stw, m,
                                                out_mf, false, Tw{}, Tw{});
  cluster_barrier();
  // phase 2: rows rank, rank+K, ...
#pragma unroll 1
  for (unsigned r = rank; r < Cfg::R; r += Cfg::K) {
    u64* row = result + poly_off + (u64)r * Cfg::C;
    row_fwd_body<MODE, Cfg::LOGC, kViaL2, kStream>(row, row, smem, threadIdx.x, (u64)Cfg::R + r, tw, m, out_mf, true);
    if (r + Cfg::K < Cfg::R) __syncthreads();       // the next row reuses the shared buffer
  }
}

template <int MODE, int LOGR>
__global__ void __launch_bounds__(FusedCfg<LOGR>::THREADS, FusedCfg<LOGR>::MIN_BLOCKS)
    ntt_fused_inv(u64* result, const u64* operand, const typename Ar<MODE>::Tw* __restrict__ tw, const Mod m,
                  int out_mf, typename Ar<MODE>::Tw inv_n, typename Ar<MODE>::Tw inv_n_w) {
  using Cfg = FusedCfg<LOGR>;
  using E = typename Ar<MODE>::E;
  using Tw = typename Ar<MODE>::Tw;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  E* smem = reinterpret_cast<E*>(smem_raw);
  __shared__ Tw stw[Cfg::R];
  const unsigned rank = blockIdx.x % Cfg::K;
  const u64 poly_off = (u64)(blockIdx.x / Cfg::K) << (Cfg::LOGC + LOGR);
  for (int l = threadIdx.x; l < Cfg::R; l += Cfg::THREADS)
    if (l) stw[l] = ld_tw(tw + l);
  // phase 1: rows (the __syncthreads inside/after each row also publishes stw)
#pragma unroll 1
  for (unsigned r = rank; r < Cfg::R; r += Cfg::K) {
    const u64 off = poly_off + (u64)r * Cfg::C;
    row_inv_body<MODE, Cfg::LOGC, kStream, kViaL2>(result + off, operand + off, smem, threadIdx.x, (u64)Cfg::R + r,
                                                   tw, m, out_mf, false, inv_n, inv_n_w, true);
    __syncthreads();
  }
  cluster_barrier();
  // phase 2: columns, root stage folded with N^-1
  constexpr int COLS = Cfg::C / Cfg::K;
#pragma unroll 1
  for (int c = threadIdx.x; c < COLS; c += Cfg::THREADS)
    col_body<MODE, LOGR, false, kViaL2, kStream>(result, result, poly_off + rank * COLS + c, Cfg::LOGC, stw, m,
                                                 out_mf, true, inv_n, inv_n_w);
}

// ------------------------------------------------ persistent pipelined single kernel
// N = R * 4096 as above, ONE launch per batch, HBM sees each coefficient once in and once out, and no
// barrier wider than a CTA.  The grid is persistent (a few CTAs per SM) and pulls work items from a
// global counter.  Items come in the order
//     block b:  the 16 column tiles of polynomial b,  then the R rows of polynomial b - D.
// A column tile is 256 columns of R
// coefficients (the top log2 R stages in registers); a row is a 4096-point transform.  The consumer of a
// polynomial waits on a per-polynomial counter its producers bump with release semantics -- but the
// producers were claimed D*(16+R) items earlier, far more than the number of CTAs in flight, so the wait
// is normally over before it starts, and since producers never wait the scheme cannot deadlock.  The
// intermediate is written and read back with .cg accesses: it lives in the 50 MB L2 (D polynomials of
// 8N bytes) and is overwritten in place by the consumer before L2 has a reason to write it back.
// Memory-bound column tiles and multiplier-bound rows of DIFFERENT polynomials share every SM at all
// times, which is what the cluster version above could not do (its two phases are serialised per CTA).
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// 64-bit words only
template <int LOGR>
struct PipeCfg {
  static constexpr int LOGC = 12, C = 1 << LOGC, R = 1 << LOGR;
  static constexpr int THREADS = 256;
  static constexpr int CT = C / THREADS;             // column tiles per polynomial
  static constexpr int SLOTS = CT + R;               // work items per block
  static constexpr int MIN_BLOCKS = FusedCfg<LOGR>::MIN_BLOCKS;
  static constexpr size_t SMEM = RowCfg<LOGC>::ROW_BYTES;
};

template <int MODE, int LOGR>
__global__ void __launch_bounds__(PipeCfg<LOGR>::THREADS, PipeCfg<LOGR>::MIN_BLOCKS)
    ntt_pipe_fwd(u64* result, const u64* operand, const typename Ar<MODE>::Tw* __restrict__ tw, const Mod m,
                 int out_mf, unsigned batch, unsigned lookahead, unsigned* counter, unsigned* done) {
  using Cfg = PipeCfg<LOGR>;
  using E = typename Ar<MODE>::E;
  using Tw = typename Ar<MODE>::Tw;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  E* smem = reinterpret_cast<E*>(smem_raw);
  __shared__ Tw stw[Cfg::R];
  __shared__ unsigned s_item;
  for (int l = threadIdx.x; l < Cfg::R; l += Cfg::THREADS)
    if (l) stw[l] = ld_tw(tw + l);                   // root sub-tree: local node == global node
  const unsigned total = (batch + lookahead) * Cfg::SLOTS;
  while (true) {
    __syncthreads();                                 // s_item and the row buffer are free again
    if (threadIdx.x == 0) s_item = atomicAdd(counter, 1u);
    __syncthreads();
    const unsigned item = s_item;
    if (item >= total) break;
    const unsigned blk = item / Cfg::SLOTS, j = item % Cfg::SLOTS;
    if (j < (unsigned)Cfg::CT) {                     // column tile j of polynomial blk
      if (blk >= batch) continue;
      const u64 poly_off = (u64)blk << (Cfg::LOGC + LOGR);
      col_body<MODE, LOGR, true, kStream, kViaL2>(result, operand, poly_off + j * Cfg::THREADS + threadIdx.x, Cfg::LOGC,
                                                  stw, m, out_mf, false, Tw{}, Tw{});
      __syncthreads();                               // every thread's stores precede the release below
      if (threadIdx.x == 0) red_release_gpu(done + blk, 1u);
    } else {                                         // row j - CT of polynomial blk - lookahead
      if (blk < lookahead) continue;
      const unsigned p = blk - lookahead, r = j - Cfg::CT;
      if (threadIdx.x == 0)
        while (ld_acquire_gpu(done + p) < (unsigned)Cfg::CT) __nanosleep(100);
      __syncthreads();
      u64* row = result + ((u64)p << (Cfg::LOGC + LOGR)) + (u64)r * Cfg::C;
      row_fwd_body<MODE, Cfg::LOGC, kViaL2, kStream>(row, row, smem, threadIdx.x, (u64)Cfg::R + r, tw, m, out_mf, true);
    }
  }
}

// ------------------------------------- fused kernels through distributed shared memory
// The whole polynomial fits in the shared memory of its cluster -- N words spread over K CTAs
// -- so the intermediate between the column phase and the row phase never leaves the SMs.
// CTA `rank` owns rows rank, rank + K, ... of the R x 4096 matrix.  Forward: the column
// phase of every CTA scatters its results straight into the owners' shared memory
// (st.shared::cluster, 128 or 256 contiguous bytes per warp and row), one cluster barrier,
// then every CTA transforms its own rows from local shared memory to HBM.  Inverse: rows
// first into local shared memory, barrier, the column phase gathers from the owners
// (ld.shared::cluster), a last barrier keeps every CTA's memory alive until its peers have
// read it.  HBM sees 8N bytes in and 8N bytes out, L2 nothing.
__device__ __forceinline__ unsigned dsmem_address(const void* local_smem, unsigned cta_rank) {
  const unsigned a = (unsigned)__cvta_generic_to_shared(local_smem);
  unsigned r;
  asm("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(cta_rank));
  return r;
}
__device__ __forceinline__ void dsmem_store(unsigned addr, unsigned v) {
  asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ void dsmem_store(unsigned addr, u64 v) {
  asm volatile("st.shared::cluster.u64 [%0], %1;" ::"r"(addr), "l"(v) : "memory");
}
template <typename E>
__device__ __forceinline__ E dsmem_load(unsigned addr) {
  E v;
  if constexpr (sizeof(E) == 8)
    asm volatile("ld.shared::cluster.u64 %0, [%1];" : "=l"(v) : "r"(addr) : "memory");
  else
    asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

// K = min(R, 8) CTAs per cluster (8 is the portable maximum), R / K rows each.  32-bit words: the owned rows are
// unpadded and the row phase has one exchange buffer of its own.  64-bit words: the owned rows are stored in the
// padded layout of the row kernels' exchanges, and each row is its own exchange buffer once it is in registers, so
// even two rows per CTA (N = 2^16: 72 KiB with the twiddle tables; 106 KiB with a separate buffer) leave room for the
// 3 CTAs per SM the 64-bit row kernels are tuned to.  One 64-bit row per CTA in clusters of 16 (non-portable) fits
// 3 CTAs per SM as well, but an H100 80GB HBM3 (400 W) schedules only 21 such clusters (336 of 396 CTA slots,
// cudaOccupancyMaxActiveClusters) against 45 clusters of 8, and at N = 2^16, 55-bit q, 2^28 coefficients, it took
// 3.86 / 4.27 ms forward / inverse against 3.97 / 4.36 for the two-kernel split.  ntt.cu (plan_single_pass) launches the
// 64-bit kernels at N = 2^14 and 2^15 only.
template <int LOGR, int MODE = kSmall>
struct DsmemCfg {
  using E = typename Ar<MODE>::E;
  using Tw = typename Ar<MODE>::Tw;
  static constexpr int LOGC = 12, C = 1 << LOGC, R = 1 << LOGR;
  static constexpr int K = R < 8 ? R : 8;            // CTAs per cluster
  static constexpr int RPC = R / K;                  // rows owned by one CTA
  static constexpr int THREADS = 256;
  static constexpr int COLS = C / K;                 // columns one CTA runs in the column phase
  static constexpr bool PAD = sizeof(E) == 8;        // owned rows in the padded exchange layout
  static constexpr int ROW_POLICY = PAD ? kSmemRowPad : kSmemRow;
  static constexpr unsigned ROW = row_elems<E>(LOGC);  // elements from one owned row to the next
  // owned rows (+ the exchange buffer of 32-bit words) + the row kernel's twiddle tables
  static constexpr size_t SMEM = (size_t)(RPC + (PAD ? 0 : 1)) * ROW * sizeof(E) + kRowTwEntries * sizeof(Tw);
  // 64-bit words: the row kernels' 3 CTAs per SM (80 registers) at every R
  static constexpr int MIN_BLOCKS = PAD ? kRowMinBlocks : (SMEM <= 56 * 1024 ? 4 : (SMEM <= 75 * 1024 ? 3 : 2));
  // where coefficient j of an owned row is stored
  static __device__ __forceinline__ unsigned slot(unsigned j) { return PAD ? j + (j >> 4) : j; }
};

template <int MODE, int LOGR>
__global__ void __launch_bounds__(DsmemCfg<LOGR, MODE>::THREADS, DsmemCfg<LOGR, MODE>::MIN_BLOCKS)
    ntt_dsmem_fwd(u64* result, const u64* operand, const typename Ar<MODE>::Tw* __restrict__ tw, const Mod m,
                  int out_mf) {
  using Cfg = DsmemCfg<LOGR, MODE>;
  using E = typename Ar<MODE>::E;
  using Tw = typename Ar<MODE>::Tw;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  E* rows = reinterpret_cast<E*>(smem_raw);  // [RPC][ROW]
  E* xbuf = rows + Cfg::RPC * Cfg::ROW;      // 32-bit words: exchange buffer, twiddle tables behind it
  Tw* const ctab = Cfg::PAD ? reinterpret_cast<Tw*>(xbuf) : nullptr;  // 64-bit words: the twiddle tables
  __shared__ Tw stw[Cfg::R];
  const unsigned rank = blockIdx.x % Cfg::K;
  const u64 poly_off = (u64)(blockIdx.x / Cfg::K) << (Cfg::LOGC + LOGR);
  // a CTA's shared memory may only be written by its peers once it is known to be running:
  // arrive now, wait just before the first remote store
  asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
  for (int l = threadIdx.x; l < Cfg::R; l += Cfg::THREADS)
    if (l) stw[l] = ld_tw(tw + l);
  __syncthreads();
  asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
  // phase 1: my columns of every row -> the row owners' shared memory
  unsigned owner_base[Cfg::K];
  static_for<0, Cfg::K>([&](auto I) { constexpr int o = I; owner_base[o] = dsmem_address(rows, o); });
#pragma unroll 1
  for (int c = threadIdx.x; c < Cfg::COLS; c += Cfg::THREADS) {
    const unsigned col = rank * Cfg::COLS + c;
    E v[Cfg::R];
    static_for<0, Cfg::R>([&](auto I) {
      constexpr int e = I;
      v[e] = (E)ld_coef<kStream>(operand + poly_off + ((u64)e << Cfg::LOGC) + col);
    });
    col_stages<MODE, LOGR, true>(v, stw, m, false, Tw{}, Tw{});
    static_for<0, Cfg::R>([&](auto I) {  // row e lives in CTA e % K, slot e / K
      constexpr int e = I;
      dsmem_store(owner_base[e % Cfg::K] + ((e / Cfg::K) * Cfg::ROW + Cfg::slot(col)) * (unsigned)sizeof(E), v[e]);
    });
  }
  cluster_barrier();
  // phase 2: my rows, shared memory -> HBM
#pragma unroll 1
  for (int lr = 0; lr < Cfg::RPC; ++lr) {
    const unsigned r = rank + lr * Cfg::K;
    E* row = rows + lr * Cfg::ROW;
    row_fwd_body<MODE, Cfg::LOGC, Cfg::ROW_POLICY, kStream>(result + poly_off + (u64)r * Cfg::C, row,
                                                            Cfg::PAD ? row : xbuf, threadIdx.x, (u64)Cfg::R + r, tw, m,
                                                            out_mf, true, ctab);
    if (lr + 1 < Cfg::RPC) __syncthreads();  // the next row reuses the exchange buffer and tables
  }
}

template <int MODE, int LOGR>
__global__ void __launch_bounds__(DsmemCfg<LOGR, MODE>::THREADS, DsmemCfg<LOGR, MODE>::MIN_BLOCKS)
    ntt_dsmem_inv(u64* result, const u64* operand, const typename Ar<MODE>::Tw* __restrict__ tw, const Mod m,
                  int out_mf, typename Ar<MODE>::Tw inv_n, typename Ar<MODE>::Tw inv_n_w) {
  using Cfg = DsmemCfg<LOGR, MODE>;
  using E = typename Ar<MODE>::E;
  using Tw = typename Ar<MODE>::Tw;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  E* rows = reinterpret_cast<E*>(smem_raw);
  E* xbuf = rows + Cfg::RPC * Cfg::ROW;
  Tw* const ctab = Cfg::PAD ? reinterpret_cast<Tw*>(xbuf) : nullptr;
  __shared__ Tw stw[Cfg::R];
  const unsigned rank = blockIdx.x % Cfg::K;
  const u64 poly_off = (u64)(blockIdx.x / Cfg::K) << (Cfg::LOGC + LOGR);
  for (int l = threadIdx.x; l < Cfg::R; l += Cfg::THREADS)
    if (l) stw[l] = ld_tw(tw + l);
  // phase 1: my rows, HBM -> local shared memory (the barriers inside publish stw as well)
#pragma unroll 1
  for (int lr = 0; lr < Cfg::RPC; ++lr) {
    const unsigned r = rank + lr * Cfg::K;
    // 64-bit words: the row is its own exchange buffer; the last exchange leaves every thread holding exactly the
    // slots it then stores to, so no thread overwrites a slot another one has still to read
    E* row = rows + lr * Cfg::ROW;
    row_inv_body<MODE, Cfg::LOGC, kStream, Cfg::ROW_POLICY>(row, operand + poly_off + (u64)r * Cfg::C,
                                                            Cfg::PAD ? row : xbuf, threadIdx.x, (u64)Cfg::R + r, tw, m,
                                                            out_mf, false, inv_n, inv_n_w, true, ctab);
    __syncthreads();
  }
  cluster_barrier();
  // phase 2: my columns gathered from the row owners, root stage folded with N^-1, -> HBM
  unsigned owner_base[Cfg::K];
  static_for<0, Cfg::K>([&](auto I) { constexpr int o = I; owner_base[o] = dsmem_address(rows, o); });
#pragma unroll 1
  for (int c = threadIdx.x; c < Cfg::COLS; c += Cfg::THREADS) {
    const unsigned col = rank * Cfg::COLS + c;
    E v[Cfg::R];
    static_for<0, Cfg::R>([&](auto I) {
      constexpr int e = I;
      v[e] = dsmem_load<E>(owner_base[e % Cfg::K] + ((e / Cfg::K) * Cfg::ROW + Cfg::slot(col)) * (unsigned)sizeof(E));
    });
    col_stages<MODE, LOGR, false>(v, stw, m, true, inv_n, inv_n_w);
    static_for<0, Cfg::R>([&](auto I) {
      constexpr int e = I;
      st_coef<kStream>(result + poly_off + ((u64)e << Cfg::LOGC) + col, inv_out<MODE>(v[e], m, out_mf));
    });
  }
  cluster_barrier();  // nobody leaves while a peer may still read its rows
}

// --------------------------------------------------------- tiny-N stage kernel
// One radix-2 stage per launch on global memory; used for N < 16 (GENERIC mode).
template <bool FWD>
__global__ void ntt_stage_simple(u64* result, const u64* src, const Twiddle* __restrict__ tw,
                                 const Mod m, int log_n, int s /*stage: m = 2^s groups*/,
                                 u64 total_bflies, int out_mf, int last, Twiddle inv_n,
                                 Twiddle inv_n_w) {
  const u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total_bflies) return;
  const int log_t = log_n - 1 - s;
  const u64 half = 1ull << (log_n - 1);
  const u64 poly = g >> (log_n - 1), k = g & (half - 1);
  const u64 i = k >> log_t, jj = k & ((1ull << log_t) - 1);
  const u64 j = (poly << log_n) + (i << (log_t + 1)) + jj;
  u64 X = src[j], Y = src[j + (1ull << log_t)];
  if (FWD) {
    fwd_bfly<kGeneric>(X, Y, ld_tw(tw + (1ull << s) + i), m);
    if (last) {
      X = fwd_out<kGeneric>(X, m, out_mf);
      Y = fwd_out<kGeneric>(Y, m, out_mf);
    }
  } else if (last) {
    inv_bfly_last<kGeneric>(X, Y, inv_n, inv_n_w, m, m.two_q);
    X = inv_out<kGeneric>(X, m, out_mf);
    Y = inv_out<kGeneric>(Y, m, out_mf);
  } else {
    inv_bfly<kGeneric>(X, Y, ld_tw(tw + (1ull << s) + i), m, m.two_q);
  }
  result[j] = X;
  result[j + (1ull << log_t)] = Y;
}

// --------------------------------------------------------------- host side

// Opt a kernel into more than 48 KiB of dynamic shared memory, once per kernel and device
// (the attribute call costs more than a launch; doing it on every call doubled the host-side
// cost of small transforms).
template <auto Kernel>
cudaError_t ensure_dynamic_smem(size_t bytes) {
  if (bytes <= 48 * 1024) return cudaSuccess;
  static std::atomic<unsigned long long> done{0};
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (done.load(std::memory_order_acquire) & bit) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e == cudaSuccess) done.fetch_or(bit, std::memory_order_release);
  return e;
}

// One launch of a persistent pipelined kernel (ntt_pipe_fwd, ntt_pipe_multi) over `units` polynomials: a grid of
// MIN_BLOCKS CTAs per SM (fewer if there are fewer work items) and a zeroed work counter and per-polynomial producer
// counters, freed in stream order after the kernel.  The kernel is called with args..., then (units, lookahead,
// counter, done).  HEXL_B200_PIPE_LOOKAHEAD = polynomials between a producer block and its consumers (default 16,
// chosen for the H100's 50 MB L2: at N = 2^17 that is 16 MiB of intermediate).
template <auto Kernel, typename Cfg, typename... Args>
cudaError_t launch_pipelined(u64 units, cudaStream_t stream, Args... args) {
  static const unsigned lookahead = [] {
    const char* v = std::getenv("HEXL_B200_PIPE_LOOKAHEAD");
    return (unsigned)std::max(1, v ? std::atoi(v) : 16);
  }();
  cudaError_t e = ensure_dynamic_smem<Kernel>(Cfg::SMEM);
  if (e != cudaSuccess) return e;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const u64 items = (units + lookahead) * Cfg::SLOTS;
  const unsigned grid = (unsigned)std::min<u64>((u64)sms * Cfg::MIN_BLOCKS, items);
  unsigned* state = nullptr;  // [0] = work counter, [1 + p] = producers of polynomial p that have finished
  const size_t bytes = (size_t)(units + 1) * sizeof(unsigned);
  if ((e = scratch_alloc_async(reinterpret_cast<void**>(&state), bytes, stream)) != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(state, 0, bytes, stream)) == cudaSuccess) {
    Kernel<<<grid, Cfg::THREADS, Cfg::SMEM, stream>>>(args..., (unsigned)units, lookahead, state, state + 1);
    count_launch();
    e = cudaGetLastError();
  }
  scratch_free_async(state, stream);
  return e;
}

inline int pick_mode(u64 q) {
  if (q < kSmallModulusLimit) return kSmall;
  if (q < kFastModulusLimit && q >= (1ull << 32)) return kFast;
  return (q >= kFastModulusLimit && q < kWideModulusLimit) ? kWide : kGeneric;
}

// the tables of a mode
template <int MODE>
struct Tab {
  static const Twiddle* fwd(const NttDeviceTables& t) { return t.fwd; }
  static const Twiddle* inv(const NttDeviceTables& t) { return t.inv; }
  static Twiddle inv_n(const NttDeviceTables& t) { return t.inv_n; }
  static Twiddle inv_n_w(const NttDeviceTables& t) { return t.inv_n_w; }
};
template <>
struct Tab<kSmall> {
  static const Twiddle32* fwd(const NttDeviceTables& t) { return t.fwd32; }
  static const Twiddle32* inv(const NttDeviceTables& t) { return t.inv32; }
  static Twiddle32 inv_n(const NttDeviceTables& t) { return t.inv_n32; }
  static Twiddle32 inv_n_w(const NttDeviceTables& t) { return t.inv_n_w32; }
};

__host__ __device__ inline Mod make_mod(u64 q, u64 mu) {
  Mod m;
  m.q = q;
  m.two_q = q << 1;
  m.four_q = q << 2;
  m.mu = mu;
  const u64 negq = 0 - q;
  m.n0 = (unsigned)negq;
  m.n1 = (unsigned)(negq >> 32);
  m.zero = 0;
  return m;
}
inline Mod make_mod(const NttDeviceTables& t) { return make_mod(t.q, t.mu); }

// Split the top (log_n - log_c) stages into column passes of at most 5 stages,
// as even as possible, larger first.
inline int plan_col_passes(int top_stages, int out[8]) {
  if (top_stages <= 0) return 0;
  const int passes = (top_stages + 4) / 5;
  int left = top_stages;
  for (int p = 0; p < passes; ++p) {
    out[p] = (left + (passes - p) - 1) / (passes - p);
    left -= out[p];
  }
  return passes;
}


}  // namespace
}  // namespace hexl_b200
