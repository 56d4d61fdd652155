// Device kernels for the SEAL-shaped composites that sit directly on top of the
// hot path (SURVEY.md 8(f)-1/-2): DyadicMultiply, the element-wise glue of
// CKKS KeySwitch, and the rescale (DivideAndRoundQLast) that shares KeySwitch's
// mod-down.  The NTTs inside them are the kernels of ntt.cu; what is here is
// memory-bound streaming work.
//   DyadicMultiply   hexl/experimental/seal/dyadic-multiply-internal.cpp:17-73
//   KeySwitch        hexl/experimental/seal/key-switch-internal.cpp:25-201
//   rescale          SEAL's RNSTool::divide_and_round_q_last(_ntt)_inplace
#include "galois.cuh"
#include "hybrid_rotation.h"
#include "internal.h"

namespace hexl_b200 {
namespace {

constexpr int kThreads = 256;

// generalised Barrett x*y mod q for x, y < q (same arithmetic as EltwiseMultMod,
// eltwise-mult-mod-internal.hpp:71-99).  WIDE: the launch has a 62-bit modulus, whose quotient estimate can be low by
// two, so the product is reduced from [0, 3q) with a second conditional subtraction (eltwise.cu:FMult).
struct MulCtx {
  u64 q, mu;
  int shift;
};
template <bool WIDE>
__device__ __forceinline__ u64 mulmod(u64 x, u64 y, const MulCtx& c) {
  const u64 lo = x * y, hi = mulhi(x, y);
  const u64 c1 = c.shift ? ((lo >> c.shift) | (hi << (64 - c.shift))) : lo;
  const u64 z = csub(lo - mulhi(c1, c.mu) * c.q, c.q);
  return WIDE ? csub(z, c.q) : z;
}

// ---- DyadicMultiply: (x0*y0, x0*y1 + x1*y0, x1*y1) for every RNS modulus.
// A thread owns VEC consecutive coefficient slots of one modulus: 4 loads and 3 stores of
// VEC*8 bytes, all coalesced and streaming (56 B of traffic per slot); inputs are read
// before any output is written, so result may alias either operand
// (test-dyadic-multiply.cpp:38-112).  VEC = 2 (128-bit accesses) when n is even and every
// pointer is 16-byte aligned, else 1.
template <int VEC>
struct Slots {
  u64 v[VEC];
};
template <int VEC>
__device__ __forceinline__ Slots<VEC> ld_slots(const u64* p) {
  Slots<VEC> r;
  if constexpr (VEC == 2) {
    const ulonglong2 t = ld_stream2(p);
    r.v[0] = t.x;
    r.v[1] = t.y;
  } else {
    r.v[0] = __ldcs(p);
  }
  return r;
}
template <int VEC>
__device__ __forceinline__ void st_slots(u64* p, const Slots<VEC>& r) {
  if constexpr (VEC == 2) {
    st_stream2(p, make_ulonglong2(r.v[0], r.v[1]));
  } else {
    __stcs(p, r.v[0]);
  }
}

template <int VEC, bool WIDE>
__global__ void __launch_bounds__(kThreads)
    dyadic_kernel(u64* result, const u64* op1, const u64* op2, u64 n, u64 num_moduli, u64 first, u64 count,
                  const __grid_constant__ DyadicModuli mods) {
  const u64 total = n * count / VEC, poly = n * num_moduli, base = first * n;
  const u64 stride = (u64)gridDim.x * kThreads;
  for (u64 i = (u64)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride) {
    const DyadicModulus& dm = mods.m[i * VEC / n];
    const MulCtx c{dm.q, dm.mu, dm.shift};
    const u64 o = base + i * VEC;
    const Slots<VEC> x0 = ld_slots<VEC>(op1 + o), x1 = ld_slots<VEC>(op1 + o + poly);
    const Slots<VEC> y0 = ld_slots<VEC>(op2 + o), y1 = ld_slots<VEC>(op2 + o + poly);
    Slots<VEC> r0, r1, r2;
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      r0.v[k] = mulmod<WIDE>(x0.v[k], y0.v[k], c);
      r1.v[k] = csub(mulmod<WIDE>(x0.v[k], y1.v[k], c) + mulmod<WIDE>(x1.v[k], y0.v[k], c), c.q);
      r2.v[k] = mulmod<WIDE>(x1.v[k], y1.v[k], c);
    }
    st_slots<VEC>(result + o, r0);
    st_slots<VEC>(result + o + poly, r1);
    st_slots<VEC>(result + o + 2 * poly, r2);
  }
}

// ---- EltwiseMultMod / AddMod / SubMod over an RNS batch: block e of per_mod elements under
// modulus e (eltwise-mult-mod-internal.hpp:33-101, eltwise-add-mod.cpp:16-40, eltwise-sub-mod.cpp:16-40
// per element; MultMod inputs < in_mf * q_e with in_mf in {1,2,4}, Add/Sub inputs < q_e).
template <int VEC, bool WIDE>
__global__ void __launch_bounds__(kThreads)
    rns_eltwise_kernel(u64* result, const u64* a, const u64* b, u64 per_mod, u64 count, int op, int in_mf,
                       const __grid_constant__ DyadicModuli mods) {
  const u64 total = per_mod * count / VEC;
  const u64 stride = (u64)gridDim.x * kThreads;
  for (u64 i = (u64)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride) {
    const DyadicModulus& dm = mods.m[i * VEC / per_mod];
    const MulCtx c{dm.q, dm.mu, dm.shift};
    const Slots<VEC> x = ld_slots<VEC>(a + i * VEC), y = ld_slots<VEC>(b + i * VEC);
    Slots<VEC> r;
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      u64 xv = x.v[k], yv = y.v[k];
      if (op == kRnsAdd) {
        r.v[k] = csub(xv + yv, c.q);
        continue;
      }
      if (op == kRnsSub) {
        r.v[k] = xv >= yv ? xv - yv : xv + c.q - yv;
        continue;
      }
      if (in_mf >= 4) {
        xv = csub(xv, c.q << 1);
        yv = csub(yv, c.q << 1);
      }
      if (in_mf >= 2) {
        xv = csub(xv, c.q);
        yv = csub(yv, c.q);
      }
      r.v[k] = mulmod<WIDE>(xv, yv, c);
    }
    st_slots<VEC>(result + i * VEC, r);
  }
}

// ---- KeySwitch glue (key-switch-internal.cpp:60-198), every kernel batched over the RNS
// moduli of one parameter block; layouts are [modulus][component or digit][n].

// (:77-85, every digit reduced into every modulus, is folded into the forward transform: NttMulti::gather)

// :93-130: lazy 128-bit multiply-accumulate of the digits with the switching keys, one
// Shoup(hi, 2^64 mod q) + Barrett(lo) at the end, two conditional subtractions.
// PERMUTE (the hoisted rotations): output slot l reads digit slot pi_g(l), the NTT-form automorphism applied to the
// transformed digits on load.  An aligned block of 2^t output slots reads one aligned block of 2^t digit slots, so the
// reads stay as coalesced as the plain ones.
template <bool PERMUTE>
__global__ void __launch_bounds__(kThreads)
    ks_mac_kernel(u64* prod, const u64* ops, u64 ops_stride, const __grid_constant__ KeyPointers keys, u64 n,
                  u64 jcount, u64 kcc, u64 key_modulus_size, u64 count, const __grid_constant__ KsModuli mods,
                  int accumulate, unsigned galois_elt) {
  const u64 per_mod = kcc * n;
  const u64 g = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (g >= per_mod * count) return;
  const u64 e = g / per_mod, r = g - e * per_mod;
  const u64 k = r / n, l = r - k * n;
  const KsModulus& md = mods.m[e];
  const u64 key_off = n * md.c + k * key_modulus_size * n + l;
  u64 src = l;
  if constexpr (PERMUTE) src = ntt_source((unsigned)l, galois_elt, (unsigned)(2 * n - 1), __ffsll((long long)n) - 1);
  const u64* op = ops + e * ops_stride + src;
  u64 lo = 0, hi = 0;
  for (u64 j = 0; j < jcount; ++j) {
    const u64 a = op[j * n];
    const u64 b = __ldcs(keys.p[j] + key_off);
    const u64 plo = a * b, phi = mulhi(a, b);
    lo += plo;
    hi += phi + (lo < plo);
  }
  u64 v = shoup_lazy(hi, md.a, md.b, md.q) + barrett64_lazy(lo, md.q, md.mu);  // < 4q
  v = csub(csub(v, md.q << 1), md.q);
  if (accumulate) v = csub(v + prod[g], md.q);
  prod[g] = v;
}

// ---- The hybrid linear transform: sum_r w_r (.) Rot_{g_r}(ct) with one mod-down for the whole sum.
// (hi, lo) += a b, unreduced
__device__ __forceinline__ void mac128(u64 a, u64 b, u64& lo, u64& hi) {
  const u64 plo = a * b;
  lo += plo;
  hi += mulhi(a, b) + (lo < plo);
}
// (hi 2^64 + lo) mod q, canonical: Shoup(hi, 2^64 mod q) + Barrett(lo) < 4q, then two conditional subtractions
__device__ __forceinline__ u64 reduce128(u64 hi, u64 lo, const KsModulus& md) {
  const u64 v = shoup_lazy(hi, md.a, md.b, md.q) + barrett64_lazy(lo, md.q, md.mu);
  return csub(csub(v, md.q << 1), md.q);
}

// A thread owns one slot l of one modulus e and both key components: per element it reads the permuted digits and the
// diagonal word once, sums the digit products unreduced (the bound of ks_mac_digits_per_launch), reduces, and adds
// w times that into a second 128-bit sum, which at most 64 canonical products cannot wrap for q < 2^61.  The
// per-element products are never written.
__global__ void __launch_bounds__(kThreads)
    ks_weighted_mac_kernel(u64* acc, const u64* ops, u64 ops_stride, const __grid_constant__ WeightedMacElts elts,
                           u64 n, u64 jcount, u64 num_elts, u64 key_modulus_size, u64 count,
                           const __grid_constant__ KsModuli mods, int accumulate) {
  const u64 g = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (g >= n * count) return;
  const u64 e = g / n, l = g - e * n;
  const KsModulus& md = mods.m[e];
  const u64 key_off = n * md.c + l, comp = key_modulus_size * n;
  const int log_n = __ffsll((long long)n) - 1;
  const u64* op = ops + e * ops_stride;
  u64 lo0 = 0, hi0 = 0, lo1 = 0, hi1 = 0;
  // (element, digit) pairs and digits fit 32 bits: at most kParamBlock of each
  for (unsigned r = 0, kp = 0; r < (unsigned)num_elts; ++r) {
    const u64* d = op + ntt_source((unsigned)l, elts.elt[r], (unsigned)(2 * n - 1), log_n);
    u64 a0 = 0, b0 = 0, a1 = 0, b1 = 0;
    for (unsigned j = 0; j < (unsigned)jcount; ++j, ++kp) {
      const u64 x = d[j * n];
      const u64* key = elts.key[kp] + key_off;
      mac128(x, __ldcs(key), a0, b0);
      mac128(x, __ldcs(key + comp), a1, b1);
    }
    const u64 w = elts.diag[r][e * n + l];
    mac128(w, reduce128(b0, a0, md), lo0, hi0);
    mac128(w, reduce128(b1, a1, md), lo1, hi1);
  }
  u64 v0 = reduce128(hi0, lo0, md), v1 = reduce128(hi1, lo1, md);
  u64* out = acc + e * 2 * n + l;
  if (accumulate) {
    v0 = csub(v0 + out[0], md.q);
    v1 = csub(v1 + out[n], md.q);
  }
  out[0] = v0;
  out[n] = v1;
}

// A thread owns one slot l of one data limb: w_r times c0 at pi_r(l) for every element, and times c1 at l for the
// identity terms, each sum in 128 bits (at most 64 canonical products) and reduced once.
__global__ void __launch_bounds__(kThreads)
    ks_permuted_sum_kernel(u64* result, const u64* ct, u64 n, u64 level, u64 i0, u64 count,
                           const __grid_constant__ PermutedSumElts elts, u64 num_elts,
                           const __grid_constant__ KsModuli mods, int accumulate) {
  const u64 g = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (g >= n * count) return;
  const u64 e = g / n, l = g - e * n;
  const KsModulus& md = mods.m[e];
  const int log_n = __ffsll((long long)n) - 1;
  const u64* c0 = ct + (i0 + e) * n;
  const u64 c1 = elts.identity ? ct[(level + i0 + e) * n + l] : 0;
  u64 lo0 = 0, hi0 = 0, lo1 = 0, hi1 = 0;
  for (u64 r = 0; r < num_elts; ++r) {
    const u64 w = elts.diag[r][e * n + l];
    mac128(w, c0[ntt_source((unsigned)l, elts.elt[r], (unsigned)(2 * n - 1), log_n)], lo0, hi0);
    if ((elts.identity >> r) & 1) mac128(w, c1, lo1, hi1);
  }
  u64 v0 = reduce128(hi0, lo0, md), v1 = reduce128(hi1, lo1, md);
  u64* out = result + (i0 + e) * n + l;
  if (accumulate) {
    v0 = csub(v0 + out[0], md.q);
    v1 = csub(v1 + out[level * n], md.q);
  }
  out[0] = v0;
  out[level * n] = v1;
}

// ---- The baby-step giant-step linear transform: one giant step's sums over its present babies.
// A thread owns one slot l of one modulus b = b0 + e of B.  Component 0 is read at pi_h(l), so the giant rotation is
// applied on load: the diagonal and the stored baby products at pi_h(l), c0 at pi_{b_i}(pi_h(l)) on the data limbs.
// Component 1 is read at l.  Each of the four sums (data-limb and extended-basis part of each component) takes at most
// 64 canonical products in 128 bits, which cannot wrap below 2^61, and is reduced once.
__global__ void __launch_bounds__(kThreads)
    ks_bsgs_sum_kernel(u64* x, u64* y, u64* x1, u64* y1, const u64* ct, const u64* prods, u64 prod_stride, u64 n,
                       u64 level, u64 b0, u64 count, unsigned giant, const __grid_constant__ BsgsSumTerms terms,
                       u64 num_terms, const __grid_constant__ KsModuli mods, int mode) {
  const u64 g = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (g >= n * count) return;
  const u64 e = g / n, l = g - e * n, b = b0 + e;
  const KsModulus& md = mods.m[e];
  const int log_n = __ffsll((long long)n) - 1;
  const unsigned mask = (unsigned)(2 * n - 1);
  const u64 pl = ntt_source((unsigned)l, giant, mask, log_n);
  const bool data = b < level;
  const u64* c0 = ct + b * n;
  const u64 c1 = data ? ct[(level + b) * n + l] : 0;
  const u64* prod_b = prods + b * 2 * n;
  u64 slo0 = 0, shi0 = 0, slo1 = 0, shi1 = 0, tlo0 = 0, thi0 = 0, tlo1 = 0, thi1 = 0;
  for (unsigned r = 0; r < (unsigned)num_terms; ++r) {  // at most kParamBlock terms per launch
    const u64* w = terms.diag[r] + e * n;
    const u64 w0 = w[pl], w1 = w[l];
    if (data) mac128(w0, c0[ntt_source((unsigned)pl, terms.elt[r], mask, log_n)], slo0, shi0);
    if (terms.prod[r] != kBsgsNoProducts) {
      const u64* p = prod_b + terms.prod[r] * prod_stride;
      mac128(w0, __ldcs(p + pl), tlo0, thi0);
      mac128(w1, __ldcs(p + n + l), tlo1, thi1);
    } else if (data) {
      mac128(w1, c1, slo1, shi1);
    }
  }
  const u64 s0 = reduce128(shi0, slo0, md), s1 = reduce128(shi1, slo1, md);
  const u64 t0 = reduce128(thi0, tlo0, md), t1 = reduce128(thi1, tlo1, md);
  const bool keyed = mode & kBsgsKeyedGiant, store1 = mode & kBsgsStore1;
  u64* yb = y + b * 2 * n + l;
  u64 v0 = csub(yb[0] + t0, md.q), v1 = yb[n];
  if (!keyed) v1 = csub(v1 + t1, md.q);
  if (data) {
    u64* xb = x + b * n + l;
    const u64 x0 = csub(xb[0] + s0, md.q);
    const u64 xs1 = keyed ? xb[level * n] : csub(xb[level * n] + s1, md.q);
    if (mode & kBsgsFold) {  // the last sum of X: y_{q_i} += [P]_{q_i} X, md.c = [P]_{q_i}; X itself is not stored
      u64 lo = 0, hi = 0;
      mac128(md.c, x0, lo, hi);
      v0 = csub(v0 + reduce128(hi, lo, md), md.q);
      lo = hi = 0;
      mac128(md.c, xs1, lo, hi);
      v1 = csub(v1 + reduce128(hi, lo, md), md.q);
    } else {
      xb[0] = x0;
      if (!keyed) xb[level * n] = xs1;
    }
    if (keyed) x1[b * n + l] = store1 ? s1 : csub(x1[b * n + l] + s1, md.q);
  }
  if (keyed) y1[b * n + l] = store1 ? t1 : csub(y1[b * n + l] + t1, md.q);
  yb[0] = v0;
  yb[n] = v1;
}

// ---- Multiply and relinearize: the key products of the tensor's last term, plus [P] times its first two terms.
// A thread owns one slot l of one modulus e and both key components: it reads each digit word once for both, keeps each
// component's sum unreduced in 128 bits (jcount within the bound of ks_mac_digits_per_launch) and reduces it.  The
// storing launch of a data modulus also reads a0, a1, b0, b1 at the slot: d_k and [P] d_k are reduced on their own
// (products of canonical words, below 2^123) and added mod q, so the digit sums' bound is untouched.
__global__ void __launch_bounds__(kThreads)
    ks_relin_mac_kernel(u64* prod, const u64* ops, u64 ops_stride, const __grid_constant__ KeyPointers keys, u64 n,
                        u64 jcount, u64 key_modulus_size, u64 count, const __grid_constant__ KsModuli mods,
                        const __grid_constant__ RelinTensor tensor, int accumulate) {
  const u64 g = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (g >= n * count) return;
  const u64 e = g / n, l = g - e * n;
  const KsModulus& md = mods.m[e];
  const u64 key_off = n * md.c + l, comp = key_modulus_size * n;
  const u64* op = ops + e * ops_stride + l;
  u64 lo0 = 0, hi0 = 0, lo1 = 0, hi1 = 0;
  for (unsigned j = 0; j < (unsigned)jcount; ++j) {  // at most kParamBlock digits per launch
    const u64 x = op[j * n];
    const u64* key = keys.p[j] + key_off;
    mac128(x, __ldcs(key), lo0, hi0);
    mac128(x, __ldcs(key + comp), lo1, hi1);
  }
  u64 v0 = reduce128(hi0, lo0, md), v1 = reduce128(hi1, lo1, md);
  u64* out = prod + e * 2 * n + l;
  if (accumulate) {
    v0 = csub(v0 + out[0], md.q);
    v1 = csub(v1 + out[n], md.q);
  } else if (e < tensor.data) {
    const u64 s = e * n + l;
    u64 d0, d1, lo = 0, hi = 0;
    if (tensor.sum) {
      d0 = tensor.sum[s];
      d1 = tensor.sum[s + tensor.comp];
    } else {
      const u64 a0 = tensor.ct1[s], a1 = tensor.ct1[s + tensor.comp];
      const u64 b0 = tensor.ct2[s], b1 = tensor.ct2[s + tensor.comp];
      mac128(a0, b0, lo, hi);
      d0 = reduce128(hi, lo, md);
      lo = hi = 0;
      mac128(a0, b1, lo, hi);
      mac128(a1, b0, lo, hi);
      d1 = reduce128(hi, lo, md);
    }
    const u64 P = tensor.p[e];
    lo = hi = 0;
    mac128(P, d0, lo, hi);
    v0 = csub(v0 + reduce128(hi, lo, md), md.q);
    lo = hi = 0;
    mac128(P, d1, lo, hi);
    v1 = csub(v1 + reduce128(hi, lo, md), md.q);
  }
  out[0] = v0;
  out[n] = v1;
}

// ---- A sum of ciphertext products: the tensor terms of a chunk of pairs, summed before one relinearization.
// A thread owns one slot l of one data limb i = i0 + e and reads the four words of every pair there.  d0 and t take one
// product per pair, d1 two: at most kRelinSumPairs pairs keep each 128-bit sum within 64 products of canonical words,
// exact below 2^61.  Each sum is reduced once; a later chunk adds mod q into what the first stored.
__global__ void __launch_bounds__(kThreads)
    relin_tensor_sum_kernel(u64* out, u64 n, u64 level, u64 i0, u64 count, const __grid_constant__ RelinSumPairs pairs,
                            u64 num_pairs, const __grid_constant__ KsModuli mods, int accumulate) {
  const u64 g = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (g >= n * count) return;
  const u64 e = g / n, l = g - e * n;
  const KsModulus& md = mods.m[e];
  const u64 comp = level * n, s = (i0 + e) * n + l;
  u64 lo0 = 0, hi0 = 0, lo1 = 0, hi1 = 0, lo2 = 0, hi2 = 0;
  for (unsigned r = 0; r < (unsigned)num_pairs; ++r) {  // at most kRelinSumPairs pairs per launch
    const u64 a0 = pairs.ct1[r][s], a1 = pairs.ct1[r][s + comp];
    const u64 b0 = pairs.ct2[r][s], b1 = pairs.ct2[r][s + comp];
    mac128(a0, b0, lo0, hi0);
    mac128(a0, b1, lo1, hi1);
    mac128(a1, b0, lo1, hi1);
    mac128(a1, b1, lo2, hi2);
  }
  u64 v0 = reduce128(hi0, lo0, md), v1 = reduce128(hi1, lo1, md), v2 = reduce128(hi2, lo2, md);
  u64* o = out + s;
  if (accumulate) {
    v0 = csub(v0 + o[0], md.q);
    v1 = csub(v1 + o[comp], md.q);
    v2 = csub(v2 + o[2 * comp], md.q);
  }
  o[0] = v0;
  o[comp] = v1;
  o[2 * comp] = v2;
}

// ---- The inner sum: one bit of the rotate-and-sum recurrence, A' = A + Rot_d(A) and R += Rot_s(A).
// A thread owns one slot l of one modulus b = b0 + e of B and handles X (data moduli) and Y there.  It reads A's
// component 0 at l, pi_d(l) and pi_s(l) and component 1 at l, once each; component 1 moves to A' unchanged, or doubled
// when d = 1.  Only additions of canonical words, except the fold's [P] X_R, one 128-bit product reduced once.
struct SumPart {
  u64 a0, ad, as, a1;  // A0 at l, pi_d(l), pi_s(l); A1 at l
};
__device__ __forceinline__ SumPart sum_read(const u64* a0, const u64* a1, u64 l, u64 pd, u64 ps) {
  return SumPart{a0[l], a0[pd], a0[ps], a1[l]};
}
__global__ void __launch_bounds__(kThreads)
    inner_sum_step_kernel(const u64* xa, const u64* ya, u64* xn, u64* yn, u64* xr, u64* yr, u64* y1, u64 n, u64 level,
                          u64 b0, u64 count, unsigned dbl, unsigned shift, const __grid_constant__ KsModuli mods,
                          int mode) {
  const u64 g = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (g >= n * count) return;
  const u64 e = g / n, l = g - e * n, b = b0 + e;
  const KsModulus& md = mods.m[e];
  const u64 q = md.q;
  const int log_n = __ffsll((long long)n) - 1;
  const unsigned mask = (unsigned)(2 * n - 1);
  const u64 pd = ntt_source((unsigned)l, dbl, mask, log_n), ps = ntt_source((unsigned)l, shift, mask, log_n);
  const bool twice = mode & kSumDoubleId, shift_id = mode & kSumShiftId;
  u64 xr0 = 0, xr1 = 0;  // X_R after this bit, for the fold
  if (b < level) {
    const u64 comp = level * n;
    const SumPart x = sum_read(xa + b * n, xa + comp + b * n, l, pd, ps);
    if (mode & kSumNext) {
      xn[b * n + l] = csub(x.a0 + x.ad, q);
      xn[comp + b * n + l] = twice ? csub(x.a1 + x.a1, q) : x.a1;
    }
    if (mode & kSumR) {
      u64* r = xr + b * n + l;
      xr0 = x.as;
      xr1 = shift_id ? x.a1 : 0;
      if (!(mode & kSumRStore)) {
        xr0 = csub(xr0 + r[0], q);
        xr1 = csub(xr1 + r[comp], q);
      }
      if (!(mode & kSumFold)) {
        r[0] = xr0;
        r[comp] = xr1;
      }
    }
  }
  const bool y_next = (mode & kSumNext) && (mode & kSumNextY), y_r = (mode & kSumR) && (mode & kSumRYWrite);
  if (!y_next && !y_r && !(mode & kSumCopy1)) return;
  const SumPart y = (mode & kSumYA) ? sum_read(ya + b * 2 * n, ya + b * 2 * n + n, l, pd, ps) : SumPart{0, 0, 0, 0};
  if (y_next) {
    yn[b * 2 * n + l] = csub(y.a0 + y.ad, q);
    yn[b * 2 * n + n + l] = twice ? csub(y.a1 + y.a1, q) : y.a1;
  }
  if (y_r) {
    u64* r = yr + b * 2 * n + l;
    u64 v0 = y.as, v1 = shift_id ? y.a1 : 0;
    if (mode & kSumRY) {
      v0 = csub(v0 + r[0], q);
      v1 = csub(v1 + r[n], q);
    }
    if ((mode & kSumFold) && b < level) {  // y_{q_i} += [P]_{q_i} X_R, md.c = [P]_{q_i}
      u64 lo = 0, hi = 0;
      mac128(md.c, xr0, lo, hi);
      v0 = csub(v0 + reduce128(hi, lo, md), q);
      lo = hi = 0;
      mac128(md.c, xr1, lo, hi);
      v1 = csub(v1 + reduce128(hi, lo, md), q);
    }
    r[0] = v0;
    r[n] = v1;
  }
  if (mode & kSumCopy1) y1[b * n + l] = y.a1;
}

// The two halves of the mod-down by the last modulus, shared by the kernels below.
// round: a coefficient of the last modulus's part (coefficient form, [0, 2 q_last)) rounded and moved into modulus q:
//   t = (x + q_last/2) mod q_last;  out = (t mod q) + add,  add = q - (q_last/2 mod q);  out < 2q
__device__ __forceinline__ u64 round_into(u64 x, u64 q_last, u64 mu_last, u64 q, u64 mu, u64 add) {
  x += q_last >> 1;
  x = csub(barrett64_lazy(x, q_last, mu_last), q_last);
  if (q_last > q) x = csub(barrett64_lazy(x, q, mu), q);
  return x + add;
}
// finish: (x + 4q - t) * factor mod q, canonical, for x < 4q and t < 4q (the operand is < 8q, so q < 2^61)
__device__ __forceinline__ u64 finish_value(u64 x, u64 t, u64 q, u64 w, u64 wp) {
  x = reduce_from<8>(x + (q << 2) - t, q);
  return csub(shoup_lazy(x, w, wp, q), q);
}

// :148-178: the special prime's part, rounded and moved into modulus e
__global__ void __launch_bounds__(kThreads)
    ks_round_kernel(u64* tmp, const u64* t_last, u64 per_mod /* kcc*n */, u64 q_last, u64 mu_last, u64 count,
                    const __grid_constant__ KsModuli mods) {
  const u64 g = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (g >= per_mod * count) return;
  const u64 e = g / per_mod, r = g - e * per_mod;
  const KsModulus& md = mods.m[e];
  tmp[g] = round_into(t_last[r], q_last, mu_last, md.q, md.mu, md.a);
}

// :183-197:  v = (in + 4 q_e - t_ntt) * modswitch mod q_e;  result[n (res_stride k + i0 + e) + l] (+)= v mod q_e.
// `in` is either modulus-major like tmp (KeySwitch's prod) or, with in_like_result, laid out like result (the operand
// of DivideAndRoundQLast, which may be result itself).  accumulate: add into result (KeySwitch) or store (rescale).
__global__ void __launch_bounds__(kThreads)
    ks_finish_kernel(u64* result, const u64* in, const u64* tmp, u64 n, u64 kcc, u64 res_stride, u64 i0, u64 count,
                     const __grid_constant__ KsModuli mods, int in_like_result, int accumulate) {
  const u64 per_mod = kcc * n;
  const u64 g = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (g >= per_mod * count) return;
  const u64 e = g / per_mod, r = g - e * per_mod;
  const u64 k = r / n, l = r - k * n;
  const KsModulus& md = mods.m[e];
  const u64 d = n * (res_stride * k + i0 + e) + l;
  const u64 v = finish_value(in[in_like_result ? d : g], tmp[g], md.q, md.a, md.b);
  result[d] = accumulate ? csub(result[d] + v, md.q) : v;
}

// DivideAndRoundQLast in coefficient form: polynomial p of `polys` holds rns limbs of n words; every thread reads limb
// rns-1 and limb i0+e of one coefficient, rounds and finishes in registers and stores limb i0+e.  Limb rns-1 is never
// written, so result may be operand.  mods.m[e]: a, b = q_last^-1 mod q and its Shoup factor, c = the round's `add`.
__global__ void __launch_bounds__(kThreads)
    rescale_coef_kernel(u64* result, const u64* operand, u64 n, u64 rns, u64 i0, u64 count, u64 polys, u64 q_last,
                        u64 mu_last, const __grid_constant__ KsModuli mods) {
  const u64 per_poly = count * n;
  const u64 g = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (g >= per_poly * polys) return;
  const u64 p = g / per_poly, r = g - p * per_poly;
  const u64 e = r / n, l = r - e * n;
  const KsModulus& md = mods.m[e];
  const u64 base = p * rns * n + l, d = base + (i0 + e) * n;
  const u64 t = round_into(operand[base + (rns - 1) * n], q_last, mu_last, md.q, md.mu, md.c);
  result[d] = finish_value(operand[d], t, md.q, md.a, md.b);
}

unsigned blocks_for(u64 items) { return (unsigned)((items + kThreads - 1) / kThreads); }

// the block needs mulmod<true>: one of its moduli has 62 bits (shift = bits(q) - 2 = 60)
bool has_62_bit_modulus(const DyadicModuli& mods, u64 count) {
  for (u64 e = 0; e < count; ++e)
    if (mods.m[e].shift == 60) return true;
  return false;
}

}  // namespace

cudaError_t launch_dyadic_multiply(u64* result, const u64* op1, const u64* op2, u64 n, u64 num_moduli, u64 first,
                                   u64 count, const DyadicModuli& mods, cudaStream_t stream) {
  const u64 total = n * count;
  if (total == 0) return cudaSuccess;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const bool vec = n % 2 == 0 &&
                   ((reinterpret_cast<uintptr_t>(result) | reinterpret_cast<uintptr_t>(op1) |
                     reinterpret_cast<uintptr_t>(op2)) & 15) == 0;
  u64 blocks = blocks_for(vec ? total / 2 : total);
  if (blocks > (u64)sms * 16) blocks = (u64)sms * 16;
  auto kernel = vec ? dyadic_kernel<2, false> : dyadic_kernel<1, false>;
  if (has_62_bit_modulus(mods, count)) kernel = vec ? dyadic_kernel<2, true> : dyadic_kernel<1, true>;
  kernel<<<(unsigned)blocks, kThreads, 0, stream>>>(result, op1, op2, n, num_moduli, first, count, mods);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_rns_eltwise(int op, u64* result, const u64* a, const u64* b, u64 per_mod, u64 count, int in_mf,
                               const DyadicModuli& mods, cudaStream_t stream) {
  const u64 total = per_mod * count;
  if (total == 0) return cudaSuccess;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const bool vec = per_mod % 2 == 0 &&
                   ((reinterpret_cast<uintptr_t>(result) | reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0;
  u64 blocks = blocks_for(vec ? total / 2 : total);
  if (blocks > (u64)sms * 16) blocks = (u64)sms * 16;
  auto kernel = vec ? rns_eltwise_kernel<2, false> : rns_eltwise_kernel<1, false>;
  if (op == kRnsMult && has_62_bit_modulus(mods, count))
    kernel = vec ? rns_eltwise_kernel<2, true> : rns_eltwise_kernel<1, true>;
  kernel<<<(unsigned)blocks, kThreads, 0, stream>>>(result, a, b, per_mod, count, op, in_mf, mods);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_ks_mac(u64* prod, const u64* ops, u64 ops_stride, const KeyPointers& keys, u64 n, u64 jcount,
                          u64 kcc, u64 key_modulus_size, u64 count, const KsModuli& mods, int accumulate,
                          cudaStream_t stream, u64 galois_elt) {
  auto kernel = galois_elt ? ks_mac_kernel<true> : ks_mac_kernel<false>;
  kernel<<<blocks_for(kcc * n * count), kThreads, 0, stream>>>(prod, ops, ops_stride, keys, n, jcount, kcc,
                                                              key_modulus_size, count, mods, accumulate,
                                                              (unsigned)galois_elt);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_ks_weighted_mac(u64* acc, const u64* ops, u64 ops_stride, const WeightedMacElts& elts, u64 n,
                                   u64 jcount, u64 num_elts, u64 key_modulus_size, u64 count, const KsModuli& mods,
                                   bool accumulate, cudaStream_t stream) {
  ks_weighted_mac_kernel<<<blocks_for(n * count), kThreads, 0, stream>>>(acc, ops, ops_stride, elts, n, jcount,
                                                                        num_elts, key_modulus_size, count, mods,
                                                                        accumulate);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_ks_permuted_sum(u64* result, const u64* ct, u64 n, u64 level, u64 i0, u64 count,
                                   const PermutedSumElts& elts, u64 num_elts, const KsModuli& mods, bool accumulate,
                                   cudaStream_t stream) {
  ks_permuted_sum_kernel<<<blocks_for(n * count), kThreads, 0, stream>>>(result, ct, n, level, i0, count, elts,
                                                                        num_elts, mods, accumulate);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_ks_bsgs_sum(u64* x, u64* y, u64* x1, u64* y1, const u64* ct, const u64* prods, u64 prod_stride,
                               u64 n, u64 level, u64 b0, u64 count, u64 giant, const BsgsSumTerms& terms,
                               u64 num_terms, const KsModuli& mods, int mode, cudaStream_t stream) {
  ks_bsgs_sum_kernel<<<blocks_for(n * count), kThreads, 0, stream>>>(x, y, x1, y1, ct, prods, prod_stride, n, level, b0,
                                                                    count, (unsigned)giant, terms, num_terms, mods,
                                                                    mode);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_ks_relin_mac(u64* prod, const u64* ops, u64 ops_stride, const KeyPointers& keys, u64 n, u64 jcount,
                                u64 key_modulus_size, u64 count, const KsModuli& mods, const RelinTensor& tensor,
                                bool accumulate, cudaStream_t stream) {
  ks_relin_mac_kernel<<<blocks_for(n * count), kThreads, 0, stream>>>(prod, ops, ops_stride, keys, n, jcount,
                                                                     key_modulus_size, count, mods, tensor, accumulate);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_relin_tensor_sum(u64* out, u64 n, u64 level, u64 i0, u64 count, const RelinSumPairs& pairs,
                                    u64 num_pairs, const KsModuli& mods, bool accumulate, cudaStream_t stream) {
  relin_tensor_sum_kernel<<<blocks_for(n * count), kThreads, 0, stream>>>(out, n, level, i0, count, pairs, num_pairs,
                                                                         mods, accumulate);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_inner_sum_step(const u64* xa, const u64* ya, u64* xn, u64* yn, u64* xr, u64* yr, u64* y1, u64 n,
                                  u64 level, u64 b0, u64 count, u64 dbl, u64 shift, const KsModuli& mods, int mode,
                                  cudaStream_t stream) {
  inner_sum_step_kernel<<<blocks_for(n * count), kThreads, 0, stream>>>(xa, ya, xn, yn, xr, yr, y1, n, level, b0, count,
                                                                       (unsigned)dbl, (unsigned)shift, mods, mode);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_ks_round(u64* tmp, const u64* t_last, u64 n, u64 kcc, u64 q_last, u64 mu_last, u64 count,
                            const KsModuli& mods, cudaStream_t stream) {
  ks_round_kernel<<<blocks_for(kcc * n * count), kThreads, 0, stream>>>(tmp, t_last, kcc * n, q_last, mu_last, count,
                                                                       mods);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_ks_finish(u64* result, const u64* in, const u64* tmp, u64 n, u64 kcc, u64 res_stride, u64 i0,
                             u64 count, const KsModuli& mods, bool in_like_result, bool accumulate,
                             cudaStream_t stream) {
  ks_finish_kernel<<<blocks_for(kcc * n * count), kThreads, 0, stream>>>(result, in, tmp, n, kcc, res_stride, i0, count,
                                                                        mods, in_like_result, accumulate);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_rescale_coef(u64* result, const u64* operand, u64 n, u64 rns, u64 i0, u64 count, u64 polys,
                                u64 q_last, u64 mu_last, const KsModuli& mods, cudaStream_t stream) {
  rescale_coef_kernel<<<blocks_for(count * n * polys), kThreads, 0, stream>>>(result, operand, n, rns, i0, count, polys,
                                                                             q_last, mu_last, mods);
  count_launch();
  return cudaGetLastError();
}

}  // namespace hexl_b200
