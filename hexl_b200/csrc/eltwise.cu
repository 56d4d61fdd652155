// Element-wise modular kernels: straight HBM-bound grids.
//
// One templated streaming kernel; each op is a functor.  16-byte-aligned
// operands go through 128-bit loads/stores (ulonglong2, 4 in flight per thread
// per operand); anything else through the scalar instantiation.  Algorithmic
// traffic: 24 B/element for the two-input ops, 16 B/element for the others.
//
// Semantics follow the reference's scalar definitions:
//   AddMod      hexl/eltwise/eltwise-add-mod.cpp:16-69
//   SubMod      hexl/eltwise/eltwise-sub-mod.cpp:16-65
//   MultMod     hexl/eltwise/eltwise-mult-mod-internal.hpp:33-101
//   FMAMod      hexl/eltwise/eltwise-fma-mod-internal.hpp:11-39
//   ReduceMod   hexl/eltwise/eltwise-reduce-mod.cpp:16-79,94-99
//   CmpAdd      hexl/eltwise/eltwise-cmp-add.cpp:32-106
//   CmpSubMod   hexl/eltwise/eltwise-cmp-sub-mod.cpp:47-66
//   Montgomery  hexl/include/hexl/number-theory/number-theory.hpp:269-301; hexl/eltwise/eltwise-reduce-mod-avx512.hpp:156-352
#include "internal.h"

namespace hexl_b200 {
namespace {

constexpr int kThreads = 256;
constexpr int kUnroll = 4;

// CMPINT semantics: hexl/util/util-internal.hpp:16-42
__device__ __forceinline__ bool cmp_holds(int cmp, u64 lhs, u64 rhs) {
  switch (cmp) {
    case 0: return lhs == rhs;
    case 1: return lhs < rhs;
    case 2: return lhs <= rhs;
    case 3: return false;
    case 4: return lhs != rhs;
    case 5: return lhs >= rhs;
    case 6: return lhs > rhs;
    default: return true;
  }
}

struct FAddVV {
  u64 q;
  __device__ __forceinline__ u64 operator()(u64 a, u64 b) const { return csub(a + b, q); }
};
struct FAddVS {
  u64 q, s;
  __device__ __forceinline__ u64 operator()(u64 a, u64) const {
    u64 gap = q - s;
    return a >= gap ? a - gap : a + s;
  }
};
struct FSubVV {
  u64 q;
  __device__ __forceinline__ u64 operator()(u64 a, u64 b) const {
    return a >= b ? a - b : a + q - b;
  }
};
struct FSubVS {
  u64 q, s;
  __device__ __forceinline__ u64 operator()(u64 a, u64) const {
    return a >= s ? a - s : a + q - s;
  }
};
// generalised Barrett, alpha = 62, beta = -2 (eltwise-mult-mod-internal.hpp:52-99).  The quotient estimate is low by at
// most one while bits(q) <= 61, so z < 2q.  At 62 bits (shift == 60) alpha - bits(q) = 0 and it can be low by two:
// WIDE reduces z from [0, 3q) with a second conditional subtraction (the reference's scalar tier makes one only).
template <int IN_MF, bool WIDE>
struct FMult {
  u64 q, mu;
  int shift;
  __device__ __forceinline__ u64 operator()(u64 a, u64 b) const {
    u64 x = reduce_from<IN_MF>(a, q), y = reduce_from<IN_MF>(b, q);
    u64 lo = x * y, hi = mulhi(x, y);
    // c1 = floor(U / 2^shift); shift in [0, 60]
    u64 c1 = shift ? ((lo >> shift) | (hi << (64 - shift))) : lo;
    u64 z = csub(lo - mulhi(c1, mu) * q, q);
    return WIDE ? csub(z, q) : z;
  }
};
template <int IN_MF, bool ADD>
struct FFma {
  u64 q, s, sp;  // s = reduced arg2, sp = floor(s * 2^64 / q)
  __device__ __forceinline__ u64 operator()(u64 a, u64 c) const {
    u64 x = reduce_from<IN_MF>(a, q);
    u64 p = csub(shoup_lazy(x, s, sp, q), q);
    if (ADD) p = csub(p + reduce_from<IN_MF>(c, q), q);
    return p;
  }
};
// in_mf: 0 -> arbitrary 64-bit input (Barrett-64), 2, 4
template <int IN_MF, int OUT_MF>
struct FReduce {
  u64 q, mu;
  __device__ __forceinline__ u64 operator()(u64 x, u64) const {
    if (IN_MF == 0) {
      // for x < q the quotient estimate is 0, so the reference's `if (x >= q)`
      // guard (eltwise-reduce-mod.cpp:37,46) is implied
      u64 r = barrett64_lazy(x, q, mu);
      return OUT_MF == 1 ? csub(r, q) : r;
    }
    if (IN_MF == 2) return csub(x, q);
    x = csub(x, q << 1);
    return OUT_MF == 1 ? csub(x, q) : x;
  }
};
struct FCopy {
  __device__ __forceinline__ u64 operator()(u64 x, u64) const { return x; }
};
struct FCmpAdd {
  u64 bound, diff;
  int cmp;
  __device__ __forceinline__ u64 operator()(u64 x, u64) const {
    return cmp_holds(cmp, x, bound) ? x + diff : x;
  }
};
struct FCmpSubMod {
  u64 q, mu, bound, diff;
  int cmp;
  __device__ __forceinline__ u64 operator()(u64 x, u64) const {
    bool hit = cmp_holds(cmp, x, bound);
    // true x % q for any 64-bit x: Barrett estimate is off by at most one
    u64 r = barrett64_lazy(x, q, mu);
    r = r >= q ? r - q : r;
    return hit ? (r >= diff ? r - diff : r + q - diff) : r;
  }
};

// Montgomery reduction with R = 2^r, q < R <= 2^62 (MontgomeryReduce<64>, number-theory.hpp:269-301; the element-wise
// helpers of hexl/eltwise/eltwise-reduce-mod-avx512.hpp:156-352): T = hi:lo < q*R -> T / R mod q in [0, q).
// (T + m q) is a multiple of R below 2 q R <= 2^125; its quotient by R is assembled from the two 64-bit halves.
struct MontParams {
  u64 q, ninv;  // ninv = -q^-1 mod R
  int r;
  __device__ __forceinline__ u64 redc(u64 hi, u64 lo) const {
    const u64 mask = (1ull << r) - 1;
    const u64 mm = ((lo & mask) * ninv) & mask;
    const u64 mq_lo = mm * q, mq_hi = mulhi(mm, q);
    const u64 t_lo = lo + mq_lo;
    const u64 t_hi = hi + mq_hi + (t_lo < lo ? 1ull : 0ull);
    const u64 s = (t_hi << (64 - r)) | (t_lo >> r);
    return csub(s, q);
  }
};
struct FMontMult {
  MontParams p;
  __device__ __forceinline__ u64 operator()(u64 a, u64 b) const { return p.redc(mulhi(a, b), a * b); }
};
struct FMontIn {
  MontParams p;
  u64 r2;  // R^2 mod q
  __device__ __forceinline__ u64 operator()(u64 a, u64) const { return p.redc(mulhi(a, r2), a * r2); }
};
struct FMontOut {
  MontParams p;
  __device__ __forceinline__ u64 operator()(u64 a, u64) const { return p.redc(0, a); }
};

// NIN = number of vector inputs.  VEC = 2 -> 128-bit accesses (n counts pairs).
template <class F, int NIN, int VEC>
__global__ void __launch_bounds__(kThreads) elt_kernel(u64* r, const u64* a,
                                                       const u64* b,
                                                       u64 n_items, F f) {
  const u64 stride = (u64)gridDim.x * kThreads;
  u64 i = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (VEC == 2) {
    // full tiles: kUnroll independent 128-bit loads per operand in flight
    for (; i + (kUnroll - 1) * stride < n_items; i += kUnroll * stride) {
      ulonglong2 va[kUnroll], vb[kUnroll];
#pragma unroll
      for (int k = 0; k < kUnroll; ++k) {
        va[k] = ld_stream2(a + 2 * (i + k * stride));
        if (NIN == 2) vb[k] = ld_stream2(b + 2 * (i + k * stride));
      }
#pragma unroll
      for (int k = 0; k < kUnroll; ++k) {
        ulonglong2 o;
        o.x = f(va[k].x, NIN == 2 ? vb[k].x : 0ull);
        o.y = f(va[k].y, NIN == 2 ? vb[k].y : 0ull);
        st_stream2(r + 2 * (i + k * stride), o);
      }
    }
    for (; i < n_items; i += stride) {
      ulonglong2 va = ld_stream2(a + 2 * i), vb = va;
      if (NIN == 2) vb = ld_stream2(b + 2 * i);
      ulonglong2 o;
      o.x = f(va.x, vb.x);
      o.y = f(va.y, vb.y);
      st_stream2(r + 2 * i, o);
    }
  } else {
    for (; i < n_items; i += stride) {
      u64 x = a[i], y = NIN == 2 ? b[i] : 0ull;
      r[i] = f(x, y);
    }
  }
}

template <class F, int NIN>
cudaError_t run(const EltParams& p, F f, cudaStream_t stream) {
  if (p.n == 0) return cudaSuccess;
  auto mis = [](const void* x) { return (reinterpret_cast<uintptr_t>(x) & 15u) != 0; };
  const bool vec = !(mis(p.result) || mis(p.a) || (NIN == 2 && mis(p.b)));
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const u64 max_blocks = (u64)sms * 8;  // 8 resident CTAs of 256 threads per SM
  if (vec) {
    u64 pairs = p.n / 2;
    if (pairs) {
      u64 blocks = (pairs + (u64)kThreads * kUnroll - 1) / ((u64)kThreads * kUnroll);
      if (blocks > max_blocks) blocks = max_blocks;
      elt_kernel<F, NIN, 2><<<(unsigned)blocks, kThreads, 0, stream>>>(p.result, p.a, p.b, pairs, f);
      count_launch();
    }
    if (p.n & 1) {  // odd tail element
      u64 off = p.n - 1;
      elt_kernel<F, NIN, 1><<<1, kThreads, 0, stream>>>(p.result + off, p.a + off,
                                                       NIN == 2 ? p.b + off : nullptr, 1, f);
      count_launch();
    }
  } else {
    u64 blocks = (p.n + kThreads - 1) / kThreads;
    if (blocks > max_blocks) blocks = max_blocks;
    elt_kernel<F, NIN, 1><<<(unsigned)blocks, kThreads, 0, stream>>>(p.result, p.a, p.b, p.n, f);
    count_launch();
  }
  return cudaGetLastError();
}

template <bool WIDE>
cudaError_t run_mult(const EltParams& p, cudaStream_t s) {
  switch (p.in_mf) {
    case 1: return run<FMult<1, WIDE>, 2>(p, FMult<1, WIDE>{p.q, p.mu, p.shift}, s);
    case 2: return run<FMult<2, WIDE>, 2>(p, FMult<2, WIDE>{p.q, p.mu, p.shift}, s);
    default: return run<FMult<4, WIDE>, 2>(p, FMult<4, WIDE>{p.q, p.mu, p.shift}, s);
  }
}

}  // namespace

cudaError_t launch_eltwise(EltOp op, const EltParams& p, cudaStream_t s) {
  switch (op) {
    case EltOp::AddVV: return run<FAddVV, 2>(p, FAddVV{p.q}, s);
    case EltOp::AddVS: return run<FAddVS, 1>(p, FAddVS{p.q, p.scalar}, s);
    case EltOp::SubVV: return run<FSubVV, 2>(p, FSubVV{p.q}, s);
    case EltOp::SubVS: return run<FSubVS, 1>(p, FSubVS{p.q, p.scalar}, s);
    case EltOp::MultVV:  // shift = bits(q) - 2: 60 for the 62-bit moduli
      return p.shift == 60 ? run_mult<true>(p, s) : run_mult<false>(p, s);
    case EltOp::Fma:
      switch (p.in_mf) {
        case 1: return run<FFma<1, true>, 2>(p, FFma<1, true>{p.q, p.scalar, p.scalar_p}, s);
        case 2: return run<FFma<2, true>, 2>(p, FFma<2, true>{p.q, p.scalar, p.scalar_p}, s);
        case 4: return run<FFma<4, true>, 2>(p, FFma<4, true>{p.q, p.scalar, p.scalar_p}, s);
        default: return run<FFma<8, true>, 2>(p, FFma<8, true>{p.q, p.scalar, p.scalar_p}, s);
      }
    case EltOp::FmaNoAdd:
      switch (p.in_mf) {
        case 1: return run<FFma<1, false>, 1>(p, FFma<1, false>{p.q, p.scalar, p.scalar_p}, s);
        case 2: return run<FFma<2, false>, 1>(p, FFma<2, false>{p.q, p.scalar, p.scalar_p}, s);
        case 4: return run<FFma<4, false>, 1>(p, FFma<4, false>{p.q, p.scalar, p.scalar_p}, s);
        default: return run<FFma<8, false>, 1>(p, FFma<8, false>{p.q, p.scalar, p.scalar_p}, s);
      }
    case EltOp::Reduce:
      if (p.in_mf == 0)
        return p.out_mf == 1 ? run<FReduce<0, 1>, 1>(p, FReduce<0, 1>{p.q, p.mu}, s)
                             : run<FReduce<0, 2>, 1>(p, FReduce<0, 2>{p.q, p.mu}, s);
      if (p.in_mf == 2) return run<FReduce<2, 1>, 1>(p, FReduce<2, 1>{p.q, p.mu}, s);
      return p.out_mf == 1 ? run<FReduce<4, 1>, 1>(p, FReduce<4, 1>{p.q, p.mu}, s)
                           : run<FReduce<4, 2>, 1>(p, FReduce<4, 2>{p.q, p.mu}, s);
    case EltOp::Copy: return run<FCopy, 1>(p, FCopy{}, s);
    case EltOp::MontMult: return run<FMontMult, 2>(p, FMontMult{MontParams{p.q, p.mu, p.shift}}, s);
    case EltOp::MontIn: return run<FMontIn, 1>(p, FMontIn{MontParams{p.q, p.mu, p.shift}, p.scalar}, s);
    case EltOp::MontOut: return run<FMontOut, 1>(p, FMontOut{MontParams{p.q, p.mu, p.shift}}, s);
    case EltOp::CmpAdd: return run<FCmpAdd, 1>(p, FCmpAdd{p.scalar, p.scalar_p, p.cmp}, s);
    case EltOp::CmpSubMod:
      return run<FCmpSubMod, 1>(p, FCmpSubMod{p.q, p.mu, p.scalar, p.scalar_p, p.cmp}, s);
  }
  return cudaErrorInvalidValue;
}

}  // namespace hexl_b200
