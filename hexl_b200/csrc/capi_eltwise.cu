// Element-wise and Montgomery-form entry points, their RNS batches, DyadicMultiply and PolyMultiplyMulti.
#include <cstdlib>

#include "capi.h"

using namespace hexl_b200;

namespace hexl_b200 {

static int eltwise_dispatch(EltOp op, EltParams p, void* stream) {
  if (p.n == 0) return fail(HEXL_B200_ERR_INVALID_ARG, "Require n != 0");
  PtrInfo pi;
  if (int rc = classify_all({p.result, p.a, p.b}, &pi)) return rc;
  if (pi.where == Where::Device)
    return run_on_device(pi, stream, [&] {
      cudaError_t e = launch_eltwise(op, p, (cudaStream_t)stream);
      return e == cudaSuccess ? 0 : cuda_fail(e, "eltwise launch");
    });
  return run_host(p.result, p.a, p.b, p.n, 1, [&](int, u64, u64, auto&& run) {
    return run([&](u64* r, const u64* a, const u64* b, u64, u64 elems, cudaStream_t s) {
      EltParams q = p;
      q.result = r;
      q.a = a;
      q.b = b;
      q.n = elems;
      return launch_eltwise(op, q, s);
    });
  });
}

static EltParams mult_params(uint64_t q, int in_mf) {
  EltParams p{};
  const DyadicModulus d = dyadic_modulus(q);
  p.q = q;
  p.in_mf = in_mf;
  p.shift = d.shift;
  p.mu = d.mu;
  return p;
}

static DyadicModuli dyadic_moduli(const uint64_t* moduli, uint64_t count) {
  DyadicModuli mods;
  for (uint64_t i = 0; i < count; ++i) mods.m[i] = dyadic_modulus(moduli[i]);
  return mods;
}

static int dyadic_on_device(uint64_t* result, const uint64_t* op1, const uint64_t* op2, uint64_t n,
                            const uint64_t* moduli, uint64_t num_moduli, cudaStream_t s) {
  for (uint64_t first = 0; first < num_moduli; first += kParamBlock) {
    const uint64_t count = std::min<uint64_t>(kParamBlock, num_moduli - first);
    cudaError_t e = launch_dyadic_multiply(result, op1, op2, n, num_moduli, first, count,
                                           dyadic_moduli(moduli + first, count), s);
    if (e != cudaSuccess) return cuda_fail(e, "DyadicMultiply launch");
  }
  return 0;
}

// HEXL_B200_NO_PRODUCT_FUSION=1: the unfused chain (lazy transforms, MultMod kernel, inverse), kept for measurement
static bool product_fusion() {
  static const bool on = !(getenv("HEXL_B200_NO_PRODUCT_FUSION") && atoi(getenv("HEXL_B200_NO_PRODUCT_FUSION")) != 0);
  return on;
}

// A chunk [off, off + elems) of an RNS job is cut at the modulus boundaries it contains and every piece is launched
// under its own modulus.
int run_host_rns(RnsJob job, hexl_b200_ntt* const* handles, const uint64_t* moduli, uint64_t count,
                 u64 per_mod, u64 n, int in_mf, int out_mf, u64* result, const u64* a, const u64* b) {
  const bool need_tables = job == RnsJob::NttFwd || job == RnsJob::NttInv || job == RnsJob::PolyMul;
  // the tables of the moduli inside [lo, hi) on device dev
  return run_host(result, a, b, count * per_mod, n, [&](int dev, u64 lo, u64 hi, auto&& run) {
    std::vector<u64> q(count);
    std::vector<NttDeviceTables> t(need_tables ? count : 0);
    DeviceGuard g;
    if (need_tables)
      if (int rc = g.enter(dev)) return rc;
    for (uint64_t m = 0; m < count; ++m) {
      q[m] = moduli ? moduli[m] : handles[m]->q;
      if (need_tables && m * per_mod < hi && (m + 1) * per_mod > lo)
        if (int rc = device_tables(handles[m], dev, &t[m])) return rc;
    }
    return run([&](u64* r, const u64* a, const u64* b, u64 off, u64 elems, cudaStream_t s) {
      for (u64 pos = off; pos < off + elems;) {
        const u64 m = pos / per_mod;
        const u64 cnt = std::min(off + elems, (m + 1) * per_mod) - pos, o = pos - off;
        cudaError_t e = cudaSuccess;
        switch (job) {
          case RnsJob::NttFwd: e = launch_ntt_forward(t[m], r + o, a + o, in_mf, out_mf, cnt / n, s); break;
          case RnsJob::NttInv: e = launch_ntt_inverse(t[m], r + o, a + o, in_mf, out_mf, cnt / n, s); break;
          case RnsJob::Mult:
          case RnsJob::Add:
          case RnsJob::Sub: {
            EltParams p = job == RnsJob::Mult ? mult_params(q[m], in_mf) : EltParams{};
            p.q = q[m];
            p.result = r + o; p.a = a + o; p.b = b + o; p.n = cnt;
            e = launch_eltwise(job == RnsJob::Mult ? EltOp::MultVV : (job == RnsJob::Add ? EltOp::AddVV : EltOp::SubVV), p, s);
            break;
          }
          case RnsJob::PolyMul: {  // staged buffers: r == a (slot buffer 0), b = slot buffer 1; all in place
            u64* fa = r + o;
            u64* fb = const_cast<u64*>(b) + o;
            if (product_fusion() && q[m] >= (1ull << 30)) {  // (below 2^30 the 32-bit-word transforms win)
              if ((e = launch_ntt_forward(t[m], fa, a + o, 1, 1, cnt / n, s)) != cudaSuccess) return e;
              if ((e = launch_ntt_forward(t[m], fb, fb, 1, 1, cnt / n, s)) != cudaSuccess) return e;
              NttMulti multi{};
              multi.p[0] = t[m].dparams;
              multi.group = (unsigned)(cnt / n);
              multi.mul = fb;
              e = launch_ntt_multi(false, multi, t[m].log_n, q[m], q[m], fa, fa, 1, cnt / n, s);
              break;
            }
            if ((e = launch_ntt_forward(t[m], fa, a + o, 1, 4, cnt / n, s)) != cudaSuccess) return e;
            if ((e = launch_ntt_forward(t[m], fb, fb, 1, 4, cnt / n, s)) != cudaSuccess) return e;
            EltParams p = mult_params(q[m], 4);
            p.result = fa; p.a = fa; p.b = fb; p.n = cnt;
            if ((e = launch_eltwise(EltOp::MultVV, p, s)) != cudaSuccess) return e;
            e = launch_ntt_inverse(t[m], fa, fa, 1, 1, cnt / n, s);
            break;
          }
        }
        if (e != cudaSuccess) return e;
        pos += cnt;
      }
      return cudaSuccess;
    });
  });
}

}  // namespace hexl_b200

// =============================================================== extern "C"
extern "C" {

// ---- eltwise.  Checks mirror the HEXL_CHECKs at the top of each reference op.
int hexl_b200_eltwise_add_mod(uint64_t* result, const uint64_t* op1, const uint64_t* op2, uint64_t n,
                              uint64_t q, void* stream) {
  // eltwise-add-mod.cpp:73-81
  REQUIRE(result && op1 && op2, "Require result, operand1, operand2 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q < (1ull << 63), "Require modulus < 2**63");
  if (int rc = debug_bounds(op1, n, q, "operand1", {result, op1, op2}, stream)) return rc;
  if (int rc = debug_bounds(op2, n, q, "operand2", {result, op1, op2}, stream)) return rc;
  EltParams p{};
  p.result = result; p.a = op1; p.b = op2; p.n = n; p.q = q;
  return eltwise_dispatch(EltOp::AddVV, p, stream);
}

int hexl_b200_eltwise_add_mod_scalar(uint64_t* result, const uint64_t* op1, uint64_t op2, uint64_t n,
                                     uint64_t q, void* stream) {
  // eltwise-add-mod.cpp:95-103
  REQUIRE(result && op1, "Require result, operand1 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q < (1ull << 63), "Require modulus < 2**63");
  REQUIRE(op2 < q, "Require operand2 < modulus");
  if (int rc = debug_bounds(op1, n, q, "operand1", {result, op1}, stream)) return rc;
  EltParams p{};
  p.result = result; p.a = op1; p.n = n; p.q = q; p.scalar = op2;
  return eltwise_dispatch(EltOp::AddVS, p, stream);
}

int hexl_b200_eltwise_sub_mod(uint64_t* result, const uint64_t* op1, const uint64_t* op2, uint64_t n,
                              uint64_t q, void* stream) {
  // eltwise-sub-mod.cpp:69-77
  REQUIRE(result && op1 && op2, "Require result, operand1, operand2 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q < (1ull << 63), "Require modulus < 2**63");
  if (int rc = debug_bounds(op1, n, q, "operand1", {result, op1, op2}, stream)) return rc;
  if (int rc = debug_bounds(op2, n, q, "operand2", {result, op1, op2}, stream)) return rc;
  EltParams p{};
  p.result = result; p.a = op1; p.b = op2; p.n = n; p.q = q;
  return eltwise_dispatch(EltOp::SubVV, p, stream);
}

int hexl_b200_eltwise_sub_mod_scalar(uint64_t* result, const uint64_t* op1, uint64_t op2, uint64_t n,
                                     uint64_t q, void* stream) {
  // eltwise-sub-mod.cpp:91-99
  REQUIRE(result && op1, "Require result, operand1 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q < (1ull << 63), "Require modulus < 2**63");
  REQUIRE(op2 < q, "Require operand2 < modulus");
  if (int rc = debug_bounds(op1, n, q, "operand1", {result, op1}, stream)) return rc;
  EltParams p{};
  p.result = result; p.a = op1; p.n = n; p.q = q; p.scalar = op2;
  return eltwise_dispatch(EltOp::SubVS, p, stream);
}

int hexl_b200_eltwise_mult_mod(uint64_t* result, const uint64_t* op1, const uint64_t* op2, uint64_t n,
                               uint64_t q, uint64_t in_mf, void* stream) {
  // eltwise-mult-mod.cpp:21-36
  REQUIRE(result && op1 && op2, "Require result, operand1, operand2 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(in_mf == 1 || in_mf == 2 || in_mf == 4, "input_mod_factor must be 1, 2 or 4; got %llu", (unsigned long long)in_mf);
  REQUIRE(q < (1ull << 62), "Require modulus < (1ULL << 62)");
  REQUIRE(in_mf * q < (1ull << 63), "Require input_mod_factor * modulus < (1ULL << 63)");
  if (int rc = debug_bounds(op1, n, in_mf * q, "operand1", {result, op1, op2}, stream)) return rc;
  if (int rc = debug_bounds(op2, n, in_mf * q, "operand2", {result, op1, op2}, stream)) return rc;
  EltParams p = mult_params(q, (int)in_mf);
  p.result = result; p.a = op1; p.b = op2; p.n = n;
  return eltwise_dispatch(EltOp::MultVV, p, stream);
}

int hexl_b200_eltwise_fma_mod(uint64_t* result, const uint64_t* arg1, uint64_t arg2, const uint64_t* arg3,
                              uint64_t n, uint64_t q, uint64_t in_mf, void* stream) {
  // eltwise-fma-mod.cpp:20-40
  REQUIRE(result && arg1, "Require result, arg1 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q < (1ull << 61), "Require modulus < (1ULL << 61)");
  REQUIRE(in_mf == 1 || in_mf == 2 || in_mf == 4 || in_mf == 8,
          "input_mod_factor must be 1, 2, 4, or 8. Got %llu", (unsigned long long)in_mf);
  REQUIRE(arg2 < in_mf * q, "arg2 exceeds bound input_mod_factor * modulus");
  if (int rc = debug_bounds(arg1, n, in_mf * q, "arg1", {result, arg1, arg3}, stream)) return rc;
  if (int rc = debug_bounds(arg3, n, in_mf * q, "arg3", {result, arg1, arg3}, stream)) return rc;
  EltParams p{};
  p.result = result; p.a = arg1; p.b = arg3; p.n = n; p.q = q; p.in_mf = (int)in_mf;
  uint64_t s = arg2;  // ReduceMod<in_mf>(arg2), eltwise-fma-mod-internal.hpp:16-17
  if (in_mf >= 8 && s >= 4 * q) s -= 4 * q;
  if (in_mf >= 4 && s >= 2 * q) s -= 2 * q;
  if (in_mf >= 2 && s >= q) s -= q;
  p.scalar = s;
  p.scalar_p = nt::multiply_factor(s, 64, q);
  return eltwise_dispatch(arg3 ? EltOp::Fma : EltOp::FmaNoAdd, p, stream);
}

int hexl_b200_eltwise_reduce_mod(uint64_t* result, const uint64_t* operand, uint64_t n, uint64_t q,
                                 uint64_t in_mf, uint64_t out_mf, void* stream) {
  // eltwise-reduce-mod.cpp:84-92
  REQUIRE(result && operand, "Require result, operand != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(in_mf == q || in_mf == 2 || in_mf == 4, "input_mod_factor must be modulus or 2 or 4; got %llu",
          (unsigned long long)in_mf);
  REQUIRE(out_mf == 1 || out_mf == 2, "output_mod_factor must be 1 or 2; got %llu", (unsigned long long)out_mf);
  EltParams p{};
  p.result = result; p.a = operand; p.n = n; p.q = q; p.out_mf = (int)out_mf;
  // From q >= 2^63 on, every 64-bit word is below 2q, so input_mod_factor 4 is the 2 case; reducing from [0, 4q) would
  // subtract 2q, which wraps (as it does in every tier of the reference).
  if (in_mf == 4 && q >= (1ull << 63)) in_mf = 2;
  if (in_mf == out_mf) {  // eltwise-reduce-mod.cpp:94-99: plain copy (no-op in place)
    if (result == operand) return 0;
    return eltwise_dispatch(EltOp::Copy, p, stream);
  }
  p.in_mf = (in_mf == q) ? 0 : (int)in_mf;
  p.mu = nt::multiply_factor(1, 64, q);
  return eltwise_dispatch(EltOp::Reduce, p, stream);
}

int hexl_b200_eltwise_cmp_add(uint64_t* result, const uint64_t* op1, uint64_t n, int cmp, uint64_t bound,
                              uint64_t diff, void* stream) {
  // eltwise-cmp-add.cpp:18-21
  REQUIRE(result && op1, "Require result, operand1 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(diff != 0, "Require diff != 0");
  REQUIRE(cmp >= 0 && cmp <= 7, "cmp must be a CMPINT value (0..7)");
  EltParams p{};
  p.result = result; p.a = op1; p.n = n; p.scalar = bound; p.scalar_p = diff; p.cmp = cmp;
  return eltwise_dispatch(EltOp::CmpAdd, p, stream);
}

int hexl_b200_eltwise_cmp_sub_mod(uint64_t* result, const uint64_t* op1, uint64_t n, uint64_t q, int cmp,
                                  uint64_t bound, uint64_t diff, void* stream) {
  // eltwise-cmp-sub-mod.cpp:21-25,50-55
  REQUIRE(result && op1, "Require result, operand1 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(diff != 0, "Require diff != 0");
  REQUIRE(diff < q, "Diff >= modulus");
  REQUIRE(cmp >= 0 && cmp <= 7, "cmp must be a CMPINT value (0..7)");
  EltParams p{};
  p.result = result; p.a = op1; p.n = n; p.q = q; p.scalar = bound; p.scalar_p = diff; p.cmp = cmp;
  p.mu = nt::multiply_factor(1, 64, q);
  return eltwise_dispatch(EltOp::CmpSubMod, p, stream);
}

// ---- Montgomery-form helpers (SURVEY 8(f)-4)
uint64_t hexl_b200_hensel_lemma_2adic_root(uint32_t r, uint64_t q) {
  if (r == 0 || r > 64 || !(q & 1)) return 0;
  return nt::neg_inverse_mod_pow2(r, q);
}
uint64_t hexl_b200_montgomery_reduce(uint64_t T_hi, uint64_t T_lo, uint64_t q, int r, uint64_t inv_mod) {
  if (r < 1 || r > 62 || q < 2) return 0;
  return nt::montgomery_reduce(T_hi, T_lo, q, r, inv_mod);
}
static int mont_dispatch(EltOp op, uint64_t* result, const uint64_t* a, const uint64_t* b, uint64_t scalar, uint64_t n,
                         uint64_t q, int r, uint64_t neg_inv_mod, void* stream) {
  // checks of eltwise-reduce-mod-avx512.hpp:160-176
  REQUIRE(result && a && (op != EltOp::MontMult || b), "Require result, operands != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q & 1, "gcd(modulus, R) != 1");
  REQUIRE(r >= 1 && r <= 62, "With r > 62 internal ops might overflow");
  REQUIRE((1ull << r) > q, "Needs R bigger than q.");
  REQUIRE(((q * neg_inv_mod + 1) & ((1ull << r) - 1)) == 0, "neg_inv_mod is not -1/q mod R");
  if (int rc = debug_bounds(a, n, q, "operand a", {result, a, b}, stream)) return rc;
  if (op == EltOp::MontMult)
    if (int rc = debug_bounds(b, n, q, "operand b", {result, a, b}, stream)) return rc;
  EltParams p{};
  p.result = result; p.a = a; p.b = b; p.n = n; p.q = q; p.mu = neg_inv_mod & ((1ull << r) - 1); p.shift = r; p.scalar = scalar;
  return eltwise_dispatch(op, p, stream);
}
int hexl_b200_eltwise_mont_reduce_mod(uint64_t* result, const uint64_t* a, const uint64_t* b, uint64_t n, uint64_t q,
                                      int r, uint64_t neg_inv_mod, void* stream) {
  return mont_dispatch(EltOp::MontMult, result, a, b, 0, n, q, r, neg_inv_mod, stream);
}
int hexl_b200_eltwise_montgomery_form_in(uint64_t* result, const uint64_t* a, uint64_t R2_mod_q, uint64_t n, uint64_t q,
                                         int r, uint64_t neg_inv_mod, void* stream) {
  REQUIRE(R2_mod_q < q, "Require R2_mod_q < modulus");
  return mont_dispatch(EltOp::MontIn, result, a, nullptr, R2_mod_q, n, q, r, neg_inv_mod, stream);
}
int hexl_b200_eltwise_montgomery_form_out(uint64_t* result, const uint64_t* a, uint64_t n, uint64_t q, int r,
                                          uint64_t neg_inv_mod, void* stream) {
  return mont_dispatch(EltOp::MontOut, result, a, nullptr, 0, n, q, r, neg_inv_mod, stream);
}

// ---- SEAL-shaped composites
// device side of EltwiseMultMod over an RNS batch
static int rns_eltwise_on_device(int op, uint64_t* result, const uint64_t* a, const uint64_t* b, uint64_t per_mod,
                                 const uint64_t* moduli, uint64_t num_moduli, int in_mf, cudaStream_t s) {
  for (uint64_t first = 0; first < num_moduli; first += kParamBlock) {
    const uint64_t count = std::min<uint64_t>(kParamBlock, num_moduli - first);
    const uint64_t off = first * per_mod;
    cudaError_t e = launch_rns_eltwise(op, result + off, a + off, b + off, per_mod, count, in_mf,
                                       dyadic_moduli(moduli + first, count), s);
    if (e != cudaSuccess) return cuda_fail(e, "eltwise (RNS batch) launch");
  }
  return 0;
}

static int rns_eltwise_entry(int op, uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                             uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli, uint64_t in_mf,
                             void* stream) {
  REQUIRE(result && operand1 && operand2 && moduli, "Require result, operand1, operand2, moduli != nullptr");
  REQUIRE(n_per_modulus != 0 && num_moduli != 0, "Require n != 0");
  REQUIRE(in_mf == 1 || in_mf == 2 || in_mf == 4, "Require input_mod_factor = 1, 2, or 4");
  for (uint64_t i = 0; i < num_moduli; ++i)
    REQUIRE(moduli[i] > 1 && moduli[i] < (1ull << 62) && moduli[i] * in_mf < (1ull << 63),
            "Require 1 < modulus < 2^62 and input_mod_factor * modulus < 2^63");
  PtrInfo pi;
  if (int rc = classify_all({result, operand1, operand2}, &pi)) return rc;
  if (pi.where == Where::Device)
    return run_on_device(pi, stream, [&] {
      auto bound = [&](u64 i) { return moduli[i] * in_mf; };
      if (int rc = check_limb_bounds(operand1, 1, num_moduli, n_per_modulus, bound, pi, "operand1", stream)) return rc;
      if (int rc = check_limb_bounds(operand2, 1, num_moduli, n_per_modulus, bound, pi, "operand2", stream)) return rc;
      return rns_eltwise_on_device(op, result, operand1, operand2, n_per_modulus, moduli, num_moduli, (int)in_mf,
                                   (cudaStream_t)stream);
    });
  const RnsJob job = op == kRnsMult ? RnsJob::Mult : (op == kRnsAdd ? RnsJob::Add : RnsJob::Sub);
  return run_host_rns(job, nullptr, moduli, num_moduli, n_per_modulus, 1, (int)in_mf, 1, result, operand1, operand2);
}

int hexl_b200_eltwise_mult_mod_multi(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                                     uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli,
                                     uint64_t in_mf, void* stream) {
  return rns_eltwise_entry(kRnsMult, result, operand1, operand2, n_per_modulus, moduli, num_moduli, in_mf, stream);
}
int hexl_b200_eltwise_add_mod_multi(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                                    uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli, void* stream) {
  return rns_eltwise_entry(kRnsAdd, result, operand1, operand2, n_per_modulus, moduli, num_moduli, 1, stream);
}
int hexl_b200_eltwise_sub_mod_multi(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                                    uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli, void* stream) {
  return rns_eltwise_entry(kRnsSub, result, operand1, operand2, n_per_modulus, moduli, num_moduli, 1, stream);
}

// FwdNTT(b) into scratch, FwdNTT(a) into result, point-wise product, InvNTT: all moduli per launch.  b is read before
// result is first written, so result may be a, b or both (an in-place square)
static int poly_multiply_on_device(int dev, hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                                   const uint64_t* a, const uint64_t* b, uint64_t group, cudaStream_t s) {
  const uint64_t n = handles[0]->n, total = count * group * n;
  Scratch ws(s);
  uint64_t* fb = nullptr;
  if (int rc = ws.get(&fb, total)) return rc;
  std::vector<uint64_t> moduli(count);
  for (uint64_t i = 0; i < count; ++i) moduli[i] = handles[i]->q;
  if (product_fusion()) {
    // canonical transforms, then ONE inverse transform that multiplies on load: no MultMod kernel, and the product
    // never travels to HBM and back (dyadic-multiply-internal.cpp:17-73 folded into the transform that consumes it)
    if (int rc = ntt_multi_on_device(true, dev, handles, count, fb, b, 1, group, s)) return rc;
    if (int rc = ntt_multi_on_device(true, dev, handles, count, result, a, 1, group, s)) return rc;
    return ntt_multi_on_device(false, dev, handles, count, result, result, 1, group, s, nullptr, false, fb);
  }
  if (int rc = ntt_multi_on_device(true, dev, handles, count, fb, b, 4, group, s)) return rc;
  if (int rc = ntt_multi_on_device(true, dev, handles, count, result, a, 4, group, s)) return rc;
  if (int rc = rns_eltwise_on_device(kRnsMult, result, result, fb, group * n, moduli.data(), count, 4, s)) return rc;
  return ntt_multi_on_device(false, dev, handles, count, result, result, 1, group, s);
}

int hexl_b200_poly_multiply_multi(hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result, const uint64_t* a,
                                  const uint64_t* b, uint64_t group, void* stream) {
  REQUIRE(handles && result && a && b, "Require handles, result, a, b != nullptr");
  if (count == 0 || group == 0) return 0;
  for (uint64_t i = 0; i < count; ++i) {
    REQUIRE(handles[i] != nullptr, "Require handles[i] != nullptr");
    REQUIRE(handles[i]->n == handles[0]->n, "all handles must share one degree");
    REQUIRE(handles[i]->q < (1ull << 61), "Require modulus < 2^61 (lazy transform outputs feed the product)");
  }
  PtrInfo pi;
  if (int rc = classify_all({result, a, b}, &pi)) return rc;
  const uint64_t n = handles[0]->n;
  auto bound = [&](u64 i) { return handles[i]->q; };
  if (int rc = check_limb_bounds(a, 1, count, group * n, bound, pi, "a", stream)) return rc;
  if (int rc = check_limb_bounds(b, 1, count, group * n, bound, pi, "b", stream)) return rc;
  if (pi.where == Where::Device)
    return run_on_device(pi, stream, [&] {
      return poly_multiply_on_device(pi.device, handles, count, result, a, b, group, (cudaStream_t)stream);
    });
  // host pointers: every chunk of polynomials is copied in, transformed, multiplied, transformed back and
  // copied out on one of the rotating staging streams, so the PCIe copies of one chunk hide under the
  // kernels of the others; with host devices set the polynomials are split across the GPUs
  return run_host_rns(RnsJob::PolyMul, handles, nullptr, count, group * n, n, 1, 1, result, a, b);
}

int hexl_b200_dyadic_multiply(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2, uint64_t n,
                              const uint64_t* moduli, uint64_t num_moduli, void* stream) {
  // dyadic-multiply-internal.cpp:20-24
  REQUIRE(result && operand1 && operand2 && moduli, "Require result, operand1, operand2, moduli != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(num_moduli != 0, "Require num_moduli != 0");
  for (uint64_t i = 0; i < num_moduli; ++i)
    REQUIRE(moduli[i] > 1 && moduli[i] < (1ull << 62), "Require 1 < modulus < 2^62");
  PtrInfo pi;
  if (int rc = classify_all({result, operand1, operand2}, &pi)) return rc;
  if (pi.where == Where::Device)
    return run_on_device(pi, stream, [&] {
      return dyadic_on_device(result, operand1, operand2, n, moduli, num_moduli, (cudaStream_t)stream);
    });
  // Host pointers: blocks of moduli travel through the staging slots (stage_items) of the first host device (the
  // layout is [polynomial][modulus][n], so a block of moduli is a 2-D copy: 2 rows in, 3 rows out).
  std::vector<int> devs;
  if (int rc = host_devices(&devs)) return rc;
  u64 mb = std::max<u64>(1, (kChunkBytes / sizeof(u64)) / (3 * n));
  mb = std::min<u64>({mb, (u64)kParamBlock, num_moduli});
  const size_t row = (size_t)num_moduli * n * sizeof(u64);  // host pitch: one polynomial over all moduli
  return stage_items({devs[0]}, num_moduli, mb, [&](int, u64, u64, auto&& stage) {
    return stage([&](const StageSlot& sl, u64 m0, u64 cnt) -> int {
      const size_t w = (size_t)cnt * n * sizeof(u64);
      if (int rc = sl.reserve(0, 3 * w)) return rc;
      if (int rc = sl.reserve(1, 2 * w)) return rc;
      if (int rc = sl.reserve(2, 2 * w)) return rc;
      cudaStream_t sx = sl.stream();
      u64 *dr = sl.buf(0), *d1 = sl.buf(1), *d2 = sl.buf(2);
      CU(cudaMemcpy2DAsync(d1, w, operand1 + m0 * n, row, w, 2, cudaMemcpyHostToDevice, sx));
      CU(cudaMemcpy2DAsync(d2, w, operand2 + m0 * n, row, w, 2, cudaMemcpyHostToDevice, sx));
      if (int rc = dyadic_on_device(dr, d1, d2, n, moduli + m0, cnt, sx)) return rc;
      CU(cudaMemcpy2DAsync(result + m0 * n, row, dr, w, w, 3, cudaMemcpyDeviceToHost, sx));
      return 0;
    });
  });
}

}  // extern "C"
