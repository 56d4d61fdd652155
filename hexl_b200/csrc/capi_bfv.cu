// BFV ciphertext multiplication by BEHZ (hexl_b200_bfv_multiply): the argument rules, the bound on Bsk, the constant
// tables of the two kernels of bfv.cu (cached on each device), and the chain extension -> forward transforms -> tensor
// -> inverse transforms -> scaling.  The relinearized call (capi_hybrid.cu) runs the same chain.
#include <numeric>

#include "capi.h"

using namespace hexl_b200;

namespace hexl_b200 {

namespace {

uint64_t mul_mod(uint64_t a, uint64_t b, uint64_t m) { return (uint64_t)((unsigned __int128)a * b % m); }

// prod of `moduli` except index `skip` (none when skip >= count), mod m
uint64_t product_mod(const std::vector<uint64_t>& moduli, size_t skip, uint64_t m) {
  uint64_t r = 1 % m;
  for (size_t i = 0; i < moduli.size(); ++i)
    if (i != skip) r = mul_mod(r, moduli[i] % m, m);
  return r;
}

// (Q/q_i)^-1 mod 2^32 style products modulo 2^32: prod of moduli except `skip`, wrapping
uint32_t product_mod32(const std::vector<uint64_t>& moduli, size_t skip) {
  uint32_t r = 1;
  for (size_t i = 0; i < moduli.size(); ++i)
    if (i != skip) r *= (uint32_t)moduli[i];
  return r;
}

uint32_t inverse_mod32(uint32_t x) {  // x odd: Newton's iteration doubles the correct low bits
  uint32_t y = x;                     // correct to 3 bits
  for (int i = 0; i < 4; ++i) y *= 2 - x * y;
  return y;
}

void push_reducer(std::vector<uint64_t>& tab, uint64_t m) {  // m, floor(2^64 / m), 2^64 mod m, its Shoup factor
  const uint64_t mu = nt::multiply_factor(1, 64, m);
  const Twiddle R = make_twiddle(mu * (0 - m) % m, m);
  tab.insert(tab.end(), {m, mu, R.w, R.wp});
}

void push_twiddle(std::vector<uint64_t>& tab, uint64_t w, uint64_t m) {
  const Twiddle t = make_twiddle(w % m, m);
  tab.insert(tab.end(), {t.w, t.wp});
}

}  // namespace

bool behz_bound_holds(uint64_t n, uint64_t t, const uint64_t* q, uint64_t l, const uint64_t* b, uint64_t k,
                      uint64_t m_sk) {
  if (m_sk < 2 * k + 2) return false;
  Big lhs{1}, rhs{1};
  for (uint64_t i = 0; i < l; ++i) big_mul(lhs, q[i]);
  big_mul(lhs, n);
  big_mul(lhs, t);
  big_mul(lhs, (1ull << 32) + 2 * l);
  big_mul(lhs, (1ull << 32) + 2 * l);
  big_add_at(lhs, 1, 2 * (l + 1));  // 2 (l + 1) m~^2 = 2 (l + 1) 2^64
  for (uint64_t j = 0; j < k; ++j) big_mul(rhs, b[j]);
  big_mul(rhs, m_sk - 1 - 2 * k);
  rhs.insert(rhs.begin(), 0);  // times m~^2 = 2^64
  return big_le(lhs, rhs);
}

int bfv_check(const void* result, const void* ct1, const void* ct2, uint64_t n, const uint64_t* moduli, uint64_t l,
              const uint64_t* base_b, uint64_t k, uint64_t m_sk, uint64_t t) {
  REQUIRE(result && ct1 && ct2 && moduli && base_b, "Require non-null arguments");
  REQUIRE(n >= 2 && n <= (1ull << 20) && !(n & (n - 1)), "Require n a power of two in [2, 2^20]");
  REQUIRE(l >= 1 && l <= (uint64_t)kParamBlock, "Require 1 <= level_size <= %d", kParamBlock);
  REQUIRE(k >= 1 && k <= (uint64_t)kParamBlock, "Require 1 <= base_b_size <= %d", kParamBlock);
  REQUIRE(t >= 2 && t < (1ull << 61), "Require 2 <= plain_modulus < 2^61");
  std::vector<uint64_t> all(moduli, moduli + l);
  all.insert(all.end(), base_b, base_b + k);
  all.push_back(m_sk);
  for (size_t i = 0; i < all.size(); ++i) {
    const char* what = i < l ? "moduli" : i < l + k ? "base_b" : "m_sk";
    const unsigned long long at = i < l ? i : i < l + k ? i - l : 0;
    const char* why = "";
    REQUIRE(all[i] < (1ull << 61), "Require %s[%llu] < 2^61", what, at);
    REQUIRE(check_ntt_arguments(n, all[i], &why), "%s[%llu]: %s", what, at, why);
    for (size_t j = 0; j < i; ++j)
      REQUIRE(std::gcd(all[i], all[j]) == 1, "Require the moduli of Q, B and m_sk pairwise coprime (%s[%llu])", what,
              at);
  }
  REQUIRE(behz_bound_holds(n, t, moduli, l, base_b, k, m_sk),
          "Bsk = base_b and m_sk is too small for an exact conversion back to Q: require "
          "n t Q (2^32 + 2l)^2 + 2 (l + 1) 2^64 <= B (m_sk - 1 - 2k) 2^64");
  return 0;
}

int bfv_plan(BfvPlan* pl, uint64_t n, const uint64_t* moduli, uint64_t l, const uint64_t* base_b, uint64_t k,
             uint64_t m_sk, uint64_t t) {
  pl->n = n;
  pl->l = l;
  pl->k = k;
  const std::vector<uint64_t> Q(moduli, moduli + l), B(base_b, base_b + k);
  std::vector<uint64_t> bsk(B);
  bsk.push_back(m_sk);
  pl->mods = Q;
  pl->mods.insert(pl->mods.end(), bsk.begin(), bsk.end());
  for (size_t m = 0; m < pl->mods.size(); ++m)
    if (int rc = pl->h.load(m, n, pl->mods[m])) return rc;
  const uint64_t mt = 1ull << 32;
  // extension table
  auto& ext = pl->ext_tab;
  ext.clear();
  for (uint64_t i = 0; i < l; ++i) {
    const uint64_t q = Q[i];
    ext.push_back(q);
    push_twiddle(ext, mul_mod(mt % q, nt::inverse_mod(product_mod(Q, i, q), q), q), q);
  }
  for (uint64_t i = 0; i < l; ++i) ext.push_back(product_mod32(Q, i));
  ext.push_back((uint32_t)(0u - inverse_mod32(product_mod32(Q, l))));
  for (uint64_t m : bsk) {
    push_reducer(ext, m);
    const uint64_t Qm = product_mod(Q, l, m);
    ext.push_back(Qm);
    ext.push_back((m - mul_mod(Qm, mt % m, m)) % m);
    push_twiddle(ext, nt::inverse_mod(mt % m, m), m);
  }
  for (uint64_t m : bsk)
    for (uint64_t i = 0; i < l; ++i) ext.push_back(product_mod(Q, i, m));
  // scaling table
  auto& sc = pl->scale_tab;
  sc.clear();
  for (uint64_t i = 0; i < l; ++i) {
    const uint64_t q = Q[i];
    sc.push_back(q);
    push_twiddle(sc, mul_mod(t % q, nt::inverse_mod(product_mod(Q, i, q), q), q), q);
  }
  for (uint64_t e = 0; e <= k; ++e) {
    const uint64_t m = bsk[e], qinv = nt::inverse_mod(product_mod(Q, l, m), m);
    push_reducer(sc, m);
    push_twiddle(sc, mul_mod(t % m, qinv, m), m);
    push_twiddle(sc, (m - qinv) % m, m);
    if (e < k)
      push_twiddle(sc, nt::inverse_mod(product_mod(B, e, m), m), m);
    else
      sc.insert(sc.end(), {0, 0});
  }
  for (uint64_t m : bsk)
    for (uint64_t i = 0; i < l; ++i) sc.push_back(product_mod(Q, i, m));
  std::vector<uint64_t> targets(Q);
  targets.push_back(m_sk);
  for (uint64_t q : targets) {
    push_reducer(sc, q);
    sc.push_back(product_mod(B, k, q));
  }
  for (uint64_t q : targets)
    for (uint64_t j = 0; j < k; ++j) sc.push_back(product_mod(B, j, q));
  push_twiddle(sc, nt::inverse_mod(product_mod(B, k, m_sk), m_sk), m_sk);
  return 0;
}

int bfv_product_on_device(int dev, const BfvPlan& pl, const BfvOutputs& out, const uint64_t* ct1, const uint64_t* ct2,
                          cudaStream_t s) {
  const uint64_t n = pl.n, l = pl.l, k = pl.k, M = l + k + 1, comp = l * n, poly = M * n;
  const uint64_t *ext_tab = nullptr, *scale_tab = nullptr;
  if (int rc = device_table(pl.ext_tab, dev, s, &ext_tab, "BEHZ tables")) return rc;
  if (int rc = device_table(pl.scale_tab, dev, s, &scale_tab, "BEHZ tables")) return rc;
  const bool square = ct1 == ct2;
  const uint64_t inputs = square ? 2 : 4;
  Scratch ws(s);
  uint64_t *ext = nullptr, *tensor = nullptr;
  if (int rc = ws.get(&ext, inputs * poly)) return rc;  // [a0, a1, (b0, b1)][m][n]
  if (int rc = ws.get(&tensor, 3 * poly)) return rc;    // [d0, d1, d2][m][n]
  cudaError_t e = launch_bfv_extend(ext, poly, ct1, comp, n, 2, l, k, ext_tab, s);
  if (e == cudaSuccess && !square) e = launch_bfv_extend(ext + 2 * poly, poly, ct2, comp, n, 2, l, k, ext_tab, s);
  if (e != cudaSuccess) return cuda_fail(e, "BfvMultiply: extension launch");
  std::vector<hexl_b200_ntt*> hs;  // one handle per limb of the polynomials back to back
  for (uint64_t p = 0; p < inputs; ++p) hs.insert(hs.end(), pl.h.data(), pl.h.data() + M);
  if (int rc = ntt_multi_on_device(true, dev, hs.data(), inputs * M, ext, ext, 1, 1, s)) return rc;
  for (uint64_t first = 0; first < M; first += kParamBlock) {
    const uint64_t cnt = std::min<uint64_t>(kParamBlock, M - first);
    DyadicModuli mods;
    for (uint64_t m = 0; m < cnt; ++m) mods.m[m] = dyadic_modulus(pl.mods[first + m]);
    e = launch_dyadic_multiply(tensor, ext, square ? ext : ext + 2 * poly, n, M, first, cnt, mods, s);
    if (e != cudaSuccess) return cuda_fail(e, "BfvMultiply: tensor launch");
  }
  hs.clear();
  for (uint64_t p = 0; p < 3; ++p) hs.insert(hs.end(), pl.h.data(), pl.h.data() + M);
  if (int rc = ntt_multi_on_device(false, dev, hs.data(), 3 * M, tensor, tensor, 1, 1, s)) return rc;
  e = launch_bfv_scale(out, tensor, poly, n, 3, l, k, scale_tab, s);
  return e == cudaSuccess ? 0 : cuda_fail(e, "BfvMultiply: scaling launch");
}

}  // namespace hexl_b200

extern "C" {

int hexl_b200_bfv_multiply(uint64_t* result, const uint64_t* ct1, const uint64_t* ct2, uint64_t n,
                           const uint64_t* moduli, uint64_t level_size, const uint64_t* base_b, uint64_t base_b_size,
                           uint64_t m_sk, uint64_t plain_modulus, uint64_t batch, void* stream) {
  const uint64_t l = level_size, k = base_b_size;
  if (int rc = bfv_check(result, ct1, ct2, n, moduli, l, base_b, k, m_sk, plain_modulus)) return rc;
  if (batch == 0) return 0;
  const uint64_t comp = l * n, in_words = 2 * comp, out_words = 3 * comp;
  const uint64_t in_total = batch * in_words, out_total = batch * out_words;
  REQUIRE(result + out_total <= ct1 || ct1 + in_total <= result, "result and ct1 must not overlap");
  REQUIRE(result + out_total <= ct2 || ct2 + in_total <= result, "result and ct2 must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, ct1, ct2}, &pi)) return rc;
  auto bound = [&](u64 i) { return moduli[i]; };
  if (int rc = check_limb_bounds(ct1, 2 * batch, l, n, bound, pi, "ct1", stream)) return rc;
  if (ct2 != ct1)
    if (int rc = check_limb_bounds(ct2, 2 * batch, l, n, bound, pi, "ct2", stream)) return rc;
  BfvPlan plan(l + k + 1);
  if (int rc = bfv_plan(&plan, n, moduli, l, base_b, k, m_sk, plain_modulus)) return rc;
  auto outputs = [&](uint64_t* r) { return BfvOutputs{{r, r + comp, r + 2 * comp}}; };
  // host pointers: both ciphertexts of a pair cross PCIe in once (one copy when squaring) and the product comes back
  // from the same slot
  if (pi.where == Where::Host) {
    const bool square = ct1 == ct2;
    return key_switch_host_batch(result, out_words, false, ct1, in_words, square ? in_words : 2 * in_words, nullptr, 0,
                                 batch,
                                 [&](int dev, uint64_t* d_res, uint64_t* d_in, const uint64_t* const* const*,
                                     cudaStream_t s) {
                                   return bfv_product_on_device(dev, plan, outputs(d_res), d_in,
                                                                square ? d_in : d_in + in_words, s);
                                 },
                                 nullptr, square ? nullptr : ct2);
  }
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = bfv_product_on_device(pi.device, plan, outputs(result + c * out_words), ct1 + c * in_words,
                                         ct2 + c * in_words, (cudaStream_t)stream))
        return rc;
    return 0;
  });
}

}  // extern "C"
