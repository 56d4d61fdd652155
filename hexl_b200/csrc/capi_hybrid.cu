// Hybrid key switching (OpenFHE's KeySwitchHYBRID): digits of up to 64 data moduli and up to 64 special primes, the
// mod-up and the mod-down by fast base conversion (rns.cu); the base conversion on its own; and the rotations with
// hybrid keys: hoisted, the diagonal-weighted sum of rotations under one mod-down (the linear transform) and its
// double-hoisted baby-step giant-step form; the ciphertext product, or a sum of such products, relinearized with
// hybrid keys, its rescale optionally merged into the mod-down; the inner sum of k rotations, a rotate-and-sum kept
// in the extended basis; and the BFV product relinearized with hybrid keys in coefficient form.
#include <cstdio>
#include <numeric>

#include "capi.h"

using namespace hexl_b200;

namespace hexl_b200 {

static uint64_t mul_mod128(uint64_t a, uint64_t b, uint64_t m) { return (uint64_t)((unsigned __int128)a * b % m); }

// floor(M/2) mod m for M the product of `count` odd moduli (M odd, so floor(M/2) = (M - 1) / 2) and m odd
static uint64_t half_product_mod(const uint64_t* moduli, uint64_t count, uint64_t m) {
  uint64_t r = 1 % m;
  for (uint64_t i = 0; i < count; ++i) r = mul_mod128(r, moduli[i] % m, m);
  return mul_mod128((r + m - 1) % m, (m + 1) / 2, m);  // (m + 1) / 2 = 2^-1 mod m
}

// Base conversion of `polys` polynomials from the moduli `from` (pairwise coprime, Q their product) into the moduli
// `to`, device pointers on the current device, asynchronous on s; strides as launch_base_conv.  One launch per block of
// base_conv_targets(from_count) targets; the constants are computed here, per call.  round (the mod-down by
// P = Q): x_i + [floor(P/2)]_{q_i} on input and - [floor(P/2)]_t on output, so that an input X in [0, P) comes out as
// the centred lift of X + floor(P/2) minus floor(P/2), plus e P with 0 <= e < from_count.  plain_modulus = tau != 0
// (BGV's mod-down, round ignored): the t-corrected conversion of launch_base_conv_t instead, one launch per block of
// base_conv_t_targets(from_count) targets, which yields delta = X mod P with delta = 0 mod tau.
int base_convert_on_device(uint64_t* result, uint64_t res_limb, uint64_t res_poly, const uint64_t* operand,
                           uint64_t op_limb, uint64_t op_poly, uint64_t n, uint64_t polys, const uint64_t* from,
                           uint64_t from_count, const uint64_t* to, uint64_t to_count, bool round, cudaStream_t s,
                           uint64_t plain_modulus) {
  const uint64_t F = from_count, block = base_conv_targets(F);
  std::vector<uint64_t> prefix(F + 1), suffix(F + 1);
  BaseConvTable tab;
  // [Q/q_i]_t for every source i into row[0..F)
  auto cofactors = [&](uint64_t t, uint64_t* row) {
    prefix[0] = suffix[F] = 1 % t;
    for (uint64_t i = 0; i < F; ++i) prefix[i + 1] = mul_mod128(prefix[i], from[i] % t, t);
    for (uint64_t i = F; i-- > 0;) suffix[i] = mul_mod128(suffix[i + 1], from[i] % t, t);
    for (uint64_t i = 0; i < F; ++i) row[i] = mul_mod128(prefix[i], suffix[i + 1], t);
  };
  // t, floor(2^64 / t), 2^64 mod t and its Shoup factor into row[0..4)
  auto reducer = [](uint64_t t, uint64_t* row) {
    const uint64_t mu = nt::multiply_factor(1, 64, t);
    const Twiddle R = make_twiddle(mu * (0 - t) % t, t);
    row[0] = t;
    row[1] = mu;
    row[2] = R.w;
    row[3] = R.wp;
  };
  if (plain_modulus) {
    const uint64_t tau = plain_modulus, tblock = base_conv_t_targets(F);
    for (uint64_t i = 0; i < F; ++i) {
      const uint64_t q = from[i];
      uint64_t rest = 1 % q;
      for (uint64_t j = 0; j < F; ++j)
        if (j != i) rest = mul_mod128(rest, from[j] % q, q);
      const Twiddle inv = make_twiddle(nt::inverse_mod(rest, q), q);
      tab.w[3 * i] = q;
      tab.w[3 * i + 1] = inv.w;
      tab.w[3 * i + 2] = inv.wp;
    }
    uint64_t* trow = tab.w + 3 * F;
    reducer(tau, trow);
    uint64_t P_tau = 1 % tau;
    for (uint64_t i = 0; i < F; ++i) P_tau = mul_mod128(P_tau, from[i] % tau, tau);
    const Twiddle neg_inv = make_twiddle((tau - nt::inverse_mod(P_tau, tau)) % tau, tau);
    trow[4] = neg_inv.w;
    trow[5] = neg_inv.wp;
    cofactors(tau, trow + 6);
    for (uint64_t e0 = 0; e0 < to_count; e0 += tblock) {
      const uint64_t cnt = std::min(tblock, to_count - e0);
      uint64_t* targets = trow + 6 + F;
      uint64_t* matrix = targets + 6 * cnt;
      for (uint64_t e = 0; e < cnt; ++e) {
        const uint64_t t = to[e0 + e];
        reducer(t, targets + 6 * e);
        uint64_t P = 1 % t;
        for (uint64_t i = 0; i < F; ++i) P = mul_mod128(P, from[i] % t, t);
        const Twiddle Pt = make_twiddle(P, t);
        targets[6 * e + 4] = Pt.w;
        targets[6 * e + 5] = Pt.wp;
        cofactors(t, matrix + e * F);
      }
      const cudaError_t e = launch_base_conv_t(result + e0 * res_limb, res_limb, res_poly, operand, op_limb, op_poly,
                                               n, polys, F, cnt, tab, s);
      if (e != cudaSuccess) return cuda_fail(e, "t-corrected base conversion launch");
    }
    return 0;
  }
  // (Q/q_i)^-1 mod q_i from prefix and suffix products under q_i
  for (uint64_t i = 0; i < F; ++i) {
    const uint64_t q = from[i];
    uint64_t rest = 1 % q;
    for (uint64_t j = 0; j < F; ++j)
      if (j != i) rest = mul_mod128(rest, from[j] % q, q);
    const Twiddle inv = make_twiddle(nt::inverse_mod(rest, q), q);
    tab.w[4 * i] = q;
    tab.w[4 * i + 1] = inv.w;
    tab.w[4 * i + 2] = inv.wp;
    tab.w[4 * i + 3] = round ? half_product_mod(from, F, q) : 0;
  }
  for (uint64_t e0 = 0; e0 < to_count; e0 += block) {
    const uint64_t cnt = std::min(block, to_count - e0);
    uint64_t* targets = tab.w + 4 * F;
    uint64_t* matrix = targets + 5 * cnt;
    for (uint64_t e = 0; e < cnt; ++e) {
      const uint64_t t = to[e0 + e];
      reducer(t, targets + 5 * e);
      targets[5 * e + 4] = round ? half_product_mod(from, F, t) : 0;
      cofactors(t, matrix + e * F);
    }
    const cudaError_t e = launch_base_conv(result + e0 * res_limb, res_limb, res_poly, operand, op_limb, op_poly, n,
                                           polys, F, cnt, tab, s);
    if (e != cudaSuccess) return cuda_fail(e, "base conversion launch");
  }
  return 0;
}

// The mod-up of one target (level limbs in NTT form, device memory), steps 1 and 2 of the hybrid switch
// (include/hexl_b200.h has the definitions).  h holds the transforms of the extended basis
// B = {q_0..q_{l-1}, p_0..p_{K-1}} in that order and bmods their moduli.  The target's limbs go back to coefficients
// once; then, per round of moduli of B, every digit is converted into each modulus of the round and lazily
// transformed into ops ([e][d][n], D x n words between moduli), and mac(b0, cnt, ops, slots) multiplies them with the
// keys: moduli [b0, b0 + cnt) of B, slots[e] the key slot of modulus b0 + e.  Scratch comes from ws.  mul (nullptr:
// none; laid out like target) makes the target the point-wise product target (.) mul, multiplied in the first inverse
// transform's load, so the product is never written.  coef: the target is already in coefficient form (canonical);
// its limbs are read directly and step 1 is skipped.
template <class Mac>
static int hybrid_mod_up(int dev, const uint64_t* target, uint64_t n, uint64_t level, uint64_t q_size,
                         uint64_t p_size, uint64_t alpha, const CachedNtts& h, const uint64_t* bmods, Scratch& ws,
                         Mac&& mac, cudaStream_t s, const uint64_t* mul = nullptr, bool coef = false) {
  const uint64_t D = (level + alpha - 1) / alpha, nb = level + p_size;
  // moduli handled per round of the mod-up: bounded by the parameter block and by ~256 MiB of scratch
  const uint64_t per_mod = D * n;
  uint64_t ichunk = std::max<uint64_t>(1, (256ull << 20) / (per_mod * 8));
  ichunk = std::min<uint64_t>({ichunk, nb, (uint64_t)kParamBlock});
  uint64_t *t_coef = nullptr, *ops = nullptr;
  if (!coef)
    if (int rc = ws.get(&t_coef, level * n)) return rc;
  if (int rc = ws.get(&ops, ichunk * per_mod)) return rc;  // [e][d][n]
  // 1. the target's limbs back to coefficients, canonical
  if (!coef)
    if (int rc = ntt_multi_on_device(false, dev, h.data(), level, t_coef, target, 1, 1, s, nullptr, false, mul))
      return rc;
  const uint64_t* a = coef ? target : t_coef;
  // 2. mod-up: every digit converted into each modulus of the round, lazily transformed, multiplied with the keys.
  //    (A digit's own limbs are converted and transformed again like the others: NTT(INTT(t)) = t.)
  for (uint64_t b0 = 0; b0 < nb; b0 += ichunk) {
    const uint64_t cnt = std::min(ichunk, nb - b0);
    for (uint64_t d = 0; d < D; ++d) {
      const uint64_t lo = d * alpha, width = std::min(alpha, level - lo);
      if (int rc = base_convert_on_device(ops + d * n, per_mod, 0, a + lo * n, n, 0, n, 1, bmods + lo, width,
                                          bmods + b0, cnt, false, s))
        return rc;
    }
    if (int rc = ntt_multi_on_device(true, dev, h.data() + b0, cnt, ops, ops, 4, D, s)) return rc;
    uint64_t slots[kParamBlock];
    for (uint64_t e = 0; e < cnt; ++e) slots[e] = b0 + e < level ? b0 + e : q_size + (b0 + e - level);
    if (int rc = mac(b0, cnt, (const uint64_t*)ops, (const uint64_t*)slots)) return rc;
  }
  return 0;
}

// Step 3, the mod-down by P, of one switch's products prod ([b][k][n] over the moduli of B, kcc components): the
// special limbs back to coefficients in place, rounded and converted into each data modulus, transformed, and
// (prod - that) * P^-1 accumulated into result (kcc x level x n), or stored when !accumulate.  tmp holds
// min(level, 64) x kcc x n words.  P is the product of the p_size moduli of B after the first `level`: called with
// level - 1 and p_size + 1 it divides by q_{level-1} P as well, the mod-down merged with the rescale.  coef: result is
// in coefficient form; the products' data limbs go back to coefficients in place instead of the rounded correction
// being transformed forward, and the finish, point-wise, is the same: INTT((prod - NTT(c)) P^-1) = (INTT(prod) - c) P^-1.
// plain_modulus = tau != 0 (BGV): the t-corrected conversion in place of the rounded one, so that c = 0 mod tau.
static int hybrid_mod_down(int dev, uint64_t* result, uint64_t* prod, uint64_t* tmp, uint64_t n, uint64_t level,
                           uint64_t p_size, uint64_t kcc, const CachedNtts& h, const uint64_t* bmods, bool accumulate,
                           cudaStream_t s, bool coef = false, uint64_t plain_modulus = 0) {
  uint64_t* special = prod + level * kcc * n;  // [j][k][n]
  if (int rc = ntt_multi_on_device(false, dev, h.data() + level, p_size, special, special, 1, kcc, s)) return rc;
  for (uint64_t i0 = 0; i0 < level; i0 += kParamBlock) {
    const uint64_t cnt = std::min<uint64_t>(kParamBlock, level - i0);
    if (int rc = base_convert_on_device(tmp, kcc * n, n, special, kcc * n, n, n, kcc, bmods + level, p_size,
                                        bmods + i0, cnt, true, s, plain_modulus))
      return rc;
    if (coef) {
      uint64_t* data = prod + i0 * kcc * n;
      if (int rc = ntt_multi_on_device(false, dev, h.data() + i0, cnt, data, data, 1, kcc, s)) return rc;
    } else if (int rc = ntt_multi_on_device(true, dev, h.data() + i0, cnt, tmp, tmp, 4, kcc, s)) {
      return rc;
    }
    KsModuli fin;
    for (uint64_t e = 0; e < cnt; ++e) {
      const uint64_t q = bmods[i0 + e];
      uint64_t P = 1 % q;
      for (uint64_t j = 0; j < p_size; ++j) P = mul_mod128(P, bmods[level + j] % q, q);
      const Twiddle f = make_twiddle(nt::inverse_mod(P, q), q);
      fin.m[e] = KsModulus{q, nt::multiply_factor(1, 64, q), f.w, f.wp, 0};
    }
    const cudaError_t e =
        launch_ks_finish(result, prod + i0 * kcc * n, tmp, n, kcc, level, i0, cnt, fin, false, accumulate, s);
    if (e != cudaSuccess) return cuda_fail(e, "hybrid mod-down: finish launch");
  }
  return 0;
}

// `elts` hybrid key switches of one target, every pointer a device pointer on the current device, asynchronous on s:
// the mod-up once, then for switch r the multiply-accumulate with keys[r] (keys[r][d]: digit d's key buffer,
// kcc x (q_size + K) x n words) and one mod-down accumulated into results[r].  galois_elts[r] (nullptr: none) makes
// switch r read the transformed digits permuted by pi_g, as key_switch_elts_on_device does for the hoisted
// rotations.  Scratch: one round of transformed digits plus elts x (level + K) x kcc x n words of products.
// plain_modulus != 0: the mod-downs are BGV's t-corrected ones (hybrid_mod_down).
static int key_switch_hybrid_elts_on_device(int dev, uint64_t* const* results, const uint64_t* target, uint64_t n,
                                            uint64_t level, uint64_t q_size, uint64_t p_size, uint64_t alpha,
                                            uint64_t kcc, const CachedNtts& h, const uint64_t* bmods,
                                            const uint64_t* const* const* keys, const uint64_t* galois_elts,
                                            uint64_t elts, cudaStream_t s, uint64_t plain_modulus = 0) {
  const uint64_t D = (level + alpha - 1) / alpha, nb = level + p_size, kms = q_size + p_size;
  Scratch ws(s);
  uint64_t *prod = nullptr, *tmp = nullptr;
  if (int rc = ws.get(&prod, elts * nb * kcc * n)) return rc;                               // [r][b][k][n]
  if (int rc = ws.get(&tmp, std::min<uint64_t>(level, kParamBlock) * kcc * n)) return rc;  // [i][k][n], one block
  if (int rc = hybrid_mod_up(dev, target, n, level, q_size, p_size, alpha, h, bmods, ws,
                             [&](uint64_t b0, uint64_t cnt, const uint64_t* ops, const uint64_t* slots) {
                               return ks_mac_products(h.data() + b0, slots, cnt, kms, ops, D, n, kcc,
                                                      prod + b0 * kcc * n, nb * kcc * n, keys, galois_elts, elts, s);
                             },
                             s))
    return rc;
  for (uint64_t r = 0; r < elts; ++r)
    if (int rc =
            hybrid_mod_down(dev, results[r], prod + r * nb * kcc * n, tmp, n, level, p_size, kcc, h, bmods, true, s,
                            false, plain_modulus))
      return rc;
  return 0;  // asynchronous on s; ~Scratch returns the buffers to the pool in stream order
}

static int key_switch_hybrid_on_device(int dev, uint64_t* result, const uint64_t* target, uint64_t n, uint64_t level,
                                       uint64_t q_size, uint64_t p_size, uint64_t alpha, uint64_t kcc,
                                       const CachedNtts& h, const uint64_t* bmods, const uint64_t* const* keys,
                                       cudaStream_t s, uint64_t plain_modulus) {
  return key_switch_hybrid_elts_on_device(dev, &result, target, n, level, q_size, p_size, alpha, kcc, h, bmods, &keys,
                                          nullptr, 1, s, plain_modulus);
}

// The hoisted hybrid rotations of one ciphertext ct (two components of level limbs, NTT form, device memory) by
// `elts` elements: per element one automorphism launch of c0 straight into its output and a memset of the output's
// c1, then the shared switch of c1 with every element's keys, read through pi_g.
static int hybrid_hoisted_on_device(int dev, uint64_t* out, const uint64_t* ct, uint64_t n, uint64_t level,
                                    uint64_t q_size, uint64_t p_size, uint64_t alpha, const CachedNtts& h,
                                    const uint64_t* bmods, const uint64_t* const* const* keys,
                                    const uint64_t* galois_elts, uint64_t elts, cudaStream_t s,
                                    uint64_t plain_modulus) {
  const uint64_t comp = level * n;
  std::vector<uint64_t*> results(elts);
  for (uint64_t r = 0; r < elts; ++r) {
    results[r] = out + r * 2 * comp;
    const cudaError_t e = launch_galois_ntt(results[r], ct, floor_log2(n), level, galois_elts[r], s);
    if (e != cudaSuccess) return cuda_fail(e, "ApplyGaloisKeySwitchHybridHoisted: automorphism launch");
    CU(cudaMemsetAsync(results[r] + comp, 0, comp * sizeof(uint64_t), s));
  }
  return key_switch_hybrid_elts_on_device(dev, results.data(), ct + comp, n, level, q_size, p_size, alpha, 2, h, bmods,
                                          keys, galois_elts, elts, s, plain_modulus);
}

// The hybrid linear transform of one ciphertext ct (as above) into result (2 x level x n words, device memory):
// keys[r] is element r's key copy, or nullptr for an identity term; diag holds elts diagonals of (level + K) x n
// words.  First the weighted permuted sum of ct's limbs is stored into result (one launch per chunk of 64 elements
// and block of 64 data moduli); then, when any element has keys, the shared mod-up, the weighted multiply-accumulate
// of every keyed element into one accumulator over B (one launch per round, chunk of (element, digit) pairs and
// chunk of digits) and one mod-down of the accumulator into result.
static int linear_transform_hybrid_on_device(int dev, uint64_t* result, const uint64_t* ct, const uint64_t* diag,
                                             uint64_t n, uint64_t level, uint64_t q_size, uint64_t p_size,
                                             uint64_t alpha, const CachedNtts& h, const uint64_t* bmods,
                                             const uint64_t* const* const* keys, const uint64_t* galois_elts,
                                             uint64_t elts, cudaStream_t s) {
  const uint64_t D = (level + alpha - 1) / alpha, nb = level + p_size, kms = q_size + p_size, dstride = nb * n;
  for (uint64_t i0 = 0; i0 < level; i0 += kParamBlock) {
    const uint64_t cnt = std::min<uint64_t>(kParamBlock, level - i0);
    const KsModuli mods = ks_mac_moduli(bmods + i0, nullptr, cnt);
    for (uint64_t r0 = 0; r0 < elts; r0 += kParamBlock) {
      const uint64_t ecnt = std::min<uint64_t>(kParamBlock, elts - r0);
      PermutedSumElts ps{};
      for (uint64_t r = 0; r < ecnt; ++r) {
        ps.diag[r] = diag + (r0 + r) * dstride + i0 * n;
        ps.elt[r] = (unsigned)galois_elts[r0 + r];
        if (!keys[r0 + r]) ps.identity |= 1ull << r;
      }
      const cudaError_t e = launch_ks_permuted_sum(result, ct, n, level, i0, cnt, ps, ecnt, mods, r0 != 0, s);
      if (e != cudaSuccess) return cuda_fail(e, "LinearTransformHybrid: permuted sum launch");
    }
  }
  std::vector<uint64_t> keyed;
  for (uint64_t r = 0; r < elts; ++r)
    if (keys[r]) keyed.push_back(r);
  if (keyed.empty()) return 0;
  Scratch ws(s);
  uint64_t *acc = nullptr, *tmp = nullptr;
  if (int rc = ws.get(&acc, nb * 2 * n)) return rc;                                       // [b][k][n]
  if (int rc = ws.get(&tmp, std::min<uint64_t>(level, kParamBlock) * 2 * n)) return rc;  // [i][k][n], one block
  auto mac = [&](uint64_t b0, uint64_t cnt, const uint64_t* ops, const uint64_t* slots) -> int {
    const KsModuli mods = ks_mac_moduli(bmods + b0, slots, cnt);
    // (element, digit) pairs per launch: a digit chunk within the 128-bit bound, as many elements as fill the block
    const uint64_t jc = std::min(ks_mac_digits_per_launch(mods, cnt), D);
    const uint64_t per = std::max<uint64_t>(1, kParamBlock / jc);
    bool accumulate = false;
    for (uint64_t j0 = 0; j0 < D; j0 += jc) {
      const uint64_t jcnt = std::min(jc, D - j0);
      for (uint64_t k0 = 0; k0 < keyed.size(); k0 += per) {
        const uint64_t ecnt = std::min<uint64_t>(per, keyed.size() - k0);
        WeightedMacElts we{};
        for (uint64_t e = 0; e < ecnt; ++e) {
          const uint64_t r = keyed[k0 + e];
          for (uint64_t j = 0; j < jcnt; ++j) we.key[e * jcnt + j] = keys[r][j0 + j];
          we.diag[e] = diag + r * dstride + b0 * n;
          we.elt[e] = (unsigned)galois_elts[r];
        }
        const cudaError_t e = launch_ks_weighted_mac(acc + b0 * 2 * n, ops + j0 * n, D * n, we, n, jcnt, ecnt, kms,
                                                     cnt, mods, accumulate, s);
        if (e != cudaSuccess) return cuda_fail(e, "LinearTransformHybrid: multiply-accumulate launch");
        accumulate = true;
      }
    }
    return 0;
  };
  if (int rc = hybrid_mod_up(dev, ct + level * n, n, level, q_size, p_size, alpha, h, bmods, ws, mac, s)) return rc;
  return hybrid_mod_down(dev, result, acc, tmp, n, level, p_size, 2, h, bmods, true, s);
}

// The baby-step giant-step transform of one ciphertext ct (as above) into result (2 x (level - rescale) x n words):
// diag[j * n1 + i] is the (giant j, baby i) diagonal on this device ((level + K) x n words) or nullptr when absent;
// baby_keys[i] / giant_keys[j] a handle's copy, or nullptr for an identity term.  X (data limbs, in result, or in
// scratch with the rescale) and Y (two components over B) stay apart; include/hexl_b200.h has the definitions.
//   1. when some keyed baby has a diagonal: one mod-up of c1, its products with every such baby's keys stored
//      ([i][b][k][n]);
//   2. per giant step with a present baby: the sum launches (per block of 64 moduli of B, only the data moduli when
//      the row has no keyed baby, and per chunk of 64 present babies);
//   3. per keyed giant step: the mod-down of y_1 into x_1 (kcc = 1; none without a keyed baby), then the mod-up of
//      c1' = x_1 with its multiply-accumulate reading pi_h and adding into Y;
//   4. one mod-down of Y into result (none while Y is empty), or with the rescale, [P] X folded into Y's data limbs by
//      the last sum launch and the mod-down by q_{level-1} P that stores.
static int bsgs_hybrid_on_device(int dev, uint64_t* result, const uint64_t* ct, const uint64_t* const* diag,
                                 uint64_t n, uint64_t level, uint64_t q_size, uint64_t p_size, uint64_t alpha,
                                 bool rescale, const CachedNtts& h, const uint64_t* bmods,
                                 const uint64_t* const* const* baby_keys, const uint64_t* baby_elts, uint64_t n1,
                                 const uint64_t* const* const* giant_keys, const uint64_t* giant_elts, uint64_t n2,
                                 cudaStream_t s) {
  const uint64_t D = (level + alpha - 1) / alpha, nb = level + p_size, kms = q_size + p_size, comp = level * n;
  const uint64_t stride = nb * 2 * n;  // one baby's stored products
  // the keyed babies with a diagonal, in baby order: their index among the stored products
  std::vector<uint64_t> stored(n1, kBsgsNoProducts), used_elts;
  std::vector<const uint64_t* const*> used_keys;
  for (uint64_t i = 0; i < n1; ++i) {
    if (!baby_keys[i]) continue;
    for (uint64_t j = 0; j < n2; ++j)
      if (diag[j * n1 + i]) {
        stored[i] = used_keys.size();
        used_keys.push_back(baby_keys[i]);
        used_elts.push_back(baby_elts[i]);
        break;
      }
  }
  uint64_t last_row = n2;  // the last giant step with a present baby: its sums fold X into Y under the rescale
  for (uint64_t j = 0; j < n2; ++j)
    for (uint64_t i = 0; i < n1; ++i)
      if (diag[j * n1 + i]) last_row = j;
  Scratch ws(s);
  uint64_t *prods = nullptr, *y = nullptr, *x = result, *x1 = nullptr, *y1 = nullptr, *tmp = nullptr;
  if (!used_keys.empty())
    if (int rc = ws.get(&prods, used_keys.size() * stride)) return rc;  // [i][b][k][n]
  if (int rc = ws.get(&y, stride)) return rc;                           // [b][k][n]
  if (rescale)
    if (int rc = ws.get(&x, 2 * comp)) return rc;  // [k][i][n]
  if (int rc = ws.get(&x1, comp)) return rc;       // [i][n]
  if (int rc = ws.get(&y1, nb * n)) return rc;     // [b][n]
  if (int rc = ws.get(&tmp, std::min<uint64_t>(level, kParamBlock) * 2 * n)) return rc;  // [i][k][n], one block
  CU(cudaMemsetAsync(y, 0, stride * sizeof(uint64_t), s));
  CU(cudaMemsetAsync(x, 0, 2 * comp * sizeof(uint64_t), s));
  // 1. the baby products
  if (!used_keys.empty()) {
    Scratch wu(s);
    if (int rc = hybrid_mod_up(dev, ct + comp, n, level, q_size, p_size, alpha, h, bmods, wu,
                               [&](uint64_t b0, uint64_t cnt, const uint64_t* ops, const uint64_t* slots) {
                                 return ks_mac_products(h.data() + b0, slots, cnt, kms, ops, D, n, 2,
                                                        prods + b0 * 2 * n, stride, used_keys.data(),
                                                        used_elts.data(), used_keys.size(), s);
                               },
                               s))
      return rc;
  }
  bool y_used = false;
  for (uint64_t j = 0; j < n2; ++j) {
    std::vector<uint64_t> present;
    bool keyed_baby = false;
    for (uint64_t i = 0; i < n1; ++i)
      if (diag[j * n1 + i]) {
        present.push_back(i);
        keyed_baby = keyed_baby || baby_keys[i];
      }
    if (present.empty()) continue;  // an absent row costs nothing
    const bool keyed_giant = giant_keys[j] != nullptr, fold = rescale && j == last_row;
    // 2. the giant step's sums; without a keyed baby the special limbs would only add zeros
    const uint64_t span = keyed_baby ? nb : level;
    for (uint64_t b0 = 0; b0 < span; b0 += kParamBlock) {
      const uint64_t cnt = std::min<uint64_t>(kParamBlock, span - b0);
      KsModuli mods = ks_mac_moduli(bmods + b0, nullptr, cnt);
      if (fold)
        for (uint64_t e = 0; e < cnt && b0 + e < level; ++e) {
          const uint64_t q = bmods[b0 + e];
          uint64_t P = 1 % q;
          for (uint64_t k = 0; k < p_size; ++k) P = mul_mod128(P, bmods[level + k] % q, q);
          mods.m[e].c = P;
        }
      for (uint64_t r0 = 0; r0 < present.size(); r0 += kParamBlock) {
        const uint64_t rcnt = std::min<uint64_t>(kParamBlock, present.size() - r0);
        BsgsSumTerms terms{};
        for (uint64_t r = 0; r < rcnt; ++r) {
          const uint64_t i = present[r0 + r];
          terms.diag[r] = diag[j * n1 + i] + b0 * n;
          terms.elt[r] = (unsigned)baby_elts[i];
          terms.prod[r] = (unsigned)stored[i];
        }
        int mode = keyed_giant ? kBsgsKeyedGiant : 0;
        if (r0 == 0) mode |= kBsgsStore1;
        if (fold && r0 + rcnt == present.size()) mode |= kBsgsFold;
        const cudaError_t e = launch_ks_bsgs_sum(x, y, x1, y1, ct, prods, stride, n, level, b0, cnt, giant_elts[j],
                                                 terms, rcnt, mods, mode, s);
        if (e != cudaSuccess) return cuda_fail(e, "LinearTransformHybridBSGS: sum launch");
      }
    }
    y_used = y_used || keyed_baby || keyed_giant;
    if (!keyed_giant) continue;
    // 3. the giant step's own switch: c1' = x_1 + ModDown_P(y_1), then its mod-up multiplied with the giant's keys
    //    through pi_h and added into Y
    if (keyed_baby)
      if (int rc = hybrid_mod_down(dev, x1, y1, tmp, n, level, p_size, 1, h, bmods, true, s)) return rc;
    Scratch wu(s);
    const uint64_t h_elt = giant_elts[j];
    if (int rc = hybrid_mod_up(dev, x1, n, level, q_size, p_size, alpha, h, bmods, wu,
                               [&](uint64_t b0, uint64_t cnt, const uint64_t* ops, const uint64_t* slots) {
                                 return ks_mac_products(h.data() + b0, slots, cnt, kms, ops, D, n, 2, y + b0 * 2 * n,
                                                        stride, &giant_keys[j], &h_elt, 1, s, true);
                               },
                               s))
      return rc;
  }
  // 4. the final mod-down
  if (rescale) return hybrid_mod_down(dev, result, y, tmp, n, level - 1, p_size + 1, 2, h, bmods, false, s);
  if (!y_used) return 0;
  return hybrid_mod_down(dev, result, y, tmp, n, level, p_size, 2, h, bmods, true, s);
}

// The product of two ciphertexts ct1 = (a0, a1) and ct2 = (b0, b1) (each two components of level limbs, NTT form,
// device memory), relinearized with keys (digit d's key buffer keys[d]) and stored into result (2 x (level - rescale)
// limbs): the mod-up of a1 (.) b1, multiplied in the mod-up's first inverse transform; per round, the relinearization
// multiply-accumulate, whose storing launch adds [P] (a0 b0, a0 b1 + a1 b0) on the data moduli; and one mod-down,
// by P or, with rescale, by q_{level-1} P (q_{level-1} is the limb of B right before the special limbs).  Scratch: one
// round of transformed digits plus (level + K) x 2 x n words of products.  sum (nullptr: none) holds the tensor
// (d0, d1, t) already formed ([3][level][n], canonical): the mod-up then reads t, the storing launches read d0 and d1,
// and ct1 and ct2 are not read.  plain_modulus != 0 (BGV): the mod-down is t-corrected, and with rescale it is the
// merged modulus switch by q_{level-1} P.
static int multiply_relinearize_hybrid_on_device(int dev, uint64_t* result, const uint64_t* ct1, const uint64_t* ct2,
                                                 uint64_t n, uint64_t level, uint64_t q_size, uint64_t p_size,
                                                 uint64_t alpha, bool rescale, const CachedNtts& h,
                                                 const uint64_t* bmods, const uint64_t* const* keys, cudaStream_t s,
                                                 const uint64_t* sum = nullptr, uint64_t plain_modulus = 0) {
  const uint64_t D = (level + alpha - 1) / alpha, nb = level + p_size, kms = q_size + p_size, comp = level * n;
  Scratch ws(s);
  uint64_t *prod = nullptr, *tmp = nullptr;
  if (int rc = ws.get(&prod, nb * 2 * n)) return rc;                                       // [b][k][n]
  if (int rc = ws.get(&tmp, std::min<uint64_t>(level, kParamBlock) * 2 * n)) return rc;  // [i][k][n], one block
  auto mac = [&](uint64_t b0, uint64_t cnt, const uint64_t* ops, const uint64_t* slots) -> int {
    const KsModuli mods = ks_mac_moduli(bmods + b0, slots, cnt);
    RelinTensor tensor{};
    if (sum) {
      tensor.sum = sum + b0 * n;
    } else {
      tensor.ct1 = ct1 + b0 * n;
      tensor.ct2 = ct2 + b0 * n;
    }
    tensor.comp = comp;
    tensor.data = b0 < level ? std::min(cnt, level - b0) : 0;
    for (uint64_t e = 0; e < tensor.data; ++e) {
      const uint64_t q = bmods[b0 + e];
      uint64_t P = 1 % q;
      for (uint64_t j = 0; j < p_size; ++j) P = mul_mod128(P, bmods[level + j] % q, q);
      tensor.p[e] = P;
    }
    const uint64_t jc = std::min(ks_mac_digits_per_launch(mods, cnt), D);
    for (uint64_t j0 = 0; j0 < D; j0 += jc) {  // key pointers ride in the kernel parameters
      const uint64_t jcnt = std::min(jc, D - j0);
      KeyPointers kp;
      for (uint64_t j = 0; j < jcnt; ++j) kp.p[j] = keys[j0 + j];
      const cudaError_t e = launch_ks_relin_mac(prod + b0 * 2 * n, ops + j0 * n, D * n, kp, n, jcnt, kms, cnt, mods,
                                                tensor, j0 != 0, s);
      if (e != cudaSuccess) return cuda_fail(e, "MultiplyRelinearizeHybrid: multiply-accumulate launch");
    }
    return 0;
  };
  const int up = sum ? hybrid_mod_up(dev, sum + 2 * comp, n, level, q_size, p_size, alpha, h, bmods, ws, mac, s)
                     : hybrid_mod_up(dev, ct1 + comp, n, level, q_size, p_size, alpha, h, bmods, ws, mac, s, ct2 + comp);
  if (up) return up;
  if (plain_modulus)  // BGV: the t-corrected mod-down by P, or by q_{level-1} P (the merged modulus switch)
    return hybrid_mod_down(dev, result, prod, tmp, n, level - rescale, p_size + rescale, 2, h, bmods, false, s, false,
                           plain_modulus);
  if (rescale) return hybrid_mod_down(dev, result, prod, tmp, n, level - 1, p_size + 1, 2, h, bmods, false, s);
  return hybrid_mod_down(dev, result, prod, tmp, n, level, p_size, 2, h, bmods, false, s);
}

// The sum over `pairs` pairs of ciphertexts (ct1[r], ct2[r], laid out as above) of their products, relinearized once
// into result.  One pair is multiply_relinearize_hybrid_on_device.  Otherwise the tensor terms of every pair are summed
// into scratch (d0, d1, t) ([3][level][n]) by one launch per block of 64 data limbs and chunk of kRelinSumPairs pairs,
// and the single relinearization reads the sums: the mod-up of t, the multiply-accumulate adding [P] (d0, d1) and one
// mod-down.  Scratch: 3 x level x n words, plus what the single product takes.
static int multiply_relinearize_sum_hybrid_on_device(int dev, uint64_t* result, const uint64_t* const* ct1,
                                                     const uint64_t* const* ct2, uint64_t pairs, uint64_t n,
                                                     uint64_t level, uint64_t q_size, uint64_t p_size, uint64_t alpha,
                                                     bool rescale, const CachedNtts& h, const uint64_t* bmods,
                                                     const uint64_t* const* keys, cudaStream_t s) {
  if (pairs == 1)
    return multiply_relinearize_hybrid_on_device(dev, result, ct1[0], ct2[0], n, level, q_size, p_size, alpha, rescale,
                                                 h, bmods, keys, s);
  Scratch ws(s);
  uint64_t* sum = nullptr;
  if (int rc = ws.get(&sum, 3 * level * n)) return rc;  // [d0, d1, t][i][n]
  for (uint64_t i0 = 0; i0 < level; i0 += kParamBlock) {
    const uint64_t cnt = std::min<uint64_t>(kParamBlock, level - i0);
    const KsModuli mods = ks_mac_moduli(bmods + i0, nullptr, cnt);
    for (uint64_t r0 = 0; r0 < pairs; r0 += kRelinSumPairs) {
      const uint64_t rcnt = std::min<uint64_t>(kRelinSumPairs, pairs - r0);
      RelinSumPairs chunk{};
      for (uint64_t r = 0; r < rcnt; ++r) {
        chunk.ct1[r] = ct1[r0 + r];
        chunk.ct2[r] = ct2[r0 + r];
      }
      const cudaError_t e = launch_relin_tensor_sum(sum, n, level, i0, cnt, chunk, rcnt, mods, r0 != 0, s);
      if (e != cudaSuccess) return cuda_fail(e, "MultiplyRelinearizeSumHybrid: tensor sum launch");
    }
  }
  return multiply_relinearize_hybrid_on_device(dev, result, nullptr, nullptr, n, level, q_size, p_size, alpha, rescale,
                                               h, bmods, keys, s, sum);
}

// The BFV product of one pair (ct1, ct2: two components of level limbs, coefficient form, device memory), relinearized
// with keys (digit d's key buffer keys[d]) and stored into result (2 x level x n words, coefficient form): the BEHZ chain
// of hexl_b200_bfv_multiply stores d0 and d1 into result and d2 into scratch; the mod-up reads d2's limbs as they are;
// per round, the multiply-accumulate stores the products; the mod-down brings the products' data limbs back to
// coefficients and adds (prod - c) P^-1 into (d0, d1).  Scratch: that of hexl_b200_bfv_multiply, l x n words of d2, one
// round of converted digits and (level + K) x 2 x n words of products.
static int bfv_multiply_relinearize_on_device(int dev, uint64_t* result, const uint64_t* ct1, const uint64_t* ct2,
                                              const BfvPlan& plan, uint64_t n, uint64_t level, uint64_t q_size,
                                              uint64_t p_size, uint64_t alpha, const CachedNtts& h,
                                              const uint64_t* bmods, const uint64_t* const* keys, cudaStream_t s) {
  const uint64_t D = (level + alpha - 1) / alpha, nb = level + p_size, kms = q_size + p_size, comp = level * n;
  Scratch ws(s);
  uint64_t *d2 = nullptr, *prod = nullptr, *tmp = nullptr;
  if (int rc = ws.get(&d2, comp)) return rc;
  if (int rc = ws.get(&prod, nb * 2 * n)) return rc;                                       // [b][k][n]
  if (int rc = ws.get(&tmp, std::min<uint64_t>(level, kParamBlock) * 2 * n)) return rc;  // [i][k][n], one block
  if (int rc = bfv_product_on_device(dev, plan, BfvOutputs{{result, result + comp, d2}}, ct1, ct2, s)) return rc;
  if (int rc = hybrid_mod_up(dev, d2, n, level, q_size, p_size, alpha, h, bmods, ws,
                             [&](uint64_t b0, uint64_t cnt, const uint64_t* ops, const uint64_t* slots) {
                               return ks_mac_products(h.data() + b0, slots, cnt, kms, ops, D, n, 2,
                                                      prod + b0 * 2 * n, nb * 2 * n, &keys, nullptr, 1, s);
                             },
                             s, nullptr, true))
    return rc;
  return hybrid_mod_down(dev, result, prod, tmp, n, level, p_size, 2, h, bmods, true, s, true);
}

// The inner sum's recurrence, per bit i of k from 0 to floor(log2 k): the doubling element g^(2^i) when 2^(i+1) <= k
// (0: no doubling) and the shift element g^s when bit i is set (0: R is not updated), s the sum of the set bits below
// i.  Elements are reduced mod 2n; 1 is an identity.
struct InnerSumBit {
  uint64_t dbl, shift;
};
static std::vector<InnerSumBit> inner_sum_bits(uint64_t g, uint64_t k, uint64_t n) {
  std::vector<InnerSumBit> bits;
  const uint64_t two_n = 2 * n;
  uint64_t power = g % two_n, shift = 1;  // g^(2^i), g^s
  for (uint64_t i = 0; (k >> i) != 0; ++i) {
    InnerSumBit bit{0, 0};
    if ((k >> i) & 1) {
      bit.shift = shift;
      shift = shift * power % two_n;
    }
    if ((k >> (i + 1)) != 0) bit.dbl = power;
    power = power * power % two_n;
    bits.push_back(bit);
  }
  return bits;
}

// The inner sum of one ciphertext ct (two components of level limbs, NTT form, device memory) into result
// (2 x (level - rescale) x n words): per bit of k, with dbl_keys[i] / shift_keys[i] the keys of the bit's doubling and
// shift elements (nullptr for an identity or an absent rotation):
//   1. the step launches (per block of 64 moduli of B, only the data moduli while no Y is read or written): A' and R
//      from A's component 0 at l, pi_d(l) and pi_s(l);
//   2. with a keyed element: c1' = X_A1 + ModDown_P(Y_A1) (one component, into X_A1, which is not read again; none
//      while Y_A is empty), then one mod-up of c1' whose multiply-accumulates read pi_d and pi_s and add into Y_A' and
//      Y_R, laid out one stride apart;
//   3. after the last bit, the mod-down of Y_R adding into result, which holds X_R (none while Y_R is empty), or with
//      the rescale, [P] X_R folded into Y_R by the last step launch and the mod-down by q_{level-1} P that stores.
// A ping-pongs between two scratch pairs; at bit 0 it is ct itself, whose Y is empty.
static int inner_sum_hybrid_on_device(int dev, uint64_t* result, const uint64_t* ct, uint64_t n, uint64_t level,
                                      uint64_t q_size, uint64_t p_size, uint64_t alpha, bool rescale,
                                      const CachedNtts& h, const uint64_t* bmods, const std::vector<InnerSumBit>& bits,
                                      const uint64_t* const* const* dbl_keys, const uint64_t* const* const* shift_keys,
                                      cudaStream_t s) {
  const uint64_t D = (level + alpha - 1) / alpha, nb = level + p_size, kms = q_size + p_size, comp = level * n;
  const uint64_t stride = nb * 2 * n;  // one Y
  Scratch ws(s);
  uint64_t *xs = nullptr, *ys = nullptr, *xr = result, *y1 = nullptr, *tmp = nullptr;
  if (int rc = ws.get(&xs, 2 * 2 * comp)) return rc;  // X of the two A buffers, [2][k][i][n]
  if (int rc = ws.get(&ys, 3 * stride)) return rc;    // Y of the two A buffers, then Y_R, [3][b][k][n]
  if (rescale)
    if (int rc = ws.get(&xr, 2 * comp)) return rc;  // [k][i][n]
  if (int rc = ws.get(&y1, nb * n)) return rc;      // [b][n]
  if (int rc = ws.get(&tmp, std::min<uint64_t>(level, kParamBlock) * 2 * n)) return rc;  // [i][k][n], one block
  uint64_t* const yr = ys + 2 * stride;
  const uint64_t* xa = ct;
  uint64_t *xa_own = nullptr, *ya = nullptr;  // A in scratch (nullptr while A is ct)
  bool y_a = false, y_r = false, r_set = false;
  int next = 0;
  for (size_t i = 0; i < bits.size(); ++i) {
    const InnerSumBit& bit = bits[i];
    const bool dbl = bit.dbl != 0, upd = bit.shift != 0, fold = rescale && i + 1 == bits.size();
    const bool d_keyed = dbl && bit.dbl != 1, s_keyed = upd && bit.shift != 1;
    uint64_t *xn = xs + next * 2 * comp, *yn = ys + next * stride;
    int mode = y_a ? kSumYA : 0;
    if (dbl) {
      mode |= kSumNext;
      if (y_a || d_keyed) mode |= kSumNextY;
      if (bit.dbl == 1) mode |= kSumDoubleId;
    }
    if (upd) {
      mode |= kSumR;
      if (!r_set) mode |= kSumRStore;
      if (y_r) mode |= kSumRY;
      if (y_a || s_keyed || fold) mode |= kSumRYWrite;
      if (bit.shift == 1) mode |= kSumShiftId;
      if (fold) mode |= kSumFold;
    }
    if (y_a && (d_keyed || s_keyed)) mode |= kSumCopy1;
    // 1. the step; Y only where it is read or written
    const uint64_t span = (mode & (kSumNextY | kSumRYWrite | kSumCopy1)) ? nb : level;
    for (uint64_t b0 = 0; b0 < span; b0 += kParamBlock) {
      const uint64_t cnt = std::min<uint64_t>(kParamBlock, span - b0);
      KsModuli mods = ks_mac_moduli(bmods + b0, nullptr, cnt);
      if (fold)
        for (uint64_t e = 0; e < cnt && b0 + e < level; ++e) {
          const uint64_t q = bmods[b0 + e];
          uint64_t P = 1 % q;
          for (uint64_t j = 0; j < p_size; ++j) P = mul_mod128(P, bmods[level + j] % q, q);
          mods.m[e].c = P;
        }
      const cudaError_t e = launch_inner_sum_step(xa, ya, xn, yn, xr, yr, y1, n, level, b0, cnt, dbl ? bit.dbl : 1,
                                                  upd ? bit.shift : 1, mods, mode, s);
      if (e != cudaSuccess) return cuda_fail(e, "InnerSumHybrid: step launch");
    }
    // 2. the bit's keyed rotations, hoisted: one c1', one mod-up, the products of both elements
    if (d_keyed || s_keyed) {
      const uint64_t* c1 = xa + comp;
      if (y_a) {
        if (int rc = hybrid_mod_down(dev, xa_own + comp, y1, tmp, n, level, p_size, 1, h, bmods, true, s)) return rc;
        c1 = xa_own + comp;
      }
      const uint64_t* const* keys[2];
      uint64_t elts[2], count = 0;
      if (d_keyed) {
        keys[count] = dbl_keys[i];
        elts[count++] = bit.dbl;
      }
      if (s_keyed) {
        keys[count] = shift_keys[i];
        elts[count++] = bit.shift;
      }
      uint64_t* prod = d_keyed ? yn : yr;  // Y_A' below Y_R: the second element's products land one stride further
      const uint64_t pstride = (uint64_t)(yr - yn);
      Scratch wu(s);
      if (int rc = hybrid_mod_up(dev, c1, n, level, q_size, p_size, alpha, h, bmods, wu,
                                 [&](uint64_t b0, uint64_t cnt, const uint64_t* ops, const uint64_t* slots) {
                                   return ks_mac_products(h.data() + b0, slots, cnt, kms, ops, D, n, 2,
                                                          prod + b0 * 2 * n, pstride, keys, elts, count, s, true);
                                 },
                                 s))
        return rc;
    }
    if (dbl) {
      xa = xa_own = xn;
      ya = yn;
      y_a = (mode & kSumNextY) != 0;
      next ^= 1;
    }
    if (upd) {
      r_set = true;
      y_r = y_r || (mode & kSumRYWrite);
    }
  }
  // 3. the final mod-down
  if (rescale) return hybrid_mod_down(dev, result, yr, tmp, n, level - 1, p_size + 1, 2, h, bmods, false, s);
  if (!y_r) return 0;
  return hybrid_mod_down(dev, result, yr, tmp, n, level, p_size, 2, h, bmods, true, s);
}

// The shape rules of hexl_b200_key_switch_hybrid, without the key handle
static int hybrid_shape_check(uint64_t n, uint64_t level, uint64_t q_size, uint64_t p_size, uint64_t alpha,
                              uint64_t kcc, const uint64_t* moduli) {
  const uint64_t kms = q_size + p_size;
  REQUIRE(n >= 2 && n <= (1ull << 20) && !(n & (n - 1)), "Require n a power of two in [2, 2^20]");
  REQUIRE(level >= 1 && level <= q_size, "Require 1 <= level_size <= q_size");
  REQUIRE(alpha >= 1 && alpha <= (uint64_t)kParamBlock, "Require 1 <= digit_size <= %d", kParamBlock);
  REQUIRE(p_size >= 1 && p_size <= (uint64_t)kParamBlock, "Require 1 <= p_size <= %d", kParamBlock);
  REQUIRE(kcc >= 1, "Require key_component_count >= 1");
  for (uint64_t i = 0; i < kms; ++i) {
    const char* why = "";
    // the lazy sums of the multiply-accumulate and of the finish step (< 8q) need q < 2^61
    REQUIRE(moduli[i] < (1ull << 61), "Require moduli < 2^61 (moduli[%llu])", (unsigned long long)i);
    REQUIRE(check_ntt_arguments(n, moduli[i], &why), "moduli[%llu]: %s", (unsigned long long)i, why);
  }
  std::vector<uint64_t> sorted(moduli, moduli + kms);
  std::sort(sorted.begin(), sorted.end());
  REQUIRE(std::adjacent_find(sorted.begin(), sorted.end()) == sorted.end(), "Require distinct moduli");
  return 0;
}

int bgv_plain_modulus_check(uint64_t plain_modulus, const uint64_t* moduli, uint64_t count) {
  // the t-corrected conversion reduces its 128-bit sums mod tau with the lazy reductions of every other target
  REQUIRE(plain_modulus >= 2 && plain_modulus < (1ull << 61), "Require 2 <= plain_modulus < 2^61");
  for (uint64_t i = 0; i < count; ++i)
    REQUIRE(std::gcd(plain_modulus, moduli[i]) == 1, "Require plain_modulus coprime to moduli[%llu]",
            (unsigned long long)i);
  return 0;
}

// A hybrid key handle of the shape: ceil(q_size / digit_size) digits, kcc x (q_size + p_size) words, not sharded
static int hybrid_handle_check(const hexl_b200_keys* keys, uint64_t n, uint64_t q_size, uint64_t p_size,
                               uint64_t alpha, uint64_t kcc, const char* what) {
  REQUIRE(keys_fit(keys, n, (q_size + alpha - 1) / alpha, kcc, q_size + p_size),
          "%s was uploaded for another shape (decomp = ceil(q_size / digit_size), "
          "key_modulus_size = q_size + p_size)", what);
  REQUIRE(keys->shards.empty(), "%s: hybrid key switching does not take keys sharded by modulus: upload them with "
                                "hexl_b200_keys_upload", what);
  return 0;
}

// The extended basis B = {q_0..q_{l-1}, p_0..p_{K-1}} and its transforms
static int hybrid_basis(uint64_t n, uint64_t level, uint64_t q_size, uint64_t p_size, const uint64_t* moduli,
                        std::vector<uint64_t>* bmods, CachedNtts* h) {
  bmods->assign(moduli, moduli + level);
  bmods->insert(bmods->end(), moduli + q_size, moduli + q_size + p_size);
  for (uint64_t b = 0; b < bmods->size(); ++b)
    if (int rc = h->load(b, n, (*bmods)[b])) return rc;
  return 0;
}

// Host buffers of the base conversion: chunks of whole polynomials through stage_items, split by polynomial over the
// host devices; a slot holds a chunk of input polynomials in buffer 1 and their results in buffer 0.
static int base_convert_host(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* from,
                             uint64_t from_count, const uint64_t* to, uint64_t to_count, uint64_t count) {
  std::vector<int> devs;
  if (int rc = host_devices(&devs)) return rc;
  const uint64_t in_words = from_count * n, out_words = to_count * n;
  const uint64_t chunk = std::max<uint64_t>(1, (kChunkBytes / 8) / std::max(in_words, out_words));
  return stage_items(devs, count, chunk, [&](int, u64, u64, auto&& stage) {
    return stage([&](const StageSlot& sl, u64 p0, u64 cnt) -> int {
      if (int rc = sl.reserve(0, cnt * out_words * 8)) return rc;
      if (int rc = sl.reserve(1, cnt * in_words * 8)) return rc;
      const cudaStream_t sx = sl.stream();
      cudaError_t e =
          cudaMemcpyAsync(sl.buf(1), operand + p0 * in_words, cnt * in_words * 8, cudaMemcpyHostToDevice, sx);
      if (e != cudaSuccess) return cuda_fail(e, "FastBaseConvert H2D");
      if (int rc = base_convert_on_device(sl.buf(0), n, out_words, sl.buf(1), n, in_words, n, cnt, from, from_count,
                                          to, to_count, false, sx))
        return rc;
      e = cudaMemcpyAsync(result + p0 * out_words, sl.buf(0), cnt * out_words * 8, cudaMemcpyDeviceToHost, sx);
      return e == cudaSuccess ? 0 : cuda_fail(e, "FastBaseConvert D2H");
    });
  });
}

}  // namespace hexl_b200

// =============================================================== extern "C"
extern "C" {

int hexl_b200_fast_base_convert(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* from_moduli,
                                uint64_t from_count, const uint64_t* to_moduli, uint64_t to_count, uint64_t count,
                                void* stream) {
  REQUIRE(result && operand && from_moduli && to_moduli, "Require non-null arguments");
  REQUIRE(n >= 1, "Require n >= 1");
  REQUIRE(from_count >= 1 && from_count <= (uint64_t)kParamBlock, "Require 1 <= from_count <= %d", kParamBlock);
  REQUIRE(to_count >= 1, "Require to_count >= 1");
  for (uint64_t i = 0; i < from_count; ++i)
    REQUIRE(from_moduli[i] > 1 && from_moduli[i] < (1ull << 61), "Require 1 < from_moduli[%llu] < 2^61",
            (unsigned long long)i);
  for (uint64_t e = 0; e < to_count; ++e)
    REQUIRE(to_moduli[e] > 1 && to_moduli[e] < (1ull << 61), "Require 1 < to_moduli[%llu] < 2^61",
            (unsigned long long)e);
  for (uint64_t i = 0; i < from_count; ++i)
    for (uint64_t j = 0; j < i; ++j)
      REQUIRE(std::gcd(from_moduli[i], from_moduli[j]) == 1, "Require from_moduli pairwise coprime (%llu and %llu)",
              (unsigned long long)j, (unsigned long long)i);
  if (count == 0) return 0;
  const uint64_t in_total = count * from_count * n, out_total = count * to_count * n;
  REQUIRE(result + out_total <= operand || operand + in_total <= result, "result and operand must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, operand}, &pi)) return rc;
  if (int rc = check_limb_bounds(operand, count, from_count, n, [&](u64 i) { return from_moduli[i]; }, pi, "operand", stream))
    return rc;
  if (pi.where == Where::Device)
    return run_on_device(pi, stream, [&] {
      return base_convert_on_device(result, n, to_count * n, operand, n, from_count * n, n, count, from_moduli,
                                    from_count, to_moduli, to_count, false, (cudaStream_t)stream);
    });
  return base_convert_host(result, operand, n, from_moduli, from_count, to_moduli, to_count, count);
}

}  // extern "C"

namespace {

// hexl_b200_key_switch_hybrid, and with bgv hexl_b200_bgv_key_switch_hybrid
int key_switch_hybrid_call(uint64_t* result, const uint64_t* target, uint64_t n, uint64_t level_size, uint64_t q_size,
                           uint64_t p_size, uint64_t digit_size, uint64_t key_component_count, const uint64_t* moduli,
                           const hexl_b200_keys* keys, uint64_t batch, void* stream, bool bgv,
                           uint64_t plain_modulus) {
  const uint64_t level = level_size, alpha = digit_size, kcc = key_component_count;
  REQUIRE(result && target && moduli && keys, "Require non-null arguments");
  if (int rc = hybrid_shape_check(n, level, q_size, p_size, alpha, kcc, moduli)) return rc;
  if (bgv)
    if (int rc = bgv_plain_modulus_check(plain_modulus, moduli, q_size + p_size)) return rc;
  if (int rc = hybrid_handle_check(keys, n, q_size, p_size, alpha, kcc, "the key handle")) return rc;
  if (batch == 0) return 0;
  const uint64_t in_words = level * n, out_words = kcc * level * n;
  REQUIRE(result + batch * out_words <= target || target + batch * in_words <= result,
          "result and target must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, target}, &pi)) return rc;
  if (int rc = check_limb_bounds(target, batch, level, n, [&](u64 i) { return moduli[i]; }, pi, "target", stream)) return rc;
  std::vector<uint64_t> bmods;
  CachedNtts h(level + p_size);
  if (int rc = hybrid_basis(n, level, q_size, p_size, moduli, &bmods, &h)) return rc;
  if (pi.where == Where::Host)
    return key_switch_host_batch(result, out_words, true, target, in_words, in_words, &keys, 1, batch,
                                 [&](int dev, uint64_t* d_res, uint64_t* d_t, const uint64_t* const* const* dk,
                                     cudaStream_t s) {
                                   return key_switch_hybrid_on_device(dev, d_res, d_t, n, level, q_size, p_size,
                                                                      alpha, kcc, h, bmods.data(), dk[0], s,
                                                                      plain_modulus);
                                 });
  std::vector<const uint64_t* const*> dk;
  if (keys_on_device(&keys, 1, pi.device, &dk) < 1)
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "the key handle holds no copy on the device of result");
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = key_switch_hybrid_on_device(pi.device, result + c * out_words, target + c * in_words, n, level,
                                               q_size, p_size, alpha, kcc, h, bmods.data(), dk[0],
                                               (cudaStream_t)stream, plain_modulus))
        return rc;
    return 0;
  });
}

// The element and key-handle rules of the two hybrid rotation calls.  identity_ok: a null handle is an identity term,
// allowed for the element 1 only; otherwise every handle must be there.
int hybrid_elts_check(uint64_t n, uint64_t q_size, uint64_t p_size, uint64_t alpha, const hexl_b200_keys* const* keys,
                      const uint64_t* elts, uint64_t num_elts, bool identity_ok) {
  for (uint64_t r = 0; r < num_elts; ++r) {
    REQUIRE(elts[r] % 2 == 1 && elts[r] < 2 * n, "Require galois_elts[%llu] odd and in [1, 2n)", (unsigned long long)r);
    if (!keys[r]) {
      REQUIRE(identity_ok, "Require galois_keys[%llu] != nullptr", (unsigned long long)r);
      REQUIRE(elts[r] == 1, "galois_keys[%llu] may be null only for galois_elts[%llu] = 1 (an identity term)",
              (unsigned long long)r, (unsigned long long)r);
      continue;
    }
    char what[40];
    std::snprintf(what, sizeof what, "galois_keys[%llu]", (unsigned long long)r);
    if (int rc = hybrid_handle_check(keys[r], n, q_size, p_size, alpha, 2, what)) return rc;
  }
  return 0;
}

// Per element, the copy of its handle among `dk` (the copies of the non-null handles, in element order), or nullptr
// for an identity term
std::vector<const uint64_t* const*> per_element(const hexl_b200_keys* const* keys, uint64_t num_elts,
                                                const uint64_t* const* const* dk) {
  std::vector<const uint64_t* const*> out(num_elts, nullptr);
  for (uint64_t r = 0, k = 0; r < num_elts; ++r)
    if (keys[r]) out[r] = dk[k++];
  return out;
}

// hexl_b200_apply_galois_key_switch_hybrid_hoisted, and with bgv its BGV form
int hoisted_hybrid_call(uint64_t* results, const uint64_t* ciphertexts, uint64_t n, uint64_t level_size,
                        uint64_t q_size, uint64_t p_size, uint64_t digit_size, const uint64_t* moduli,
                        const hexl_b200_keys* const* galois_keys, const uint64_t* galois_elts, uint64_t num_elts,
                        uint64_t batch, void* stream, bool bgv, uint64_t plain_modulus) {
  const uint64_t level = level_size, alpha = digit_size;
  REQUIRE(results && ciphertexts && moduli, "Require non-null arguments");
  REQUIRE(num_elts == 0 || (galois_keys && galois_elts), "Require galois_keys, galois_elts != nullptr");
  if (int rc = hybrid_shape_check(n, level, q_size, p_size, alpha, 2, moduli)) return rc;
  if (bgv)
    if (int rc = bgv_plain_modulus_check(plain_modulus, moduli, q_size + p_size)) return rc;
  if (int rc = hybrid_elts_check(n, q_size, p_size, alpha, galois_keys, galois_elts, num_elts, false)) return rc;
  if (num_elts == 0 || batch == 0) return 0;
  const uint64_t comp = level * n, in_total = batch * 2 * comp, out_total = batch * num_elts * 2 * comp;
  REQUIRE(results + out_total <= ciphertexts || ciphertexts + in_total <= results,
          "results and ciphertexts must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({results, ciphertexts}, &pi)) return rc;
  if (int rc = check_limb_bounds(ciphertexts, 2 * batch, level, n, [&](u64 i) { return moduli[i]; }, pi,
                                 "ciphertexts", stream))
    return rc;
  std::vector<uint64_t> bmods;
  CachedNtts h(level + p_size);
  if (int rc = hybrid_basis(n, level, q_size, p_size, moduli, &bmods, &h)) return rc;
  // host pointers: each ciphertext crosses PCIe in once and its num_elts rotations come back from the same slot
  if (pi.where == Where::Host)
    return key_switch_host_batch(results, num_elts * 2 * comp, false, ciphertexts, 2 * comp, 2 * comp, galois_keys,
                                 num_elts, batch,
                                 [&](int dev, uint64_t* d_res, uint64_t* d_ct, const uint64_t* const* const* dk,
                                     cudaStream_t s) {
                                   return hybrid_hoisted_on_device(dev, d_res, d_ct, n, level, q_size, p_size, alpha,
                                                                   h, bmods.data(), dk, galois_elts, num_elts, s,
                                                                   plain_modulus);
                                 });
  std::vector<const uint64_t* const*> dk;
  const uint64_t missing = keys_on_device(galois_keys, num_elts, pi.device, &dk);
  if (missing < num_elts)
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "galois_keys[%llu] holds no copy on the device of the ciphertexts",
                (unsigned long long)missing);
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = hybrid_hoisted_on_device(pi.device, results + c * num_elts * 2 * comp, ciphertexts + c * 2 * comp, n,
                                            level, q_size, p_size, alpha, h, bmods.data(), dk.data(), galois_elts,
                                            num_elts, (cudaStream_t)stream, plain_modulus))
        return rc;
    return 0;
  });
}

}  // namespace

extern "C" {

int hexl_b200_key_switch_hybrid(uint64_t* result, const uint64_t* target, uint64_t n, uint64_t level_size,
                                uint64_t q_size, uint64_t p_size, uint64_t digit_size, uint64_t key_component_count,
                                const uint64_t* moduli, const hexl_b200_keys* keys, uint64_t batch, void* stream) {
  return key_switch_hybrid_call(result, target, n, level_size, q_size, p_size, digit_size, key_component_count, moduli,
                                keys, batch, stream, false, 0);
}

int hexl_b200_bgv_key_switch_hybrid(uint64_t* result, const uint64_t* target, uint64_t n, uint64_t level_size,
                                    uint64_t q_size, uint64_t p_size, uint64_t digit_size,
                                    uint64_t key_component_count, const uint64_t* moduli, uint64_t plain_modulus,
                                    const hexl_b200_keys* keys, uint64_t batch, void* stream) {
  return key_switch_hybrid_call(result, target, n, level_size, q_size, p_size, digit_size, key_component_count, moduli,
                                keys, batch, stream, true, plain_modulus);
}

int hexl_b200_apply_galois_key_switch_hybrid_hoisted(uint64_t* results, const uint64_t* ciphertexts, uint64_t n,
                                                     uint64_t level_size, uint64_t q_size, uint64_t p_size,
                                                     uint64_t digit_size, const uint64_t* moduli,
                                                     const hexl_b200_keys* const* galois_keys,
                                                     const uint64_t* galois_elts, uint64_t num_elts, uint64_t batch,
                                                     void* stream) {
  return hoisted_hybrid_call(results, ciphertexts, n, level_size, q_size, p_size, digit_size, moduli, galois_keys,
                             galois_elts, num_elts, batch, stream, false, 0);
}

int hexl_b200_bgv_apply_galois_key_switch_hybrid_hoisted(uint64_t* results, const uint64_t* ciphertexts, uint64_t n,
                                                         uint64_t level_size, uint64_t q_size, uint64_t p_size,
                                                         uint64_t digit_size, const uint64_t* moduli,
                                                         uint64_t plain_modulus,
                                                         const hexl_b200_keys* const* galois_keys,
                                                         const uint64_t* galois_elts, uint64_t num_elts,
                                                         uint64_t batch, void* stream) {
  return hoisted_hybrid_call(results, ciphertexts, n, level_size, q_size, p_size, digit_size, moduli, galois_keys,
                             galois_elts, num_elts, batch, stream, true, plain_modulus);
}

int hexl_b200_linear_transform_hybrid(uint64_t* result, const uint64_t* ciphertexts, uint64_t n, uint64_t level_size,
                                      uint64_t q_size, uint64_t p_size, uint64_t digit_size, const uint64_t* moduli,
                                      const hexl_b200_keys* const* galois_keys, const uint64_t* galois_elts,
                                      uint64_t num_elts, const uint64_t* diagonals, uint64_t batch, void* stream) {
  const uint64_t level = level_size, alpha = digit_size;
  REQUIRE(result && ciphertexts && moduli, "Require non-null arguments");
  REQUIRE(num_elts == 0 || (galois_keys && galois_elts && diagonals),
          "Require galois_keys, galois_elts, diagonals != nullptr");
  if (int rc = hybrid_shape_check(n, level, q_size, p_size, alpha, 2, moduli)) return rc;
  if (int rc = hybrid_elts_check(n, q_size, p_size, alpha, galois_keys, galois_elts, num_elts, true)) return rc;
  if (num_elts == 0 || batch == 0) return 0;
  const uint64_t comp = level * n, nb = level + p_size, ct_total = batch * 2 * comp, diag_total = num_elts * nb * n;
  REQUIRE(result + ct_total <= ciphertexts || ciphertexts + ct_total <= result,
          "result and ciphertexts must not overlap");
  REQUIRE(result + ct_total <= diagonals || diagonals + diag_total <= result, "result and diagonals must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, ciphertexts, diagonals}, &pi)) return rc;
  if (int rc = check_limb_bounds(ciphertexts, 2 * batch, level, n, [&](u64 i) { return moduli[i]; }, pi,
                                 "ciphertexts", stream))
    return rc;
  std::vector<uint64_t> bmods;
  CachedNtts h(nb);
  if (int rc = hybrid_basis(n, level, q_size, p_size, moduli, &bmods, &h)) return rc;
  if (int rc = check_limb_bounds(diagonals, num_elts, nb, n, [&](u64 i) { return bmods[i]; }, pi, "diagonals", stream))
    return rc;
  std::vector<const hexl_b200_keys*> keyed;  // the handles of the elements that switch keys
  for (uint64_t r = 0; r < num_elts; ++r)
    if (galois_keys[r]) keyed.push_back(galois_keys[r]);
  if (pi.where == Where::Host) {
    // host pointers: the diagonals go to each device of the split once, before its first ciphertext; each ciphertext
    // crosses PCIe in once and its result comes back from the same slot
    std::vector<std::pair<int, uint64_t*>> uploaded;
    const int rc = key_switch_host_batch(
        result, 2 * comp, false, ciphertexts, 2 * comp, 2 * comp, keyed.data(), keyed.size(), batch,
        [&](int dev, uint64_t* d_res, uint64_t* d_ct, const uint64_t* const* const* dk, cudaStream_t s) {
          const uint64_t* d_diag = nullptr;
          for (auto& u : uploaded)
            if (u.first == dev) d_diag = u.second;
          const auto keys = per_element(galois_keys, num_elts, dk);
          return linear_transform_hybrid_on_device(dev, d_res, d_ct, d_diag, n, level, q_size, p_size, alpha, h,
                                                   bmods.data(), keys.data(), galois_elts, num_elts, s);
        },
        [&](int dev) -> int {
          uint64_t* p = nullptr;
          CU(cudaMalloc(&p, diag_total * sizeof(uint64_t)));
          uploaded.emplace_back(dev, p);
          CU(cudaMemcpy(p, diagonals, diag_total * sizeof(uint64_t), cudaMemcpyHostToDevice));
          CU(cudaStreamSynchronize(nullptr));  // the staging streams do not wait for the legacy stream's copy
          return 0;
        });
    for (auto& u : uploaded) {
      DeviceGuard g;
      if (g.enter(u.first) == 0) cudaFree(u.second);
    }
    return rc;
  }
  std::vector<const uint64_t* const*> dk;
  const uint64_t found = keys_on_device(keyed.data(), keyed.size(), pi.device, &dk);
  if (found < keyed.size())
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "a key handle holds no copy on the device of the ciphertexts");
  const auto keys = per_element(galois_keys, num_elts, dk.data());
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = linear_transform_hybrid_on_device(pi.device, result + c * 2 * comp, ciphertexts + c * 2 * comp,
                                                     diagonals, n, level, q_size, p_size, alpha, h, bmods.data(),
                                                     keys.data(), galois_elts, num_elts, (cudaStream_t)stream))
        return rc;
    return 0;
  });
}

int hexl_b200_linear_transform_hybrid_bsgs(uint64_t* result, const uint64_t* ciphertexts, uint64_t n,
                                           uint64_t level_size, uint64_t q_size, uint64_t p_size, uint64_t digit_size,
                                           const uint64_t* moduli, const hexl_b200_keys* const* baby_keys,
                                           const uint64_t* baby_elts, uint64_t num_baby,
                                           const hexl_b200_keys* const* giant_keys, const uint64_t* giant_elts,
                                           uint64_t num_giant, const uint64_t* const* diagonals, int rescale,
                                           uint64_t batch, void* stream) {
  const uint64_t level = level_size, alpha = digit_size, n1 = num_baby, n2 = num_giant;
  REQUIRE(result && ciphertexts && moduli, "Require non-null arguments");
  REQUIRE(n1 == 0 || (baby_keys && baby_elts), "Require baby_keys, baby_elts != nullptr");
  REQUIRE(n2 == 0 || (giant_keys && giant_elts), "Require giant_keys, giant_elts != nullptr");
  REQUIRE(n1 * n2 == 0 || diagonals, "Require diagonals != nullptr");
  if (int rc = hybrid_shape_check(n, level, q_size, p_size, alpha, 2, moduli)) return rc;
  if (int rc = hybrid_elts_check(n, q_size, p_size, alpha, baby_keys, baby_elts, n1, true)) return rc;
  if (int rc = hybrid_elts_check(n, q_size, p_size, alpha, giant_keys, giant_elts, n2, true)) return rc;
  REQUIRE(rescale == 0 || rescale == 1, "Require rescale = 0 or 1");
  REQUIRE(!rescale || level >= 2, "rescale = 1 requires level_size >= 2");
  REQUIRE(!rescale || p_size < (uint64_t)kParamBlock, "rescale = 1 requires p_size <= %d", kParamBlock - 1);
  if (n1 == 0 || n2 == 0 || batch == 0) return 0;
  const uint64_t comp = level * n, nb = level + p_size, in_words = 2 * comp, out_words = 2 * (level - rescale) * n;
  const uint64_t in_total = batch * in_words, out_total = batch * out_words, dwords = nb * n;
  REQUIRE(result + out_total <= ciphertexts || ciphertexts + in_total <= result,
          "result and ciphertexts must not overlap");
  std::vector<uint64_t> present;  // the indices of the present diagonals in diagonals[]
  for (uint64_t r = 0; r < n1 * n2; ++r)
    if (diagonals[r]) {
      present.push_back(r);
      REQUIRE(result + out_total <= diagonals[r] || diagonals[r] + dwords <= result,
              "result and diagonals[%llu] must not overlap", (unsigned long long)r);
    }
  PtrInfo pi;
  if (int rc = classify_all({result, ciphertexts}, &pi)) return rc;
  for (uint64_t r : present) {
    PtrInfo pd;
    if (int rc = classify_all({result, diagonals[r]}, &pd)) return rc;
  }
  if (int rc = check_limb_bounds(ciphertexts, 2 * batch, level, n, [&](u64 i) { return moduli[i]; }, pi,
                                 "ciphertexts", stream))
    return rc;
  std::vector<uint64_t> bmods;
  CachedNtts h(nb);
  if (int rc = hybrid_basis(n, level, q_size, p_size, moduli, &bmods, &h)) return rc;
  for (uint64_t r : present)
    if (int rc = check_limb_bounds(diagonals[r], 1, nb, n, [&](u64 i) { return bmods[i]; }, pi, "diagonals", stream)) return rc;
  // the handles that switch keys: the keyed babies', then the keyed giants'
  std::vector<const hexl_b200_keys*> keyed;
  for (uint64_t i = 0; i < n1; ++i)
    if (baby_keys[i]) keyed.push_back(baby_keys[i]);
  const uint64_t keyed_babies = keyed.size();
  for (uint64_t j = 0; j < n2; ++j)
    if (giant_keys[j]) keyed.push_back(giant_keys[j]);
  const bool rs = rescale != 0;
  if (pi.where == Where::Host) {
    // host pointers: the present diagonals go to each device of the split once, before its first ciphertext; each
    // ciphertext crosses PCIe in once and its result comes back from the same slot
    std::vector<std::pair<int, uint64_t*>> uploaded;
    std::vector<std::vector<const uint64_t*>> tables;  // per uploaded device: diagonals[] on that device
    const int rc = key_switch_host_batch(
        result, out_words, false, ciphertexts, in_words, in_words, keyed.data(), keyed.size(), batch,
        [&](int dev, uint64_t* d_res, uint64_t* d_ct, const uint64_t* const* const* dk, cudaStream_t s) {
          const std::vector<const uint64_t*>* d_diag = nullptr;
          for (size_t u = 0; u < uploaded.size(); ++u)
            if (uploaded[u].first == dev) d_diag = &tables[u];
          const auto babies = per_element(baby_keys, n1, dk);
          const auto giants = per_element(giant_keys, n2, dk + keyed_babies);
          return bsgs_hybrid_on_device(dev, d_res, d_ct, d_diag->data(), n, level, q_size, p_size, alpha, rs, h,
                                       bmods.data(), babies.data(), baby_elts, n1, giants.data(), giant_elts, n2, s);
        },
        [&](int dev) -> int {
          uint64_t* p = nullptr;
          CU(cudaMalloc(&p, std::max<uint64_t>(1, present.size()) * dwords * sizeof(uint64_t)));
          uploaded.emplace_back(dev, p);
          tables.emplace_back(n1 * n2, nullptr);
          for (size_t k = 0; k < present.size(); ++k) {
            CU(cudaMemcpy(p + k * dwords, diagonals[present[k]], dwords * sizeof(uint64_t), cudaMemcpyHostToDevice));
            tables.back()[present[k]] = p + k * dwords;
          }
          CU(cudaStreamSynchronize(nullptr));  // the staging streams do not wait for the legacy stream's copies
          return 0;
        });
    for (auto& u : uploaded) {
      DeviceGuard g;
      if (g.enter(u.first) == 0) cudaFree(u.second);
    }
    return rc;
  }
  std::vector<const uint64_t* const*> dk;
  const uint64_t found = keys_on_device(keyed.data(), keyed.size(), pi.device, &dk);
  if (found < keyed.size())
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "a key handle holds no copy on the device of the ciphertexts");
  const auto babies = per_element(baby_keys, n1, dk.data());
  const auto giants = per_element(giant_keys, n2, dk.data() + keyed_babies);
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = bsgs_hybrid_on_device(pi.device, result + c * out_words, ciphertexts + c * in_words, diagonals, n,
                                         level, q_size, p_size, alpha, rs, h, bmods.data(), babies.data(), baby_elts,
                                         n1, giants.data(), giant_elts, n2, (cudaStream_t)stream))
        return rc;
    return 0;
  });
}

}  // extern "C"

namespace {

// hexl_b200_multiply_relinearize_hybrid, and with bgv hexl_b200_bgv_multiply_relinearize_hybrid, whose merged mod-down
// is the modulus switch (the messages name rescale mod_switch there)
int multiply_relinearize_hybrid_call(uint64_t* result, const uint64_t* ct1, const uint64_t* ct2, uint64_t n,
                                     uint64_t level_size, uint64_t q_size, uint64_t p_size, uint64_t digit_size,
                                     const uint64_t* moduli, const hexl_b200_keys* relin_keys, int rescale,
                                     uint64_t batch, void* stream, bool bgv, uint64_t plain_modulus) {
  const uint64_t level = level_size, alpha = digit_size;
  const char* flag = bgv ? "mod_switch" : "rescale";
  REQUIRE(result && ct1 && ct2 && moduli && relin_keys, "Require non-null arguments");
  if (int rc = hybrid_shape_check(n, level, q_size, p_size, alpha, 2, moduli)) return rc;
  if (bgv)
    if (int rc = bgv_plain_modulus_check(plain_modulus, moduli, q_size + p_size)) return rc;
  if (int rc = hybrid_handle_check(relin_keys, n, q_size, p_size, alpha, 2, "relin_keys")) return rc;
  REQUIRE(rescale == 0 || rescale == 1, "Require %s = 0 or 1", flag);
  // the merged rescale divides by q_{l-1} too: a level to drop, and K + 1 sources of one base conversion
  REQUIRE(!rescale || level >= 2, "%s = 1 requires level_size >= 2", flag);
  REQUIRE(!rescale || p_size < (uint64_t)kParamBlock, "%s = 1 requires p_size <= %d", flag, kParamBlock - 1);
  if (batch == 0) return 0;
  const uint64_t in_words = 2 * level * n, out_words = 2 * (level - rescale) * n;
  const uint64_t in_total = batch * in_words, out_total = batch * out_words;
  REQUIRE(ct1 == ct2 || ct1 + in_total <= ct2 || ct2 + in_total <= ct1,
          "ct1 and ct2 must be the same ciphertexts or not overlap");
  REQUIRE(result + out_total <= ct1 || ct1 + in_total <= result, "result and ct1 must not overlap");
  REQUIRE(result + out_total <= ct2 || ct2 + in_total <= result, "result and ct2 must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, ct1, ct2}, &pi)) return rc;
  auto bound = [&](u64 i) { return moduli[i]; };
  if (int rc = check_limb_bounds(ct1, 2 * batch, level, n, bound, pi, "ct1", stream)) return rc;
  if (ct2 != ct1)
    if (int rc = check_limb_bounds(ct2, 2 * batch, level, n, bound, pi, "ct2", stream)) return rc;
  std::vector<uint64_t> bmods;
  CachedNtts h(level + p_size);
  if (int rc = hybrid_basis(n, level, q_size, p_size, moduli, &bmods, &h)) return rc;
  const bool rs = rescale != 0;
  // host pointers: both ciphertexts of a pair cross PCIe in once (one copy when squaring) and the product comes back
  // from the same slot
  if (pi.where == Where::Host) {
    const bool square = ct1 == ct2;
    return key_switch_host_batch(result, out_words, false, ct1, in_words, square ? in_words : 2 * in_words,
                                 &relin_keys, 1, batch,
                                 [&](int dev, uint64_t* d_res, uint64_t* d_in, const uint64_t* const* const* dk,
                                     cudaStream_t s) {
                                   return multiply_relinearize_hybrid_on_device(
                                       dev, d_res, d_in, square ? d_in : d_in + in_words, n, level, q_size, p_size,
                                       alpha, rs, h, bmods.data(), dk[0], s, nullptr, plain_modulus);
                                 },
                                 nullptr, square ? nullptr : ct2);
  }
  std::vector<const uint64_t* const*> dk;
  if (keys_on_device(&relin_keys, 1, pi.device, &dk) < 1)
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "relin_keys holds no copy on the device of the ciphertexts");
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = multiply_relinearize_hybrid_on_device(pi.device, result + c * out_words, ct1 + c * in_words,
                                                         ct2 + c * in_words, n, level, q_size, p_size, alpha, rs, h,
                                                         bmods.data(), dk[0], (cudaStream_t)stream, nullptr,
                                                         plain_modulus))
        return rc;
    return 0;
  });
}

}  // namespace

extern "C" {

int hexl_b200_multiply_relinearize_hybrid(uint64_t* result, const uint64_t* ct1, const uint64_t* ct2, uint64_t n,
                                          uint64_t level_size, uint64_t q_size, uint64_t p_size, uint64_t digit_size,
                                          const uint64_t* moduli, const hexl_b200_keys* relin_keys, int rescale,
                                          uint64_t batch, void* stream) {
  return multiply_relinearize_hybrid_call(result, ct1, ct2, n, level_size, q_size, p_size, digit_size, moduli,
                                          relin_keys, rescale, batch, stream, false, 0);
}

int hexl_b200_bgv_multiply_relinearize_hybrid(uint64_t* result, const uint64_t* ct1, const uint64_t* ct2, uint64_t n,
                                              uint64_t level_size, uint64_t q_size, uint64_t p_size,
                                              uint64_t digit_size, const uint64_t* moduli, uint64_t plain_modulus,
                                              const hexl_b200_keys* relin_keys, int mod_switch, uint64_t batch,
                                              void* stream) {
  return multiply_relinearize_hybrid_call(result, ct1, ct2, n, level_size, q_size, p_size, digit_size, moduli,
                                          relin_keys, mod_switch, batch, stream, true, plain_modulus);
}

int hexl_b200_multiply_relinearize_sum_hybrid(uint64_t* result, const uint64_t* const* ct1, const uint64_t* const* ct2,
                                              uint64_t num_pairs, uint64_t n, uint64_t level_size, uint64_t q_size,
                                              uint64_t p_size, uint64_t digit_size, const uint64_t* moduli,
                                              const hexl_b200_keys* relin_keys, int rescale, uint64_t batch,
                                              void* stream) {
  const uint64_t level = level_size, alpha = digit_size, k = num_pairs, total = batch * num_pairs;
  REQUIRE(result && moduli && relin_keys, "Require non-null arguments");
  REQUIRE(total == 0 || (ct1 && ct2), "Require ct1, ct2 != nullptr");
  if (int rc = hybrid_shape_check(n, level, q_size, p_size, alpha, 2, moduli)) return rc;
  if (int rc = hybrid_handle_check(relin_keys, n, q_size, p_size, alpha, 2, "relin_keys")) return rc;
  REQUIRE(rescale == 0 || rescale == 1, "Require rescale = 0 or 1");
  REQUIRE(!rescale || level >= 2, "rescale = 1 requires level_size >= 2");
  REQUIRE(!rescale || p_size < (uint64_t)kParamBlock, "rescale = 1 requires p_size <= %d", kParamBlock - 1);
  if (total == 0) return 0;
  const uint64_t in_words = 2 * level * n, out_words = 2 * (level - rescale) * n, out_total = batch * out_words;
  // the distinct input ciphertexts, each read (and checked, and on host buffers uploaded) once
  std::vector<const uint64_t*> inputs;
  for (uint64_t x = 0; x < total; ++x) {
    REQUIRE(ct1[x] && ct2[x], "Require ct1[%llu], ct2[%llu] != nullptr", (unsigned long long)x, (unsigned long long)x);
    inputs.push_back(ct1[x]);
    inputs.push_back(ct2[x]);
  }
  std::sort(inputs.begin(), inputs.end());
  inputs.erase(std::unique(inputs.begin(), inputs.end()), inputs.end());
  for (const uint64_t* p : inputs)
    REQUIRE(result + out_total <= p || p + in_words <= result, "result must not overlap an input ciphertext");
  PtrInfo pi;
  if (int rc = classify_all({result, inputs[0]}, &pi)) return rc;
  for (const uint64_t* p : inputs) {
    PtrInfo pp;
    if (int rc = classify_all({result, p}, &pp)) return rc;
    pi.managed = pi.managed || pp.managed;
  }
  for (const uint64_t* p : inputs)
    if (int rc = check_limb_bounds(p, 2, level, n, [&](u64 i) { return moduli[i]; }, pi, "an input ciphertext", stream))
      return rc;
  std::vector<uint64_t> bmods;
  CachedNtts h(level + p_size);
  if (int rc = hybrid_basis(n, level, q_size, p_size, moduli, &bmods, &h)) return rc;
  const bool rs = rescale != 0;
  if (pi.where == Where::Host) {
    // host pointers: the distinct inputs go to each device of the split once, before its first output; each output is
    // computed in a staging slot and comes back from it.  key_switch_host_batch runs the outputs in order, so the
    // calls of `run` count them.
    std::vector<uint64_t> slot1(total), slot2(total);  // entry x's index among the distinct inputs
    for (uint64_t x = 0; x < total; ++x) {
      slot1[x] = std::lower_bound(inputs.begin(), inputs.end(), ct1[x]) - inputs.begin();
      slot2[x] = std::lower_bound(inputs.begin(), inputs.end(), ct2[x]) - inputs.begin();
    }
    std::vector<std::pair<int, uint64_t*>> uploaded;
    uint64_t c = 0;
    const int rc = key_switch_host_batch(
        result, out_words, false, nullptr, 0, 0, &relin_keys, 1, batch,
        [&](int dev, uint64_t* d_res, uint64_t*, const uint64_t* const* const* dk, cudaStream_t s) {
          const uint64_t* base = nullptr;
          for (auto& u : uploaded)
            if (u.first == dev) base = u.second;
          std::vector<const uint64_t*> a(k), b(k);
          for (uint64_t r = 0; r < k; ++r) {
            a[r] = base + slot1[c * k + r] * in_words;
            b[r] = base + slot2[c * k + r] * in_words;
          }
          ++c;
          return multiply_relinearize_sum_hybrid_on_device(dev, d_res, a.data(), b.data(), k, n, level, q_size, p_size,
                                                           alpha, rs, h, bmods.data(), dk[0], s);
        },
        [&](int dev) -> int {
          uint64_t* p = nullptr;
          CU(cudaMalloc(&p, inputs.size() * in_words * sizeof(uint64_t)));
          uploaded.emplace_back(dev, p);
          for (size_t i = 0; i < inputs.size(); ++i)
            CU(cudaMemcpy(p + i * in_words, inputs[i], in_words * sizeof(uint64_t), cudaMemcpyHostToDevice));
          CU(cudaStreamSynchronize(nullptr));  // the staging streams do not wait for the legacy stream's copies
          return 0;
        });
    for (auto& u : uploaded) {
      DeviceGuard g;
      if (g.enter(u.first) == 0) cudaFree(u.second);
    }
    return rc;
  }
  std::vector<const uint64_t* const*> dk;
  if (keys_on_device(&relin_keys, 1, pi.device, &dk) < 1)
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "relin_keys holds no copy on the device of the ciphertexts");
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = multiply_relinearize_sum_hybrid_on_device(pi.device, result + c * out_words, ct1 + c * k,
                                                             ct2 + c * k, k, n, level, q_size, p_size, alpha, rs, h,
                                                             bmods.data(), dk[0], (cudaStream_t)stream))
        return rc;
    return 0;
  });
}

int hexl_b200_inner_sum_hybrid(uint64_t* result, const uint64_t* ciphertexts, uint64_t n, uint64_t level_size,
                               uint64_t q_size, uint64_t p_size, uint64_t digit_size, const uint64_t* moduli,
                               uint64_t galois_elt, uint64_t sum_count, const hexl_b200_keys* const* galois_keys,
                               const uint64_t* key_elts, uint64_t num_keys, int rescale, uint64_t batch,
                               void* stream) {
  const uint64_t level = level_size, alpha = digit_size, g = galois_elt;
  REQUIRE(result && ciphertexts && moduli, "Require non-null arguments");
  REQUIRE(num_keys == 0 || (galois_keys && key_elts), "Require galois_keys, key_elts != nullptr");
  if (int rc = hybrid_shape_check(n, level, q_size, p_size, alpha, 2, moduli)) return rc;
  REQUIRE(g % 2 == 1 && g < 2 * n, "Require galois_elt odd and in [1, 2n)");
  REQUIRE(rescale == 0 || rescale == 1, "Require rescale = 0 or 1");
  REQUIRE(!rescale || level >= 2, "rescale = 1 requires level_size >= 2");
  REQUIRE(!rescale || p_size < (uint64_t)kParamBlock, "rescale = 1 requires p_size <= %d", kParamBlock - 1);
  // the keys of every element the recurrence rotates by, looked up in the table: used[] the distinct handles, and per
  // bit the index of its doubling's and its shift's handle among them (-1: identity or none)
  const std::vector<InnerSumBit> bits = inner_sum_bits(g, sum_count, n);
  std::vector<const hexl_b200_keys*> used;
  std::vector<int64_t> dbl_slot(bits.size(), -1), shift_slot(bits.size(), -1);
  auto lookup = [&](uint64_t elt, int64_t* slot) -> int {
    if (elt <= 1) return 0;
    uint64_t r = 0;
    while (r < num_keys && key_elts[r] != elt) ++r;
    REQUIRE(r < num_keys, "no key for the Galois element %llu, which the sum of %llu rotations by %llu needs",
            (unsigned long long)elt, (unsigned long long)sum_count, (unsigned long long)g);
    REQUIRE(galois_keys[r], "Require galois_keys[%llu] != nullptr (the key of element %llu)", (unsigned long long)r,
            (unsigned long long)elt);
    char what[40];
    std::snprintf(what, sizeof what, "galois_keys[%llu]", (unsigned long long)r);
    if (int rc = hybrid_handle_check(galois_keys[r], n, q_size, p_size, alpha, 2, what)) return rc;
    const auto it = std::find(used.begin(), used.end(), galois_keys[r]);
    *slot = it - used.begin();
    if (it == used.end()) used.push_back(galois_keys[r]);
    return 0;
  };
  for (size_t i = 0; i < bits.size(); ++i) {
    if (int rc = lookup(bits[i].dbl, &dbl_slot[i])) return rc;
    if (int rc = lookup(bits[i].shift, &shift_slot[i])) return rc;
  }
  if (sum_count == 0 || batch == 0) return 0;
  const uint64_t in_words = 2 * level * n, out_words = 2 * (level - rescale) * n;
  REQUIRE(result + batch * out_words <= ciphertexts || ciphertexts + batch * in_words <= result,
          "result and ciphertexts must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, ciphertexts}, &pi)) return rc;
  if (int rc = check_limb_bounds(ciphertexts, 2 * batch, level, n, [&](u64 i) { return moduli[i]; }, pi,
                                 "ciphertexts", stream))
    return rc;
  std::vector<uint64_t> bmods;
  CachedNtts h(level + p_size);
  if (int rc = hybrid_basis(n, level, q_size, p_size, moduli, &bmods, &h)) return rc;
  const bool rs = rescale != 0;
  // one ciphertext on one device: dk[u] is used[u]'s copy there
  auto run = [&](int dev, uint64_t* res, const uint64_t* ct, const uint64_t* const* const* dk, cudaStream_t s) {
    std::vector<const uint64_t* const*> dbl_keys(bits.size(), nullptr), shift_keys(bits.size(), nullptr);
    for (size_t i = 0; i < bits.size(); ++i) {
      if (dbl_slot[i] >= 0) dbl_keys[i] = dk[dbl_slot[i]];
      if (shift_slot[i] >= 0) shift_keys[i] = dk[shift_slot[i]];
    }
    return inner_sum_hybrid_on_device(dev, res, ct, n, level, q_size, p_size, alpha, rs, h, bmods.data(), bits,
                                      dbl_keys.data(), shift_keys.data(), s);
  };
  // host pointers: each ciphertext crosses PCIe in once and its sum comes back from the same slot
  if (pi.where == Where::Host)
    return key_switch_host_batch(result, out_words, false, ciphertexts, in_words, in_words, used.data(), used.size(),
                                 batch,
                                 [&](int dev, uint64_t* d_res, uint64_t* d_ct, const uint64_t* const* const* dk,
                                     cudaStream_t s) { return run(dev, d_res, d_ct, dk, s); });
  std::vector<const uint64_t* const*> dk;
  if (keys_on_device(used.data(), used.size(), pi.device, &dk) < used.size())
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "a key handle holds no copy on the device of the ciphertexts");
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = run(pi.device, result + c * out_words, ciphertexts + c * in_words, dk.data(), (cudaStream_t)stream))
        return rc;
    return 0;
  });
}

int hexl_b200_bfv_multiply_relinearize_hybrid(uint64_t* result, const uint64_t* ct1, const uint64_t* ct2, uint64_t n,
                                              uint64_t level_size, uint64_t q_size, uint64_t p_size,
                                              uint64_t digit_size, const uint64_t* moduli, const uint64_t* base_b,
                                              uint64_t base_b_size, uint64_t m_sk, uint64_t plain_modulus,
                                              const hexl_b200_keys* relin_keys, uint64_t batch, void* stream) {
  const uint64_t level = level_size, alpha = digit_size, k = base_b_size;
  REQUIRE(result && ct1 && ct2 && moduli && base_b && relin_keys, "Require non-null arguments");
  if (int rc = hybrid_shape_check(n, level, q_size, p_size, alpha, 2, moduli)) return rc;
  if (int rc = hybrid_handle_check(relin_keys, n, q_size, p_size, alpha, 2, "relin_keys")) return rc;
  if (int rc = bfv_check(result, ct1, ct2, n, moduli, level, base_b, k, m_sk, plain_modulus)) return rc;
  if (batch == 0) return 0;
  const uint64_t comp = level * n, words = 2 * comp, total = batch * words;
  REQUIRE(result + total <= ct1 || ct1 + total <= result, "result and ct1 must not overlap");
  REQUIRE(result + total <= ct2 || ct2 + total <= result, "result and ct2 must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, ct1, ct2}, &pi)) return rc;
  auto bound = [&](u64 i) { return moduli[i]; };
  if (int rc = check_limb_bounds(ct1, 2 * batch, level, n, bound, pi, "ct1", stream)) return rc;
  if (ct2 != ct1)
    if (int rc = check_limb_bounds(ct2, 2 * batch, level, n, bound, pi, "ct2", stream)) return rc;
  BfvPlan plan(level + k + 1);
  if (int rc = bfv_plan(&plan, n, moduli, level, base_b, k, m_sk, plain_modulus)) return rc;
  std::vector<uint64_t> bmods;
  CachedNtts h(level + p_size);
  if (int rc = hybrid_basis(n, level, q_size, p_size, moduli, &bmods, &h)) return rc;
  // host pointers: both ciphertexts of a pair cross PCIe in once (one copy when squaring) and the product comes back
  // from the same slot
  if (pi.where == Where::Host) {
    const bool square = ct1 == ct2;
    return key_switch_host_batch(result, words, false, ct1, words, square ? words : 2 * words, &relin_keys, 1, batch,
                                 [&](int dev, uint64_t* d_res, uint64_t* d_in, const uint64_t* const* const* dk,
                                     cudaStream_t s) {
                                   return bfv_multiply_relinearize_on_device(
                                       dev, d_res, d_in, square ? d_in : d_in + words, plan, n, level, q_size, p_size,
                                       alpha, h, bmods.data(), dk[0], s);
                                 },
                                 nullptr, square ? nullptr : ct2);
  }
  std::vector<const uint64_t* const*> dk;
  if (keys_on_device(&relin_keys, 1, pi.device, &dk) < 1)
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "relin_keys holds no copy on the device of the ciphertexts");
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = bfv_multiply_relinearize_on_device(pi.device, result + c * words, ct1 + c * words,
                                                      ct2 + c * words, plan, n, level, q_size, p_size, alpha, h,
                                                      bmods.data(), dk[0], (cudaStream_t)stream))
        return rc;
    return 0;
  });
}

}  // extern "C"
