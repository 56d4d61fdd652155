// ApplyGalois, the rotation of ciphertexts with its key switch, and the hoisted rotations of one ciphertext.
#include "capi.h"

using namespace hexl_b200;

namespace {

int galois_elt_check(uint64_t n, uint64_t galois_elt) {
  REQUIRE(galois_elt % 2 == 1 && galois_elt < 2 * n, "Require galois_elt odd and in [1, 2n)");
  return 0;
}

// g^-1 mod 2n (g odd): Newton's iteration doubles the correct low bits of an inverse mod 2^64 (g is its own inverse
// mod 8), so five steps give all 64
uint64_t galois_inverse(uint64_t g, uint64_t n) {
  uint64_t inv = g;
  for (int i = 0; i < 5; ++i) inv *= 2 - g * inv;
  return inv & (2 * n - 1);
}

// `count` polynomials of rns limbs x n words, device pointers on the current device.  NTT form: one launch over every
// limb; coefficient form: one launch per block of kParamBlock moduli.  In place, the polynomials are first copied into
// pool scratch (at most ~256 MiB at a time, whole polynomials) and permuted from there back into result.
int apply_galois_on_device(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                           uint64_t rns, uint64_t count, uint64_t galois_elt, bool ntt_form, cudaStream_t s) {
  const int log_n = floor_log2(n);
  const uint64_t g_inv = galois_inverse(galois_elt, n), unit = rns * n;
  auto permute = [&](uint64_t* r, const uint64_t* a, uint64_t polys) -> int {
    if (ntt_form) {
      cudaError_t e = launch_galois_ntt(r, a, log_n, polys * rns, galois_elt, s);
      if (e != cudaSuccess) return cuda_fail(e, "ApplyGalois launch");
      return 0;
    }
    for (uint64_t i0 = 0; i0 < rns; i0 += kParamBlock) {
      const uint64_t cnt = std::min<uint64_t>(kParamBlock, rns - i0);
      GaloisModuli mods;
      for (uint64_t e = 0; e < cnt; ++e) mods.q[e] = moduli[i0 + e];
      cudaError_t e = launch_galois_coef(r, a, log_n, rns, i0, cnt, polys, g_inv, mods, s);
      if (e != cudaSuccess) return cuda_fail(e, "ApplyGalois launch");
    }
    return 0;
  };
  if (result != operand) return permute(result, operand, count);
  const uint64_t chunk = std::min<uint64_t>(count, std::max<uint64_t>(1, (256ull << 20) / (unit * 8)));
  Scratch ws(s);
  uint64_t* copy = nullptr;
  if (int rc = ws.get(&copy, chunk * unit)) return rc;
  for (uint64_t p0 = 0; p0 < count; p0 += chunk) {
    const uint64_t cnt = std::min(chunk, count - p0);
    CU(cudaMemcpyAsync(copy, result + p0 * unit, cnt * unit * 8, cudaMemcpyDeviceToDevice, s));
    if (int rc = permute(result + p0 * unit, copy, cnt)) return rc;
  }
  return 0;  // ~Scratch returns the copy to the pool in stream order
}

// The rotation of one ciphertext (two components of decomp limbs in NTT form, device memory): sigma_g of both
// components into perm (2 x decomp x n words of scratch) in one launch, then c0 <- sigma_g(c0), c1 <- 0 by stream
// copies and the key switch of t_target = sigma_g(c1), which accumulates KS(sigma_g(c1)) into both components.
int galois_key_switch_on_device(int dev, uint64_t* ct, uint64_t* perm, uint64_t n, uint64_t decomp,
                                uint64_t key_modulus_size, uint64_t rns, const uint64_t* moduli,
                                const uint64_t* const* d_key_ptrs_host, const uint64_t* modswitch,
                                uint64_t galois_elt, cudaStream_t s) {
  const uint64_t comp = decomp * n;
  const cudaError_t e = launch_galois_ntt(perm, ct, floor_log2(n), 2 * decomp, galois_elt, s);
  if (e != cudaSuccess) return cuda_fail(e, "ApplyGaloisKeySwitch: automorphism launch");
  CU(cudaMemcpyAsync(ct, perm, comp * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
  CU(cudaMemsetAsync(ct + comp, 0, comp * sizeof(uint64_t), s));
  return key_switch_on_device(dev, ct, perm + comp, n, decomp, key_modulus_size, rns, 2, moduli, d_key_ptrs_host,
                              modswitch, s);
}

// The hoisted rotations of one ciphertext ct (device memory, as above) by num_elts elements: out + r * 2 * decomp * n
// gets [sigma_g(c0), 0] + ModDown(sum_j pi_g(D_j) K_r[j]) for g = galois_elts[r], with the digits D_j of c1 decomposed
// and transformed once for every element.  Per element: one automorphism launch over c0 straight into the output, a
// memset of the output's c1, then its multiply-accumulates and mod-down inside the shared key switch.
int hoisted_rotations_on_device(int dev, uint64_t* out, const uint64_t* ct, uint64_t n, uint64_t decomp,
                                uint64_t key_modulus_size, uint64_t rns, const uint64_t* moduli,
                                const uint64_t* const* const* d_key_ptrs, const uint64_t* galois_elts,
                                uint64_t num_elts, const uint64_t* modswitch, cudaStream_t s) {
  const uint64_t comp = decomp * n;
  std::vector<uint64_t*> results(num_elts);
  for (uint64_t r = 0; r < num_elts; ++r) {
    results[r] = out + r * 2 * comp;
    const cudaError_t e = launch_galois_ntt(results[r], ct, floor_log2(n), decomp, galois_elts[r], s);
    if (e != cudaSuccess) return cuda_fail(e, "ApplyGaloisKeySwitchHoisted: automorphism launch");
    CU(cudaMemsetAsync(results[r] + comp, 0, comp * sizeof(uint64_t), s));
  }
  return key_switch_elts_on_device(dev, results.data(), ct + comp, n, decomp, key_modulus_size, rns, 2, moduli,
                                   d_key_ptrs, galois_elts, num_elts, modswitch, s);
}

}  // namespace

// =============================================================== extern "C"
extern "C" {

int hexl_b200_apply_galois(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                           uint64_t rns_modulus_size, uint64_t count, uint64_t galois_elt, int ntt_form, void* stream) {
  REQUIRE(result && operand && moduli, "Require result, operand, moduli != nullptr");
  REQUIRE(rns_modulus_size >= 1, "Require rns_modulus_size >= 1");
  REQUIRE(ntt_form == 0 || ntt_form == 1, "Require ntt_form = 0 or 1");
  REQUIRE(n >= 2 && n <= (1ull << 20) && !(n & (n - 1)), "Require n a power of two in [2, 2^20]");
  const uint64_t rns = rns_modulus_size;
  for (uint64_t i = 0; i < rns; ++i)
    REQUIRE(moduli[i] > 1 && moduli[i] < (1ull << 62), "Require 1 < moduli[%llu] < 2^62", (unsigned long long)i);
  if (int rc = galois_elt_check(n, galois_elt)) return rc;
  if (count == 0) return 0;
  const uint64_t unit = rns * n, total = count * unit;
  REQUIRE(result == operand || result + total <= operand || operand + total <= result,
          "result and operand must be the same buffer or not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, operand}, &pi)) return rc;
  if (int rc = check_limb_bounds(operand, count, rns, n, [&](u64 i) { return moduli[i]; }, pi, "operand", stream)) return rc;
  const bool ntt = ntt_form != 0;
  if (pi.where == Where::Device)
    return run_on_device(pi, stream, [&] {
      return apply_galois_on_device(result, operand, n, moduli, rns, count, galois_elt, ntt, (cudaStream_t)stream);
    });
  // host pointers: whole polynomials through the staging slots (split over the host devices when set); the staged
  // polynomials are permuted in place on the device
  return run_host(result, operand, nullptr, total, unit, [&](int, u64, u64, auto&& run) {
    return run([&](u64* r, const u64* a, const u64*, u64, u64 elems, cudaStream_t s) {
      return apply_galois_on_device(r, a, n, moduli, rns, elems / unit, galois_elt, ntt, s);
    });
  });
}

int hexl_b200_apply_galois_key_switch(uint64_t* ciphertexts, uint64_t n, uint64_t decomp_modulus_size,
                                      uint64_t key_modulus_size, uint64_t rns_modulus_size,
                                      uint64_t key_component_count, const uint64_t* moduli,
                                      const hexl_b200_keys* galois_keys, const uint64_t* modswitch_factors,
                                      uint64_t galois_elt, uint64_t batch, void* stream) {
  const uint64_t decomp = decomp_modulus_size, rns = rns_modulus_size, kcc = key_component_count;
  if (int rc = key_switch_check(ciphertexts, ciphertexts, n, decomp, key_modulus_size, rns, kcc, moduli,
                                modswitch_factors))
    return rc;
  REQUIRE(kcc == 2, "Require key_component_count == 2 (a ciphertext of two components)");
  REQUIRE(n <= (1ull << 20), "Require n <= 2^20");
  if (int rc = galois_elt_check(n, galois_elt)) return rc;
  REQUIRE(galois_keys != nullptr, "Require galois_keys != nullptr");
  REQUIRE(keys_fit(galois_keys, n, decomp, kcc, key_modulus_size), "the key handle was uploaded for another shape");
  REQUIRE(galois_keys->shards.empty(),
          "ApplyGaloisKeySwitch does not take keys sharded by modulus: upload them with hexl_b200_keys_upload");
  if (batch == 0) return 0;
  PtrInfo pi;
  if (int rc = classify_all({ciphertexts}, &pi)) return rc;
  const uint64_t comp = decomp * n;
  if (int rc = check_limb_bounds(ciphertexts, 2 * batch, decomp, n, [&](u64 i) { return moduli[i]; }, pi,
                                 "ciphertexts", stream))
    return rc;
  // host pointers: only the ciphertext crosses PCIe, and the slot's second buffer holds both permuted components
  if (pi.where == Where::Host)
    return key_switch_host_batch(ciphertexts, 2 * comp, true, nullptr, 0, 2 * comp, &galois_keys, 1, batch,
                                 [&](int dev, uint64_t* d_ct, uint64_t* perm, const uint64_t* const* const* dk,
                                     cudaStream_t s) {
                                   return galois_key_switch_on_device(dev, d_ct, perm, n, decomp, key_modulus_size,
                                                                      rns, moduli, dk[0], modswitch_factors,
                                                                      galois_elt, s);
                                 });
  std::vector<const uint64_t* const*> dk;
  if (keys_on_device(&galois_keys, 1, pi.device, &dk) < 1)
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "the key handle holds no copy on the device of the ciphertexts");
  return run_on_device(pi, stream, [&] {
    Scratch ws((cudaStream_t)stream);
    uint64_t* perm = nullptr;
    if (int rc = ws.get(&perm, 2 * comp)) return rc;
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = galois_key_switch_on_device(pi.device, ciphertexts + c * 2 * comp, perm, n, decomp,
                                               key_modulus_size, rns, moduli, dk[0], modswitch_factors, galois_elt,
                                               (cudaStream_t)stream))
        return rc;
    return 0;
  });
}

int hexl_b200_apply_galois_key_switch_hoisted(uint64_t* results, const uint64_t* ciphertexts, uint64_t n,
                                              uint64_t decomp_modulus_size, uint64_t key_modulus_size,
                                              uint64_t rns_modulus_size, uint64_t key_component_count,
                                              const uint64_t* moduli, const hexl_b200_keys* const* galois_keys,
                                              const uint64_t* galois_elts, uint64_t num_elts,
                                              const uint64_t* modswitch_factors, uint64_t batch, void* stream) {
  const uint64_t decomp = decomp_modulus_size, rns = rns_modulus_size, kcc = key_component_count;
  if (int rc = key_switch_check(results, ciphertexts, n, decomp, key_modulus_size, rns, kcc, moduli,
                                modswitch_factors))
    return rc;
  REQUIRE(kcc == 2, "Require key_component_count == 2 (a ciphertext of two components)");
  REQUIRE(n <= (1ull << 20), "Require n <= 2^20");
  REQUIRE(num_elts == 0 || (galois_keys && galois_elts), "Require galois_keys, galois_elts != nullptr");
  for (uint64_t r = 0; r < num_elts; ++r) {
    if (int rc = galois_elt_check(n, galois_elts[r])) return rc;
    const hexl_b200_keys* k = galois_keys[r];
    REQUIRE(k != nullptr, "Require galois_keys[%llu] != nullptr", (unsigned long long)r);
    REQUIRE(keys_fit(k, n, decomp, kcc, key_modulus_size), "galois_keys[%llu] was uploaded for another shape",
            (unsigned long long)r);
    REQUIRE(k->shards.empty(),
            "ApplyGaloisKeySwitchHoisted does not take keys sharded by modulus: upload them with hexl_b200_keys_upload");
  }
  if (num_elts == 0 || batch == 0) return 0;
  const uint64_t comp = decomp * n, in_total = batch * 2 * comp, out_total = batch * num_elts * 2 * comp;
  REQUIRE(results + out_total <= ciphertexts || ciphertexts + in_total <= results,
          "results and ciphertexts must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({results, ciphertexts}, &pi)) return rc;
  if (int rc = check_limb_bounds(ciphertexts, 2 * batch, decomp, n, [&](u64 i) { return moduli[i]; }, pi,
                                 "ciphertexts", stream))
    return rc;
  // host pointers: each input ciphertext crosses PCIe in once and its num_elts rotations come back from the same slot
  if (pi.where == Where::Host)
    return key_switch_host_batch(results, num_elts * 2 * comp, false, ciphertexts, 2 * comp, 2 * comp, galois_keys,
                                 num_elts, batch,
                                 [&](int dev, uint64_t* d_res, uint64_t* d_ct, const uint64_t* const* const* dk,
                                     cudaStream_t s) {
                                   return hoisted_rotations_on_device(dev, d_res, d_ct, n, decomp, key_modulus_size,
                                                                      rns, moduli, dk, galois_elts, num_elts,
                                                                      modswitch_factors, s);
                                 });
  std::vector<const uint64_t* const*> dk;
  const uint64_t missing = keys_on_device(galois_keys, num_elts, pi.device, &dk);
  if (missing < num_elts)
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "galois_keys[%llu] holds no copy on the device of the ciphertexts",
                (unsigned long long)missing);
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = hoisted_rotations_on_device(pi.device, results + c * num_elts * 2 * comp, ciphertexts + c * 2 * comp,
                                               n, decomp, key_modulus_size, rns, moduli, dk.data(), galois_elts,
                                               num_elts, modswitch_factors, (cudaStream_t)stream))
        return rc;
    return 0;
  });
}

}  // extern "C"
