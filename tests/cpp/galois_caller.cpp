// A C++ caller of intel::hexl::ApplyGalois and ApplyGaloisKeySwitch through include/hexl/hexl.hpp, on host
// AlignedVector64 buffers.  ApplyGalois runs in coefficient form (out of place) and NTT form (in place) on two
// polynomials of three limbs; every word is checked against a loop of the definition.  ApplyGaloisKeySwitch rotates
// two ciphertexts with a KeySwitchKeys handle and is checked against the same rotation chained from ApplyGalois and
// KeySwitch.  Built without arguments it only has to link; `run` calls the library (needs a GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "hexl/hexl.hpp"

using intel::hexl::AlignedVector64;

static uint64_t rev(uint64_t x, int bits) {
  uint64_t r = 0;
  for (int b = 0; b < bits; ++b) r |= ((x >> b) & 1) << (bits - 1 - b);
  return r;
}

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1024, log_n = 10, rns = 3, count = 2, g = 5;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(rns, 50, true, n);
  AlignedVector64<uint64_t> a(count * rns * n), coef(a.size()), ntt(a.size()), want_coef(a.size()), want_ntt(a.size());
  uint64_t s = 2024;
  for (uint64_t p = 0; p < count; ++p)
    for (uint64_t i = 0; i < rns; ++i)
      for (uint64_t l = 0; l < n; ++l) {
        s = s * 6364136223846793005ull + 1442695040888963407ull;
        const uint64_t v = l % 7 == 0 ? 0 : (s >> 11) % q[i];
        const uint64_t base = (p * rns + i) * n;
        a[base + l] = v;
        const uint64_t k = l * g % (2 * n);  // coefficient form: X^l -> X^(l g), X^n = -1
        if (k < n) want_coef[base + k] = v;
        else want_coef[base + k - n] = v ? q[i] - v : 0;
      }
  // NTT form: slot j reads slot pi_g(j)
  for (uint64_t p = 0; p < count; ++p)
    for (uint64_t i = 0; i < rns; ++i)
      for (uint64_t j = 0; j < n; ++j) {
        const uint64_t k = g * (2 * rev(j, log_n) + 1) % (2 * n);
        const uint64_t base = (p * rns + i) * n;
        want_ntt[base + j] = a[base + rev((k - 1) / 2, log_n)];
      }
  intel::hexl::ApplyGalois(coef.data(), a.data(), n, q.data(), rns, count, g, false);
  ntt = a;
  intel::hexl::ApplyGalois(ntt.data(), ntt.data(), n, q.data(), rns, count, g, true);
  uint64_t wrong = 0;
  for (size_t k = 0; k < a.size(); ++k) wrong += (coef[k] != want_coef[k]) + (ntt[k] != want_ntt[k]);
  std::printf("galois_caller: ApplyGalois: %llu of %zu words differ\n", (unsigned long long)wrong, 2 * a.size());

  // rotation: decomp = 2 digits + the special prime, random keys; two ciphertexts of 2 x 2 limbs
  const uint64_t decomp = 2, kms = rns, kcc = 2, batch = 2, comp = decomp * n;
  std::vector<AlignedVector64<uint64_t>> keys(decomp, AlignedVector64<uint64_t>(kcc * kms * n));
  for (auto& key : keys)
    for (uint64_t k = 0; k < kcc; ++k)
      for (uint64_t i = 0; i < kms; ++i)
        for (uint64_t l = 0; l < n; ++l) {
          s = s * 6364136223846793005ull + 1442695040888963407ull;
          key[(k * kms + i) * n + l] = (s >> 11) % q[i];
        }
  std::vector<const uint64_t*> key_ptrs = {keys[0].data(), keys[1].data()};
  std::vector<uint64_t> modswitch(decomp);
  for (uint64_t i = 0; i < decomp; ++i) modswitch[i] = intel::hexl::InverseMod(q[kms - 1] % q[i], q[i]);
  AlignedVector64<uint64_t> ct(batch * kcc * comp);
  for (uint64_t c = 0; c < batch * kcc; ++c)
    for (uint64_t i = 0; i < decomp; ++i)
      for (uint64_t l = 0; l < n; ++l) {
        s = s * 6364136223846793005ull + 1442695040888963407ull;
        ct[(c * decomp + i) * n + l] = (s >> 11) % q[i];
      }
  intel::hexl::b200::KeySwitchKeys handle(key_ptrs.data(), n, decomp, kms, kcc);
  // the chain: sigma of both components, r = [sigma(c0), 0], KeySwitch(r, sigma(c1))
  AlignedVector64<uint64_t> perm(ct.size()), chained(ct.size(), 0), digits(batch * comp);
  intel::hexl::ApplyGalois(perm.data(), ct.data(), n, q.data(), decomp, batch * kcc, g, true);
  for (uint64_t c = 0; c < batch; ++c) {
    std::memcpy(&chained[c * kcc * comp], &perm[c * kcc * comp], comp * 8);
    std::memcpy(&digits[c * comp], &perm[(c * kcc + 1) * comp], comp * 8);
  }
  intel::hexl::KeySwitch(chained.data(), digits.data(), n, decomp, kms, decomp + 1, kcc, q.data(), handle,
                         modswitch.data(), batch);
  intel::hexl::ApplyGaloisKeySwitch(ct.data(), n, decomp, kms, decomp + 1, kcc, q.data(), handle, modswitch.data(), g,
                                    batch);
  uint64_t wrong_ks = 0;
  for (size_t k = 0; k < ct.size(); ++k) wrong_ks += ct[k] != chained[k];
  std::printf("galois_caller: ApplyGaloisKeySwitch: %llu of %zu words differ from the chain\n",
              (unsigned long long)wrong_ks, ct.size());
  return wrong == 0 && wrong_ks == 0 ? 0 : 1;
}
