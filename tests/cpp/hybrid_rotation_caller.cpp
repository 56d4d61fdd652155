// A C++ caller of intel::hexl::b200::ApplyGaloisKeySwitchHybridHoisted and LinearTransformHybrid through
// include/hexl/hexl.hpp, on host AlignedVector64 buffers.  With digit size 1 and one special prime the hoisted hybrid
// rotations of two ciphertexts must equal ApplyGaloisKeySwitchHoisted bit for bit; with digit size 2 and two special
// primes the linear transform of one element with a diagonal of ones must equal the hoisted call, and an identity term
// alone (no key) must weight the ciphertext by its diagonal.  Built without arguments it only has to link; `run` calls
// the library (needs a GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "hexl/hexl.hpp"

using intel::hexl::AlignedVector64;
using intel::hexl::b200::KeySwitchKeys;

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1024, L = 4, batch = 2, comp = L * n;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(L + 2, 50, true, n);
  uint64_t s = 2025;
  auto next = [&](uint64_t bound) {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    return (s >> 11) % bound;
  };
  // keys for K special primes and digits of alpha moduli: ceil(L / alpha) buffers of 2 x (L + K) x n
  auto make_keys = [&](const std::vector<uint64_t>& mods, uint64_t alpha) {
    std::vector<AlignedVector64<uint64_t>> keys((L + alpha - 1) / alpha, AlignedVector64<uint64_t>(2 * mods.size() * n));
    for (auto& key : keys)
      for (uint64_t k = 0; k < 2; ++k)
        for (uint64_t i = 0; i < mods.size(); ++i)
          for (uint64_t l = 0; l < n; ++l) key[(k * mods.size() + i) * n + l] = next(mods[i]);
    return keys;
  };
  auto pointers = [](const std::vector<AlignedVector64<uint64_t>>& keys) {
    std::vector<const uint64_t*> p;
    for (auto& k : keys) p.push_back(k.data());
    return p;
  };
  AlignedVector64<uint64_t> ct(batch * 2 * comp);
  for (uint64_t c = 0; c < 2 * batch; ++c)
    for (uint64_t i = 0; i < L; ++i)
      for (uint64_t l = 0; l < n; ++l) ct[(c * L + i) * n + l] = next(q[i]);
  uint64_t wrong = 0;

  // alpha = 1, K = 1 against the SEAL-shaped hoisted rotations
  const std::vector<uint64_t> q1(q.begin(), q.begin() + L + 1);
  const auto keys1 = make_keys(q1, 1);
  auto ptrs1 = pointers(keys1);
  const KeySwitchKeys h1(ptrs1.data(), n, L, L + 1, 2);
  const KeySwitchKeys* handles1[2] = {&h1, &h1};
  const uint64_t elts[2] = {3, 2 * n - 1};
  std::vector<uint64_t> modswitch(L);
  for (uint64_t i = 0; i < L; ++i) modswitch[i] = intel::hexl::InverseMod(q1[L] % q[i], q[i]);
  AlignedVector64<uint64_t> hybrid(batch * 2 * 2 * comp), seal(batch * 2 * 2 * comp, 1);
  intel::hexl::b200::ApplyGaloisKeySwitchHybridHoisted(hybrid.data(), ct.data(), n, L, L, 1, 1, q1.data(), handles1,
                                                       elts, 2, batch);
  intel::hexl::b200::ApplyGaloisKeySwitchHoisted(seal.data(), ct.data(), n, L, L + 1, L + 1, 2, q1.data(), handles1,
                                                 elts, 2, modswitch.data(), batch);
  for (uint64_t k = 0; k < hybrid.size(); ++k) wrong += hybrid[k] != seal[k];

  // alpha = 2, K = 2: one element with a unit diagonal equals the hoisted call
  const auto keys2 = make_keys(q, 2);
  auto ptrs2 = pointers(keys2);
  const KeySwitchKeys h2(ptrs2.data(), n, keys2.size(), L + 2, 2);
  const KeySwitchKeys* handles2[1] = {&h2};
  const uint64_t g5[1] = {5};
  AlignedVector64<uint64_t> ones((L + 2) * n, 1), rot(batch * 2 * comp), lin(batch * 2 * comp, 7);
  intel::hexl::b200::ApplyGaloisKeySwitchHybridHoisted(rot.data(), ct.data(), n, L, L, 2, 2, q.data(), handles2, g5, 1,
                                                       batch);
  intel::hexl::b200::LinearTransformHybrid(lin.data(), ct.data(), n, L, L, 2, 2, q.data(), handles2, g5, 1,
                                           ones.data(), batch);
  for (uint64_t k = 0; k < rot.size(); ++k) wrong += rot[k] != lin[k];

  // an identity term alone: w (.) ct, no key switch
  const KeySwitchKeys* none[1] = {nullptr};
  const uint64_t g1[1] = {1};
  AlignedVector64<uint64_t> w((L + 2) * n), id(batch * 2 * comp);
  for (uint64_t i = 0; i < L + 2; ++i)
    for (uint64_t l = 0; l < n; ++l) w[i * n + l] = next(q[i]);
  intel::hexl::b200::LinearTransformHybrid(id.data(), ct.data(), n, L, L, 2, 2, q.data(), none, g1, 1, w.data(),
                                           batch);
  for (uint64_t c = 0; c < 2 * batch; ++c)
    for (uint64_t i = 0; i < L; ++i)
      for (uint64_t l = 0; l < n; ++l) {
        const uint64_t k = (c * L + i) * n + l;
        wrong += id[k] != intel::hexl::MultiplyMod(w[i * n + l], ct[k], q[i]);
      }

  std::printf("hybrid_rotation_caller: %llu words differ\n", (unsigned long long)wrong);
  return wrong == 0 ? 0 : 1;
}
