// A C++ caller of intel::hexl::b200::KeySwitchHybrid and FastBaseConvert through include/hexl/hexl.hpp, on host
// AlignedVector64 buffers.  With digit size 1 and one special prime the hybrid switch of two ciphertexts must equal
// KeySwitch on resident keys bit for bit; with digit size 2 and two special primes it must equal two calls of one
// ciphertext each; and a base conversion into the source moduli themselves must return its input.  Built without
// arguments it only has to link; `run` calls the library (needs a GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "hexl/hexl.hpp"

using intel::hexl::AlignedVector64;
using intel::hexl::b200::KeySwitchKeys;

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1024, L = 4, kcc = 2, batch = 2;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(L + 2, 50, true, n);
  uint64_t s = 2024;
  auto next = [&](uint64_t bound) {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    return (s >> 11) % bound;
  };
  // keys for K special primes and digits of alpha moduli: ceil(L / alpha) buffers of kcc x (L + K) x n
  auto make_keys = [&](const std::vector<uint64_t>& mods, uint64_t alpha) {
    std::vector<AlignedVector64<uint64_t>> keys((L + alpha - 1) / alpha,
                                                AlignedVector64<uint64_t>(kcc * mods.size() * n));
    for (auto& key : keys)
      for (uint64_t k = 0; k < kcc; ++k)
        for (uint64_t i = 0; i < mods.size(); ++i)
          for (uint64_t l = 0; l < n; ++l) key[(k * mods.size() + i) * n + l] = next(mods[i]);
    return keys;
  };
  auto pointers = [](const std::vector<AlignedVector64<uint64_t>>& keys) {
    std::vector<const uint64_t*> p;
    for (auto& k : keys) p.push_back(k.data());
    return p;
  };
  AlignedVector64<uint64_t> target(batch * L * n), result(batch * kcc * L * n);
  for (uint64_t c = 0; c < batch; ++c)
    for (uint64_t i = 0; i < L; ++i)
      for (uint64_t l = 0; l < n; ++l) target[(c * L + i) * n + l] = next(q[i]);
  for (uint64_t c = 0; c < batch * kcc; ++c)
    for (uint64_t i = 0; i < L; ++i)
      for (uint64_t l = 0; l < n; ++l) result[(c * L + i) * n + l] = next(q[i]);
  uint64_t wrong = 0;

  // alpha = 1, K = 1 against KeySwitch on resident keys
  const std::vector<uint64_t> q1(q.begin(), q.begin() + L + 1);
  const auto keys1 = make_keys(q1, 1);
  auto ptrs1 = pointers(keys1);
  const KeySwitchKeys h1(ptrs1.data(), n, L, L + 1, kcc);
  std::vector<uint64_t> modswitch(L);
  for (uint64_t i = 0; i < L; ++i) modswitch[i] = intel::hexl::InverseMod(q1[L] % q[i], q[i]);
  AlignedVector64<uint64_t> hybrid = result, resident = result;
  intel::hexl::b200::KeySwitchHybrid(hybrid.data(), target.data(), n, L, L, 1, 1, kcc, q1.data(), h1, batch);
  intel::hexl::KeySwitch(resident.data(), target.data(), n, L, L + 1, L + 1, kcc, q1.data(), h1, modswitch.data(),
                         batch);
  for (uint64_t k = 0; k < hybrid.size(); ++k) wrong += hybrid[k] != resident[k];

  // alpha = 2, K = 2: a batch of two equals two single calls
  const auto keys2 = make_keys(q, 2);
  auto ptrs2 = pointers(keys2);
  const KeySwitchKeys h2(ptrs2.data(), n, keys2.size(), L + 2, kcc);
  AlignedVector64<uint64_t> both = result, one = result;
  intel::hexl::b200::KeySwitchHybrid(both.data(), target.data(), n, L, L, 2, 2, kcc, q.data(), h2, batch);
  for (uint64_t c = 0; c < batch; ++c)
    intel::hexl::b200::KeySwitchHybrid(one.data() + c * kcc * L * n, target.data() + c * L * n, n, L, L, 2, 2, kcc,
                                       q.data(), h2);
  for (uint64_t k = 0; k < both.size(); ++k) wrong += both[k] != one[k];

  // a base conversion into the source moduli returns the input
  AlignedVector64<uint64_t> back(target.size());
  intel::hexl::b200::FastBaseConvert(back.data(), target.data(), n, q.data(), L, q.data(), L, batch);
  for (uint64_t k = 0; k < back.size(); ++k) wrong += back[k] != target[k];

  std::printf("hybrid_caller: %llu words differ\n", (unsigned long long)wrong);
  return wrong == 0 ? 0 : 1;
}
