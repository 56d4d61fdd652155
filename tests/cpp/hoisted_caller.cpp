// A C++ caller of intel::hexl::b200::ApplyGaloisKeySwitchHoisted through include/hexl/hexl.hpp, on host
// AlignedVector64 buffers.  Two ciphertexts are rotated by the elements {1, 5, 1} with two key handles in one call.
// The outputs for g = 1 must equal ApplyGaloisKeySwitch with g = 1 bit for bit, the output for g = 5 must equal a
// hoisted call with {5} alone, and the input must come back unchanged.  Built without arguments it only has to link;
// `run` calls the library (needs a GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "hexl/hexl.hpp"

using intel::hexl::AlignedVector64;
using intel::hexl::b200::KeySwitchKeys;

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1024, decomp = 3, kms = decomp + 1, kcc = 2, batch = 2, comp = decomp * n, per = kcc * comp;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(kms, 50, true, n);
  uint64_t s = 2024;
  auto next = [&](uint64_t bound) {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    return (s >> 11) % bound;
  };
  std::vector<std::vector<AlignedVector64<uint64_t>>> keys(2, std::vector<AlignedVector64<uint64_t>>(
                                                                  decomp, AlignedVector64<uint64_t>(kcc * kms * n)));
  for (auto& set : keys)
    for (auto& key : set)
      for (uint64_t k = 0; k < kcc; ++k)
        for (uint64_t i = 0; i < kms; ++i)
          for (uint64_t l = 0; l < n; ++l) key[(k * kms + i) * n + l] = next(q[i]);
  std::vector<const uint64_t*> ptrs0, ptrs1;
  for (uint64_t j = 0; j < decomp; ++j) {
    ptrs0.push_back(keys[0][j].data());
    ptrs1.push_back(keys[1][j].data());
  }
  KeySwitchKeys h1(ptrs0.data(), n, decomp, kms, kcc), h5(ptrs1.data(), n, decomp, kms, kcc);
  std::vector<uint64_t> modswitch(decomp);
  for (uint64_t i = 0; i < decomp; ++i) modswitch[i] = intel::hexl::InverseMod(q[kms - 1] % q[i], q[i]);
  AlignedVector64<uint64_t> ct(batch * per);
  for (uint64_t c = 0; c < batch * kcc; ++c)
    for (uint64_t i = 0; i < decomp; ++i)
      for (uint64_t l = 0; l < n; ++l) ct[(c * decomp + i) * n + l] = next(q[i]);
  const AlignedVector64<uint64_t> input = ct;

  const uint64_t elts[] = {1, 5, 1}, five[] = {5};
  const KeySwitchKeys* handles[] = {&h1, &h5, &h1};
  const KeySwitchKeys* handle5[] = {&h5};
  AlignedVector64<uint64_t> out(batch * 3 * per), alone(batch * per);
  intel::hexl::b200::ApplyGaloisKeySwitchHoisted(out.data(), ct.data(), n, decomp, kms, kms, kcc, q.data(), handles,
                                                 elts, 3, modswitch.data(), batch);
  intel::hexl::b200::ApplyGaloisKeySwitchHoisted(alone.data(), ct.data(), n, decomp, kms, kms, kcc, q.data(), handle5,
                                                 five, 1, modswitch.data(), batch);
  const bool input_kept = std::memcmp(ct.data(), input.data(), ct.size() * 8) == 0;
  intel::hexl::ApplyGaloisKeySwitch(ct.data(), n, decomp, kms, kms, kcc, q.data(), h1, modswitch.data(), 1, batch);
  uint64_t wrong = 0;
  for (uint64_t c = 0; c < batch; ++c)
    for (uint64_t k = 0; k < per; ++k) {
      const uint64_t* o = &out[c * 3 * per];
      wrong += (o[k] != ct[c * per + k]) + (o[2 * per + k] != ct[c * per + k]) + (o[per + k] != alone[c * per + k]);
    }
  std::printf("hoisted_caller: %llu of %zu words differ; input %s\n", (unsigned long long)wrong, out.size(),
              input_kept ? "unchanged" : "CHANGED");
  return wrong == 0 && input_kept ? 0 : 1;
}
