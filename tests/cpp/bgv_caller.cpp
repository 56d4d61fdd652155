// A C++ caller of the BGV calls of intel::hexl::b200 through include/hexl/hexl.hpp, on host AlignedVector64 buffers.
// BgvMultiplyRelinearizeHybrid without the modulus switch must equal DyadicMultiply followed by BgvKeySwitchHybrid of
// d2 into (d0, d1) bit for bit; the hoisted rotation by 1 must equal BgvKeySwitchHybrid of c1 into (c0, 0); with the
// modulus switch, and after BgvModSwitch in place, every word must be below its modulus.  Built without arguments it
// only has to link; `run` calls the library (needs a GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "hexl/hexl.hpp"

using intel::hexl::AlignedVector64;
using intel::hexl::b200::KeySwitchKeys;

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1024, L = 4, K = 2, alpha = 2, batch = 2, comp = L * n, t = 65537;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(L + K, 50, true, n);
  uint64_t s = 2027;
  auto next = [&](uint64_t bound) {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    return (s >> 11) % bound;
  };
  std::vector<AlignedVector64<uint64_t>> keys((L + alpha - 1) / alpha, AlignedVector64<uint64_t>(2 * (L + K) * n));
  for (auto& key : keys)
    for (uint64_t k = 0; k < 2; ++k)
      for (uint64_t i = 0; i < L + K; ++i)
        for (uint64_t l = 0; l < n; ++l) key[(k * (L + K) + i) * n + l] = next(q[i]);
  std::vector<const uint64_t*> ptrs;
  for (auto& k : keys) ptrs.push_back(k.data());
  const KeySwitchKeys relin(ptrs.data(), n, keys.size(), L + K, 2);
  AlignedVector64<uint64_t> ct1(batch * 2 * comp), ct2(batch * 2 * comp);
  for (auto* ct : {&ct1, &ct2})
    for (uint64_t c = 0; c < 2 * batch; ++c)
      for (uint64_t i = 0; i < L; ++i)
        for (uint64_t l = 0; l < n; ++l) (*ct)[(c * L + i) * n + l] = next(q[i]);
  uint64_t wrong = 0;

  // mod_switch = 0 against the chain, and the hoisted rotation by 1 against the key switch of c1
  AlignedVector64<uint64_t> fused(batch * 2 * comp), rot(batch * 2 * comp);
  intel::hexl::b200::BgvMultiplyRelinearizeHybrid(fused.data(), ct1.data(), ct2.data(), n, L, L, K, alpha, q.data(), t,
                                                  relin, false, batch);
  const uint64_t one = 1;
  const KeySwitchKeys* gk[] = {&relin};
  intel::hexl::b200::BgvApplyGaloisKeySwitchHybridHoisted(rot.data(), ct1.data(), n, L, L, K, alpha, q.data(), t, gk,
                                                          &one, 1, batch);
  for (uint64_t c = 0; c < batch; ++c) {
    AlignedVector64<uint64_t> d(3 * comp);
    intel::hexl::DyadicMultiply(d.data(), ct1.data() + c * 2 * comp, ct2.data() + c * 2 * comp, n, q.data(), L);
    intel::hexl::b200::BgvKeySwitchHybrid(d.data(), d.data() + 2 * comp, n, L, L, K, alpha, 2, q.data(), t, relin);
    for (uint64_t k = 0; k < 2 * comp; ++k) wrong += fused[c * 2 * comp + k] != d[k];
    AlignedVector64<uint64_t> r(2 * comp, 0);
    std::memcpy(r.data(), ct1.data() + c * 2 * comp, comp * sizeof(uint64_t));
    intel::hexl::b200::BgvKeySwitchHybrid(r.data(), ct1.data() + c * 2 * comp + comp, n, L, L, K, alpha, 2, q.data(),
                                          t, relin);
    for (uint64_t k = 0; k < 2 * comp; ++k) wrong += rot[c * 2 * comp + k] != r[k];
  }

  // mod_switch = 1 and the modulus switch in place: canonical
  const uint64_t out = 2 * (L - 1) * n;
  AlignedVector64<uint64_t> sw(batch * out);
  intel::hexl::b200::BgvMultiplyRelinearizeHybrid(sw.data(), ct1.data(), ct1.data(), n, L, L, K, alpha, q.data(), t,
                                                  relin, true, batch);
  intel::hexl::b200::BgvModSwitch(ct2.data(), ct2.data(), n, q.data(), L, t, 2 * batch, true);
  for (uint64_t c = 0; c < 2 * batch; ++c)
    for (uint64_t i = 0; i < L - 1; ++i)
      for (uint64_t l = 0; l < n; ++l)
        wrong += sw[(c * (L - 1) + i) * n + l] >= q[i] || ct2[(c * L + i) * n + l] >= q[i];

  std::printf("bgv_caller: %llu words differ\n", (unsigned long long)wrong);
  return wrong == 0 ? 0 : 1;
}
