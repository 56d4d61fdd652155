// A C++ caller of intel::hexl::b200::BfvMultiply and BfvMultiplyRelinearizeHybrid through include/hexl/hexl.hpp, on
// host AlignedVector64 buffers.  The relinearized product must equal BfvMultiply, the forward transform of d2,
// KeySwitchHybrid, the inverse transform and the addition of (d0, d1) bit for bit; squaring one ciphertext must equal
// the product of two copies of it.  Built without arguments it only has to link; `run` calls the library (needs a GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "hexl/hexl.hpp"

using intel::hexl::AlignedVector64;
using intel::hexl::b200::KeySwitchKeys;

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1024, L = 3, K = 1, alpha = 1, batch = 2, comp = L * n, t = 65537;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(L + K, 55, true, n);
  // B = 3 primes, then m_sk, all in [2^60, 2^61)
  const std::vector<uint64_t> bsk = intel::hexl::GeneratePrimes(L + 1, 60, true, n);
  uint64_t s = 2027;
  auto next = [&](uint64_t bound) {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    return (s >> 11) % bound;
  };
  std::vector<AlignedVector64<uint64_t>> keys(L, AlignedVector64<uint64_t>(2 * (L + K) * n));
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

  AlignedVector64<uint64_t> d(batch * 3 * comp), fused(batch * 2 * comp);
  intel::hexl::b200::BfvMultiply(d.data(), ct1.data(), ct2.data(), n, q.data(), L, bsk.data(), L, bsk[L], t, batch);
  intel::hexl::b200::BfvMultiplyRelinearizeHybrid(fused.data(), ct1.data(), ct2.data(), n, L, L, K, alpha, q.data(),
                                                  bsk.data(), L, bsk[L], t, relin, batch);
  std::vector<intel::hexl::NTT> ntts;
  for (uint64_t i = 0; i < L; ++i) ntts.emplace_back(n, q[i]);
  for (uint64_t c = 0; c < batch; ++c) {
    const uint64_t* dc = d.data() + c * 3 * comp;
    AlignedVector64<uint64_t> t2(comp), ks(2 * comp, 0);
    for (uint64_t i = 0; i < L; ++i) ntts[i].ComputeForward(t2.data() + i * n, dc + (2 * L + i) * n, 1, 1);
    intel::hexl::b200::KeySwitchHybrid(ks.data(), t2.data(), n, L, L, K, alpha, 2, q.data(), relin);
    for (uint64_t k = 0; k < 2; ++k)
      for (uint64_t i = 0; i < L; ++i) {
        uint64_t* x = ks.data() + (k * L + i) * n;
        ntts[i].ComputeInverse(x, x, 1, 1);
        intel::hexl::EltwiseAddMod(x, x, dc + (k * L + i) * n, n, q[i]);
      }
    for (uint64_t k = 0; k < 2 * comp; ++k) wrong += fused[c * 2 * comp + k] != ks[k];
  }

  AlignedVector64<uint64_t> sq(batch * 3 * comp), copies(batch * 3 * comp, 1);
  const AlignedVector64<uint64_t> copy = ct1;
  intel::hexl::b200::BfvMultiply(sq.data(), ct1.data(), ct1.data(), n, q.data(), L, bsk.data(), L, bsk[L], t, batch);
  intel::hexl::b200::BfvMultiply(copies.data(), ct1.data(), copy.data(), n, q.data(), L, bsk.data(), L, bsk[L], t,
                                 batch);
  for (uint64_t k = 0; k < batch * 3 * comp; ++k) wrong += sq[k] != copies[k];

  std::printf("bfv_caller: %llu words differ\n", (unsigned long long)wrong);
  return wrong == 0 ? 0 : 1;
}
