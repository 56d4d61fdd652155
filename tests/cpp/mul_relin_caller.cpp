// A C++ caller of intel::hexl::b200::MultiplyRelinearizeHybrid through include/hexl/hexl.hpp, on host AlignedVector64
// buffers.  Without rescale the product of two pairs must equal DyadicMultiply followed by KeySwitchHybrid of d2 into
// (d0, d1) bit for bit; with rescale every word must be below its modulus and squaring one ciphertext must equal the
// product of two copies of it.  Built without arguments it only has to link; `run` calls the library (needs a GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "hexl/hexl.hpp"

using intel::hexl::AlignedVector64;
using intel::hexl::b200::KeySwitchKeys;

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1024, L = 4, K = 2, alpha = 2, batch = 2, comp = L * n;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(L + K, 50, true, n);
  uint64_t s = 2026;
  auto next = [&](uint64_t bound) {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    return (s >> 11) % bound;
  };
  // relinearization keys: ceil(L / alpha) buffers of 2 x (L + K) x n
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

  // rescale = 0 against the chain, pair by pair
  AlignedVector64<uint64_t> fused(batch * 2 * comp);
  intel::hexl::b200::MultiplyRelinearizeHybrid(fused.data(), ct1.data(), ct2.data(), n, L, L, K, alpha, q.data(), relin,
                                               false, batch);
  for (uint64_t c = 0; c < batch; ++c) {
    AlignedVector64<uint64_t> d(3 * comp);
    intel::hexl::DyadicMultiply(d.data(), ct1.data() + c * 2 * comp, ct2.data() + c * 2 * comp, n, q.data(), L);
    intel::hexl::b200::KeySwitchHybrid(d.data(), d.data() + 2 * comp, n, L, L, K, alpha, 2, q.data(), relin);
    for (uint64_t k = 0; k < 2 * comp; ++k) wrong += fused[c * 2 * comp + k] != d[k];
  }

  // rescale = 1: canonical, and squaring equals the product of two copies
  const uint64_t out = 2 * (L - 1) * n;
  AlignedVector64<uint64_t> sq(batch * out), copies(batch * out, 1);
  const AlignedVector64<uint64_t> copy = ct1;
  intel::hexl::b200::MultiplyRelinearizeHybrid(sq.data(), ct1.data(), ct1.data(), n, L, L, K, alpha, q.data(), relin,
                                               true, batch);
  intel::hexl::b200::MultiplyRelinearizeHybrid(copies.data(), ct1.data(), copy.data(), n, L, L, K, alpha, q.data(),
                                               relin, true, batch);
  for (uint64_t c = 0; c < 2 * batch; ++c)
    for (uint64_t i = 0; i < L - 1; ++i)
      for (uint64_t l = 0; l < n; ++l) {
        const uint64_t k = (c * (L - 1) + i) * n + l;
        wrong += sq[k] != copies[k] || sq[k] >= q[i];
      }

  std::printf("mul_relin_caller: %llu words differ\n", (unsigned long long)wrong);
  return wrong == 0 ? 0 : 1;
}
