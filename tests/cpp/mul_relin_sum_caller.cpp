// A C++ caller of intel::hexl::b200::MultiplyRelinearizeSumHybrid through include/hexl/hexl.hpp, on host AlignedVector64
// buffers.  Two outputs of three pairs each, the second output reusing the first's ciphertexts and squaring one.
// Without rescale each output must equal DyadicMultiply of every pair, the sums with EltwiseAddMod, then
// KeySwitchHybrid of the summed d2 into the summed (d0, d1), bit for bit; with rescale one pair per output must equal
// MultiplyRelinearizeHybrid bit for bit.  Built without arguments it only has to link; `run` calls the library (needs
// a GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "hexl/hexl.hpp"

using intel::hexl::AlignedVector64;
using intel::hexl::b200::KeySwitchKeys;

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1024, L = 4, K = 2, alpha = 2, pairs = 3, batch = 2, comp = L * n;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(L + K, 50, true, n);
  uint64_t s = 2027;
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
  std::vector<AlignedVector64<uint64_t>> cts(5, AlignedVector64<uint64_t>(2 * comp));
  for (auto& ct : cts)
    for (uint64_t c = 0; c < 2; ++c)
      for (uint64_t i = 0; i < L; ++i)
        for (uint64_t l = 0; l < n; ++l) ct[(c * L + i) * n + l] = next(q[i]);
  // output 0: (0, 1), (2, 3), (4, 0); output 1: (1, 1), (2, 3), (0, 4)
  const int i1[batch * pairs] = {0, 2, 4, 1, 2, 0}, i2[batch * pairs] = {1, 3, 0, 1, 3, 4};
  std::vector<const uint64_t*> a, b;
  for (uint64_t x = 0; x < batch * pairs; ++x) {
    a.push_back(cts[i1[x]].data());
    b.push_back(cts[i2[x]].data());
  }
  uint64_t wrong = 0;

  // rescale = 0 against the chain, output by output
  AlignedVector64<uint64_t> fused(batch * 2 * comp);
  intel::hexl::b200::MultiplyRelinearizeSumHybrid(fused.data(), a.data(), b.data(), pairs, n, L, L, K, alpha, q.data(),
                                                  relin, false, batch);
  for (uint64_t c = 0; c < batch; ++c) {
    AlignedVector64<uint64_t> acc(3 * comp), d(3 * comp);
    intel::hexl::DyadicMultiply(acc.data(), a[c * pairs], b[c * pairs], n, q.data(), L);
    for (uint64_t r = 1; r < pairs; ++r) {
      intel::hexl::DyadicMultiply(d.data(), a[c * pairs + r], b[c * pairs + r], n, q.data(), L);
      for (uint64_t k = 0; k < 3; ++k)
        for (uint64_t i = 0; i < L; ++i)
          intel::hexl::EltwiseAddMod(acc.data() + (k * L + i) * n, acc.data() + (k * L + i) * n,
                                     d.data() + (k * L + i) * n, n, q[i]);
    }
    intel::hexl::b200::KeySwitchHybrid(acc.data(), acc.data() + 2 * comp, n, L, L, K, alpha, 2, q.data(), relin);
    for (uint64_t k = 0; k < 2 * comp; ++k) wrong += fused[c * 2 * comp + k] != acc[k];
  }

  // rescale = 1, one pair per output: MultiplyRelinearizeHybrid
  const uint64_t out = 2 * (L - 1) * n;
  AlignedVector64<uint64_t> one(batch * out), single(batch * out, 1), x1(batch * 2 * comp), x2(batch * 2 * comp);
  const uint64_t* a1[batch] = {a[0], a[1]};
  const uint64_t* b1[batch] = {b[0], b[1]};
  for (uint64_t c = 0; c < batch; ++c) {
    std::memcpy(x1.data() + c * 2 * comp, a1[c], 2 * comp * sizeof(uint64_t));
    std::memcpy(x2.data() + c * 2 * comp, b1[c], 2 * comp * sizeof(uint64_t));
  }
  intel::hexl::b200::MultiplyRelinearizeSumHybrid(one.data(), a1, b1, 1, n, L, L, K, alpha, q.data(), relin, true,
                                                  batch);
  intel::hexl::b200::MultiplyRelinearizeHybrid(single.data(), x1.data(), x2.data(), n, L, L, K, alpha, q.data(), relin,
                                               true, batch);
  for (uint64_t k = 0; k < batch * out; ++k) wrong += one[k] != single[k];

  std::printf("mul_relin_sum_caller: %llu words differ\n", (unsigned long long)wrong);
  return wrong == 0 ? 0 : 1;
}
