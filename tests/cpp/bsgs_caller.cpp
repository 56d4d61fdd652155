// A C++ caller of intel::hexl::b200::LinearTransformHybridBSGS through include/hexl/hexl.hpp, on host AlignedVector64
// buffers, digit size 2 and two special primes.  One identity giant over three babies (an identity baby and an absent
// pair included) must equal LinearTransformHybrid over the babies with the absent diagonal as a zero one; one identity
// baby under two keyed giants with diagonals of ones must equal LinearTransformHybrid over the giants.  Built without
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
  const uint64_t n = 1024, L = 4, K = 2, batch = 2, comp = L * n, nb = L + K;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(L + K, 50, true, n);
  uint64_t s = 2026;
  auto next = [&](uint64_t bound) {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    return (s >> 11) % bound;
  };
  // keys for digits of 2 moduli: 2 buffers of 2 x (L + K) x n
  std::vector<std::vector<AlignedVector64<uint64_t>>> keys(3);
  std::vector<std::vector<const uint64_t*>> ptrs(3);
  for (uint64_t r = 0; r < 3; ++r) {
    keys[r].assign(2, AlignedVector64<uint64_t>(2 * nb * n));
    for (auto& key : keys[r])
      for (uint64_t k = 0; k < 2; ++k)
        for (uint64_t i = 0; i < nb; ++i)
          for (uint64_t l = 0; l < n; ++l) key[(k * nb + i) * n + l] = next(q[i]);
    for (auto& key : keys[r]) ptrs[r].push_back(key.data());
  }
  const KeySwitchKeys h0(ptrs[0].data(), n, 2, nb, 2), h1(ptrs[1].data(), n, 2, nb, 2), h2(ptrs[2].data(), n, 2, nb, 2);
  AlignedVector64<uint64_t> ct(batch * 2 * comp);
  for (uint64_t c = 0; c < 2 * batch; ++c)
    for (uint64_t i = 0; i < L; ++i)
      for (uint64_t l = 0; l < n; ++l) ct[(c * L + i) * n + l] = next(q[i]);
  auto diagonals = [&](uint64_t count, bool ones) {
    AlignedVector64<uint64_t> w(count * nb * n);
    for (uint64_t r = 0; r < count; ++r)
      for (uint64_t i = 0; i < nb; ++i)
        for (uint64_t l = 0; l < n; ++l) w[(r * nb + i) * n + l] = ones ? 1 : next(q[i]);
    return w;
  };
  uint64_t wrong = 0;
  const KeySwitchKeys* none[1] = {nullptr};
  const uint64_t g1[1] = {1};

  // one identity giant: babies 3 (keyed), 1 (identity) and 5 (keyed, absent)
  const KeySwitchKeys* babies[3] = {&h0, nullptr, &h1};
  const uint64_t belts[3] = {3, 1, 5};
  AlignedVector64<uint64_t> w = diagonals(3, false);
  for (uint64_t k = 2 * nb * n; k < 3 * nb * n; ++k) w[k] = 0;
  const uint64_t* grid[3] = {w.data(), w.data() + nb * n, nullptr};
  AlignedVector64<uint64_t> a(batch * 2 * comp), b(batch * 2 * comp, 7);
  intel::hexl::b200::LinearTransformHybridBSGS(a.data(), ct.data(), n, L, L, K, 2, q.data(), babies, belts, 3, none,
                                               g1, 1, grid, false, batch);
  intel::hexl::b200::LinearTransformHybrid(b.data(), ct.data(), n, L, L, K, 2, q.data(), babies, belts, 3, w.data(),
                                           batch);
  for (uint64_t k = 0; k < a.size(); ++k) wrong += a[k] != b[k];

  // one identity baby under keyed giants 2n - 1 and 9, diagonals of ones
  const KeySwitchKeys* giants[2] = {&h2, &h0};
  const uint64_t gelts[2] = {2 * n - 1, 9};
  AlignedVector64<uint64_t> ones = diagonals(2, true);
  const uint64_t* column[2] = {ones.data(), ones.data() + nb * n};
  intel::hexl::b200::LinearTransformHybridBSGS(a.data(), ct.data(), n, L, L, K, 2, q.data(), none, g1, 1, giants,
                                               gelts, 2, column, false, batch);
  intel::hexl::b200::LinearTransformHybrid(b.data(), ct.data(), n, L, L, K, 2, q.data(), giants, gelts, 2, ones.data(),
                                           batch);
  for (uint64_t k = 0; k < a.size(); ++k) wrong += a[k] != b[k];

  // the rescale: 2 x (L - 1) limbs per ciphertext, every word below its modulus
  AlignedVector64<uint64_t> r(batch * 2 * (L - 1) * n, ~0ull);
  intel::hexl::b200::LinearTransformHybridBSGS(r.data(), ct.data(), n, L, L, K, 2, q.data(), babies, belts, 3, giants,
                                               gelts, 1, grid, true, batch);
  for (uint64_t k = 0; k < r.size(); ++k) wrong += r[k] >= q[(k / n) % (L - 1)];

  std::printf("bsgs_caller: %llu words differ\n", (unsigned long long)wrong);
  return wrong == 0 ? 0 : 1;
}
