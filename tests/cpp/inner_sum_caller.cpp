// A C++ caller of intel::hexl::b200::InnerSumHybrid through include/hexl/hexl.hpp, on host AlignedVector64 buffers,
// digit size 2 and two special primes, with a key table of the powers 3, 9 and 81 of g = 3 and an unused element.
// k = 2 must equal LinearTransformHybrid over {1, g} with unit diagonals, and k = 4 LinearTransformHybridBSGS over
// babies {1, g} and giants {1, g^2} with unit diagonals; with the rescale every word of 2 x (L - 1) limbs is below its
// modulus, and a missing key throws.  Built without arguments it only has to link; `run` calls the library (needs a
// GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <vector>

#include "hexl/hexl.hpp"

using intel::hexl::AlignedVector64;
using intel::hexl::b200::KeySwitchKeys;

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1024, L = 4, K = 2, batch = 2, comp = L * n, nb = L + K, g = 3;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(L + K, 50, true, n);
  uint64_t s = 2027;
  auto next = [&](uint64_t bound) {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    return (s >> 11) % bound;
  };
  // four key sets for digits of 2 moduli: 2 buffers of 2 x (L + K) x n
  std::vector<std::vector<AlignedVector64<uint64_t>>> keys(4);
  std::vector<std::vector<const uint64_t*>> ptrs(4);
  for (uint64_t r = 0; r < 4; ++r) {
    keys[r].assign(2, AlignedVector64<uint64_t>(2 * nb * n));
    for (auto& key : keys[r])
      for (uint64_t k = 0; k < 2; ++k)
        for (uint64_t i = 0; i < nb; ++i)
          for (uint64_t l = 0; l < n; ++l) key[(k * nb + i) * n + l] = next(q[i]);
    for (auto& key : keys[r]) ptrs[r].push_back(key.data());
  }
  const KeySwitchKeys h0(ptrs[0].data(), n, 2, nb, 2), h1(ptrs[1].data(), n, 2, nb, 2), h2(ptrs[2].data(), n, 2, nb, 2),
      h3(ptrs[3].data(), n, 2, nb, 2);
  const KeySwitchKeys* table[4] = {&h3, &h0, &h1, &h2};
  const uint64_t elts[4] = {5, g, g * g, g * g * g * g % (2 * n)};
  AlignedVector64<uint64_t> ct(batch * 2 * comp);
  for (uint64_t c = 0; c < 2 * batch; ++c)
    for (uint64_t i = 0; i < L; ++i)
      for (uint64_t l = 0; l < n; ++l) ct[(c * L + i) * n + l] = next(q[i]);
  AlignedVector64<uint64_t> ones(2 * nb * n, 1);
  uint64_t wrong = 0;

  // k = 2: the linear transform over {1, g}
  AlignedVector64<uint64_t> a(batch * 2 * comp), b(batch * 2 * comp, 7);
  intel::hexl::b200::InnerSumHybrid(a.data(), ct.data(), n, L, L, K, 2, q.data(), g, 2, table, elts, 4, false, batch);
  const KeySwitchKeys* lt_keys[2] = {nullptr, &h0};
  const uint64_t lt_elts[2] = {1, g};
  intel::hexl::b200::LinearTransformHybrid(b.data(), ct.data(), n, L, L, K, 2, q.data(), lt_keys, lt_elts, 2,
                                           ones.data(), batch);
  for (uint64_t k = 0; k < a.size(); ++k) wrong += a[k] != b[k];

  // k = 4: BSGS over babies {1, g} and giants {1, g^2}
  intel::hexl::b200::InnerSumHybrid(a.data(), ct.data(), n, L, L, K, 2, q.data(), g, 4, table, elts, 4, false, batch);
  const KeySwitchKeys* giants[2] = {nullptr, &h1};
  const uint64_t gelts[2] = {1, g * g};
  const uint64_t* grid[4] = {ones.data(), ones.data(), ones.data(), ones.data()};
  intel::hexl::b200::LinearTransformHybridBSGS(b.data(), ct.data(), n, L, L, K, 2, q.data(), lt_keys, lt_elts, 2,
                                               giants, gelts, 2, grid, false, batch);
  for (uint64_t k = 0; k < a.size(); ++k) wrong += a[k] != b[k];

  // k = 8 with the rescale: 2 x (L - 1) limbs per ciphertext, every word below its modulus
  AlignedVector64<uint64_t> r(batch * 2 * (L - 1) * n, ~0ull);
  intel::hexl::b200::InnerSumHybrid(r.data(), ct.data(), n, L, L, K, 2, q.data(), g, 8, table, elts, 4, true, batch);
  uint64_t bad = 0;
  for (uint64_t k = 0; k < r.size(); ++k) bad += r[k] >= q[(k / n) % (L - 1)];
  wrong += bad;

  // k = 7 shifts by g^3 at its top bit: not in the table
  bool threw = false;
  try {
    intel::hexl::b200::InnerSumHybrid(a.data(), ct.data(), n, L, L, K, 2, q.data(), g, 7, table, elts, 4, false, 1);
  } catch (const std::runtime_error&) {
    threw = true;
  }
  wrong += !threw;

  std::printf("inner_sum_caller: %llu words differ%s\n", (unsigned long long)wrong,
              threw ? "" : ", and a missing key did not throw");
  return wrong == 0 ? 0 : 1;
}
