// A C++ caller of intel::hexl::DivideAndRoundQLast through include/hexl/hexl.hpp: three 30-bit moduli,
// coefficient form, host vectors, two polynomials rescaled in place; every word is checked against the definition
// floor((X + q_2/2) / q_2) mod q_i computed with __int128.  Built without arguments it only has to link; `run` calls
// the library (needs a GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "hexl/hexl.hpp"

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1000, rns = 3, count = 2;
  const uint64_t q[rns] = {1073741789ull, 1073741783ull, 1073741741ull};  // 30-bit primes
  typedef unsigned __int128 u128;
  const u128 Q = (u128)q[0] * q[1] * q[2];
  std::vector<uint64_t> data(count * rns * n), want(count * rns * n);
  uint64_t s = 12345;
  for (uint64_t p = 0; p < count; ++p)
    for (uint64_t l = 0; l < n; ++l) {
      s = s * 6364136223846793005ull + 1442695040888963407ull;
      u128 X = (((u128)s << 64) | (s ^ (s >> 17))) % Q;
      if (l == 0) X = 0;
      if (l == 1) X = Q - 1;
      if (l == 2) X = (u128)q[2] * 77 + q[2] / 2;  // exactly on the rounding boundary
      for (uint64_t i = 0; i < rns; ++i) data[(p * rns + i) * n + l] = (uint64_t)(X % q[i]);
      const u128 y = (X + q[2] / 2) / q[2];
      for (uint64_t i = 0; i < rns; ++i)
        want[(p * rns + i) * n + l] = i + 1 < rns ? (uint64_t)(y % q[i]) : data[(p * rns + i) * n + l];
    }
  intel::hexl::DivideAndRoundQLast(data.data(), data.data(), n, q, rns, count, false);
  uint64_t wrong = 0;
  for (size_t k = 0; k < data.size(); ++k) wrong += data[k] != want[k];
  std::printf("rescale_caller: %llu of %zu words differ\n", (unsigned long long)wrong, data.size());
  return wrong == 0 ? 0 : 1;
}
