// A C++ caller of intel::hexl::b200::PlainLift, BfvAddPlain and BfvMultiplyPlain through include/hexl/hexl.hpp, on host
// AlignedVector64 buffers.  BfvMultiplyPlain must equal PlainLift in NTT form, the forward transform of the ciphertext,
// EltwiseMultMod and the inverse transform bit for bit, with the plaintext in either form; BfvAddPlain in place must
// equal it out of place, and sub_plain must undo add_plain.  Built without arguments it only has to link; `run` calls
// the library (needs a GPU).
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "hexl/hexl.hpp"

using intel::hexl::AlignedVector64;

int main(int argc, char** argv) {
  if (argc < 2 || std::strcmp(argv[1], "run") != 0) return 0;
  const uint64_t n = 1024, L = 3, batch = 2, comp = L * n, t = 65537, pcc = n / 2 + 1;
  const std::vector<uint64_t> q = intel::hexl::GeneratePrimes(L, 55, true, n);
  uint64_t s = 4049;
  auto next = [&](uint64_t bound) {
    s = s * 6364136223846793005ull + 1442695040888963407ull;
    return (s >> 11) % bound;
  };
  AlignedVector64<uint64_t> ct(batch * 2 * comp), plain(pcc);
  for (uint64_t c = 0; c < 2 * batch; ++c)
    for (uint64_t i = 0; i < L; ++i)
      for (uint64_t l = 0; l < n; ++l) ct[(c * L + i) * n + l] = next(q[i]);
  for (auto& m : plain) m = next(t);
  uint64_t wrong = 0;

  AlignedVector64<uint64_t> lifted(comp), fused(batch * 2 * comp), ready(batch * 2 * comp);
  intel::hexl::b200::PlainLift(lifted.data(), plain.data(), pcc, n, q.data(), L, t, 1, true);
  intel::hexl::b200::BfvMultiplyPlain(fused.data(), ct.data(), plain.data(), pcc, 1, false, n, q.data(), L, t, batch);
  intel::hexl::b200::BfvMultiplyPlain(ready.data(), ct.data(), lifted.data(), pcc, 1, true, n, q.data(), L, t, batch);
  std::vector<intel::hexl::NTT> ntts;
  for (uint64_t i = 0; i < L; ++i) ntts.emplace_back(n, q[i]);
  for (uint64_t c = 0; c < 2 * batch; ++c)
    for (uint64_t i = 0; i < L; ++i) {
      const uint64_t off = (c * L + i) * n;
      AlignedVector64<uint64_t> x(n);
      ntts[i].ComputeForward(x.data(), ct.data() + off, 1, 1);
      intel::hexl::EltwiseMultMod(x.data(), x.data(), lifted.data() + i * n, n, q[i], 1);
      ntts[i].ComputeInverse(x.data(), x.data(), 1, 1);
      for (uint64_t l = 0; l < n; ++l) wrong += (fused[off + l] != x[l]) + (ready[off + l] != x[l]);
    }

  AlignedVector64<uint64_t> out(batch * 2 * comp), inplace = ct;
  intel::hexl::b200::BfvAddPlain(out.data(), ct.data(), plain.data(), pcc, 1, n, q.data(), L, t, false, batch);
  intel::hexl::b200::BfvAddPlain(inplace.data(), inplace.data(), plain.data(), pcc, 1, n, q.data(), L, t, false, batch);
  for (uint64_t k = 0; k < batch * 2 * comp; ++k) wrong += out[k] != inplace[k];
  intel::hexl::b200::BfvAddPlain(inplace.data(), inplace.data(), plain.data(), pcc, 1, n, q.data(), L, t, true, batch);
  for (uint64_t k = 0; k < batch * 2 * comp; ++k) wrong += inplace[k] != ct[k];

  std::printf("plain_caller: %llu words differ\n", (unsigned long long)wrong);
  return wrong == 0 ? 0 : 1;
}
