// One caller of the intel::hexl C++ API, compiled unchanged against the reference's headers and library and against
// include/hexl/** and libhexl_b200.so; tests/test_cpp_api_parity.py runs both programs and compares what they write.
//
//   api_parity <outdir> [--host-only]
//
// Every record is a file <outdir>/<tag>.bin of little-endian 64-bit words and a line "tag kind q out_mf" in
// <outdir>/index.txt.  kind is
//   exact     the two programs must write the same words;
//   lazy      every word is below out_mf * q, and the two programs' words are congruent mod q;
//   property  the words are (degree, modulus, root) triples and each root must be a primitive degree-th root.
// --host-only runs what a caller compiles into its own binary or computes on the host: the inline arithmetic of the
// headers, the number theory, and the NTT tables and constants.  Without it the GPU entry points run too, called the
// way SEAL calls them: one polynomial per call on std::vector buffers.
//
// Only names both trees declare are used.  The one exception is the element-wise Montgomery family, which the
// reference keeps in an internal AVX-512 header: against the reference this program computes those records with the
// public MontgomeryReduce<64>, element by element, which is the operation the three calls are specified to perform.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "hexl/hexl.hpp"
#include "hexl/experimental/seal/locks.hpp"
#include "hexl/experimental/seal/ntt-cache.hpp"

#if __has_include("hexl/b200/hexl_api.hpp")
#define API_PARITY_HAS_ELTWISE_MONTGOMERY 1
#endif

using namespace intel::hexl;
using Words = std::vector<uint64_t>;

namespace {

std::string g_dir;
FILE* g_index = nullptr;
size_t g_records = 0;

void Rec(const std::string& tag, const char* kind, uint64_t q, uint64_t out_mf, const uint64_t* w, size_t n) {
  const std::string path = g_dir + "/" + tag + ".bin";
  FILE* f = std::fopen(path.c_str(), "wb");
  if (!f || (n && std::fwrite(w, sizeof(uint64_t), n, f) != n) || std::fclose(f)) {
    std::fprintf(stderr, "cannot write %s\n", path.c_str());
    std::exit(2);
  }
  std::fprintf(g_index, "%s %s %llu %llu\n", tag.c_str(), kind, (unsigned long long)q, (unsigned long long)out_mf);
  ++g_records;
}
template <class V>
void Exact(const std::string& tag, const V& v, uint64_t q = 0) {
  Rec(tag, "exact", q, 0, v.data(), v.size());
}
template <class V>
void Lazy(const std::string& tag, const V& v, uint64_t q, uint64_t out_mf) {
  Rec(tag, "lazy", q, out_mf, v.data(), v.size());
}
std::string S(uint64_t v) { return std::to_string(v); }

// splitmix64: the same operands on both sides
struct Rng {
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed * 0x9E3779B97F4A7C15ULL + 1) {}
  uint64_t Next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ULL);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    return z ^ (z >> 31);
  }
  uint64_t Below(uint64_t bound) { return bound ? Next() % bound : Next(); }  // bound 0 means 2^64
};

uint64_t PrimeBelow(uint64_t x) {
  uint64_t p = x - 1;
  while (!IsPrime(p)) --p;
  return p;
}
uint64_t PrimeAbove(uint64_t x) {
  uint64_t p = x + 1;
  while (!IsPrime(p)) ++p;
  return p;
}

// 2, 3, 769, the primes on both sides of 2^30, 2^32, 2^50, 2^52, 2^56 and 2^61, and the largest 62-bit prime
Words EdgeModuli() {
  Words m{2, 3, 769};
  for (int k : {30, 32, 50, 52, 56, 61}) {
    m.push_back(PrimeBelow(1ULL << k));
    m.push_back(PrimeAbove(1ULL << k));
  }
  m.push_back(PrimeBelow(1ULL << 62));
  return m;
}

// words where 64- and 128-bit arithmetic goes wrong: 0, 1, 2^k - 1, 2^k, 2^k + 1, 2^63, 2^64 - 1 and a few others
Words EdgeWords() {
  Words w{0, 1, 2, 3};
  for (int k : {31, 32, 52, 62, 63}) {
    w.push_back((1ULL << k) - 1);
    w.push_back(1ULL << k);
    w.push_back((1ULL << k) + 1);
  }
  w.push_back(~0ULL);
  w.push_back(~0ULL - 1);
  Rng r(1);
  for (int i = 0; i < 4; ++i) w.push_back(r.Next());
  return w;
}

// operands below bound = factor * q: 0, 1, q - 1, q, q + 1 and the top of the range where they fit, then uniform
Words ModWords(uint64_t q, uint64_t factor, size_t extra, uint64_t seed) {
  const uint64_t bound = q * factor;
  Words w;
  for (uint64_t v : Words{uint64_t(0), uint64_t(1), q - 1, q, q + 1, 2 * q - 1, 2 * q, 4 * q - 1, bound - 2, bound - 1})
    if (v < bound) w.push_back(v);
  Rng r(seed);
  for (size_t i = 0; i < extra; ++i) w.push_back(r.Below(bound));
  return w;
}

// ------------------------------------------------------------------------------------------ inline arithmetic
void InlineArithmetic(const Words& moduli) {
  const Words G = EdgeWords();
  Words hi32, hi52, hi64, mul, add;
  for (uint64_t x : G)
    for (uint64_t y : G) {
      hi32.push_back(MultiplyUInt64Hi<32>(x, y));
      hi52.push_back(MultiplyUInt64Hi<52>(x, y));
      hi64.push_back(MultiplyUInt64Hi<64>(x, y));
      uint64_t ph = 0, pl = 0;
      MultiplyUInt64(x, y, &ph, &pl);
      const uint128_t p = MultiplyUInt64(x, y);
      mul.insert(mul.end(), {ph, pl, static_cast<uint64_t>(p >> 64), static_cast<uint64_t>(p)});
      uint64_t s = 0;
      const unsigned char carry = AddUInt64(x, y, &s);
      add.insert(add.end(), {s, carry});
    }
  Exact("MultiplyUInt64Hi_32", hi32);
  Exact("MultiplyUInt64Hi_52", hi52);
  Exact("MultiplyUInt64Hi_64", hi64);
  Exact("MultiplyUInt64", mul);
  Exact("AddUInt64", add);

  Words maxv, bits;
  for (uint64_t b = 0; b <= 64; ++b) maxv.push_back(MaximumValue(b));
  // MSB and Log2 of 0 are undefined (the reference takes log2 of 0)
  Words msb_in;
  for (int k = 0; k < 64; ++k) msb_in.insert(msb_in.end(), {1ULL << k, (1ULL << k) + 1, ((1ULL << k) - 1) | 1});
  for (uint64_t x : G)
    if (x) msb_in.push_back(x);
  for (uint64_t x : msb_in) bits.insert(bits.end(), {x, MSB(x), Log2(x)});
  Exact("MaximumValue", maxv);
  Exact("MSB_Log2", bits);
  Words pow2;
  for (uint64_t x : msb_in) pow2.insert(pow2.end(), {x, IsPowerOfTwo(x), IsPowerOfFour(x)});
  pow2.insert(pow2.end(), {0, IsPowerOfTwo(0), IsPowerOfFour(0)});
  Exact("IsPowerOfTwo_IsPowerOfFour", pow2);
  Words nots;
  for (int c = 0; c < 8; ++c) nots.push_back(static_cast<uint64_t>(Not(static_cast<CMPINT>(c))));
  Exact("CMPINT_Not", nots);

  Words div;
  for (uint64_t q : moduli)
    for (uint64_t x1 : G)
      for (uint64_t x0 : Words{uint64_t(0), uint64_t(1), ~0ULL, x1 ^ 0x5555555555555555ULL}) {
        // DivideUInt128UInt64Lo keeps the low word of the quotient; BarrettReduce128 takes any 128-bit input
        div.push_back(DivideUInt128UInt64Lo(x1 % q, x0, q));
        div.push_back(DivideUInt128UInt64Lo(x1, x0, q));
        div.push_back(BarrettReduce128(x1, x0, q));
      }
  Exact("DivideUInt128UInt64Lo_BarrettReduce128", div);

  for (uint64_t q : moduli) {
    const std::string sq = "_q" + S(q);
    const Words xs = ModWords(q, 1, 24, q);
    const uint64_t twice = 2 * q, four = 4 * q;
    Words mm, lazy[3], lazy2[3], mf;
    for (uint64_t x : xs)
      for (uint64_t y : xs) {
        const uint64_t y_precon = MultiplyFactor(y, 64, q).BarrettFactor();
        mm.push_back(MultiplyMod(x, y, y_precon, q));
        const int shifts[3] = {32, 52, 64};
        for (int s = 0; s < 3; ++s) {
          // MultiplyModLazy<BitShift> needs q and x at most 2^BitShift - 1
          if (shifts[s] < 64 && q > MaximumValue(shifts[s])) continue;
          const uint64_t factor = MultiplyFactor(y, shifts[s], q).BarrettFactor();
          // x below q and x at the top of the BitShift-bit range
          for (uint64_t xl : Words{x, MaximumValue(shifts[s]) - x}) {
            if (s == 0) {
              lazy[s].push_back(MultiplyModLazy<32>(xl, y, factor, q));
              lazy2[s].push_back(MultiplyModLazy<32>(xl, y, q));
            } else if (s == 1) {
              lazy[s].push_back(MultiplyModLazy<52>(xl, y, factor, q));
              lazy2[s].push_back(MultiplyModLazy<52>(xl, y, q));
            } else {
              lazy[s].push_back(MultiplyModLazy<64>(xl, y, factor, q));
              lazy2[s].push_back(MultiplyModLazy<64>(xl, y, q));
            }
          }
        }
      }
    Exact("MultiplyMod_precon" + sq, mm, q);
    const char* names[3] = {"32", "52", "64"};
    for (int s = 0; s < 3; ++s) {
      if (lazy[s].empty()) continue;
      Exact(std::string("MultiplyModLazy_factor_") + names[s] + sq, lazy[s], q);
      Exact(std::string("MultiplyModLazy_") + names[s] + sq, lazy2[s], q);
    }

    // Barrett reduction of any 64-bit word, fully and to [0, 2q)
    const uint64_t q_barr = MultiplyFactor(1, 64, q).BarrettFactor();
    Words b1, b2;
    Rng r(q ^ 77);
    Words ins = G;
    for (int i = 0; i < 256; ++i) ins.push_back(r.Next());
    for (uint64_t k = 1; k < 8; ++k) ins.insert(ins.end(), {k * q - 1, k * q, k * q + 1});
    for (uint64_t x : ins) {
      b1.push_back(BarrettReduce64<1>(x, q, q_barr));
      b2.push_back(BarrettReduce64<2>(x, q, q_barr));
    }
    Exact("BarrettReduce64_1" + sq, b1, q);
    Exact("BarrettReduce64_2" + sq, b2, q);

    // ReduceMod<InputModFactor> on [0, factor * q)
    for (uint64_t f : {1, 2, 4, 8}) {
      if (q > ~0ULL / f) continue;
      Words red;
      for (uint64_t x : ModWords(q, f, 64, q + f)) {
        if (f == 1) red.push_back(ReduceMod<1>(x, q, &twice, &four));
        if (f == 2) red.push_back(ReduceMod<2>(x, q, &twice, &four));
        if (f == 4) red.push_back(ReduceMod<4>(x, q, &twice, &four));
        if (f == 8) red.push_back(ReduceMod<8>(x, q, &twice, &four));
      }
      Exact("ReduceMod_" + S(f) + sq, red, q);
    }

    for (uint64_t shift : {32, 52, 64}) {
      for (uint64_t op : ModWords(q, 1, 8, q + shift)) {
        MultiplyFactor m(op, shift, q);
        mf.insert(mf.end(), {m.Operand(), m.BarrettFactor()});
      }
      MultiplyFactor m(q, shift, q);  // operand == modulus is allowed
      mf.insert(mf.end(), {m.Operand(), m.BarrettFactor()});
    }
    Exact("MultiplyFactor" + sq, mf, q);
  }
}

// names a caller reaches through the reference's headers besides the arithmetic: the NTT cache's key hash and lock,
// and the loop-unrolling macros
void ReachableNames() {
  RWLock lock;
  { ReadLock reader = lock.AcquireRead(); }
  { WriteLock writer = lock.AcquireWrite(); }
  { ReadLock reader = lock.TryAcquireRead(); }
  { WriteLock writer = lock.TryAcquireWrite(); }
  Words h;
  HEXL_LOOP_UNROLL_4
  for (uint64_t i = 0; i < 8; ++i) h.push_back(HashPair::hash_combine(i * 0x9E3779B97F4A7C15ULL, ~i));
  HEXL_LOOP_UNROLL_8
  for (uint64_t i = 0; i < 8; ++i) h.push_back(HashPair{}(std::make_pair(uint64_t(1) << i, uint64_t(1) << (63 - i))));
  Exact("HashPair", h);
}

// ------------------------------------------------------------------------------------------ number theory
void NumberTheory(const Words& moduli) {
  Words rev;
  Rng r(5);
  for (uint64_t w = 0; w <= 64; ++w) {
    const uint64_t mask = MaximumValue(w);
    for (uint64_t x : Words{uint64_t(0), uint64_t(1), mask, w ? 1ULL << (w - 1) : 0, r.Next() & mask, r.Next() & mask})
      rev.push_back(ReverseBits(x & mask, w));
  }
  Exact("ReverseBits", rev);

  for (uint64_t q : moduli) {
    const std::string sq = "_q" + S(q);
    const Words xs = ModWords(q, 1, 16, q * 3);
    Words inv, mul, add, sub, pw;
    for (uint64_t x : xs) {
      if (x % q) inv.push_back(InverseMod(x, q));
      for (uint64_t y : xs) {
        if (x >= q || y >= q) continue;
        mul.push_back(MultiplyMod(x, y, q));
        add.push_back(AddUIntMod(x, y, q));
        sub.push_back(SubUIntMod(x, y, q));
      }
      if (x < q)
        for (uint64_t e : Words{uint64_t(0), uint64_t(1), uint64_t(2), q - 2, q - 1, q, ~0ULL, 0x123456789abcdefULL})
          pw.push_back(PowMod(x, e, q));
    }
    Exact("InverseMod" + sq, inv, q);
    Exact("MultiplyMod" + sq, mul, q);
    Exact("AddUIntMod" + sq, add, q);
    Exact("SubUIntMod" + sq, sub, q);
    Exact("PowMod" + sq, pw, q);

    // Hensel's lemma and Montgomery reduction for every r with 2^r > q
    if (q % 2 == 1) {
      Words hensel, mont;
      for (uint32_t rr = 1; rr <= 63; ++rr) hensel.push_back(HenselLemma2adicRoot(rr, q));
      for (int rr : {31, 46, 52, 61, 62, 63}) {
        if ((1ULL << rr) <= q) continue;
        const uint64_t inv_mod = HenselLemma2adicRoot(rr, q);
        const uint64_t mask = (1ULL << rr) - 1;
        for (uint64_t a : ModWords(q, 1, 12, q + rr))
          for (uint64_t b : Words{uint64_t(0), uint64_t(1), q - 1, a >> 1}) {
            if (a >= q) continue;
            uint64_t hi = 0, lo = 0;
            MultiplyUInt64(a, b, &hi, &lo);
            mont.push_back(MontgomeryReduce<64>(hi, lo, q, rr, mask, inv_mod));
          }
      }
      Exact("HenselLemma2adicRoot" + sq, hensel, q);
      Exact("MontgomeryReduce_64" + sq, mont, q);
    }
  }

  // primes, Carmichael numbers, squares of primes, strong pseudoprimes to small bases, 2^64 - 1
  Words primes{0, 2, 3, 4, 5, 9, 25, 49, 91, 97, 561, 1105, 1729, 2047, 2465, 2821, 6601, 8911, 41041, 62745, 825265,
               3215031751ULL, 321197185ULL, 3825123056546413051ULL, 18446744073709551557ULL,
               65537ULL * 65537ULL, 4294967291ULL * 4294967291ULL, 3037000493ULL * 3037000493ULL,
               4294967291ULL * 4294967279ULL, (1ULL << 61) - 1, (1ULL << 31) - 1, ~0ULL, ~0ULL - 58};
  for (uint64_t q : moduli) primes.insert(primes.end(), {q, q + 2, q - 2});
  Words is_prime;
  for (uint64_t n : primes) is_prime.insert(is_prime.end(), {n, IsPrime(n)});
  Exact("IsPrime", is_prime);

  Words gen;
  for (size_t bits : {30, 40, 50, 55, 59, 60, 61})
    for (bool small : {true, false})
      for (size_t ntt_size : {1, 1024, 1 << 16}) {
        const Words p = GeneratePrimes(3, bits, small, ntt_size);
        gen.insert(gen.end(), p.begin(), p.end());
      }
  Exact("GeneratePrimes", gen);

  // roots of unity: the minimal one, which candidates are primitive, and a random one (a property record)
  const Words ntt_moduli{769, GeneratePrimes(1, 29, false, 1 << 17)[0], GeneratePrimes(1, 55, true, 1 << 17)[0],
                         GeneratePrimes(1, 61, false, 1 << 17)[0]};
  Words minimal, prim, random_roots;
  for (uint64_t q : ntt_moduli)
    for (uint64_t degree = 2; degree <= (1ULL << 18) && (q - 1) % degree == 0; degree <<= 1) {
      const uint64_t root = MinimalPrimitiveRoot(degree, q);
      minimal.insert(minimal.end(), {degree, q, root});
      for (uint64_t cand : {root, PowMod(root, 2, q), PowMod(root, 3, q), uint64_t(1), q - 1, uint64_t(0), uint64_t(2)})
        prim.push_back(IsPrimitiveRoot(cand, degree, q));
      random_roots.insert(random_roots.end(), {degree, q, GeneratePrimitiveRoot(degree, q)});
    }
  Exact("MinimalPrimitiveRoot", minimal);
  Exact("IsPrimitiveRoot", prim);
  Rec("GeneratePrimitiveRoot", "property", 0, 0, random_roots.data(), random_roots.size());
}

// ------------------------------------------------------------------------------------------ NTT host side
void NttTables(const std::string& tag, NTT& ntt) {
  const uint64_t q = ntt.GetModulus();
  Exact(tag + "_scalars", Words{ntt.GetDegree(), q, ntt.GetMinimalRootOfUnity(), ntt.GetRootOfUnityPower(0),
                                ntt.GetRootOfUnityPower(ntt.GetDegree() - 1), ntt.GetInvRootOfUnityPower(0),
                                ntt.GetInvRootOfUnityPower(ntt.GetDegree() - 1)},
        q);
  Exact(tag + "_RootOfUnityPowers", ntt.GetRootOfUnityPowers(), q);
  Exact(tag + "_Precon32RootOfUnityPowers", ntt.GetPrecon32RootOfUnityPowers(), q);
  Exact(tag + "_Precon64RootOfUnityPowers", ntt.GetPrecon64RootOfUnityPowers(), q);
  Exact(tag + "_AVX512RootOfUnityPowers", ntt.GetAVX512RootOfUnityPowers(), q);
  Exact(tag + "_AVX512Precon32RootOfUnityPowers", ntt.GetAVX512Precon32RootOfUnityPowers(), q);
  Exact(tag + "_AVX512Precon52RootOfUnityPowers", ntt.GetAVX512Precon52RootOfUnityPowers(), q);
  Exact(tag + "_AVX512Precon64RootOfUnityPowers", ntt.GetAVX512Precon64RootOfUnityPowers(), q);
  Exact(tag + "_InvRootOfUnityPowers", ntt.GetInvRootOfUnityPowers(), q);
  Exact(tag + "_Precon32InvRootOfUnityPowers", ntt.GetPrecon32InvRootOfUnityPowers(), q);
  Exact(tag + "_Precon52InvRootOfUnityPowers", ntt.GetPrecon52InvRootOfUnityPowers(), q);
  Exact(tag + "_Precon64InvRootOfUnityPowers", ntt.GetPrecon64InvRootOfUnityPowers(), q);
}

void NttHost() {
  const Words moduli{GeneratePrimes(1, 29, false, 1 << 17)[0], GeneratePrimes(1, 61, false, 1 << 17)[0]};
  for (uint64_t n = 2; n <= (1 << 17); n <<= 1)
    for (size_t m = 0; m < moduli.size(); ++m) {
      const uint64_t q = moduli[m];
      NTT minimal(n, q);
      NttTables("NTT_n" + S(n) + "_q" + S(q), minimal);
      if (m == 1) {
        NTT other(n, q, PowMod(MinimalPrimitiveRoot(2 * n, q), 3, q));
        NttTables("NTT_root3_n" + S(n) + "_q" + S(q), other);
      }
    }
  {
    const uint64_t n = 1 << 20, q = GeneratePrimes(1, 59, true, n)[0];
    NTT big(n, q);
    NttTables("NTT_n" + S(n) + "_q" + S(q), big);
  }

  // copies, moves and assignments keep the tables, also after the source is gone
  {
    const uint64_t n = 64, q = GeneratePrimes(1, 50, true, n)[0];
    NTT copy, assigned, moved_to;
    {
      NTT src(n, q);
      copy = src;
      NTT tmp(src);
      NTT moved(std::move(tmp));
      moved_to = std::move(moved);
      assigned = NTT(n, q);
    }
    NttTables("NTT_copy", copy);
    NttTables("NTT_move", moved_to);
    NttTables("NTT_assign", assigned);
  }

  // CheckArguments on both sides of each precondition: power of two, degree <= 2^20, q <= 2^62, q = 1 mod 2n, prime
  Words check;
  const uint64_t q20 = GeneratePrimes(1, 40, true, 1 << 20)[0];
  struct Case {
    uint64_t degree, q;
  } cases[] = {{8, 769},     {7, 769},       {12, 769},      {1, 769},          {1 << 20, q20}, {1 << 21, q20},
               {8, 770},     {8, 771},       {8, 17},        {8, 7 * 16 + 1},   {2, 5},         {16, 769 * 97},
               {8, PrimeBelow(1ULL << 62) }, {8, 0}};
  for (const Case& c : cases) check.insert(check.end(), {c.degree, c.q, NTT::CheckArguments(c.degree, c.q)});
  Exact("NTT_CheckArguments", check);

  Exact("NTT_constants",
        Words{NTT::MaxDegreeBits(), NTT::MaxModulusBits(), NTT::s_default_shift_bits, NTT::s_ifma_shift_bits,
              NTT::s_max_fwd_32_modulus, NTT::s_max_inv_32_modulus, NTT::s_max_fwd_ifma_modulus,
              NTT::s_max_inv_ifma_modulus, NTT::s_max_inv_dq_modulus, NTT::s_max_fwd_modulus(32),
              NTT::s_max_fwd_modulus(52), NTT::s_max_fwd_modulus(64), NTT::s_max_inv_modulus(32),
              NTT::s_max_inv_modulus(52), NTT::s_max_inv_modulus(64)});
}

// ------------------------------------------------------------------------------------------ GPU entry points
// one prime per arithmetic mode: below 2^30; just above 2^32 and just below 2^56; just below 2^61 and 2^62
Words TransformModuli() {
  const uint64_t n = 1 << 17;
  return {GeneratePrimes(1, 29, false, n)[0], GeneratePrimes(1, 32, true, n)[0], GeneratePrimes(1, 55, false, n)[0],
          GeneratePrimes(1, 60, false, n)[0], GeneratePrimes(1, 61, false, n)[0]};
}

Words Operand(uint64_t n, uint64_t bound, uint64_t seed) {
  // every fourth word at the top of the range, the others uniform below it
  Rng r(seed);
  Words v(n);
  for (uint64_t i = 0; i < n; ++i)
    v[i] = (i % 4 != 1) ? r.Below(bound) : bound ? bound - 1 - (i & 7) % bound : ~0ULL - (i & 7);
  return v;
}

void Transforms() {
  for (uint64_t q : TransformModuli())
    for (uint64_t n = 2; n <= (1 << 17); n <<= 1) {
      const std::string t = "_n" + S(n) + "_q" + S(q);
      NTT ntt(n, q);
      for (uint64_t in : {1, 2, 4})
        for (uint64_t out : {1, 4}) {
          const Words x = Operand(n, in * q, n + q + in);
          Words y(n, 0);
          ntt.ComputeForward(y.data(), x.data(), in, out);
          const std::string tag = "Forward_in" + S(in) + "_out" + S(out) + t;
          if (out == 1) Exact(tag, y, q); else Lazy(tag, y, q, out);
        }
      for (uint64_t in : {1, 2})
        for (uint64_t out : {1, 2}) {
          const Words x = Operand(n, in * q, n + q + 10 * in);
          Words y(n, 0);
          ntt.ComputeInverse(y.data(), x.data(), in, out);
          const std::string tag = "Inverse_in" + S(in) + "_out" + S(out) + t;
          if (out == 1) Exact(tag, y, q); else Lazy(tag, y, q, out);
        }
      // in place, through the SEAL cache, and with a root other than the minimal one
      Words x = Operand(n, q, n ^ q);
      GetNTT(n, q).ComputeForward(x.data(), x.data(), 1, 1);
      Exact("Forward_inplace_cached" + t, x, q);
      GetNTT(n, q).ComputeInverse(x.data(), x.data(), 2, 1);
      Exact("Inverse_inplace_cached" + t, x, q);
      NTT other(n, q, PowMod(ntt.GetMinimalRootOfUnity(), 5, q));
      Words y(n, 0);
      other.ComputeForward(y.data(), x.data(), 1, 1);
      Exact("Forward_root5" + t, y, q);
      other.ComputeInverse(x.data(), y.data(), 1, 1);
      Exact("Inverse_root5" + t, x, q);
    }
}

void MontgomeryCalls(const std::string& t, uint64_t q, int r, const Words& a, const Words& b) {
  const uint64_t n = a.size();
  const uint64_t inv_mod = HenselLemma2adicRoot(r, q);
  const uint64_t R = (r == 64) ? 0 : (1ULL << r) % q;
  const uint64_t R2 = MultiplyMod(R, R, q);
  Words prod(n), in(n), out(n);
#ifdef API_PARITY_HAS_ELTWISE_MONTGOMERY
  EltwiseMontReduceMod(prod.data(), a.data(), b.data(), n, q, r, inv_mod);
  EltwiseMontgomeryFormIn(in.data(), a.data(), R2, n, q, r, inv_mod);
  EltwiseMontgomeryFormOut(out.data(), a.data(), n, q, r, inv_mod);
#else
  const uint64_t mask = (1ULL << r) - 1;
  for (uint64_t i = 0; i < n; ++i) {
    uint64_t hi = 0, lo = 0;
    MultiplyUInt64(a[i], b[i], &hi, &lo);
    prod[i] = MontgomeryReduce<64>(hi, lo, q, r, mask, inv_mod);
    MultiplyUInt64(a[i], R2, &hi, &lo);
    in[i] = MontgomeryReduce<64>(hi, lo, q, r, mask, inv_mod);
    out[i] = MontgomeryReduce<64>(0, a[i], q, r, mask, inv_mod);
  }
#endif
  Exact("EltwiseMontReduceMod" + t, prod, q);
  Exact("EltwiseMontgomeryFormIn" + t, in, q);
  Exact("EltwiseMontgomeryFormOut" + t, out, q);
}

void Eltwise() {
  // the largest modulus each operation accepts bounds its set: MultMod and DyadicMultiply q < 2^62, AddMod and SubMod
  // q < 2^63, FMAMod q < 2^61, ReduceMod and CmpSubMod any q > 1.  4084223049772944437 is a 62-bit prime at which the
  // reference's one conditional subtraction leaves some products in [q, 2q).
  const Words base{3, 769, PrimeBelow(1ULL << 30), PrimeAbove(1ULL << 32), PrimeBelow(1ULL << 52),
                   PrimeBelow(1ULL << 56), PrimeBelow(1ULL << 61)};
  Words mult = base, add = base, reduce = base;
  mult.insert(mult.end(), {PrimeBelow(1ULL << 62), 4084223049772944437ULL});
  add.insert(add.end(), {PrimeBelow(1ULL << 62), PrimeBelow(1ULL << 63)});
  reduce.insert(reduce.end(), {PrimeBelow(1ULL << 63), PrimeAbove(1ULL << 63), PrimeBelow(~0ULL)});

  for (uint64_t n : {1, 7, 4099, (1 << 16) + 1}) {
    const std::string sn = "_n" + S(n);
    for (uint64_t q : add) {
      const std::string t = sn + "_q" + S(q);
      const Words a = Operand(n, q, q + n), b = Operand(n, q, q + n + 1);
      const uint64_t s = q - 1 - (n % q);
      Words r(n);
      EltwiseAddMod(r.data(), a.data(), b.data(), n, q);
      Exact("EltwiseAddMod" + t, r, q);
      EltwiseAddMod(r.data(), a.data(), s, n, q);
      Exact("EltwiseAddMod_scalar" + t, r, q);
      EltwiseSubMod(r.data(), a.data(), b.data(), n, q);
      Exact("EltwiseSubMod" + t, r, q);
      EltwiseSubMod(r.data(), a.data(), s, n, q);
      Exact("EltwiseSubMod_scalar" + t, r, q);
      // SEAL's in-place call
      Words c = a;
      EltwiseAddMod(c.data(), c.data(), b.data(), n, q);
      Exact("EltwiseAddMod_inplace" + t, c, q);
    }
    for (uint64_t q : mult)
      for (uint64_t f : {1, 2, 4}) {
        if (f * q >= (1ULL << 63)) continue;
        const std::string t = "_in" + S(f) + sn + "_q" + S(q);
        const Words a = Operand(n, f * q, q + n + f), b = Operand(n, f * q, q + n + f + 7);
        Words r(n);
        EltwiseMultMod(r.data(), a.data(), b.data(), n, q, f);
        Exact("EltwiseMultMod" + t, r, q);
        if (q >= (3ULL << 60)) {  // the operands for the exact check of the 62-bit products
          Exact("EltwiseMultMod_a" + t, a, q);
          Exact("EltwiseMultMod_b" + t, b, q);
        }
      }
    for (uint64_t q : base)
      for (uint64_t f : {1, 2, 4, 8}) {
        if (q >= (1ULL << 61)) continue;
        const std::string t = "_in" + S(f) + sn + "_q" + S(q);
        const Words a = Operand(n, f * q, q + n + 3 * f), c = Operand(n, q, q + n + 5);
        const uint64_t arg2 = q - 2 - (q > 2 ? n % (q - 2) : 0);
        Words r(n);
        EltwiseFMAMod(r.data(), a.data(), arg2, c.data(), n, q, f);
        Exact("EltwiseFMAMod" + t, r, q);
        EltwiseFMAMod(r.data(), a.data(), arg2, nullptr, n, q, f);
        Exact("EltwiseFMAMod_noarg3" + t, r, q);
      }
    for (uint64_t q : reduce)
      for (uint64_t f : Words{q, uint64_t(2), uint64_t(4)})
        for (uint64_t out : {1, 2}) {
          if (f == out) continue;  // input_mod_factor must differ from output_mod_factor
          const std::string t = "_in" + S(f == q ? 0 : f) + "_out" + S(out) + sn + "_q" + S(q);
          // input_mod_factor q takes any word; 2 and 4 take words below that multiple of q where it fits
          const uint64_t bound = (f == q || f * (q >> 1) >= (1ULL << 63)) ? 0 : f * q;
          const Words a = Operand(n, bound, q + n + f + out);
          Words r(n);
          EltwiseReduceMod(r.data(), a.data(), n, q, f, out);
          const std::string tag = "EltwiseReduceMod" + t;
          if (out == 1) Exact(tag, r, q); else Lazy(tag, r, q, out);
          if (q >> 63) Exact("EltwiseReduceMod_a" + t, a, q);  // the operand for the exact check
        }
    {
      const uint64_t q = PrimeBelow(1ULL << 50);
      const Words a = Operand(n, 0, n + 11);
      for (int c = 0; c < 8; ++c)
        for (uint64_t bound : Words{uint64_t(0), q, a[0]}) {
          const std::string t = "_cmp" + S(c) + "_bound" + S(bound) + sn;
          const uint64_t diff = 1 + (bound % 1000);
          Words r(n);
          EltwiseCmpAdd(r.data(), a.data(), n, static_cast<CMPINT>(c), bound, diff);
          Exact("EltwiseCmpAdd" + t, r);
          EltwiseCmpSubMod(r.data(), a.data(), n, q, static_cast<CMPINT>(c), bound, diff);
          Exact("EltwiseCmpSubMod" + t, r, q);
        }
    }
    for (uint64_t q : Words{769ULL, PrimeBelow(1ULL << 46), PrimeBelow(1ULL << 61)}) {
      const Words a = Operand(n, q, n + q + 21), b = Operand(n, q, n + q + 22);
      for (int r : {46, 62})
        if ((1ULL << r) > q) MontgomeryCalls("_r" + S(r) + sn + "_q" + S(q), q, r, a, b);
    }
  }

  // SEAL's DyadicMultiply: 3 moduli, n = 2^12 .. 2^15; operands hold 2 polynomials, the result 3
  for (uint64_t n = 1 << 12; n <= (1 << 15); n <<= 1)
    for (size_t bits : {30, 50, 60}) {
      const Words mods = GeneratePrimes(3, bits, false, n);
      Words a(2 * 3 * n), b(2 * 3 * n), r(3 * 3 * n, 0);
      for (uint64_t p = 0; p < 2; ++p)
        for (uint64_t i = 0; i < 3; ++i) {
          const Words x = Operand(n, mods[i], n + 100 * p + i), y = Operand(n, mods[i], n + 100 * p + i + 50);
          std::copy(x.begin(), x.end(), a.begin() + (p * 3 + i) * n);
          std::copy(y.begin(), y.end(), b.begin() + (p * 3 + i) * n);
        }
      DyadicMultiply(r.data(), a.data(), b.data(), n, mods.data(), 3);
      Exact("DyadicMultiply_n" + S(n) + "_bits" + S(bits), r, mods[2]);
      if (n == (1 << 12)) {
        Words r2(3 * 3 * n, 0);
        internal::DyadicMultiply(r2.data(), a.data(), b.data(), n, mods.data(), 3);
        Exact("internal_DyadicMultiply_n" + S(n) + "_bits" + S(bits), r2, mods[2]);
      }
    }
}

// SEAL's KeySwitch: the reference known answer's shape (n = 16, decomp 2, three key moduli) and n = 2^12, decomp 3
void KeySwitches() {
  struct Shape {
    uint64_t n, decomp, bits;
  } shapes[] = {{16, 2, 59}, {1 << 12, 3, 50}, {1 << 12, 3, 59}};
  for (const Shape& s : shapes) {
    const uint64_t n = s.n, decomp = s.decomp, kms = decomp + 1, rns = decomp + 1, kcc = 2;
    const Words moduli = GeneratePrimes(kms, s.bits, true, n);
    std::vector<Words> keys(decomp);
    std::vector<const uint64_t*> key_ptrs(decomp);
    for (uint64_t j = 0; j < decomp; ++j) {
      for (uint64_t k = 0; k < kcc; ++k)
        for (uint64_t i = 0; i < kms; ++i) {
          const Words w = Operand(n, moduli[i], 1000 * j + 10 * k + i);
          keys[j].insert(keys[j].end(), w.begin(), w.end());
        }
      key_ptrs[j] = keys[j].data();
    }
    Words t, result, modswitch(decomp);
    for (uint64_t j = 0; j < decomp; ++j) {
      const Words w = Operand(n, moduli[j], 77 + j);
      t.insert(t.end(), w.begin(), w.end());
      modswitch[j] = InverseMod(moduli[kms - 1] % moduli[j], moduli[j]);
    }
    for (uint64_t k = 0; k < kcc; ++k)
      for (uint64_t i = 0; i < decomp; ++i) {
        const Words w = Operand(n, moduli[i], 500 + 10 * k + i);
        result.insert(result.end(), w.begin(), w.end());
      }
    Words result2 = result;
    KeySwitch(result.data(), t.data(), n, decomp, kms, rns, kcc, moduli.data(), key_ptrs.data(), modswitch.data());
    Exact("KeySwitch_n" + S(n) + "_decomp" + S(decomp) + "_bits" + S(s.bits), result, moduli[0]);
    if (n == 16) {
      internal::KeySwitch(result2.data(), t.data(), n, decomp, kms, rns, kcc, moduli.data(), key_ptrs.data(),
                          modswitch.data());
      Exact("internal_KeySwitch_n" + S(n) + "_decomp" + S(decomp) + "_bits" + S(s.bits), result2, moduli[0]);
    }
  }
}

}  // namespace

int main(int argc, char** argv) {
  if (argc < 2) {
    std::fprintf(stderr, "usage: %s <outdir> [--host-only]\n", argv[0]);
    return 2;
  }
  g_dir = argv[1];
  const bool host_only = argc > 2 && std::strcmp(argv[2], "--host-only") == 0;
  g_index = std::fopen((g_dir + "/index.txt").c_str(), "w");
  if (!g_index) {
    std::fprintf(stderr, "cannot write %s/index.txt\n", argv[1]);
    return 2;
  }
  const Words moduli = EdgeModuli();
  Exact("EdgeModuli", moduli);
  InlineArithmetic(moduli);
  ReachableNames();
  NumberTheory(moduli);
  NttHost();
  if (!host_only) {
    Transforms();
    Eltwise();
    KeySwitches();
  }
  std::fclose(g_index);
  std::printf("%zu records\n", g_records);
  return 0;
}
