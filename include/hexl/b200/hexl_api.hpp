// intel::hexl source-compatible API on top of libhexl_b200.so.
//
// This single header re-creates the public surface of the reference's
// hexl/include/hexl/ tree for the NTT + Eltwise*Mod hot path (class NTT, the
// Eltwise* free functions, CMPINT, the allocator hooks, the number-theory
// helpers those signatures mention).  Every compute entry point is an inline
// forwarder to the extern "C" ABI in include/hexl_b200.h; nothing is computed
// on the CPU except O(1) scalar helpers and one-off table construction.  The
// per-file headers a reference user includes (hexl/hexl.hpp, hexl/ntt/ntt.hpp,
// hexl/eltwise/eltwise-*.hpp, ...) are one-line includes of this file.
//
// Differences a caller can observe (see INTEGRATION.md):
//  * buffers may be host OR device pointers;
//  * failures (bad arguments -- the reference's HEXL_CHECK conditions -- and CUDA
//    errors) always throw std::runtime_error; the reference throws only in
//    HEXL_DEBUG builds and is undefined otherwise;
//  * NTT::ComputeForward/Inverse and Eltwise* gain optional trailing
//    `batch` / `stream` arguments (defaults keep the reference signatures).
#pragma once

#include <stdint.h>

#include <cmath>
#include <cstdlib>
#include <functional>
#include <limits>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../hexl_b200.h"

#ifndef HEXL_UNUSED
#define HEXL_UNUSED(x) (void)(x)
#endif
// The reference's HEXL_CHECK macros compile to nothing in release builds
// (hexl/include/hexl/util/check.hpp:37-42); argument checking lives behind the ABI.
#ifndef HEXL_CHECK
#define HEXL_CHECK(cond, expr) \
  {}
#define HEXL_CHECK_BOUNDS(...) \
  {}
#endif
#ifndef HEXL_VLOG
#define HEXL_VLOG(N, rest) \
  {}
#endif
// hexl/include/hexl/util/gcc.hpp:55-56
#ifndef HEXL_LOOP_UNROLL_4
#define HEXL_LOOP_UNROLL_4 _Pragma("GCC unroll 4")
#define HEXL_LOOP_UNROLL_8 _Pragma("GCC unroll 8")
#endif

namespace intel {
namespace hexl {

namespace b200_detail {
inline void Throw(int status) {
  if (status != 0) throw std::runtime_error(std::string("hexl-b200: ") + hexl_b200_last_error());
}
}  // namespace b200_detail

// ------------------------------------------------------------------- types
// hexl/include/hexl/util/types.hpp:10-13
#if defined(__SIZEOF_INT128__)
__extension__ typedef __int128 int128_t;
__extension__ typedef unsigned __int128 uint128_t;
#endif

// -------------------------------------------------------------------- CMPINT
// hexl/include/hexl/util/util.hpp:16-50
#undef TRUE
#undef FALSE
enum class CMPINT { EQ = 0, LT = 1, LE = 2, FALSE = 3, NE = 4, NLT = 5, NLE = 6, TRUE = 7 };

inline CMPINT Not(CMPINT cmp) {
  // the predicates pair up as (k, k ^ 4)
  int k = static_cast<int>(cmp);
  return (k >= 0 && k <= 7) ? static_cast<CMPINT>(k ^ 4) : CMPINT::FALSE;
}

// ---------------------------------------------------------------- allocators
// hexl/include/hexl/util/allocator.hpp:12-51
struct AllocatorBase {
  virtual ~AllocatorBase() noexcept {}
  virtual void* allocate(size_t bytes_count) = 0;
  virtual void deallocate(void* p, size_t n) = 0;
};

template <class AllocatorImpl>
struct AllocatorInterface : public AllocatorBase {
  void* allocate(size_t bytes_count) override {
    return static_cast<AllocatorImpl*>(this)->allocate_impl(bytes_count);
  }
  void deallocate(void* p, size_t n) override { static_cast<AllocatorImpl*>(this)->deallocate_impl(p, n); }

 private:
  void* allocate_impl(size_t) { return nullptr; }
  void deallocate_impl(void*, size_t) {}
};

// hexl/include/hexl/util/aligned-allocator.hpp:18-107
struct MallocStrategy : AllocatorBase {
  void* allocate(size_t bytes_count) final { return std::malloc(bytes_count); }
  void deallocate(void* p, size_t) final { std::free(p); }
};

using AllocatorStrategyPtr = std::shared_ptr<AllocatorBase>;

// GPU-aware strategies for the same hook (not in the reference).  Buffers of an
// AlignedVector64 built on PinnedStrategy stream over PCIe at full rate through the
// host-pointer path; buffers built on ManagedStrategy are unified memory and are
// worked on in place by the kernels, no staging copy at all:
//   AlignedVector64<uint64_t> v(n, 0, AlignedAllocator<uint64_t, 64>(std::make_shared<b200::ManagedStrategy>()));
namespace b200 {
struct PinnedStrategy : AllocatorBase {
  void* allocate(size_t bytes_count) final { return hexl_b200_host_alloc(bytes_count); }
  void deallocate(void* p, size_t) final { hexl_b200_host_free(p); }
};
struct ManagedStrategy : AllocatorBase {
  void* allocate(size_t bytes_count) final { return hexl_b200_managed_alloc(bytes_count); }
  void deallocate(void* p, size_t) final { hexl_b200_managed_free(p); }
};
}  // namespace b200

inline AllocatorStrategyPtr& DefaultMallocStrategy() {
  static AllocatorStrategyPtr s = AllocatorStrategyPtr(new MallocStrategy);
  return s;
}
// the reference exposes this as an extern global (ntt-internal.cpp:22)
static AllocatorStrategyPtr& mallocStrategy = DefaultMallocStrategy();

template <typename T, uint64_t Alignment>
class AlignedAllocator {
 public:
  template <typename, uint64_t>
  friend class AlignedAllocator;
  using value_type = T;

  explicit AlignedAllocator(AllocatorStrategyPtr strategy = nullptr) noexcept
      : m_alloc_impl(strategy ? strategy : DefaultMallocStrategy()) {}
  AlignedAllocator(const AlignedAllocator&) = default;
  AlignedAllocator& operator=(const AlignedAllocator&) = default;
  template <typename U>
  AlignedAllocator(const AlignedAllocator<U, Alignment>& src) : m_alloc_impl(src.m_alloc_impl) {}
  ~AlignedAllocator() {}

  template <typename U>
  struct rebind {
    using other = AlignedAllocator<U, Alignment>;
  };
  bool operator==(const AlignedAllocator&) { return true; }
  bool operator!=(const AlignedAllocator&) { return false; }

  // Over-allocate by Alignment + one pointer; remember the raw block just below
  // the aligned address so deallocate can hand it back to the strategy.
  T* allocate(size_t n) {
    if (Alignment == 0 || (Alignment & (Alignment - 1))) return nullptr;
    const size_t payload = sizeof(T) * n;
    char* raw = static_cast<char*>(m_alloc_impl->allocate(payload + Alignment + sizeof(void*)));
    if (!raw) return nullptr;
    uintptr_t a = reinterpret_cast<uintptr_t>(raw + sizeof(void*));
    a = (a + Alignment - 1) & ~static_cast<uintptr_t>(Alignment - 1);
    reinterpret_cast<void**>(a)[-1] = raw;
    return reinterpret_cast<T*>(a);
  }
  void deallocate(T* p, size_t n) {
    if (p) m_alloc_impl->deallocate(reinterpret_cast<void**>(p)[-1], n);
  }

 private:
  AllocatorStrategyPtr m_alloc_impl;
};

template <typename T>
using AlignedVector64 = std::vector<T, AlignedAllocator<T, 64>>;

// ------------------------------------------------------------- number theory
// hexl/include/hexl/util/gcc.hpp:14-60 (128-bit helpers) and
// hexl/include/hexl/number-theory/number-theory.hpp
inline uint64_t MSB(uint64_t input) { return input ? 63u - static_cast<uint64_t>(__builtin_clzll(input)) : 0; }
inline bool IsPowerOfTwo(uint64_t num) { return num && !(num & (num - 1)); }
inline uint64_t Log2(uint64_t x) { return MSB(x); }
inline bool IsPowerOfFour(uint64_t num) { return IsPowerOfTwo(num) && (Log2(num) % 2 == 0); }
inline uint64_t MaximumValue(uint64_t bits) {
  return bits >= 64 ? (std::numeric_limits<uint64_t>::max)() : (1ULL << bits) - 1;
}

#if defined(__SIZEOF_INT128__)
inline uint128_t MultiplyUInt64(uint64_t x, uint64_t y) { return uint128_t(x) * y; }
inline void MultiplyUInt64(uint64_t x, uint64_t y, uint64_t* prod_hi, uint64_t* prod_lo) {
  uint128_t p = uint128_t(x) * y;
  *prod_hi = static_cast<uint64_t>(p >> 64);
  *prod_lo = static_cast<uint64_t>(p);
}
template <int BitShift>
inline uint64_t MultiplyUInt64Hi(uint64_t x, uint64_t y) {
  return static_cast<uint64_t>((uint128_t(x) * y) >> BitShift);
}
inline uint64_t BarrettReduce128(uint64_t input_hi, uint64_t input_lo, uint64_t modulus) {
  return static_cast<uint64_t>(((uint128_t(input_hi) << 64) | input_lo) % modulus);
}
inline uint64_t DivideUInt128UInt64Lo(uint64_t x1, uint64_t x0, uint64_t y) {
  return static_cast<uint64_t>(((uint128_t(x1) << 64) | x0) / y);
}
#endif

inline uint64_t ReverseBits(uint64_t x, uint64_t bit_width) { return hexl_b200_reverse_bits(x, bit_width); }
inline uint64_t InverseMod(uint64_t x, uint64_t modulus) { return hexl_b200_inverse_mod(x, modulus); }
inline uint64_t MultiplyMod(uint64_t x, uint64_t y, uint64_t modulus) { return hexl_b200_multiply_mod(x, y, modulus); }
inline uint64_t AddUIntMod(uint64_t x, uint64_t y, uint64_t modulus) { return hexl_b200_add_uint_mod(x, y, modulus); }
inline uint64_t SubUIntMod(uint64_t x, uint64_t y, uint64_t modulus) { return hexl_b200_sub_uint_mod(x, y, modulus); }
inline uint64_t PowMod(uint64_t base, uint64_t exp, uint64_t modulus) { return hexl_b200_pow_mod(base, exp, modulus); }
inline bool IsPrimitiveRoot(uint64_t root, uint64_t degree, uint64_t modulus) {
  return hexl_b200_is_primitive_root(root, degree, modulus) != 0;
}
inline uint64_t GeneratePrimitiveRoot(uint64_t degree, uint64_t modulus) {
  return hexl_b200_generate_primitive_root(degree, modulus);
}
inline uint64_t MinimalPrimitiveRoot(uint64_t degree, uint64_t modulus) {
  return hexl_b200_minimal_primitive_root(degree, modulus);
}
inline bool IsPrime(uint64_t n) { return hexl_b200_is_prime(n) != 0; }
inline std::vector<uint64_t> GeneratePrimes(size_t num_primes, size_t bit_size, bool prefer_small_primes,
                                            size_t ntt_size = 1) {
  std::vector<uint64_t> out(num_primes);
  int got = hexl_b200_generate_primes(out.data(), num_primes, bit_size, prefer_small_primes ? 1 : 0, ntt_size);
  if (got < 0) got = 0;
  out.resize(static_cast<size_t>(got));
  if (out.size() != num_primes) throw std::runtime_error("hexl-b200: Failed to find enough primes");
  return out;
}

// number-theory.hpp:19-51
class MultiplyFactor {
 public:
  MultiplyFactor() = default;
  MultiplyFactor(uint64_t operand, uint64_t bit_shift, uint64_t modulus)
      : m_operand(operand), m_barrett_factor(hexl_b200_multiply_factor(operand, bit_shift, modulus)) {}
  inline uint64_t BarrettFactor() const { return m_barrett_factor; }
  inline uint64_t Operand() const { return m_operand; }

 private:
  uint64_t m_operand = 0;
  uint64_t m_barrett_factor = 0;
};

#if defined(__SIZEOF_INT128__)
// number-theory.cpp:54-59
inline uint64_t MultiplyMod(uint64_t x, uint64_t y, uint64_t y_precon, uint64_t modulus) {
  uint64_t r = x * y - MultiplyUInt64Hi<64>(x, y_precon) * modulus;
  return r >= modulus ? r - modulus : r;
}
// number-theory.hpp:127-165
template <int BitShift>
inline uint64_t MultiplyModLazy(uint64_t x, uint64_t y_operand, uint64_t y_barrett_factor, uint64_t modulus) {
  return y_operand * x - MultiplyUInt64Hi<BitShift>(x, y_barrett_factor) * modulus;
}
template <int BitShift>
inline uint64_t MultiplyModLazy(uint64_t x, uint64_t y, uint64_t modulus) {
  return MultiplyModLazy<BitShift>(x, y, MultiplyFactor(y, BitShift, modulus).BarrettFactor(), modulus);
}
// number-theory.hpp:195-205
template <int OutputModFactor = 1>
uint64_t BarrettReduce64(uint64_t input, uint64_t modulus, uint64_t q_barr) {
  uint64_t r = input - MultiplyUInt64Hi<64>(input, q_barr) * modulus;
  if (OutputModFactor == 2) return r;
  return r >= modulus ? r - modulus : r;
}
#endif

inline unsigned char AddUInt64(uint64_t operand1, uint64_t operand2, uint64_t* result) {
  *result = operand1 + operand2;
  return static_cast<unsigned char>(*result < operand1);
}

// number-theory.hpp:214-258
template <int InputModFactor>
uint64_t ReduceMod(uint64_t x, uint64_t modulus, const uint64_t* twice_modulus = nullptr,
                   const uint64_t* four_times_modulus = nullptr) {
  if (InputModFactor >= 8 && x >= *four_times_modulus) x -= *four_times_modulus;
  if (InputModFactor >= 4 && x >= *twice_modulus) x -= *twice_modulus;
  if (InputModFactor >= 2 && x >= modulus) x -= modulus;
  return x;
}

// ----------------------------------------------------------------------- NTT
// hexl/include/hexl/ntt/ntt.hpp:22-293
class NTT {
 public:
  template <class Adaptee, class... Args>
  struct AllocatorAdapter : public AllocatorInterface<AllocatorAdapter<Adaptee, Args...>> {
    explicit AllocatorAdapter(Adaptee&& _a, Args&&... args);
    AllocatorAdapter(const Adaptee& _a, Args&... args);
    void* allocate_impl(size_t bytes_count);
    void deallocate_impl(void* p, size_t n);

   private:
    Adaptee alloc;
  };

  NTT() = default;
  ~NTT() { Drop(); }
  NTT(const NTT& o) : m_handle(o.m_handle), m_alloc(o.m_alloc), m_tables(o.m_tables) {
    if (m_handle) hexl_b200_ntt_retain(m_handle);
  }
  NTT(NTT&& o) noexcept : m_handle(o.m_handle), m_alloc(std::move(o.m_alloc)), m_tables(std::move(o.m_tables)) {
    o.m_handle = nullptr;
  }
  NTT& operator=(NTT o) noexcept {
    std::swap(m_handle, o.m_handle);
    std::swap(m_alloc, o.m_alloc);
    std::swap(m_tables, o.m_tables);
    return *this;
  }

  NTT(uint64_t degree, uint64_t q, std::shared_ptr<AllocatorBase> alloc_ptr = {}) : m_alloc(alloc_ptr) {
    b200_detail::Throw(hexl_b200_ntt_create(&m_handle, degree, q));
    InitTables();
  }
  template <class Allocator, class... AllocatorArgs>
  NTT(uint64_t degree, uint64_t q, Allocator&& a, AllocatorArgs&&... args)
      : NTT(degree, q,
            std::static_pointer_cast<AllocatorBase>(std::make_shared<AllocatorAdapter<Allocator, AllocatorArgs...>>(
                std::move(a), std::forward<AllocatorArgs>(args)...))) {}
  NTT(uint64_t degree, uint64_t q, uint64_t root_of_unity, std::shared_ptr<AllocatorBase> alloc_ptr = {})
      : m_alloc(alloc_ptr) {
    b200_detail::Throw(hexl_b200_ntt_create_with_root(&m_handle, degree, q, root_of_unity));
    InitTables();
  }
  template <class Allocator, class... AllocatorArgs>
  NTT(uint64_t degree, uint64_t q, uint64_t root_of_unity, Allocator&& a, AllocatorArgs&&... args)
      : NTT(degree, q, root_of_unity,
            std::static_pointer_cast<AllocatorBase>(std::make_shared<AllocatorAdapter<Allocator, AllocatorArgs...>>(
                std::move(a), std::forward<AllocatorArgs>(args)...))) {}

  static bool CheckArguments(uint64_t degree, uint64_t modulus) {
    return hexl_b200_ntt_check_arguments(degree, modulus) != 0;
  }

  // The reference signature is the first four parameters; `batch` polynomials
  // back to back and the CUDA stream (device pointers) are extensions.
  void ComputeForward(uint64_t* result, const uint64_t* operand, uint64_t input_mod_factor,
                      uint64_t output_mod_factor, uint64_t batch = 1, void* stream = nullptr) {
    b200_detail::Throw(
        hexl_b200_ntt_forward(m_handle, result, operand, input_mod_factor, output_mod_factor, batch, stream));
  }
  void ComputeInverse(uint64_t* result, const uint64_t* operand, uint64_t input_mod_factor,
                      uint64_t output_mod_factor, uint64_t batch = 1, void* stream = nullptr) {
    b200_detail::Throw(
        hexl_b200_ntt_inverse(m_handle, result, operand, input_mod_factor, output_mod_factor, batch, stream));
  }

  // RNS batches in one launch (not in the reference, which needs one call per polynomial and
  // modulus): of the count * batch_per_modulus polynomials laid out back to back, polynomial u
  // is transformed under ntts[u / batch_per_modulus].
  static void ComputeForwardMulti(const NTT* const* ntts, size_t count, uint64_t* result, const uint64_t* operand,
                                  uint64_t input_mod_factor, uint64_t output_mod_factor,
                                  uint64_t batch_per_modulus = 1, void* stream = nullptr) {
    std::vector<hexl_b200_ntt*> hs(count);
    for (size_t i = 0; i < count; ++i) hs[i] = ntts[i]->m_handle;
    b200_detail::Throw(hexl_b200_ntt_forward_multi(hs.data(), count, result, operand, input_mod_factor,
                                                   output_mod_factor, batch_per_modulus, stream));
  }
  static void ComputeInverseMulti(const NTT* const* ntts, size_t count, uint64_t* result, const uint64_t* operand,
                                  uint64_t input_mod_factor, uint64_t output_mod_factor,
                                  uint64_t batch_per_modulus = 1, void* stream = nullptr) {
    std::vector<hexl_b200_ntt*> hs(count);
    for (size_t i = 0; i < count; ++i) hs[i] = ntts[i]->m_handle;
    b200_detail::Throw(hexl_b200_ntt_inverse_multi(hs.data(), count, result, operand, input_mod_factor,
                                                   output_mod_factor, batch_per_modulus, stream));
  }

  // result = InvNTT(FwdNTT(a) .* FwdNTT(b)) for count * batch_per_modulus polynomials (negacyclic
  // products, polynomial u under ntts[u / batch_per_modulus]): the FwdNTT -> EltwiseMultMod -> InvNTT
  // pipeline as one call and a handful of launches.  result may be a, b or a separate buffer, and a may be b
  // (a square), with or without result.
  static void PolyMultiplyMulti(const NTT* const* ntts, size_t count, uint64_t* result, const uint64_t* a,
                                const uint64_t* b, uint64_t batch_per_modulus = 1, void* stream = nullptr) {
    std::vector<hexl_b200_ntt*> hs(count);
    for (size_t i = 0; i < count; ++i) hs[i] = ntts[i]->m_handle;
    b200_detail::Throw(hexl_b200_poly_multiply_multi(hs.data(), count, result, a, b, batch_per_modulus, stream));
  }

  uint64_t GetMinimalRootOfUnity() const { return hexl_b200_ntt_minimal_root(m_handle); }
  uint64_t GetDegree() const { return hexl_b200_ntt_degree(m_handle); }
  uint64_t GetModulus() const { return hexl_b200_ntt_modulus(m_handle); }

  const AlignedVector64<uint64_t>& GetRootOfUnityPowers() const { return m_tables->w; }
  uint64_t GetRootOfUnityPower(size_t i) { return GetRootOfUnityPowers()[i]; }
  const AlignedVector64<uint64_t>& GetPrecon32RootOfUnityPowers() const { return Lazy(m_tables->w32, m_tables->w, 32); }
  const AlignedVector64<uint64_t>& GetPrecon64RootOfUnityPowers() const { return m_tables->w64; }
  const AlignedVector64<uint64_t>& GetAVX512RootOfUnityPowers() const { return Avx(); }
  const AlignedVector64<uint64_t>& GetAVX512Precon32RootOfUnityPowers() const { return Lazy(m_tables->a32, Avx(), 32); }
  const AlignedVector64<uint64_t>& GetAVX512Precon52RootOfUnityPowers() const { return Lazy(m_tables->a52, Avx(), 52); }
  const AlignedVector64<uint64_t>& GetAVX512Precon64RootOfUnityPowers() const { return Lazy(m_tables->a64, Avx(), 64); }
  const AlignedVector64<uint64_t>& GetInvRootOfUnityPowers() const { return m_tables->iw; }
  uint64_t GetInvRootOfUnityPower(size_t i) { return GetInvRootOfUnityPowers()[i]; }
  const AlignedVector64<uint64_t>& GetPrecon32InvRootOfUnityPowers() const { return Lazy(m_tables->iw32, m_tables->iw, 32); }
  const AlignedVector64<uint64_t>& GetPrecon52InvRootOfUnityPowers() const { return Lazy(m_tables->iw52, m_tables->iw, 52); }
  const AlignedVector64<uint64_t>& GetPrecon64InvRootOfUnityPowers() const { return m_tables->iw64; }

  static size_t MaxDegreeBits() { return 20; }
  static size_t MaxModulusBits() { return 62; }
  static const size_t s_default_shift_bits{64};
  static const size_t s_ifma_shift_bits{52};
  static const size_t s_max_fwd_32_modulus{1ULL << (32 - 2)};
  static const size_t s_max_inv_32_modulus{1ULL << (32 - 2)};
  static const size_t s_max_fwd_ifma_modulus{1ULL << (s_ifma_shift_bits - 2)};
  static const size_t s_max_inv_ifma_modulus{1ULL << (s_ifma_shift_bits - 2)};
  static const size_t s_max_inv_dq_modulus{1ULL << (s_default_shift_bits - 2)};
  static size_t s_max_fwd_modulus(int bit_shift) { return ModulusCap(bit_shift); }
  static size_t s_max_inv_modulus(int bit_shift) { return ModulusCap(bit_shift); }

  // extension: the underlying C handle (e.g. to pass across an FFI)
  hexl_b200_ntt* Handle() const { return m_handle; }
  // extension: upload the tables to `device` (-1 = current) now, e.g. before capturing calls into a CUDA graph
  void Prepare(int device = -1) { b200_detail::Throw(hexl_b200_ntt_prepare(m_handle, device)); }
  // extension: the process-wide cached object for (N, modulus) -- GetNTT below
  static NTT FromCache(uint64_t degree, uint64_t q) {
    NTT t;
    b200_detail::Throw(hexl_b200_ntt_get_cached(&t.m_handle, degree, q));
    t.InitTables();
    return t;
  }

 private:
  using Vec = AlignedVector64<uint64_t>;
  struct Tables {
    explicit Tables(const AlignedAllocator<uint64_t, 64>& a)
        : w(a), w64(a), iw(a), iw64(a), w32(a), iw32(a), iw52(a), avx(a), a32(a), a52(a), a64(a) {}
    Vec w, w64, iw, iw64;                      // filled at construction
    Vec w32, iw32, iw52, avx, a32, a52, a64;   // filled on first use
    uint64_t q = 0;
    std::mutex mu;
  };

  static size_t ModulusCap(int bit_shift) {
    if (bit_shift == 32) return s_max_fwd_32_modulus;
    if (bit_shift == 52) return s_max_fwd_ifma_modulus;
    if (bit_shift == 64) return 1ULL << MaxModulusBits();
    return 0;
  }
  void Drop() {
    if (m_handle) hexl_b200_ntt_release(m_handle);
    m_handle = nullptr;
  }
  void InitTables() {
    AlignedAllocator<uint64_t, 64> a(m_alloc);
    m_tables = std::make_shared<Tables>(a);
    m_tables->q = GetModulus();
    const uint64_t n = GetDegree();
    Vec* dst[4] = {&m_tables->w, &m_tables->w64, &m_tables->iw, &m_tables->iw64};
    for (int k = 0; k < 4; ++k) {
      const uint64_t* src = hexl_b200_ntt_table(m_handle, k);
      dst[k]->assign(src, src + n);
    }
  }
  // floor(v * 2^shift / q) for every entry (ntt-internal.cpp:113-139)
  const Vec& Lazy(Vec& out, const Vec& in, uint64_t shift) const {
    std::lock_guard<std::mutex> lk(m_tables->mu);
    if (out.empty() && !in.empty()) {
      out.reserve(in.size());
      for (uint64_t v : in) out.push_back(hexl_b200_multiply_factor(v, shift, m_tables->q));
    }
    return out;
  }
  // the reference's AVX-512 table: entries [N/8,N/4) x4 and [N/4,N/2) x2 (ntt-internal.cpp:75-111)
  const Vec& Avx() const {
    std::lock_guard<std::mutex> lk(m_tables->mu);
    Vec& out = m_tables->avx;
    if (out.empty()) {
      const Vec& w = m_tables->w;
      const size_t n = w.size();
      for (size_t i = 0; i < n; ++i) {
        const size_t copies = (i >= n / 8 && i < n / 4) ? 4 : ((i >= n / 4 && i < n / 2) ? 2 : 1);
        for (size_t c = 0; c < copies; ++c) out.push_back(w[i]);
      }
    }
    return out;
  }

  hexl_b200_ntt* m_handle = nullptr;
  std::shared_ptr<AllocatorBase> m_alloc;
  std::shared_ptr<Tables> m_tables;
};

// ------------------------------------------------------------------ eltwise
// hexl/include/hexl/eltwise/eltwise-add-mod.hpp:22,36
inline void EltwiseAddMod(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2, uint64_t n,
                          uint64_t modulus, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_eltwise_add_mod(result, operand1, operand2, n, modulus, stream));
}
inline void EltwiseAddMod(uint64_t* result, const uint64_t* operand1, uint64_t operand2, uint64_t n, uint64_t modulus,
                          void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_eltwise_add_mod_scalar(result, operand1, operand2, n, modulus, stream));
}
// hexl/include/hexl/eltwise/eltwise-sub-mod.hpp:22,36
inline void EltwiseSubMod(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2, uint64_t n,
                          uint64_t modulus, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_eltwise_sub_mod(result, operand1, operand2, n, modulus, stream));
}
inline void EltwiseSubMod(uint64_t* result, const uint64_t* operand1, uint64_t operand2, uint64_t n, uint64_t modulus,
                          void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_eltwise_sub_mod_scalar(result, operand1, operand2, n, modulus, stream));
}
// hexl/include/hexl/eltwise/eltwise-mult-mod.hpp:23
// Exact for every accepted input (q < 2^62, input_mod_factor * q < 2^63).  For 62-bit moduli the generalised Barrett
// quotient estimate can be low by two and the product takes a second conditional subtraction; the reference's scalar
// tier takes one and returns words in [q, 2q) for some operands near q at some moduli above about 2^61.7.
inline void EltwiseMultMod(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2, uint64_t n,
                           uint64_t modulus, uint64_t input_mod_factor, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_eltwise_mult_mod(result, operand1, operand2, n, modulus, input_mod_factor, stream));
}
// hexl/include/hexl/eltwise/eltwise-fma-mod.hpp:22
inline void EltwiseFMAMod(uint64_t* result, const uint64_t* arg1, uint64_t arg2, const uint64_t* arg3, uint64_t n,
                          uint64_t modulus, uint64_t input_mod_factor, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_eltwise_fma_mod(result, arg1, arg2, arg3, n, modulus, input_mod_factor, stream));
}
// hexl/include/hexl/eltwise/eltwise-reduce-mod.hpp:24
// Exact for every modulus above 1.  For q >= 2^63 every 64-bit word is below 2q, so input_mod_factor 4 is treated as
// 2; every tier of the reference subtracts 2q there, which wraps.
inline void EltwiseReduceMod(uint64_t* result, const uint64_t* operand, uint64_t n, uint64_t modulus,
                             uint64_t input_mod_factor, uint64_t output_mod_factor, void* stream = nullptr) {
  b200_detail::Throw(
      hexl_b200_eltwise_reduce_mod(result, operand, n, modulus, input_mod_factor, output_mod_factor, stream));
}
// hexl/include/hexl/eltwise/eltwise-cmp-add.hpp:22
inline void EltwiseCmpAdd(uint64_t* result, const uint64_t* operand1, uint64_t n, CMPINT cmp, uint64_t bound,
                          uint64_t diff, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_eltwise_cmp_add(result, operand1, n, static_cast<int>(cmp), bound, diff, stream));
}
// hexl/include/hexl/eltwise/eltwise-cmp-sub-mod.hpp:24
inline void EltwiseCmpSubMod(uint64_t* result, const uint64_t* operand1, uint64_t n, uint64_t modulus, CMPINT cmp,
                             uint64_t bound, uint64_t diff, void* stream = nullptr) {
  b200_detail::Throw(
      hexl_b200_eltwise_cmp_sub_mod(result, operand1, n, modulus, static_cast<int>(cmp), bound, diff, stream));
}

// Montgomery-form helpers.  In the reference the element-wise ones are internal AVX-512 templates on <BitShift, r>
// (hexl/eltwise/eltwise-reduce-mod-avx512.hpp:156-352); here r is a run-time argument and BitShift is 64.
inline uint64_t HenselLemma2adicRoot(uint32_t r, uint64_t q) { return hexl_b200_hensel_lemma_2adic_root(r, q); }
#if defined(__SIZEOF_INT128__)
// number-theory.hpp:269-301, inline like the reference's, for every r with q < 2^r <= 2^63: T * 2^-r mod q for
// T = T_hi * 2^64 + T_lo < q * 2^r, by REDC on the 128-bit sum T + m * q (below 2^128 because q * 2^r < 2^127).
template <int BitShift>
inline uint64_t MontgomeryReduce(uint64_t T_hi, uint64_t T_lo, uint64_t q, int r, uint64_t mod_R_msk,
                                 uint64_t inv_mod) {
  static_assert(BitShift == 64, "only the 64-bit form exists on the GPU path");
  const uint64_t m = ((T_lo & mod_R_msk) * inv_mod) & mod_R_msk;
  const uint64_t s = static_cast<uint64_t>((((uint128_t(T_hi) << 64) | T_lo) + uint128_t(m) * q) >> r);
  return s >= q ? s - q : s;
}
#endif
inline void EltwiseMontReduceMod(uint64_t* result, const uint64_t* a, const uint64_t* b, uint64_t n, uint64_t modulus,
                                 int r, uint64_t neg_inv_mod, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_eltwise_mont_reduce_mod(result, a, b, n, modulus, r, neg_inv_mod, stream));
}
inline void EltwiseMontgomeryFormIn(uint64_t* result, const uint64_t* a, uint64_t R2_mod_q, uint64_t n, uint64_t modulus,
                                    int r, uint64_t neg_inv_mod, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_eltwise_montgomery_form_in(result, a, R2_mod_q, n, modulus, r, neg_inv_mod, stream));
}
inline void EltwiseMontgomeryFormOut(uint64_t* result, const uint64_t* a, uint64_t n, uint64_t modulus, int r,
                                     uint64_t neg_inv_mod, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_eltwise_montgomery_form_out(result, a, n, modulus, r, neg_inv_mod, stream));
}

// ------------------------------------------------ SEAL-shaped composites
// hexl/include/hexl/experimental/seal/ntt-cache.hpp:27-53.  The reference returns
// NTT& into a process-wide map; here the cache lives behind the ABI and a cheap
// handle copy is returned.
inline NTT GetNTT(size_t N, uint64_t modulus) { return NTT::FromCache(N, modulus); }

// hexl/include/hexl/experimental/seal/ntt-cache.hpp:13-25: the key hash of the reference's cache map
struct HashPair {
  template <class T1, class T2>
  std::size_t operator()(const std::pair<T1, T2>& p) const {
    return hash_combine(std::hash<T1>{}(p.first), std::hash<T2>{}(p.second));
  }
  static std::size_t hash_combine(std::size_t lhs, std::size_t rhs) {
    return lhs ^ (rhs + 0x9e3779b9 + (lhs << 6) + (lhs >> 2));
  }
};

// hexl/include/hexl/experimental/seal/locks.hpp: the reader-writer lock the reference's cache is guarded by
using Lock = std::shared_mutex;
using WriteLock = std::unique_lock<Lock>;
using ReadLock = std::shared_lock<Lock>;
class RWLock {
 public:
  RWLock() = default;
  RWLock(const RWLock&) = delete;
  RWLock& operator=(const RWLock&) = delete;
  ReadLock AcquireRead() { return ReadLock(m_mutex); }
  WriteLock AcquireWrite() { return WriteLock(m_mutex); }
  ReadLock TryAcquireRead() noexcept { return ReadLock(m_mutex, std::try_to_lock); }
  WriteLock TryAcquireWrite() noexcept { return WriteLock(m_mutex, std::try_to_lock); }

 private:
  Lock m_mutex{};
};

// hexl/include/hexl/experimental/seal/dyadic-multiply.hpp:26
// Exact for every modulus below 2^62, like EltwiseMultMod: for 62-bit moduli the products take the second conditional
// subtraction the reference's scalar tier lacks.
inline void DyadicMultiply(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2, uint64_t n,
                           const uint64_t* moduli, uint64_t num_moduli, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_dyadic_multiply(result, operand1, operand2, n, moduli, num_moduli, stream));
}

// hexl/include/hexl/experimental/seal/key-switch.hpp:34
// Every modulus the switch uses must be below 2^61.  The result is exact for every accepted input; it differs from the
// reference only where the reference's unreduced 128-bit sum of digit x key products wraps (moduli above 2^60 with
// more than floor((2^128 - 1) / ((4q - 1)(q - 1))) digits, 16 just below 2^61).  The same holds for the resident-key
// overload below.
inline void KeySwitch(uint64_t* result, const uint64_t* t_target_iter_ptr, uint64_t n, uint64_t decomp_modulus_size,
                      uint64_t key_modulus_size, uint64_t rns_modulus_size, uint64_t key_component_count,
                      const uint64_t* moduli, const uint64_t** k_switch_keys, const uint64_t* modswitch_factors,
                      const uint64_t* root_of_unity_powers_ptr = nullptr, void* stream = nullptr) {
  if (root_of_unity_powers_ptr != nullptr)  // key-switch-internal.cpp:31-34
    throw std::invalid_argument("Parameter root_of_unity_powers_ptr is not supported yet.");
  b200_detail::Throw(hexl_b200_key_switch(result, t_target_iter_ptr, n, decomp_modulus_size, key_modulus_size,
                                          rns_modulus_size, key_component_count, moduli, k_switch_keys,
                                          modswitch_factors, stream));
}

// hexl/include/hexl/experimental/seal/{dyadic-multiply,key-switch}-internal.hpp, which the reference's hexl.hpp
// includes: the same operations under intel::hexl::internal
namespace internal {
inline void DyadicMultiply(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2, uint64_t n,
                           const uint64_t* moduli, uint64_t num_moduli) {
  intel::hexl::DyadicMultiply(result, operand1, operand2, n, moduli, num_moduli);
}
inline void KeySwitch(uint64_t* result, const uint64_t* t_target_iter_ptr, uint64_t n, uint64_t decomp_modulus_size,
                      uint64_t key_modulus_size, uint64_t rns_modulus_size, uint64_t key_component_count,
                      const uint64_t* moduli, const uint64_t** k_switch_keys, const uint64_t* modswitch_factors,
                      const uint64_t* root_of_unity_powers_ptr = nullptr) {
  intel::hexl::KeySwitch(result, t_target_iter_ptr, n, decomp_modulus_size, key_modulus_size, rns_modulus_size,
                         key_component_count, moduli, k_switch_keys, modswitch_factors, root_of_unity_powers_ptr);
}
}  // namespace internal

// extension: rescale by the last RNS modulus, SEAL's RNSTool::divide_and_round_q_last(_ntt)_inplace batched over
// `count` polynomials of rns_modulus_size limbs each (hexl_b200_divide_and_round_q_last in include/hexl_b200.h has the
// layout and the argument rules).  Limb rns_modulus_size - 1 of result is not written; result may be operand.
inline void DivideAndRoundQLast(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                                uint64_t rns_modulus_size, uint64_t count, bool ntt_form, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_divide_and_round_q_last(result, operand, n, moduli, rns_modulus_size, count,
                                                       ntt_form ? 1 : 0, stream));
}

// extension: key-switch keys resident on the GPU(s).  The reference reads the keys from caller memory on every
// call (key-switch.hpp:34-39); a host caller uploads them once here and then switches any number of
// ciphertexts (`batch` of them back to back per call) without the keys crossing PCIe again.
namespace b200 {
class KeySwitchKeys {
 public:
  KeySwitchKeys() = default;
  // sharded_by_modulus: the RNS moduli of ONE switch are spread over the devices of hexl_b200_set_host_devices
  // (digit all-gather + special-prime broadcast over NVLink); lowers the latency of a single switch on host buffers
  KeySwitchKeys(const uint64_t** k_switch_keys, uint64_t n, uint64_t decomp_modulus_size, uint64_t key_modulus_size,
                uint64_t key_component_count, bool sharded_by_modulus = false) {
    b200_detail::Throw((sharded_by_modulus ? hexl_b200_keys_upload_sharded : hexl_b200_keys_upload)(
        &m_keys, k_switch_keys, n, decomp_modulus_size, key_modulus_size, key_component_count));
  }
  ~KeySwitchKeys() { hexl_b200_keys_release(m_keys); }
  KeySwitchKeys(KeySwitchKeys&& o) noexcept : m_keys(o.m_keys) { o.m_keys = nullptr; }
  KeySwitchKeys& operator=(KeySwitchKeys&& o) noexcept {
    std::swap(m_keys, o.m_keys);
    return *this;
  }
  KeySwitchKeys(const KeySwitchKeys&) = delete;
  KeySwitchKeys& operator=(const KeySwitchKeys&) = delete;
  const hexl_b200_keys* Handle() const { return m_keys; }

 private:
  hexl_b200_keys* m_keys = nullptr;
};
}  // namespace b200

inline void KeySwitch(uint64_t* result, const uint64_t* t_target_iter_ptr, uint64_t n, uint64_t decomp_modulus_size,
                      uint64_t key_modulus_size, uint64_t rns_modulus_size, uint64_t key_component_count,
                      const uint64_t* moduli, const b200::KeySwitchKeys& keys, const uint64_t* modswitch_factors,
                      uint64_t batch = 1, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_key_switch_resident(result, t_target_iter_ptr, n, decomp_modulus_size, key_modulus_size,
                                                   rns_modulus_size, key_component_count, moduli, keys.Handle(),
                                                   modswitch_factors, batch, stream));
}

// extension: the Galois automorphism a(X) -> a(X^galois_elt) of `count` polynomials of rns_modulus_size limbs each,
// in NTT or coefficient form (hexl_b200_apply_galois in include/hexl_b200.h has the layout, the formulas and the
// argument rules); result may be operand.
inline void ApplyGalois(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                        uint64_t rns_modulus_size, uint64_t count, uint64_t galois_elt, bool ntt_form,
                        void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_apply_galois(result, operand, n, moduli, rns_modulus_size, count, galois_elt,
                                            ntt_form ? 1 : 0, stream));
}

// extension: rotation or conjugation of `batch` ciphertexts in NTT form, in place -- SEAL's apply_galois_inplace:
// c0 <- sigma(c0) + KS_0(sigma(c1)), c1 <- KS_1(sigma(c1)) with the Galois keys of galois_elt
// (hexl_b200_apply_galois_key_switch).  key_component_count must be 2; sharded key handles are refused.
inline void ApplyGaloisKeySwitch(uint64_t* ciphertexts, uint64_t n, uint64_t decomp_modulus_size,
                                 uint64_t key_modulus_size, uint64_t rns_modulus_size, uint64_t key_component_count,
                                 const uint64_t* moduli, const b200::KeySwitchKeys& galois_keys,
                                 const uint64_t* modswitch_factors, uint64_t galois_elt, uint64_t batch = 1,
                                 void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_apply_galois_key_switch(ciphertexts, n, decomp_modulus_size, key_modulus_size,
                                                       rns_modulus_size, key_component_count, moduli,
                                                       galois_keys.Handle(), modswitch_factors, galois_elt, batch,
                                                       stream));
}

namespace b200 {
// extension: hoisted rotations -- each of `batch` ciphertexts rotated by every galois_elts[r] with *galois_keys[r],
// its digits decomposed once for all elements; rotation r of ciphertext c goes to
// results + (c * num_elts + r) * 2 * decomp_modulus_size * n (hexl_b200_apply_galois_key_switch_hoisted has the
// formula).  Not bit-identical to ApplyGaloisKeySwitch: the digits are lifted to signed integers under sigma_g (equal
// for g = 1; the same noise bound).  key_component_count must be 2; sharded key handles are refused.
inline void ApplyGaloisKeySwitchHoisted(uint64_t* results, const uint64_t* ciphertexts, uint64_t n,
                                        uint64_t decomp_modulus_size, uint64_t key_modulus_size,
                                        uint64_t rns_modulus_size, uint64_t key_component_count,
                                        const uint64_t* moduli, const KeySwitchKeys* const* galois_keys,
                                        const uint64_t* galois_elts, uint64_t num_elts,
                                        const uint64_t* modswitch_factors, uint64_t batch = 1,
                                        void* stream = nullptr) {
  std::vector<const hexl_b200_keys*> handles(num_elts);
  for (uint64_t r = 0; r < num_elts; ++r) handles[r] = galois_keys[r] ? galois_keys[r]->Handle() : nullptr;
  b200_detail::Throw(hexl_b200_apply_galois_key_switch_hoisted(
      results, ciphertexts, n, decomp_modulus_size, key_modulus_size, rns_modulus_size, key_component_count, moduli,
      handles.data(), galois_elts, num_elts, modswitch_factors, batch, stream));
}

// extension: fast base conversion of `count` polynomials from from_count moduli into to_count moduli, coefficient form
// (hexl_b200_fast_base_convert has the layout and the formula).  result and operand must not overlap.
inline void FastBaseConvert(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* from_moduli,
                            uint64_t from_count, const uint64_t* to_moduli, uint64_t to_count, uint64_t count = 1,
                            void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_fast_base_convert(result, operand, n, from_moduli, from_count, to_moduli, to_count,
                                                 count, stream));
}

// extension: hybrid key switch of `batch` ciphertexts at level level_size -- digits of digit_size data moduli and
// p_size special primes, moduli = data moduli then special primes; keys uploaded with decomp = ceil(q_size /
// digit_size) and key_modulus_size = q_size + p_size (hexl_b200_key_switch_hybrid has the definitions).  result
// (key_component_count x level_size limbs per ciphertext) is accumulated into.
inline void KeySwitchHybrid(uint64_t* result, const uint64_t* target, uint64_t n, uint64_t level_size, uint64_t q_size,
                            uint64_t p_size, uint64_t digit_size, uint64_t key_component_count, const uint64_t* moduli,
                            const KeySwitchKeys& keys, uint64_t batch = 1, void* stream = nullptr) {
  b200_detail::Throw(hexl_b200_key_switch_hybrid(result, target, n, level_size, q_size, p_size, digit_size,
                                                 key_component_count, moduli, keys.Handle(), batch, stream));
}

// extension: hoisted rotations with hybrid keys -- each of `batch` ciphertexts (2 x level_size limbs) rotated by every
// galois_elts[r] with *galois_keys[r] (hybrid keys, key_component_count 2), its mod-up done once for all elements;
// rotation r of ciphertext c goes to results + (c * num_elts + r) * 2 * level_size * n
// (hexl_b200_apply_galois_key_switch_hybrid_hoisted has the formula).  Not bit-identical to ApplyGalois followed by
// KeySwitchHybrid for g != 1 (signed digit lift, the same noise bound).
inline void ApplyGaloisKeySwitchHybridHoisted(uint64_t* results, const uint64_t* ciphertexts, uint64_t n,
                                              uint64_t level_size, uint64_t q_size, uint64_t p_size,
                                              uint64_t digit_size, const uint64_t* moduli,
                                              const KeySwitchKeys* const* galois_keys, const uint64_t* galois_elts,
                                              uint64_t num_elts, uint64_t batch = 1, void* stream = nullptr) {
  std::vector<const hexl_b200_keys*> handles(num_elts);
  for (uint64_t r = 0; r < num_elts; ++r) handles[r] = galois_keys[r] ? galois_keys[r]->Handle() : nullptr;
  b200_detail::Throw(hexl_b200_apply_galois_key_switch_hybrid_hoisted(results, ciphertexts, n, level_size, q_size,
                                                                      p_size, digit_size, moduli, handles.data(),
                                                                      galois_elts, num_elts, batch, stream));
}

// extension: sum_r w_r (.) Rot_{g_r}(ct) with hybrid keys and one mod-down for the whole sum, for each of `batch`
// ciphertexts; diagonals holds num_elts x (level_size + p_size) x n words in NTT form, and a null galois_keys[r] with
// galois_elts[r] = 1 is an identity term (hexl_b200_linear_transform_hybrid has the formula).
inline void LinearTransformHybrid(uint64_t* result, const uint64_t* ciphertexts, uint64_t n, uint64_t level_size,
                                  uint64_t q_size, uint64_t p_size, uint64_t digit_size, const uint64_t* moduli,
                                  const KeySwitchKeys* const* galois_keys, const uint64_t* galois_elts,
                                  uint64_t num_elts, const uint64_t* diagonals, uint64_t batch = 1,
                                  void* stream = nullptr) {
  std::vector<const hexl_b200_keys*> handles(num_elts);
  for (uint64_t r = 0; r < num_elts; ++r) handles[r] = galois_keys[r] ? galois_keys[r]->Handle() : nullptr;
  b200_detail::Throw(hexl_b200_linear_transform_hybrid(result, ciphertexts, n, level_size, q_size, p_size, digit_size,
                                                       moduli, handles.data(), galois_elts, num_elts, diagonals,
                                                       batch, stream));
}
}  // namespace b200

}  // namespace hexl
}  // namespace intel
