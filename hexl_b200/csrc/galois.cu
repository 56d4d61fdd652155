// The Galois automorphism sigma_g : a(X) -> a(X^g) (g odd, 1 <= g < 2n) of RNS polynomials, the permutation behind
// every CKKS / BFV / BGV rotation and conjugation (SEAL's Evaluator::apply_galois_inplace does it in a scalar loop;
// the reference has no counterpart).  Every kernel here is pure data movement: 16 B of HBM traffic per word.
//
//   NTT form          result[j] = operand[pi_g(j)],  pi_g(j) = rev(((g (2 rev(j) + 1)) mod 2n - 1) / 2)
//   coefficient form  coefficient i moves to k = i g mod 2n, negated when k >= n.  Written as a gather:
//                     result[k] = +-operand[t mod n],  t = k g^-1 mod 2n, negated when t >= n (because n g = n mod 2n)
// rev is the bit reversal on log2 n bits.  Every index fits 32 bits (n <= 2^20) and every product is only needed mod
// 2n, which divides 2^32, so the index arithmetic is 32-bit and wraps harmlessly.
//
// V16: every buffer of the launch is 16-byte aligned, so a thread moves its output pair (2m, 2m+1) with one 16-byte
// store (and, in NTT form, one 16-byte load); otherwise the same pairs move a word at a time.
#include "galois.cuh"
#include "internal.h"

namespace hexl_b200 {
namespace {

constexpr int kThreads = 256;
constexpr int kSmemThreads = 1024;

template <bool V16>
__device__ __forceinline__ void st_pair(u64* p, u64 a, u64 b) {
  if constexpr (V16) {
    st_stream2(p, make_ulonglong2(a, b));
  } else {
    __stcs(p, a);
    __stcs(p + 1, b);
  }
}

// NTT form, `polys` polynomials of n words in one launch; a thread stores the output pair (2m, 2m+1).  Every aligned
// block of 2^t output slots reads one aligned block of 2^t input slots, so pi_g(2m+1) = pi_g(2m) ^ 1: the pair is one
// aligned input pair, swapped when pi_g(2m) is odd, and a warp's 64 slots read one aligned 512-byte block.
template <bool V16>
__global__ void __launch_bounds__(kThreads)
    galois_ntt_kernel(u64* __restrict__ result, const u64* __restrict__ operand, u64 polys, int log_n, unsigned g) {
  const u64 total = polys << (log_n - 1);
  const unsigned two_n_mask = (2u << log_n) - 1u;
  const u64 stride = (u64)gridDim.x * kThreads;
  for (u64 i = (u64)blockIdx.x * kThreads + threadIdx.x; i < total; i += stride) {
    const u64 p = i >> (log_n - 1);
    const unsigned j = (unsigned)(i - (p << (log_n - 1))) * 2u;
    const u64* src = operand + (p << log_n);
    const unsigned s = ntt_source(j, g, two_n_mask, log_n);
    u64 a, b;
    if constexpr (V16) {
      const ulonglong2 v = ld_stream2(src + (s & ~1u));
      a = v.x;
      b = v.y;
    } else {
      a = __ldcs(src + (s & ~1u));
      b = __ldcs(src + (s | 1u));
    }
    if (s & 1u) st_pair<V16>(result + (p << log_n) + j, b, a);
    else st_pair<V16>(result + (p << log_n) + j, a, b);
  }
}

__device__ __forceinline__ u64 signed_word(u64 v, bool neg, u64 q) { return neg && v ? q - v : v; }

// Coefficient form up to kGaloisSmemMaxN: one CTA per limb stages the limb in shared memory with coalesced loads, then
// gathers from it and stores coalesced pairs.  Limb e of polynomial p of the launch is limb i0 + e of the buffer (rns
// limbs per polynomial), under mods.q[e].
template <bool V16>
__global__ void __launch_bounds__(kSmemThreads)
    galois_coef_smem_kernel(u64* __restrict__ result, const u64* __restrict__ operand, u64 rns, u64 i0, u64 cnt,
                            int log_n, unsigned g_inv, const __grid_constant__ GaloisModuli mods) {
  extern __shared__ ulonglong2 stage2[];
  u64* stage = reinterpret_cast<u64*>(stage2);
  const u64 p = blockIdx.x / cnt, e = blockIdx.x - p * cnt;
  const unsigned n = 1u << log_n, half = n >> 1, two_n_mask = 2u * n - 1u;
  const u64 off = (p * rns + i0 + e) << log_n;
  const u64 q = mods.q[e];
  for (unsigned m = threadIdx.x; m < half; m += kSmemThreads) {
    if constexpr (V16) {
      stage2[m] = ld_stream2(operand + off + 2 * m);
    } else {
      stage[2 * m] = __ldcs(operand + off + 2 * m);
      stage[2 * m + 1] = __ldcs(operand + off + 2 * m + 1);
    }
  }
  __syncthreads();
  for (unsigned m = threadIdx.x; m < half; m += kSmemThreads) {
    const unsigned t0 = (2u * m * g_inv) & two_n_mask, t1 = ((2u * m + 1u) * g_inv) & two_n_mask;
    st_pair<V16>(result + off + 2 * m, signed_word(stage[t0 & (n - 1u)], t0 & n, q),
                 signed_word(stage[t1 & (n - 1u)], t1 & n, q));
  }
}

// Coefficient form above kGaloisSmemMaxN: one thread per output pair, gathering its two words from global memory.  The
// grid walks the output in order, so the CTAs in flight cover a few consecutive limbs, whose words stay in L2 until
// every gather of them has been served: HBM still sees each input word about once.
template <bool V16>
__global__ void __launch_bounds__(kThreads)
    galois_coef_gather_kernel(u64* __restrict__ result, const u64* __restrict__ operand, u64 rns, u64 i0, u64 cnt,
                              u64 polys, int log_n, unsigned g_inv, const __grid_constant__ GaloisModuli mods) {
  const unsigned n = 1u << log_n, two_n_mask = 2u * n - 1u;
  const u64 i = (u64)blockIdx.x * kThreads + threadIdx.x;
  if (i >= (polys * cnt) << (log_n - 1)) return;
  const u64 limb = i >> (log_n - 1);  // limb of the launch: polynomial limb / cnt, entry limb % cnt
  const u64 p = limb / cnt, e = limb - p * cnt;
  const unsigned k = (unsigned)(i - (limb << (log_n - 1))) * 2u;
  const u64 off = (p * rns + i0 + e) << log_n;
  const u64 q = mods.q[e];
  const unsigned t0 = (k * g_inv) & two_n_mask, t1 = ((k + 1u) * g_inv) & two_n_mask;
  st_pair<V16>(result + off + k, signed_word(__ldg(operand + off + (t0 & (n - 1u))), t0 & n, q),
               signed_word(__ldg(operand + off + (t1 & (n - 1u))), t1 & n, q));
}

unsigned blocks_for(u64 items) { return (unsigned)((items + kThreads - 1) / kThreads); }

bool aligned16(const void* a, const void* b) {
  return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0;
}

}  // namespace

cudaError_t launch_galois_ntt(u64* result, const u64* operand, int log_n, u64 polys, u64 galois_elt,
                              cudaStream_t stream) {
  if (polys == 0) return cudaSuccess;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  u64 blocks = blocks_for(polys << (log_n - 1));
  if (blocks > (u64)sms * 16) blocks = (u64)sms * 16;
  auto kernel = aligned16(result, operand) ? galois_ntt_kernel<true> : galois_ntt_kernel<false>;
  kernel<<<(unsigned)blocks, kThreads, 0, stream>>>(result, operand, polys, log_n, (unsigned)galois_elt);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_galois_coef(u64* result, const u64* operand, int log_n, u64 rns, u64 i0, u64 cnt, u64 polys,
                               u64 galois_inv, const GaloisModuli& mods, cudaStream_t stream) {
  if (polys == 0 || cnt == 0) return cudaSuccess;
  const u64 n = 1ull << log_n;
  const bool v16 = aligned16(result, operand);
  if (n <= kGaloisSmemMaxN) {
    auto kernel = v16 ? galois_coef_smem_kernel<true> : galois_coef_smem_kernel<false>;
    const size_t smem = n * sizeof(u64);
    if (smem > 48 * 1024) {
      const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
    }
    kernel<<<(unsigned)(polys * cnt), kSmemThreads, smem, stream>>>(result, operand, rns, i0, cnt, log_n,
                                                                    (unsigned)galois_inv, mods);
  } else {
    auto kernel = v16 ? galois_coef_gather_kernel<true> : galois_coef_gather_kernel<false>;
    kernel<<<blocks_for((polys * cnt * n) / 2), kThreads, 0, stream>>>(result, operand, rns, i0, cnt, polys, log_n,
                                                                       (unsigned)galois_inv, mods);
  }
  count_launch();
  return cudaGetLastError();
}

}  // namespace hexl_b200
