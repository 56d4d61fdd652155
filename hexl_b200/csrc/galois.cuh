// The NTT-form slot permutation of the Galois automorphism sigma_g, shared by the automorphism kernels (galois.cu) and
// the permuted multiply-accumulate of the hoisted rotations (seal.cu).  Every index fits 32 bits (n <= 2^20) and every
// product is only needed mod 2n, which divides 2^32, so the arithmetic is 32-bit and wraps harmlessly.
#pragma once

namespace hexl_b200 {

__device__ __forceinline__ unsigned rev_bits(unsigned x, int log_n) { return __brev(x) >> (32 - log_n); }

// pi_g(j) for the NTT-form slot j: result[j] = operand[pi_g(j)], pi_g(j) = rev(((g (2 rev(j) + 1)) mod 2n - 1) / 2)
__device__ __forceinline__ unsigned ntt_source(unsigned j, unsigned g, unsigned two_n_mask, int log_n) {
  const unsigned k = (g * (2u * rev_bits(j, log_n) + 1u)) & two_n_mask;  // odd
  return rev_bits(k >> 1, log_n);
}

}  // namespace hexl_b200
