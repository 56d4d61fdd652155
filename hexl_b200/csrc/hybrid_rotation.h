// Launchers of the two kernels of the hybrid linear transform (seal.cu): the weighted multi-element
// multiply-accumulate and the weighted permuted sum of the ciphertext's limbs; of the giant-step sums of the
// baby-step giant-step transform; of the multiply-accumulate of the multiply-relinearize call, which adds the
// tensor terms; of the tensor sums of a sum of products; and of the per-bit step of the inner sum (a rotate-and-sum
// kept in the extended basis).  All take two-component ciphertexts (key component count 2)
// in NTT form, every word canonical, every modulus below 2^61.
#pragma once
#include "internal.h"

namespace hexl_b200 {

// One launch covers up to kParamBlock (element, digit) pairs: `elts` elements of a chunk times the digits
// [j0, j0 + jcount) of a digit chunk.  key[r * jcount + j] is digit j0 + j's key of element r (2 x kms x n words),
// diag[r] element r's diagonal at the limb of the round's first modulus, elt[r] its Galois element.
struct WeightedMacElts {
  const u64* key[kParamBlock];
  const u64* diag[kParamBlock];
  unsigned elt[kParamBlock];
};
// For the `count` moduli of a mod-up round (mods as for launch_ks_mac: a, b = 2^64 mod q and its Shoup factor, c =
// the modulus's slot in the keys), every slot l and both key components k:
//   acc[e][k][l] (+)= sum_r w_r[e][l] ( sum_{j < jcount} ops[e][j][pi_r(l)] key_{r,j}[k][c_e][l] mod q_e )  mod q_e
// ops_stride = elements between e's.  The digit sum stays unreduced in 128 bits, so jcount must respect the bound of
// ks_mac_digits_per_launch; the weighted sum of at most 64 canonical products cannot wrap below 2^61.
cudaError_t launch_ks_weighted_mac(u64* acc, const u64* ops, u64 ops_stride, const WeightedMacElts& elts, u64 n,
                                   u64 jcount, u64 num_elts, u64 key_modulus_size, u64 count, const KsModuli& mods,
                                   bool accumulate, cudaStream_t stream);

// Up to kParamBlock elements of one launch: diag[r] element r's diagonal at the limb of the block's first modulus,
// elt[r] its Galois element; bit r of `identity` marks an identity term (g = 1 with no key), which adds w_r c1 too.
struct PermutedSumElts {
  const u64* diag[kParamBlock];
  unsigned elt[kParamBlock];
  u64 identity;
};
// For the data limbs [i0, i0 + count) of one ciphertext ct (two components of `level` limbs, mods.m[e] describing
// limb i0 + e with a, b = 2^64 mod q and its Shoup factor), every slot l:
//   result_0[i][l] (+)= sum_r w_r[i][l] c0_i[pi_r(l)],   result_1[i][l] (+)= sum_{r identity} w_r[i][l] c1_i[l]
// canonical; accumulate adds into result (later chunks of elements), else stores.  result must not overlap ct.
cudaError_t launch_ks_permuted_sum(u64* result, const u64* ct, u64 n, u64 level, u64 i0, u64 count,
                                   const PermutedSumElts& elts, u64 num_elts, const KsModuli& mods, bool accumulate,
                                   cudaStream_t stream);

// Up to kParamBlock present (giant, baby) pairs of one giant step: diag[r] the pair's diagonal at the limb of the
// block's first modulus, elt[r] the baby's Galois element, prod[r] the index of the baby's stored products among the
// keyed babies, or kBsgsNoProducts for an identity baby (element 1 without a key).
constexpr unsigned kBsgsNoProducts = ~0u;
struct BsgsSumTerms {
  const u64* diag[kParamBlock];
  unsigned elt[kParamBlock];
  unsigned prod[kParamBlock];
};
// mode bits: kBsgsKeyedGiant: component 1 goes to (x1, y1) for the giant's own key switch instead of into (X1, Y1);
// kBsgsStore1: store into (x1, y1) (the giant's first chunk of babies) instead of adding; kBsgsFold: the last sum
// launch of X with the merged rescale, which adds [P]_{q_i} X_{k,i} into Y's data limbs (mods.m[e].c = [P]_{q_i})
// and leaves X unwritten.
enum : int { kBsgsKeyedGiant = 1, kBsgsStore1 = 2, kBsgsFold = 4 };
// One giant step h over the moduli [b0, b0 + count) of B = {q_0..q_{l-1}, p_0..p_{K-1}} (l = level; mods.m[e] describes
// modulus b0 + e with a, b = 2^64 mod q and its Shoup factor), every slot l, the sums over the terms r (babies b_r):
//   X0_i[l]   += sum_r w_r[pi_h(l)] c0_i[pi_{b_r}(pi_h(l))]                       data limbs, x ([k][i][n])
//   Y0_b[l]   += sum_{r keyed} w_r[pi_h(l)] prod_r[b][0][pi_h(l)]                  every b, y ([b][k][n])
//   s1_i[l]    = sum_{r identity} w_r[l] c1_i[l],  t1_b[l] = sum_{r keyed} w_r[l] prod_r[b][1][l]
// s1 and t1 go into X1 and Y1, or into x1 ([i][n]) and y1 ([b][n]) under kBsgsKeyedGiant.  prod_r is
// prods + terms.prod[r] * prod_stride, laid out [b][k][n].  Everything canonical; ct is two components of level limbs.
cudaError_t launch_ks_bsgs_sum(u64* x, u64* y, u64* x1, u64* y1, const u64* ct, const u64* prods, u64 prod_stride,
                               u64 n, u64 level, u64 b0, u64 count, u64 giant, const BsgsSumTerms& terms,
                               u64 num_terms, const KsModuli& mods, int mode, cudaStream_t stream);

// The tensor terms of the multiply-relinearize call for the first `data` moduli of a mod-up round (the data moduli
// q_i, i = b0 + e): ct1 and ct2 point at limb b0 of component 0 of the two ciphertexts, component 1 is comp words
// further, and p[e] = [P]_{q_i} for P the product of the special primes.  sum (nullptr: none) holds (d0, d1) already
// formed, canonical, laid out like ct1 (d1 comp words after d0); ct1 and ct2 are then not read.
struct RelinTensor {
  const u64* ct1;
  const u64* ct2;
  u64 comp;
  u64 data;
  u64 p[kParamBlock];
  const u64* sum;
};
// For the `count` moduli of a mod-up round (mods as for launch_ks_mac), every slot l and both key components k:
//   prod[e][k][l] (+)= sum_{j < jcount} ops[e][j][l] keys.p[j][k][c_e][l]  (+ [P]_{q_i} d_k[i][l] when storing and
//                      e < tensor.data)   mod q_e,
// d_0 = a0 b0 and d_1 = a0 b1 + a1 b0 at limb i = b0 + e, (a0, a1) = ct1, (b0, b1) = ct2, or d_k read from tensor.sum.
// The digit sum stays unreduced in 128 bits (the bound of ks_mac_digits_per_launch); the tensor term is reduced on its
// own and added mod q.
cudaError_t launch_ks_relin_mac(u64* prod, const u64* ops, u64 ops_stride, const KeyPointers& keys, u64 n, u64 jcount,
                                u64 key_modulus_size, u64 count, const KsModuli& mods, const RelinTensor& tensor,
                                bool accumulate, cudaStream_t stream);

// Up to kRelinSumPairs pairs of ciphertexts of one sum of products: ct1[r] and ct2[r] point at pair r's ciphertexts
// (two components of `level` limbs each).  d1 takes two products per pair, so a launch's 128-bit sums hold at most 64
// products of canonical words, which cannot wrap below 2^61.
constexpr int kRelinSumPairs = 32;
struct RelinSumPairs {
  const u64* ct1[kRelinSumPairs];
  const u64* ct2[kRelinSumPairs];
};
// For the data limbs [i0, i0 + count) (mods.m[e] describing limb i0 + e with a, b = 2^64 mod q and its Shoup factor),
// every slot l, over the num_pairs pairs r, (a0, a1) = ct1[r], (b0, b1) = ct2[r]:
//   out[0][i][l] (+)= sum_r a0 b0,  out[1][i][l] (+)= sum_r (a0 b1 + a1 b0),  out[2][i][l] (+)= sum_r a1 b1   mod q_i
// canonical; out is [3][level][n]; accumulate adds into out (later chunks of pairs), else stores.
cudaError_t launch_relin_tensor_sum(u64* out, u64 n, u64 level, u64 i0, u64 count, const RelinSumPairs& pairs,
                                    u64 num_pairs, const KsModuli& mods, bool accumulate, cudaStream_t stream);

// One bit of the inner sum's rotate-and-sum recurrence.  The pairs A (the current partial sum, read), A' (A + Rot_d(A),
// written) and R (the result so far, R += Rot_s(A)) each hold X, two components on the data limbs ([k][i][n], level
// limbs), and Y, two components over B ([b][k][n]).  mode bits:
//   kSumYA         A has Y (else Y_A reads as zero)
//   kSumNext       write A'; kSumNextY: A' has Y (writes it over B); kSumDoubleId: d = 1, so component 1 doubles
//   kSumR          update R; kSumRStore: X_R is stored (the first set bit); kSumRY: R had Y before (else Y_R is stored);
//                  kSumRYWrite: write Y_R over B; kSumShiftId: s = 1, so component 1 of A adds into R too
//   kSumCopy1      store Y_A's component 1 into y1 ([b][n]), the input of the one-component mod-down of c1'
//   kSumFold       R's last update under the merged rescale: Y_R's data limbs take [P]_{q_i} X_R (mods.m[e].c),
//                  X_R is not stored
enum : int {
  kSumYA = 1, kSumNext = 2, kSumNextY = 4, kSumDoubleId = 8, kSumR = 16, kSumRStore = 32, kSumRY = 64,
  kSumRYWrite = 128, kSumShiftId = 256, kSumCopy1 = 512, kSumFold = 1024
};
// Over the moduli [b0, b0 + count) of B (l = level; mods.m[e] describes modulus b0 + e with a, b = 2^64 mod q and its
// Shoup factor), every slot l, with d and s the doubling and shift elements (1 when absent):
//   A'0[l] = A0[l] + A0[pi_d(l)],  A'1[l] = A1[l] (2 A1[l] under kSumDoubleId)
//   R0[l] (+)= A0[pi_s(l)],        R1[l] (+)= A1[l] under kSumShiftId
// on X for the data moduli and on Y where Y is written; everything canonical.  xa, ya (A) are only read.
cudaError_t launch_inner_sum_step(const u64* xa, const u64* ya, u64* xn, u64* yn, u64* xr, u64* yr, u64* y1, u64 n,
                                  u64 level, u64 b0, u64 count, u64 dbl, u64 shift, const KsModuli& mods, int mode,
                                  cudaStream_t stream);

}  // namespace hexl_b200
