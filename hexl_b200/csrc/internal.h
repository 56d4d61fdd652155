// Internal interfaces between the C ABI (capi*.cu) and the kernel launchers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "modarith.cuh"

namespace hexl_b200 {

// ------------------------------------------------------------------ eltwise
enum class EltOp : int {
  AddVV, AddVS, SubVV, SubVS, MultVV, Fma, FmaNoAdd, Reduce, Copy, CmpAdd, CmpSubMod,
  MontMult, MontIn, MontOut  // Montgomery form, R = 2^shift: a*b/R, a*scalar/R (scalar = R^2 mod q), a/R; mu = -q^-1 mod R
};

struct EltParams {
  u64* result;
  const u64* a;
  const u64* b;  // second vector operand (AddVV/SubVV/MultVV: op2; Fma: arg3)
  u64 n;
  u64 q;
  u64 scalar;    // AddVS/SubVS: operand2; Fma: reduced arg2; Cmp*: bound
  u64 scalar_p;  // Fma: floor(arg2*2^64/q); Cmp*: diff
  u64 mu;        // MultVV: generalised-Barrett mu; Reduce/CmpSubMod: floor(2^64/q)
  int in_mf;     // MultVV/Fma: 1,2,4,8; Reduce: 0 means "== q", else 2 or 4
  int out_mf;    // Reduce: 1 or 2
  int shift;     // MultVV: ceil_log2(q) - 2
  int cmp;       // CMPINT 0..7
};

cudaError_t launch_eltwise(EltOp op, const EltParams& p, cudaStream_t stream);

// ---------------------------------------------------------------------- NTT
// Device-resident tables of one (N, q, root) on one device.
//   fwd[k], k in [1, N): forward twiddle of tree node k  ( = psi^bitrev(k), the
//           reference's root_of_unity_powers[k], ntt-internal.cpp:60-72 )
//   inv[k]: its modular inverse (the reference stores these re-ordered,
//           ntt-internal.cpp:144-154; here they keep the tree indexing)
// The children of node k are 2k and 2k+1; a sub-transform rooted at node b uses
// node b*2^s + i for its stage s, group i.
// Device copies are in node order except where twiddle_lanes_major(log_n): there, entry i of each of the deepest
// four tree levels (depth log_n - 4 + j, j = 0..3) is stored at lane_major(i >> j, i & (2^j - 1), j) of that level
// instead of at i.  Those levels are read only by the last register pass of the 4096-point rows (reg_stages, LB = 0),
// where global thread-row U = (row in polynomial) * 256 + u reads entry U * 2^j + g of level j for g < 2^j: in node
// order adjacent lanes are 2^j entries apart, in this order they are adjacent for every g.  The host trees (and the
// getters of the C ABI) keep node order.
//
// NttDeviceParams: what a kernel needs to know about one (N, q), resident in device
// memory next to the tables, so that ONE launch can transform polynomials of several
// moduli (RNS batches): the launch carries a short list of pointers to these records.
struct NttDeviceParams {
  const Twiddle* fwd;
  const Twiddle* inv;
  u64 q, mu;
  Twiddle inv_n, inv_n_w;
  // generalised-Barrett constants of the point-wise product (eltwise-mult-mod-internal.hpp:52-99, alpha = 62,
  // beta = -2): prod_shift = bits(q) - 2, prod_mu = floor(2^(prod_shift + 64) / q).  Used by the inverse transform
  // that multiplies on load (NttMulti::mul).
  u64 prod_mu;
  int prod_shift;
};
struct NttDeviceTables {
  const Twiddle* fwd;
  const Twiddle* inv;
  const Twiddle32* fwd32;  // 32-bit copies of both tables, only for q < 2^30 (else nullptr)
  const Twiddle32* inv32;
  u64 n;
  int log_n;
  u64 q;
  u64 mu;           // floor(2^64 / q)
  Twiddle inv_n;    // N^-1 and its Shoup factor
  Twiddle inv_n_w;  // N^-1 * inv[1] and its Shoup factor
  Twiddle32 inv_n32, inv_n_w32;
  const NttDeviceParams* dparams;  // the same facts as a device-resident record
};
constexpr u64 kSmallModulusLimit = 1ull << 30;  // below: 4q < 2^32, the 32-bit kernels apply

// log2 of the row length used for a transform of size 2^log_n: the whole polynomial up to 8192 coefficients, else
// 4096-point rows after the column passes
constexpr int pick_row_log(int log_n) { return log_n <= 13 ? log_n : 12; }
// The transforms whose rows are 4096 points store their deepest four twiddle levels lane-major.
constexpr bool twiddle_lanes_major(int log_n) { return pick_row_log(log_n) == 12; }
// Position inside level j (of the deepest four) of the entry that thread-row U reads for group g < 2^j: warps of
// 32 thread-rows own blocks of 32 * 2^j entries, g-major inside the block.  The three terms occupy disjoint bits, so
// lane_major(U, g, j) = lane_major(U, 0, j) + (g << 5): the kernels add g << 5 to the address as an immediate offset.
__host__ __device__ constexpr unsigned lane_major(unsigned U, unsigned g, int j) {
  return ((U >> 5) << (j + 5)) + (g << 5) + (U & 31);
}

// result/operand: `batch` polynomials back to back on the current device.
cudaError_t launch_ntt_forward(const NttDeviceTables& t, u64* result, const u64* operand,
                               int in_mf, int out_mf, u64 batch, cudaStream_t stream);
cudaError_t launch_ntt_inverse(const NttDeviceTables& t, u64* result, const u64* operand,
                               int in_mf, int out_mf, u64 batch, cudaStream_t stream);

// Multi-modulus launch: polynomial u (of `units` back to back) belongs to entry u / group.
// At most kParamBlock entries per call; all moduli share the degree 2^log_n.
constexpr int kParamBlock = 64;
constexpr int kMaxMirrors = 15;
struct NttMulti {
  const NttDeviceParams* p[kParamBlock];
  unsigned group;
  // Inverse transforms only: the kernel that writes the final values also writes them to `mirrors` more buffers at the
  // same offsets -- peer-mapped memory of other GPUs (P2P stores over NVLink).  This is how the sharded key switch
  // all-gathers its digits inside the transform that produces them instead of copying afterwards.
  unsigned mirrors;
  u64* mirror[kMaxMirrors];
  // Forward transforms only: when non-zero, unit u READS polynomial (u % gather) of `operand` (result still goes to
  // unit u) and every value is first reduced into its own modulus (any 64-bit value -> [0, q)).  This is KeySwitch's
  // "every digit into every modulus" step (key-switch-internal.cpp:77-85) folded into the transform that consumes it:
  // the digits are read from L2 instead of a decomp x rns x n intermediate being written to and read back from HBM.
  unsigned gather;
  // Inverse transforms only: when non-null, the kernel that reads `operand` multiplies every value by the value at the
  // same offset of `mul` (both canonical, i.e. forward outputs with output_mod_factor 1) before its first butterfly:
  // InvNTT(a (.) b) in one pass over the data -- the FwdNTT -> MultMod -> InvNTT chain of
  // dyadic-multiply-internal.cpp:17-73 / the product pipelines of the callers without the MultMod kernel and without
  // the product's round trip through HBM (24 B per coefficient less).
  const u64* mul;
};
// max_q = the largest modulus of the call: it selects the butterflies every entry can run
cudaError_t launch_ntt_multi(bool forward, const NttMulti& multi, int log_n, u64 min_q, u64 max_q, u64* result,
                             const u64* operand, int out_mf, u64 units, cudaStream_t stream);

// ----------------------------------------------------- SEAL-shaped composites
struct DyadicModulus {  // per RNS modulus: q and its generalised-Barrett constants
  u64 q, mu;
  int shift;
};
// Small per-call tables travel as kernel parameters (no upload, no synchronisation, capturable
// in a CUDA graph); longer lists are processed in blocks of kParamBlock entries.
struct DyadicModuli {
  DyadicModulus m[kParamBlock];
};
struct KeyPointers {
  const u64* p[kParamBlock];
};
// moduli [first, first + count) of a DyadicMultiply over `num_moduli` moduli
cudaError_t launch_dyadic_multiply(u64* result, const u64* op1, const u64* op2, u64 n, u64 num_moduli, u64 first,
                                   u64 count, const DyadicModuli& mods, cudaStream_t stream);
// EltwiseMultMod / AddMod / SubMod of `count` blocks of per_mod elements, block e under mods.m[e]
enum : int { kRnsMult = 0, kRnsAdd = 1, kRnsSub = 2 };
cudaError_t launch_rns_eltwise(int op, u64* result, const u64* a, const u64* b, u64 per_mod, u64 count, int in_mf,
                               const DyadicModuli& mods, cudaStream_t stream);

// KeySwitch glue, batched over the RNS moduli of one parameter block (entry e of `mods`
// describes modulus i0 + e).  KsModulus.a/b/c mean, per kernel:
//   reduce: -            mac: a,b = 2^64 mod q and its Shoup factor, c = slot of q in the key
//   round:  a = q - (q_last/2 mod q)        finish: a,b = mod-switch factor and its Shoup factor
//   rescale_coef: a,b = q_last^-1 mod q and its Shoup factor, c = q - (q_last/2 mod q)
struct KsModulus {
  u64 q, mu, a, b, c;
};
struct KsModuli {
  KsModulus m[kParamBlock];
};
// prod[e][k][l] (+)= sum_{j < jcount} ops[e][j][l] * keys[j][k][c_e][l]  mod q_e ; ops_stride = elements between e's.
// galois_elt = g != 0: ops[e][j][pi_g(l)] instead, pi_g the NTT-form automorphism of launch_galois_ntt.
cudaError_t launch_ks_mac(u64* prod, const u64* ops, u64 ops_stride, const KeyPointers& keys, u64 n, u64 jcount,
                          u64 kcc, u64 key_modulus_size, u64 count, const KsModuli& mods, int accumulate,
                          cudaStream_t stream, u64 galois_elt = 0);
// tmp[e][k][l] = ((t_last[k][l] + q_last/2) mod q_last) mod q_e + a_e
cudaError_t launch_ks_round(u64* tmp, const u64* t_last, u64 n, u64 kcc, u64 q_last, u64 mu_last, u64 count,
                            const KsModuli& mods, cudaStream_t stream);
// result[k][i0+e][l] = ([result +] (in + 4 q_e - tmp[e][k][l]) * a_e) mod q_e ; result has `res_stride` moduli per k.
// in: in[e][k][l] (modulus-major, like tmp), or in[k][i0+e][l] laid out like result when in_like_result (may be result).
// accumulate: add into result (KeySwitch) or store (DivideAndRoundQLast).
cudaError_t launch_ks_finish(u64* result, const u64* in, const u64* tmp, u64 n, u64 kcc, u64 res_stride, u64 i0,
                             u64 count, const KsModuli& mods, bool in_like_result, bool accumulate,
                             cudaStream_t stream);
// DivideAndRoundQLast in coefficient form, fused: `polys` polynomials of rns limbs x n words; limbs [i0, i0 + count)
// of result = round(limb rns-1) and finish(limb i0+e) of operand, one pass; limb rns-1 of result is not written
cudaError_t launch_rescale_coef(u64* result, const u64* operand, u64 n, u64 rns, u64 i0, u64 count, u64 polys,
                                u64 q_last, u64 mu_last, const KsModuli& mods, cudaStream_t stream);

// Fast base conversion (rns.cu) of `polys` polynomials from `from` <= kParamBlock source moduli q_i (Q = their product)
// into `to` target moduli t_e, coefficient form; limb i of polynomial p is operand[p op_poly + i op_limb + l], limb e
// of its result is result[p res_poly + e res_limb + l]:
//   result_e = [ sum_i [(x_i + add_i) (Q/q_i)^-1]_{q_i} [Q/q_i]_{t_e} - sub_e ]_{t_e},  every modulus below 2^61.
// The constants travel in the kernel parameters (capturable, no upload); the table holds, in this order:
//   per source i (4 words):  q_i, (Q/q_i)^-1 mod q_i, its Shoup factor, add_i < q_i
//   per target e (5 words):  t_e, floor(2^64 / t_e), 2^64 mod t_e, its Shoup factor, sub_e < t_e
//   per target e (from words): [Q/q_i]_{t_e} for every source i
// so one launch takes at most base_conv_targets(from) targets; the mod-down's rounding sets add and sub (capi_hybrid.cu).
constexpr int kBaseConvWords = 480;  // 3840 bytes: with the other arguments inside the 4 KiB of kernel parameters
struct BaseConvTable {
  u64 w[kBaseConvWords];
};
inline u64 base_conv_targets(u64 from) { return (kBaseConvWords - 4 * from) / (5 + from); }
cudaError_t launch_base_conv(u64* result, u64 res_limb, u64 res_poly, const u64* operand, u64 op_limb, u64 op_poly,
                             u64 n, u64 polys, u64 from, u64 to, const BaseConvTable& tab, cudaStream_t stream);
// The t-corrected conversion (BGV's mod-down by P_T = Q, tau the plain modulus), same strides and result layout:
//   y_i = [x_i (P_T/q_i)^-1]_{q_i},  X~_m = [sum_i y_i [P_T/q_i]_m]_m,  k = [-X~_tau P_T^-1]_tau,
//   result_e = [X~_e + [P_T]_{t_e} k]_{t_e},  canonical,
// the residues of delta = X~ + P_T k: delta = x mod P_T, delta = 0 mod tau, 0 <= delta < P_T (from + tau - 1).  Table:
//   per source i (3 words):  q_i, (P_T/q_i)^-1 mod q_i, its Shoup factor
//   tau (6 + from words):    tau, floor(2^64 / tau), 2^64 mod tau, its Shoup factor, [-P_T^-1]_tau, its Shoup factor,
//                            then [P_T/q_i]_tau for every source i
//   per target e (6 words):  t_e, floor(2^64 / t_e), 2^64 mod t_e, its Shoup factor, [P_T]_{t_e}, its Shoup factor
//   per target e (from words): [P_T/q_i]_{t_e} for every source i
// so one launch takes at most base_conv_t_targets(from) targets: 67 for one source, 27 for 10, 3 for 64.
inline u64 base_conv_t_targets(u64 from) { return (kBaseConvWords - 4 * from - 6) / (6 + from); }
cudaError_t launch_base_conv_t(u64* result, u64 res_limb, u64 res_poly, const u64* operand, u64 op_limb, u64 op_poly,
                               u64 n, u64 polys, u64 from, u64 to, const BaseConvTable& tab, cudaStream_t stream);

// BFV multiplication by BEHZ (bfv.cu), coefficient form, every modulus below 2^61, l = |Q| and k = |B| in [1, 64].
// The constants are too many for the kernel parameters (l = k = 64 takes ~9000 words), so they live in a device table
// (capi_bfv.cu caches one per parameter set and device).  Extension table, in words:
//   per q_i (3):        q_i, [m~ (Q/q_i)^-1]_{q_i}, its Shoup factor
//   per q_i (1):        [Q/q_i] mod 2^32;  then 1 word: [-Q^-1] mod 2^32
//   per m of Bsk (8):   m, floor(2^64 / m), 2^64 mod m, its Shoup factor, [Q]_m, [-Q 2^32]_m, [2^-32]_m, its Shoup factor
//   per m of Bsk (l):   [Q/q_i]_m for every i
// Scaling table, in words:
//   per q_i (3):        q_i, [t (Q/q_i)^-1]_{q_i}, its Shoup factor
//   per m of Bsk (10):  m, floor(2^64 / m), 2^64 mod m, its Shoup factor, [t Q^-1]_m, Shoup, [-Q^-1]_m, Shoup,
//                       [(B/b_j)^-1]_{b_j} and its Shoup factor (m = b_j; zeros for m_sk)
//   per m of Bsk (l):   [Q/q_i]_m for every i
//   per q_i, then m_sk (5): q, floor(2^64 / q), 2^64 mod q, its Shoup factor, [B]_q
//   per q_i, then m_sk (k): [B/b_j]_q for every j
//   2 words:            [B^-1]_{m_sk}, its Shoup factor
// Bsk is ordered b_0..b_{k-1}, m_sk, and a lifted polynomial is l + k + 1 limbs: Q, then Bsk.
constexpr unsigned kBehzTile = 32;
// `polys` polynomials: polynomial p reads l limbs at operand + p op_poly and writes l + k + 1 limbs at
// result + p res_poly (limb stride n both), its Q limbs copied
cudaError_t launch_bfv_extend(u64* result, u64 res_poly, const u64* operand, u64 op_poly, u64 n, u64 polys, u64 l,
                              u64 k, const u64* tab, cudaStream_t stream);
// `polys` <= 3 tensor polynomials of l + k + 1 limbs, d_poly words apart, scaled by t/Q into l limbs at out.p[p]
struct BfvOutputs {
  u64* p[3];
};
cudaError_t launch_bfv_scale(const BfvOutputs& out, const u64* tensor, u64 d_poly, u64 n, u64 polys, u64 l, u64 k,
                             const u64* tab, cudaStream_t stream);

// Plaintexts of BFV and BGV (plain.cu), coefficient form, every modulus below 2^61, t in [2, 2^61), l <= 64.
// The lift of `count` plaintexts of pcc <= n words each (back to back) into l limbs of n words each:
//   m' = [m cf]_t (cf_shoup = floor(cf 2^64 / t)),  limb i = m' >= ceil(t/2) ? [m' - t]_{q_i} : [m']_{q_i}
struct PlainModuli {
  u64 q[kParamBlock];
  u64 mu[kParamBlock];  // floor(2^64 / q)
};
cudaError_t launch_plain_lift(u64* result, const u64* plain, u64 pcc, u64 n, u64 count, u64 l, u64 t, u64 cf,
                              u64 cf_shoup, const PlainModuli& mods, cudaStream_t stream);
// BFV add_plain / sub_plain on c0 of `batch` ciphertexts (2 l limbs of n words each): slots [0, cover) of c0 get
// +- round(Q m / t) mod q_i; ciphertext c reads its plaintext at plain + c plain_stride.  result may be ct.  tab: the
// device table capi_plain.cu builds (plain.cu states its layout).
cudaError_t launch_bfv_add_plain(u64* result, const u64* ct, const u64* plain, u64 pcc, u64 plain_stride, u64 n,
                                 u64 cover, u64 batch, u64 l, bool subtract, const u64* tab, cudaStream_t stream);

// Galois automorphism sigma_g (galois.cu).  NTT form: `polys` polynomials of 2^log_n words, one launch, words move
// unchanged (result[j] = operand[pi_g(j)]).  Coefficient form: limbs [i0, i0 + cnt) of `polys` polynomials of rns
// limbs each, limb i0 + e under mods.q[e]; galois_inv = g^-1 mod 2n.  result and operand must not overlap.
constexpr u64 kGaloisSmemMaxN = 1ull << 14;  // coefficient form: a limb is staged in shared memory up to this degree
struct GaloisModuli {
  u64 q[kParamBlock];
};
cudaError_t launch_galois_ntt(u64* result, const u64* operand, int log_n, u64 polys, u64 galois_elt,
                              cudaStream_t stream);
cudaError_t launch_galois_coef(u64* result, const u64* operand, int log_n, u64 rns, u64 i0, u64 cnt, u64 polys,
                               u64 galois_inv, const GaloisModuli& mods, cudaStream_t stream);

// Stream-ordered scratch from the library's own memory pool (capi.cu): kept warm between calls, capturable.
cudaError_t scratch_alloc_async(void** p, size_t bytes, cudaStream_t stream);
void scratch_free_async(void* p, cudaStream_t stream);

// launches issued so far (all kernels of this library)
void count_launch(unsigned n = 1);
uint64_t launches_so_far();

}  // namespace hexl_b200
