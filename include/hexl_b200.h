/* hexl_b200.h -- C ABI of libhexl_b200.so, the Hopper (sm_90a) drop-in for the
 * intel/hexl hot path: NTT::ComputeForward / ComputeInverse, the seven Eltwise*Mod
 * operations, and the SEAL-shaped callers built on them (DyadicMultiply, KeySwitch,
 * the NTT cache).
 *
 * Every entry point names the reference interface it replaces (file:line relative
 * to the intel/hexl v1.2.5 tree).  The C++ headers under include/hexl/ re-create
 * the reference's `intel::hexl` API (same names, overloads, defaults) as inline
 * forwarders to these symbols, so SEAL/OpenFHE-style callers re-link unchanged;
 * INTEGRATION.md shows the binding a maintainer would add on the reference side.
 *
 * Conventions
 *  - Plain pointers and sizes only; no C++ or torch types.
 *  - Every data pointer may be a DEVICE pointer (cudaMalloc / torch tensor
 *    storage; the call is enqueued on `stream` and returns without synchronising)
 *    or a HOST pointer (pageable or pinned; the call stages the buffers through
 *    the GPU -- H2D, kernel, D2H, chunked so copies and kernels overlap -- and
 *    returns when `result` is complete).  Unified-memory pointers
 *    (hexl_b200_managed_alloc) are worked on in place like device pointers, and
 *    with stream == NULL the call returns with the result complete.  All data
 *    pointers of one call must be of the same kind.  `result` may alias an input (in place), as in the
 *    reference (test/test-ntt.cpp:240-243).
 *  - `stream` is a cudaStream_t passed as void*; NULL = the legacy default stream.
 *  - Batched calls take `batch` independent units laid out back to back
 *    (unit u at offset u*n elements); batch = 1 is the reference's one-call shape.
 *  - Return value: 0 on success, negative hexl_b200_status otherwise;
 *    hexl_b200_last_error() returns a thread-local message.  There is NO CPU
 *    fallback: without a usable CUDA device every compute entry point fails
 *    with HEXL_B200_ERR_NO_DEVICE.
 *  - Argument validation mirrors the reference's HEXL_CHECKs
 *    (e.g. hexl/ntt/ntt-internal.cpp:191-200, hexl/eltwise/eltwise-fma-mod.cpp:20-40).
 *    Cheap checks (null, n == 0, mod factors, modulus range) are always on;
 *    the O(n) input-range checks only when hexl_b200_set_debug(1) was called
 *    (the reference does them only in HEXL_DEBUG builds, check.hpp:12-44).
 *    On device pointers the range checks run on `stream`, after the work the
 *    caller queued there, and the host waits for the checks (that stream
 *    only) before the call goes on or refuses: the work queued before a debug
 *    call is complete when it returns.  The result itself is still computed
 *    asynchronously on `stream`, as without the checks.  A debug call on a
 *    stream that is being captured into a CUDA graph is refused with
 *    HEXL_B200_ERR_INVALID_ARG before anything is queued, and the capture
 *    stays valid; turn the checks off to capture.
 */
#ifndef HEXL_B200_H
#define HEXL_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum hexl_b200_status {
  HEXL_B200_OK = 0,
  HEXL_B200_ERR_INVALID_ARG = -1, /* a HEXL_CHECK of the reference would fire */
  HEXL_B200_ERR_NO_DEVICE = -2,   /* no CUDA device / driver */
  HEXL_B200_ERR_CUDA = -3,        /* a CUDA runtime call failed */
  HEXL_B200_ERR_ALLOC = -4,
  HEXL_B200_ERR_MIXED_POINTERS = -5 /* host and device pointers in one call */
} hexl_b200_status;

typedef struct hexl_b200_ntt hexl_b200_ntt; /* opaque, reference-counted */

/* ---- library / device management (no counterpart in the reference: it is CPU-only) */
const char* hexl_b200_version(void);
const char* hexl_b200_last_error(void);
int hexl_b200_device_count(void);
/* Devices used for HOST-pointer calls with batch > 1: units are split into
 * contiguous blocks, one block per listed device (no inter-GPU traffic).
 * Default: the calling thread's current device only. */
int hexl_b200_set_host_devices(const int* devices, int count);
void hexl_b200_set_debug(int on); /* O(n) input-range checks, like HEXL_DEBUG */
int hexl_b200_sync(void* stream);
/* Pinned host memory so host-pointer calls DMA at full PCIe rate (the
 * reference's AllocatorBase hook, hexl/include/hexl/util/allocator.hpp:12-24,
 * is the place a caller would plug these in). */
void* hexl_b200_host_alloc(size_t bytes);
void hexl_b200_host_free(void* p);
/* Unified (managed) memory: one pointer valid on the host and on every GPU, so a
 * caller's buffers are device-visible with no staging copy.  Calls on managed
 * buffers with stream == NULL return after the result is complete (the
 * reference's synchronous semantics); with a stream they are asynchronous. */
void* hexl_b200_managed_alloc(size_t bytes);
void hexl_b200_managed_free(void* p);
/* number of kernel launches this library has issued in this process */
uint64_t hexl_b200_launch_count(void);

/* ---- number theory (host side; hexl/include/hexl/number-theory/number-theory.hpp) */
uint64_t hexl_b200_multiply_mod(uint64_t x, uint64_t y, uint64_t q);      /* :83  */
uint64_t hexl_b200_add_uint_mod(uint64_t x, uint64_t y, uint64_t q);      /* :95  */
uint64_t hexl_b200_sub_uint_mod(uint64_t x, uint64_t y, uint64_t q);      /* :99  */
uint64_t hexl_b200_pow_mod(uint64_t base, uint64_t exp, uint64_t q);      /* :102 */
uint64_t hexl_b200_inverse_mod(uint64_t x, uint64_t q);                   /* :79  */
uint64_t hexl_b200_reverse_bits(uint64_t x, uint64_t bit_width);          /* :75  */
int hexl_b200_is_prime(uint64_t n);                                       /* :166 */
int hexl_b200_is_primitive_root(uint64_t root, uint64_t degree, uint64_t q); /* :108 */
uint64_t hexl_b200_generate_primitive_root(uint64_t degree, uint64_t q);  /* :112 */
uint64_t hexl_b200_minimal_primitive_root(uint64_t degree, uint64_t q);   /* :117 */
/* floor(operand * 2^bit_shift / q), bit_shift in {32, 52, 64} (MultiplyFactor, :19-51) */
uint64_t hexl_b200_multiply_factor(uint64_t operand, uint64_t bit_shift, uint64_t q);
/* GeneratePrimes (:181): writes up to num primes, returns how many were found */
int hexl_b200_generate_primes(uint64_t* out, size_t num, size_t bit_size, int prefer_small,
                              size_t ntt_size);

/* ---- NTT object (class NTT, hexl/include/hexl/ntt/ntt.hpp:22-293) ---------------- */
/* NTT(degree, q): ntt.hpp:54 -- uses the minimal primitive 2N-th root */
int hexl_b200_ntt_create(hexl_b200_ntt** out, uint64_t degree, uint64_t q);
/* NTT(degree, q, root_of_unity): ntt.hpp:75 */
int hexl_b200_ntt_create_with_root(hexl_b200_ntt** out, uint64_t degree, uint64_t q,
                                   uint64_t root_of_unity);
void hexl_b200_ntt_retain(hexl_b200_ntt* h);  /* NTT is copyable in the reference */
void hexl_b200_ntt_release(hexl_b200_ntt* h); /* ~NTT */
/* NTT::CheckArguments (ntt.hpp:90, ntt-internal.cpp:171-186): 1 if valid */
int hexl_b200_ntt_check_arguments(uint64_t degree, uint64_t q);
uint64_t hexl_b200_ntt_degree(const hexl_b200_ntt* h);           /* GetDegree  :119 */
uint64_t hexl_b200_ntt_modulus(const hexl_b200_ntt* h);          /* GetModulus :122 */
uint64_t hexl_b200_ntt_minimal_root(const hexl_b200_ntt* h);     /* GetMinimalRootOfUnity :116 */
/* Host copies of the tables in the reference's layouts (getters ntt.hpp:125-194).
 * `which`: 0 root powers (bit-reversed slots), 1 their 64-bit Shoup factors,
 * 2 inverse root powers (stage-sequential order of ntt-internal.cpp:144-154),
 * 3 their 64-bit Shoup factors.  Returns a pointer valid for the handle's life. */
const uint64_t* hexl_b200_ntt_table(const hexl_b200_ntt* h, int which);

/* Uploads the handle's tables to `device` (-1: the calling thread's current device) now instead of on
 * the first transform there.  The first use of a handle on a device allocates and copies synchronously,
 * which is not allowed while a stream is being captured into a CUDA graph: warm the handles (this call,
 * or one ordinary call) before capturing.  No counterpart in the reference (its tables live in host
 * memory, ntt-internal.cpp:54-169). */
int hexl_b200_ntt_prepare(hexl_b200_ntt* h, int device);

/* NTT::ComputeForward (ntt.hpp:99; ntt-internal.cpp:188-250): natural-order input,
 * bit-reversed output.  in_mf in {1,2,4}: inputs < in_mf*q; out_mf in {1,4}:
 * outputs in [0, out_mf*q).  `batch` polynomials back to back. */
int hexl_b200_ntt_forward(hexl_b200_ntt* h, uint64_t* result, const uint64_t* operand,
                          uint64_t input_mod_factor, uint64_t output_mod_factor,
                          uint64_t batch, void* stream);
/* NTT::ComputeInverse (ntt.hpp:109; ntt-internal.cpp:252-310): bit-reversed input,
 * natural-order output, includes the 1/N scale.  in_mf in {1,2}, out_mf in {1,2}. */
int hexl_b200_ntt_inverse(hexl_b200_ntt* h, uint64_t* result, const uint64_t* operand,
                          uint64_t input_mod_factor, uint64_t output_mod_factor,
                          uint64_t batch, void* stream);

/* RNS batches in ONE launch (the shape of the reference's callers: every ciphertext
 * polynomial exists once per modulus, key-switch-internal.cpp:49-55,82-88): `count`
 * handles of the same degree; of the count * batch_per_modulus polynomials laid out back
 * to back, polynomial u is transformed under handles[u / batch_per_modulus], with the
 * semantics of hexl_b200_ntt_forward / _inverse.  Device (or unified) pointers run as one
 * launch per kernel stage regardless of `count`; host pointers fall back to one staged
 * call per handle. */
int hexl_b200_ntt_forward_multi(hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                                const uint64_t* operand, uint64_t input_mod_factor,
                                uint64_t output_mod_factor, uint64_t batch_per_modulus, void* stream);
int hexl_b200_ntt_inverse_multi(hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                                const uint64_t* operand, uint64_t input_mod_factor,
                                uint64_t output_mod_factor, uint64_t batch_per_modulus, void* stream);

/* The other two steps of an RNS polynomial product, with the same batching (not in the
 * reference, whose callers loop over the moduli: dyadic-multiply-internal.cpp:50-72):
 * EltwiseMultMod (eltwise-mult-mod.hpp:23) over `num_moduli` blocks of n_per_modulus
 * elements, block e under moduli[e], in one launch;  and the whole negacyclic product
 * result = InvNTT(FwdNTT(a) .* FwdNTT(b)) of count * batch_per_modulus polynomials,
 * polynomial u under handles[u / batch_per_modulus] (BASELINE configs[3]: FwdNTT ->
 * EltwiseMultMod -> InvNTT; the point-wise product is folded into the inverse transform,
 * which multiplies on load), 4 to 6 launches whatever `count`.  Inputs < q, outputs
 * in [0, q); result may be a, b or a separate buffer, and a may be b (a square), with or
 * without result. */
int hexl_b200_eltwise_mult_mod_multi(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                                     uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli,
                                     uint64_t input_mod_factor, void* stream);
/* EltwiseAddMod / EltwiseSubMod (eltwise-add-mod.hpp:22, eltwise-sub-mod.hpp:22) over an RNS batch */
int hexl_b200_eltwise_add_mod_multi(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                                    uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli, void* stream);
int hexl_b200_eltwise_sub_mod_multi(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                                    uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli, void* stream);
int hexl_b200_poly_multiply_multi(hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                                  const uint64_t* a, const uint64_t* b, uint64_t batch_per_modulus, void* stream);

/* ---- element-wise operations (hexl/include/hexl/eltwise/ *.hpp) -------------------
 * n = number of elements (for batched use pass n = batch * N: the ops are
 * position-independent). */
/* EltwiseAddMod vector-vector, eltwise-add-mod.hpp:22 */
int hexl_b200_eltwise_add_mod(uint64_t* result, const uint64_t* operand1,
                              const uint64_t* operand2, uint64_t n, uint64_t modulus,
                              void* stream);
/* EltwiseAddMod vector-scalar, eltwise-add-mod.hpp:36 */
int hexl_b200_eltwise_add_mod_scalar(uint64_t* result, const uint64_t* operand1,
                                     uint64_t operand2, uint64_t n, uint64_t modulus,
                                     void* stream);
/* EltwiseSubMod vector-vector, eltwise-sub-mod.hpp:22 */
int hexl_b200_eltwise_sub_mod(uint64_t* result, const uint64_t* operand1,
                              const uint64_t* operand2, uint64_t n, uint64_t modulus,
                              void* stream);
/* EltwiseSubMod vector-scalar, eltwise-sub-mod.hpp:36 */
int hexl_b200_eltwise_sub_mod_scalar(uint64_t* result, const uint64_t* operand1,
                                     uint64_t operand2, uint64_t n, uint64_t modulus,
                                     void* stream);
/* EltwiseMultMod, eltwise-mult-mod.hpp:23; in_mf in {1,2,4}, q < 2^62, in_mf * q < 2^63.
 * Exact for every accepted input; the same holds for hexl_b200_eltwise_mult_mod_multi and
 * hexl_b200_dyadic_multiply.  For 62-bit moduli the generalised Barrett quotient estimate can be low
 * by two and the product takes a second conditional subtraction; the reference's scalar tier takes one
 * and returns words in [q, 2q) for some operands near q at some moduli above about 2^61.7. */
int hexl_b200_eltwise_mult_mod(uint64_t* result, const uint64_t* operand1,
                               const uint64_t* operand2, uint64_t n, uint64_t modulus,
                               uint64_t input_mod_factor, void* stream);
/* EltwiseFMAMod, eltwise-fma-mod.hpp:22; arg3 may be NULL; in_mf in {1,2,4,8} */
int hexl_b200_eltwise_fma_mod(uint64_t* result, const uint64_t* arg1, uint64_t arg2,
                              const uint64_t* arg3, uint64_t n, uint64_t modulus,
                              uint64_t input_mod_factor, void* stream);
/* EltwiseReduceMod, eltwise-reduce-mod.hpp:24; in_mf in {modulus,2,4}, out_mf in {1,2}.
 * Exact for every q > 1.  For q >= 2^63 every 64-bit word is below 2q and in_mf 4 is treated as 2;
 * every tier of the reference subtracts 2q there, which wraps. */
int hexl_b200_eltwise_reduce_mod(uint64_t* result, const uint64_t* operand, uint64_t n,
                                 uint64_t modulus, uint64_t input_mod_factor,
                                 uint64_t output_mod_factor, void* stream);
/* EltwiseCmpAdd, eltwise-cmp-add.hpp:22; cmp = CMPINT value 0..7 (util.hpp:16-25) */
int hexl_b200_eltwise_cmp_add(uint64_t* result, const uint64_t* operand1, uint64_t n,
                              int cmp, uint64_t bound, uint64_t diff, void* stream);
/* EltwiseCmpSubMod, eltwise-cmp-sub-mod.hpp:24 */
int hexl_b200_eltwise_cmp_sub_mod(uint64_t* result, const uint64_t* operand1, uint64_t n,
                                  uint64_t modulus, int cmp, uint64_t bound, uint64_t diff,
                                  void* stream);

/* ---- Montgomery-form helpers (R = 2^r > q, q odd, r <= 62: the BitShift = 64 forms of the reference)
 * HenselLemma2adicRoot (number-theory.hpp:303): x in [0, 2^r) with q*x = -1 mod 2^r; 0 for invalid arguments */
uint64_t hexl_b200_hensel_lemma_2adic_root(uint32_t r, uint64_t q);
/* MontgomeryReduce<64> (number-theory.hpp:269-301): T * 2^-r mod q for T = T_hi*2^64 + T_lo < q * 2^r */
uint64_t hexl_b200_montgomery_reduce(uint64_t T_hi, uint64_t T_lo, uint64_t q, int r, uint64_t inv_mod);
/* EltwiseMontReduceModAVX512<64, r> (hexl/eltwise/eltwise-reduce-mod-avx512.hpp:156): result = a*b*R^-1 mod q;
 * EltwiseMontgomeryFormInAVX512 (:227): result = a*R mod q, given R^2 mod q;
 * EltwiseMontgomeryFormOutAVX512 (:298): result = a*R^-1 mod q.  Inputs < q, outputs in [0, q). */
int hexl_b200_eltwise_mont_reduce_mod(uint64_t* result, const uint64_t* a, const uint64_t* b, uint64_t n,
                                      uint64_t modulus, int r, uint64_t neg_inv_mod, void* stream);
int hexl_b200_eltwise_montgomery_form_in(uint64_t* result, const uint64_t* a, uint64_t R2_mod_q, uint64_t n,
                                         uint64_t modulus, int r, uint64_t neg_inv_mod, void* stream);
int hexl_b200_eltwise_montgomery_form_out(uint64_t* result, const uint64_t* a, uint64_t n, uint64_t modulus, int r,
                                          uint64_t neg_inv_mod, void* stream);

/* ---- SEAL-shaped composites built on the hot path (hexl/include/hexl/experimental/seal/)
 * `moduli`, `modswitch_factors` and the array `k_switch_keys` itself are small HOST
 * arrays; the coefficient buffers (result, operands, t_target, every k_switch_keys[j])
 * are all device pointers or all host pointers. */
/* NTT cache, GetNTT(N, modulus): ntt-cache.hpp:27-53.  Returns a retained handle
 * shared by every caller; release it with hexl_b200_ntt_release. */
int hexl_b200_ntt_get_cached(hexl_b200_ntt** out, uint64_t degree, uint64_t q);
/* DyadicMultiply, dyadic-multiply.hpp:26: (x0*y0, x0*y1 + x1*y0, x1*y1) per modulus;
 * operands hold 2 polynomials x num_moduli x n, result 3; result may alias an operand. */
int hexl_b200_dyadic_multiply(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                              uint64_t n, const uint64_t* moduli, uint64_t num_moduli, void* stream);
/* KeySwitch, key-switch.hpp:34 (CKKS): result (key_component_count x decomp x n) is
 * updated in place; t_target_iter_ptr holds decomp x n digits in NTT form;
 * k_switch_keys[j] holds key_component_count x key_modulus_size x n.
 * Every modulus the switch uses must be below 2^61 (HEXL_B200_ERR_INVALID_ARG otherwise).  The result is exact for
 * every accepted input.  It differs from the reference only where the reference's unreduced 128-bit sum of digit x
 * key products wraps: moduli above 2^60 with more than J(q) = floor((2^128 - 1) / ((4q - 1)(q - 1))) digits (16 just
 * below 2^61), where this library adds the digits up in chunks of at most J(q) instead. */
int hexl_b200_key_switch(uint64_t* result, const uint64_t* t_target_iter_ptr, uint64_t n,
                         uint64_t decomp_modulus_size, uint64_t key_modulus_size, uint64_t rns_modulus_size,
                         uint64_t key_component_count, const uint64_t* moduli,
                         const uint64_t* const* k_switch_keys, const uint64_t* modswitch_factors,
                         void* stream);

/* Rescale by the last RNS modulus (extension; SEAL's RNSTool::divide_and_round_q_last_inplace and
 * divide_and_round_q_last_ntt_inplace): the CKKS rescale after every multiplication, and BFV modulus switching.
 * operand holds `count` polynomials back to back, each of rns_modulus_size = L + 1 limbs of n words; limb i of
 * polynomial p is at (p * (L + 1) + i) * n and lies under moduli[i]; q_L = moduli[L] is the modulus dropped (the two
 * components of a ciphertext are two consecutive polynomials).  result has the same layout: limbs 0..L-1 of every
 * polynomial get floor((X + floor(q_L / 2)) / q_L) mod q_i, canonical, with X the CRT lift of the coefficient's limbs
 * in [0, q_0 ... q_L); limb L is not written.  result == operand is allowed; otherwise the buffers must not overlap.
 * ntt_form = 1 (CKKS): input and output limbs are in the forward-NTT form of GetNTT(n, q_i), as KeySwitch takes them;
 * ntt_form = 0: plain coefficients.  Inputs must be below their modulus (checked under hexl_b200_set_debug(1)).
 * HEXL_B200_ERR_INVALID_ARG unless every modulus is in (1, 2^61) and coprime to q_L, and in NTT form n is a power of
 * two in [2, 2^20] and every modulus NTT-friendly for n (n >= 1 in coefficient form).  count = 0 does nothing.  The
 * library computes q_L^-1 mod q_i itself.  Host buffers are staged by whole polynomials. */
int hexl_b200_divide_and_round_q_last(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                                      uint64_t rns_modulus_size, uint64_t count, int ntt_form, void* stream);

/* Galois automorphism sigma_g : a(X) -> a(X^g) of RNS polynomials (extension; the permutation of SEAL's
 * Evaluator::apply_galois_inplace, behind every rotation and conjugation of CKKS, BFV and BGV).  Layout as for
 * hexl_b200_divide_and_round_q_last: `count` polynomials back to back, each of rns_modulus_size limbs of n words, limb
 * i under moduli[i].  galois_elt = g is odd with 1 <= g < 2n; n is a power of two in [2, 2^20].
 *   ntt_form = 0 (coefficients): coefficient i moves to k = i g mod 2n; result[k] = operand[i] if k < n, otherwise
 *     result[k - n] = (q - operand[i]) mod q.  Inputs must be below q; outputs are canonical.
 *   ntt_form = 1 (the forward-NTT order of GetNTT(n, q), slot j holding a(psi^(2 rev(j) + 1))):
 *     result[j] = operand[pi_g(j)], pi_g(j) = rev(((g (2 rev(j) + 1)) mod 2n - 1) / 2), rev the bit reversal on
 *     log2 n bits.  Words move unchanged; pi_g depends neither on q nor on the root, so the moduli are read only by
 *     the range check.
 * Inputs are checked below their modulus under hexl_b200_set_debug(1).  HEXL_B200_ERR_INVALID_ARG unless every
 * pointer is non-null, every modulus is in (1, 2^62), g is as above and result == operand or the buffers do not
 * overlap.  count = 0 does nothing.  NTT form is one launch for the whole call; coefficient form one per block of 64
 * moduli.  In place (result == operand) the polynomials are first copied into library scratch and permuted from
 * there: one device copy of the data more than out of place.  Host buffers are staged by whole polynomials (and
 * permuted in place on the device) and split by polynomial over the devices of hexl_b200_set_host_devices. */
int hexl_b200_apply_galois(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                           uint64_t rns_modulus_size, uint64_t count, uint64_t galois_elt, int ntt_form, void* stream);

/* Key-switch keys resident on the GPU.  The reference keeps the keys in caller memory and reads them on every
 * call (key-switch.hpp:34-39); a host caller of hexl_b200_key_switch therefore pays decomp x key_component_count
 * x key_modulus_size x n words of PCIe traffic per call.  hexl_b200_keys_upload copies the `decomp` key buffers
 * (host or device pointers, the layout KeySwitch takes) once to the current device -- to every device listed with
 * hexl_b200_set_host_devices when that was called -- and hexl_b200_key_switch_resident runs `batch` key switches
 * against them: ciphertext c uses result + c * key_component_count * decomp * n and t_target + c * decomp * n.
 * Host buffers are pipelined (copies of one ciphertext under the kernels of its neighbours) and split across the
 * devices holding the keys; device buffers run on `stream` on their own device.  Moduli, exactness and the difference
 * from the reference are as for hexl_b200_key_switch, sharded handles included.
 * The upload (sharded or not) is synchronous: it first waits for every device that owns a device or managed key
 * buffer (cudaDeviceSynchronize there), so keys the caller has just written on any stream of that device, blocking or
 * not, are the ones copied; the handle is complete when the call returns. */
typedef struct hexl_b200_keys hexl_b200_keys;
int hexl_b200_keys_upload(hexl_b200_keys** out, const uint64_t* const* k_switch_keys, uint64_t n,
                          uint64_t decomp_modulus_size, uint64_t key_modulus_size, uint64_t key_component_count);
/* The same keys SHARDED BY RNS MODULUS over the devices of hexl_b200_set_host_devices (one shard per listed device; a
 * device listed twice carries two shards): shard s keeps only the key slices of its moduli.  ONE key switch then runs on
 * all shards at once -- the decomposed digits are all-gathered and the special prime's part is broadcast with P2P stores
 * over NVLink from the kernels that produce them (the exchange of key-switch-internal.cpp:60-131,134-198) -- which cuts
 * the latency of a single switch;
 * hexl_b200_key_switch_resident takes such a handle with HOST result / t_target buffers. */
int hexl_b200_keys_upload_sharded(hexl_b200_keys** out, const uint64_t* const* k_switch_keys, uint64_t n,
                                  uint64_t decomp_modulus_size, uint64_t key_modulus_size,
                                  uint64_t key_component_count);
void hexl_b200_keys_release(hexl_b200_keys* keys);
int hexl_b200_key_switch_resident(uint64_t* result, const uint64_t* t_target_iter_ptr, uint64_t n,
                                  uint64_t decomp_modulus_size, uint64_t key_modulus_size, uint64_t rns_modulus_size,
                                  uint64_t key_component_count, const uint64_t* moduli, const hexl_b200_keys* keys,
                                  const uint64_t* modswitch_factors, uint64_t batch, void* stream);

/* Rotation or conjugation of `batch` ciphertexts in place (extension; SEAL's Evaluator::apply_galois_inplace for a
 * ciphertext in NTT form).  Ciphertext c is at ciphertexts + c * 2 * decomp * n, laid out like KeySwitch's result:
 * components c0 and c1 of decomp limbs in NTT form, limb i under moduli[i], every word canonical (checked under
 * hexl_b200_set_debug(1)).  For each ciphertext:
 *   c0 <- sigma_g(c0) + KS_0(sigma_g(c1)),  c1 <- KS_1(sigma_g(c1)),
 * with sigma_g the NTT-form automorphism of hexl_b200_apply_galois and KS the function of hexl_b200_key_switch
 * applied to a zero result; bit for bit the chain r = [sigma_g(c0), 0]; hexl_b200_key_switch_resident(r, sigma_g(c1)).
 * galois_keys: the key-switch keys for g, uploaded with hexl_b200_keys_upload.  HEXL_B200_ERR_INVALID_ARG on the
 * shape rules of hexl_b200_key_switch_resident, unless key_component_count == 2 and n <= 2^20, for g outside the
 * rules of hexl_b200_apply_galois, and for a handle sharded by modulus (not supported here).  On the device, one
 * automorphism launch over both components into scratch, a copy and a memset, then the key switch: one launch more
 * per ciphertext than hexl_b200_key_switch_resident.  Host buffers cross PCIe once each way per ciphertext, pipelined
 * and split over the devices holding the keys as for hexl_b200_key_switch_resident. */
int hexl_b200_apply_galois_key_switch(uint64_t* ciphertexts, uint64_t n, uint64_t decomp_modulus_size,
                                      uint64_t key_modulus_size, uint64_t rns_modulus_size,
                                      uint64_t key_component_count, const uint64_t* moduli,
                                      const hexl_b200_keys* galois_keys, const uint64_t* modswitch_factors,
                                      uint64_t galois_elt, uint64_t batch, void* stream);

/* Hoisted rotations (extension; OpenFHE's EvalFastRotationPrecompute + EvalFastRotation): each of `batch` ciphertexts
 * rotated by each of num_elts Galois elements in one call, its digits decomposed and transformed ONCE for every
 * element.  Input ciphertext c is at ciphertexts + c * 2 * decomp * n, laid out as for
 * hexl_b200_apply_galois_key_switch; its rotation by galois_elts[r] with galois_keys[r] is written to
 * results + (c * num_elts + r) * 2 * decomp * n.  Out of place: ciphertexts is not modified.  For c = (c0, c1):
 *   a_j        = INTT_{q_j}(c1_j)                          digit j < decomp, in [0, q_j)
 *   D_{j,i}    = NTT_{q_i}(a_j mod q_i)                    every modulus i of the switch
 *   prod_{i,k} = sum_j pi_g(D_{j,i}) (.) K[j][k][i]  mod q_i
 *   out        = [sigma_g(c0), 0] + ModDown(prod)           (the mod-down of hexl_b200_key_switch)
 * with pi_g / sigma_g the NTT-form automorphism of hexl_b200_apply_galois.  This is the key switch of sigma_g(c1)
 * with digit j's coefficients lifted to the signed integers sigma_g(a_j) (entries +-a_j[t], below q_j in magnitude)
 * instead of to [0, q_j), so it is NOT bit-identical to hexl_b200_apply_galois_key_switch: the two differ where
 * sigma_g negates a nonzero coefficient, by q_j mod q_i in digit j's extended limbs; for g = 1 they are equal bit for
 * bit.  The decryption noise bound is the same.  HEXL_B200_ERR_INVALID_ARG on the shape rules of
 * hexl_b200_apply_galois_key_switch applied to every key handle (null, another shape, or sharded by modulus), for any
 * element outside the rules of hexl_b200_apply_galois, and when results overlaps ciphertexts.  Elements may repeat.
 * num_elts = 0 or batch = 0 does nothing.  Inputs are checked below their modulus under hexl_b200_set_debug(1).
 * On the device, per ciphertext: one inverse transform of the digits and one gathered forward transform per round of
 * moduli, shared by every element; per element, its multiply-accumulates, one automorphism launch of c0 straight into
 * the output, a memset of the output's c1 and its mod-down.  For one element these are the launches of
 * hexl_b200_apply_galois_key_switch.  Library scratch is one round of transformed digits, as for the key switch, plus
 * num_elts x rns x 2 x n words of products: about the size of one ciphertext's results.  Host buffers: each ciphertext
 * crosses PCIe in once and its num_elts rotations come back on the same staging stream, pipelined and split by
 * ciphertext over the devices of hexl_b200_set_host_devices where every key handle holds a copy. */
int hexl_b200_apply_galois_key_switch_hoisted(uint64_t* results, const uint64_t* ciphertexts, uint64_t n,
                                              uint64_t decomp_modulus_size, uint64_t key_modulus_size,
                                              uint64_t rns_modulus_size, uint64_t key_component_count,
                                              const uint64_t* moduli, const hexl_b200_keys* const* galois_keys,
                                              const uint64_t* galois_elts, uint64_t num_elts,
                                              const uint64_t* modswitch_factors, uint64_t batch, void* stream);

/* Fast base conversion (extension; OpenFHE's ApproxSwitchCRTBasis, SEAL's BaseConverter::fast_convert_array),
 * coefficient form: `count` polynomials; polynomial p reads from_count limbs of n words at operand + p*from_count*n
 * (limb i under from_moduli[i]) and writes to_count limbs at result + p*to_count*n (limb e under to_moduli[e]):
 *   result_e = [ sum_i [x_i (Q/q_i)^-1]_{q_i} [Q/q_i]_{t_e} ]_{t_e},  Q = prod from_moduli,
 * canonical.  That is X + u Q mod t_e, X the CRT lift of the x_i in [0, Q) and 0 <= u < from_count.  A target equal to
 * a source modulus q_i gets x_i back.  HEXL_B200_ERR_INVALID_ARG unless every pointer is non-null, n >= 1,
 * 1 <= from_count <= 64, to_count >= 1, every modulus is in (1, 2^61), the from_moduli are pairwise coprime, and result
 * and operand do not overlap.  Inputs must be below their modulus (checked under hexl_b200_set_debug(1)).  count = 0
 * does nothing.  One launch per block of targets (up to 79 for from_count = 1, 3 for from_count = 64: the constants
 * travel in the kernel parameters, so a device call can be captured into a CUDA graph).  Host buffers are staged by
 * whole polynomials and split by polynomial over the devices of hexl_b200_set_host_devices. */
int hexl_b200_fast_base_convert(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* from_moduli,
                                uint64_t from_count, const uint64_t* to_moduli, uint64_t to_count, uint64_t count,
                                void* stream);

/* Hybrid key switch (extension; OpenFHE's KeySwitchHYBRID) of `batch` ciphertexts at level level_size = l.  moduli
 * holds q_size data moduli q_0..q_{L-1} and then p_size special primes p_0..p_{K-1} (P = prod p_k), all distinct,
 * NTT-friendly for n and below 2^61.  Digit d covers the data moduli [d a, min((d+1) a, L)), a = digit_size; the key
 * handle holds dnum = ceil(L / a) buffers of key_component_count x (L + K) x n words in NTT form, limb i < L under q_i
 * and limb L + k under p_k (hexl_b200_keys_upload with decomp = dnum, key_modulus_size = L + K).  Ciphertext c reads
 * its target, l limbs in NTT form, canonical, at target + c*l*n, and accumulates into key_component_count x l limbs at
 * result + c*key_component_count*l*n.  With S_d = [d a, min((d+1) a, l)) for d < D = ceil(l / a), Q_d = prod_{S_d} q_i
 * and B = {q_0..q_{l-1}, p_0..p_{K-1}}:
 *   a_i        = INTT_{q_i}(t_i)
 *   D_{d,m}    = NTT_m([ sum_{i in S_d} [a_i (Q_d/q_i)^-1]_{q_i} [Q_d/q_i]_m ]_m)     mod-up, every m in B
 *   prod_{m,k} = sum_{d<D} D_{d,m} keys[d][k][slot(m)] mod m,  slot(q_i) = i, slot(p_j) = L + j
 *   x_j        = INTT_{p_j}(prod_{p_j,k}),  z_j = [(x_j + floor(P/2)) (P/p_j)^-1]_{p_j}
 *   c_i        = [ sum_j z_j [P/p_j]_{q_i} - floor(P/2) ]_{q_i}                       mod-down, rounded
 *   result_{k,i} += (prod_{q_i,k} - NTT_{q_i}(c_i)) P^-1 mod q_i, canonical.
 * With digit_size = 1 and p_size = 1 this is bit for bit hexl_b200_key_switch_resident with decomp = l,
 * key_modulus_size = L + 1 and modswitch factors p^-1 mod q_i.  The library computes every constant itself.
 * HEXL_B200_ERR_INVALID_ARG for a null pointer, n not a power of two in [2, 2^20], level_size outside [1, q_size],
 * digit_size or p_size outside [1, 64], key_component_count = 0, a modulus that is not NTT-friendly, is >= 2^61 or
 * repeats, a handle of another shape or sharded by modulus, and result overlapping target.  batch = 0 does nothing.
 * Inputs are checked below their modulus under hexl_b200_set_debug(1).  On the device, per ciphertext: one inverse
 * transform of the target; per round of at most 64 moduli of B (and ~256 MiB of scratch), one base-conversion launch
 * per digit and block of targets, one forward transform and the multiply-accumulates; then one inverse transform of
 * the special limbs and, per block of 64 data moduli, the rounding base conversion, one forward transform and the
 * finish step.  Device calls capture into a CUDA graph once the transforms are warm.  Host buffers are pipelined and
 * split by ciphertext over the devices holding the keys, as for hexl_b200_key_switch_resident. */
int hexl_b200_key_switch_hybrid(uint64_t* result, const uint64_t* target, uint64_t n, uint64_t level_size,
                                uint64_t q_size, uint64_t p_size, uint64_t digit_size, uint64_t key_component_count,
                                const uint64_t* moduli, const hexl_b200_keys* keys, uint64_t batch, void* stream);

/* Hoisted rotations with hybrid keys (extension; OpenFHE's EvalFastRotation with KeySwitchHYBRID): each of `batch`
 * ciphertexts rotated by each of num_elts Galois elements, its mod-up done ONCE for every element.  The moduli, digits
 * and shape rules are those of hexl_b200_key_switch_hybrid with key_component_count = 2; galois_keys[r] is a hybrid key
 * handle (dnum = ceil(q_size / digit_size) buffers of 2 x (q_size + p_size) x n words) that switches s(X^g) back to s
 * for g = galois_elts[r].  Ciphertext c is two components of l = level_size limbs in NTT form, canonical, at
 * ciphertexts + c * 2 * l * n; its rotation by galois_elts[r] is written to results + (c * num_elts + r) * 2 * l * n.
 * Out of place: ciphertexts is not modified.  With the mod-up D_{d,m} and ModDown_P of hexl_b200_key_switch_hybrid
 * applied to t = c1:
 *   prod^r_{m,k} = sum_d pi_g(D_{d,m}) (.) K_r[d][k][slot(m)]  mod m,  every m in B
 *   out_r        = [sigma_g(c0), 0] + ModDown_P(prod^r)
 * with pi_g / sigma_g the NTT-form automorphism of hexl_b200_apply_galois.  Permuting the converted digits lifts digit
 * d to the signed integers sigma_g(X + u Q_d) instead of sigma_g applied after an unsigned lift, so for g != 1 this is
 * NOT bit-identical to the chain hexl_b200_apply_galois + hexl_b200_key_switch_hybrid; the lift is below alpha Q_d in
 * magnitude either way, so the decryption noise bound is the same.  For g = 1 it is that chain bit for bit, and with
 * digit_size = 1 and p_size = 1 it is hexl_b200_apply_galois_key_switch_hoisted bit for bit (decomp = l,
 * key_modulus_size = q_size + 1, modswitch factors p^-1 mod q_i).  Elements may repeat.  num_elts = 0 or batch = 0
 * does nothing.  HEXL_B200_ERR_INVALID_ARG on the shape rules of hexl_b200_key_switch_hybrid applied to every handle
 * (null, another shape, or sharded by modulus), for an element outside the rules of hexl_b200_apply_galois, and when
 * results overlaps ciphertexts.  Inputs are checked below their modulus under hexl_b200_set_debug(1).  On the device,
 * per ciphertext: the mod-up of hexl_b200_key_switch_hybrid once; per element, one automorphism launch of c0 into the
 * output, a memset of the output's c1, its multiply-accumulates and its mod-down.  Library scratch: one round of
 * converted digits plus num_elts x (l + p_size) x 2 x n words of products.  Device calls capture into a CUDA graph
 * once the transforms are warm.  Host buffers: each ciphertext crosses PCIe in once and its rotations come back on the
 * same staging stream, split by ciphertext over the devices of hexl_b200_set_host_devices where every handle holds a
 * copy. */
int hexl_b200_apply_galois_key_switch_hybrid_hoisted(uint64_t* results, const uint64_t* ciphertexts, uint64_t n,
                                                     uint64_t level_size, uint64_t q_size, uint64_t p_size,
                                                     uint64_t digit_size, const uint64_t* moduli,
                                                     const hexl_b200_keys* const* galois_keys,
                                                     const uint64_t* galois_elts, uint64_t num_elts, uint64_t batch,
                                                     void* stream);

/* Linear transform with hybrid keys (extension; Lattigo's MultiplyByDiagMatrix, OpenFHE's EvalLinearTransform): the
 * plaintext-matrix x ciphertext product in diagonal form, sum_r w_r (.) Rot_{g_r}(ct), for each of `batch`
 * ciphertexts, with ONE mod-down for the whole sum.  Arguments, layouts and rules as for
 * hexl_b200_apply_galois_key_switch_hybrid_hoisted, plus diagonals: num_elts x (l + p_size) x n words in NTT form,
 * canonical; limb i < l of diagonal r is under q_i and limb l + j under p_j.  Ciphertext c goes to
 * result + c * 2 * l * n.  With prod^r of the hoisted call and I the identity terms (g_r = 1 with galois_keys[r] null,
 * which add w_r (.) ct and switch no key):
 *   acc_{m,k} = sum_{r not in I} w_{r,m} (.) prod^r_{m,k}  mod m,  every m in B
 *   result    = [sum_r w_r (.) sigma_{g_r}(c0), sum_{r in I} w_r (.) c1] + ModDown_P(acc)
 * canonical; when every term is an identity term there is no key switch and no ModDown term.  Weighting in the
 * extended basis and rounding once is what makes the single mod-down possible, so the result is NOT the sum of
 * weighted hoisted rotations bit for bit (that rounds once per element); with one element and every diagonal word 1 it
 * equals hexl_b200_apply_galois_key_switch_hybrid_hoisted bit for bit.  A null handle for g != 1 is refused
 * (HEXL_B200_ERR_INVALID_ARG), as are the refusals of the hoisted call and a result overlapping the ciphertexts or the
 * diagonals.  Elements may repeat.  num_elts = 0 or batch = 0 does nothing.  Inputs, the diagonals included, are
 * checked below their modulus under hexl_b200_set_debug(1).  On the device, per ciphertext: one weighted permuted-sum
 * launch per chunk of 64 elements and block of 64 data moduli (stores [sum w sigma(c0), sum_I w c1]); then, when some
 * element has keys, the mod-up once, per round of moduli one weighted multiply-accumulate launch per chunk of
 * (element, digit) pairs (at most 64 pairs, each launch adding into one accumulator of (l + p_size) x 2 x n words
 * without writing per-element products), and one mod-down.  Device calls capture into a CUDA graph once the transforms
 * are warm.  Host buffers: the diagonals go to each device once per call, before its first ciphertext; the ciphertexts
 * are pipelined and split over the devices as for the hoisted call. */
int hexl_b200_linear_transform_hybrid(uint64_t* result, const uint64_t* ciphertexts, uint64_t n, uint64_t level_size,
                                      uint64_t q_size, uint64_t p_size, uint64_t digit_size, const uint64_t* moduli,
                                      const hexl_b200_keys* const* galois_keys, const uint64_t* galois_elts,
                                      uint64_t num_elts, const uint64_t* diagonals, uint64_t batch, void* stream);

/* Baby-step giant-step linear transform with hybrid keys, double-hoisted (extension; Bossuat et al., Eurocrypt 2021,
 * Alg. 6; Lattigo's MultiplyByDiagMatrixBSGS; OpenFHE's EvalFastRotationExt + KeySwitchDown): the plaintext-matrix x
 * ciphertext product sum_j sigma_{h_j}( sum_i w_{j,i} (.) sigma_{b_i}(ct) ) over a num_giant x num_baby grid of
 * diagonals, for each of `batch` ciphertexts, with n1 + n2 Galois keys instead of the n1 n2 of
 * hexl_b200_linear_transform_hybrid.  The baby rotations' mod-up runs once, their products and the inner sums stay in
 * the extended basis B = {q_0..q_{l-1}, p_0..p_{K-1}}, each giant step takes only its c1 part down to Q, and the result
 * is rounded once at the end.  The moduli, digits, shape rules, key handles and layouts are those of
 * hexl_b200_apply_galois_key_switch_hybrid_hoisted: baby_keys[i] switches s(X^{b_i}) to s for b_i = baby_elts[i], and
 * giant_keys[j] s(X^{h_j}) to s for h_j = giant_elts[j].  A null handle is an identity term, allowed for the element 1
 * only, on either side.  Every element is odd and in [1, 2n); elements may repeat.  diagonals is a host array of
 * num_giant x num_baby pointers: diagonals[j * num_baby + i] is null (the pair is absent and costs nothing) or points at
 * (l + p_size) x n words in NTT form, canonical, limb i < l under q_i and limb l + j under p_j, in the memory kind of
 * the ciphertexts.  Ciphertext c (two components of l = level_size limbs, NTT form, canonical) is read at
 * ciphertexts + c * 2 * l * n and its result STORED at result + c * 2 * l' * n, l' = l - rescale.
 * With the mod-up D_{d,m} of hexl_b200_key_switch_hybrid, prod^b_{m,k} = sum_d pi_b(D_{d,m}(c1)) (.) K_b[d][k][slot(m)]
 * the products of the hoisted call, and R_j the babies with a diagonal in row j, a pair (X, Y) with X on the data limbs
 * (from 0) and Y two components over B (from empty):
 *   x0_j  = sum_{i in R_j} w_{j,i} (.) sigma_{b_i}(c0),  x1_j = sum_{i in R_j, b_i identity} w_{j,i} (.) c1
 *   y_j,k = sum_{i in R_j, b_i keyed} w_{j,i} (.) prod^{b_i}_k                                     every m in B
 *   identity giant:  X += (x0_j, x1_j);  Y += (y_j,0, y_j,1)
 *   keyed giant h:   c1'_j = x1_j + ModDown_P(y_j,1)          (no ModDown when R_j has no keyed baby)
 *                    X0 += sigma_h(x0_j);  Y0 += sigma_h(y_j,0)   (pi_h on the special limbs too)
 *                    Y_k += sum_d pi_h(D_{d,m}(c1'_j)) (.) K_h[d][k][slot(m)]  (a fresh mod-up of c1'_j)
 *   rescale = 0:     result = X + ModDown_P(Y)                  (result = X while Y is empty)
 *   rescale = 1:     ext_{q_i,k} = Y_{q_i,k} + [P]_{q_i} X_{k,i},  ext_{p_j,k} = Y_{p_j,k};  result = the mod-down of
 *                    ext by q_{l-1} P of hexl_b200_multiply_relinearize_hybrid (l - 1 limbs)
 * canonical; a row without a present diagonal adds nothing.  X is kept apart from Y because ModDown_P(P x) need not
 * be x for K > 1 (its rounded base conversion of zero special limbs gives u P, 0 <= u < K), while
 * ModDown_P(P x + y) = x + ModDown_P(y) bit for bit.  Hence, bit for bit: with one identity giant (element 1, null key)
 * this is hexl_b200_linear_transform_hybrid over the babies with the absent diagonals as zero ones; with one identity
 * baby and every diagonal word 1 it is hexl_b200_linear_transform_hybrid over the giants with unit diagonals, and with
 * one giant as well, hexl_b200_apply_galois_key_switch_hybrid_hoisted.  It decrypts to
 * sum_j sigma_{h_j}(sum_i w_{j,i} (.) sigma_{b_i}(phase(ct))), divided by q_{l-1} and rounded with rescale = 1, within
 * the linear transform's bound plus, per keyed giant, one key switch and the rounding of c1'_j times s.
 * HEXL_B200_ERR_INVALID_ARG on the refusals of the hoisted call applied to every non-null handle (another shape,
 * sharded by modulus), a null handle for an element other than 1, rescale other than 0 or 1, rescale = 1 with
 * level_size < 2 or p_size > 63, a null diagonals array when num_baby x num_giant > 0, and result overlapping the
 * ciphertexts or a present diagonal.  num_baby = 0, num_giant = 0 or batch = 0 does nothing.  Inputs, the present
 * diagonals included, are checked below their modulus under hexl_b200_set_debug(1).
 * On the device, per ciphertext: (1) when some keyed baby has a diagonal, the mod-up of c1 once, and per round the
 * multiply-accumulates of those babies, their products stored; (2) per giant step with a present diagonal, one sum
 * launch per block of 64 moduli of B (of the data moduli only when the row has no keyed baby) and chunk of 64 present
 * babies, which applies pi_h on load; (3) per keyed giant step, the mod-down of y_j,1 into x1_j (one component, none
 * without a keyed baby), then the mod-up of c1'_j with multiply-accumulates adding into Y through pi_h; (4) the
 * mod-down of Y, adding into result (none while Y is empty), or with rescale = 1 the [P] X fold in the last sum launch
 * and the mod-down by q_{l-1} P that stores.  Library scratch: n1' x (l + p_size) x 2 x n words of stored baby
 * products, n1' the keyed babies with a diagonal (336 MB at n1' = 8, l = 30, K = 10, n = 2^16), plus Y, one round of
 * converted digits and a few l x n buffers.  Device calls capture into a CUDA graph once the transforms are warm.
 * Host buffers: the present diagonals go to each device once per call, before its first ciphertext; the ciphertexts
 * are pipelined and split by ciphertext over the devices of hexl_b200_set_host_devices where every non-null handle
 * holds a copy.  Managed buffers take the device path.  Not covered: keys sharded by modulus (refused), encoding the
 * diagonals (pre-rotating them by -h_j is the caller's), and mapping rotation steps to elements. */
int hexl_b200_linear_transform_hybrid_bsgs(uint64_t* result, const uint64_t* ciphertexts, uint64_t n,
                                           uint64_t level_size, uint64_t q_size, uint64_t p_size, uint64_t digit_size,
                                           const uint64_t* moduli, const hexl_b200_keys* const* baby_keys,
                                           const uint64_t* baby_elts, uint64_t num_baby,
                                           const hexl_b200_keys* const* giant_keys, const uint64_t* giant_elts,
                                           uint64_t num_giant, const uint64_t* const* diagonals, int rescale,
                                           uint64_t batch, void* stream);

/* Ciphertext multiplication with relinearization by hybrid keys (extension; CKKS HMult: SEAL's multiply + relinearize
 * [+ rescale_to_next], OpenFHE's EvalMult), optionally rescaled in the same mod-down, for each of `batch` pairs.  The
 * moduli, digits and shape rules are those of hexl_b200_key_switch_hybrid with key_component_count = 2; relin_keys is
 * a hybrid key handle (dnum = ceil(q_size / digit_size) buffers of 2 x (q_size + p_size) x n words) that switches s^2
 * to s.  Pair c reads ct1 + c * 2 * l * n and ct2 + c * 2 * l * n (two components of l = level_size limbs each, NTT
 * form, canonical) and its product is STORED at result + c * 2 * l' * n, l' = l - rescale.  With (a0, a1) = ct1,
 * (b0, b1) = ct2, the mod-up D_{d,m}, keys K and slot(m) of hexl_b200_key_switch_hybrid, and P = prod p_j:
 *   d0 = a0 (.) b0,  d1 = a0 (.) b1 + a1 (.) b0,  t = a1 (.) b1           per data limb, canonical
 *   prod_{m,k} = sum_d D_{d,m}(t) (.) K[d][k][slot(m)]  mod m,             every m in B
 *   ext_{m,k}  = prod_{m,k} + [P]_m d_{k,m} for m = q_i, i < l;  ext_{p_j,k} = prod_{p_j,k}
 *   T = {p_0..p_{K-1}} (rescale = 0) or {q_{l-1}, p_0..p_{K-1}} (rescale = 1),  P_T = prod T
 *   x_t = INTT_t(ext_{t,k}),  z_t = [(x_t + floor(P_T/2)) (P_T/t)^-1]_t                          every t in T
 *   c_i = [ sum_t z_t [P_T/t]_{q_i} - floor(P_T/2) ]_{q_i},  result_{k,i} = (ext_{q_i,k} - NTT_{q_i}(c_i)) P_T^-1
 *   mod q_i, canonical, for i < l'.
 * rescale = 0 is bit for bit hexl_b200_dyadic_multiply followed by hexl_b200_key_switch_hybrid of d2 into (d0, d1): the
 * mod-down reads only the special limbs, where ext = prod, and (prod + P d - NTT(c)) P^-1 = (prod - NTT(c)) P^-1 + d
 * mod q_i with both sides canonical.  At digit_size = 1 with one special prime it is therefore hexl_b200_dyadic_multiply
 * followed by hexl_b200_key_switch_resident (SEAL's multiply + relinearize) bit for bit.  rescale = 1 is NOT that
 * chain followed by hexl_b200_divide_and_round_q_last bit for bit: it rounds once, by q_{l-1} P, where the chain rounds
 * by P and then by q_{l-1}.  It decrypts to round(phase(ct1) phase(ct2) / q_{l-1}) within the key switch's error
 * divided by q_{l-1} plus one rounding term of K + 1 sources.  ct1 == ct2 (squaring) is allowed; any other overlap
 * of the inputs, and any overlap of result with an input, is refused.  HEXL_B200_ERR_INVALID_ARG on the refusals of
 * hexl_b200_key_switch_hybrid with key_component_count = 2, on rescale other than 0 or 1, on rescale = 1 with
 * level_size < 2 or p_size > 63 (the merged mod-down converts from K + 1 <= 64 moduli), and on those overlaps.
 * batch = 0 does nothing.  Inputs are checked below their modulus under hexl_b200_set_debug(1).  On the device, per
 * pair: the mod-up of hexl_b200_key_switch_hybrid applied to t, whose first inverse transform multiplies a1 by b1 on
 * load (t is never written); per round of moduli of B, one multiply-accumulate launch per chunk of digits within the
 * 128-bit bound, the first of which reads a0, a1, b0, b1 on the data moduli and adds [P] d; then one mod-down by P_T
 * that stores into result.  These are the launches of hexl_b200_key_switch_hybrid, with K + 1 special limbs and l - 1
 * targets in the mod-down when rescale = 1.  Library scratch: one round of converted digits plus (l + p_size) x 2 x n
 * words of products.  Device calls capture into a CUDA graph once the transforms are warm.  Host buffers: both
 * ciphertexts of a pair cross PCIe in once (one copy when squaring) and the product comes back on the same staging
 * stream, split by pair over the devices of hexl_b200_set_host_devices where the handle holds a copy. */
int hexl_b200_multiply_relinearize_hybrid(uint64_t* result, const uint64_t* ct1, const uint64_t* ct2, uint64_t n,
                                          uint64_t level_size, uint64_t q_size, uint64_t p_size, uint64_t digit_size,
                                          const uint64_t* moduli, const hexl_b200_keys* relin_keys, int rescale,
                                          uint64_t batch, void* stream);

/* A sum of ciphertext products relinearized once with hybrid keys (extension; lazy relinearization: Lattigo's MulThenAdd
 * followed by one Relinearize, OpenFHE's EvalMultNoRelin + EvalAdd + Relinearize), optionally rescaled in the same
 * mod-down, for each of `batch` outputs: the inner products, the k-sums of matrix products and the sums of products of
 * polynomial evaluation.  Relinearization is linear in the tensor's last term, so one key switch serves the whole sum.
 * ct1 and ct2 are host arrays of batch x num_pairs pointers: entry c * num_pairs + r is pair r of output c and points at
 * one ciphertext (two components of l = level_size limbs, NTT form, canonical, in the memory kind of result).  Output c
 * is STORED at result + c * 2 * l' * n, l' = l - rescale.  The moduli, digits, key handle (one relinearization key,
 * s^2 -> s) and shape rules are those of hexl_b200_multiply_relinearize_hybrid.  With (a0_r, a1_r) = ct1[c * num_pairs
 * + r] and (b0_r, b1_r) = ct2[c * num_pairs + r], per data limb i < l:
 *   d0 = sum_r a0_r (.) b0_r,  d1 = sum_r (a0_r (.) b1_r + a1_r (.) b0_r),  t = sum_r a1_r (.) b1_r      mod q_i, canonical
 * and from there the steps of hexl_b200_multiply_relinearize_hybrid from "prod = the mod-up of t times the keys" on,
 * unchanged: ext = prod + [P] d on the data limbs, then the mod-down by P or by q_{l-1} P.  Hence, bit for bit:
 * num_pairs = 1 is hexl_b200_multiply_relinearize_hybrid in both rescale modes; rescale = 0 is hexl_b200_dyadic_multiply
 * of every pair, the three components summed with hexl_b200_eltwise_add_mod_multi, then hexl_b200_key_switch_hybrid of
 * the summed d2 into the summed (d0, d1).  It is NOT the sum of the num_pairs products of
 * hexl_b200_multiply_relinearize_hybrid bit for bit: that sum rounds num_pairs times and carries num_pairs key-switch
 * errors.  It decrypts to sum_r phase(ct1_r) phase(ct2_r), divided by q_{l-1} and rounded with rescale = 1, within the
 * bound of ONE relinearization.  Inputs are only read: they may repeat and overlap freely (a ciphertext may appear in
 * several pairs and outputs, and ct1[x] == ct2[x] squares it); result must not overlap any of them.
 * HEXL_B200_ERR_INVALID_ARG on every refusal of hexl_b200_multiply_relinearize_hybrid (shape, handle, rescale other than
 * 0 or 1, rescale = 1 with level_size < 2 or p_size > 63), a null array when batch x num_pairs > 0, a null entry in
 * either array, and result overlapping an input; HEXL_B200_ERR_MIXED_POINTERS when result and the entries are not all
 * of one memory kind (and device).  num_pairs = 0 or batch = 0 does nothing.  Every distinct input is checked below its
 * modulus under hexl_b200_set_debug(1).  On the device, per output: num_pairs = 1 runs the launches of
 * hexl_b200_multiply_relinearize_hybrid.  Otherwise one tensor-sum launch per block of 64 data limbs and chunk of 32
 * pairs (d1's 128-bit sum takes two products per pair: 64 x (2^61 - 1)^2 < 2^128, so the sums are exact for every
 * modulus below 2^61 and every num_pairs) stores (d0, d1, t), then the launches of hexl_b200_multiply_relinearize_hybrid,
 * whose mod-up reads t (its first inverse transform launches as with the multiply on load) and whose storing
 * multiply-accumulate reads d0 and d1: ceil(l / 64) x ceil(num_pairs / 32) launches more than one product.  Library
 * scratch: 3 x l x n words plus that of hexl_b200_multiply_relinearize_hybrid.  Device calls capture into a CUDA graph
 * once the transforms are warm.  Host buffers: every distinct input goes to each device of the
 * hexl_b200_set_host_devices split once per call, before its first output; the outputs are split by output over the
 * devices where the handle holds a copy and each comes back from its staging slot.  Managed buffers take the device
 * path.  Not covered: keys sharded by modulus (refused), plaintext-weighted sums, and an in-place variant. */
int hexl_b200_multiply_relinearize_sum_hybrid(uint64_t* result, const uint64_t* const* ct1, const uint64_t* const* ct2,
                                              uint64_t num_pairs, uint64_t n, uint64_t level_size, uint64_t q_size,
                                              uint64_t p_size, uint64_t digit_size, const uint64_t* moduli,
                                              const hexl_b200_keys* relin_keys, int rescale, uint64_t batch,
                                              void* stream);

/* The inner sum of k = sum_count rotations with hybrid keys (extension; Lattigo's InnerSum, OpenFHE's EvalSum, the last
 * step of EvalInnerProduct): sum_{j<k} sigma_{g^j}(ct) for g = galois_elt, for each of `batch` ciphertexts, by the
 * log-step recurrence A <- A + Rot(A) kept in the extended basis B = {q_0..q_{l-1}, p_0..p_{K-1}} and rounded once at
 * the end, the rescale optionally merged into that mod-down.  The moduli, digits, shape rules, handle rules (non-null,
 * the right shape, not sharded), layouts, rescale (l' = l - rescale), memory kinds, batch splitting and debug checks are
 * those of hexl_b200_linear_transform_hybrid_bsgs: ciphertext c (two components of l = level_size limbs, NTT form,
 * canonical) is read at ciphertexts + c * 2 * l * n and its sum STORED at result + c * 2 * l' * n.
 * (key_elts[r], galois_keys[r]) for r < num_keys is a table of available keys (galois_keys[r] switches s(X^e) to s for
 * e = key_elts[r]); the call looks up the elements it needs there (the first match), so one set of keys for the powers
 * g^(2^i) serves every sum_count.  With pi_e / sigma_e the NTT-form automorphism of hexl_b200_apply_galois, elements
 * reduced mod 2n, the mod-up D_{d,m} and keys K of hexl_b200_key_switch_hybrid, and a pair (X, Y) as in the BSGS call
 * (X two components on the data limbs, Y two components over B or empty, val = X + ModDown_P(Y)):
 *   Rot_1(X, Y)  = (X, Y)                                                       (no key)
 *   Rot_e(X, Y)  = ((sigma_e X0, 0), (pi_e Y0 + M_e,0, M_e,1)),  c1' = X1 + ModDown_P(Y1) (X1 while Y is empty),
 *                  M_e,k = sum_d pi_e(D_{d,m}(c1')) (.) K_e[d][k][slot(m)]                         every m in B
 *   A = (ct, empty);  R = none;  s = 0
 *   for i = 0 .. floor(log2 k):
 *     if bit i of k is set:  R = Rot_{g^s}(A) (R none) or R + Rot_{g^s}(A);  s += 2^i
 *     if 2^(i+1) <= k:       A = A + Rot_{g^(2^i)}(A)
 *   rescale = 0:  result = X_R + ModDown_P(Y_R)      (X_R while Y_R is empty)
 *   rescale = 1:  [P] X_R folded into Y_R's data limbs and the mod-down by q_{l-1} P, as in the BSGS call
 * Pairs add component-wise, an empty Y as zero.  Both rotations of one bit read the same A, so they share one c1' and
 * one mod-up (hoisted).  The needed elements are g^(2^i) for 2^(i+1) <= k and g^s at every set bit but the lowest; one
 * equal to 1 (mod 2n) is an identity and needs no key (the conjugation 2n - 1 squared is 1).  It decrypts to
 * sum_{j<k} sigma_{g^j}(phase(ct)), divided by q_{l-1} and rounded with rescale = 1, within one key switch and one
 * rounding of c1' times s per keyed rotation, carried through the sum.  Canonical modular sums do not depend on their
 * order, so bit for bit: k = 1 is hexl_b200_linear_transform_hybrid_bsgs with one identity baby, one identity giant and
 * a unit diagonal (a copy of ct with rescale = 0); k = 2 is hexl_b200_apply_galois_key_switch_hybrid_hoisted by g plus
 * hexl_b200_eltwise_add_mod_multi with ct, and hexl_b200_linear_transform_hybrid over {1, g} with unit diagonals;
 * k = 3 is the BSGS call with babies {1, g}, giants {1, g}, unit diagonals and the (giant 1, baby g) pair absent, and
 * k = 4 the BSGS call with babies {1, g}, giants {1, g^2} and four unit diagonals, both in both rescale modes.  For
 * k >= 5 it is a nested chain of such steps, not one BSGS call.  It is NOT the chain of separately rounded hoisted
 * rotations and additions bit for bit: that rounds once per rotation.
 * HEXL_B200_ERR_INVALID_ARG on the shape refusals of hexl_b200_key_switch_hybrid, galois_elt even or outside [1, 2n),
 * a needed element other than 1 missing from key_elts (the message names it), a null or misshapen handle for a needed
 * element, rescale other than 0 or 1, rescale = 1 with level_size < 2 or p_size > 63, null galois_keys or key_elts with
 * num_keys > 0, and result overlapping the ciphertexts.  sum_count = 0 or batch = 0 does nothing.
 * On the device, per ciphertext and bit i of k: one step launch per block of 64 moduli of B (of the data moduli only
 * while no Y is read or written), which writes A' = A + pi_d(A0) into the other buffer of a ping-pong pair and adds
 * pi_s(A0) into R; then, when the bit has a keyed element, the one-component mod-down of Y_A1 (none while Y_A is empty)
 * and one mod-up of c1' whose multiply-accumulates add the products of the bit's one or two keyed elements into Y_A'
 * and Y_R; after the last bit, the mod-down of Y_R (none while it is empty), or the merged one with rescale = 1.  So a
 * ciphertext takes sum_i (ceil(span_i / 64) + [keyed_i] (down_1 [Y_A non-empty] + up(e_i))) + down_2 launches, span_i
 * = l or l + K, e_i <= 2 its keyed elements, up(e) the launches of the mod-up of hexl_b200_key_switch_hybrid with e
 * multiply-accumulate sets (ceil(l / alpha) digits) and down_c those of its mod-down of c components (0 while Y_R is
 * empty without the rescale).  Library scratch: two pairs for A and R (5 x (l + K) x 2 x n words and less), one round of
 * converted digits and a few l x n buffers.  Device calls capture into a CUDA graph once the transforms are warm.  Host
 * buffers: each ciphertext crosses PCIe in once and its sum comes back on the same staging stream, split by ciphertext
 * over the devices of hexl_b200_set_host_devices where every needed handle holds a copy.  Managed buffers take the
 * device path.  Not covered: keys sharded by modulus (refused), mapping rotation steps to elements, sums over other
 * than the powers of one element, and an in-place variant. */
int hexl_b200_inner_sum_hybrid(uint64_t* result, const uint64_t* ciphertexts, uint64_t n, uint64_t level_size,
                               uint64_t q_size, uint64_t p_size, uint64_t digit_size, const uint64_t* moduli,
                               uint64_t galois_elt, uint64_t sum_count, const hexl_b200_keys* const* galois_keys,
                               const uint64_t* key_elts, uint64_t num_keys, int rescale, uint64_t batch, void* stream);

/* BFV ciphertext multiplication by BEHZ (extension; Bajard, Eynard, Hasan, Zucca 2016; SEAL's Evaluator::multiply for
 * BFV with its RNSTool): the tensor of two ciphertexts scaled by t/Q, integer arithmetic only, for each of `batch`
 * pairs.  Q = q_0..q_{l-1} (moduli, l = level_size), B = b_0..b_{k-1} (base_b, k = base_b_size), Bsk = B u {m_sk},
 * m~ = 2^32 and t = plain_modulus.  Pair c reads ct1 + c*2*l*n and ct2 + c*2*l*n, two components of l limbs each in
 * COEFFICIENT form (SEAL's BFV form), canonical; its product is STORED at result + c*3*l*n as (d0, d1, d2), l limbs
 * each, coefficient form, canonical.  With FBC the conversion of hexl_b200_fast_base_convert, per input polynomial x:
 *   y_i  = [x_i m~]_{q_i},  z_m = FBC(y; Q -> m) for m in Bsk u {m~}
 *   r    = [-z_m~ Q^-1]_m~,  r_c = r - m~ if r >= m~/2 else r
 *   x'_m = [(z_m + [Q]_m r_c) m~^-1]_m for m in Bsk,  x'_{q_i} = x_i                       (SEAL's sm_mrq)
 * per modulus m of Q u Bsk, (a0, a1) and (b0, b1) the lifted inputs, negacyclic products mod m (forward NTT, dyadic,
 * inverse NTT):
 *   D0 = a0 b0,  D1 = a0 b1 + a1 b0,  D2 = a1 b1
 * and per output polynomial D over Q u Bsk:
 *   u_i   = [t D_{q_i}]_{q_i},  w_m = [(t D_m - FBC(u; Q -> m)) [Q^-1]_m]_m for m in Bsk    (fast_floor)
 *   c_i   = FBC(w_B; B -> q_i),  gamma = FBC(w_B; B -> m_sk),  alpha = [(gamma - w_{m_sk}) [B^-1]_{m_sk}]_{m_sk}
 *   out_i = [c_i + [B]_{q_i} (m_sk - alpha)]_{q_i} if alpha > floor(m_sk/2), else [c_i - [B]_{q_i} alpha]_{q_i}
 *                                                                                                (fastbconv_sk)
 * Each out coefficient is floor(t D / Q) - v mod Q with 0 <= v < l, D the integer tensor of the lifts, exactly when
 * Bsk passes this bound, which the call checks with exact integers:
 *   n t Q (m~ + 2l)^2 + 2 (l + 1) m~^2 <= B (m_sk - 1 - 2k) m~^2.
 * Why: the lift is x' = x mod Q with -Q/2 <= x' < lambda Q, lambda = 1/2 + l/m~; so |D| < 2 n lambda^2 Q^2 (D1 sums 2n
 * products); the fast floor gives w = floor(t D / Q) - v, |w| < 2 n t lambda^2 Q + l + 1; Shenoy-Kumaresan returns w
 * exactly when |w| <= B ((m_sk - 1)/2 - k).  Multiplied through by 2 m~^2 that is the test.  Every B of SEAL's rule
 * (|B| = l, or l + 1 when 32 + bits(t) + bits(Q) >= 61 (l + 1), 61-bit primes, and a 61-bit m_sk) passes it.
 * ct1 == ct2 (squaring) is allowed; the inputs are only read.  batch = 0 does nothing.  HEXL_B200_ERR_INVALID_ARG for a
 * null pointer, n not a power of two in [2, 2^20], l or k outside [1, 64], plain_modulus outside [2, 2^61), a modulus of
 * Q u Bsk that is >= 2^61, not NTT-friendly for n or not coprime to the others, result overlapping an input, and Bsk
 * failing the bound.  Inputs are checked below their modulus under hexl_b200_set_debug(1).  On the device, per pair: one
 * extension launch per input ciphertext (one when squaring) that reads the l limbs and writes all l + k + 1; one
 * forward transform of the four (two) lifted polynomials (ceil(4 (l + k + 1) / 64) launches); one DyadicMultiply
 * launch per block of 64 moduli; one inverse transform of the tensor (ceil(3 (l + k + 1) / 64) launches); and one
 * scaling launch that reads l + k + 1 limbs and writes l.  The kernels' constants live in a device table built and
 * uploaded on first use per (Q, B, m_sk, t) and device, so device calls capture into a CUDA graph once the call has
 * run once on that device and the transforms are warm.  Library scratch: 7 x (l + k + 1) x n words (5 when squaring).
 * Host buffers: both ciphertexts of a pair cross PCIe in once (one copy when squaring) and the product comes back on
 * the same staging stream, split by pair over the devices of hexl_b200_set_host_devices.  Managed buffers take the
 * device path.  Not covered: HPS or other floating-point scaling, BGV, inputs of more than two components, choosing B
 * or m_sk (the caller's context does), and an in-place variant. */
int hexl_b200_bfv_multiply(uint64_t* result, const uint64_t* ct1, const uint64_t* ct2, uint64_t n,
                           const uint64_t* moduli, uint64_t level_size, const uint64_t* base_b, uint64_t base_b_size,
                           uint64_t m_sk, uint64_t plain_modulus, uint64_t batch, void* stream);

/* BFV ciphertext multiplication relinearized with hybrid keys (extension; SEAL's multiply + relinearize for BFV): the
 * product of hexl_b200_bfv_multiply followed by the key switch of its d2.  The moduli, digits, key handle (one
 * relinearization key, s^2 -> s, key_component_count 2) and shape rules are those of
 * hexl_b200_multiply_relinearize_hybrid; Q is the first l = level_size data moduli and base_b, m_sk, plain_modulus are
 * the BEHZ bases and plain modulus of hexl_b200_bfv_multiply for that level.  Pair c reads ct1 + c*2*l*n and
 * ct2 + c*2*l*n (coefficient form, canonical) and its result is STORED at result + c*2*l*n, coefficient form,
 * canonical:
 *   (d0, d1, d2) = hexl_b200_bfv_multiply(ct1, ct2)
 *   result       = (d0, d1) + KS(d2)
 * with KS the switch of hexl_b200_key_switch_hybrid taken in coefficient form: the mod-up reads d2's limbs directly,
 * and the mod-down brings the data limbs of the products back to coefficients and adds (INTT(prod) - c) P^-1, c the
 * rounded conversion of the special limbs.  Every step is canonical and the NTT a bijection, so this is bit for bit the
 * chain hexl_b200_bfv_multiply; hexl_b200_ntt_forward_multi of d2; hexl_b200_key_switch_hybrid into a zeroed
 * two-component result; hexl_b200_ntt_inverse_multi; hexl_b200_eltwise_add_mod_multi with (d0, d1).  At digit_size = 1
 * with one special prime it is therefore SEAL's multiply + relinearize with hexl_b200_key_switch_resident.  It decrypts
 * under (1, s) to the product's message within the product's noise plus one key switch's.  HEXL_B200_ERR_INVALID_ARG
 * on the refusals of hexl_b200_multiply_relinearize_hybrid (rescale aside) and of hexl_b200_bfv_multiply.  ct1 == ct2
 * squares; batch = 0 does nothing.  On the device, per pair: the launches of hexl_b200_bfv_multiply, then those of
 * hexl_b200_key_switch_hybrid with kcc = 2 less its first inverse transform, and in the mod-down an inverse transform
 * of the products' data limbs in place of the forward transform of the correction.  Library scratch: that of
 * hexl_b200_bfv_multiply plus l x n words of d2, one round of converted digits and (l + p_size) x 2 x n words of
 * products.  Device calls capture into a CUDA graph once the call has run once on that device.  Host buffers: as for
 * hexl_b200_bfv_multiply, split by pair over the devices where the handle holds a copy.  Not covered: keys sharded by
 * modulus (refused), a relinearize-only call for three-component coefficient-form ciphertexts, BFV rotations, and an
 * in-place variant. */
int hexl_b200_bfv_multiply_relinearize_hybrid(uint64_t* result, const uint64_t* ct1, const uint64_t* ct2, uint64_t n,
                                              uint64_t level_size, uint64_t q_size, uint64_t p_size,
                                              uint64_t digit_size, const uint64_t* moduli, const uint64_t* base_b,
                                              uint64_t base_b_size, uint64_t m_sk, uint64_t plain_modulus,
                                              const hexl_b200_keys* relin_keys, uint64_t batch, void* stream);

/* ---------------------------------------------------------------------------------------------------------- BGV
 * BGV keeps the message mod the plain modulus tau = plain_modulus (SEAL's t) in the low part of the phase, so every
 * division by a modulus product P_T must subtract a correction delta with delta = 0 (mod tau); the rounded correction of
 * the CKKS calls is not, and its error, not a multiple of tau, destroys the message.  The calls below replace it by the
 * t-corrected mod-down.  T is the set of moduli dropped, P_T = prod T, and x_t (t in T) the T-limbs in coefficient form,
 * canonical (an inverse transform of them in NTT form):
 *   y_t   = [x_t (P_T/t)^-1]_t                                                   (no rounding offset)
 *   X~_m  = [ sum_t y_t [P_T/t]_m ]_m   for m in {q_i : i < l'} and m = tau       (one integer X~ = X + u P_T, 0 <= u < |T|)
 *   k     = [ -X~_tau P_T^-1 ]_tau
 *   delta_i = [ X~_i + [P_T]_{q_i} k ]_{q_i}
 *   out_i = (ext_i - NTT_{q_i}(delta_i)) P_T^-1 mod q_i  (NTT form)   or   (ext_i - delta_i) P_T^-1 mod q_i  (coefficients)
 * The integer delta = X~ + P_T k satisfies delta = X (mod P_T), delta = 0 (mod tau) and 0 <= delta < P_T (|T| + tau - 1),
 * so out is exactly (X_ext - delta) / P_T, and the message mod tau is multiplied by [P_T^-1]_tau.  With T one prime p the
 * conversion returns x itself (u = 0): k = [-x p^-1]_tau and delta = x + p k, SEAL's formula
 * (RNSTool::mod_t_and_divide_q_last_ntt_inplace and the BGV branch of Evaluator::switch_key_inplace), so digit_size = 1
 * with one special prime is SEAL's BGV relinearization and rotation bit for bit.  OpenFHE's BGV takes
 * delta = tau FBC([x tau^-1]_P) instead: its results differ from these bit for bit, with the same noise bound.
 * Exactness, for every modulus below 2^61, every tau in [2, 2^61) and |T| <= 64: each sum of |T| products
 * y_t [P_T/t]_m < (2^61 - 1)^2 is below 64 (2^61 - 1)^2 < 2^128 and is reduced once; k [P_T]_{q_i} is added after that
 * reduction (a Shoup product, exact for any 64-bit k, and one conditional subtraction), never as a 65th term of the
 * 128-bit sum, which could then exceed 2^128.  The constants travel in the kernel parameters: one conversion launch
 * takes at most floor((474 - 4 |T|) / (6 + |T|)) targets (67 for |T| = 1, 27 for 10, 3 for 64), where the rounded
 * conversion of the CKKS calls takes floor((480 - 4 |T|) / (5 + |T|)); device calls capture into CUDA graphs.
 * Every BGV call refuses (HEXL_B200_ERR_INVALID_ARG) plain_modulus outside [2, 2^61) and plain_modulus sharing a factor
 * with any modulus it is given, on top of the refusals of its CKKS counterpart.  The caller tracks the correction
 * factor [P_T^-1]_tau, as SEAL does.  Not covered: BGV forms of the linear transforms, the inner sum and the lazy
 * relinearization, the SEAL-shaped KeySwitch, sharded key handles (refused), key generation, encoding, encryption and
 * decryption. */

/* BGV modulus switch by the last modulus (extension; SEAL's RNSTool::mod_t_and_divide_q_last_inplace and
 * mod_t_and_divide_q_last_ntt_inplace, OpenFHE's BGV ModReduce): the layout, forms, in-place rule and refusals of
 * hexl_b200_divide_and_round_q_last, with the rounding replaced by the t-correction of T = {q_L}: limbs 0..L-1 of every
 * polynomial get (X - delta) / q_L mod q_i, canonical, delta = x_L + q_L [-x_L q_L^-1]_tau with x_L the last limb in
 * coefficient form; limb L is not written.  The message mod tau is multiplied by [q_L^-1]_tau.  In NTT form this is bit
 * for bit the inverse transform, the coefficient-form call and the forward transform.  On the device, per chunk of
 * polynomials (~256 MiB of scratch): in NTT form one gathering copy and one inverse transform of the last limbs; then per
 * block of 64 moduli one conversion launch, in NTT form one forward transform of delta, and one finish launch. */
int hexl_b200_bgv_mod_switch(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                             uint64_t rns_modulus_size, uint64_t plain_modulus, uint64_t count, int ntt_form,
                             void* stream);

/* BGV hybrid key switch (extension; SEAL's Evaluator::switch_key_inplace for BGV with OpenFHE's hybrid digits): the
 * arguments, layouts, definitions and launches of hexl_b200_key_switch_hybrid, with ModDown_P the t-corrected mod-down
 * (T = {p_0..p_{K-1}}) in place of the rounded one; its conversion launches are per block of base_conv_t targets.  It
 * is BGV's relinearization of a three-component ciphertext (d2 into (d0, d1), key_component_count = 2) and, after
 * hexl_b200_apply_galois, the non-hoisted rotation.  Refusals: those of hexl_b200_key_switch_hybrid and the BGV ones. */
int hexl_b200_bgv_key_switch_hybrid(uint64_t* result, const uint64_t* target, uint64_t n, uint64_t level_size,
                                    uint64_t q_size, uint64_t p_size, uint64_t digit_size,
                                    uint64_t key_component_count, const uint64_t* moduli, uint64_t plain_modulus,
                                    const hexl_b200_keys* keys, uint64_t batch, void* stream);

/* BGV hoisted rotations with hybrid keys (extension; SEAL's rotate_rows / rotate_columns for several elements with one
 * mod-up): hexl_b200_apply_galois_key_switch_hybrid_hoisted with the t-corrected ModDown_P:
 *   out_r = [sigma_g(c0), 0] + ModDown^tau_P(prod^r).
 * For g = 1 it is hexl_b200_bgv_key_switch_hybrid of c1 into (c0, 0) bit for bit.  Arguments, layouts, launches,
 * scratch, host staging and refusals as for the CKKS call, plus the BGV refusals. */
int hexl_b200_bgv_apply_galois_key_switch_hybrid_hoisted(uint64_t* results, const uint64_t* ciphertexts, uint64_t n,
                                                         uint64_t level_size, uint64_t q_size, uint64_t p_size,
                                                         uint64_t digit_size, const uint64_t* moduli,
                                                         uint64_t plain_modulus,
                                                         const hexl_b200_keys* const* galois_keys,
                                                         const uint64_t* galois_elts, uint64_t num_elts,
                                                         uint64_t batch, void* stream);

/* BGV ciphertext multiplication with relinearization by hybrid keys (extension; SEAL's multiply + relinearize
 * [+ mod_switch_to_next] for BGV), optionally modulus-switched in the same mod-down: hexl_b200_multiply_relinearize_hybrid
 * with the t-corrected mod-down, mod_switch in the place of rescale.  With the tensor d, prod and ext of that call:
 *   T = {p_0..p_{K-1}} (mod_switch = 0) or {q_{l-1}, p_0..p_{K-1}} (mod_switch = 1),  result = ModDown^tau_T(ext), stored,
 * l' = l - mod_switch limbs.  mod_switch = 0 is bit for bit hexl_b200_dyadic_multiply followed by
 * hexl_b200_bgv_key_switch_hybrid of d2 into (d0, d1) (delta depends only on the limbs of T, where ext = prod, and
 * (prod + P d - delta) P^-1 = (prod - delta) P^-1 + d).  mod_switch = 1 drops q_{l-1} in the same mod-down as P, with one
 * t-correction instead of the two of that chain followed by hexl_b200_bgv_mod_switch, so it is NOT the chain bit for bit;
 * the message picks up [(q_{l-1})^-1]_tau and the key switch's error is divided by q_{l-1}.  Launches, scratch, host
 * staging and squaring as for the CKKS call; refusals as for it (mod_switch other than 0 or 1, mod_switch = 1 with
 * level_size < 2 or p_size > 63) plus the BGV ones. */
int hexl_b200_bgv_multiply_relinearize_hybrid(uint64_t* result, const uint64_t* ct1, const uint64_t* ct2, uint64_t n,
                                              uint64_t level_size, uint64_t q_size, uint64_t p_size,
                                              uint64_t digit_size, const uint64_t* moduli, uint64_t plain_modulus,
                                              const hexl_b200_keys* relin_keys, int mod_switch, uint64_t batch,
                                              void* stream);

/* The lift of BFV / BGV plaintexts into the RNS basis of a ciphertext (extension; SEAL's transform_to_ntt_inplace
 * (Plaintext&, parms_id) and the lift inside BFV and BGV multiply_plain and BGV add_plain).  Plaintext p is
 * plain_coeff_count = pcc words at plain + p*pcc, coefficients mod t = plain_modulus (SEAL's Plaintext buffer, its
 * coeff_count(); the coefficients from pcc to n are zero), and its lift is STORED at result + p*l*n, l = level_size
 * limbs of n words.  With c = correction_factor, per coefficient m and limb i:
 *   m' = [m c]_t,   out_i = [m' - t]_{q_i} if m' >= floor((t + 1) / 2), else [m']_{q_i}
 * (the centred lift of m'; c = 1 is no correction, BGV's add_plain passes its correction factor).  Exact for every order
 * of t and the q_i (t may exceed some q_i).  ntt_form = 1 then applies the forward transform (hexl_b200_ntt_forward_multi,
 * canonical output) to every limb: the plaintext operand of BGV's add_plain / multiply_plain and of
 * hexl_b200_bfv_multiply_plain(plain_ntt_form = 1).  Moduli below 2^61 (NTT-friendly for n when ntt_form = 1), t in
 * [2, 2^61), l in [1, 64].  count = 0 does nothing.  HEXL_B200_ERR_INVALID_ARG for a null pointer, n not a power of two
 * in [2, 2^20], l outside [1, 64], t outside [2, 2^61), correction_factor outside [1, t), pcc outside [1, n], ntt_form
 * other than 0 or 1, a modulus outside [2, 2^61) (or not NTT-friendly with ntt_form = 1), and result overlapping plain;
 * plaintext words >= t under hexl_b200_set_debug(1).  On the device: one launch for all count plaintexts (a thread per
 * coefficient slot looping over the limbs), then with ntt_form = 1 the forward transform of the count x l limbs
 * (ceil(count l / 64) transform launches); no library scratch.  Device calls capture into a CUDA graph once the
 * transforms are warm.  Host buffers: one plaintext per staging step, split by plaintext over the devices of
 * hexl_b200_set_host_devices.  Not covered: in place (the lift grows each plaintext from pcc to l x n words), encoding
 * (the caller's BatchEncoder produced the plaintext), CKKS plaintexts (already in RNS form). */
int hexl_b200_plain_lift(uint64_t* result, const uint64_t* plain, uint64_t plain_coeff_count, uint64_t n,
                         const uint64_t* moduli, uint64_t level_size, uint64_t plain_modulus,
                         uint64_t correction_factor, int ntt_form, uint64_t count, void* stream);

/* BFV add_plain / sub_plain (extension; SEAL's Evaluator::add_plain / sub_plain for BFV,
 * multiply_add_plain_with_scaling_variant / multiply_sub_plain_with_scaling_variant): c0 +- round(Q m / t) for each of
 * `batch` ciphertexts.  Q = q_0..q_{l-1} (moduli, l = level_size: the ciphertext's level), t = plain_modulus.
 * Ciphertext c is two components of l limbs of n words at ct + c*2*l*n, COEFFICIENT form, canonical; its plaintext is
 * plain_coeff_count = pcc words at plain (plain_count = 1: one plaintext for every ciphertext) or at plain + c*pcc
 * (plain_count = batch), coefficients below t, the coefficients from pcc to n zero.  Per coefficient j < pcc and limb i,
 * with r = Q mod t and h = floor((t + 1) / 2):
 *   fix = floor((m_j r + h) / t),   s = [m_j [floor(Q/t)]_{q_i} + fix]_{q_i},   c0_i[j] = [c0_i[j] +- s]_{q_i}
 * (- with subtract = 1); m floor(Q/t) + fix = floor((Q m + h) / t), so this is SEAL's formula bit for bit.  The result
 * is STORED at result + c*2*l*n: result == ct (SEAL's in-place operation) changes only those pcc slots of c0; any other
 * result gets c0 in full and a copy of c1.  A result overlapping ct without being equal to it is refused.  fix is
 * computed without a 128-bit division: a Shoup quotient of m r by t, corrected by at most one, plus [rem + h >= t]
 * (plain.cu states the proof).  Moduli below 2^61 (any, not only NTT-friendly), t in [2, 2^61), l in [1, 64].
 * batch = 0 does nothing.  HEXL_B200_ERR_INVALID_ARG for a null pointer, n not a power of two in [2, 2^20], l outside
 * [1, 64], t outside [2, 2^61), pcc outside [1, n], plain_count other than 1 or batch, subtract other than 0 or 1, a
 * modulus outside [2, 2^61), result partly overlapping ct, and result overlapping plain; ciphertext words >= their
 * modulus and plaintext words >= t under hexl_b200_set_debug(1).  On the device: one launch for the whole batch (a
 * thread per coefficient slot, fix computed once and applied to the l limbs), plus one device-to-device copy of the c1
 * components when result != ct.  The constants (per limb q_i, floor(2^64 / q_i), [floor(Q/t)]_{q_i} and its Shoup
 * factor; r, floor(r 2^64 / t), h) live in a device table built and uploaded on first use per (Q, t) and device, so a
 * device call captures into a CUDA graph once it has run once on that device.  No library scratch.  Host buffers: one
 * ciphertext per staging step (in and out on the same stream), a broadcast plaintext uploaded once per device, split by
 * ciphertext over the devices of hexl_b200_set_host_devices.  Not covered: NTT-form BFV ciphertexts (SEAL refuses them
 * too), BGV and CKKS add_plain (hexl_b200_plain_lift with the correction factor, then hexl_b200_eltwise_add_mod_multi
 * on c0; CKKS plaintexts are already RNS), and sums of several plaintexts in one pass. */
int hexl_b200_bfv_add_plain(uint64_t* result, const uint64_t* ct, const uint64_t* plain, uint64_t plain_coeff_count,
                            uint64_t plain_count, uint64_t n, const uint64_t* moduli, uint64_t level_size,
                            uint64_t plain_modulus, int subtract, uint64_t batch, void* stream);

/* BFV multiply_plain (extension; SEAL's Evaluator::multiply_plain for BFV, multiply_plain_normal): each of `batch`
 * coefficient-form ciphertexts times a plaintext, the product in coefficient form.  Layouts, Q, t, pcc and plain_count
 * as for hexl_b200_bfv_add_plain.  Per component k and limb i, negacyclic products mod q_i:
 *   result_k,i = INTT(NTT(ct_k,i) . NTT(lift(m)_i)),   lift that of hexl_b200_plain_lift with correction factor 1,
 * canonical.  plain_ntt_form = 1 takes plaintexts that hexl_b200_plain_lift(ntt_form = 1) produced instead: l x n words
 * each at plain (+ c*l*n), canonical; pcc is then not read (a PIR server transforms its database once).  result may
 * equal ct; partial overlap is refused.  Bit for bit the chain hexl_b200_plain_lift(ntt_form = 1);
 * hexl_b200_ntt_forward_multi of ct; hexl_b200_eltwise_mult_mod_multi of each component by the lifted plaintext;
 * hexl_b200_ntt_inverse_multi.  Moduli below 2^61 and NTT-friendly for n; otherwise the refusals of
 * hexl_b200_bfv_add_plain (subtract aside) and plain_ntt_form other than 0 or 1; plaintext words (NTT form: >= q_i)
 * refused under hexl_b200_set_debug(1) like the ciphertext's.  On the device: each coefficient-form plaintext is lifted
 * and transformed once (one lift launch and ceil(l / 64) forward transform launches; once per call when broadcast);
 * per ciphertext, one forward transform of its two components into result (ceil(2l / 64) launches) and one inverse
 * transform per component that multiplies by the transformed plaintext on load (2 ceil(l / 64) launches): there is no
 * separate product pass, and the product never makes a round trip through HBM.  Library scratch: l x n words (none with
 * plain_ntt_form = 1).  Device calls capture into a CUDA graph once the transforms are warm.  Host buffers: one
 * ciphertext per staging step; a broadcast plaintext is uploaded, lifted and transformed once per device.  Not covered:
 * NTT-form BFV ciphertexts, plaintext-weighted sums sum_i pt_i . ct_i in one pass, SEAL's fast path for monomial
 * plaintexts (the same result), and BGV (hexl_b200_plain_lift(ntt_form = 1), then hexl_b200_eltwise_mult_mod_multi on
 * both components). */
int hexl_b200_bfv_multiply_plain(uint64_t* result, const uint64_t* ct, const uint64_t* plain,
                                 uint64_t plain_coeff_count, uint64_t plain_count, int plain_ntt_form, uint64_t n,
                                 const uint64_t* moduli, uint64_t level_size, uint64_t plain_modulus, uint64_t batch,
                                 void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HEXL_B200_H */
