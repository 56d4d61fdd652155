// KeySwitch and its mod-down: on device pointers, as a batch on host pointers, and sharded by RNS modulus over several
// GPUs; the key handles; and the rescale by the last modulus (DivideAndRoundQLast), which shares the mod-down.
#include <cstdlib>
#include <numeric>

#include "capi.h"

using namespace hexl_b200;

namespace hexl_b200 {

// RNS modulus i of a key switch lives in slot key_slot(i) of the key / moduli arrays (key-switch-internal.cpp:62-63);
// the slots between decomp and the special prime are not touched by the switch
static uint64_t key_slot(uint64_t i, uint64_t decomp, uint64_t key_modulus_size) {
  return i == decomp ? key_modulus_size - 1 : i;
}

// The cached transforms of the decomp + 1 RNS moduli of a key switch, h[i] for RNS index i
static int key_switch_ntts(CachedNtts& h, uint64_t n, const uint64_t* moduli, uint64_t decomp,
                           uint64_t key_modulus_size) {
  for (uint64_t i = 0; i <= decomp; ++i) {
    const uint64_t slot = key_slot(i, decomp, key_modulus_size);
    // lazy sums of the glue kernels (v < 4q in the MAC, < 8q in the final step) need 8q < 2^64
    if (moduli[slot] >= (1ull << 61))
      return fail(HEXL_B200_ERR_INVALID_ARG, "KeySwitch: Require moduli < 2^61 (slot %llu)", (unsigned long long)slot);
    if (int rc = h.load(i, n, moduli[slot])) return rc;
  }
  return 0;
}

// Digits one ks_mac_kernel launch may add up for the `count` moduli of `mods`.  Each product is a lazy forward-transform
// output (< 4q) times a key word (< q) and the kernel sums them unreduced in 128 bits, so at most
// (2^128 - 1) / ((4q - 1)(q - 1)) of them fit for the largest q: the whole 64-entry key block below 2^60, down to 16
// just below 2^61.  Launches beyond the first add their reduced sums into prod (the `accumulate` flag).
uint64_t ks_mac_digits_per_launch(const KsModuli& mods, uint64_t count) {
  uint64_t q = 0;
  for (uint64_t e = 0; e < count; ++e) q = std::max(q, mods.m[e].q);
  const unsigned __int128 largest_product = (unsigned __int128)(4 * q - 1) * (q - 1);
  return (uint64_t)std::min<unsigned __int128>(kParamBlock, ~(unsigned __int128)0 / largest_product);
}

// One round of step 2 of the key switch (key-switch-internal.cpp:60-131) for `cnt` <= kParamBlock RNS moduli, hs[e]
// their transforms and slots[e] their slots in keys of kms slots: every digit of t_coef (decomp x n words,
// coefficient form) reduced into each modulus and lazily forward-transformed into ops ([e][j][n]), then multiplied
// with the keys of each of `elts` switches and accumulated into prod + r * prod_stride ([e][k][n]).  keys[r][j] is
// digit j's key of switch r; galois_elts[r] (nullptr: none) makes switch r read the digits permuted by pi_g.
static int ks_mac_round(int dev, hexl_b200_ntt* const* hs, const uint64_t* slots, uint64_t cnt, uint64_t kms,
                        uint64_t* ops, const uint64_t* t_coef, uint64_t decomp, uint64_t n, uint64_t kcc, uint64_t* prod,
                        uint64_t prod_stride, const uint64_t* const* const* keys, const uint64_t* galois_elts,
                        uint64_t elts, cudaStream_t s) {
  // every digit into every modulus of the round (:77-85) happens inside the transform: it reads the digits from
  // t_coef (L2-resident) and reduces on load, instead of a reduce kernel writing decomp x cnt x n words for it
  if (int rc = ntt_multi_on_device(true, dev, hs, cnt, ops, t_coef, 4, decomp, s, nullptr, true)) return rc;
  return ks_mac_products(hs, slots, cnt, kms, ops, decomp, n, kcc, prod, prod_stride, keys, galois_elts, elts, s);
}

KsModuli ks_mac_moduli(const uint64_t* moduli, const uint64_t* slots, uint64_t cnt) {
  KsModuli mods;
  for (uint64_t e = 0; e < cnt; ++e) {
    const uint64_t q = moduli[e], mu = nt::multiply_factor(1, 64, q);
    const uint64_t r64 = mu * (0 - q);  // 2^64 - floor(2^64/q)*q = 2^64 mod q
    const Twiddle R = make_twiddle(r64 % q, q);
    mods.m[e] = KsModulus{q, mu, R.w, R.wp, slots ? slots[e] : 0};
  }
  return mods;
}

int ks_mac_products(hexl_b200_ntt* const* hs, const uint64_t* slots, uint64_t cnt, uint64_t kms, const uint64_t* ops,
                    uint64_t decomp, uint64_t n, uint64_t kcc, uint64_t* prod, uint64_t prod_stride,
                    const uint64_t* const* const* keys, const uint64_t* galois_elts, uint64_t elts, cudaStream_t s,
                    bool accumulate) {
  uint64_t q[kParamBlock];
  for (uint64_t e = 0; e < cnt; ++e) q[e] = hs[e]->q;
  const KsModuli mods = ks_mac_moduli(q, slots, cnt);
  const uint64_t per_mod = decomp * n, jmax = ks_mac_digits_per_launch(mods, cnt);
  for (uint64_t r = 0; r < elts; ++r)
    for (uint64_t j0 = 0; j0 < decomp; j0 += jmax) {  // key pointers ride in the kernel parameters
      const uint64_t jc = std::min<uint64_t>(jmax, decomp - j0);
      KeyPointers kp;
      for (uint64_t j = 0; j < jc; ++j) kp.p[j] = keys[r][j0 + j];
      const cudaError_t e = launch_ks_mac(prod + r * prod_stride, ops + j0 * n, per_mod, kp, n, jc, kcc, kms, cnt,
                                          mods, accumulate || j0 != 0, s, galois_elts ? galois_elts[r] : 0);
      if (e != cudaSuccess) return cuda_fail(e, "KeySwitch: multiply-accumulate launch");
    }
  return 0;
}

// The blocks of the mod-down by q_last: for each block of at most kParamBlock target moduli i (h_targets[i],
// target_moduli[i], factors[i] = q_last^-1 mod q_i), ks_round of t_last ([p][n], coefficient form) into tmp ([e][p][n],
// room for one block), one lazy multi-modulus forward transform of tmp, and
// ks_finish: result[n (res_stride p + i) + l] (+)= (in - tmp) * factors[i] mod q_i.
// `in`, in_like_result and accumulate are those of launch_ks_finish (modulus-major `in` starts at target 0).
static int mod_down_blocks(int dev, uint64_t* result, uint64_t res_stride, const uint64_t* in, bool in_like_result,
                           bool accumulate, const uint64_t* t_last, uint64_t* tmp, uint64_t n, uint64_t group,
                           uint64_t q_last, hexl_b200_ntt* const* h_targets, const uint64_t* target_moduli,
                           const uint64_t* factors, uint64_t targets, cudaStream_t s) {
  const uint64_t mu_last = nt::multiply_factor(1, 64, q_last);
  for (uint64_t i0 = 0; i0 < targets; i0 += kParamBlock) {
    const uint64_t cnt = std::min<uint64_t>(kParamBlock, targets - i0);
    KsModuli round_mods, fin_mods;
    for (uint64_t e = 0; e < cnt; ++e) {
      const uint64_t qi = target_moduli[i0 + e], mu_i = nt::multiply_factor(1, 64, qi);
      round_mods.m[e] = KsModulus{qi, mu_i, qi - ((q_last >> 1) % qi), 0, 0};
      const Twiddle ms = make_twiddle(factors[i0 + e] % qi, qi);
      fin_mods.m[e] = KsModulus{qi, mu_i, ms.w, ms.wp, 0};
    }
    cudaError_t e = launch_ks_round(tmp, t_last, n, group, q_last, mu_last, cnt, round_mods, s);
    if (e != cudaSuccess) return cuda_fail(e, "mod-down: round launch");
    if (int rc = ntt_multi_on_device(true, dev, h_targets + i0, cnt, tmp, tmp, 4, group, s)) return rc;
    e = launch_ks_finish(result, in_like_result ? in : in + i0 * group * n, tmp, n, group, res_stride, i0, cnt,
                         fin_mods, in_like_result, accumulate, s);
    if (e != cudaSuccess) return cuda_fail(e, "mod-down: finish launch");
  }
  return 0;
}

// Mod-down of `group` polynomials by their last modulus q_last = h_last->q, every step batched over the target moduli
// (key-switch-internal.cpp:134-198; SEAL's divide_and_round_q_last_ntt_inplace): t_last, the polynomials' last part in
// NTT form ([p][n] contiguous, < 2 q_last), is inverse-transformed in place, then mod_down_blocks.  About 1 + 3
// launches per block, whatever `group` is.  Device pointers on the current device, asynchronous on s.
static int mod_down_on_device(int dev, uint64_t* result, uint64_t res_stride, const uint64_t* in, bool in_like_result,
                              bool accumulate, uint64_t* t_last, uint64_t* tmp, uint64_t n, uint64_t group,
                              hexl_b200_ntt* h_last, hexl_b200_ntt* const* h_targets, const uint64_t* target_moduli,
                              const uint64_t* factors, uint64_t targets, cudaStream_t s) {
  NttDeviceTables tl;
  if (int rc = device_tables(h_last, dev, &tl, s)) return rc;
  const cudaError_t e = launch_ntt_inverse(tl, t_last, t_last, 2, 2, group, s);
  if (e != cudaSuccess) return cuda_fail(e, "mod-down: inverse NTT launch");
  return mod_down_blocks(dev, result, res_stride, in, in_like_result, accumulate, t_last, tmp, n, group, h_last->q,
                         h_targets, target_moduli, factors, targets, s);
}

// key-switch-internal.cpp:25-201 as a short chain of launches on the caller's stream, every
// step batched over the RNS moduli (multi-modulus NTTs + the glue kernels of seal.cu): about a
// dozen launches whatever the number of moduli, instead of ~10 per modulus.  Every pointer is
// a device pointer on the current device.  Scratch layouts are [modulus][digit or component][n].
// `elts` switches share the digits t_target, decomposed once (steps 1 and 2's transforms): switch r multiplies them
// with the keys d_key_ptrs[r] and accumulates into results[r].  galois_elts (the hoisted rotations; nullptr: none)
// makes switch r read the transformed digits permuted by pi_{galois_elts[r]}.  Scratch: one round of transformed
// digits plus elts x rns x kcc x n words of products.
int key_switch_elts_on_device(int dev, uint64_t* const* results, const uint64_t* t_target, uint64_t n,
                              uint64_t decomp, uint64_t key_modulus_size, uint64_t rns, uint64_t kcc,
                              const uint64_t* moduli, const uint64_t* const* const* d_key_ptrs,
                              const uint64_t* galois_elts, uint64_t elts, const uint64_t* modswitch,
                              cudaStream_t s) {
  CachedNtts h(rns);
  if (int rc = key_switch_ntts(h, n, moduli, decomp, key_modulus_size)) return rc;
  // moduli handled per round of step 2: bounded by the parameter block and by ~256 MiB of scratch
  const uint64_t per_mod = decomp * n;
  uint64_t ichunk = std::max<uint64_t>(1, (256ull << 20) / (per_mod * 8));
  ichunk = std::min<uint64_t>({ichunk, rns, (uint64_t)kParamBlock});
  Scratch ws(s);
  uint64_t *t_coef = nullptr, *ops = nullptr, *prod = nullptr, *tmp = nullptr;
  if (int rc = ws.get(&t_coef, per_mod)) return rc;
  if (int rc = ws.get(&ops, ichunk * per_mod)) return rc;
  if (int rc = ws.get(&prod, elts * rns * kcc * n)) return rc;                                // [r][i][k][n]
  if (int rc = ws.get(&tmp, std::min<uint64_t>(decomp, kParamBlock) * kcc * n)) return rc;  // [i][k][n], one block
  // 1. digits back to coefficient form, each under its own modulus (:49-55)
  if (int rc = ntt_multi_on_device(false, dev, h.data(), decomp, t_coef, t_target, 1, 1, s)) return rc;
  // 2. every digit under every modulus: reduce, lazy forward NTT, multiply-accumulate with the keys (:60-131).
  //    (The digit that already lives in modulus i is re-derived like the others: NTT(INTT(x)) = x mod q_i.)
  for (uint64_t i0 = 0; i0 < rns; i0 += ichunk) {
    const uint64_t cnt = std::min(ichunk, rns - i0);
    uint64_t slots[kParamBlock];
    for (uint64_t e = 0; e < cnt; ++e) slots[e] = key_slot(i0 + e, decomp, key_modulus_size);
    if (int rc = ks_mac_round(dev, h.data() + i0, slots, cnt, key_modulus_size, ops, t_coef, decomp, n, kcc,
                              prod + i0 * kcc * n, rns * kcc * n, d_key_ptrs, galois_elts, elts, s))
      return rc;
  }
  // 3. mod-down by the special prime and accumulate into result (:134-198); prod's last part is [k][n], contiguous
  for (uint64_t r = 0; r < elts; ++r) {
    uint64_t* prod_r = prod + r * rns * kcc * n;
    if (int rc = mod_down_on_device(dev, results[r], decomp, prod_r, false, true, prod_r + decomp * kcc * n, tmp, n,
                                    kcc, h[decomp], h.data(), moduli, modswitch, decomp, s))
      return rc;
  }
  return 0;  // asynchronous on s; ~Scratch returns the buffers to the pool in stream order
}

int key_switch_on_device(int dev, uint64_t* result, const uint64_t* t_target, uint64_t n, uint64_t decomp,
                         uint64_t key_modulus_size, uint64_t rns, uint64_t kcc, const uint64_t* moduli,
                         const uint64_t* const* d_key_ptrs_host, const uint64_t* modswitch, cudaStream_t s) {
  return key_switch_elts_on_device(dev, &result, t_target, n, decomp, key_modulus_size, rns, kcc, moduli,
                                   &d_key_ptrs_host, nullptr, 1, modswitch, s);
}

bool keys_fit(const hexl_b200_keys* k, uint64_t n, uint64_t decomp, uint64_t kcc, uint64_t key_modulus_size) {
  return k->n == n && k->decomp >= decomp && k->kcc == kcc && k->kms == key_modulus_size;
}

uint64_t keys_on_device(const hexl_b200_keys* const* keys, uint64_t count, int dev,
                        std::vector<const uint64_t* const*>* dk) {
  dk->assign(count, nullptr);
  for (uint64_t r = 0; r < count; ++r) {
    auto it = keys[r]->dev.find(dev);
    if (it == keys[r]->dev.end()) return r;
    (*dk)[r] = it->second.data();
  }
  return count;
}

// One or more key switches on HOST buffers against keys already on the devices, one ciphertext per staging chunk
// (stage_items), split by ciphertext over the host devices holding every key.  Ciphertext c's result block
// (res_words words at result + c * res_words, in the slot's buffer 0) crosses PCIe out, and in as well when
// result_in; in_words words of `in` (in + c * in_words; nothing when in is null) go into the slot's buffer 1, which
// holds buf_words words, followed by in_words words of in2 (in2 + c * in_words) when in2 is not null.
int key_switch_host_batch(uint64_t* result, uint64_t res_words, bool result_in, const uint64_t* in,
                          uint64_t in_words, uint64_t buf_words, const hexl_b200_keys* const* keys,
                          uint64_t num_keys, uint64_t batch, const HostSwitch& run,
                          const std::function<int(int)>& prepare, const uint64_t* in2) {
  std::vector<int> devs;
  if (int rc = host_devices(&devs)) return rc;
  std::vector<const uint64_t* const*> dk;
  std::vector<int> use;
  for (int d : devs)
    if (keys_on_device(keys, num_keys, d, &dk) == num_keys) use.push_back(d);
  if (use.empty()) return fail(HEXL_B200_ERR_INVALID_ARG, "the key handle holds no copy on the device(s) used for host calls");
  return stage_items(use, batch, 1, [&](int dev, u64, u64, auto&& stage) {
    keys_on_device(keys, num_keys, dev, &dk);
    if (prepare)
      if (int rc = prepare(dev)) return rc;
    return stage([&](const StageSlot& sl, u64 c, u64) -> int {
      if (int rc = sl.reserve(0, res_words * 8)) return rc;
      if (int rc = sl.reserve(1, buf_words * 8)) return rc;
      cudaStream_t sx = sl.stream();
      u64 *d_res = sl.buf(0), *d_in = sl.buf(1);
      cudaError_t e = cudaSuccess;
      if (in) e = cudaMemcpyAsync(d_in, in + c * in_words, in_words * 8, cudaMemcpyHostToDevice, sx);
      if (e == cudaSuccess && in2)
        e = cudaMemcpyAsync(d_in + in_words, in2 + c * in_words, in_words * 8, cudaMemcpyHostToDevice, sx);
      if (e == cudaSuccess && result_in)
        e = cudaMemcpyAsync(d_res, result + c * res_words, res_words * 8, cudaMemcpyHostToDevice, sx);
      if (e != cudaSuccess) return cuda_fail(e, "KeySwitch H2D");
      if (int rc = run(dev, d_res, d_in, dk.data(), sx)) return rc;
      e = cudaMemcpyAsync(result + c * res_words, d_res, res_words * 8, cudaMemcpyDeviceToHost, sx);
      return e == cudaSuccess ? 0 : cuda_fail(e, "KeySwitch D2H");
    });
  });
}

int key_switch_check(const void* result, const void* t_target, uint64_t n, uint64_t decomp,
                     uint64_t key_modulus_size, uint64_t rns, uint64_t kcc, const uint64_t* moduli,
                     const uint64_t* modswitch) {
  REQUIRE(result && t_target && moduli && modswitch, "Require non-null arguments");
  REQUIRE(n >= 2 && !(n & (n - 1)), "Require n a power of two");
  REQUIRE(decomp >= 1 && kcc >= 1, "Require decomp_modulus_size, key_component_count >= 1");
  REQUIRE(rns == decomp + 1, "Require rns_modulus_size == decomp_modulus_size + 1");
  REQUIRE(key_modulus_size >= rns, "Require key_modulus_size >= rns_modulus_size");
  return 0;
}

// KeySwitch of a host batch: ciphertext c's digits (decomp x n words) in, its result (kcc x decomp x n) in and out
static int key_switch_host(uint64_t* result, const uint64_t* t_target, uint64_t n, uint64_t decomp,
                           uint64_t key_modulus_size, uint64_t rns, uint64_t kcc, const uint64_t* moduli,
                           const hexl_b200_keys* keys, const uint64_t* modswitch, uint64_t batch) {
  return key_switch_host_batch(result, kcc * decomp * n, true, t_target, decomp * n, decomp * n, &keys, 1, batch,
                               [&](int dev, uint64_t* d_res, uint64_t* d_t, const uint64_t* const* const* dk,
                                   cudaStream_t s) {
                                 return key_switch_on_device(dev, d_res, d_t, n, decomp, key_modulus_size, rns, kcc,
                                                             moduli, dk[0], modswitch, s);
                               });
}

// ---------------------------------------------------------------- one key switch sharded by RNS modulus
// The reference's loop nest (key-switch-internal.cpp:60-131) makes every output modulus consume every decomposed digit:
// with the moduli of ONE switch spread over several GPUs that is an all-gather of the digits in coefficient form
// (decomp x n words) -- the only exchange on this path (SURVEY 8(e)) -- plus a broadcast of the special prime's part
// (kcc x n words) before the final step (:134-198).  Both ride NVLink as peer copies issued from the producing shard's
// stream right behind the kernel that produced the data; consumers wait on an event, never on the host.
//   shard s, moduli [lo, hi):   H2D its digits + its slices of result
//     A  inverse NTT of its digits                       -> its rows of t_coef on EVERY shard        (all-gather)
//     B  every digit reduced into its moduli, lazy forward NTTs, multiply-accumulate with ITS key slices -> prod
//     C  (owner of the special prime) inverse NTT of that part -> t_last on every shard               (broadcast)
//     D  round, forward NTT, mod-switch, accumulate into its slices of result; D2H
static int key_switch_sharded(uint64_t* result, const uint64_t* t_target, uint64_t n, uint64_t decomp,
                              uint64_t key_modulus_size, uint64_t rns, uint64_t kcc, const uint64_t* moduli,
                              hexl_b200_keys* keys, const uint64_t* modswitch) {
  std::lock_guard<std::mutex> lk(keys->mu);
  auto& S = keys->shards;
  CachedNtts h(rns);
  if (int rc = key_switch_ntts(h, n, moduli, decomp, key_modulus_size)) return rc;
  const size_t row = (size_t)decomp * n * sizeof(uint64_t);  // host pitch of result: one key component over all moduli
  const uint64_t q_last = moduli[key_modulus_size - 1];

  // Every shard's operations are issued by its own host thread; the threads meet at two points, because an event must
  // have been RECORDED before another stream is told to wait for it.
  std::atomic<int> first_error{0};
  std::mutex err_mu;
  std::string err_text;
  std::atomic<unsigned> arrived{0};
  const unsigned nshards = (unsigned)S.size();
  auto meet = [&](unsigned round) {  // all threads have issued everything of the rounds before `round`
    arrived.fetch_add(1, std::memory_order_acq_rel);
    while (arrived.load(std::memory_order_acquire) < round * nshards) std::this_thread::yield();
  };
  auto worker = [&](size_t si) {
    auto& z = S[si];
    int rc = 0;
    auto bad = [&](int code) {
      if (code && !rc) {
        rc = code;
        int expected = 0;
        if (first_error.compare_exchange_strong(expected, code)) {
          std::lock_guard<std::mutex> g(err_mu);
          err_text = t_error;  // the message lives in this worker's thread-local slot
        }
      }
      return code != 0;
    };
    auto cu = [&](cudaError_t e, const char* what) { return e != cudaSuccess && bad(cuda_fail(e, what)); };
    const uint64_t dhi = std::min<uint64_t>(z.hi, decomp), nd = dhi > z.lo ? dhi - z.lo : 0;
    const uint64_t cnt = z.hi - z.lo, per_mod = decomp * n;
    const bool last = si + 1 == S.size();
    cu(cudaSetDevice(z.device), "cudaSetDevice");
    // A: digits and result slices in, inverse NTT of the digits, all-gather to every peer
    if (!rc && nd) {
      cu(cudaMemcpyAsync(z.t_coef + z.lo * n, t_target + z.lo * n, nd * n * 8, cudaMemcpyHostToDevice, z.stream), "H2D digits");
      if (!rc) cu(cudaMemcpy2DAsync(z.res, nd * n * 8, result + z.lo * n, row, nd * n * 8, kcc, cudaMemcpyHostToDevice, z.stream), "H2D result");
      // the all-gather: the transform's last kernel stores every coefficient into all peers as well (P2P stores over
      // NVLink, fused into the producing kernel); copy-engine peer copies behind the transform where P2P is unavailable
      std::vector<uint64_t*> peers;
      if (keys->p2p)
        for (size_t pi = 0; pi < S.size(); ++pi)
          if (pi != si) peers.push_back(S[pi].t_coef + z.lo * n);
      if (!rc) bad(ntt_multi_on_device(false, z.device, h.data() + z.lo, nd, z.t_coef + z.lo * n, z.t_coef + z.lo * n, 1, 1, z.stream,
                                       keys->p2p ? &peers : nullptr));
      for (size_t pi = 0; pi < S.size() && !rc && !keys->p2p; ++pi)
        if (pi != si)
          cu(cudaMemcpyPeerAsync(S[pi].t_coef + z.lo * n, S[pi].device, z.t_coef + z.lo * n, z.device, nd * n * 8, z.stream), "all-gather");
    }
    if (!rc) cu(cudaEventRecord(z.gathered, z.stream), "cudaEventRecord");
    meet(1);
    // B: wait for everybody's digits; reduce them into my moduli, transform, multiply-accumulate with my key slices
    for (size_t pi = 0; pi < S.size() && !rc && !first_error.load(); ++pi)
      if (pi != si) cu(cudaStreamWaitEvent(z.stream, S[pi].gathered, 0), "cudaStreamWaitEvent");
    const uint64_t* const* zk = z.keys.data();
    for (uint64_t e0 = 0; e0 < cnt && !rc && !first_error.load(); e0 += kParamBlock) {
      const uint64_t c = std::min<uint64_t>(kParamBlock, cnt - e0);
      uint64_t slots[kParamBlock];
      for (uint64_t e = 0; e < c; ++e) slots[e] = e0 + e;  // key slot = index inside the shard
      bad(ks_mac_round(z.device, h.data() + z.lo + e0, slots, c, cnt, z.ops + e0 * per_mod, z.t_coef, decomp, n, kcc,
                       z.prod + e0 * kcc * n, 0, &zk, nullptr, 1, z.stream));
    }
    // C: the owner of the special prime brings that part back to coefficients and sends it to everybody
    if (last && !rc && !first_error.load()) {
      std::vector<uint64_t*> peers;
      if (keys->p2p)
        for (size_t pi = 0; pi < S.size(); ++pi)
          if (pi != si) peers.push_back(S[pi].t_last);
      hexl_b200_ntt* hl = h[decomp];
      bad(ntt_multi_on_device(false, z.device, &hl, 1, z.t_last, z.prod + (decomp - z.lo) * kcc * n, 2, kcc, z.stream,
                              keys->p2p ? &peers : nullptr));
      for (size_t pi = 0; pi < S.size() && !rc && !keys->p2p; ++pi)
        if (pi != si) cu(cudaMemcpyPeerAsync(S[pi].t_last, S[pi].device, z.t_last, z.device, kcc * n * 8, z.stream), "broadcast");
      if (!rc) cu(cudaEventRecord(z.special, z.stream), "cudaEventRecord");
    }
    meet(2);
    // D: mod-down by the special prime, accumulate into my slices of result, results out
    if (nd && !rc && !first_error.load()) {
      if (!last) cu(cudaStreamWaitEvent(z.stream, S.back().special, 0), "cudaStreamWaitEvent");
      if (!rc)
        bad(mod_down_blocks(z.device, z.res, nd, z.prod, false, true, z.t_last, z.tmp, n, kcc, q_last, h.data() + z.lo,
                            moduli + z.lo, modswitch + z.lo, nd, z.stream));
      if (!rc) cu(cudaMemcpy2DAsync(result + z.lo * n, row, z.res, nd * n * 8, nd * n * 8, kcc, cudaMemcpyDeviceToHost, z.stream), "D2H result");
    }
    const cudaError_t e = cudaStreamSynchronize(z.stream);  // always drain: host buffers are in flight
    if (e != cudaSuccess) cu(e, "cudaStreamSynchronize");
  };
  keys->pool.run(worker);
  if (const int rc = first_error.load()) {
    t_error = err_text;
    return rc;
  }
  return 0;
}

static void free_shards(hexl_b200_keys* k) {
  k->pool.shutdown();
  for (auto& z : k->shards) {
    if (cudaSetDevice(z.device) != cudaSuccess) continue;
    for (uint64_t* p : z.keys) cudaFree(p);
    for (uint64_t* p : {z.t_coef, z.ops, z.prod, z.tmp, z.t_last, z.res, z.digits}) cudaFree(p);
    if (z.stream) cudaStreamDestroy(z.stream);
    if (z.gathered) cudaEventDestroy(z.gathered);
    if (z.special) cudaEventDestroy(z.special);
  }
  k->shards.clear();
}

// ---------------------------------------------------------------- rescale by the last modulus
// `count` polynomials of rns limbs x n words (limb i under moduli[i]), device pointers on the current device; limbs
// [0, rns - 1) of result get floor((X + q_last/2) / q_last) mod q_i.  NTT form: the gathered last limbs of a chunk of
// polynomials run through the shared mod-down (mod_down_on_device); coefficient form: one fused kernel per block of
// moduli.  h: the cached transforms of every modulus (NTT form only).
static int divide_and_round_on_device(int dev, uint64_t* result, const uint64_t* operand, uint64_t n,
                                      const uint64_t* moduli, uint64_t rns, uint64_t count, bool ntt_form,
                                      hexl_b200_ntt* const* h, cudaStream_t s) {
  const uint64_t L = rns - 1, q_last = moduli[L], mu_last = nt::multiply_factor(1, 64, q_last);
  std::vector<uint64_t> inv(L);
  for (uint64_t i = 0; i < L; ++i) inv[i] = nt::inverse_mod(q_last % moduli[i], moduli[i]);
  if (!ntt_form) {
    for (uint64_t i0 = 0; i0 < L; i0 += kParamBlock) {
      const uint64_t cnt = std::min<uint64_t>(kParamBlock, L - i0);
      KsModuli mods;
      for (uint64_t e = 0; e < cnt; ++e) {
        const uint64_t qi = moduli[i0 + e];
        const Twiddle f = make_twiddle(inv[i0 + e], qi);
        mods.m[e] = KsModulus{qi, nt::multiply_factor(1, 64, qi), f.w, f.wp, qi - ((q_last >> 1) % qi)};
      }
      cudaError_t e = launch_rescale_coef(result, operand, n, rns, i0, cnt, count, q_last, mu_last, mods, s);
      if (e != cudaSuccess) return cuda_fail(e, "DivideAndRoundQLast launch");
    }
    return 0;
  }
  // polynomials per round: the last limbs plus one block of rounded limbs stay within ~256 MiB of scratch
  const uint64_t block = std::min<uint64_t>(L, kParamBlock);
  uint64_t chunk = std::max<uint64_t>(1, (256ull << 20) / ((block + 1) * n * 8));
  chunk = std::min(chunk, count);
  Scratch ws(s);
  uint64_t *t_last = nullptr, *tmp = nullptr;
  if (int rc = ws.get(&t_last, chunk * n)) return rc;        // [p][n]
  if (int rc = ws.get(&tmp, block * chunk * n)) return rc;   // [e][p][n]
  for (uint64_t p0 = 0; p0 < count; p0 += chunk) {
    const uint64_t cnt = std::min(chunk, count - p0);
    const uint64_t* op = operand + p0 * rns * n;
    CU(cudaMemcpy2DAsync(t_last, n * 8, op + L * n, rns * n * 8, n * 8, cnt, cudaMemcpyDeviceToDevice, s));
    if (int rc = mod_down_on_device(dev, result + p0 * rns * n, rns, op, true, false, t_last, tmp, n, cnt, h[L], h,
                                    moduli, inv.data(), L, s))
      return rc;
  }
  return 0;  // ~Scratch returns the buffers to the pool in stream order
}

// BGV's modulus switch by the last modulus, same layout: limbs [0, rns - 1) of result get (x_i - delta) q_L^-1 mod q_i,
// with delta = x_L + q_L [-x_L q_L^-1]_tau the t-corrected conversion of the last limb (T = {q_L}, one source).  Per
// chunk of polynomials: in NTT form the last limbs are gathered and transformed back to coefficients (canonical); per
// block of 64 moduli, one conversion launch reads every polynomial's last limb through its strides, delta is
// transformed forward (NTT form only) and the finish stores, reading the operand laid out like the result (in place
// works: limb rns - 1 is neither written nor read after the conversions of the chunk).
static int bgv_mod_switch_on_device(int dev, uint64_t* result, const uint64_t* operand, uint64_t n,
                                    const uint64_t* moduli, uint64_t rns, uint64_t count, bool ntt_form,
                                    uint64_t plain_modulus, hexl_b200_ntt* const* h, cudaStream_t s) {
  const uint64_t L = rns - 1, q_last = moduli[L];
  const uint64_t block = std::min<uint64_t>(L, kParamBlock);
  uint64_t chunk = std::max<uint64_t>(1, (256ull << 20) / ((block + 1) * n * 8));
  chunk = std::min(chunk, count);
  Scratch ws(s);
  uint64_t *t_last = nullptr, *tmp = nullptr;
  if (ntt_form)
    if (int rc = ws.get(&t_last, chunk * n)) return rc;    // [p][n]
  if (int rc = ws.get(&tmp, block * chunk * n)) return rc;  // [e][p][n]
  for (uint64_t p0 = 0; p0 < count; p0 += chunk) {
    const uint64_t cnt = std::min(chunk, count - p0);
    const uint64_t* op = operand + p0 * rns * n;
    const uint64_t* last = op + L * n;
    uint64_t last_poly = rns * n;
    if (ntt_form) {
      CU(cudaMemcpy2DAsync(t_last, n * 8, last, rns * n * 8, n * 8, cnt, cudaMemcpyDeviceToDevice, s));
      if (int rc = ntt_multi_on_device(false, dev, h + L, 1, t_last, t_last, 1, cnt, s)) return rc;
      last = t_last;
      last_poly = n;
    }
    for (uint64_t i0 = 0; i0 < L; i0 += kParamBlock) {
      const uint64_t cm = std::min<uint64_t>(kParamBlock, L - i0);
      if (int rc = base_convert_on_device(tmp, cnt * n, n, last, n, last_poly, n, cnt, &q_last, 1, moduli + i0, cm,
                                          false, s, plain_modulus))
        return rc;
      if (ntt_form)
        if (int rc = ntt_multi_on_device(true, dev, h + i0, cm, tmp, tmp, 4, cnt, s)) return rc;
      KsModuli fin;
      for (uint64_t e = 0; e < cm; ++e) {
        const uint64_t qi = moduli[i0 + e];
        const Twiddle f = make_twiddle(nt::inverse_mod(q_last % qi, qi), qi);
        fin.m[e] = KsModulus{qi, nt::multiply_factor(1, 64, qi), f.w, f.wp, 0};
      }
      const cudaError_t e =
          launch_ks_finish(result + p0 * rns * n, op, tmp, n, cnt, rns, i0, cm, fin, true, false, s);
      if (e != cudaSuccess) return cuda_fail(e, "BgvModSwitch: finish launch");
    }
  }
  return 0;  // ~Scratch returns the buffers to the pool in stream order
}

// The caller may have written device (or managed) key sources on any stream of their device, and the upload's copies
// run on the legacy default stream, which does not wait for non-blocking streams: wait for every device that owns a
// source before copying from it.
static int wait_for_key_sources(const uint64_t* const* k_switch_keys, uint64_t decomp) {
  std::vector<int> owners;
  for (uint64_t j = 0; j < decomp; ++j) {
    PtrInfo pi;
    if (int rc = classify(k_switch_keys[j], &pi)) return rc;
    if (pi.where == Where::Device && std::find(owners.begin(), owners.end(), pi.device) == owners.end())
      owners.push_back(pi.device);
  }
  for (int dev : owners) {
    DeviceGuard g;
    if (int rc = g.enter(dev)) return rc;
    CU(cudaDeviceSynchronize());
  }
  return 0;
}

}  // namespace hexl_b200

// =============================================================== extern "C"
extern "C" {

int hexl_b200_keys_upload(hexl_b200_keys** out, const uint64_t* const* k_switch_keys, uint64_t n,
                          uint64_t decomp, uint64_t key_modulus_size, uint64_t kcc) {
  REQUIRE(out && k_switch_keys, "Require out, k_switch_keys != nullptr");
  *out = nullptr;
  REQUIRE(n >= 1 && decomp >= 1 && kcc >= 1 && key_modulus_size >= 1, "Require non-zero sizes");
  for (uint64_t j = 0; j < decomp; ++j) REQUIRE(k_switch_keys[j] != nullptr, "Require k_switch_keys[j] != nullptr");
  if (int rc = wait_for_key_sources(k_switch_keys, decomp)) return rc;
  std::vector<int> devs;
  if (int rc = host_devices(&devs)) return rc;
  std::sort(devs.begin(), devs.end());
  devs.erase(std::unique(devs.begin(), devs.end()), devs.end());
  hexl_b200_keys* k = new (std::nothrow) hexl_b200_keys();
  if (!k) return fail(HEXL_B200_ERR_ALLOC, "out of host memory");
  k->n = n; k->decomp = decomp; k->kcc = kcc; k->kms = key_modulus_size;
  const size_t bytes = (size_t)kcc * key_modulus_size * n * sizeof(uint64_t);
  int rc = 0;
  for (int dev : devs) {
    DeviceGuard g;
    if ((rc = g.enter(dev))) break;
    std::vector<uint64_t*>& v = k->dev[dev];
    v.assign(decomp, nullptr);
    for (uint64_t j = 0; j < decomp && !rc; ++j) {
      cudaError_t e = cudaMalloc(&v[j], bytes);
      if (e == cudaSuccess) e = cudaMemcpy(v[j], k_switch_keys[j], bytes, cudaMemcpyDefault);  // host or device source
      if (e != cudaSuccess) rc = cuda_fail(e, "hexl_b200_keys_upload");
    }
    if (!rc) {
      cudaError_t e = cudaDeviceSynchronize();
      if (e != cudaSuccess) rc = cuda_fail(e, "hexl_b200_keys_upload");
    }
    if (rc) break;
  }
  if (rc) {
    hexl_b200_keys_release(k);
    return rc;
  }
  *out = k;
  return 0;
}

void hexl_b200_keys_release(hexl_b200_keys* k) {
  if (!k || k->refs.fetch_sub(1) != 1) return;
  int prev = -1;
  cudaGetDevice(&prev);
  free_shards(k);
  for (auto& kv : k->dev)
    if (cudaSetDevice(kv.first) == cudaSuccess)
      for (uint64_t* p : kv.second) cudaFree(p);
  if (prev >= 0) cudaSetDevice(prev);
  cudaGetLastError();
  delete k;
}

int hexl_b200_keys_upload_sharded(hexl_b200_keys** out, const uint64_t* const* k_switch_keys, uint64_t n,
                                  uint64_t decomp, uint64_t key_modulus_size, uint64_t kcc) {
  REQUIRE(out && k_switch_keys, "Require out, k_switch_keys != nullptr");
  *out = nullptr;
  REQUIRE(n >= 2 && !(n & (n - 1)), "Require n a power of two");
  REQUIRE(decomp >= 1 && kcc >= 1 && key_modulus_size >= decomp + 1, "Require decomp, kcc >= 1 and key_modulus_size > decomp");
  for (uint64_t j = 0; j < decomp; ++j) REQUIRE(k_switch_keys[j] != nullptr, "Require k_switch_keys[j] != nullptr");
  if (int rc = wait_for_key_sources(k_switch_keys, decomp)) return rc;
  std::vector<int> devs;
  if (int rc = host_devices(&devs)) return rc;
  const uint64_t rns = decomp + 1;
  if (devs.size() > rns) devs.resize(rns);
  hexl_b200_keys* k = new (std::nothrow) hexl_b200_keys();
  if (!k) return fail(HEXL_B200_ERR_ALLOC, "out of host memory");
  k->n = n; k->decomp = decomp; k->kcc = kcc; k->kms = key_modulus_size;
  int prev = 0;
  cudaGetDevice(&prev);
  int rc = 0;
  const size_t src_pitch = (size_t)key_modulus_size * n * 8;
  bool p2p_all = devs.size() - 1 <= (size_t)kMaxMirrors;
  for (size_t si = 0; si < devs.size() && !rc; ++si) {
    k->shards.emplace_back();
    auto& z = k->shards.back();
    z.device = devs[si];
    z.lo = rns * si / devs.size();
    z.hi = rns * (si + 1) / devs.size();
    const uint64_t cnt = z.hi - z.lo, nd = std::min<uint64_t>(z.hi, decomp) > z.lo ? std::min<uint64_t>(z.hi, decomp) - z.lo : 0;
    cudaError_t e = cudaSetDevice(z.device);
    for (size_t pj = 0; pj < si && e == cudaSuccess; ++pj)  // NVLink peer mappings in both directions (ignore "already enabled")
      if (devs[pj] != z.device) {
        int ab = 0, ba = 0;
        cudaDeviceCanAccessPeer(&ab, z.device, devs[pj]);
        cudaDeviceCanAccessPeer(&ba, devs[pj], z.device);
        if (!ab || !ba) p2p_all = false;
        cudaDeviceEnablePeerAccess(devs[pj], 0);
        cudaGetLastError();
        cudaSetDevice(devs[pj]);
        cudaDeviceEnablePeerAccess(z.device, 0);
        cudaGetLastError();
        cudaSetDevice(z.device);
      }
    auto alloc = [&](uint64_t** p, uint64_t words) {
      if (e == cudaSuccess) e = cudaMalloc(p, std::max<uint64_t>(words, 1) * 8);
    };
    alloc(&z.t_coef, decomp * n);
    alloc(&z.ops, cnt * decomp * n);
    alloc(&z.prod, cnt * kcc * n);
    alloc(&z.tmp, cnt * kcc * n);
    alloc(&z.t_last, kcc * n);
    alloc(&z.res, kcc * std::max<uint64_t>(nd, 1) * n);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&z.stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&z.gathered, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&z.special, cudaEventDisableTiming);
    z.keys.assign(decomp, nullptr);
    for (uint64_t j = 0; j < decomp && e == cudaSuccess; ++j) {
      alloc(&z.keys[j], kcc * cnt * n);
      // key slot of RNS index i is i, except the special prime (index decomp) which sits in the last slot
      if (nd && e == cudaSuccess)
        e = cudaMemcpy2D(z.keys[j], cnt * n * 8, k_switch_keys[j] + z.lo * n, src_pitch, nd * n * 8, kcc, cudaMemcpyDefault);
      if (z.hi == rns && e == cudaSuccess)
        e = cudaMemcpy2D(z.keys[j] + (decomp - z.lo) * n, cnt * n * 8, k_switch_keys[j] + (key_modulus_size - 1) * n, src_pitch,
                         n * 8, kcc, cudaMemcpyDefault);
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e != cudaSuccess) rc = cuda_fail(e, "hexl_b200_keys_upload_sharded");
  }
  cudaSetDevice(prev);
  if (rc) {
    hexl_b200_keys_release(k);
    return rc;
  }
  static const bool no_p2p_stores = std::getenv("HEXL_B200_KS_PEER_COPIES") != nullptr;  // force the copy-engine exchange
  k->p2p = p2p_all && !no_p2p_stores;
  k->pool.start(k->shards.size());
  *out = k;
  return 0;
}

int hexl_b200_key_switch_resident(uint64_t* result, const uint64_t* t_target_iter_ptr, uint64_t n, uint64_t decomp,
                                  uint64_t key_modulus_size, uint64_t rns, uint64_t kcc, const uint64_t* moduli,
                                  const hexl_b200_keys* keys, const uint64_t* modswitch_factors, uint64_t batch,
                                  void* stream) {
  if (int rc = key_switch_check(result, t_target_iter_ptr, n, decomp, key_modulus_size, rns, kcc, moduli, modswitch_factors))
    return rc;
  REQUIRE(keys != nullptr, "Require keys != nullptr");
  REQUIRE(keys_fit(keys, n, decomp, kcc, key_modulus_size), "the key handle was uploaded for another shape");
  if (batch == 0) return 0;
  PtrInfo pi;
  if (int rc = classify_all({result, t_target_iter_ptr}, &pi)) return rc;
  if (!keys->shards.empty()) {
    REQUIRE(pi.where == Where::Host, "keys sharded by modulus take host buffers (every shard receives its own slices)");
    REQUIRE(keys->decomp == decomp, "keys sharded by modulus were uploaded for another decomp_modulus_size");
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = key_switch_sharded(result + c * kcc * decomp * n, t_target_iter_ptr + c * decomp * n, n, decomp,
                                      key_modulus_size, rns, kcc, moduli, const_cast<hexl_b200_keys*>(keys), modswitch_factors))
        return rc;
    return 0;
  }
  if (pi.where == Where::Host)
    return key_switch_host(result, t_target_iter_ptr, n, decomp, key_modulus_size, rns, kcc, moduli, keys,
                           modswitch_factors, batch);
  std::vector<const uint64_t* const*> dk;
  if (keys_on_device(&keys, 1, pi.device, &dk) < 1)
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "the key handle holds no copy on the device of result");
  return run_on_device(pi, stream, [&] {
    for (uint64_t c = 0; c < batch; ++c)
      if (int rc = key_switch_on_device(pi.device, result + c * kcc * decomp * n, t_target_iter_ptr + c * decomp * n, n,
                                        decomp, key_modulus_size, rns, kcc, moduli, dk[0], modswitch_factors,
                                        (cudaStream_t)stream))
        return rc;
    return 0;
  });
}

int hexl_b200_key_switch(uint64_t* result, const uint64_t* t_target_iter_ptr, uint64_t n, uint64_t decomp,
                         uint64_t key_modulus_size, uint64_t rns, uint64_t kcc, const uint64_t* moduli,
                         const uint64_t* const* k_switch_keys, const uint64_t* modswitch_factors, void* stream) {
  if (int rc = key_switch_check(result, t_target_iter_ptr, n, decomp, key_modulus_size, rns, kcc, moduli, modswitch_factors))
    return rc;
  REQUIRE(k_switch_keys != nullptr, "Require non-null arguments");
  for (uint64_t j = 0; j < decomp; ++j) REQUIRE(k_switch_keys[j] != nullptr, "Require k_switch_keys[j] != nullptr");
  PtrInfo pi;
  if (int rc = classify_all({result, t_target_iter_ptr}, &pi)) return rc;
  for (uint64_t j = 0; j < decomp; ++j) {
    PtrInfo pk;
    if (int rc = classify(k_switch_keys[j], &pk)) return rc;
    if (pk.where != pi.where || (pk.where == Where::Device && pk.device != pi.device))
      return fail(HEXL_B200_ERR_MIXED_POINTERS, "k_switch_keys[%llu] lives elsewhere than result", (unsigned long long)j);
  }
  if (pi.where == Where::Device)
    return run_on_device(pi, stream, [&] {
      return key_switch_on_device(pi.device, result, t_target_iter_ptr, n, decomp, key_modulus_size, rns, kcc, moduli,
                                  k_switch_keys, modswitch_factors, (cudaStream_t)stream);
    });
  // Host pointers, the reference's call shape (key-switch.hpp:34-39 keeps the keys in caller memory): the keys
  // cross PCIe on every call.  A caller that switches more than once with the same keys uploads them once
  // (hexl_b200_keys_upload) and calls hexl_b200_key_switch_resident.
  hexl_b200_keys* tmp = nullptr;
  if (int rc = hexl_b200_keys_upload(&tmp, k_switch_keys, n, decomp, key_modulus_size, kcc)) return rc;
  const int rc = key_switch_host(result, t_target_iter_ptr, n, decomp, key_modulus_size, rns, kcc, moduli, tmp,
                                 modswitch_factors, 1);
  hexl_b200_keys_release(tmp);
  return rc;
}

}  // extern "C"

namespace {

// hexl_b200_divide_and_round_q_last (plain_modulus = 0) and hexl_b200_bgv_mod_switch (plain_modulus checked)
int last_modulus_call(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                      uint64_t rns_modulus_size, uint64_t count, int ntt_form, void* stream, uint64_t plain_modulus) {
  REQUIRE(result && operand && moduli, "Require result, operand, moduli != nullptr");
  REQUIRE(rns_modulus_size >= 2, "Require rns_modulus_size >= 2");
  REQUIRE(ntt_form == 0 || ntt_form == 1, "Require ntt_form = 0 or 1");
  const uint64_t rns = rns_modulus_size, L = rns - 1, q_last = moduli[L];
  for (uint64_t i = 0; i < rns; ++i)
    // the lazy sums of the round and finish steps (< 8q) need q < 2^61
    REQUIRE(moduli[i] > 1 && moduli[i] < (1ull << 61), "Require 1 < moduli[%llu] < 2^61", (unsigned long long)i);
  for (uint64_t i = 0; i < L; ++i)
    REQUIRE(std::gcd(moduli[i], q_last) == 1, "Require moduli[%llu] coprime to the last modulus",
            (unsigned long long)i);
  if (ntt_form) {
    REQUIRE(n >= 2 && n <= (1ull << 20) && !(n & (n - 1)), "Require n a power of two in [2, 2^20]");
    for (uint64_t i = 0; i < rns; ++i) {
      const char* why = "";
      REQUIRE(check_ntt_arguments(n, moduli[i], &why), "moduli[%llu]: %s", (unsigned long long)i, why);
    }
  } else {
    REQUIRE(n >= 1, "Require n >= 1");
  }
  if (count == 0) return 0;
  const uint64_t unit = rns * n, total = count * unit;
  REQUIRE(result == operand || result + total <= operand || operand + total <= result,
          "result and operand must be the same buffer or not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, operand}, &pi)) return rc;
  CachedNtts h(ntt_form ? rns : 0);
  for (uint64_t i = 0; i < h.h.size(); ++i)
    if (int rc = h.load(i, n, moduli[i])) return rc;
  if (int rc = check_limb_bounds(operand, count, rns, n, [&](u64 i) { return moduli[i]; }, pi, "operand", stream)) return rc;
  const bool ntt = ntt_form != 0;
  auto on_device = [&](int dev, uint64_t* r, const uint64_t* a, uint64_t polys, cudaStream_t s) {
    return plain_modulus ? bgv_mod_switch_on_device(dev, r, a, n, moduli, rns, polys, ntt, plain_modulus, h.data(), s)
                         : divide_and_round_on_device(dev, r, a, n, moduli, rns, polys, ntt, h.data(), s);
  };
  if (pi.where == Where::Device)
    return run_on_device(pi, stream, [&] { return on_device(pi.device, result, operand, count, (cudaStream_t)stream); });
  // host pointers: whole polynomials through the staging slots (split over the host devices when set); only limbs
  // [0, L) of each polynomial are copied back, so limb L of result is left as it was
  return run_host(result, operand, nullptr, total, unit, [&](int dev, u64, u64, auto&& run) {
    return run([&, dev](u64* r, const u64* a, const u64*, u64, u64 elems, cudaStream_t s) {
      return on_device(dev, r, a, elems / unit, s);
    });
  }, L * n);
}

}  // namespace

extern "C" {

int hexl_b200_divide_and_round_q_last(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                                      uint64_t rns_modulus_size, uint64_t count, int ntt_form, void* stream) {
  return last_modulus_call(result, operand, n, moduli, rns_modulus_size, count, ntt_form, stream, 0);
}

int hexl_b200_bgv_mod_switch(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                             uint64_t rns_modulus_size, uint64_t plain_modulus, uint64_t count, int ntt_form,
                             void* stream) {
  REQUIRE(moduli, "Require result, operand, moduli != nullptr");
  if (int rc = bgv_plain_modulus_check(plain_modulus, moduli, rns_modulus_size)) return rc;
  return last_modulus_call(result, operand, n, moduli, rns_modulus_size, count, ntt_form, stream, plain_modulus);
}

}  // extern "C"
