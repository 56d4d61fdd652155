// The plaintext operands of BFV and BGV (hexl_b200_plain_lift, hexl_b200_bfv_add_plain, hexl_b200_bfv_multiply_plain):
// the argument rules, the constants of plain.cu's two kernels (the add_plain table cached on each device), the device
// chains and their host staging.
#include "capi.h"

using namespace hexl_b200;

namespace hexl_b200 {

namespace {

constexpr uint64_t kLimit = 1ull << 61;

bool disjoint(const void* a, uint64_t a_words, const void* b, uint64_t b_words) {
  const uint64_t *x = static_cast<const uint64_t*>(a), *y = static_cast<const uint64_t*>(b);
  return x + a_words <= y || y + b_words <= x;
}

// The refusals every plaintext call shares; ntt: the moduli must carry a transform of degree n
int plain_check(const void* result, const void* in, const void* plain, uint64_t pcc, uint64_t n,
                const uint64_t* moduli, uint64_t l, uint64_t t, bool ntt) {
  REQUIRE(result && in && plain && moduli, "Require non-null arguments");
  REQUIRE(n >= 2 && n <= (1ull << 20) && !(n & (n - 1)), "Require n a power of two in [2, 2^20]");
  REQUIRE(l >= 1 && l <= (uint64_t)kParamBlock, "Require 1 <= level_size <= %d", kParamBlock);
  REQUIRE(t >= 2 && t < kLimit, "Require 2 <= plain_modulus < 2^61");
  REQUIRE(pcc >= 1 && pcc <= n, "Require 1 <= plain_coeff_count <= n");
  for (uint64_t i = 0; i < l; ++i) {
    const char* why = "";
    REQUIRE(moduli[i] >= 2 && moduli[i] < kLimit, "Require 2 <= moduli[%llu] < 2^61", (unsigned long long)i);
    if (ntt) REQUIRE(check_ntt_arguments(n, moduli[i], &why), "moduli[%llu]: %s", (unsigned long long)i, why);
  }
  return 0;
}

// What a call needs: the lift's moduli and, for the calls that transform, the transforms of the l moduli
struct PlainPlan {
  uint64_t n, l, t, cf, cf_shoup;
  PlainModuli mods{};
  CachedNtts h;
  PlainPlan(uint64_t n_, const uint64_t* moduli, uint64_t l_, uint64_t t_, uint64_t cf_)
      : n(n_), l(l_), t(t_), cf(cf_), cf_shoup(nt::multiply_factor(cf_, 64, t_)), h(l_) {
    for (uint64_t i = 0; i < l; ++i) {
      mods.q[i] = moduli[i];
      mods.mu[i] = nt::multiply_factor(1, 64, moduli[i]);
    }
  }
  int load() {
    for (uint64_t i = 0; i < l; ++i)
      if (int rc = h.load(i, n, mods.q[i])) return rc;
    return 0;
  }
};

// `count` plaintexts of pcc words into count x l x n words at result, then (ntt) their forward transforms in place
int lift_on_device(int dev, uint64_t* result, const uint64_t* plain, uint64_t pcc, uint64_t count,
                   const PlainPlan& pl, bool ntt, cudaStream_t s) {
  cudaError_t e = launch_plain_lift(result, plain, pcc, pl.n, count, pl.l, pl.t, pl.cf, pl.cf_shoup, pl.mods, s);
  if (e != cudaSuccess) return cuda_fail(e, "PlainLift launch");
  if (!ntt) return 0;
  std::vector<hexl_b200_ntt*> hs;  // the l handles once per plaintext
  for (uint64_t p = 0; p < count; ++p) hs.insert(hs.end(), pl.h.data(), pl.h.data() + pl.l);
  return ntt_multi_on_device(true, dev, hs.data(), hs.size(), result, result, 1, 1, s);
}

// The constants of bfv_add_plain_kernel (plain.cu states the layout), from Q = q_0 ... q_{l-1}
std::vector<uint64_t> add_plain_table(const uint64_t* moduli, uint64_t l, uint64_t t) {
  Big Q{1};
  for (uint64_t i = 0; i < l; ++i) big_mul(Q, moduli[i]);
  const uint64_t r = big_divmod(Q, t);  // Q is now floor(Q / t)
  std::vector<uint64_t> tab;
  for (uint64_t i = 0; i < l; ++i) {
    const uint64_t q = moduli[i], delta = big_mod(Q, q);
    tab.insert(tab.end(), {q, nt::multiply_factor(1, 64, q), delta, nt::multiply_factor(delta, 64, q)});
  }
  tab.insert(tab.end(), {t, r, nt::multiply_factor(r, 64, t), (t + 1) / 2});
  return tab;
}

// ct times the transformed plaintext fplain (l x n words, canonical), result may be ct: one forward transform of both
// components into result, then one inverse transform per component that multiplies by fplain on load
int multiply_plain_one(int dev, uint64_t* result, const uint64_t* ct, const uint64_t* fplain, const PlainPlan& pl,
                       cudaStream_t s) {
  const uint64_t l = pl.l, comp = l * pl.n;
  std::vector<hexl_b200_ntt*> hs(pl.h.data(), pl.h.data() + l);
  hs.insert(hs.end(), pl.h.data(), pl.h.data() + l);
  if (int rc = ntt_multi_on_device(true, dev, hs.data(), 2 * l, result, ct, 1, 1, s)) return rc;
  for (uint64_t k = 0; k < 2; ++k)
    if (int rc = ntt_multi_on_device(false, dev, hs.data(), l, result + k * comp, result + k * comp, 1, 1, s, nullptr,
                                     false, fplain))
      return rc;
  return 0;
}

// Host buffers, through stage_items one item (ciphertext, or PlainLift's plaintext) per slot step, split by item over
// the host devices.  Item c's in_words words of `in` (optional) go to slot buffer 0, which run() leaves holding the
// item's res_words words of result; its plaintext (plain_words words at plain + c plain_words) goes to buffer 1.  A
// broadcast plaintext goes to each device of the split once, before its first item, at `front` words into a buffer of
// its own; prep (optional) then fills the front words from it on that device, and run() reads the front instead.
using PlainPrep = std::function<int(int, const uint64_t*, uint64_t*)>;
using PlainRun = std::function<int(int, uint64_t*, const uint64_t*, cudaStream_t)>;
int plain_host(uint64_t* result, uint64_t res_words, const uint64_t* in, uint64_t in_words, const uint64_t* plain,
               uint64_t plain_words, bool broadcast, uint64_t items, uint64_t front, const PlainPrep& prep,
               const PlainRun& run) {
  std::vector<int> devs;
  if (int rc = host_devices(&devs)) return rc;
  std::vector<std::pair<int, uint64_t*>> uploaded;
  const int rc = stage_items(devs, items, 1, [&](int dev, u64, u64, auto&& stage) -> int {
    const uint64_t* shared = nullptr;
    if (broadcast) {
      uint64_t* p = nullptr;
      CU(cudaMalloc(&p, (front + plain_words) * sizeof(uint64_t)));
      uploaded.emplace_back(dev, p);
      CU(cudaMemcpy(p + front, plain, plain_words * sizeof(uint64_t), cudaMemcpyHostToDevice));
      if (prep)
        if (int rc = prep(dev, p + front, p)) return rc;
      CU(cudaStreamSynchronize(nullptr));  // the staging streams do not wait for the legacy stream
      shared = prep ? p : p + front;
    }
    return stage([&](const StageSlot& sl, u64 c, u64) -> int {
      if (int rc = sl.reserve(0, std::max(res_words, in_words) * sizeof(uint64_t))) return rc;
      if (!broadcast)
        if (int rc = sl.reserve(1, plain_words * sizeof(uint64_t))) return rc;
      const cudaStream_t sx = sl.stream();
      if (in) CU(cudaMemcpyAsync(sl.buf(0), in + c * in_words, in_words * 8, cudaMemcpyHostToDevice, sx));
      if (!broadcast)
        CU(cudaMemcpyAsync(sl.buf(1), plain + c * plain_words, plain_words * 8, cudaMemcpyHostToDevice, sx));
      if (int rc = run(dev, sl.buf(0), broadcast ? shared : sl.buf(1), sx)) return rc;
      CU(cudaMemcpyAsync(result + c * res_words, sl.buf(0), res_words * 8, cudaMemcpyDeviceToHost, sx));
      return 0;
    });
  });
  for (auto& u : uploaded) {
    DeviceGuard g;
    if (g.enter(u.first) == 0) cudaFree(u.second);
  }
  return rc;
}

// The debug checks of a ciphertext batch and its plaintexts (coefficient form: below t; NTT form: below each q_i)
int plain_bounds(const uint64_t* ct, uint64_t batch, const uint64_t* plain, uint64_t plain_count, uint64_t pcc,
                 bool plain_ntt, const uint64_t* moduli, uint64_t l, uint64_t n, uint64_t t, const PtrInfo& pi,
                 void* stream) {
  auto bound = [&](u64 i) { return moduli[i]; };
  if (ct)
    if (int rc = check_limb_bounds(ct, 2 * batch, l, n, bound, pi, "ct", stream)) return rc;
  if (plain_ntt) return check_limb_bounds(plain, plain_count, l, n, bound, pi, "plain", stream);
  return check_bounds(plain, plain_count * pcc, t, pi, "plain", stream);
}

}  // namespace

}  // namespace hexl_b200

extern "C" {

int hexl_b200_plain_lift(uint64_t* result, const uint64_t* plain, uint64_t plain_coeff_count, uint64_t n,
                         const uint64_t* moduli, uint64_t level_size, uint64_t plain_modulus,
                         uint64_t correction_factor, int ntt_form, uint64_t count, void* stream) {
  const uint64_t l = level_size, pcc = plain_coeff_count, t = plain_modulus;
  if (int rc = plain_check(result, plain, plain, pcc, n, moduli, l, t, ntt_form != 0)) return rc;
  REQUIRE(correction_factor >= 1 && correction_factor < t, "Require 1 <= correction_factor < plain_modulus");
  REQUIRE(ntt_form == 0 || ntt_form == 1, "Require ntt_form 0 or 1");
  if (count == 0) return 0;
  const uint64_t out_words = l * n;
  REQUIRE(disjoint(result, count * out_words, plain, count * pcc), "result and plain must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, plain}, &pi)) return rc;
  if (int rc = check_bounds(plain, count * pcc, t, pi, "plain", stream)) return rc;
  PlainPlan pl(n, moduli, l, t, correction_factor);
  if (ntt_form)
    if (int rc = pl.load()) return rc;
  if (pi.where == Where::Host)
    return plain_host(result, out_words, nullptr, 0, plain, pcc, false, count, 0, nullptr,
                      [&](int dev, uint64_t* d_res, const uint64_t* d_plain, cudaStream_t s) {
                        return lift_on_device(dev, d_res, d_plain, pcc, 1, pl, ntt_form != 0, s);
                      });
  return run_on_device(pi, stream, [&] {
    return lift_on_device(pi.device, result, plain, pcc, count, pl, ntt_form != 0, (cudaStream_t)stream);
  });
}

int hexl_b200_bfv_add_plain(uint64_t* result, const uint64_t* ct, const uint64_t* plain, uint64_t plain_coeff_count,
                            uint64_t plain_count, uint64_t n, const uint64_t* moduli, uint64_t level_size,
                            uint64_t plain_modulus, int subtract, uint64_t batch, void* stream) {
  const uint64_t l = level_size, pcc = plain_coeff_count, t = plain_modulus;
  if (int rc = plain_check(result, ct, plain, pcc, n, moduli, l, t, false)) return rc;
  REQUIRE(subtract == 0 || subtract == 1, "Require subtract 0 or 1");
  if (batch == 0) return 0;
  REQUIRE(plain_count == 1 || plain_count == batch, "Require plain_count 1 or batch");
  const uint64_t comp = l * n, ct_words = 2 * comp, total = batch * ct_words;
  REQUIRE(result == ct || disjoint(result, total, ct, total), "result must be ct or not overlap it");
  REQUIRE(disjoint(result, total, plain, plain_count * pcc), "result and plain must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, ct, plain}, &pi)) return rc;
  if (int rc = plain_bounds(ct, batch, plain, plain_count, pcc, false, moduli, l, n, t, pi, stream)) return rc;
  const std::vector<uint64_t> tab = add_plain_table(moduli, l, t);
  const bool broadcast = plain_count == 1;
  auto table = [&](int dev, cudaStream_t s, const uint64_t** out) {
    return device_table(tab, dev, s, out, "BfvAddPlain constants");
  };
  if (pi.where == Where::Host)
    return plain_host(result, ct_words, ct, ct_words, plain, pcc, broadcast, batch, 0, nullptr,
                      [&](int dev, uint64_t* d_ct, const uint64_t* d_plain, cudaStream_t s) {
                        const uint64_t* d_tab = nullptr;
                        if (int rc = table(dev, s, &d_tab)) return rc;
                        const cudaError_t e =
                            launch_bfv_add_plain(d_ct, d_ct, d_plain, pcc, 0, n, pcc, 1, l, subtract, d_tab, s);
                        return e == cudaSuccess ? 0 : cuda_fail(e, "BfvAddPlain launch");
                      });
  return run_on_device(pi, stream, [&] {
    const cudaStream_t s = (cudaStream_t)stream;
    const uint64_t* d_tab = nullptr;
    if (int rc = table(pi.device, s, &d_tab)) return rc;
    const bool in_place = result == ct;
    // in place only the plaintext's slots of c0 change; otherwise the kernel writes all of c0 and c1 is copied
    cudaError_t e = launch_bfv_add_plain(result, ct, plain, pcc, broadcast ? 0 : pcc, n, in_place ? pcc : n, batch, l,
                                         subtract, d_tab, s);
    if (e == cudaSuccess && !in_place)
      e = cudaMemcpy2DAsync(result + comp, ct_words * 8, ct + comp, ct_words * 8, comp * 8, batch,
                            cudaMemcpyDeviceToDevice, s);
    return e == cudaSuccess ? 0 : cuda_fail(e, "BfvAddPlain");
  });
}

int hexl_b200_bfv_multiply_plain(uint64_t* result, const uint64_t* ct, const uint64_t* plain,
                                 uint64_t plain_coeff_count, uint64_t plain_count, int plain_ntt_form, uint64_t n,
                                 const uint64_t* moduli, uint64_t level_size, uint64_t plain_modulus, uint64_t batch,
                                 void* stream) {
  const uint64_t l = level_size, t = plain_modulus;
  REQUIRE(plain_ntt_form == 0 || plain_ntt_form == 1, "Require plain_ntt_form 0 or 1");
  const bool ready = plain_ntt_form == 1;  // the plaintexts are PlainLift's NTT-form output: l x n words each
  const uint64_t pcc = ready ? n : plain_coeff_count;
  if (int rc = plain_check(result, ct, plain, pcc, n, moduli, l, t, true)) return rc;
  if (batch == 0) return 0;
  REQUIRE(plain_count == 1 || plain_count == batch, "Require plain_count 1 or batch");
  const uint64_t comp = l * n, ct_words = 2 * comp, total = batch * ct_words;
  const uint64_t plain_words = ready ? comp : pcc;
  REQUIRE(result == ct || disjoint(result, total, ct, total), "result must be ct or not overlap it");
  REQUIRE(disjoint(result, total, plain, plain_count * plain_words), "result and plain must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, ct, plain}, &pi)) return rc;
  if (int rc = plain_bounds(ct, batch, plain, plain_count, pcc, ready, moduli, l, n, t, pi, stream)) return rc;
  PlainPlan pl(n, moduli, l, t, 1);
  if (int rc = pl.load()) return rc;
  const bool broadcast = plain_count == 1;
  // a coefficient-form plaintext lifted and transformed into `lifted` (l x n words), then ct times it
  auto lifted_product = [&](int dev, uint64_t* res, const uint64_t* c, const uint64_t* p, uint64_t* lifted,
                            cudaStream_t s) {
    if (int rc = lift_on_device(dev, lifted, p, pcc, 1, pl, true, s)) return rc;
    return multiply_plain_one(dev, res, c, lifted, pl, s);
  };
  if (pi.where == Where::Host) {
    // a broadcast plaintext is lifted and transformed once per device, in front of its raw copy
    PlainPrep prep = nullptr;
    if (broadcast && !ready)
      prep = [&](int dev, const uint64_t* raw, uint64_t* out) { return lift_on_device(dev, out, raw, pcc, 1, pl, true, nullptr); };
    return plain_host(result, ct_words, ct, ct_words, plain, plain_words, broadcast, batch,
                      broadcast && !ready ? comp : 0, prep,
                      [&](int dev, uint64_t* d_ct, const uint64_t* d_plain, cudaStream_t s) {
                        if (ready || broadcast) return multiply_plain_one(dev, d_ct, d_ct, d_plain, pl, s);
                        Scratch ws(s);
                        uint64_t* lifted = nullptr;
                        if (int rc = ws.get(&lifted, comp)) return rc;
                        return lifted_product(dev, d_ct, d_ct, d_plain, lifted, s);
                      });
  }
  return run_on_device(pi, stream, [&] {
    const cudaStream_t s = (cudaStream_t)stream;
    Scratch ws(s);
    uint64_t* lifted = nullptr;
    if (!ready)
      if (int rc = ws.get(&lifted, comp)) return rc;
    for (uint64_t c = 0; c < batch; ++c) {
      uint64_t* res = result + c * ct_words;
      const uint64_t* in = ct + c * ct_words;
      const uint64_t* p = plain + (broadcast ? 0 : c * plain_words);
      int rc;
      if (ready)
        rc = multiply_plain_one(pi.device, res, in, p, pl, s);
      else if (broadcast && c > 0)  // lifted for the first ciphertext
        rc = multiply_plain_one(pi.device, res, in, lifted, pl, s);
      else
        rc = lifted_product(pi.device, res, in, p, lifted, s);
      if (rc) return rc;
    }
    return 0;
  });
}

}  // extern "C"
