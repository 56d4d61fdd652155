// What the host sources of the C ABI (include/hexl_b200.h) share: capi.cu (library state, staging, scratch pool),
// capi_ntt.cu, capi_eltwise.cu, capi_keyswitch.cu (key switch, key handles, rescale), capi_galois.cu and
// capi_hybrid.cu (hybrid key switch, fast base conversion, rotations and multiplication with hybrid keys, CKKS and BGV),
// capi_bfv.cu (BFV multiplication) and capi_plain.cu (the plaintext operands of BFV and BGV).
// Host-side responsibilities, all one-off or O(1) per call:
//   * argument validation mirroring the reference's HEXL_CHECKs,
//   * NTT handle = (N, q, root) -> twiddle tables, built on the host exactly as
//     hexl/ntt/ntt-internal.cpp:54-169 defines them, uploaded once per device,
//   * pointer classification: device pointers are launched on in place and
//     asynchronously; host pointers are staged through the GPU in pipelined
//     chunks (H2D / kernel / D2H on rotating streams) and, for batched calls,
//     optionally split across several GPUs with no inter-GPU traffic.
// There is no CPU compute path here: without a CUDA device every compute entry
// point returns HEXL_B200_ERR_NO_DEVICE.
#pragma once
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include "../../include/hexl_b200.h"
#include "hybrid_rotation.h"
#include "internal.h"
#include "numtheory.h"

// ------------------------------------------------------------------ handle types
struct hexl_b200_ntt {
  std::atomic<int> refs{1};
  uint64_t n = 0, q = 0, root = 0;
  int log_n = 0;
  // reference layouts (host), returned by hexl_b200_ntt_table
  std::vector<uint64_t> w, w_precon, inv_seq, inv_seq_precon;
  // tree layouts for the device: node k -> {value, Shoup factor}
  std::vector<hexl_b200::Twiddle> fwd_tree, inv_tree;
  hexl_b200::Twiddle inv_n{}, inv_n_w{};
  std::mutex mu;
  struct Dev {
    hexl_b200::Twiddle* fwd = nullptr;
    hexl_b200::Twiddle* inv = nullptr;
    hexl_b200::Twiddle32* fwd32 = nullptr;  // q < 2^30 only
    hexl_b200::Twiddle32* inv32 = nullptr;
    hexl_b200::NttDeviceParams* params = nullptr;
    hexl_b200::NttDeviceTables view{};
    void free() {  // on the current device, which must be the one the tables live on
      cudaFree(fwd);
      cudaFree(inv);
      cudaFree(fwd32);
      cudaFree(inv32);
      cudaFree(params);
    }
  };
  std::map<int, Dev> dev;  // device ordinal -> uploaded tables
};

// KeySwitch keys resident on the GPUs (hexl_b200_keys_upload): decomp buffers of kcc x key_modulus_size x n
struct hexl_b200_keys {
  std::atomic<int> refs{1};
  uint64_t n = 0, decomp = 0, kcc = 0, kms = 0;
  std::map<int, std::vector<uint64_t*>> dev;  // device ordinal -> decomp device buffers
  // Sharded by RNS modulus (hexl_b200_keys_upload_sharded): shard s owns the RNS moduli [lo, hi) of ONE key switch,
  // holds only their slices of the keys and a private workspace, on device `device` (a device may carry several shards).
  struct Shard {
    int device = 0;
    uint64_t lo = 0, hi = 0;                 // RNS modulus indices (index decomp = the special prime)
    std::vector<uint64_t*> keys;             // [j] -> kcc x (hi - lo) x n
    uint64_t *t_coef = nullptr, *ops = nullptr, *prod = nullptr, *tmp = nullptr, *t_last = nullptr, *res = nullptr,
             *digits = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t gathered = nullptr, special = nullptr;
  };
  std::vector<Shard> shards;
  bool p2p = false;                          // every shard can store straight into every other shard's memory
  std::mutex mu;                             // one sharded switch at a time per handle (the workspaces are per handle)
  // One host thread per shard issues that shard's copies and launches: a switch is ~30 stream operations per shard,
  // and a single issuing thread (240 operations at ~2.7 us on 8 GPUs) was the whole latency of the first version.
  struct Pool {
    std::vector<std::thread> threads;
    std::mutex m;
    std::condition_variable cv_go, cv_done;
    std::function<void(size_t)> job;
    uint64_t generation = 0;
    size_t pending = 0;
    bool stop = false;
    void start(size_t count) {
      for (size_t i = 0; i < count; ++i)
        threads.emplace_back([this, i] {
          uint64_t seen = 0;
          for (;;) {
            std::unique_lock<std::mutex> lk(m);
            cv_go.wait(lk, [&] { return stop || generation != seen; });
            if (stop) return;
            seen = generation;
            auto fn = job;
            lk.unlock();
            fn(i);
            lk.lock();
            if (--pending == 0) cv_done.notify_all();
          }
        });
    }
    void run(std::function<void(size_t)> fn) {
      std::unique_lock<std::mutex> lk(m);
      job = std::move(fn);
      pending = threads.size();
      ++generation;
      cv_go.notify_all();
      cv_done.wait(lk, [&] { return pending == 0; });
    }
    void shutdown() {
      {
        std::lock_guard<std::mutex> lk(m);
        stop = true;
      }
      cv_go.notify_all();
      for (auto& t : threads) t.join();
      threads.clear();
    }
  } pool;
};

namespace hexl_b200 {

extern thread_local std::string t_error;  // the message hexl_b200_last_error returns
extern std::atomic<int> g_debug;          // hexl_b200_set_debug: bounds checks of the inputs

int fail(int code, const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);

#define CU(call)                                         \
  do {                                                   \
    cudaError_t e__ = (call);                            \
    if (e__ != cudaSuccess) return cuda_fail(e__, #call); \
  } while (0)

#define REQUIRE(cond, ...) \
  if (!(cond)) return fail(HEXL_B200_ERR_INVALID_ARG, __VA_ARGS__)

// ------------------------------------------------------------- pointer kinds
enum class Where { Host, Device };
struct PtrInfo {
  Where where;
  int device;            // valid for Device
  bool managed = false;  // unified memory: the host may read it right after the call
};

int classify(const void* p, PtrInfo* out);
// All non-null pointers of a call must live in the same place.
int classify_all(std::initializer_list<const void*> ptrs, PtrInfo* out);

struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  int enter(int dev) {
    CU(cudaGetDevice(&prev));
    if (prev != dev) {
      CU(cudaSetDevice(dev));
      switched = true;
    }
    return 0;
  }
  ~DeviceGuard() {
    if (switched) cudaSetDevice(prev);
  }
};

// The device-pointer branch of an entry point: run() on the device of the call's buffers.  Unified-memory buffers are
// what a host caller of the reference API reads back immediately (hexl_b200_managed_alloc / the ManagedStrategy
// allocator): with no explicit stream the call keeps the reference's synchronous semantics.
template <class Run>
int run_on_device(const PtrInfo& pi, void* stream, Run&& run) {
  DeviceGuard g;
  if (int rc = g.enter(pi.device)) return rc;
  if (int rc = run()) return rc;
  const cudaError_t e = pi.managed && stream == nullptr ? cudaStreamSynchronize(nullptr) : cudaSuccess;
  return e == cudaSuccess ? 0 : cuda_fail(e, "cudaStreamSynchronize");
}

// the devices listed with hexl_b200_set_host_devices, or else the current one
int host_devices(std::vector<int>* out);

// ----------------------------------------------------------- host-pointer staging
// One staging context per device: kSlots rotating {stream, device buffers}, used only through stage_items.
constexpr int kSlots = 3;
constexpr size_t kChunkBytes = 32u << 20;  // per buffer per slot

struct StageCtx {
  std::mutex mu;
  cudaStream_t stream[kSlots] = {};
  u64* buf[kSlots][3] = {};  // [slot][result/in-place a, b, c]
  size_t cap[kSlots][3] = {};
  bool ready = false;
  int init() {
    if (ready) return 0;
    for (int s = 0; s < kSlots; ++s) CU(cudaStreamCreateWithFlags(&stream[s], cudaStreamNonBlocking));
    ready = true;
    return 0;
  }
  int reserve(int slot, int which, size_t bytes) {
    if (cap[slot][which] >= bytes) return 0;
    if (buf[slot][which]) CU(cudaFree(buf[slot][which]));
    buf[slot][which] = nullptr;
    cap[slot][which] = 0;
    CU(cudaMalloc(&buf[slot][which], bytes));
    cap[slot][which] = bytes;
    return 0;
  }
};

StageCtx* stage_for(int dev);
int sync_stage(int dev);  // waits for every slot stream of dev

// Slot i of a device's staging context, as a step of stage_items sees it
struct StageSlot {
  StageCtx* st;
  int i;
  cudaStream_t stream() const { return st->stream[i]; }
  u64* buf(int which) const { return st->buf[i][which]; }
  int reserve(int which, size_t bytes) const { return st->reserve(i, which, bytes); }
};

// The one staging loop of the host-pointer calls.  Items [0, items) are split over devs by contiguous blocks (no
// inter-GPU traffic): device d of nd = min(|devs|, items) takes [items d / nd, items (d + 1) / nd), the rule
// hexl_b200/sharding.py states.  On each device, with it current and its staging lock held, prepare(dev, lo, hi, stage)
// readies what its block needs and returns an error code or stage(step), which runs step(slot, first, count) for
// chunks of at most per_chunk items on the rotating slots, so the copies of one chunk overlap the kernels of its
// neighbours.  Returns the first error, always after waiting for every slot stream of every device of the split:
// copies into the caller's buffers may still be queued when a step fails.
template <class Prepare>
int stage_items(const std::vector<int>& devs, u64 items, u64 per_chunk, Prepare&& prepare) {
  const u64 nd = std::min<u64>(devs.size(), items);
  int rc = 0;
  for (u64 d = 0; d < nd && !rc; ++d) {
    const u64 lo = items * d / nd, hi = items * (d + 1) / nd;
    DeviceGuard g;
    if ((rc = g.enter(devs[d]))) break;
    StageCtx* st = stage_for(devs[d]);
    std::lock_guard<std::mutex> lk(st->mu);
    if ((rc = st->init())) break;
    rc = prepare(devs[d], lo, hi, [&](auto&& step) {
      int slot = 0;
      for (u64 first = lo; first < hi; first += per_chunk, slot = (slot + 1) % kSlots)
        if (int e = step(StageSlot{st, slot}, first, std::min(per_chunk, hi - first))) return e;
      return 0;
    });
  }
  for (u64 d = 0; d < nd; ++d) {
    const int rc2 = sync_stage(devs[d]);
    if (!rc) rc = rc2;
  }
  return rc;
}

// A host-pointer job of `total` elements in whole units of `unit` elements, through stage_items: split over the host
// devices by unit, in chunks of whole units up to kChunkBytes (or of one unit).  a is always present; b optional;
// result may alias a or b.  make(dev, lo, hi, run) prepares device dev for the elements [lo, hi) of the job and
// returns either an error code or run(launch).  launch(dev_result, dev_a, dev_b, off, elems, stream) enqueues the
// kernel(s) for the elements [off, off + elems) of the whole job, staged in the slot's buffer 0 (b in buffer 1); it
// returns a cudaError_t, or an int error code whose message it has already set.
// unit_out (non-zero): only the first unit_out elements of every unit are copied back.
template <class MakeLaunch>
int run_host(u64* result, const u64* a, const u64* b, u64 total, u64 unit, MakeLaunch&& make, u64 unit_out = 0) {
  std::vector<int> devs;
  if (int rc = host_devices(&devs)) return rc;
  const u64 per_chunk = std::max<u64>(1, (kChunkBytes / sizeof(u64)) / unit);
  return stage_items(devs, total / unit, per_chunk, [&](int dev, u64 lo, u64 hi, auto&& stage) {
    return make(dev, lo * unit, hi * unit, [&](auto&& launch) {
      return stage([&](const StageSlot& sl, u64 first, u64 count) -> int {
        const u64 off = first * unit, elems = count * unit;
        const size_t bytes = elems * sizeof(u64);
        if (int rc = sl.reserve(0, bytes)) return rc;
        if (b)
          if (int rc = sl.reserve(1, bytes)) return rc;
        cudaStream_t s = sl.stream();
        CU(cudaMemcpyAsync(sl.buf(0), a + off, bytes, cudaMemcpyHostToDevice, s));
        if (b) CU(cudaMemcpyAsync(sl.buf(1), b + off, bytes, cudaMemcpyHostToDevice, s));
        const auto e = launch(sl.buf(0), sl.buf(0), b ? sl.buf(1) : nullptr, off, elems, s);
        if constexpr (std::is_same_v<std::decay_t<decltype(e)>, int>) {
          if (e) return e;
        } else if (e != cudaSuccess) {
          return cuda_fail(e, "kernel launch");
        }
        if (unit_out && unit_out < unit)
          CU(cudaMemcpy2DAsync(result + off, unit * sizeof(u64), sl.buf(0), unit * sizeof(u64),
                               unit_out * sizeof(u64), count, cudaMemcpyDeviceToHost, s));
        else
          CU(cudaMemcpyAsync(result + off, sl.buf(0), bytes, cudaMemcpyDeviceToHost, s));
        return 0;
      });
    });
  });
}

// ---------------------------------------------------------------- debug checks
// HEXL_CHECK_BOUNDS analogue (check.hpp:33-36): every element < bound.  Device data is checked on the call's
// `stream`, after what the caller queued there before the call, and the check waits for that stream only; a stream
// being captured into a CUDA graph is refused (HEXL_B200_ERR_INVALID_ARG) before anything is queued on it.
int check_bounds(const u64* p, u64 n, u64 bound, const PtrInfo& pi, const char* what, void* stream);
// check_bounds of p against bound when debug checks are on, classifying the call's pointers `all` first
int debug_bounds(const u64* p, u64 n, u64 bound, const char* what, std::initializer_list<const void*> all,
                 void* stream);
// check_bounds of `polys` polynomials of `limbs` blocks of `words` words each, back to back: block i < bound(i)
template <class Bound>
int check_limb_bounds(const u64* p, u64 polys, u64 limbs, u64 words, Bound&& bound, const PtrInfo& pi,
                      const char* what, void* stream) {
  if (!g_debug.load()) return 0;
  for (u64 c = 0; c < polys; ++c)
    for (u64 i = 0; i < limbs; ++i)
      if (int rc = check_bounds(p + (c * limbs + i) * words, words, bound(i), pi, what, stream)) return rc;
  return 0;
}

// A device copy of a constant table, one per table content and device, kept for the life of the process like the NTT
// tables (capi.cu).  The cold path uploads synchronously on a private stream, so it is refused inside a capture of
// user_stream; `what` names the table in that refusal.
int device_table(const std::vector<uint64_t>& tab, int dev, cudaStream_t user_stream, const uint64_t** out,
                 const char* what);

// Little-endian multi-word integers (capi.cu), for the host-side constants of the BFV calls
using Big = std::vector<uint64_t>;
void big_mul(Big& a, uint64_t x);                    // a *= x
void big_add_at(Big& a, size_t word, uint64_t x);    // a += x 2^(64 word)
bool big_le(Big a, Big b);                           // a <= b
uint64_t big_divmod(Big& a, uint64_t d);             // a = floor(a / d); returns the remainder (d >= 1)
uint64_t big_mod(const Big& a, uint64_t m);          // a mod m (m >= 1)

int scratch_pool(cudaMemPool_t* out);  // the library's pool on the current device

struct Scratch {
  cudaStream_t s;
  std::vector<void*> ptrs;
  explicit Scratch(cudaStream_t st) : s(st) {}
  template <class T>
  int get(T** p, size_t count) {
    cudaMemPool_t pool;
    if (int rc = scratch_pool(&pool)) return rc;
    void* v = nullptr;
    CU(cudaMallocFromPoolAsync(&v, count * sizeof(T) + 16, pool, s));
    ptrs.push_back(v);
    *p = static_cast<T*>(v);
    return 0;
  }
  ~Scratch() {
    for (void* v : ptrs) cudaFreeAsync(v, s);
  }
};

inline int floor_log2(uint64_t x) { return 63 - __builtin_clzll(x); }
inline Twiddle make_twiddle(uint64_t v, uint64_t q) { return Twiddle{v, nt::multiply_factor(v, 64, q)}; }
// q and its generalised-Barrett constants, eltwise-mult-mod-internal.hpp:52-69
inline DyadicModulus dyadic_modulus(uint64_t q) {
  const int L = floor_log2(q) + 1;
  return DyadicModulus{q, nt::multiply_factor(1ull << (L - 2), 64, q), L - 2};
}

bool check_ntt_arguments(uint64_t degree, uint64_t q, const char** why);
// Uploads the tables of h to device `dev` (the current device) on first use.  The cold path allocates and
// copies synchronously, so it must not run inside a stream capture: hexl_b200_ntt_prepare warms a handle
// explicitly, and a cold handle met during a capture is reported instead of invalidating the capture.
int device_tables(hexl_b200_ntt* h, int dev, NttDeviceTables* out, cudaStream_t user_stream = nullptr);
// GetNTT(N, modulus) of the reference: one reference to the process-wide handle of (n, q)
int cached_ntt(hexl_b200_ntt** out, uint64_t n, uint64_t q);

struct CachedNtts {  // cached_ntt references held for the length of a call
  std::vector<hexl_b200_ntt*> h;
  explicit CachedNtts(size_t count) : h(count, nullptr) {}
  CachedNtts(const CachedNtts&) = delete;
  ~CachedNtts() {
    for (auto* p : h)
      if (p) hexl_b200_ntt_release(p);
  }
  int load(size_t i, uint64_t n, uint64_t q) { return cached_ntt(&h[i], n, q); }
  hexl_b200_ntt* const* data() const { return h.data(); }
  hexl_b200_ntt* operator[](size_t i) const { return h[i]; }
};

// `count` handles x `group` polynomials each, device pointers on device `dev`, in blocks of kParamBlock handles
// mirrors (inverse only): buffers laid out like `result` that receive the final values too (peer memory: NttMulti::mirror)
int ntt_multi_on_device(bool forward, int dev, hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                        const uint64_t* operand, int out_mf, uint64_t group, cudaStream_t s,
                        const std::vector<uint64_t*>* mirrors = nullptr, bool gather = false,
                        const uint64_t* mul = nullptr);

// `count` moduli x per_mod elements (modulus m owns [m*per_mod, (m+1)*per_mod)) through the same chunked, multi-stream,
// multi-device staging as the single-modulus calls, in whole units of n elements.  The moduli are moduli[m], or the
// handles' when moduli is null; the NTT jobs and PolyMul use the handles' tables.
enum class RnsJob { NttFwd, NttInv, Mult, Add, Sub, PolyMul };
int run_host_rns(RnsJob job, hexl_b200_ntt* const* handles, const uint64_t* moduli, uint64_t count, u64 per_mod, u64 n,
                 int in_mf, int out_mf, u64* result, const u64* a, const u64* b);

int key_switch_check(const void* result, const void* t_target, uint64_t n, uint64_t decomp, uint64_t key_modulus_size,
                     uint64_t rns, uint64_t kcc, const uint64_t* moduli, const uint64_t* modswitch);
bool keys_fit(const hexl_b200_keys* k, uint64_t n, uint64_t decomp, uint64_t kcc, uint64_t key_modulus_size);
// the copies of keys[0, count) on device dev; returns count, or the first r whose handle holds none there
uint64_t keys_on_device(const hexl_b200_keys* const* keys, uint64_t count, int dev,
                        std::vector<const uint64_t* const*>* dk);
int key_switch_on_device(int dev, uint64_t* result, const uint64_t* t_target, uint64_t n, uint64_t decomp,
                         uint64_t key_modulus_size, uint64_t rns, uint64_t kcc, const uint64_t* moduli,
                         const uint64_t* const* d_key_ptrs_host, const uint64_t* modswitch, cudaStream_t s);
// The multiply-accumulate of one step-2 round: ops ([e][j][n], lazily transformed digits under the round's cnt moduli,
// hs[e] their transforms and slots[e] their slots in keys of kms slots) times the keys of each of `elts` switches,
// into prod + r * prod_stride ([e][k][n]); chunked by ks_mac_digits_per_launch.  keys[r][j]: digit j's key of switch
// r; galois_elts[r] (nullptr: none) makes switch r read the digits permuted by pi_g.  accumulate: every launch adds
// into prod, the first digit chunk's too (otherwise that one stores).
// The multiply-accumulate's constants of cnt <= kParamBlock moduli: q, floor(2^64 / q), 2^64 mod q and its Shoup
// factor, and c = slots[e] (0 when slots is null)
KsModuli ks_mac_moduli(const uint64_t* moduli, const uint64_t* slots, uint64_t cnt);
// Digits one multiply-accumulate launch may sum unreduced in 128 bits for the moduli of mods: 64 below 2^60, down to
// 16 just below 2^61
uint64_t ks_mac_digits_per_launch(const KsModuli& mods, uint64_t count);
int ks_mac_products(hexl_b200_ntt* const* hs, const uint64_t* slots, uint64_t cnt, uint64_t kms, const uint64_t* ops,
                    uint64_t decomp, uint64_t n, uint64_t kcc, uint64_t* prod, uint64_t prod_stride,
                    const uint64_t* const* const* keys, const uint64_t* galois_elts, uint64_t elts, cudaStream_t s,
                    bool accumulate = false);
int key_switch_elts_on_device(int dev, uint64_t* const* results, const uint64_t* t_target, uint64_t n, uint64_t decomp,
                              uint64_t key_modulus_size, uint64_t rns, uint64_t kcc, const uint64_t* moduli,
                              const uint64_t* const* const* d_key_ptrs, const uint64_t* galois_elts, uint64_t elts,
                              const uint64_t* modswitch, cudaStream_t s);
// run(dev, device result block, device input block, the key handles' copies on dev, stream): one ciphertext's switch,
// called for the ciphertexts in order, 0 to batch - 1.
// prepare(dev) (optional) runs once on each device of the split, with it current, before its first ciphertext.
// in2 (optional): a second input of in_words words per ciphertext, copied into the input block after the first.
using HostSwitch = std::function<int(int, uint64_t*, uint64_t*, const uint64_t* const* const*, cudaStream_t)>;
int key_switch_host_batch(uint64_t* result, uint64_t res_words, bool result_in, const uint64_t* in, uint64_t in_words,
                          uint64_t buf_words, const hexl_b200_keys* const* keys, uint64_t num_keys, uint64_t batch,
                          const HostSwitch& run, const std::function<int(int)>& prepare = nullptr,
                          const uint64_t* in2 = nullptr);

// Fast base conversion of `polys` polynomials from the moduli `from` into the moduli `to` (capi_hybrid.cu): plain
// (round = false), rounded (the CKKS mod-down) or, with plain_modulus = tau != 0, t-corrected (the BGV mod-down and
// modulus switch); strides as launch_base_conv, device pointers on the current device, asynchronous on s.
int base_convert_on_device(uint64_t* result, uint64_t res_limb, uint64_t res_poly, const uint64_t* operand,
                           uint64_t op_limb, uint64_t op_poly, uint64_t n, uint64_t polys, const uint64_t* from,
                           uint64_t from_count, const uint64_t* to, uint64_t to_count, bool round, cudaStream_t s,
                           uint64_t plain_modulus = 0);
// The BGV refusal of a plain modulus: outside [2, 2^61), or sharing a factor with one of moduli[0, count)
int bgv_plain_modulus_check(uint64_t plain_modulus, const uint64_t* moduli, uint64_t count);

// BFV multiplication by BEHZ (capi_bfv.cu).  The refusals of hexl_b200_bfv_multiply that do not depend on the
// buffers' memory: null pointers, shapes, moduli, plain modulus and the bound on Bsk.
bool behz_bound_holds(uint64_t n, uint64_t t, const uint64_t* q, uint64_t l, const uint64_t* b, uint64_t k,
                      uint64_t m_sk);
int bfv_check(const void* result, const void* ct1, const void* ct2, uint64_t n, const uint64_t* moduli, uint64_t l,
              const uint64_t* base_b, uint64_t k, uint64_t m_sk, uint64_t t);
// What one call needs: the transforms of Q u Bsk (l + k + 1 moduli, Q first, then b_0..b_{k-1}, m_sk) and the
// constant tables of the two kernels (internal.h), uploaded to each device on first use
struct BfvPlan {
  uint64_t n = 0, l = 0, k = 0;
  std::vector<uint64_t> mods, ext_tab, scale_tab;
  CachedNtts h;
  explicit BfvPlan(size_t count) : h(count) {}
};
int bfv_plan(BfvPlan* plan, uint64_t n, const uint64_t* moduli, uint64_t l, const uint64_t* base_b, uint64_t k,
             uint64_t m_sk, uint64_t t);
// One pair (ct1, ct2: two components of l limbs, coefficient form, device memory; ct1 == ct2 squares) into d0, d1, d2
// at out.p[0..2] (l limbs each), asynchronous on s: the extension launches, one forward transform of the lifted
// inputs, the tensor, one inverse transform and the scaling launch.  Scratch: 7 (or 5 when squaring) x (l + k + 1) x n
// words.
int bfv_product_on_device(int dev, const BfvPlan& plan, const BfvOutputs& out, const uint64_t* ct1,
                          const uint64_t* ct2, cudaStream_t s);

}  // namespace hexl_b200
