// extern "C" boundary of libhexl_b200.so (declared in include/hexl_b200.h).
//
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
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <thread>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <numeric>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/hexl_b200.h"
#include "internal.h"
#include "numtheory.h"

using namespace hexl_b200;

namespace hexl_b200 {
static std::atomic<uint64_t> g_launches{0};
void count_launch(unsigned n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
uint64_t launches_so_far() { return g_launches.load(std::memory_order_relaxed); }
}  // namespace hexl_b200

// ------------------------------------------------------------------ handle type
struct hexl_b200_ntt {
  std::atomic<int> refs{1};
  uint64_t n = 0, q = 0, root = 0;
  int log_n = 0;
  // reference layouts (host), returned by hexl_b200_ntt_table
  std::vector<uint64_t> w, w_precon, inv_seq, inv_seq_precon;
  // tree layouts for the device: node k -> {value, Shoup factor}
  std::vector<Twiddle> fwd_tree, inv_tree;
  Twiddle inv_n{}, inv_n_w{};
  std::mutex mu;
  struct Dev {
    Twiddle* fwd = nullptr;
    Twiddle* inv = nullptr;
    Twiddle32* fwd32 = nullptr;  // q < 2^30 only
    Twiddle32* inv32 = nullptr;
    NttDeviceParams* params = nullptr;
    NttDeviceTables view{};
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

extern "C" {
static void free_shards(hexl_b200_keys* k);
}

namespace {

thread_local std::string t_error;
std::atomic<int> g_debug{0};
std::mutex g_cfg_mu;
std::vector<int> g_host_devices;  // empty = current device only

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  t_error = buf;
  return code;
}

int cuda_fail(cudaError_t e, const char* what) {
  if (e == cudaErrorNoDevice || e == cudaErrorInsufficientDriver || e == cudaErrorInitializationError)
    return fail(HEXL_B200_ERR_NO_DEVICE, "%s: no usable CUDA device (%s)", what, cudaGetErrorString(e));
  return fail(HEXL_B200_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
}

#define CU(call)                                         \
  do {                                                   \
    cudaError_t e__ = (call);                            \
    if (e__ != cudaSuccess) return cuda_fail(e__, #call); \
  } while (0)

// ------------------------------------------------------------- pointer kinds
enum class Where { Host, Device };
struct PtrInfo {
  Where where;
  int device;            // valid for Device
  bool managed = false;  // unified memory: the host may read it right after the call
};

int classify(const void* p, PtrInfo* out) {
  cudaPointerAttributes a;
  cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return cuda_fail(e, "cudaPointerGetAttributes");
  }
  if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) {
    out->where = Where::Device;
    out->device = a.device;
    out->managed = a.type == cudaMemoryTypeManaged;
  } else {
    out->where = Where::Host;
    out->device = -1;
  }
  return 0;
}

// All non-null pointers of a call must live in the same place.
int classify_all(std::initializer_list<const void*> ptrs, PtrInfo* out) {
  bool have = false;
  for (const void* p : ptrs) {
    if (!p) continue;
    PtrInfo pi;
    int rc = classify(p, &pi);
    if (rc) return rc;
    if (!have) {
      *out = pi;
      have = true;
    } else if (pi.where == out->where && pi.where == Where::Device && pi.device == out->device) {
      out->managed = out->managed || pi.managed;
    } else if (pi.where != out->where || (pi.where == Where::Device && pi.device != out->device)) {
      return fail(HEXL_B200_ERR_MIXED_POINTERS, "host and device pointers (or two devices) mixed in one call");
    }
  }
  return 0;
}

// Unified-memory buffers are what a host caller of the reference API reads back
// immediately (hexl_b200_managed_alloc / the ManagedStrategy allocator): with no
// explicit stream the call keeps the reference's synchronous semantics.
int finish_device_call(const PtrInfo& pi, void* stream) {
  if (pi.managed && stream == nullptr) {
    cudaError_t e = cudaStreamSynchronize(nullptr);
    if (e != cudaSuccess) return cuda_fail(e, "cudaStreamSynchronize");
  }
  return 0;
}

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

// ----------------------------------------------------------- host-pointer staging
// One staging context per device: kSlots rotating {stream, device buffers}.
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

std::mutex g_stage_mu;
std::map<int, StageCtx*> g_stage;

StageCtx* stage_for(int dev) {
  std::lock_guard<std::mutex> lk(g_stage_mu);
  auto it = g_stage.find(dev);
  if (it == g_stage.end()) it = g_stage.emplace(dev, new StageCtx()).first;
  return it->second;
}

// A host-pointer job: `total` elements, processed in chunks that are multiples
// of `unit` elements.  a is always present; b optional; result may alias a or b.
// launch(dev_result, dev_a, dev_b, off, elems, stream) enqueues the kernel(s) for the
// elements [off, off + elems) of the whole job (`base` = offset of this device's block);
// it returns a cudaError_t, or an int error code whose message it has already set.
// unit_out (non-zero): only the first unit_out elements of every unit are copied back.
template <class Launch>
int run_host_on_device(int dev, u64* result, const u64* a, const u64* b, u64 total, u64 unit,
                       Launch&& launch, bool wait, u64 base = 0, u64 unit_out = 0) {
  DeviceGuard g;
  if (int rc = g.enter(dev)) return rc;
  StageCtx* st = stage_for(dev);
  std::lock_guard<std::mutex> lk(st->mu);
  if (int rc = st->init()) return rc;
  u64 chunk = (kChunkBytes / sizeof(u64)) / unit * unit;
  if (chunk == 0) chunk = unit;
  int slot = 0;
  for (u64 off = 0; off < total; off += chunk, slot = (slot + 1) % kSlots) {
    const u64 elems = (total - off < chunk) ? total - off : chunk;
    const size_t bytes = elems * sizeof(u64);
    if (int rc = st->reserve(slot, 0, bytes)) return rc;
    if (b)
      if (int rc = st->reserve(slot, 1, bytes)) return rc;
    cudaStream_t s = st->stream[slot];
    CU(cudaMemcpyAsync(st->buf[slot][0], a + off, bytes, cudaMemcpyHostToDevice, s));
    if (b) CU(cudaMemcpyAsync(st->buf[slot][1], b + off, bytes, cudaMemcpyHostToDevice, s));
    const auto e = launch(st->buf[slot][0], st->buf[slot][0], b ? st->buf[slot][1] : nullptr, base + off, elems, s);
    if constexpr (std::is_same_v<std::decay_t<decltype(e)>, int>) {
      if (e) return e;
    } else if (e != cudaSuccess) {
      return cuda_fail(e, "kernel launch");
    }
    if (unit_out && unit_out < unit)
      CU(cudaMemcpy2DAsync(result + off, unit * sizeof(u64), st->buf[slot][0], unit * sizeof(u64),
                           unit_out * sizeof(u64), elems / unit, cudaMemcpyDeviceToHost, s));
    else
      CU(cudaMemcpyAsync(result + off, st->buf[slot][0], bytes, cudaMemcpyDeviceToHost, s));
  }
  if (wait)
    for (int s = 0; s < kSlots; ++s) CU(cudaStreamSynchronize(st->stream[s]));
  return 0;
}

int sync_stage(int dev) {
  DeviceGuard g;
  if (int rc = g.enter(dev)) return rc;
  StageCtx* st = stage_for(dev);
  std::lock_guard<std::mutex> lk(st->mu);
  if (!st->ready) return 0;
  for (int s = 0; s < kSlots; ++s) CU(cudaStreamSynchronize(st->stream[s]));
  return 0;
}

std::vector<int> host_devices() {
  std::lock_guard<std::mutex> lk(g_cfg_mu);
  return g_host_devices;
}

// Split a host-pointer job over the configured devices by contiguous blocks of
// whole units (no inter-GPU traffic), enqueue everything, then wait.
template <class MakeLaunch>
int run_host(u64* result, const u64* a, const u64* b, u64 total, u64 unit, MakeLaunch&& make, u64 unit_out = 0) {
  std::vector<int> devs = host_devices();
  if (devs.empty() || total / unit < 2) {
    int cur = 0;
    CU(cudaGetDevice(&cur));
    if (!devs.empty()) cur = devs[0];
    auto launch = make(cur, (u64)0, total);
    if (!launch.ok) return launch.rc;
    return run_host_on_device(cur, result, a, b, total, unit, launch, true, 0, unit_out);
  }
  const u64 units = total / unit;
  const u64 ndev = devs.size() < units ? devs.size() : units;
  int rc = 0;
  for (u64 d = 0; d < ndev && !rc; ++d) {
    const u64 lo = units * d / ndev * unit, hi = units * (d + 1) / ndev * unit;
    auto launch = make(devs[d], lo, hi);
    if (!launch.ok) {
      rc = launch.rc;  // fall through: copies already enqueued on other devices still target `result`
      break;
    }
    rc = run_host_on_device(devs[d], result + lo, a + lo, b ? b + lo : nullptr, hi - lo, unit, launch, false, lo,
                            unit_out);
  }
  for (u64 d = 0; d < ndev; ++d) {
    int rc2 = sync_stage(devs[d]);
    if (!rc) rc = rc2;
  }
  return rc;
}

// ---------------------------------------------------------------- debug checks
__global__ void bounds_kernel(const u64* p, u64 n, u64 bound, int* flag) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  bool bad = false;
  for (; i < n; i += stride) bad |= p[i] >= bound;
  if (bad) atomicExch(flag, 1);
}

// HEXL_CHECK_BOUNDS analogue (check.hpp:33-36): every element < bound
int check_bounds(const u64* p, u64 n, u64 bound, const PtrInfo& pi, const char* what) {
  if (!g_debug.load() || !p) return 0;
  if (pi.where == Where::Host) {
    for (u64 i = 0; i < n; ++i)
      if (p[i] >= bound) return fail(HEXL_B200_ERR_INVALID_ARG, "%s: element %llu exceeds bound", what, (unsigned long long)i);
    return 0;
  }
  DeviceGuard g;
  if (int rc = g.enter(pi.device)) return rc;
  int* flag = nullptr;
  CU(cudaMalloc(&flag, sizeof(int)));
  CU(cudaMemset(flag, 0, sizeof(int)));
  bounds_kernel<<<296, 256>>>(p, n, bound, flag);
  count_launch();
  int h = 0;
  cudaError_t e = cudaMemcpy(&h, flag, sizeof(int), cudaMemcpyDeviceToHost);
  cudaFree(flag);
  if (e != cudaSuccess) return cuda_fail(e, "bounds check");
  if (h) return fail(HEXL_B200_ERR_INVALID_ARG, "%s: an element exceeds its bound", what);
  return 0;
}

// --------------------------------------------------------------- NTT tables
int floor_log2(uint64_t x) { return 63 - __builtin_clzll(x); }
DyadicModulus dyadic_modulus(uint64_t q);

bool check_ntt_arguments(uint64_t degree, uint64_t q, const char** why) {
  // NTT::CheckArguments, hexl/ntt/ntt-internal.cpp:171-186
  if (degree < 2 || (degree & (degree - 1))) { *why = "degree is not a power of 2 (>= 2)"; return false; }
  if (degree > (1ull << 20)) { *why = "degree should be at most 2^20"; return false; }
  if (q > (1ull << 62)) { *why = "modulus should be at most 2^62"; return false; }
  if (q % (2 * degree) != 1) { *why = "modulus mod 2n != 1"; return false; }
  if (!nt::is_prime(q)) { *why = "modulus is not prime"; return false; }
  return true;
}

Twiddle make_twiddle(uint64_t v, uint64_t q) { return Twiddle{v, nt::multiply_factor(v, 64, q)}; }
Twiddle32 make_twiddle32(uint64_t v, uint64_t q) { return Twiddle32{(uint32_t)v, (uint32_t)((v << 32) / q)}; }

// hexl/ntt/ntt-internal.cpp:54-169 restated: psi^i goes to slot bitrev(i); the
// inverse powers are additionally listed in the order the reference's inverse
// transform consumes them (m = N/2 groups first, ..., m = 1 last).
void build_tables(hexl_b200_ntt* h) {
  const uint64_t n = h->n, q = h->q;
  h->w.assign(n, 0);
  h->w_precon.assign(n, 0);
  h->inv_seq.assign(n, 0);
  h->inv_seq_precon.assign(n, 0);
  h->fwd_tree.assign(n, Twiddle{0, 0});
  h->inv_tree.assign(n, Twiddle{0, 0});
  const uint64_t root_inv = nt::inverse_mod(h->root, q);
  uint64_t pw = 1, ipw = 1;
  for (uint64_t i = 0; i < n; ++i) {
    const uint64_t slot = nt::reverse_bits(i, h->log_n);
    h->fwd_tree[slot] = make_twiddle(pw, q);
    h->inv_tree[slot] = make_twiddle(ipw, q);  // (psi^i)^-1 = (psi^-1)^i
    pw = nt::mul_mod(pw, h->root, q);
    ipw = nt::mul_mod(ipw, root_inv, q);
  }
  for (uint64_t k = 0; k < n; ++k) {
    h->w[k] = h->fwd_tree[k].w;
    h->w_precon[k] = h->fwd_tree[k].wp;
  }
  uint64_t pos = 0;
  h->inv_seq[pos] = h->inv_tree[0].w;
  h->inv_seq_precon[pos++] = h->inv_tree[0].wp;
  for (uint64_t m = n >> 1; m > 0; m >>= 1)
    for (uint64_t i = 0; i < m; ++i, ++pos) {
      h->inv_seq[pos] = h->inv_tree[m + i].w;
      h->inv_seq_precon[pos] = h->inv_tree[m + i].wp;
    }
  const uint64_t inv_n = nt::inverse_mod(n, q);
  h->inv_n = make_twiddle(inv_n, q);
  h->inv_n_w = make_twiddle(nt::mul_mod(inv_n, h->inv_tree[1].w, q), q);
}

// Uploads the tables of h to device `dev` (the current device) on first use.  The cold path allocates and
// copies synchronously, so it must not run inside a stream capture: hexl_b200_ntt_prepare warms a handle
// explicitly, and a cold handle met during a capture is reported instead of invalidating the capture.
int device_tables(hexl_b200_ntt* h, int dev, NttDeviceTables* out, cudaStream_t user_stream = nullptr) {
  std::lock_guard<std::mutex> lk(h->mu);
  auto it = h->dev.find(dev);
  if (it == h->dev.end()) {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    // (the legacy default stream cannot be captured, and querying it during someone else's capture would
    // invalidate that capture)
    if (user_stream && cudaStreamIsCapturing(user_stream, &cap) != cudaSuccess) cudaGetLastError();
    if (cap != cudaStreamCaptureStatusNone)
      return fail(HEXL_B200_ERR_INVALID_ARG,
                  "NTT tables for this device are not uploaded yet and the stream is being captured: call "
                  "hexl_b200_ntt_prepare (or run the call once) before capturing");
    hexl_b200_ntt::Dev d;
    auto release = [&d]() {
      cudaFree(d.fwd);
      cudaFree(d.inv);
      cudaFree(d.fwd32);
      cudaFree(d.inv32);
      cudaFree(d.params);
    };
#define CU_T(call)                                        \
  do {                                                    \
    cudaError_t e__ = (call);                             \
    if (e__ != cudaSuccess) {                             \
      release();                                          \
      return cuda_fail(e__, #call);                       \
    }                                                     \
  } while (0)
    const size_t bytes = h->n * sizeof(Twiddle);
    CU_T(cudaMalloc(&d.fwd, bytes));
    CU_T(cudaMalloc(&d.inv, bytes));
    CU_T(cudaMemcpy(d.fwd, h->fwd_tree.data(), bytes, cudaMemcpyHostToDevice));
    CU_T(cudaMemcpy(d.inv, h->inv_tree.data(), bytes, cudaMemcpyHostToDevice));
    if (h->q < kSmallModulusLimit) {
      std::vector<Twiddle32> f32(h->n), i32(h->n);
      for (uint64_t k = 0; k < h->n; ++k) {
        f32[k] = make_twiddle32(h->fwd_tree[k].w, h->q);
        i32[k] = make_twiddle32(h->inv_tree[k].w, h->q);
      }
      CU_T(cudaMalloc(&d.fwd32, h->n * sizeof(Twiddle32)));
      CU_T(cudaMalloc(&d.inv32, h->n * sizeof(Twiddle32)));
      CU_T(cudaMemcpy(d.fwd32, f32.data(), h->n * sizeof(Twiddle32), cudaMemcpyHostToDevice));
      CU_T(cudaMemcpy(d.inv32, i32.data(), h->n * sizeof(Twiddle32), cudaMemcpyHostToDevice));
    }
    const DyadicModulus pm = dyadic_modulus(h->q);
    NttDeviceParams hp{d.fwd, d.inv, h->q, nt::multiply_factor(1, 64, h->q), h->inv_n, h->inv_n_w, pm.mu, pm.shift};
    CU_T(cudaMalloc(&d.params, sizeof(NttDeviceParams)));
    CU_T(cudaMemcpy(d.params, &hp, sizeof(NttDeviceParams), cudaMemcpyHostToDevice));
    // A pageable-source cudaMemcpy may return once the data sits in the driver's staging buffer; the
    // kernels that read these tables run on non-blocking streams, which are not ordered against the
    // legacy default stream.  Wait for the DMA to land before anybody can launch on the tables.
    CU_T(cudaDeviceSynchronize());
#undef CU_T
    NttDeviceTables& t = d.view;  // everything a launch needs, computed once
    t.dparams = d.params;
    t.fwd = d.fwd;
    t.inv = d.inv;
    t.fwd32 = d.fwd32;
    t.inv32 = d.inv32;
    t.inv_n32 = h->q < kSmallModulusLimit ? make_twiddle32(h->inv_n.w, h->q) : Twiddle32{0, 0};
    t.inv_n_w32 = h->q < kSmallModulusLimit ? make_twiddle32(h->inv_n_w.w, h->q) : Twiddle32{0, 0};
    t.n = h->n;
    t.log_n = h->log_n;
    t.q = h->q;
    t.mu = hp.mu;
    t.inv_n = h->inv_n;
    t.inv_n_w = h->inv_n_w;
    it = h->dev.emplace(dev, d).first;
  }
  *out = it->second.view;
  return 0;
}

int create_common(hexl_b200_ntt** out, uint64_t degree, uint64_t q, uint64_t root, bool have_root) {
  if (!out) return fail(HEXL_B200_ERR_INVALID_ARG, "out == nullptr");
  *out = nullptr;
  const char* why = "";
  if (!check_ntt_arguments(degree, q, &why)) return fail(HEXL_B200_ERR_INVALID_ARG, "NTT(%llu, %llu): %s",
                                                         (unsigned long long)degree, (unsigned long long)q, why);
  if (!have_root) root = nt::minimal_primitive_root(2 * degree, q);
  if (!nt::is_primitive_root(root, 2 * degree, q))
    return fail(HEXL_B200_ERR_INVALID_ARG, "%llu is not a primitive 2*%llu'th root of unity",
                (unsigned long long)root, (unsigned long long)degree);
  hexl_b200_ntt* h = new (std::nothrow) hexl_b200_ntt();
  if (!h) return fail(HEXL_B200_ERR_ALLOC, "out of host memory");
  h->n = degree;
  h->q = q;
  h->root = root;
  h->log_n = floor_log2(degree);
  build_tables(h);
  *out = h;
  return 0;
}

struct NttLaunch {
  bool ok = true;
  int rc = 0;
  NttDeviceTables t{};
  bool forward = true;
  int in_mf = 1, out_mf = 1;
  u64 n = 0;
  cudaError_t operator()(u64* r, const u64* a, const u64*, u64 /*off*/, u64 elems, cudaStream_t s) const {
    return forward ? launch_ntt_forward(t, r, a, in_mf, out_mf, elems / n, s)
                   : launch_ntt_inverse(t, r, a, in_mf, out_mf, elems / n, s);
  }
};

int ntt_compute(bool forward, hexl_b200_ntt* h, uint64_t* result, const uint64_t* operand,
                uint64_t in_mf, uint64_t out_mf, uint64_t batch, void* stream) {
  // checks of ntt-internal.cpp:191-200 (forward) / :255-262 (inverse)
  if (!h) return fail(HEXL_B200_ERR_INVALID_ARG, "ntt handle == nullptr");
  if (!result) return fail(HEXL_B200_ERR_INVALID_ARG, "result == nullptr");
  if (!operand) return fail(HEXL_B200_ERR_INVALID_ARG, "operand == nullptr");
  if (forward) {
    if (!(in_mf == 1 || in_mf == 2 || in_mf == 4))
      return fail(HEXL_B200_ERR_INVALID_ARG, "input_mod_factor must be 1, 2 or 4; got %llu", (unsigned long long)in_mf);
    if (!(out_mf == 1 || out_mf == 4))
      return fail(HEXL_B200_ERR_INVALID_ARG, "output_mod_factor must be 1 or 4; got %llu", (unsigned long long)out_mf);
  } else {
    if (!(in_mf == 1 || in_mf == 2))
      return fail(HEXL_B200_ERR_INVALID_ARG, "input_mod_factor must be 1 or 2; got %llu", (unsigned long long)in_mf);
    if (!(out_mf == 1 || out_mf == 2))
      return fail(HEXL_B200_ERR_INVALID_ARG, "output_mod_factor must be 1 or 2; got %llu", (unsigned long long)out_mf);
  }
  if (batch == 0) return 0;
  PtrInfo pi;
  if (int rc = classify_all({result, operand}, &pi)) return rc;
  if (int rc = check_bounds(operand, batch * h->n, h->q * in_mf, pi, "operand")) return rc;
  if (pi.where == Where::Device) {
    DeviceGuard g;
    if (int rc = g.enter(pi.device)) return rc;
    NttDeviceTables t;
    if (int rc = device_tables(h, pi.device, &t, (cudaStream_t)stream)) return rc;
    cudaError_t e = forward ? launch_ntt_forward(t, result, operand, (int)in_mf, (int)out_mf, batch, (cudaStream_t)stream)
                            : launch_ntt_inverse(t, result, operand, (int)in_mf, (int)out_mf, batch, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "NTT launch");
    return finish_device_call(pi, stream);
  }
  return run_host(result, operand, nullptr, batch * h->n, h->n, [&](int dev, u64, u64) {
    NttLaunch L;
    L.forward = forward;
    L.in_mf = (int)in_mf;
    L.out_mf = (int)out_mf;
    L.n = h->n;
    DeviceGuard g;
    int rc = g.enter(dev);
    if (!rc) rc = device_tables(h, dev, &L.t);
    if (rc) {
      L.ok = false;
      L.rc = rc;
    }
    return L;
  });
}

// ------------------------------------------------------------------ eltwise
struct EltLaunch {
  bool ok = true;
  int rc = 0;
  EltOp op;
  EltParams p;
  cudaError_t operator()(u64* r, const u64* a, const u64* b, u64 /*off*/, u64 elems, cudaStream_t s) const {
    EltParams q = p;
    q.result = r;
    q.a = a;
    q.b = b;
    q.n = elems;
    return launch_eltwise(op, q, s);
  }
};

int eltwise_dispatch(EltOp op, EltParams p, void* stream) {
  if (p.n == 0) return fail(HEXL_B200_ERR_INVALID_ARG, "Require n != 0");
  PtrInfo pi;
  if (int rc = classify_all({p.result, p.a, p.b}, &pi)) return rc;
  if (pi.where == Where::Device) {
    DeviceGuard g;
    if (int rc = g.enter(pi.device)) return rc;
    cudaError_t e = launch_eltwise(op, p, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_fail(e, "eltwise launch");
    return finish_device_call(pi, stream);
  }
  return run_host(p.result, p.a, p.b, p.n, 1, [&](int, u64, u64) {
    EltLaunch L;
    L.op = op;
    L.p = p;
    return L;
  });
}

#define REQUIRE(cond, ...) \
  if (!(cond)) return fail(HEXL_B200_ERR_INVALID_ARG, __VA_ARGS__)

// ------------------------------------------------------------ NTT cache
// GetNTT(N, modulus) of the reference (hexl/include/hexl/experimental/seal/ntt-cache.hpp:27-53)
std::mutex g_cache_mu;
std::map<std::pair<uint64_t, uint64_t>, hexl_b200_ntt*> g_ntt_cache;

int cached_ntt(hexl_b200_ntt** out, uint64_t n, uint64_t q) {
  std::lock_guard<std::mutex> lk(g_cache_mu);
  auto key = std::make_pair(n, q);
  auto it = g_ntt_cache.find(key);
  if (it == g_ntt_cache.end()) {
    hexl_b200_ntt* h = nullptr;
    if (int rc = create_common(&h, n, q, 0, false)) return rc;
    it = g_ntt_cache.emplace(key, h).first;  // the cache keeps its own reference for the process lifetime
  }
  it->second->refs.fetch_add(1);
  *out = it->second;
  return 0;
}

// Stream-ordered scratch memory for the composites, from a pool of our own per device
// (release threshold = keep everything: a KeySwitch re-uses the same few buffers call
// after call; the process-wide default pool, which other libraries may tune, is left alone).
std::mutex g_pool_mu;
std::map<int, cudaMemPool_t> g_pools;
int scratch_pool(cudaMemPool_t* out) {
  int dev = 0;
  CU(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(g_pool_mu);
  auto it = g_pools.find(dev);
  if (it == g_pools.end()) {
    cudaMemPoolProps props = {};
    props.allocType = cudaMemAllocationTypePinned;
    props.handleTypes = cudaMemHandleTypeNone;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    cudaMemPool_t pool;
    CU(cudaMemPoolCreate(&pool, &props));
    uint64_t keep = ~0ull;
    CU(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
    it = g_pools.emplace(dev, pool).first;
  }
  *out = it->second;
  return 0;
}

}  // namespace
namespace hexl_b200 {
cudaError_t scratch_alloc_async(void** p, size_t bytes, cudaStream_t stream) {
  cudaMemPool_t pool;
  if (scratch_pool(&pool)) return cudaErrorMemoryAllocation;
  return cudaMallocFromPoolAsync(p, bytes, pool, stream);
}
void scratch_free_async(void* p, cudaStream_t stream) {
  if (p) cudaFreeAsync(p, stream);
}
}  // namespace hexl_b200
namespace {

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

DyadicModulus dyadic_modulus(uint64_t q) {
  const int L = floor_log2(q) + 1;
  return DyadicModulus{q, nt::multiply_factor(1ull << (L - 2), 64, q), L - 2};
}

int dyadic_on_device(uint64_t* result, const uint64_t* op1, const uint64_t* op2, uint64_t n, const uint64_t* moduli,
                     uint64_t num_moduli, cudaStream_t s) {
  for (uint64_t first = 0; first < num_moduli; first += kParamBlock) {
    const uint64_t count = std::min<uint64_t>(kParamBlock, num_moduli - first);
    DyadicModuli mods;
    for (uint64_t i = 0; i < count; ++i) mods.m[i] = dyadic_modulus(moduli[first + i]);
    cudaError_t e = launch_dyadic_multiply(result, op1, op2, n, num_moduli, first, count, mods, s);
    if (e != cudaSuccess) return cuda_fail(e, "DyadicMultiply launch");
  }
  return 0;
}

int ntt_multi_on_device(bool forward, int dev, hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                        const uint64_t* operand, int out_mf, uint64_t group, cudaStream_t s,
                        const std::vector<uint64_t*>* mirrors = nullptr, bool gather = false,
                        const uint64_t* mul = nullptr);

// Digits one ks_mac_kernel launch may add up for the `count` moduli of `mods`.  Each product is a lazy forward-transform
// output (< 4q) times a key word (< q) and the kernel sums them unreduced in 128 bits, so at most
// (2^128 - 1) / ((4q - 1)(q - 1)) of them fit for the largest q: the whole 64-entry key block below 2^60, down to 16
// just below 2^61.  Launches beyond the first add their reduced sums into prod (the `accumulate` flag).
static uint64_t ks_mac_digits_per_launch(const KsModuli& mods, uint64_t count) {
  uint64_t q = 0;
  for (uint64_t e = 0; e < count; ++e) q = std::max(q, mods.m[e].q);
  const unsigned __int128 largest_product = (unsigned __int128)(4 * q - 1) * (q - 1);
  return (uint64_t)std::min<unsigned __int128>(kParamBlock, ~(unsigned __int128)0 / largest_product);
}

// Mod-down of `group` polynomials by their last modulus q_last = h_last->q, every step batched over the target moduli
// (key-switch-internal.cpp:134-198; SEAL's divide_and_round_q_last_ntt_inplace):
//   t_last: the polynomials' last part in NTT form, [p][n] contiguous, < 2 q_last; inverse-transformed in place;
//   for each block of at most kParamBlock target moduli i (h_targets[i], q_i, factors[i] = q_last^-1 mod q_i):
//     ks_round into tmp ([e][p][n], room for one block), one lazy multi-modulus forward transform of tmp, and
//     ks_finish: result[n (res_stride p + i) + l] (+)= (in - tmp) * factors[i] mod q_i.
// `in`, in_like_result and accumulate are those of launch_ks_finish (modulus-major `in` starts at target 0).
// About 1 + 3 launches per block, whatever `group` is.  Device pointers on the current device, asynchronous on s.
int mod_down_on_device(int dev, uint64_t* result, uint64_t res_stride, const uint64_t* in, bool in_like_result,
                       bool accumulate, uint64_t* t_last, uint64_t* tmp, uint64_t n, uint64_t group,
                       hexl_b200_ntt* h_last, hexl_b200_ntt* const* h_targets, const uint64_t* target_moduli,
                       const uint64_t* factors, uint64_t targets, cudaStream_t s) {
#define LAUNCH(expr)                                                    \
  do {                                                                  \
    cudaError_t e__ = (expr);                                           \
    if (e__ != cudaSuccess) return cuda_fail(e__, "mod-down: " #expr); \
  } while (0)
  const uint64_t q_last = h_last->q, mu_last = nt::multiply_factor(1, 64, q_last);
  {
    NttDeviceTables tl;
    if (int rc = device_tables(h_last, dev, &tl, s)) return rc;
    LAUNCH(launch_ntt_inverse(tl, t_last, t_last, 2, 2, group, s));
  }
  for (uint64_t i0 = 0; i0 < targets; i0 += kParamBlock) {
    const uint64_t cnt = std::min<uint64_t>(kParamBlock, targets - i0);
    KsModuli round_mods, fin_mods;
    for (uint64_t e = 0; e < cnt; ++e) {
      const uint64_t qi = target_moduli[i0 + e], mu_i = nt::multiply_factor(1, 64, qi);
      round_mods.m[e] = KsModulus{qi, mu_i, qi - ((q_last >> 1) % qi), 0, 0};
      const Twiddle ms = make_twiddle(factors[i0 + e] % qi, qi);
      fin_mods.m[e] = KsModulus{qi, mu_i, ms.w, ms.wp, 0};
    }
    LAUNCH(launch_ks_round(tmp, t_last, n, group, q_last, mu_last, cnt, round_mods, s));
    if (int rc = ntt_multi_on_device(true, dev, h_targets + i0, cnt, tmp, tmp, 4, group, s)) return rc;
    LAUNCH(launch_ks_finish(result, in_like_result ? in : in + i0 * group * n, tmp, n, group, res_stride, i0, cnt,
                            fin_mods, in_like_result, accumulate, s));
  }
#undef LAUNCH
  return 0;
}

// key-switch-internal.cpp:25-201 as a short chain of launches on the caller's stream, every
// step batched over the RNS moduli (multi-modulus NTTs + the glue kernels of seal.cu): about a
// dozen launches whatever the number of moduli, instead of ~10 per modulus.  Every pointer is
// a device pointer on the current device.  Scratch layouts are [modulus][digit or component][n].
// `elts` switches share the digits t_target, decomposed once (steps 1 and 2's transforms): switch r multiplies them
// with the keys d_key_ptrs[r] and accumulates into results[r].  galois_elts (the hoisted rotations; nullptr: none)
// makes switch r read the transformed digits permuted by pi_{galois_elts[r]}.  Scratch: one round of transformed
// digits plus elts x rns x kcc x n words of products.
static int key_switch_elts_on_device(int dev, uint64_t* const* results, const uint64_t* t_target, uint64_t n,
                                     uint64_t decomp, uint64_t key_modulus_size, uint64_t rns, uint64_t kcc,
                                     const uint64_t* moduli, const uint64_t* const* const* d_key_ptrs,
                                     const uint64_t* galois_elts, uint64_t elts, const uint64_t* modswitch,
                                     cudaStream_t s) {
  std::vector<hexl_b200_ntt*> h(key_modulus_size, nullptr);
  struct Release {
    std::vector<hexl_b200_ntt*>& v;
    ~Release() {
      for (auto* p : v)
        if (p) hexl_b200_ntt_release(p);
    }
  } release{h};
  // RNS modulus i of the computation lives in slot ki(i) of the key / moduli arrays (:62-63); the slots
  // between decomp and the special prime are not touched by this key switch
  auto ki = [&](uint64_t i) { return i == decomp ? key_modulus_size - 1 : i; };
  for (uint64_t i = 0; i < rns; ++i) {
    // lazy sums of the glue kernels (v < 4q in the MAC, < 8q in the final step) need 8q < 2^64
    if (moduli[ki(i)] >= (1ull << 61))
      return fail(HEXL_B200_ERR_INVALID_ARG, "KeySwitch: Require moduli < 2^61 (slot %llu)", (unsigned long long)ki(i));
    if (int rc = cached_ntt(&h[ki(i)], n, moduli[ki(i)])) return rc;
  }
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
#define LAUNCH(expr)                                                    \
  do {                                                                  \
    cudaError_t e__ = (expr);                                           \
    if (e__ != cudaSuccess) return cuda_fail(e__, "KeySwitch: " #expr); \
  } while (0)
  // 1. digits back to coefficient form, each under its own modulus (:49-55)
  if (int rc = ntt_multi_on_device(false, dev, h.data(), decomp, t_coef, t_target, 1, 1, s)) return rc;
  // 2. every digit under every modulus: reduce, lazy forward NTT, multiply-accumulate with the keys (:60-131).
  //    (The digit that already lives in modulus i is re-derived like the others: NTT(INTT(x)) = x mod q_i.)
  for (uint64_t i0 = 0; i0 < rns; i0 += ichunk) {
    const uint64_t cnt = std::min(ichunk, rns - i0);
    KsModuli mods;
    std::vector<hexl_b200_ntt*> hs(cnt);
    for (uint64_t e = 0; e < cnt; ++e) {
      const uint64_t slot = ki(i0 + e), q = moduli[slot], mu = nt::multiply_factor(1, 64, q);
      const uint64_t r64 = mu * (0 - q);  // 2^64 - floor(2^64/q)*q = 2^64 mod q
      const Twiddle R = make_twiddle(r64 % q, q);
      mods.m[e] = KsModulus{q, mu, R.w, R.wp, slot};
      hs[e] = h[slot];
    }
    // every digit into every modulus of the round (:77-85) happens inside the transform: it reads the digits from
    // t_coef (L2-resident) and reduces on load, instead of a reduce kernel writing decomp x cnt x n words for it
    if (int rc = ntt_multi_on_device(true, dev, hs.data(), cnt, ops, t_coef, 4, decomp, s, nullptr, true)) return rc;
    const uint64_t jmax = ks_mac_digits_per_launch(mods, cnt);
    for (uint64_t r = 0; r < elts; ++r) {
      uint64_t* prod_r = prod + r * rns * kcc * n;
      for (uint64_t j0 = 0; j0 < decomp; j0 += jmax) {  // key pointers ride in the kernel parameters
        const uint64_t jc = std::min<uint64_t>(jmax, decomp - j0);
        KeyPointers kp;
        for (uint64_t j = 0; j < jc; ++j) kp.p[j] = d_key_ptrs[r][j0 + j];
        LAUNCH(launch_ks_mac(prod_r + i0 * kcc * n, ops + j0 * n, per_mod, kp, n, jc, kcc, key_modulus_size, cnt,
                             mods, j0 != 0, s, galois_elts ? galois_elts[r] : 0));
      }
    }
  }
#undef LAUNCH
  // 3. mod-down by the special prime and accumulate into result (:134-198); prod's last part is [k][n], contiguous
  for (uint64_t r = 0; r < elts; ++r) {
    uint64_t* prod_r = prod + r * rns * kcc * n;
    if (int rc = mod_down_on_device(dev, results[r], decomp, prod_r, false, true, prod_r + decomp * kcc * n, tmp, n,
                                    kcc, h[key_modulus_size - 1], h.data(), moduli, modswitch, decomp, s))
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


// `count` handles x `group` polynomials each, device pointers on device `dev`, in blocks of kParamBlock handles
// mirrors (inverse only): buffers laid out like `result` that receive the final values too (peer memory: NttMulti::mirror)
int ntt_multi_on_device(bool forward, int dev, hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                        const uint64_t* operand, int out_mf, uint64_t group, cudaStream_t s,
                        const std::vector<uint64_t*>* mirrors, bool gather, const uint64_t* mul) {
  // mul (inverse only): laid out like `operand`; the transform multiplies by it on load (NttMulti::mul)
  // gather (forward only): `operand` holds ONE group of polynomials; every handle's group reads it and reduces the
  // values into its own modulus on load (NttMulti::gather)
  const uint64_t n = handles[0]->n;
  if (gather && !forward) return fail(HEXL_B200_ERR_INVALID_ARG, "gather: forward transforms only");
  if (mul && forward) return fail(HEXL_B200_ERR_INVALID_ARG, "multiply on load: inverse transforms only");
  if (mirrors && (forward || mirrors->size() > (size_t)kMaxMirrors))
    return fail(HEXL_B200_ERR_INVALID_ARG, "mirrored stores: inverse transforms only, at most %d mirrors", kMaxMirrors);
  for (uint64_t first = 0; first < count; first += kParamBlock) {
    const uint64_t cnt = std::min<uint64_t>(kParamBlock, count - first);
    NttMulti multi{};
    multi.group = (unsigned)group;
    if (mirrors) {
      multi.mirrors = (unsigned)mirrors->size();
      for (size_t p = 0; p < mirrors->size(); ++p) multi.mirror[p] = (*mirrors)[p] + first * group * n;
    }
    uint64_t min_q = ~0ull, max_q = 0;
    for (uint64_t i = 0; i < cnt; ++i) {
      NttDeviceTables t;
      if (int rc = device_tables(handles[first + i], dev, &t, s)) return rc;
      multi.p[i] = t.dparams;
      min_q = std::min(min_q, t.q);
      max_q = std::max(max_q, t.q);
    }
    const uint64_t off = first * group * n;
    multi.gather = gather ? (unsigned)group : 0u;
    multi.mul = mul ? mul + off : nullptr;
    cudaError_t e = launch_ntt_multi(forward, multi, handles[0]->log_n, min_q, max_q, result + off,
                                     gather ? operand : operand + off, out_mf, cnt * group, s);
    if (e != cudaSuccess) return cuda_fail(e, "multi-modulus NTT launch");
  }
  return 0;
}

// Host-pointer RNS jobs (count moduli x per_mod elements, modulus m owns [m*per_mod, (m+1)*per_mod)) go through
// the same chunked, multi-stream, multi-device staging as the single-modulus calls: a chunk [off, off + elems)
// is cut at the modulus boundaries it contains and every piece is launched under its own modulus.
// HEXL_B200_NO_PRODUCT_FUSION=1: the unfused chain (lazy transforms, MultMod kernel, inverse), kept for measurement
static bool product_fusion() {
  static const bool on = !(getenv("HEXL_B200_NO_PRODUCT_FUSION") && atoi(getenv("HEXL_B200_NO_PRODUCT_FUSION")) != 0);
  return on;
}
enum class RnsJob { NttFwd, NttInv, Mult, Add, Sub, PolyMul };
EltParams mult_params(uint64_t q, int in_mf) {
  EltParams p{};
  p.q = q;
  p.in_mf = in_mf;
  const int L = floor_log2(q) + 1;  // generalised Barrett constants, eltwise-mult-mod-internal.hpp:52-69
  p.shift = L - 2;
  p.mu = nt::multiply_factor(1ull << (L - 2), 64, q);
  return p;
}
struct RnsSegLaunch {
  bool ok = true;
  int rc = 0;
  RnsJob job = RnsJob::Mult;
  u64 per_mod = 0, n = 1;
  int in_mf = 1, out_mf = 1;
  std::vector<u64> moduli;
  std::vector<NttDeviceTables> t;  // per modulus, filled for the moduli this device touches (NTT jobs)
  cudaError_t operator()(u64* r, const u64* a, const u64* b, u64 off, u64 elems, cudaStream_t s) const {
    for (u64 pos = off; pos < off + elems;) {
      const u64 m = pos / per_mod;
      const u64 cnt = std::min(off + elems, (m + 1) * per_mod) - pos, o = pos - off;
      cudaError_t e = cudaSuccess;
      switch (job) {
        case RnsJob::NttFwd: e = launch_ntt_forward(t[m], r + o, a + o, in_mf, out_mf, cnt / n, s); break;
        case RnsJob::NttInv: e = launch_ntt_inverse(t[m], r + o, a + o, in_mf, out_mf, cnt / n, s); break;
        case RnsJob::Mult:
        case RnsJob::Add:
        case RnsJob::Sub: {
          EltParams p = job == RnsJob::Mult ? mult_params(moduli[m], in_mf) : EltParams{};
          p.q = moduli[m];
          p.result = r + o; p.a = a + o; p.b = b + o; p.n = cnt;
          e = launch_eltwise(job == RnsJob::Mult ? EltOp::MultVV : (job == RnsJob::Add ? EltOp::AddVV : EltOp::SubVV), p, s);
          break;
        }
        case RnsJob::PolyMul: {  // staged buffers: r == a (slot buffer 0), b = slot buffer 1; all in place
          u64* fa = r + o;
          u64* fb = const_cast<u64*>(b) + o;
          if (product_fusion() && moduli[m] >= (1ull << 30)) {  // (below 2^30 the 32-bit-word transforms win)
            if ((e = launch_ntt_forward(t[m], fa, a + o, 1, 1, cnt / n, s)) != cudaSuccess) return e;
            if ((e = launch_ntt_forward(t[m], fb, fb, 1, 1, cnt / n, s)) != cudaSuccess) return e;
            NttMulti multi{};
            multi.p[0] = t[m].dparams;
            multi.group = (unsigned)(cnt / n);
            multi.mul = fb;
            e = launch_ntt_multi(false, multi, t[m].log_n, moduli[m], moduli[m], fa, fa, 1, cnt / n, s);
            break;
          }
          if ((e = launch_ntt_forward(t[m], fa, a + o, 1, 4, cnt / n, s)) != cudaSuccess) return e;
          if ((e = launch_ntt_forward(t[m], fb, fb, 1, 4, cnt / n, s)) != cudaSuccess) return e;
          EltParams p = mult_params(moduli[m], 4);
          p.result = fa; p.a = fa; p.b = fb; p.n = cnt;
          if ((e = launch_eltwise(EltOp::MultVV, p, s)) != cudaSuccess) return e;
          e = launch_ntt_inverse(t[m], fa, fa, 1, 1, cnt / n, s);
          break;
        }
      }
      if (e != cudaSuccess) return e;
      pos += cnt;
    }
    return cudaSuccess;
  }
};

// the launcher factory run_host wants: tables of the moduli inside [lo, hi) on device dev
template <class Handles>
auto rns_seg_factory(RnsJob job, const Handles& handles, const uint64_t* moduli, uint64_t count, u64 per_mod, u64 n,
                     int in_mf, int out_mf) {
  return [=, &handles](int dev, u64 lo, u64 hi) {
    RnsSegLaunch L;
    L.job = job;
    L.per_mod = per_mod;
    L.n = n;
    L.in_mf = in_mf;
    L.out_mf = out_mf;
    L.moduli.resize(count);
    const bool need_tables = job == RnsJob::NttFwd || job == RnsJob::NttInv || job == RnsJob::PolyMul;
    if (need_tables) L.t.resize(count);
    DeviceGuard g;
    int rc = need_tables ? g.enter(dev) : 0;
    for (uint64_t m = 0; m < count && !rc; ++m) {
      L.moduli[m] = moduli ? moduli[m] : handles[m]->q;
      if (need_tables && m * per_mod < hi && (m + 1) * per_mod > lo) rc = device_tables(handles[m], dev, &L.t[m]);
    }
    if (rc) {
      L.ok = false;
      L.rc = rc;
    }
    return L;
  };
}

int ntt_compute_multi(bool forward, hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                      const uint64_t* operand, uint64_t in_mf, uint64_t out_mf, uint64_t group, void* stream) {
  if (!handles) return fail(HEXL_B200_ERR_INVALID_ARG, "handles == nullptr");
  if (count == 0 || group == 0) return 0;
  for (uint64_t i = 0; i < count; ++i) {
    if (!handles[i]) return fail(HEXL_B200_ERR_INVALID_ARG, "handles[%llu] == nullptr", (unsigned long long)i);
    if (handles[i]->n != handles[0]->n) return fail(HEXL_B200_ERR_INVALID_ARG, "all handles must share one degree");
  }
  if (count == 1) return ntt_compute(forward, handles[0], result, operand, in_mf, out_mf, group, stream);
  if (!result) return fail(HEXL_B200_ERR_INVALID_ARG, "result == nullptr");
  if (!operand) return fail(HEXL_B200_ERR_INVALID_ARG, "operand == nullptr");
  const bool in_ok = forward ? (in_mf == 1 || in_mf == 2 || in_mf == 4) : (in_mf == 1 || in_mf == 2);
  const bool out_ok = forward ? (out_mf == 1 || out_mf == 4) : (out_mf == 1 || out_mf == 2);
  if (!in_ok || !out_ok) return fail(HEXL_B200_ERR_INVALID_ARG, "bad input/output_mod_factor");
  PtrInfo pi;
  if (int rc = classify_all({result, operand}, &pi)) return rc;
  const uint64_t n = handles[0]->n;
  if (pi.where == Where::Host) {  // staged, chunked and (with host devices set) split across GPUs like a single-modulus call
    if (g_debug.load())
      for (uint64_t i = 0; i < count; ++i)
        if (int rc = check_bounds(operand + i * group * n, group * n, handles[i]->q * in_mf, pi, "operand")) return rc;
    return run_host(result, operand, nullptr, count * group * n, n,
                    rns_seg_factory(forward ? RnsJob::NttFwd : RnsJob::NttInv, handles, nullptr, count, group * n, n,
                                    (int)in_mf, (int)out_mf));
  }
  for (uint64_t i = 0; i < count; ++i)
    if (int rc = check_bounds(operand + i * group * n, group * n, handles[i]->q * in_mf, pi, "operand")) return rc;
  DeviceGuard g;
  if (int rc = g.enter(pi.device)) return rc;
  if (int rc = ntt_multi_on_device(forward, pi.device, handles, count, result, operand, (int)out_mf, group,
                                   (cudaStream_t)stream))
    return rc;
  return finish_device_call(pi, stream);
}

int debug_bounds(const u64* p, u64 n, u64 bound, const char* what, std::initializer_list<const void*> all) {
  if (!g_debug.load()) return 0;
  PtrInfo pi;
  if (int rc = classify_all(all, &pi)) return rc;
  return check_bounds(p, n, bound, pi, what);
}

}  // namespace

// =============================================================== extern "C"
extern "C" {

const char* hexl_b200_version(void) { return "hexl-b200 0.1 (sm_90a; API of intel/hexl 1.2.5)"; }
const char* hexl_b200_last_error(void) { return t_error.c_str(); }

int hexl_b200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}

int hexl_b200_set_host_devices(const int* devices, int count) {
  int n = hexl_b200_device_count();
  std::vector<int> v;
  for (int i = 0; i < count; ++i) {
    if (!devices || devices[i] < 0 || devices[i] >= n)
      return fail(HEXL_B200_ERR_INVALID_ARG, "device ordinal out of range");
    v.push_back(devices[i]);
  }
  std::lock_guard<std::mutex> lk(g_cfg_mu);
  g_host_devices = v;
  return 0;
}

void hexl_b200_set_debug(int on) { g_debug.store(on ? 1 : 0); }

int hexl_b200_sync(void* stream) {
  CU(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

void* hexl_b200_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}
void hexl_b200_host_free(void* p) {
  if (p) cudaFreeHost(p);
}
void* hexl_b200_managed_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocManaged(&p, bytes ? bytes : 1, cudaMemAttachGlobal) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}
void hexl_b200_managed_free(void* p) {
  if (p) cudaFree(p);
}

uint64_t hexl_b200_launch_count(void) { return launches_so_far(); }

// ---- number theory
uint64_t hexl_b200_multiply_mod(uint64_t x, uint64_t y, uint64_t q) { return nt::mul_mod(x, y, q); }
uint64_t hexl_b200_add_uint_mod(uint64_t x, uint64_t y, uint64_t q) { return nt::add_mod(x, y, q); }
uint64_t hexl_b200_sub_uint_mod(uint64_t x, uint64_t y, uint64_t q) { return nt::sub_mod(x, y, q); }
uint64_t hexl_b200_pow_mod(uint64_t b, uint64_t e, uint64_t q) { return nt::pow_mod(b, e, q); }
uint64_t hexl_b200_inverse_mod(uint64_t x, uint64_t q) { return nt::inverse_mod(x, q); }
uint64_t hexl_b200_reverse_bits(uint64_t x, uint64_t w) { return nt::reverse_bits(x, w); }
int hexl_b200_is_prime(uint64_t n) { return nt::is_prime(n) ? 1 : 0; }
int hexl_b200_is_primitive_root(uint64_t r, uint64_t d, uint64_t q) { return nt::is_primitive_root(r, d, q) ? 1 : 0; }
uint64_t hexl_b200_generate_primitive_root(uint64_t d, uint64_t q) { return nt::generate_primitive_root(d, q); }
uint64_t hexl_b200_minimal_primitive_root(uint64_t d, uint64_t q) { return nt::minimal_primitive_root(d, q); }
uint64_t hexl_b200_multiply_factor(uint64_t operand, uint64_t bit_shift, uint64_t q) {
  return nt::multiply_factor(operand, bit_shift, q);
}
int hexl_b200_generate_primes(uint64_t* out, size_t num, size_t bit_size, int prefer_small, size_t ntt_size) {
  std::vector<uint64_t> p = nt::generate_primes(num, bit_size, prefer_small != 0, ntt_size);
  for (size_t i = 0; i < p.size(); ++i) out[i] = p[i];
  return (int)p.size();
}

// ---- NTT object
int hexl_b200_ntt_create(hexl_b200_ntt** out, uint64_t degree, uint64_t q) {
  return create_common(out, degree, q, 0, false);
}
int hexl_b200_ntt_create_with_root(hexl_b200_ntt** out, uint64_t degree, uint64_t q, uint64_t root) {
  return create_common(out, degree, q, root, true);
}
void hexl_b200_ntt_retain(hexl_b200_ntt* h) {
  if (h) h->refs.fetch_add(1);
}
void hexl_b200_ntt_release(hexl_b200_ntt* h) {
  if (!h || h->refs.fetch_sub(1) != 1) return;
  int prev = -1;
  cudaGetDevice(&prev);
  for (auto& kv : h->dev) {
    if (cudaSetDevice(kv.first) == cudaSuccess) {
      cudaFree(kv.second.fwd);
      cudaFree(kv.second.inv);
      cudaFree(kv.second.fwd32);  // nullptr unless q < 2^30
      cudaFree(kv.second.inv32);
      cudaFree(kv.second.params);
    }
  }
  if (prev >= 0) cudaSetDevice(prev);
  cudaGetLastError();
  delete h;
}
int hexl_b200_ntt_check_arguments(uint64_t degree, uint64_t q) {
  const char* why = "";
  return check_ntt_arguments(degree, q, &why) ? 1 : 0;
}
uint64_t hexl_b200_ntt_degree(const hexl_b200_ntt* h) { return h ? h->n : 0; }
uint64_t hexl_b200_ntt_modulus(const hexl_b200_ntt* h) { return h ? h->q : 0; }
uint64_t hexl_b200_ntt_minimal_root(const hexl_b200_ntt* h) { return h ? h->root : 0; }
const uint64_t* hexl_b200_ntt_table(const hexl_b200_ntt* h, int which) {
  if (!h) return nullptr;
  switch (which) {
    case 0: return h->w.data();
    case 1: return h->w_precon.data();
    case 2: return h->inv_seq.data();
    case 3: return h->inv_seq_precon.data();
  }
  return nullptr;
}

int hexl_b200_ntt_prepare(hexl_b200_ntt* h, int device) {
  if (!h) return fail(HEXL_B200_ERR_INVALID_ARG, "ntt handle == nullptr");
  if (device < 0) CU(cudaGetDevice(&device));
  if (device >= hexl_b200_device_count()) return fail(HEXL_B200_ERR_INVALID_ARG, "device ordinal out of range");
  DeviceGuard g;
  if (int rc = g.enter(device)) return rc;
  NttDeviceTables t;
  return device_tables(h, device, &t);
}

int hexl_b200_ntt_forward(hexl_b200_ntt* h, uint64_t* result, const uint64_t* operand, uint64_t in_mf,
                          uint64_t out_mf, uint64_t batch, void* stream) {
  return ntt_compute(true, h, result, operand, in_mf, out_mf, batch, stream);
}
int hexl_b200_ntt_inverse(hexl_b200_ntt* h, uint64_t* result, const uint64_t* operand, uint64_t in_mf,
                          uint64_t out_mf, uint64_t batch, void* stream) {
  return ntt_compute(false, h, result, operand, in_mf, out_mf, batch, stream);
}

int hexl_b200_ntt_forward_multi(hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                                const uint64_t* operand, uint64_t in_mf, uint64_t out_mf, uint64_t batch_per_modulus,
                                void* stream) {
  return ntt_compute_multi(true, handles, count, result, operand, in_mf, out_mf, batch_per_modulus, stream);
}
int hexl_b200_ntt_inverse_multi(hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                                const uint64_t* operand, uint64_t in_mf, uint64_t out_mf, uint64_t batch_per_modulus,
                                void* stream) {
  return ntt_compute_multi(false, handles, count, result, operand, in_mf, out_mf, batch_per_modulus, stream);
}

// ---- eltwise.  Checks mirror the HEXL_CHECKs at the top of each reference op.
int hexl_b200_eltwise_add_mod(uint64_t* result, const uint64_t* op1, const uint64_t* op2, uint64_t n,
                              uint64_t q, void* stream) {
  // eltwise-add-mod.cpp:73-81
  REQUIRE(result && op1 && op2, "Require result, operand1, operand2 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q < (1ull << 63), "Require modulus < 2**63");
  if (int rc = debug_bounds(op1, n, q, "operand1", {result, op1, op2})) return rc;
  if (int rc = debug_bounds(op2, n, q, "operand2", {result, op1, op2})) return rc;
  EltParams p{};
  p.result = result; p.a = op1; p.b = op2; p.n = n; p.q = q;
  return eltwise_dispatch(EltOp::AddVV, p, stream);
}

int hexl_b200_eltwise_add_mod_scalar(uint64_t* result, const uint64_t* op1, uint64_t op2, uint64_t n,
                                     uint64_t q, void* stream) {
  // eltwise-add-mod.cpp:95-103
  REQUIRE(result && op1, "Require result, operand1 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q < (1ull << 63), "Require modulus < 2**63");
  REQUIRE(op2 < q, "Require operand2 < modulus");
  if (int rc = debug_bounds(op1, n, q, "operand1", {result, op1})) return rc;
  EltParams p{};
  p.result = result; p.a = op1; p.n = n; p.q = q; p.scalar = op2;
  return eltwise_dispatch(EltOp::AddVS, p, stream);
}

int hexl_b200_eltwise_sub_mod(uint64_t* result, const uint64_t* op1, const uint64_t* op2, uint64_t n,
                              uint64_t q, void* stream) {
  // eltwise-sub-mod.cpp:69-77
  REQUIRE(result && op1 && op2, "Require result, operand1, operand2 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q < (1ull << 63), "Require modulus < 2**63");
  if (int rc = debug_bounds(op1, n, q, "operand1", {result, op1, op2})) return rc;
  if (int rc = debug_bounds(op2, n, q, "operand2", {result, op1, op2})) return rc;
  EltParams p{};
  p.result = result; p.a = op1; p.b = op2; p.n = n; p.q = q;
  return eltwise_dispatch(EltOp::SubVV, p, stream);
}

int hexl_b200_eltwise_sub_mod_scalar(uint64_t* result, const uint64_t* op1, uint64_t op2, uint64_t n,
                                     uint64_t q, void* stream) {
  // eltwise-sub-mod.cpp:91-99
  REQUIRE(result && op1, "Require result, operand1 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q < (1ull << 63), "Require modulus < 2**63");
  REQUIRE(op2 < q, "Require operand2 < modulus");
  if (int rc = debug_bounds(op1, n, q, "operand1", {result, op1})) return rc;
  EltParams p{};
  p.result = result; p.a = op1; p.n = n; p.q = q; p.scalar = op2;
  return eltwise_dispatch(EltOp::SubVS, p, stream);
}

int hexl_b200_eltwise_mult_mod(uint64_t* result, const uint64_t* op1, const uint64_t* op2, uint64_t n,
                               uint64_t q, uint64_t in_mf, void* stream) {
  // eltwise-mult-mod.cpp:21-36
  REQUIRE(result && op1 && op2, "Require result, operand1, operand2 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(in_mf == 1 || in_mf == 2 || in_mf == 4, "input_mod_factor must be 1, 2 or 4; got %llu", (unsigned long long)in_mf);
  REQUIRE(q < (1ull << 62), "Require modulus < (1ULL << 62)");
  REQUIRE(in_mf * q < (1ull << 63), "Require input_mod_factor * modulus < (1ULL << 63)");
  if (int rc = debug_bounds(op1, n, in_mf * q, "operand1", {result, op1, op2})) return rc;
  if (int rc = debug_bounds(op2, n, in_mf * q, "operand2", {result, op1, op2})) return rc;
  EltParams p{};
  p.result = result; p.a = op1; p.b = op2; p.n = n; p.q = q; p.in_mf = (int)in_mf;
  // generalised Barrett constants, eltwise-mult-mod-internal.hpp:52-69
  const int L = floor_log2(q) + 1;
  p.shift = L - 2;
  p.mu = nt::multiply_factor(1ull << (L - 2), 64, q);
  return eltwise_dispatch(EltOp::MultVV, p, stream);
}

int hexl_b200_eltwise_fma_mod(uint64_t* result, const uint64_t* arg1, uint64_t arg2, const uint64_t* arg3,
                              uint64_t n, uint64_t q, uint64_t in_mf, void* stream) {
  // eltwise-fma-mod.cpp:20-40
  REQUIRE(result && arg1, "Require result, arg1 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q < (1ull << 61), "Require modulus < (1ULL << 61)");
  REQUIRE(in_mf == 1 || in_mf == 2 || in_mf == 4 || in_mf == 8,
          "input_mod_factor must be 1, 2, 4, or 8. Got %llu", (unsigned long long)in_mf);
  REQUIRE(arg2 < in_mf * q, "arg2 exceeds bound input_mod_factor * modulus");
  if (int rc = debug_bounds(arg1, n, in_mf * q, "arg1", {result, arg1, arg3})) return rc;
  if (int rc = debug_bounds(arg3, n, in_mf * q, "arg3", {result, arg1, arg3})) return rc;
  EltParams p{};
  p.result = result; p.a = arg1; p.b = arg3; p.n = n; p.q = q; p.in_mf = (int)in_mf;
  uint64_t s = arg2;  // ReduceMod<in_mf>(arg2), eltwise-fma-mod-internal.hpp:16-17
  if (in_mf >= 8 && s >= 4 * q) s -= 4 * q;
  if (in_mf >= 4 && s >= 2 * q) s -= 2 * q;
  if (in_mf >= 2 && s >= q) s -= q;
  p.scalar = s;
  p.scalar_p = nt::multiply_factor(s, 64, q);
  return eltwise_dispatch(arg3 ? EltOp::Fma : EltOp::FmaNoAdd, p, stream);
}

int hexl_b200_eltwise_reduce_mod(uint64_t* result, const uint64_t* operand, uint64_t n, uint64_t q,
                                 uint64_t in_mf, uint64_t out_mf, void* stream) {
  // eltwise-reduce-mod.cpp:84-92
  REQUIRE(result && operand, "Require result, operand != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(in_mf == q || in_mf == 2 || in_mf == 4, "input_mod_factor must be modulus or 2 or 4; got %llu",
          (unsigned long long)in_mf);
  REQUIRE(out_mf == 1 || out_mf == 2, "output_mod_factor must be 1 or 2; got %llu", (unsigned long long)out_mf);
  EltParams p{};
  p.result = result; p.a = operand; p.n = n; p.q = q; p.out_mf = (int)out_mf;
  // From q >= 2^63 on, every 64-bit word is below 2q, so input_mod_factor 4 is the 2 case; reducing from [0, 4q) would
  // subtract 2q, which wraps (as it does in every tier of the reference).
  if (in_mf == 4 && q >= (1ull << 63)) in_mf = 2;
  if (in_mf == out_mf) {  // eltwise-reduce-mod.cpp:94-99: plain copy (no-op in place)
    if (result == operand) return 0;
    return eltwise_dispatch(EltOp::Copy, p, stream);
  }
  p.in_mf = (in_mf == q) ? 0 : (int)in_mf;
  p.mu = nt::multiply_factor(1, 64, q);
  return eltwise_dispatch(EltOp::Reduce, p, stream);
}

int hexl_b200_eltwise_cmp_add(uint64_t* result, const uint64_t* op1, uint64_t n, int cmp, uint64_t bound,
                              uint64_t diff, void* stream) {
  // eltwise-cmp-add.cpp:18-21
  REQUIRE(result && op1, "Require result, operand1 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(diff != 0, "Require diff != 0");
  REQUIRE(cmp >= 0 && cmp <= 7, "cmp must be a CMPINT value (0..7)");
  EltParams p{};
  p.result = result; p.a = op1; p.n = n; p.scalar = bound; p.scalar_p = diff; p.cmp = cmp;
  return eltwise_dispatch(EltOp::CmpAdd, p, stream);
}

int hexl_b200_eltwise_cmp_sub_mod(uint64_t* result, const uint64_t* op1, uint64_t n, uint64_t q, int cmp,
                                  uint64_t bound, uint64_t diff, void* stream) {
  // eltwise-cmp-sub-mod.cpp:21-25,50-55
  REQUIRE(result && op1, "Require result, operand1 != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(diff != 0, "Require diff != 0");
  REQUIRE(diff < q, "Diff >= modulus");
  REQUIRE(cmp >= 0 && cmp <= 7, "cmp must be a CMPINT value (0..7)");
  EltParams p{};
  p.result = result; p.a = op1; p.n = n; p.q = q; p.scalar = bound; p.scalar_p = diff; p.cmp = cmp;
  p.mu = nt::multiply_factor(1, 64, q);
  return eltwise_dispatch(EltOp::CmpSubMod, p, stream);
}

// ---- Montgomery-form helpers (SURVEY 8(f)-4)
uint64_t hexl_b200_hensel_lemma_2adic_root(uint32_t r, uint64_t q) {
  if (r == 0 || r > 64 || !(q & 1)) return 0;
  return nt::neg_inverse_mod_pow2(r, q);
}
uint64_t hexl_b200_montgomery_reduce(uint64_t T_hi, uint64_t T_lo, uint64_t q, int r, uint64_t inv_mod) {
  if (r < 1 || r > 62 || q < 2) return 0;
  return nt::montgomery_reduce(T_hi, T_lo, q, r, inv_mod);
}
static int mont_dispatch(EltOp op, uint64_t* result, const uint64_t* a, const uint64_t* b, uint64_t scalar, uint64_t n,
                         uint64_t q, int r, uint64_t neg_inv_mod, void* stream) {
  // checks of eltwise-reduce-mod-avx512.hpp:160-176
  REQUIRE(result && a && (op != EltOp::MontMult || b), "Require result, operands != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(q > 1, "Require modulus > 1");
  REQUIRE(q & 1, "gcd(modulus, R) != 1");
  REQUIRE(r >= 1 && r <= 62, "With r > 62 internal ops might overflow");
  REQUIRE((1ull << r) > q, "Needs R bigger than q.");
  REQUIRE(((q * neg_inv_mod + 1) & ((1ull << r) - 1)) == 0, "neg_inv_mod is not -1/q mod R");
  if (int rc = debug_bounds(a, n, q, "operand a", {result, a, b})) return rc;
  if (op == EltOp::MontMult)
    if (int rc = debug_bounds(b, n, q, "operand b", {result, a, b})) return rc;
  EltParams p{};
  p.result = result; p.a = a; p.b = b; p.n = n; p.q = q; p.mu = neg_inv_mod & ((1ull << r) - 1); p.shift = r; p.scalar = scalar;
  return eltwise_dispatch(op, p, stream);
}
int hexl_b200_eltwise_mont_reduce_mod(uint64_t* result, const uint64_t* a, const uint64_t* b, uint64_t n, uint64_t q,
                                      int r, uint64_t neg_inv_mod, void* stream) {
  return mont_dispatch(EltOp::MontMult, result, a, b, 0, n, q, r, neg_inv_mod, stream);
}
int hexl_b200_eltwise_montgomery_form_in(uint64_t* result, const uint64_t* a, uint64_t R2_mod_q, uint64_t n, uint64_t q,
                                         int r, uint64_t neg_inv_mod, void* stream) {
  REQUIRE(R2_mod_q < q, "Require R2_mod_q < modulus");
  return mont_dispatch(EltOp::MontIn, result, a, nullptr, R2_mod_q, n, q, r, neg_inv_mod, stream);
}
int hexl_b200_eltwise_montgomery_form_out(uint64_t* result, const uint64_t* a, uint64_t n, uint64_t q, int r,
                                          uint64_t neg_inv_mod, void* stream) {
  return mont_dispatch(EltOp::MontOut, result, a, nullptr, 0, n, q, r, neg_inv_mod, stream);
}

// ---- SEAL-shaped composites
int hexl_b200_ntt_get_cached(hexl_b200_ntt** out, uint64_t degree, uint64_t q) {
  if (!out) return fail(HEXL_B200_ERR_INVALID_ARG, "out == nullptr");
  return cached_ntt(out, degree, q);
}

// device side of EltwiseMultMod over an RNS batch
static int rns_eltwise_on_device(int op, uint64_t* result, const uint64_t* a, const uint64_t* b, uint64_t per_mod,
                                 const uint64_t* moduli, uint64_t num_moduli, int in_mf, cudaStream_t s) {
  for (uint64_t first = 0; first < num_moduli; first += kParamBlock) {
    const uint64_t count = std::min<uint64_t>(kParamBlock, num_moduli - first);
    DyadicModuli mods;
    for (uint64_t i = 0; i < count; ++i) mods.m[i] = dyadic_modulus(moduli[first + i]);
    const uint64_t off = first * per_mod;
    cudaError_t e = launch_rns_eltwise(op, result + off, a + off, b + off, per_mod, count, in_mf, mods, s);
    if (e != cudaSuccess) return cuda_fail(e, "eltwise (RNS batch) launch");
  }
  return 0;
}

static int rns_eltwise_entry(int op, uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                             uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli, uint64_t in_mf,
                             void* stream) {
  REQUIRE(result && operand1 && operand2 && moduli, "Require result, operand1, operand2, moduli != nullptr");
  REQUIRE(n_per_modulus != 0 && num_moduli != 0, "Require n != 0");
  REQUIRE(in_mf == 1 || in_mf == 2 || in_mf == 4, "Require input_mod_factor = 1, 2, or 4");
  for (uint64_t i = 0; i < num_moduli; ++i)
    REQUIRE(moduli[i] > 1 && moduli[i] < (1ull << 62) && moduli[i] * in_mf < (1ull << 63),
            "Require 1 < modulus < 2^62 and input_mod_factor * modulus < 2^63");
  PtrInfo pi;
  if (int rc = classify_all({result, operand1, operand2}, &pi)) return rc;
  const uint64_t total = n_per_modulus * num_moduli;
  if (pi.where == Where::Device) {
    DeviceGuard g;
    if (int rc = g.enter(pi.device)) return rc;
    for (uint64_t i = 0; i < num_moduli; ++i) {
      if (int rc = check_bounds(operand1 + i * n_per_modulus, n_per_modulus, moduli[i] * in_mf, pi, "operand1")) return rc;
      if (int rc = check_bounds(operand2 + i * n_per_modulus, n_per_modulus, moduli[i] * in_mf, pi, "operand2")) return rc;
    }
    if (int rc = rns_eltwise_on_device(op, result, operand1, operand2, n_per_modulus, moduli, num_moduli, (int)in_mf,
                                       (cudaStream_t)stream))
      return rc;
    return finish_device_call(pi, stream);
  }
  struct NoHandles {
    hexl_b200_ntt* operator[](uint64_t) const { return nullptr; }
  } none;
  const RnsJob job = op == kRnsMult ? RnsJob::Mult : (op == kRnsAdd ? RnsJob::Add : RnsJob::Sub);
  return run_host(result, operand1, operand2, total, 1,
                  rns_seg_factory(job, none, moduli, num_moduli, n_per_modulus, 1, (int)in_mf, 1));
}

int hexl_b200_eltwise_mult_mod_multi(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                                     uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli,
                                     uint64_t in_mf, void* stream) {
  return rns_eltwise_entry(kRnsMult, result, operand1, operand2, n_per_modulus, moduli, num_moduli, in_mf, stream);
}
int hexl_b200_eltwise_add_mod_multi(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                                    uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli, void* stream) {
  return rns_eltwise_entry(kRnsAdd, result, operand1, operand2, n_per_modulus, moduli, num_moduli, 1, stream);
}
int hexl_b200_eltwise_sub_mod_multi(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2,
                                    uint64_t n_per_modulus, const uint64_t* moduli, uint64_t num_moduli, void* stream) {
  return rns_eltwise_entry(kRnsSub, result, operand1, operand2, n_per_modulus, moduli, num_moduli, 1, stream);
}

// FwdNTT(b) into scratch, FwdNTT(a) into result, point-wise product, InvNTT: all moduli per launch.  b is read before
// result is first written, so result may be a, b or both (an in-place square)
static int poly_multiply_on_device(int dev, hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
                                   const uint64_t* a, const uint64_t* b, uint64_t group, cudaStream_t s) {
  const uint64_t n = handles[0]->n, total = count * group * n;
  Scratch ws(s);
  uint64_t* fb = nullptr;
  if (int rc = ws.get(&fb, total)) return rc;
  std::vector<uint64_t> moduli(count);
  for (uint64_t i = 0; i < count; ++i) moduli[i] = handles[i]->q;
  if (product_fusion()) {
    // canonical transforms, then ONE inverse transform that multiplies on load: no MultMod kernel, and the product
    // never travels to HBM and back (dyadic-multiply-internal.cpp:17-73 folded into the transform that consumes it)
    if (int rc = ntt_multi_on_device(true, dev, handles, count, fb, b, 1, group, s)) return rc;
    if (int rc = ntt_multi_on_device(true, dev, handles, count, result, a, 1, group, s)) return rc;
    return ntt_multi_on_device(false, dev, handles, count, result, result, 1, group, s, nullptr, false, fb);
  }
  if (int rc = ntt_multi_on_device(true, dev, handles, count, fb, b, 4, group, s)) return rc;
  if (int rc = ntt_multi_on_device(true, dev, handles, count, result, a, 4, group, s)) return rc;
  if (int rc = rns_eltwise_on_device(kRnsMult, result, result, fb, group * n, moduli.data(), count, 4, s)) return rc;
  return ntt_multi_on_device(false, dev, handles, count, result, result, 1, group, s);
}

int hexl_b200_poly_multiply_multi(hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result, const uint64_t* a,
                                  const uint64_t* b, uint64_t group, void* stream) {
  REQUIRE(handles && result && a && b, "Require handles, result, a, b != nullptr");
  if (count == 0 || group == 0) return 0;
  for (uint64_t i = 0; i < count; ++i) {
    REQUIRE(handles[i] != nullptr, "Require handles[i] != nullptr");
    REQUIRE(handles[i]->n == handles[0]->n, "all handles must share one degree");
    REQUIRE(handles[i]->q < (1ull << 61), "Require modulus < 2^61 (lazy transform outputs feed the product)");
  }
  PtrInfo pi;
  if (int rc = classify_all({result, a, b}, &pi)) return rc;
  const uint64_t n = handles[0]->n, total = count * group * n;
  if (pi.where == Where::Device) {
    DeviceGuard g;
    if (int rc = g.enter(pi.device)) return rc;
    for (uint64_t i = 0; i < count; ++i) {
      if (int rc = check_bounds(a + i * group * n, group * n, handles[i]->q, pi, "a")) return rc;
      if (int rc = check_bounds(b + i * group * n, group * n, handles[i]->q, pi, "b")) return rc;
    }
    if (int rc = poly_multiply_on_device(pi.device, handles, count, result, a, b, group, (cudaStream_t)stream)) return rc;
    return finish_device_call(pi, stream);
  }
  if (g_debug.load())
    for (uint64_t i = 0; i < count; ++i) {
      if (int rc = check_bounds(a + i * group * n, group * n, handles[i]->q, pi, "a")) return rc;
      if (int rc = check_bounds(b + i * group * n, group * n, handles[i]->q, pi, "b")) return rc;
    }
  // host pointers: every chunk of polynomials is copied in, transformed, multiplied, transformed back and
  // copied out on one of the rotating staging streams, so the PCIe copies of one chunk hide under the
  // kernels of the others; with host devices set the polynomials are split across the GPUs
  return run_host(result, a, b, total, n, rns_seg_factory(RnsJob::PolyMul, handles, nullptr, count, group * n, n, 1, 1));
}

int hexl_b200_dyadic_multiply(uint64_t* result, const uint64_t* operand1, const uint64_t* operand2, uint64_t n,
                              const uint64_t* moduli, uint64_t num_moduli, void* stream) {
  // dyadic-multiply-internal.cpp:20-24
  REQUIRE(result && operand1 && operand2 && moduli, "Require result, operand1, operand2, moduli != nullptr");
  REQUIRE(n != 0, "Require n != 0");
  REQUIRE(num_moduli != 0, "Require num_moduli != 0");
  for (uint64_t i = 0; i < num_moduli; ++i)
    REQUIRE(moduli[i] > 1 && moduli[i] < (1ull << 62), "Require 1 < modulus < 2^62");
  PtrInfo pi;
  if (int rc = classify_all({result, operand1, operand2}, &pi)) return rc;
  if (pi.where == Where::Device) {
    DeviceGuard g;
    if (int rc = g.enter(pi.device)) return rc;
    if (int rc = dyadic_on_device(result, operand1, operand2, n, moduli, num_moduli, (cudaStream_t)stream)) return rc;
    return finish_device_call(pi, stream);
  }
  // Host pointers: blocks of moduli travel through the rotating staging slots (the layout is
  // [polynomial][modulus][n], so a block of moduli is a 2-D copy: 2 rows in, 3 rows out).
  int cur = 0;
  CU(cudaGetDevice(&cur));
  {
    const std::vector<int> devs = host_devices();
    if (!devs.empty()) cur = devs[0];
  }
  DeviceGuard g;
  if (int rc = g.enter(cur)) return rc;
  StageCtx* st = stage_for(cur);
  std::lock_guard<std::mutex> lk(st->mu);
  if (int rc = st->init()) return rc;
  u64 mb = std::max<u64>(1, (kChunkBytes / sizeof(u64)) / (3 * n));
  mb = std::min<u64>({mb, (u64)kParamBlock, num_moduli});
  const size_t row = (size_t)num_moduli * n * sizeof(u64);  // host pitch: one polynomial over all moduli
  int slot = 0;
  for (u64 m0 = 0; m0 < num_moduli; m0 += mb, slot = (slot + 1) % kSlots) {
    const u64 cnt = std::min(mb, num_moduli - m0);
    const size_t w = (size_t)cnt * n * sizeof(u64);
    if (int rc = st->reserve(slot, 0, 3 * w)) return rc;
    if (int rc = st->reserve(slot, 1, 2 * w)) return rc;
    if (int rc = st->reserve(slot, 2, 2 * w)) return rc;
    cudaStream_t sx = st->stream[slot];
    u64 *dr = st->buf[slot][0], *d1 = st->buf[slot][1], *d2 = st->buf[slot][2];
    CU(cudaMemcpy2DAsync(d1, w, operand1 + m0 * n, row, w, 2, cudaMemcpyHostToDevice, sx));
    CU(cudaMemcpy2DAsync(d2, w, operand2 + m0 * n, row, w, 2, cudaMemcpyHostToDevice, sx));
    if (int rc = dyadic_on_device(dr, d1, d2, n, moduli + m0, cnt, sx)) return rc;
    CU(cudaMemcpy2DAsync(result + m0 * n, row, dr, w, w, 3, cudaMemcpyDeviceToHost, sx));
  }
  for (int k = 0; k < kSlots; ++k) CU(cudaStreamSynchronize(st->stream[k]));
  return 0;
}

// The rotation of one ciphertext (two components of decomp limbs in NTT form, device memory): sigma_g of both
// components into perm (2 x decomp x n words of scratch) in one launch, then c0 <- sigma_g(c0), c1 <- 0 by stream
// copies and the key switch of t_target = sigma_g(c1), which accumulates KS(sigma_g(c1)) into both components.
static int galois_key_switch_on_device(int dev, uint64_t* ct, uint64_t* perm, uint64_t n, uint64_t decomp,
                                       uint64_t key_modulus_size, uint64_t rns, const uint64_t* moduli,
                                       const uint64_t* const* d_key_ptrs_host, const uint64_t* modswitch,
                                       uint64_t galois_elt, cudaStream_t s) {
  const uint64_t comp = decomp * n;
  const cudaError_t e = launch_galois_ntt(perm, ct, floor_log2(n), 2 * decomp, galois_elt, s);
  if (e != cudaSuccess) return cuda_fail(e, "ApplyGaloisKeySwitch: automorphism launch");
  CU(cudaMemcpyAsync(ct, perm, comp * sizeof(uint64_t), cudaMemcpyDeviceToDevice, s));
  CU(cudaMemsetAsync(ct + comp, 0, comp * sizeof(uint64_t), s));
  return key_switch_on_device(dev, ct, perm + comp, n, decomp, key_modulus_size, rns, 2, moduli, d_key_ptrs_host,
                              modswitch, s);
}

// The hoisted rotations of one ciphertext ct (device memory, as above) by num_elts elements: out + r * 2 * decomp * n
// gets [sigma_g(c0), 0] + ModDown(sum_j pi_g(D_j) K_r[j]) for g = galois_elts[r], with the digits D_j of c1 decomposed
// and transformed once for every element.  Per element: one automorphism launch over c0 straight into the output, a
// memset of the output's c1, then its multiply-accumulates and mod-down inside the shared key switch.
static int hoisted_rotations_on_device(int dev, uint64_t* out, const uint64_t* ct, uint64_t n, uint64_t decomp,
                                       uint64_t key_modulus_size, uint64_t rns, const uint64_t* moduli,
                                       const uint64_t* const* const* d_key_ptrs, const uint64_t* galois_elts,
                                       uint64_t num_elts, const uint64_t* modswitch, cudaStream_t s) {
  const uint64_t comp = decomp * n;
  std::vector<uint64_t*> results(num_elts);
  for (uint64_t r = 0; r < num_elts; ++r) {
    results[r] = out + r * 2 * comp;
    const cudaError_t e = launch_galois_ntt(results[r], ct, floor_log2(n), decomp, galois_elts[r], s);
    if (e != cudaSuccess) return cuda_fail(e, "ApplyGaloisKeySwitchHoisted: automorphism launch");
    CU(cudaMemsetAsync(results[r] + comp, 0, comp * sizeof(uint64_t), s));
  }
  return key_switch_elts_on_device(dev, results.data(), ct + comp, n, decomp, key_modulus_size, rns, 2, moduli,
                                   d_key_ptrs, galois_elts, num_elts, modswitch, s);
}

// One or more key switches on HOST buffers against keys already on the devices: ciphertext c occupies
// result[c * kcc*decomp*n ...] and t_target[c * decomp*n ...].  Each ciphertext runs on one of the rotating
// staging streams (digits in, result in, ~12 kernels, result out), so the copies of one ciphertext overlap the
// kernels of its neighbours; with host devices set the batch is split across the GPUs holding the keys.
// galois_elt != 0: the rotation of ApplyGaloisKeySwitch instead (kcc = 2, t_target unused): only the ciphertext
// crosses PCIe, and the slot's second buffer holds both permuted components.
// hoisted_elts != nullptr: the num_elts hoisted rotations of ApplyGaloisKeySwitchHoisted instead (kcc = 2, keys[r] for
// hoisted_elts[r]): t_target holds the input ciphertexts (2 x decomp x n words each); each crosses PCIe in once and
// its num_elts rotations come back from the same slot.  The batch is split over the devices holding every key.
static int key_switch_host_batch(uint64_t* result, const uint64_t* t_target, uint64_t n, uint64_t decomp,
                                 uint64_t key_modulus_size, uint64_t rns, uint64_t kcc, const uint64_t* moduli,
                                 const hexl_b200_keys* const* keys, const uint64_t* modswitch, uint64_t batch,
                                 uint64_t galois_elt = 0, const uint64_t* hoisted_elts = nullptr,
                                 uint64_t num_elts = 1) {
  std::vector<int> devs = host_devices();
  if (devs.empty()) {
    int cur = 0;
    CU(cudaGetDevice(&cur));
    devs.push_back(cur);
  }
  const bool hoisted = hoisted_elts != nullptr;
  std::vector<int> use;
  for (int d : devs) {
    bool all = true;
    for (uint64_t r = 0; r < num_elts; ++r) all = all && keys[r]->dev.count(d);
    if (all) use.push_back(d);
  }
  if (use.empty()) return fail(HEXL_B200_ERR_INVALID_ARG, "the key handle holds no copy on the device(s) used for host calls");
  if (use.size() > batch) use.resize(batch);
  const u64 res_elems = (hoisted ? num_elts : 1) * kcc * decomp * n, t_elems = (hoisted ? 2 : 1) * decomp * n;
  int rc = 0;
  for (size_t di = 0; di < use.size() && !rc; ++di) {
    const int dev = use[di];
    const u64 c_lo = batch * di / use.size(), c_hi = batch * (di + 1) / use.size();
    DeviceGuard g;
    if ((rc = g.enter(dev))) break;
    StageCtx* st = stage_for(dev);
    std::lock_guard<std::mutex> lk(st->mu);
    if ((rc = st->init())) break;
    std::vector<const uint64_t* const*> dk(num_elts);
    for (uint64_t r = 0; r < num_elts; ++r) dk[r] = keys[r]->dev.at(dev).data();
    int slot = 0;
    for (u64 c = c_lo; c < c_hi && !rc; ++c, slot = (slot + 1) % kSlots) {
      if ((rc = st->reserve(slot, 0, res_elems * 8))) break;
      if ((rc = st->reserve(slot, 1, (galois_elt ? 2 : 1) * t_elems * 8))) break;
      cudaStream_t sx = st->stream[slot];
      u64 *d_res = st->buf[slot][0], *d_t = st->buf[slot][1];
      cudaError_t e = cudaSuccess;
      if (!galois_elt) e = cudaMemcpyAsync(d_t, t_target + c * t_elems, t_elems * 8, cudaMemcpyHostToDevice, sx);
      if (e == cudaSuccess && !hoisted)
        e = cudaMemcpyAsync(d_res, result + c * res_elems, res_elems * 8, cudaMemcpyHostToDevice, sx);
      if (e != cudaSuccess) {
        rc = cuda_fail(e, "KeySwitch H2D");
        break;
      }
      if (hoisted)
        rc = hoisted_rotations_on_device(dev, d_res, d_t, n, decomp, key_modulus_size, rns, moduli, dk.data(),
                                         hoisted_elts, num_elts, modswitch, sx);
      else if (galois_elt)
        rc = galois_key_switch_on_device(dev, d_res, d_t, n, decomp, key_modulus_size, rns, moduli, dk[0], modswitch,
                                         galois_elt, sx);
      else
        rc = key_switch_on_device(dev, d_res, d_t, n, decomp, key_modulus_size, rns, kcc, moduli, dk[0], modswitch, sx);
      if (rc) break;
      e = cudaMemcpyAsync(result + c * res_elems, d_res, res_elems * 8, cudaMemcpyDeviceToHost, sx);
      if (e != cudaSuccess) rc = cuda_fail(e, "KeySwitch D2H");
    }
  }
  for (int dev : use) {
    int rc2 = sync_stage(dev);
    if (!rc) rc = rc2;
  }
  return rc;
}

static int key_switch_check(const void* result, const void* t_target, uint64_t n, uint64_t decomp,
                            uint64_t key_modulus_size, uint64_t rns, uint64_t kcc, const uint64_t* moduli,
                            const uint64_t* modswitch) {
  REQUIRE(result && t_target && moduli && modswitch, "Require non-null arguments");
  REQUIRE(n >= 2 && !(n & (n - 1)), "Require n a power of two");
  REQUIRE(decomp >= 1 && kcc >= 1, "Require decomp_modulus_size, key_component_count >= 1");
  REQUIRE(rns == decomp + 1, "Require rns_modulus_size == decomp_modulus_size + 1");
  REQUIRE(key_modulus_size >= rns, "Require key_modulus_size >= rns_modulus_size");
  return 0;
}

int hexl_b200_keys_upload(hexl_b200_keys** out, const uint64_t* const* k_switch_keys, uint64_t n,
                          uint64_t decomp, uint64_t key_modulus_size, uint64_t kcc) {
  REQUIRE(out && k_switch_keys, "Require out, k_switch_keys != nullptr");
  *out = nullptr;
  REQUIRE(n >= 1 && decomp >= 1 && kcc >= 1 && key_modulus_size >= 1, "Require non-zero sizes");
  for (uint64_t j = 0; j < decomp; ++j) REQUIRE(k_switch_keys[j] != nullptr, "Require k_switch_keys[j] != nullptr");
  std::vector<int> devs = host_devices();
  if (devs.empty()) {
    int cur = 0;
    CU(cudaGetDevice(&cur));
    devs.push_back(cur);
  }
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
  auto ki = [&](uint64_t i) { return i == decomp ? key_modulus_size - 1 : i; };
  std::vector<hexl_b200_ntt*> h(rns, nullptr);
  struct Release {
    std::vector<hexl_b200_ntt*>& v;
    ~Release() {
      for (auto* p : v)
        if (p) hexl_b200_ntt_release(p);
    }
  } release{h};
  for (uint64_t i = 0; i < rns; ++i) {
    if (moduli[ki(i)] >= (1ull << 61)) return fail(HEXL_B200_ERR_INVALID_ARG, "KeySwitch: Require moduli < 2^61");
    if (int rc = cached_ntt(&h[i], n, moduli[ki(i)])) return rc;
  }
  const size_t row = (size_t)decomp * n * sizeof(uint64_t);  // host pitch of result: one key component over all moduli
  const uint64_t q_last = moduli[key_modulus_size - 1], mu_last = nt::multiply_factor(1, 64, q_last);

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
    for (uint64_t e0 = 0; e0 < cnt && !rc && !first_error.load(); e0 += kParamBlock) {
      const uint64_t c = std::min<uint64_t>(kParamBlock, cnt - e0);
      KsModuli mods;
      for (uint64_t e = 0; e < c; ++e) {
        const uint64_t q = moduli[ki(z.lo + e0 + e)], mu = nt::multiply_factor(1, 64, q);
        const Twiddle R = make_twiddle((mu * (0 - q)) % q, q);  // 2^64 mod q
        mods.m[e] = KsModulus{q, mu, R.w, R.wp, e0 + e};        // key slot = index inside the shard
      }
      if (bad(ntt_multi_on_device(true, z.device, h.data() + z.lo + e0, c, z.ops + e0 * per_mod, z.t_coef, 4, decomp, z.stream, nullptr, true))) break;
      const uint64_t jmax = ks_mac_digits_per_launch(mods, c);
      for (uint64_t j0 = 0; j0 < decomp && !rc; j0 += jmax) {
        const uint64_t jc = std::min<uint64_t>(jmax, decomp - j0);
        KeyPointers kp;
        for (uint64_t j = 0; j < jc; ++j) kp.p[j] = z.keys[j0 + j];
        cu(launch_ks_mac(z.prod + e0 * kcc * n, z.ops + e0 * per_mod + j0 * n, per_mod, kp, n, jc, kcc, cnt, c, mods, j0 != 0, z.stream), "ks_mac");
      }
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
      for (uint64_t e0 = 0; e0 < nd && !rc; e0 += kParamBlock) {
        const uint64_t c = std::min<uint64_t>(kParamBlock, nd - e0);
        KsModuli round_mods, fin_mods;
        for (uint64_t e = 0; e < c; ++e) {
          const uint64_t i = z.lo + e0 + e, qi = moduli[i], mu_i = nt::multiply_factor(1, 64, qi);
          round_mods.m[e] = KsModulus{qi, mu_i, qi - ((q_last >> 1) % qi), 0, 0};
          const Twiddle ms = make_twiddle(modswitch[i] % qi, qi);
          fin_mods.m[e] = KsModulus{qi, mu_i, ms.w, ms.wp, 0};
        }
        uint64_t* tmp_c = z.tmp + e0 * kcc * n;
        if (cu(launch_ks_round(tmp_c, z.t_last, n, kcc, q_last, mu_last, c, round_mods, z.stream), "ks_round")) break;
        if (bad(ntt_multi_on_device(true, z.device, h.data() + z.lo + e0, c, tmp_c, tmp_c, 4, kcc, z.stream))) break;
        cu(launch_ks_finish(z.res, z.prod + e0 * kcc * n, tmp_c, n, kcc, nd, e0, c, fin_mods, false, true, z.stream),
           "ks_finish");
      }
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

int hexl_b200_keys_upload_sharded(hexl_b200_keys** out, const uint64_t* const* k_switch_keys, uint64_t n,
                                  uint64_t decomp, uint64_t key_modulus_size, uint64_t kcc) {
  REQUIRE(out && k_switch_keys, "Require out, k_switch_keys != nullptr");
  *out = nullptr;
  REQUIRE(n >= 2 && !(n & (n - 1)), "Require n a power of two");
  REQUIRE(decomp >= 1 && kcc >= 1 && key_modulus_size >= decomp + 1, "Require decomp, kcc >= 1 and key_modulus_size > decomp");
  for (uint64_t j = 0; j < decomp; ++j) REQUIRE(k_switch_keys[j] != nullptr, "Require k_switch_keys[j] != nullptr");
  std::vector<int> devs = host_devices();
  if (devs.empty()) {
    int cur = 0;
    CU(cudaGetDevice(&cur));
    devs.push_back(cur);
  }
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
  REQUIRE(keys->n == n && keys->decomp >= decomp && keys->kcc == kcc && keys->kms == key_modulus_size,
          "the key handle was uploaded for another shape");
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
    return key_switch_host_batch(result, t_target_iter_ptr, n, decomp, key_modulus_size, rns, kcc, moduli, &keys,
                                 modswitch_factors, batch);
  auto it = keys->dev.find(pi.device);
  if (it == keys->dev.end()) return fail(HEXL_B200_ERR_MIXED_POINTERS, "the key handle holds no copy on the device of result");
  DeviceGuard g;
  if (int rc = g.enter(pi.device)) return rc;
  for (uint64_t c = 0; c < batch; ++c)
    if (int rc = key_switch_on_device(pi.device, result + c * kcc * decomp * n, t_target_iter_ptr + c * decomp * n, n, decomp,
                                      key_modulus_size, rns, kcc, moduli, it->second.data(), modswitch_factors,
                                      (cudaStream_t)stream))
      return rc;
  return finish_device_call(pi, stream);
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
  if (pi.where == Where::Device) {
    DeviceGuard g;
    if (int rc = g.enter(pi.device)) return rc;
    if (int rc = key_switch_on_device(pi.device, result, t_target_iter_ptr, n, decomp, key_modulus_size, rns, kcc,
                                      moduli, k_switch_keys, modswitch_factors, (cudaStream_t)stream))
      return rc;
    return finish_device_call(pi, stream);
  }
  // Host pointers, the reference's call shape (key-switch.hpp:34-39 keeps the keys in caller memory): the keys
  // cross PCIe on every call.  A caller that switches more than once with the same keys uploads them once
  // (hexl_b200_keys_upload) and calls hexl_b200_key_switch_resident.
  hexl_b200_keys* tmp = nullptr;
  if (int rc = hexl_b200_keys_upload(&tmp, k_switch_keys, n, decomp, key_modulus_size, kcc)) return rc;
  const int rc = key_switch_host_batch(result, t_target_iter_ptr, n, decomp, key_modulus_size, rns, kcc, moduli, &tmp,
                                       modswitch_factors, 1);
  hexl_b200_keys_release(tmp);
  return rc;
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

int hexl_b200_divide_and_round_q_last(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                                      uint64_t rns_modulus_size, uint64_t count, int ntt_form, void* stream) {
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
  std::vector<hexl_b200_ntt*> h(ntt_form ? rns : 0, nullptr);
  struct Release {
    std::vector<hexl_b200_ntt*>& v;
    ~Release() {
      for (auto* p : v)
        if (p) hexl_b200_ntt_release(p);
    }
  } release{h};
  for (uint64_t i = 0; i < h.size(); ++i)
    if (int rc = cached_ntt(&h[i], n, moduli[i])) return rc;
  if (g_debug.load())
    for (uint64_t p = 0; p < count; ++p)
      for (uint64_t i = 0; i < rns; ++i)
        if (int rc = check_bounds(operand + p * unit + i * n, n, moduli[i], pi, "operand")) return rc;
  const bool ntt = ntt_form != 0;
  if (pi.where == Where::Device) {
    DeviceGuard g;
    if (int rc = g.enter(pi.device)) return rc;
    if (int rc = divide_and_round_on_device(pi.device, result, operand, n, moduli, rns, count, ntt, h.data(),
                                            (cudaStream_t)stream))
      return rc;
    return finish_device_call(pi, stream);
  }
  // host pointers: whole polynomials through the staging slots (split over the host devices when set); only limbs
  // [0, L) of each polynomial are copied back, so limb L of result is left as it was
  struct Launch {
    bool ok = true;
    int rc = 0;
    int dev;
    uint64_t n, rns, unit;
    const uint64_t* moduli;
    bool ntt;
    hexl_b200_ntt* const* h;
    int operator()(u64* r, const u64* a, const u64*, u64, u64 elems, cudaStream_t s) const {
      return divide_and_round_on_device(dev, r, a, n, moduli, rns, elems / unit, ntt, h, s);
    }
  };
  return run_host(result, operand, nullptr, total, unit,
                  [&](int dev, u64, u64) { return Launch{true, 0, dev, n, rns, unit, moduli, ntt, h.data()}; },
                  L * n);
}

// ---------------------------------------------------------------- Galois automorphisms
static int galois_elt_check(uint64_t n, uint64_t galois_elt) {
  REQUIRE(galois_elt % 2 == 1 && galois_elt < 2 * n, "Require galois_elt odd and in [1, 2n)");
  return 0;
}

// g^-1 mod 2n (g odd): Newton's iteration doubles the correct low bits of an inverse mod 2^64 (g is its own inverse
// mod 8), so five steps give all 64
static uint64_t galois_inverse(uint64_t g, uint64_t n) {
  uint64_t inv = g;
  for (int i = 0; i < 5; ++i) inv *= 2 - g * inv;
  return inv & (2 * n - 1);
}

// `count` polynomials of rns limbs x n words, device pointers on the current device.  NTT form: one launch over every
// limb; coefficient form: one launch per block of kParamBlock moduli.  In place, the polynomials are first copied into
// pool scratch (at most ~256 MiB at a time, whole polynomials) and permuted from there back into result.
static int apply_galois_on_device(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                                  uint64_t rns, uint64_t count, uint64_t galois_elt, bool ntt_form, cudaStream_t s) {
  const int log_n = floor_log2(n);
  const uint64_t g_inv = galois_inverse(galois_elt, n), unit = rns * n;
  auto permute = [&](uint64_t* r, const uint64_t* a, uint64_t polys) -> int {
    if (ntt_form) {
      cudaError_t e = launch_galois_ntt(r, a, log_n, polys * rns, galois_elt, s);
      if (e != cudaSuccess) return cuda_fail(e, "ApplyGalois launch");
      return 0;
    }
    for (uint64_t i0 = 0; i0 < rns; i0 += kParamBlock) {
      const uint64_t cnt = std::min<uint64_t>(kParamBlock, rns - i0);
      GaloisModuli mods;
      for (uint64_t e = 0; e < cnt; ++e) mods.q[e] = moduli[i0 + e];
      cudaError_t e = launch_galois_coef(r, a, log_n, rns, i0, cnt, polys, g_inv, mods, s);
      if (e != cudaSuccess) return cuda_fail(e, "ApplyGalois launch");
    }
    return 0;
  };
  if (result != operand) return permute(result, operand, count);
  const uint64_t chunk = std::min<uint64_t>(count, std::max<uint64_t>(1, (256ull << 20) / (unit * 8)));
  Scratch ws(s);
  uint64_t* copy = nullptr;
  if (int rc = ws.get(&copy, chunk * unit)) return rc;
  for (uint64_t p0 = 0; p0 < count; p0 += chunk) {
    const uint64_t cnt = std::min(chunk, count - p0);
    CU(cudaMemcpyAsync(copy, result + p0 * unit, cnt * unit * 8, cudaMemcpyDeviceToDevice, s));
    if (int rc = permute(result + p0 * unit, copy, cnt)) return rc;
  }
  return 0;  // ~Scratch returns the copy to the pool in stream order
}

int hexl_b200_apply_galois(uint64_t* result, const uint64_t* operand, uint64_t n, const uint64_t* moduli,
                           uint64_t rns_modulus_size, uint64_t count, uint64_t galois_elt, int ntt_form, void* stream) {
  REQUIRE(result && operand && moduli, "Require result, operand, moduli != nullptr");
  REQUIRE(rns_modulus_size >= 1, "Require rns_modulus_size >= 1");
  REQUIRE(ntt_form == 0 || ntt_form == 1, "Require ntt_form = 0 or 1");
  REQUIRE(n >= 2 && n <= (1ull << 20) && !(n & (n - 1)), "Require n a power of two in [2, 2^20]");
  const uint64_t rns = rns_modulus_size;
  for (uint64_t i = 0; i < rns; ++i)
    REQUIRE(moduli[i] > 1 && moduli[i] < (1ull << 62), "Require 1 < moduli[%llu] < 2^62", (unsigned long long)i);
  if (int rc = galois_elt_check(n, galois_elt)) return rc;
  if (count == 0) return 0;
  const uint64_t unit = rns * n, total = count * unit;
  REQUIRE(result == operand || result + total <= operand || operand + total <= result,
          "result and operand must be the same buffer or not overlap");
  PtrInfo pi;
  if (int rc = classify_all({result, operand}, &pi)) return rc;
  if (g_debug.load())
    for (uint64_t p = 0; p < count; ++p)
      for (uint64_t i = 0; i < rns; ++i)
        if (int rc = check_bounds(operand + p * unit + i * n, n, moduli[i], pi, "operand")) return rc;
  const bool ntt = ntt_form != 0;
  if (pi.where == Where::Device) {
    DeviceGuard g;
    if (int rc = g.enter(pi.device)) return rc;
    if (int rc = apply_galois_on_device(result, operand, n, moduli, rns, count, galois_elt, ntt, (cudaStream_t)stream))
      return rc;
    return finish_device_call(pi, stream);
  }
  // host pointers: whole polynomials through the staging slots (split over the host devices when set); the staged
  // polynomials are permuted in place on the device
  struct Launch {
    bool ok = true;
    int rc = 0;
    uint64_t n, rns, unit, galois_elt;
    const uint64_t* moduli;
    bool ntt;
    int operator()(u64* r, const u64* a, const u64*, u64, u64 elems, cudaStream_t s) const {
      return apply_galois_on_device(r, a, n, moduli, rns, elems / unit, galois_elt, ntt, s);
    }
  };
  return run_host(result, operand, nullptr, total, unit,
                  [&](int, u64, u64) { return Launch{true, 0, n, rns, unit, galois_elt, moduli, ntt}; });
}

int hexl_b200_apply_galois_key_switch(uint64_t* ciphertexts, uint64_t n, uint64_t decomp_modulus_size,
                                      uint64_t key_modulus_size, uint64_t rns_modulus_size,
                                      uint64_t key_component_count, const uint64_t* moduli,
                                      const hexl_b200_keys* galois_keys, const uint64_t* modswitch_factors,
                                      uint64_t galois_elt, uint64_t batch, void* stream) {
  const uint64_t decomp = decomp_modulus_size, rns = rns_modulus_size, kcc = key_component_count;
  if (int rc = key_switch_check(ciphertexts, ciphertexts, n, decomp, key_modulus_size, rns, kcc, moduli,
                                modswitch_factors))
    return rc;
  REQUIRE(kcc == 2, "Require key_component_count == 2 (a ciphertext of two components)");
  REQUIRE(n <= (1ull << 20), "Require n <= 2^20");
  if (int rc = galois_elt_check(n, galois_elt)) return rc;
  REQUIRE(galois_keys != nullptr, "Require galois_keys != nullptr");
  REQUIRE(galois_keys->n == n && galois_keys->decomp >= decomp && galois_keys->kcc == kcc &&
              galois_keys->kms == key_modulus_size,
          "the key handle was uploaded for another shape");
  REQUIRE(galois_keys->shards.empty(),
          "ApplyGaloisKeySwitch does not take keys sharded by modulus: upload them with hexl_b200_keys_upload");
  if (batch == 0) return 0;
  PtrInfo pi;
  if (int rc = classify_all({ciphertexts}, &pi)) return rc;
  const uint64_t comp = decomp * n;
  if (g_debug.load())
    for (uint64_t c = 0; c < 2 * batch; ++c)
      for (uint64_t i = 0; i < decomp; ++i)
        if (int rc = check_bounds(ciphertexts + c * comp + i * n, n, moduli[i], pi, "ciphertexts")) return rc;
  if (pi.where == Where::Host)
    return key_switch_host_batch(ciphertexts, nullptr, n, decomp, key_modulus_size, rns, kcc, moduli, &galois_keys,
                                 modswitch_factors, batch, galois_elt);
  auto it = galois_keys->dev.find(pi.device);
  if (it == galois_keys->dev.end())
    return fail(HEXL_B200_ERR_MIXED_POINTERS, "the key handle holds no copy on the device of the ciphertexts");
  DeviceGuard g;
  if (int rc = g.enter(pi.device)) return rc;
  Scratch ws((cudaStream_t)stream);
  uint64_t* perm = nullptr;
  if (int rc = ws.get(&perm, 2 * comp)) return rc;
  for (uint64_t c = 0; c < batch; ++c)
    if (int rc = galois_key_switch_on_device(pi.device, ciphertexts + c * 2 * comp, perm, n, decomp, key_modulus_size,
                                             rns, moduli, it->second.data(), modswitch_factors, galois_elt,
                                             (cudaStream_t)stream))
      return rc;
  return finish_device_call(pi, stream);
}

int hexl_b200_apply_galois_key_switch_hoisted(uint64_t* results, const uint64_t* ciphertexts, uint64_t n,
                                              uint64_t decomp_modulus_size, uint64_t key_modulus_size,
                                              uint64_t rns_modulus_size, uint64_t key_component_count,
                                              const uint64_t* moduli, const hexl_b200_keys* const* galois_keys,
                                              const uint64_t* galois_elts, uint64_t num_elts,
                                              const uint64_t* modswitch_factors, uint64_t batch, void* stream) {
  const uint64_t decomp = decomp_modulus_size, rns = rns_modulus_size, kcc = key_component_count;
  if (int rc = key_switch_check(results, ciphertexts, n, decomp, key_modulus_size, rns, kcc, moduli,
                                modswitch_factors))
    return rc;
  REQUIRE(kcc == 2, "Require key_component_count == 2 (a ciphertext of two components)");
  REQUIRE(n <= (1ull << 20), "Require n <= 2^20");
  REQUIRE(num_elts == 0 || (galois_keys && galois_elts), "Require galois_keys, galois_elts != nullptr");
  for (uint64_t r = 0; r < num_elts; ++r) {
    if (int rc = galois_elt_check(n, galois_elts[r])) return rc;
    const hexl_b200_keys* k = galois_keys[r];
    REQUIRE(k != nullptr, "Require galois_keys[%llu] != nullptr", (unsigned long long)r);
    REQUIRE(k->n == n && k->decomp >= decomp && k->kcc == kcc && k->kms == key_modulus_size,
            "galois_keys[%llu] was uploaded for another shape", (unsigned long long)r);
    REQUIRE(k->shards.empty(),
            "ApplyGaloisKeySwitchHoisted does not take keys sharded by modulus: upload them with hexl_b200_keys_upload");
  }
  if (num_elts == 0 || batch == 0) return 0;
  const uint64_t comp = decomp * n, in_total = batch * 2 * comp, out_total = batch * num_elts * 2 * comp;
  REQUIRE(results + out_total <= ciphertexts || ciphertexts + in_total <= results,
          "results and ciphertexts must not overlap");
  PtrInfo pi;
  if (int rc = classify_all({results, ciphertexts}, &pi)) return rc;
  if (g_debug.load())
    for (uint64_t c = 0; c < 2 * batch; ++c)
      for (uint64_t i = 0; i < decomp; ++i)
        if (int rc = check_bounds(ciphertexts + c * comp + i * n, n, moduli[i], pi, "ciphertexts")) return rc;
  if (pi.where == Where::Host)
    return key_switch_host_batch(results, ciphertexts, n, decomp, key_modulus_size, rns, kcc, moduli, galois_keys,
                                 modswitch_factors, batch, 0, galois_elts, num_elts);
  std::vector<const uint64_t* const*> dk(num_elts);
  for (uint64_t r = 0; r < num_elts; ++r) {
    auto it = galois_keys[r]->dev.find(pi.device);
    if (it == galois_keys[r]->dev.end())
      return fail(HEXL_B200_ERR_MIXED_POINTERS, "galois_keys[%llu] holds no copy on the device of the ciphertexts",
                  (unsigned long long)r);
    dk[r] = it->second.data();
  }
  DeviceGuard g;
  if (int rc = g.enter(pi.device)) return rc;
  for (uint64_t c = 0; c < batch; ++c)
    if (int rc = hoisted_rotations_on_device(pi.device, results + c * num_elts * 2 * comp, ciphertexts + c * 2 * comp,
                                             n, decomp, key_modulus_size, rns, moduli, dk.data(), galois_elts,
                                             num_elts, modswitch_factors, (cudaStream_t)stream))
      return rc;
  return finish_device_call(pi, stream);
}

}  // extern "C"
