// The C ABI's library state (errors, devices, allocation, number theory) and what every operation shares: pointer
// classification, host-pointer staging contexts, the debug bounds checks and the scratch pool.
#include <cstdarg>
#include <cstdio>

#include "capi.h"

using namespace hexl_b200;

namespace {
__global__ void bounds_kernel(const u64* p, u64 n, u64 bound, int* flag) {
  u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  const u64 stride = (u64)gridDim.x * blockDim.x;
  bool bad = false;
  for (; i < n; i += stride) bad |= p[i] >= bound;
  if (bad) atomicExch(flag, 1);
}
}  // namespace

namespace hexl_b200 {
static std::atomic<uint64_t> g_launches{0};
void count_launch(unsigned n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
uint64_t launches_so_far() { return g_launches.load(std::memory_order_relaxed); }

thread_local std::string t_error;
std::atomic<int> g_debug{0};

static std::mutex g_cfg_mu;
static std::vector<int> g_host_devices;  // empty = current device only

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

// ------------------------------------------------------------- pointer kinds
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

int host_devices(std::vector<int>* out) {
  {
    std::lock_guard<std::mutex> lk(g_cfg_mu);
    *out = g_host_devices;
  }
  if (out->empty()) {
    int cur = 0;
    CU(cudaGetDevice(&cur));
    out->push_back(cur);
  }
  return 0;
}

// ----------------------------------------------------------- host-pointer staging
static std::mutex g_stage_mu;
static std::map<int, StageCtx*> g_stage;

StageCtx* stage_for(int dev) {
  std::lock_guard<std::mutex> lk(g_stage_mu);
  auto it = g_stage.find(dev);
  if (it == g_stage.end()) it = g_stage.emplace(dev, new StageCtx()).first;
  return it->second;
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

// ---------------------------------------------------------------- debug checks
int check_bounds(const u64* p, u64 n, u64 bound, const PtrInfo& pi, const char* what, void* stream) {
  if (!g_debug.load() || !p) return 0;
  if (pi.where == Where::Host) {
    for (u64 i = 0; i < n; ++i)
      if (p[i] >= bound) return fail(HEXL_B200_ERR_INVALID_ARG, "%s: element %llu exceeds bound", what, (unsigned long long)i);
    return 0;
  }
  // The check reads the operand in the order of the call's stream, so it sees what the caller queued there before the
  // call, and the host waits for that stream alone.  A capture cannot be waited for, so it is refused before anything
  // is queued on it.  (The legacy default stream cannot be captured, and querying it during another thread's capture
  // would invalidate that capture.)
  const cudaStream_t s = (cudaStream_t)stream;
  if (s) {
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    CU(cudaStreamIsCapturing(s, &cap));
    if (cap != cudaStreamCaptureStatusNone)
      return fail(HEXL_B200_ERR_INVALID_ARG,
                  "%s: the range checks of hexl_b200_set_debug(1) wait for the stream, which is being captured into a "
                  "CUDA graph: turn debug checks off to capture",
                  what);
  }
  DeviceGuard g;
  if (int rc = g.enter(pi.device)) return rc;
  int* flag = nullptr;
  CU(scratch_alloc_async(reinterpret_cast<void**>(&flag), sizeof(int), s));
  int h = 0;
  cudaError_t e = cudaMemsetAsync(flag, 0, sizeof(int), s);
  if (e == cudaSuccess) {
    bounds_kernel<<<296, 256, 0, s>>>(p, n, bound, flag);
    count_launch();
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&h, flag, sizeof(int), cudaMemcpyDeviceToHost, s);
  scratch_free_async(flag, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) return cuda_fail(e, "bounds check");
  if (h) return fail(HEXL_B200_ERR_INVALID_ARG, "%s: an element exceeds its bound", what);
  return 0;
}

int debug_bounds(const u64* p, u64 n, u64 bound, const char* what, std::initializer_list<const void*> all,
                 void* stream) {
  if (!g_debug.load()) return 0;
  PtrInfo pi;
  if (int rc = classify_all(all, &pi)) return rc;
  return check_bounds(p, n, bound, pi, what, stream);
}

// ---------------------------------------------------------------- constant tables
static std::mutex g_table_mu;
static std::map<std::vector<uint64_t>, std::map<int, uint64_t*>> g_tables;

int device_table(const std::vector<uint64_t>& tab, int dev, cudaStream_t user_stream, const uint64_t** out,
                 const char* what) {
  std::lock_guard<std::mutex> lk(g_table_mu);
  auto& per_dev = g_tables[tab];
  auto it = per_dev.find(dev);
  if (it != per_dev.end()) {
    *out = it->second;
    return 0;
  }
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (user_stream && cudaStreamIsCapturing(user_stream, &cap) != cudaSuccess) cudaGetLastError();
  if (cap != cudaStreamCaptureStatusNone)
    return fail(HEXL_B200_ERR_INVALID_ARG,
                "%s for these moduli are not uploaded to this device yet and the stream is being captured: "
                "run the call once before capturing",
                what);
  uint64_t* p = nullptr;
  cudaStream_t s = nullptr;
  CU(cudaMalloc(&p, tab.size() * sizeof(uint64_t)));
  cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMemcpyAsync(p, tab.data(), tab.size() * sizeof(uint64_t), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);  // the copy has landed before any kernel can read the table
  if (s) cudaStreamDestroy(s);
  if (e != cudaSuccess) {
    cudaFree(p);
    return cuda_fail(e, what);
  }
  per_dev[dev] = p;
  *out = p;
  return 0;
}

// ---------------------------------------------------------------- multi-word integers
void big_mul(Big& a, uint64_t x) {
  unsigned __int128 carry = 0;
  for (auto& w : a) {
    carry += (unsigned __int128)w * x;
    w = (uint64_t)carry;
    carry >>= 64;
  }
  if (carry) a.push_back((uint64_t)carry);
}
void big_add_at(Big& a, size_t word, uint64_t x) {
  if (a.size() <= word) a.resize(word + 1, 0);
  for (size_t i = word; x; ++i) {
    if (i == a.size()) a.push_back(0);
    a[i] += x;
    x = a[i] < x ? 1 : 0;
  }
}
bool big_le(Big a, Big b) {
  while (!a.empty() && a.back() == 0) a.pop_back();
  while (!b.empty() && b.back() == 0) b.pop_back();
  if (a.size() != b.size()) return a.size() < b.size();
  for (size_t i = a.size(); i-- > 0;)
    if (a[i] != b[i]) return a[i] < b[i];
  return true;
}
uint64_t big_divmod(Big& a, uint64_t d) {
  unsigned __int128 rem = 0;
  for (size_t i = a.size(); i-- > 0;) {
    const unsigned __int128 cur = (rem << 64) | a[i];
    a[i] = (uint64_t)(cur / d);
    rem = cur % d;
  }
  return (uint64_t)rem;
}
uint64_t big_mod(const Big& a, uint64_t m) {
  unsigned __int128 rem = 0;
  for (size_t i = a.size(); i-- > 0;) rem = ((rem << 64) | a[i]) % m;
  return (uint64_t)rem;
}

// ---------------------------------------------------------------- scratch pool
// Stream-ordered scratch memory for the composites, from a pool of our own per device
// (release threshold = keep everything: a KeySwitch re-uses the same few buffers call
// after call; the process-wide default pool, which other libraries may tune, is left alone).
static std::mutex g_pool_mu;
static std::map<int, cudaMemPool_t> g_pools;

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

cudaError_t scratch_alloc_async(void** p, size_t bytes, cudaStream_t stream) {
  cudaMemPool_t pool;
  if (scratch_pool(&pool)) return cudaErrorMemoryAllocation;
  return cudaMallocFromPoolAsync(p, bytes, pool, stream);
}
void scratch_free_async(void* p, cudaStream_t stream) {
  if (p) cudaFreeAsync(p, stream);
}
}  // namespace hexl_b200

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

}  // extern "C"
