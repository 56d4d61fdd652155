// NTT handles, their tables and the cache of GetNTT, and the single- and multi-modulus transforms.
#include "capi.h"

using namespace hexl_b200;

namespace hexl_b200 {

bool check_ntt_arguments(uint64_t degree, uint64_t q, const char** why) {
  // NTT::CheckArguments, hexl/ntt/ntt-internal.cpp:171-186
  if (degree < 2 || (degree & (degree - 1))) { *why = "degree is not a power of 2 (>= 2)"; return false; }
  if (degree > (1ull << 20)) { *why = "degree should be at most 2^20"; return false; }
  if (q > (1ull << 62)) { *why = "modulus should be at most 2^62"; return false; }
  if (q % (2 * degree) != 1) { *why = "modulus mod 2n != 1"; return false; }
  if (!nt::is_prime(q)) { *why = "modulus is not prime"; return false; }
  return true;
}

static Twiddle32 make_twiddle32(uint64_t v, uint64_t q) { return Twiddle32{(uint32_t)v, (uint32_t)((v << 32) / q)}; }

// hexl/ntt/ntt-internal.cpp:54-169 restated: psi^i goes to slot bitrev(i); the
// inverse powers are additionally listed in the order the reference's inverse
// transform consumes them (m = N/2 groups first, ..., m = 1 last).
static void build_tables(hexl_b200_ntt* h) {
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

// A tree in the order of its device copy (internal.h): the deepest four levels lane-major where the rows are 4096
// points, node order elsewhere.
static std::vector<Twiddle> device_order(const std::vector<Twiddle>& tree, int log_n) {
  std::vector<Twiddle> out(tree);
  if (!twiddle_lanes_major(log_n)) return out;
  for (int j = 0; j < 4; ++j) {
    const uint64_t level = 1ull << (log_n - 4 + j);
    for (uint64_t i = 0; i < level; ++i)
      out[level + lane_major((unsigned)(i >> j), (unsigned)(i & ((1u << j) - 1)), j)] = tree[level + i];
  }
  return out;
}

int device_tables(hexl_b200_ntt* h, int dev, NttDeviceTables* out, cudaStream_t user_stream) {
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
#define CU_T(call)                                        \
  do {                                                    \
    cudaError_t e__ = (call);                             \
    if (e__ != cudaSuccess) {                             \
      d.free();                                           \
      return cuda_fail(e__, #call);                       \
    }                                                     \
  } while (0)
    const size_t bytes = h->n * sizeof(Twiddle);
    const std::vector<Twiddle> fwd = device_order(h->fwd_tree, h->log_n), inv = device_order(h->inv_tree, h->log_n);
    CU_T(cudaMalloc(&d.fwd, bytes));
    CU_T(cudaMalloc(&d.inv, bytes));
    CU_T(cudaMemcpy(d.fwd, fwd.data(), bytes, cudaMemcpyHostToDevice));
    CU_T(cudaMemcpy(d.inv, inv.data(), bytes, cudaMemcpyHostToDevice));
    if (h->q < kSmallModulusLimit) {
      std::vector<Twiddle32> f32(h->n), i32(h->n);
      for (uint64_t k = 0; k < h->n; ++k) {
        f32[k] = make_twiddle32(fwd[k].w, h->q);
        i32[k] = make_twiddle32(inv[k].w, h->q);
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

static int create_common(hexl_b200_ntt** out, uint64_t degree, uint64_t q, uint64_t root, bool have_root) {
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

// ------------------------------------------------------------ NTT cache
// GetNTT(N, modulus) of the reference (hexl/include/hexl/experimental/seal/ntt-cache.hpp:27-53)
static std::mutex g_cache_mu;
static std::map<std::pair<uint64_t, uint64_t>, hexl_b200_ntt*> g_ntt_cache;

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

static int ntt_compute(bool forward, hexl_b200_ntt* h, uint64_t* result, const uint64_t* operand,
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
  if (int rc = check_bounds(operand, batch * h->n, h->q * in_mf, pi, "operand", stream)) return rc;
  const uint64_t n = h->n;
  auto launch = [&](const NttDeviceTables& t, u64* r, const u64* a, u64 polys, cudaStream_t s) {
    return forward ? launch_ntt_forward(t, r, a, (int)in_mf, (int)out_mf, polys, s)
                   : launch_ntt_inverse(t, r, a, (int)in_mf, (int)out_mf, polys, s);
  };
  if (pi.where == Where::Device)
    return run_on_device(pi, stream, [&] {
      NttDeviceTables t;
      if (int rc = device_tables(h, pi.device, &t, (cudaStream_t)stream)) return rc;
      cudaError_t e = launch(t, result, operand, batch, (cudaStream_t)stream);
      return e == cudaSuccess ? 0 : cuda_fail(e, "NTT launch");
    });
  return run_host(result, operand, nullptr, batch * n, n, [&](int dev, u64, u64, auto&& run) {
    DeviceGuard g;
    NttDeviceTables t;
    if (int rc = g.enter(dev)) return rc;
    if (int rc = device_tables(h, dev, &t)) return rc;
    return run([&](u64* r, const u64* a, const u64*, u64, u64 elems, cudaStream_t s) {
      return launch(t, r, a, elems / n, s);
    });
  });
}

static int ntt_compute_multi(bool forward, hexl_b200_ntt* const* handles, uint64_t count, uint64_t* result,
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
  if (int rc = check_limb_bounds(operand, 1, count, group * n, [&](u64 i) { return handles[i]->q * in_mf; }, pi,
                                 "operand", stream))
    return rc;
  if (pi.where == Where::Host)  // staged, chunked and (with host devices set) split across GPUs like a single-modulus call
    return run_host_rns(forward ? RnsJob::NttFwd : RnsJob::NttInv, handles, nullptr, count, group * n, n, (int)in_mf,
                        (int)out_mf, result, operand, nullptr);
  return run_on_device(pi, stream, [&] {
    return ntt_multi_on_device(forward, pi.device, handles, count, result, operand, (int)out_mf, group,
                               (cudaStream_t)stream);
  });
}

}  // namespace hexl_b200

// =============================================================== extern "C"
extern "C" {

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
  for (auto& kv : h->dev)
    if (cudaSetDevice(kv.first) == cudaSuccess) kv.second.free();
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

int hexl_b200_ntt_get_cached(hexl_b200_ntt** out, uint64_t degree, uint64_t q) {
  if (!out) return fail(HEXL_B200_ERR_INVALID_ARG, "out == nullptr");
  return cached_ntt(out, degree, q);
}

}  // extern "C"
