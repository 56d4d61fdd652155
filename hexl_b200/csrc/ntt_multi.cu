// Multi-modulus NTT launches: ONE launch transforms `units` polynomials back to back,
// polynomial u under the modulus of entry u / group.  This is the RNS shape of the
// callers of the reference's NTT (every ciphertext polynomial exists once per modulus;
// KeySwitch re-transforms every digit under every modulus, key-switch-internal.cpp:60-131):
// with one launch per (polynomial, modulus) those workloads are bound by launch latency,
// not by arithmetic.  Same kernels bodies as ntt.cu; the only difference is where the
// twiddle pointer and the modulus constants come from -- a device-resident record per
// (N, q) (NttDeviceParams) found through a pointer list in the kernel parameters.
#include "ntt_kernels.cuh"

namespace hexl_b200 {
namespace {

// Each thread loads the record of its own polynomial.  A column CTA lies inside one sub-block of one polynomial, but a
// row CTA can span several: below N = 4096 a polynomial is one row of N / 16 threads and a CTA holds 4096 / N rows, so
// with a small group its rows belong to polynomials under different moduli.
__device__ __forceinline__ NttDeviceParams load_params(const NttMulti& multi, u64 poly) {
  return *multi.p[poly / multi.group];
}

// each row takes the modulus of its own polynomial (load_params per row), so a CTA may span moduli
// MUL (inverse only): multiply by multi.mul on load -- a separate instantiation, so the plain inverse keeps its code
template <int MODE, int LOGC, bool FWD, bool MUL = false>
__global__ void __launch_bounds__(RowCfg<LOGC, MODE>::THREADS, RowCfg<LOGC, MODE>::MIN_BLOCKS)
    ntt_row_multi(u64* result, const u64* operand, const __grid_constant__ NttMulti multi, u64 total_rows,
                  unsigned rows_per_poly, int out_mf, int fold, unsigned gather) {
  using Cfg = RowCfg<LOGC, MODE>;
  extern __shared__ __align__(16) unsigned char smem[];
  const unsigned row_local = threadIdx.x / Cfg::T, u = threadIdx.x % Cfg::T;
  u64 row = (u64)blockIdx.x * Cfg::ROWS + row_local;
  const bool active = row < total_rows;
  if (!active) row = total_rows - 1;
  const NttDeviceParams P = load_params(multi, row / rows_per_poly);
  const Mod m = make_mod(P.q, P.mu);
  const u64 base = (u64)rows_per_poly + (row % rows_per_poly);
  typename Cfg::E* srow = reinterpret_cast<typename Cfg::E*>(smem + (size_t)row_local * Cfg::ROW_BYTES);
  if (FWD) {
    // gather (first kernel of a forward transform only): read the same row of polynomial (poly % gather)
    const u64 poly = row / rows_per_poly;
    const u64 src_row = gather ? (poly % gather) * rows_per_poly + row % rows_per_poly : row;
    row_fwd_body<MODE, LOGC, kStream, kStream>(result + row * Cfg::C, operand + src_row * Cfg::C, srow, u, base, P.fwd, m,
                                               out_mf, active, nullptr, gather != 0);
  } else {
    const MirrorList mir{multi.mirror, multi.mirrors, row * Cfg::C};
    const ProdIn prod{MUL ? multi.mul + row * Cfg::C : nullptr, P.prod_mu, P.prod_shift};
    row_inv_body<MODE, LOGC, kStream, kStream>(result + row * Cfg::C, operand + row * Cfg::C, srow, u, base, P.inv, m,
                                               out_mf, fold != 0, P.inv_n, P.inv_n_w, active, nullptr,
                                               &mir, MUL ? &prod : nullptr);
  }
}

template <int MODE, int LOGR, bool FWD>
__global__ void __launch_bounds__(256)
    ntt_col_multi(u64* result, const u64* operand, const __grid_constant__ NttMulti multi, int log_n, int log_s,
                  u64 total_cols, int out_mf, int fold, unsigned gather) {
  constexpr int R = 1 << LOGR;
  __shared__ Twiddle stw[R];
  const int log_cols = log_s - LOGR;
  const u64 g0 = (u64)blockIdx.x * blockDim.x;
  const u64 blk = g0 >> log_cols;                    // sub-block index over the whole batch
  const u64 blocks_per_poly = 1ull << (log_n - log_s);
  const NttDeviceParams P = load_params(multi, blk >> (log_n - log_s));
  const Mod m = make_mod(P.q, P.mu);
  const Twiddle* tw = FWD ? P.fwd : P.inv;
  const u64 base = blocks_per_poly + (blk & (blocks_per_poly - 1));
  for (int l = threadIdx.x; l < R; l += blockDim.x) {
    if (l == 0) continue;
    const int s = 31 - __clz(l);
    stw[l] = ld_tw(tw + (base << s) + (l - (1 << s)));
  }
  __syncthreads();
  const u64 g = g0 + threadIdx.x;
  if (g >= total_cols) return;
  const u64 c = g & ((1ull << log_cols) - 1);
  const MirrorList mir{multi.mirror, multi.mirrors, 0};
  // gather (first column pass of a forward transform: log_s == log_n, one sub-block per polynomial): the source is
  // polynomial (poly % gather); col_body adds the same offset to both pointers, so the operand base is shifted
  const u64 poly = blk >> (log_n - log_s);
  const u64* src = (FWD && gather) ? operand + (((poly % gather) - poly) << log_n) : operand;
  col_body<MODE, LOGR, FWD, kStream, kStream>(result, src, (blk << log_s) + c, log_cols, stw, m, out_mf,
                                              !FWD && fold && log_s == log_n, P.inv_n, P.inv_n_w,
                                              FWD ? nullptr : &mir, FWD && gather != 0);
}

// The persistent pipelined forward kernel of ntt_kernels.cuh (ntt_pipe_fwd) for RNS batches: the same work queue,
// producer/consumer counters and L2-resident intermediate; the modulus record of a work item comes from the
// polynomial it belongs to, and the root sub-tree twiddles are re-staged when a CTA's next item has another modulus.
template <int MODE, int LOGR>
__global__ void __launch_bounds__(PipeCfg<LOGR>::THREADS, PipeCfg<LOGR>::MIN_BLOCKS)
    ntt_pipe_multi(u64* result, const u64* operand, const __grid_constant__ NttMulti multi, int out_mf, unsigned units,
                   unsigned lookahead, unsigned* counter, unsigned* done) {
  using Cfg = PipeCfg<LOGR>;
  using E = typename Ar<MODE>::E;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  E* smem = reinterpret_cast<E*>(smem_raw);
  __shared__ Twiddle stw[Cfg::R];
  __shared__ unsigned s_item;
  const unsigned total = (units + lookahead) * Cfg::SLOTS;
  unsigned staged = ~0u;                              // modulus entry whose root twiddles sit in stw
  while (true) {
    __syncthreads();
    if (threadIdx.x == 0) s_item = atomicAdd(counter, 1u);
    __syncthreads();
    const unsigned item = s_item;
    if (item >= total) break;
    const unsigned blk = item / Cfg::SLOTS, j = item % Cfg::SLOTS;
    const bool producer = j < (unsigned)Cfg::CT;      // column tile j of polynomial blk, else row j - CT of blk - D
    if (producer ? blk >= units : blk < lookahead) continue;
    const unsigned poly = producer ? blk : blk - lookahead;
    const unsigned entry = poly / multi.group;
    const NttDeviceParams P = *multi.p[entry];
    const Mod m = make_mod(P.q, P.mu);
    if (entry != staged) {                            // uniform across the CTA
      for (int l = threadIdx.x; l < Cfg::R; l += Cfg::THREADS)
        if (l) stw[l] = ld_tw(P.fwd + l);
      staged = entry;
      __syncthreads();
    }
    const u64 poly_off = (u64)poly << (Cfg::LOGC + LOGR);
    if (!producer) {
      if (threadIdx.x == 0)
        while (ld_acquire_gpu(done + poly) < (unsigned)Cfg::CT) __nanosleep(100);
      __syncthreads();
    }
    if (producer) {
      col_body<MODE, LOGR, true, kStream, kViaL2>(result, operand, poly_off + j * Cfg::THREADS + threadIdx.x, Cfg::LOGC,
                                                  stw, m, out_mf, false, Twiddle{}, Twiddle{});
    } else {
      const unsigned r = j - Cfg::CT;
      u64* row = result + poly_off + (u64)r * Cfg::C;
      row_fwd_body<MODE, Cfg::LOGC, kViaL2, kStream>(row, row, smem, threadIdx.x, (u64)Cfg::R + r, P.fwd, m, out_mf,
                                                     true);
    }
    if (producer) {
      __syncthreads();
      if (threadIdx.x == 0) red_release_gpu(done + poly, 1u);
    }
  }
}

// N = 2^LOGN < 16: one thread per polynomial, everything in registers (launch-bound shapes only)
template <bool FWD, int LOGN>
__global__ void ntt_tiny_multi(u64* result, const u64* operand, const __grid_constant__ NttMulti multi, u64 units,
                               int out_mf) {
  const u64 unit = (u64)blockIdx.x * blockDim.x + threadIdx.x;
  if (unit >= units) return;
  const NttDeviceParams P = *multi.p[unit / multi.group];
  const Mod m = make_mod(P.q, P.mu);
  constexpr int n = 1 << LOGN;
  u64 v[n];
  const u64 src_unit = (FWD && multi.gather) ? unit % multi.gather : unit;
  static_for<0, n>([&](auto I) {
    constexpr int e = I;
    v[e] = operand[src_unit * n + e];
    if (FWD && multi.gather) v[e] %= P.q;
    if (!FWD && multi.mul) v[e] = prod_lazy<kGeneric>(v[e], multi.mul[unit * n + e], m, P.prod_mu, P.prod_shift);
  });
  static_for<0, LOGN>([&](auto K) {
    constexpr int k = K;
    constexpr int s = FWD ? k : LOGN - 1 - k;  // stage: 2^s groups, span t
    constexpr int t = n >> (s + 1);
    static_for<0, (1 << s)>([&](auto I) {
      constexpr int i = I;
      static_for<0, t>([&](auto J) {
        constexpr int j = J;
        u64& X = v[2 * i * t + j];
        u64& Y = v[2 * i * t + j + t];
        if constexpr (FWD)
          fwd_bfly<kGeneric>(X, Y, P.fwd[(1 << s) + i], m);
        else if constexpr (s == 0)
          inv_bfly_last<kGeneric>(X, Y, P.inv_n, P.inv_n_w, m, m.two_q);
        else
          inv_bfly<kGeneric>(X, Y, P.inv[(1 << s) + i], m, m.two_q);
      });
    });
  });
  static_for<0, n>([&](auto I) {
    constexpr int e = I;
    result[unit * n + e] = FWD ? fwd_out<kGeneric>(v[e], m, out_mf) : inv_out<kGeneric>(v[e], m, out_mf);
  });
  if (!FWD)
    for (unsigned p = 0; p < multi.mirrors; ++p)
      static_for<0, n>([&](auto I) {
        constexpr int e = I;
        multi.mirror[p][unit * n + e] = inv_out<kGeneric>(v[e], m, out_mf);
      });
}

template <int MODE, int LOGC>
cudaError_t launch_row_multi(bool fwd, const NttMulti& multi, int log_n, u64* result, const u64* operand, u64 units,
                             int out_mf, int fold, cudaStream_t stream, unsigned gather = 0) {
  using Cfg = RowCfg<LOGC, MODE>;
  const unsigned rows_per_poly = 1u << (log_n - LOGC);
  const u64 total_rows = units * rows_per_poly;
  const unsigned grid = (unsigned)((total_rows + Cfg::ROWS - 1) / Cfg::ROWS);
  if (fwd) {
    if (cudaError_t e = ensure_dynamic_smem<ntt_row_multi<MODE, LOGC, true>>(Cfg::SMEM)) return e;
    ntt_row_multi<MODE, LOGC, true><<<grid, Cfg::THREADS, Cfg::SMEM, stream>>>(result, operand, multi, total_rows,
                                                                               rows_per_poly, out_mf, fold, gather);
  } else if (multi.mul) {
    if (cudaError_t e = ensure_dynamic_smem<ntt_row_multi<MODE, LOGC, false, true>>(Cfg::SMEM)) return e;
    ntt_row_multi<MODE, LOGC, false, true><<<grid, Cfg::THREADS, Cfg::SMEM, stream>>>(result, operand, multi, total_rows,
                                                                                      rows_per_poly, out_mf, fold, 0u);
  } else {
    if (cudaError_t e = ensure_dynamic_smem<ntt_row_multi<MODE, LOGC, false>>(Cfg::SMEM)) return e;
    ntt_row_multi<MODE, LOGC, false><<<grid, Cfg::THREADS, Cfg::SMEM, stream>>>(result, operand, multi, total_rows,
                                                                                rows_per_poly, out_mf, fold, 0u);
  }
  count_launch();
  return cudaGetLastError();
}

template <int MODE>
cudaError_t launch_row_multi_dyn(int log_c, bool fwd, const NttMulti& multi, int log_n, u64* result,
                                 const u64* operand, u64 units, int out_mf, int fold, cudaStream_t stream,
                                 unsigned gather = 0) {
  switch (log_c) {
#define ROW_CASE(L) \
  case L: return launch_row_multi<MODE, L>(fwd, multi, log_n, result, operand, units, out_mf, fold, stream, gather);
    ROW_CASE(4) ROW_CASE(5) ROW_CASE(6) ROW_CASE(7) ROW_CASE(8) ROW_CASE(9) ROW_CASE(10)
    ROW_CASE(11) ROW_CASE(12) ROW_CASE(13)
#undef ROW_CASE
  }
  return cudaErrorInvalidValue;
}

template <int MODE, int LOGR>
cudaError_t launch_col_multi(bool fwd, const NttMulti& multi, int log_n, u64* result, const u64* operand, u64 units,
                             int log_s, int out_mf, int fold, cudaStream_t stream, unsigned gather = 0) {
  const u64 total_cols = (units << log_n) >> LOGR;
  const u64 cols_per_block = 1ull << (log_s - LOGR);
  const unsigned threads = (unsigned)(cols_per_block < 256 ? cols_per_block : 256);
  const unsigned grid = (unsigned)((total_cols + threads - 1) / threads);
  if (fwd)
    ntt_col_multi<MODE, LOGR, true><<<grid, threads, 0, stream>>>(result, operand, multi, log_n, log_s, total_cols,
                                                                  out_mf, fold, gather);
  else
    ntt_col_multi<MODE, LOGR, false><<<grid, threads, 0, stream>>>(result, operand, multi, log_n, log_s, total_cols,
                                                                   out_mf, fold, 0u);
  count_launch();
  return cudaGetLastError();
}

template <int MODE>
cudaError_t launch_col_multi_dyn(int log_r, bool fwd, const NttMulti& multi, int log_n, u64* result,
                                 const u64* operand, u64 units, int log_s, int out_mf, int fold, cudaStream_t stream,
                                 unsigned gather = 0) {
  switch (log_r) {
#define COL_CASE(L) \
  case L: return launch_col_multi<MODE, L>(fwd, multi, log_n, result, operand, units, log_s, out_mf, fold, stream, gather);
    COL_CASE(2) COL_CASE(3) COL_CASE(4) COL_CASE(5)
#undef COL_CASE
  }
  return cudaErrorInvalidValue;
}

template <int MODE>
cudaError_t multi_impl(bool fwd, const NttMulti& multi, int log_n, u64* result, const u64* operand, int out_mf,
                       u64 units, cudaStream_t stream) {
  const unsigned gather = fwd ? multi.gather : 0u;
  // the pipelined kernel: the forward transform at N = 2^17 of a batch deep enough for the pipeline, without gather
  // (multiply-on-load is inverse only)
  if (fwd && !gather && log_n == 17 && units >= 64 && units < (1ull << 31))
    return launch_pipelined<ntt_pipe_multi<MODE, 5>, PipeCfg<5>>(units, stream, result, operand, multi, out_mf);
  const int log_c = pick_row_log(log_n);
  int radices[8];
  const int ncol = plan_col_passes(log_n - log_c, radices);
  if (fwd) {
    const u64* src = operand;
    int log_s = log_n;
    for (int p = 0; p < ncol; ++p) {
      cudaError_t e = launch_col_multi_dyn<MODE>(radices[p], true, multi, log_n, result, src, units, log_s, out_mf, 0, stream,
                                                 p == 0 ? gather : 0u);
      if (e != cudaSuccess) return e;
      log_s -= radices[p];
      src = result;
    }
    return launch_row_multi_dyn<MODE>(log_c, true, multi, log_n, result, src, units, out_mf, 0, stream, ncol == 0 ? gather : 0u);
  }
  cudaError_t e = launch_row_multi_dyn<MODE>(log_c, false, multi, log_n, result, operand, units, out_mf, ncol == 0, stream);
  if (e != cudaSuccess) return e;
  int log_s = log_c;
  for (int p = ncol - 1; p >= 0; --p) {
    log_s += radices[p];
    e = launch_col_multi_dyn<MODE>(radices[p], false, multi, log_n, result, result, units, log_s, out_mf, p == 0, stream);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace

cudaError_t launch_ntt_multi(bool forward, const NttMulti& multi, int log_n, u64 min_q, u64 max_q, u64* result,
                             const u64* operand, int out_mf, u64 units, cudaStream_t stream) {
  if (units == 0) return cudaSuccess;
  if (log_n < 4) {
    const unsigned threads = 128, grid = (unsigned)((units + threads - 1) / threads);
    switch (log_n) {
#define TINY_CASE(L)                                                                                 \
  case L:                                                                                            \
    if (forward)                                                                                     \
      ntt_tiny_multi<true, L><<<grid, threads, 0, stream>>>(result, operand, multi, units, out_mf);  \
    else                                                                                             \
      ntt_tiny_multi<false, L><<<grid, threads, 0, stream>>>(result, operand, multi, units, out_mf); \
    break;
      TINY_CASE(0) TINY_CASE(1) TINY_CASE(2) TINY_CASE(3)
#undef TINY_CASE
      default: return cudaErrorInvalidValue;
    }
    count_launch();
    return cudaGetLastError();
  }
  // FAST needs every modulus in [2^32, 2^56), WIDE every modulus below 2^61 (its doubled lazy ranges
  // are valid for any smaller q as well), GENERIC runs everything
  if (min_q >= (1ull << 32) && max_q < kFastModulusLimit)
    return multi_impl<kFast>(forward, multi, log_n, result, operand, out_mf, units, stream);
  if (max_q < kWideModulusLimit)
    return multi_impl<kWide>(forward, multi, log_n, result, operand, out_mf, units, stream);
  return multi_impl<kGeneric>(forward, multi, log_n, result, operand, out_mf, units, stream);
}

}  // namespace hexl_b200
