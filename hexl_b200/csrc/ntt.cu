// Single-modulus NTT launchers (the kernels are in ntt_kernels.cuh).
#include <algorithm>

#include "ntt_kernels.cuh"

namespace hexl_b200 {
namespace {

template <int MODE, int LOGC>
cudaError_t launch_row(bool fwd, const NttDeviceTables& t, u64* result, const u64* operand,
                       u64 batch, int out_mf, int fold, cudaStream_t stream) {
  using Cfg = RowCfg<LOGC, MODE>;
  const unsigned rows_per_poly = (unsigned)(t.n >> LOGC);
  const u64 total_rows = batch * rows_per_poly;
  const unsigned grid = (unsigned)((total_rows + Cfg::ROWS - 1) / Cfg::ROWS);
  const Mod m = make_mod(t);
  if (fwd) {
    if (cudaError_t e = ensure_dynamic_smem<ntt_row_fwd<MODE, LOGC>>(Cfg::SMEM)) return e;
    ntt_row_fwd<MODE, LOGC><<<grid, Cfg::THREADS, Cfg::SMEM, stream>>>(result, operand, Tab<MODE>::fwd(t), m,
                                                                       total_rows, rows_per_poly, out_mf);
  } else {
    if (cudaError_t e = ensure_dynamic_smem<ntt_row_inv<MODE, LOGC>>(Cfg::SMEM)) return e;
    ntt_row_inv<MODE, LOGC><<<grid, Cfg::THREADS, Cfg::SMEM, stream>>>(
        result, operand, Tab<MODE>::inv(t), m, total_rows, rows_per_poly, out_mf, fold, Tab<MODE>::inv_n(t),
        Tab<MODE>::inv_n_w(t));
  }
  count_launch();
  return cudaGetLastError();
}

template <int MODE>
cudaError_t launch_row_dyn(int log_c, bool fwd, const NttDeviceTables& t, u64* result,
                           const u64* operand, u64 batch, int out_mf, int fold,
                           cudaStream_t stream) {
  switch (log_c) {
#define ROW_CASE(L) \
  case L: return launch_row<MODE, L>(fwd, t, result, operand, batch, out_mf, fold, stream);
    ROW_CASE(4) ROW_CASE(5) ROW_CASE(6) ROW_CASE(7) ROW_CASE(8) ROW_CASE(9) ROW_CASE(10)
    ROW_CASE(11) ROW_CASE(12) ROW_CASE(13) ROW_CASE(14)
#undef ROW_CASE
  }
  return cudaErrorInvalidValue;
}

template <int MODE, int LOGR>
cudaError_t launch_col(bool fwd, const NttDeviceTables& t, u64* result, const u64* operand,
                       u64 batch, int log_s, int out_mf, int fold, cudaStream_t stream) {
  const u64 total_cols = (batch << t.log_n) >> LOGR;
  const u64 cols_per_block = 1ull << (log_s - LOGR);
  const unsigned threads = (unsigned)(cols_per_block < 256 ? cols_per_block : 256);
  const unsigned grid = (unsigned)((total_cols + threads - 1) / threads);
  const Mod m = make_mod(t);
  if (fwd)
    ntt_col<MODE, LOGR, true><<<grid, threads, 0, stream>>>(result, operand, Tab<MODE>::fwd(t), m, t.log_n, log_s,
                                                            total_cols, out_mf, fold, Tab<MODE>::inv_n(t),
                                                            Tab<MODE>::inv_n_w(t));
  else
    ntt_col<MODE, LOGR, false><<<grid, threads, 0, stream>>>(result, operand, Tab<MODE>::inv(t), m, t.log_n, log_s,
                                                             total_cols, out_mf, fold, Tab<MODE>::inv_n(t),
                                                             Tab<MODE>::inv_n_w(t));
  count_launch();
  return cudaGetLastError();
}

template <int MODE>
cudaError_t launch_col_dyn(int log_r, bool fwd, const NttDeviceTables& t, u64* result,
                           const u64* operand, u64 batch, int log_s, int out_mf, int fold,
                           cudaStream_t stream) {
  switch (log_r) {
    case 1: return launch_col<MODE, 1>(fwd, t, result, operand, batch, log_s, out_mf, fold, stream);
    case 2: return launch_col<MODE, 2>(fwd, t, result, operand, batch, log_s, out_mf, fold, stream);
    case 3: return launch_col<MODE, 3>(fwd, t, result, operand, batch, log_s, out_mf, fold, stream);
    case 4: return launch_col<MODE, 4>(fwd, t, result, operand, batch, log_s, out_mf, fold, stream);
    case 5: return launch_col<MODE, 5>(fwd, t, result, operand, batch, log_s, out_mf, fold, stream);
  }
  return cudaErrorInvalidValue;
}

cudaError_t simple_transform(bool fwd, const NttDeviceTables& t, u64* result, const u64* operand,
                             int out_mf, u64 batch, cudaStream_t stream) {
  const u64 total = batch << (t.log_n - 1);
  const unsigned threads = 128, grid = (unsigned)((total + threads - 1) / threads);
  const u64* src = operand;
  const Mod m = make_mod(t);
  for (int k = 0; k < t.log_n; ++k) {
    const int s = fwd ? k : t.log_n - 1 - k;
    const int last = k == t.log_n - 1;
    if (fwd)
      ntt_stage_simple<true><<<grid, threads, 0, stream>>>(result, src, t.fwd, m, t.log_n, s, total,
                                                           out_mf, last, t.inv_n, t.inv_n_w);
    else
      ntt_stage_simple<false><<<grid, threads, 0, stream>>>(result, src, t.inv, m, t.log_n, s, total,
                                                            out_mf, last, t.inv_n, t.inv_n_w);
    count_launch();
    src = result;
  }
  return cudaGetLastError();
}

template <int MODE, int LOGR>
cudaError_t launch_fused(bool fwd, const NttDeviceTables& t, u64* result, const u64* operand, u64 batch,
                         int out_mf, cudaStream_t stream) {
  using Cfg = FusedCfg<LOGR, MODE>;
  const Mod m = make_mod(t);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(batch * Cfg::K));
  cfg.blockDim = dim3(Cfg::THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM;
  cfg.stream = stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = Cfg::K;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  cudaError_t e;
  if (fwd)
    e = cudaLaunchKernelEx(&cfg, ntt_fused_fwd<MODE, LOGR>, result, operand, Tab<MODE>::fwd(t), m, out_mf);
  else
    e = cudaLaunchKernelEx(&cfg, ntt_fused_inv<MODE, LOGR>, result, operand, Tab<MODE>::inv(t), m, out_mf,
                           Tab<MODE>::inv_n(t), Tab<MODE>::inv_n_w(t));
  count_launch();
  return e != cudaSuccess ? e : cudaGetLastError();
}

// The persistent pipelined kernel: one launch, work items from a global counter (ntt_kernels.cuh).
// HEXL_B200_PIPE: see pipe_log_r below; HEXL_B200_PIPE_LOOKAHEAD = polynomials
// between a producer block and its consumers (default 16, chosen for the H100's 50 MB L2: at N = 2^17 that is 16 MiB
// of intermediate), HEXL_B200_PIPE_CTAS = CTAs per SM (default: the
// kernel's launch bound).
template <int MODE, int LOGR>
cudaError_t launch_pipe(bool fwd, const NttDeviceTables& t, u64* result, const u64* operand, u64 batch, int out_mf,
                        cudaStream_t stream) {
  using Cfg = PipeCfg<LOGR, MODE>;
  static const int lookahead_env = env_int("HEXL_B200_PIPE_LOOKAHEAD", 16);
  static const int ctas_env = env_int("HEXL_B200_PIPE_CTAS", 0);
  const Mod m = make_mod(t);
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const unsigned lookahead = (unsigned)std::max(1, lookahead_env);
  const u64 items = (batch + lookahead) * Cfg::SLOTS;
  const int per_sm = ctas_env > 0 ? ctas_env : Cfg::MIN_BLOCKS;
  const unsigned grid = (unsigned)std::min<u64>((u64)sms * per_sm, items);
  unsigned* state = nullptr;  // [0] = work counter, [1 + p] = producers of polynomial p that have finished
  const size_t bytes = (size_t)(batch + 1) * sizeof(unsigned);
  cudaError_t e = scratch_alloc_async(reinterpret_cast<void**>(&state), bytes, stream);
  if (e != cudaSuccess) return e;
  if ((e = cudaMemsetAsync(state, 0, bytes, stream)) != cudaSuccess) return e;
  if (fwd) {
    if ((e = ensure_dynamic_smem<ntt_pipe_fwd<MODE, LOGR>>(Cfg::SMEM)) != cudaSuccess) return e;
    ntt_pipe_fwd<MODE, LOGR><<<grid, Cfg::THREADS, Cfg::SMEM, stream>>>(result, operand, Tab<MODE>::fwd(t), m, out_mf,
                                                                        (unsigned)batch, lookahead, state, state + 1);
  } else {
    if ((e = ensure_dynamic_smem<ntt_pipe_inv<MODE, LOGR>>(Cfg::SMEM)) != cudaSuccess) return e;
    ntt_pipe_inv<MODE, LOGR><<<grid, Cfg::THREADS, Cfg::SMEM, stream>>>(result, operand, Tab<MODE>::inv(t), m, out_mf,
                                                                        Tab<MODE>::inv_n(t), Tab<MODE>::inv_n_w(t),
                                                                        (unsigned)batch, lookahead, state, state + 1);
  }
  count_launch();
  e = cudaGetLastError();
  scratch_free_async(state, stream);
  return e;
}

template <int MODE>
cudaError_t launch_pipe_dyn(int log_r, bool fwd, const NttDeviceTables& t, u64* result, const u64* operand, u64 batch,
                            int out_mf, cudaStream_t stream) {
  switch (log_r) {
    case 2: return launch_pipe<MODE, 2>(fwd, t, result, operand, batch, out_mf, stream);
    case 3: return launch_pipe<MODE, 3>(fwd, t, result, operand, batch, out_mf, stream);
    case 4: return launch_pipe<MODE, 4>(fwd, t, result, operand, batch, out_mf, stream);
    case 5: return launch_pipe<MODE, 5>(fwd, t, result, operand, batch, out_mf, stream);
  }
  return cudaErrorInvalidValue;
}

// log2(N / 4096) for which the pipelined kernel is used; 0 = none.  HEXL_B200_PIPE: 1 = always (N = 2^14..2^17),
// 0 = never, unset = the 64-bit modes' forward at N = 2^15..2^17.  One H100 80GB HBM3 (power limit not recorded), 2^28
// coefficients, 55-bit q (tools/tune_split.py, ms, pipelined vs the two-kernel split), with the coefficient arrays in
// registers: N = 2^17 forward 3.10 vs 3.67, inverse 3.58 vs 3.71.  (Before, with the arrays in local memory: 2^17
// forward 14.9 vs 17.2, inverse 15.5 vs 15.4.)  At N = 2^14..2^16 see dsmem_log_r for every candidate: the pipelined
// forward is the fastest at 2^15 and 2^16, its inverse never is.  32-bit words use the distributed-shared-memory
// kernel instead.  A batch of fewer polynomials than the pipeline is deep gains nothing from it.
template <int MODE>
inline int pipe_log_r(int log_n, u64 batch, bool forward) {
  static const int mode = env_int("HEXL_B200_PIPE", -1);
  static const int min_batch = env_int("HEXL_B200_PIPE_MIN_BATCH", 64);
  const int lr = log_n - 12;
  if (mode == 0 || lr < 2 || lr > 5 || batch < (u64)min_batch || batch >= (1ull << 31)) return 0;
  if (mode > 0) return lr;
  const bool wins = MODE != kSmall && forward && log_n >= 15;
  return wins ? lr : 0;
}

// The single kernel that keeps the intermediate in the cluster's shared memory
template <int MODE, int LOGR>
cudaError_t launch_dsmem(bool fwd, const NttDeviceTables& t, u64* result, const u64* operand, u64 batch, int out_mf,
                         cudaStream_t stream) {
  using Cfg = DsmemCfg<LOGR, MODE>;
  const Mod m = make_mod(t);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(batch * Cfg::K));
  cfg.blockDim = dim3(Cfg::THREADS);
  cfg.dynamicSmemBytes = Cfg::SMEM;
  cfg.stream = stream;
  cudaLaunchAttribute attr;
  attr.id = cudaLaunchAttributeClusterDimension;
  attr.val.clusterDim.x = Cfg::K;
  attr.val.clusterDim.y = 1;
  attr.val.clusterDim.z = 1;
  cfg.attrs = &attr;
  cfg.numAttrs = 1;
  cudaError_t e;
  if (fwd) {
    if ((e = ensure_dynamic_smem<ntt_dsmem_fwd<MODE, LOGR>>(Cfg::SMEM)) != cudaSuccess) return e;
    e = cudaLaunchKernelEx(&cfg, ntt_dsmem_fwd<MODE, LOGR>, result, operand, Tab<MODE>::fwd(t), m, out_mf);
  } else {
    if ((e = ensure_dynamic_smem<ntt_dsmem_inv<MODE, LOGR>>(Cfg::SMEM)) != cudaSuccess) return e;
    e = cudaLaunchKernelEx(&cfg, ntt_dsmem_inv<MODE, LOGR>, result, operand, Tab<MODE>::inv(t), m, out_mf,
                           Tab<MODE>::inv_n(t), Tab<MODE>::inv_n_w(t));
  }
  count_launch();
  return e != cudaSuccess ? e : cudaGetLastError();
}

template <int MODE>
cudaError_t launch_dsmem_dyn(int log_r, bool fwd, const NttDeviceTables& t, u64* result, const u64* operand,
                             u64 batch, int out_mf, cudaStream_t stream) {
  switch (log_r) {
    case 2: return launch_dsmem<MODE, 2>(fwd, t, result, operand, batch, out_mf, stream);
    case 3: return launch_dsmem<MODE, 3>(fwd, t, result, operand, batch, out_mf, stream);
  }
  if constexpr (MODE == kSmall) {
    if (log_r == 4) return launch_dsmem<MODE, 4>(fwd, t, result, operand, batch, out_mf, stream);
    if (log_r == 5) return launch_dsmem<MODE, 5>(fwd, t, result, operand, batch, out_mf, stream);
  }
  return cudaErrorInvalidValue;
}

// log2(N / 4096) for which the distributed-shared-memory kernel is used; 0 = none.  HEXL_B200_DSMEM=0 disables it.
// SMALL mode (32-bit words):
// One H100 SXM at 400 W, 2^28 coefficients, 29-bit q, forward / inverse ms vs the cluster kernel that keeps the
// intermediate in L2: N = 2^14 6.41 / 6.69 vs 6.90 / 7.26, 2^15 6.42 / 6.77 vs 6.83 / 7.29, 2^16 7.54 / 7.84 vs
// 7.99 / 8.15, 2^17 7.81 / 8.10 vs 8.25 / 8.42 (and vs 7.79 / 8.23, 8.10 / 8.30 for the pipelined kernel at 2^16 /
// 2^17), so it is the default at every size.  Re-timed on an H100 80GB HBM3 (power limit not recorded) with the
// coefficient arrays in registers: N = 2^16 1.76 / 1.79 vs 1.97 / 1.94, 2^17 1.94 / 2.08 vs 2.22 / 2.13 (pipelined
// 2.05 / 2.15).
// 64-bit words, one H100 80GB HBM3 at 700 W (1980 MHz maximum SM clock), 2^28 coefficients, q of 55 (FAST) / 60 (WIDE)
// / 61 (GENERIC) bits, forward / inverse ms, this kernel | the fused kernel through L2 | pipelined | two-kernel split:
//   N = 2^14  FAST 2.96 / 2.75 | 3.01 / 2.90 | 3.20 / 5.92 | 3.49 / 3.71   WIDE 3.45 / 3.24 | 3.28 / 3.32 | 3.43 / 6.26
//             GENERIC 3.35 / 3.37 | 3.41 / 3.57 | 3.48 / 6.54
//   N = 2^15  FAST 3.02 / 2.93 | 3.04 / 2.93 | 2.95 / 4.38 | 3.49 / 3.73   WIDE 3.51 / 3.43 | 3.35 / 3.47 | 3.24 / 4.70
//             GENERIC 3.46 / 3.60 | 3.46 / 3.67 | 3.28 / 4.98
//   N = 2^16  FAST 3.23 / 3.43 | 3.07 / 3.13 | 2.88 / 3.54 | 3.49 / 3.73   WIDE 3.57 / 4.01 | 3.41 / 3.56 | 3.26 / 3.87
//             GENERIC 3.71 / 4.20 | 3.54 / 3.82 | 3.27 / 4.07
// So the 64-bit modes use it at N = 2^14 (except where the WIDE forward is 5 % behind the fused kernel, kept for one
// rule per size) and for the 2^15 inverse (the 2^15 forward takes the pipelined kernel when the batch is deep enough
// for it, this one otherwise).  At 2^16 it loses both ways -- its column phase stores to the peers' shared memory in
// 8-byte words, and each CTA's phases are serialised at the cluster barrier -- to the pipelined forward and the fused
// inverse.  On the benchmark's step (8192 polynomials at 2^16, 55-bit) this kernel in both directions took 13.2 ms
// against 14.4 ms for the split.
template <int MODE>
int dsmem_log_r(int log_n) {
  static const int mode = env_int("HEXL_B200_DSMEM", 1);
  const int lr = log_n - DsmemCfg<2>::LOGC;
  if (mode == 0 || lr < 2) return 0;
  if constexpr (MODE == kSmall) return lr <= 5 ? lr : 0;
  return lr <= 3 ? lr : 0;
}

// log2(N / 4096) for which the single fused kernel is used; 0 = none.  The 64-bit modes use it at N = 2^16 (the
// inverse, and the forward of batches too shallow for the pipelined kernel; timings at dsmem_log_r);
// HEXL_B200_FUSED=1 enables it at N = 2^14..2^17, 0 disables it.  One H100 80GB HBM3 (power limit not recorded),
// 2^28 coefficients, 55-bit q: N = 2^17 inverse 3.91 vs 3.71 ms for the split.
template <int MODE>
int fused_log_r(int log_n) {
  static const int mode = MODE == kSmall ? env_int("HEXL_B200_FUSED_SMALL", 1) : env_int("HEXL_B200_FUSED", -1);
  const int lr = log_n - FusedCfg<2>::LOGC;
  if (mode == 0 || lr < 2 || lr > 5) return 0;
  return (mode > 0 || log_n == 16) ? lr : 0;
}

template <int MODE>
cudaError_t launch_fused_dyn(int log_r, bool fwd, const NttDeviceTables& t, u64* result, const u64* operand,
                             u64 batch, int out_mf, cudaStream_t stream) {
  switch (log_r) {
    case 2: return launch_fused<MODE, 2>(fwd, t, result, operand, batch, out_mf, stream);
    case 3: return launch_fused<MODE, 3>(fwd, t, result, operand, batch, out_mf, stream);
    case 4: return launch_fused<MODE, 4>(fwd, t, result, operand, batch, out_mf, stream);
    case 5: return launch_fused<MODE, 5>(fwd, t, result, operand, batch, out_mf, stream);
  }
  return cudaErrorInvalidValue;
}

template <int MODE>
cudaError_t forward_impl(const NttDeviceTables& t, u64* result, const u64* operand, int out_mf,
                         u64 batch, cudaStream_t stream) {
  if (const int lr = pipe_log_r<MODE>(t.log_n, batch, true)) return launch_pipe_dyn<MODE>(lr, true, t, result, operand, batch, out_mf, stream);
  if (const int lr = dsmem_log_r<MODE>(t.log_n)) return launch_dsmem_dyn<MODE>(lr, true, t, result, operand, batch, out_mf, stream);
  if (const int lr = fused_log_r<MODE>(t.log_n)) return launch_fused_dyn<MODE>(lr, true, t, result, operand, batch, out_mf, stream);
  const int log_c = pick_row_log(t.log_n);
  int radices[8];
  const int ncol = plan_col_passes(t.log_n - log_c, radices);
  const u64* src = operand;
  int log_s = t.log_n;
  for (int p = 0; p < ncol; ++p) {
    cudaError_t e = launch_col_dyn<MODE>(radices[p], true, t, result, src, batch, log_s, out_mf, 0, stream);
    if (e != cudaSuccess) return e;
    log_s -= radices[p];
    src = result;
  }
  return launch_row_dyn<MODE>(log_c, true, t, result, src, batch, out_mf, 0, stream);
}

template <int MODE>
cudaError_t inverse_impl(const NttDeviceTables& t, u64* result, const u64* operand, int out_mf,
                         u64 batch, cudaStream_t stream) {
  if (const int lr = pipe_log_r<MODE>(t.log_n, batch, false)) return launch_pipe_dyn<MODE>(lr, false, t, result, operand, batch, out_mf, stream);
  if (const int lr = dsmem_log_r<MODE>(t.log_n)) return launch_dsmem_dyn<MODE>(lr, false, t, result, operand, batch, out_mf, stream);
  if (const int lr = fused_log_r<MODE>(t.log_n)) return launch_fused_dyn<MODE>(lr, false, t, result, operand, batch, out_mf, stream);
  const int log_c = pick_row_log(t.log_n);
  int radices[8];
  const int ncol = plan_col_passes(t.log_n - log_c, radices);
  // the kernel that contains the root stage folds N^-1 and applies out_mf
  cudaError_t e = launch_row_dyn<MODE>(log_c, false, t, result, operand, batch, out_mf, ncol == 0, stream);
  if (e != cudaSuccess) return e;
  // column passes in reverse: innermost (smallest sub-blocks) first
  int log_s = log_c;
  for (int p = ncol - 1; p >= 0; --p) {
    log_s += radices[p];
    e = launch_col_dyn<MODE>(radices[p], false, t, result, result, batch, log_s, out_mf, p == 0, stream);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace

cudaError_t launch_ntt_forward(const NttDeviceTables& t, u64* result, const u64* operand,
                               int /*in_mf*/, int out_mf, u64 batch, cudaStream_t stream) {
  if (batch == 0) return cudaSuccess;
  if (t.log_n < 4) return simple_transform(true, t, result, operand, out_mf, batch, stream);
  switch (pick_mode(t.q)) {
    case kFast: return forward_impl<kFast>(t, result, operand, out_mf, batch, stream);
    case kSmall: return forward_impl<kSmall>(t, result, operand, out_mf, batch, stream);
    case kWide: return forward_impl<kWide>(t, result, operand, out_mf, batch, stream);
  }
  return forward_impl<kGeneric>(t, result, operand, out_mf, batch, stream);
}

cudaError_t launch_ntt_inverse(const NttDeviceTables& t, u64* result, const u64* operand,
                               int /*in_mf*/, int out_mf, u64 batch, cudaStream_t stream) {
  if (batch == 0) return cudaSuccess;
  if (t.log_n < 4) return simple_transform(false, t, result, operand, out_mf, batch, stream);
  switch (pick_mode(t.q)) {
    case kFast: return inverse_impl<kFast>(t, result, operand, out_mf, batch, stream);
    case kSmall: return inverse_impl<kSmall>(t, result, operand, out_mf, batch, stream);
    case kWide: return inverse_impl<kWide>(t, result, operand, out_mf, batch, stream);
  }
  return inverse_impl<kGeneric>(t, result, operand, out_mf, batch, stream);
}

}  // namespace hexl_b200
