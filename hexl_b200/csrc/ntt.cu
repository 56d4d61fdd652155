// Single-modulus NTT launchers (the kernels are in ntt_kernels.cuh).
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
    ROW_CASE(11) ROW_CASE(12) ROW_CASE(13)
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
    case 3: return launch_col<MODE, 3>(fwd, t, result, operand, batch, log_s, out_mf, fold, stream);
    case 4: return launch_col<MODE, 4>(fwd, t, result, operand, batch, log_s, out_mf, fold, stream);
  }
  // a radix-32 pass splits N = 2^17 only, where SMALL takes its distributed-shared-memory kernel instead
  if constexpr (MODE != kSmall)
    if (log_r == 5) return launch_col<MODE, 5>(fwd, t, result, operand, batch, log_s, out_mf, fold, stream);
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
  using Cfg = FusedCfg<LOGR>;
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

// The persistent pipelined kernel: one launch, work items from a global counter (ntt_kernels.cuh).  Forward only.
template <int MODE, int LOGR>
cudaError_t launch_pipe(const NttDeviceTables& t, u64* result, const u64* operand, u64 batch, int out_mf,
                        cudaStream_t stream) {
  return launch_pipelined<ntt_pipe_fwd<MODE, LOGR>, PipeCfg<LOGR>>(batch, stream, result, operand, Tab<MODE>::fwd(t),
                                                                  make_mod(t), out_mf);
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

// ------------------------------------------------------------------------------------------------ launch choice
// Which kernel transforms a batch of polynomials of N = 2^log_n >= 16 coefficients: a single-pass kernel with
// R = N / 4096 = 2^log_r, or the split (column passes of plan_col_passes, then rows of pick_row_log; a single row
// kernel up to N = 2^13).  "Deep" is 64 <= batch < 2^31.
//
//   N      64-bit modes (FAST, WIDE, GENERIC)                                          SMALL (q < 2^30)
//   2^14   distributed shared memory                                                  distributed shared memory
//   2^15   forward: pipelined if deep, else distributed shared memory;                distributed shared memory
//          inverse: distributed shared memory
//   2^16   forward: pipelined if deep, else fused through L2; inverse: fused          distributed shared memory
//   2^17   forward: pipelined if deep, else split; inverse: split                     distributed shared memory
//   else   split                                                                      split
//
// SMALL mode (32-bit words), distributed shared memory vs the fused kernel that keeps the intermediate in L2, forward /
// inverse ms, 2^28 coefficients, 29-bit q.  One H100 SXM at 400 W: N = 2^14 6.41 / 6.69 vs 6.90 / 7.26, 2^15 6.42 /
// 6.77 vs 6.83 / 7.29, 2^16 7.54 / 7.84 vs 7.99 / 8.15, 2^17 7.81 / 8.10 vs 8.25 / 8.42 (and vs 7.79 / 8.23, 8.10 /
// 8.30 for the pipelined kernel at 2^16 / 2^17), so it is the default at every size.  Re-timed on an H100 80GB HBM3
// (power limit not recorded) with the coefficient arrays in registers: N = 2^16 1.76 / 1.79 vs 1.97 / 1.94, 2^17 1.94
// / 2.08 vs 2.22 / 2.13 (pipelined 2.05 / 2.15).
// 64-bit words, one H100 80GB HBM3 at 700 W (1980 MHz maximum SM clock), 2^28 coefficients, q of 55 (FAST) / 60 (WIDE)
// / 61 (GENERIC) bits, forward / inverse ms, distributed shared memory | fused through L2 | pipelined | two-kernel
// split:
//   N = 2^14  FAST 2.96 / 2.75 | 3.01 / 2.90 | 3.20 / 5.92 | 3.49 / 3.71   WIDE 3.45 / 3.24 | 3.28 / 3.32 | 3.43 / 6.26
//             GENERIC 3.35 / 3.37 | 3.41 / 3.57 | 3.48 / 6.54
//   N = 2^15  FAST 3.02 / 2.93 | 3.04 / 2.93 | 2.95 / 4.38 | 3.49 / 3.73   WIDE 3.51 / 3.43 | 3.35 / 3.47 | 3.24 / 4.70
//             GENERIC 3.46 / 3.60 | 3.46 / 3.67 | 3.28 / 4.98
//   N = 2^16  FAST 3.23 / 3.43 | 3.07 / 3.13 | 2.88 / 3.54 | 3.49 / 3.73   WIDE 3.57 / 4.01 | 3.41 / 3.56 | 3.26 / 3.87
//             GENERIC 3.71 / 4.20 | 3.54 / 3.82 | 3.27 / 4.07
// So the 64-bit modes use distributed shared memory at N = 2^14 (except where the WIDE forward is 5 % behind the fused
// kernel, kept for one rule per size) and for the 2^15 inverse (the 2^15 forward takes the pipelined kernel when the
// batch is deep enough for it, this one otherwise).  At 2^16 it loses both ways -- its column phase stores to the
// peers' shared memory in 8-byte words, and each CTA's phases are serialised at the cluster barrier -- to the
// pipelined forward and the fused inverse.  On the benchmark's step (8192 polynomials at 2^16, 55-bit) the distributed-
// shared-memory kernel in both directions took 13.2 ms against 14.4 ms for the split.
// N = 2^17, one H100 80GB HBM3 (power limit not recorded), 2^28 coefficients, 55-bit q, against the two-kernel split,
// with the coefficient arrays in registers: pipelined forward 3.10 vs 3.67, pipelined inverse 3.58 vs 3.71, fused
// inverse 3.91 vs 3.71.  (Before, with the arrays in local memory: pipelined forward 14.9 vs 17.2, inverse 15.5 vs
// 15.4.)  A batch of fewer polynomials than the pipeline is deep gains nothing from it.
enum : int { kSplit, kPipe, kFused, kDsmem };
struct SinglePass {
  int kernel, log_r;
};
template <int MODE>
SinglePass plan_single_pass(int log_n, u64 batch, bool forward) {
  const int lr = log_n - 12;
  if (lr < 2 || lr > 5) return {kSplit, 0};
  if (MODE == kSmall) return {kDsmem, lr};
  if (forward && lr >= 3 && batch >= 64 && batch < (1ull << 31)) return {kPipe, lr};
  if (lr <= 3) return {kDsmem, lr};
  if (lr == 4) return {kFused, lr};
  return {kSplit, 0};
}

// Only what plan_single_pass returns is instantiated.
template <int MODE>
cudaError_t launch_single_pass(SinglePass p, bool fwd, const NttDeviceTables& t, u64* result, const u64* operand,
                               u64 batch, int out_mf, cudaStream_t stream) {
  if constexpr (MODE == kSmall) {
    switch (p.log_r) {
      case 2: return launch_dsmem<MODE, 2>(fwd, t, result, operand, batch, out_mf, stream);
      case 3: return launch_dsmem<MODE, 3>(fwd, t, result, operand, batch, out_mf, stream);
      case 4: return launch_dsmem<MODE, 4>(fwd, t, result, operand, batch, out_mf, stream);
      case 5: return launch_dsmem<MODE, 5>(fwd, t, result, operand, batch, out_mf, stream);
    }
  } else if (p.kernel == kPipe && fwd) {
    switch (p.log_r) {
      case 3: return launch_pipe<MODE, 3>(t, result, operand, batch, out_mf, stream);
      case 4: return launch_pipe<MODE, 4>(t, result, operand, batch, out_mf, stream);
      case 5: return launch_pipe<MODE, 5>(t, result, operand, batch, out_mf, stream);
    }
  } else if (p.kernel == kFused && p.log_r == 4) {
    return launch_fused<MODE, 4>(fwd, t, result, operand, batch, out_mf, stream);
  } else if (p.kernel == kDsmem) {
    switch (p.log_r) {
      case 2: return launch_dsmem<MODE, 2>(fwd, t, result, operand, batch, out_mf, stream);
      case 3: return launch_dsmem<MODE, 3>(fwd, t, result, operand, batch, out_mf, stream);
    }
  }
  return cudaErrorInvalidValue;
}

template <int MODE>
cudaError_t forward_impl(const NttDeviceTables& t, u64* result, const u64* operand, int out_mf,
                         u64 batch, cudaStream_t stream) {
  const SinglePass sp = plan_single_pass<MODE>(t.log_n, batch, true);
  if (sp.kernel != kSplit) return launch_single_pass<MODE>(sp, true, t, result, operand, batch, out_mf, stream);
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
  const SinglePass sp = plan_single_pass<MODE>(t.log_n, batch, false);
  if (sp.kernel != kSplit) return launch_single_pass<MODE>(sp, false, t, result, operand, batch, out_mf, stream);
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
