// The plaintext kernels of BFV and BGV: the lift of plaintexts (coefficients mod t) into the RNS basis of a ciphertext,
// and the BFV addition of round(Q m / t) to c0.  include/hexl_b200.h (hexl_b200_plain_lift, hexl_b200_bfv_add_plain)
// has the definitions; capi_plain.cu builds the constants.
#include "internal.h"

namespace hexl_b200 {
namespace {

constexpr int kThreads = 256;

// [x]_q for any x below 2^64 (mu = floor(2^64 / q)): the Barrett quotient is low by at most one
__device__ __forceinline__ u64 reduce64(u64 x, u64 q, u64 mu) { return csub(barrett64_lazy(x, q, mu), q); }

// One thread per coefficient slot j of one plaintext p, looping over the l limbs (adjacent threads write adjacent words
// of each limb).  m' = [m c]_t by a Shoup product (c = correction factor < t, m < t: the quotient estimate is low by at
// most one, so m c - est t is in [0, 2t)); then limb i gets [m']_{q_i}, or [m' - t]_{q_i} = q_i - [t - m']_{q_i} (0 when
// that is 0) for m' >= ceil(t/2).  Both reductions take a value below t < 2^61, so they are exact for every order of t
// and q_i.  Slots at and above pcc are zero.
__global__ void __launch_bounds__(kThreads)
    plain_lift_kernel(u64* result, const u64* plain, u64 pcc, u64 n, u64 total, unsigned l, u64 t, u64 cf,
                      u64 cf_shoup, PlainModuli mods) {
  const u64 half = (t + 1) >> 1;
  for (u64 idx = (u64)blockIdx.x * kThreads + threadIdx.x; idx < total; idx += (u64)gridDim.x * kThreads) {
    const u64 p = idx / n, j = idx - p * n;
    const u64 m = j < pcc ? csub(shoup_lazy(plain[p * pcc + j], cf, cf_shoup, t), t) : 0;
    const bool neg = m >= half;
    const u64 v = neg ? t - m : m;
    u64* dst = result + p * l * n + j;
    for (unsigned i = 0; i < l; ++i) {
      const u64 q = mods.q[i], r = reduce64(v, q, mods.mu[i]);
      dst[(u64)i * n] = neg && r ? q - r : r;
    }
  }
}

// c0 of ciphertext c at slot j < cover, per limb i: c0 +- [m [floor(Q/t)]_{q_i} + fix]_{q_i}, where
//   fix = floor((m r + h) / t),  r = Q mod t,  h = floor((t + 1) / 2)
// (SEAL's multiply_add_plain_with_scaling_variant; m [floor(Q/t)] + fix = floor((Q m + h) / t) = round(Q m / t)).
// fix without a 128-bit division: with r' = floor(r 2^64 / t), est = hi64(m r') is floor(m r / t) or one less (r' is
// low by less than one, so m r' / 2^64 is low by less than m / 2^64 < 1, and flooring loses less than one more); the
// remainder m r - est t is below 2t, so its low 64 bits are exact and one conditional subtraction leaves
// m r = a t + rem with 0 <= rem < t.  Then fix = a + floor((rem + h) / t), and since rem < t and h <= t/2 + 1,
// rem + h < 2t for t >= 2, so that floor is [rem + h >= t].  Table: per limb i (4 words) q_i, floor(2^64 / q_i), [floor(Q/t)]_{q_i}, its Shoup
// factor; then t, r, r', h.
__global__ void __launch_bounds__(kThreads)
    bfv_add_plain_kernel(u64* result, const u64* ct, const u64* plain, u64 pcc, u64 plain_stride, u64 n, u64 cover,
                         u64 total, unsigned l, int subtract, const u64* __restrict__ tab) {
  const u64* g = tab + 4 * l;
  const u64 t = g[0], r = g[1], r_shoup = g[2], h = g[3];
  for (u64 idx = (u64)blockIdx.x * kThreads + threadIdx.x; idx < total; idx += (u64)gridDim.x * kThreads) {
    const u64 c = idx / cover, j = idx - c * cover;
    const u64 m = j < pcc ? plain[c * plain_stride + j] : 0;
    u64 a = mulhi(m, r_shoup);
    u64 rem = m * r - a * t;
    if (rem >= t) {
      rem -= t;
      ++a;
    }
    const u64 fix = a + (rem + h >= t ? 1 : 0);
    const u64 off = c * 2 * l * n + j;
    for (unsigned i = 0; i < l; ++i) {
      const u64* k = tab + 4 * i;
      const u64 q = k[0];
      const u64 s = csub(csub(shoup_lazy(m, k[2], k[3], q), q) + reduce64(fix, q, k[1]), q);
      const u64 x = ct[off + (u64)i * n];
      result[off + (u64)i * n] = subtract ? (x >= s ? x - s : x + q - s) : csub(x + s, q);
    }
  }
}

unsigned grid_for(u64 total) {
  const u64 blocks = (total + kThreads - 1) / kThreads;
  return (unsigned)(blocks < 4096 ? blocks : 4096);
}

}  // namespace

cudaError_t launch_plain_lift(u64* result, const u64* plain, u64 pcc, u64 n, u64 count, u64 l, u64 t, u64 cf,
                              u64 cf_shoup, const PlainModuli& mods, cudaStream_t stream) {
  const u64 total = count * n;
  if (total == 0) return cudaSuccess;
  plain_lift_kernel<<<grid_for(total), kThreads, 0, stream>>>(result, plain, pcc, n, total, (unsigned)l, t, cf,
                                                              cf_shoup, mods);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_bfv_add_plain(u64* result, const u64* ct, const u64* plain, u64 pcc, u64 plain_stride, u64 n,
                                 u64 cover, u64 batch, u64 l, bool subtract, const u64* tab, cudaStream_t stream) {
  const u64 total = batch * cover;
  if (total == 0) return cudaSuccess;
  bfv_add_plain_kernel<<<grid_for(total), kThreads, 0, stream>>>(result, ct, plain, pcc, plain_stride, n, cover, total,
                                                                 (unsigned)l, subtract ? 1 : 0, tab);
  count_launch();
  return cudaGetLastError();
}

}  // namespace hexl_b200
