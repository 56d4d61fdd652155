// The two integer kernels of BFV multiplication by BEHZ (Bajard, Eynard, Hasan, Zucca 2016; SEAL's RNSTool): the lift
// of a polynomial from Q into Bsk = B u {m_sk} with the overflow removed by Montgomery reduction modulo m~ = 2^32, and
// the scaling of the tensor by t/Q (fast floor into Bsk, Shenoy-Kumaresan back to Q).  include/hexl_b200.h
// (hexl_b200_bfv_multiply) has the definitions; capi_bfv.cu builds the constant tables laid out as internal.h states.
#include "internal.h"

namespace hexl_b200 {
namespace {

constexpr int kThreads = 256;
constexpr unsigned kTile = kBehzTile;  // coefficient slots per CTA: one warp covers one limb of the tile

// [hi * 2^64 + lo]_m for any 128-bit value; c = {m, floor(2^64 / m), 2^64 mod m, its Shoup factor}, m < 2^62
__device__ __forceinline__ u64 reduce128(u64 hi, u64 lo, const u64* c) {
  const u64 m = c[0];
  const u64 r = shoup_lazy(hi, c[2], c[3], m) + barrett64_lazy(lo, m, c[1]);  // < 4m
  return csub(csub(r, m << 1), m);
}

// sum_i a[i * kTile] b[i] over `count` terms, unreduced in 128 bits: count <= 64 products of canonical words below
// 2^61 stay below 2^128
__device__ __forceinline__ void dot128(const u64* a, const u64* b, unsigned count, u64& hi, u64& lo) {
  hi = lo = 0;
#pragma unroll 4
  for (unsigned i = 0; i < count; ++i) {
    const u64 x = a[i * kTile], y = b[i];
    const u64 plo = x * y;
    lo += plo;
    hi += mulhi(x, y) + (lo < plo);
  }
}

// One CTA lifts kTile slots of one polynomial x over Q (l limbs) to Q u Bsk (l + k + 1 limbs, the Q limbs copied).
// Phase 1 reads each source limb once and stages v_i = [x_i m~ (Q/q_i)^-1]_{q_i}; phase 2 forms r = [-z Q^-1]_{m~}
// per slot, z = sum_i v_i [Q/q_i]_{m~} (wrapping 32-bit arithmetic is exact modulo m~ = 2^32); phase 3 gives each warp
// one target m of Bsk: x'_m = [(z_m + [Q]_m r_c) m~^-1]_m with r_c the centred r.
__global__ void __launch_bounds__(kThreads)
    bfv_extend_kernel(u64* result, u64 res_poly, const u64* operand, u64 op_poly, u64 n, u64 tiles, unsigned l,
                      unsigned kb, const u64* __restrict__ tab) {
  extern __shared__ __align__(16) u64 smem[];
  u64* v = smem;             // [i][slot]
  u64* rr = smem + l * kTile;  // [slot]
  const u64 p = blockIdx.x / tiles, s0 = (blockIdx.x - p * tiles) * kTile;
  const unsigned width = (unsigned)min((u64)kTile, n - s0);
  const u64* src = operand + p * op_poly + s0;
  u64* dst = result + p * res_poly + s0;
  const u64* mt = tab + 3 * l;               // [Q/q_i] mod 2^32
  const u64* tgt = tab + 4 * l + 1;          // per target: m, mu, 2^64 mod m, Shoup, [Q]_m, m - [Q m~]_m, m~^-1, Shoup
  const u64* matrix = tgt + 8 * kb;          // [e][i]: [Q/q_i]_m
  for (unsigned idx = threadIdx.x; idx < l * kTile; idx += kThreads) {
    const unsigned i = idx / kTile, s = idx - i * kTile;
    if (s >= width) continue;
    const u64* c = tab + 3 * i;  // q_i, [m~ (Q/q_i)^-1]_{q_i}, its Shoup factor
    const u64 x = __ldcs(src + i * n + s);
    dst[i * n + s] = x;
    v[i * kTile + s] = csub(shoup_lazy(x, c[1], c[2], c[0]), c[0]);
  }
  __syncthreads();
  const uint32_t neg_qinv = (uint32_t)tab[4 * l];
  for (unsigned s = threadIdx.x; s < width; s += kThreads) {
    uint32_t z = 0;
    for (unsigned i = 0; i < l; ++i) z += (uint32_t)v[i * kTile + s] * (uint32_t)mt[i];
    rr[s] = z * neg_qinv;
  }
  __syncthreads();
  for (unsigned idx = threadIdx.x; idx < kb * kTile; idx += kThreads) {
    const unsigned e = idx / kTile, s = idx - e * kTile;
    if (s >= width) continue;
    const u64* t = tgt + 8 * e;
    u64 hi, lo;
    dot128(v + s, matrix + (u64)e * l, l, hi, lo);
    const u64 z = reduce128(hi, lo, t);
    const u64 r = rr[s];
    // z + [Q]_m r_c as a 128-bit value below 2^94: r_c = r - 2^32 adds m - [Q 2^32]_m
    lo = t[4] * r;
    hi = mulhi(t[4], r);
    const u64 add = z + (r >> 31 ? t[5] : 0);
    lo += add;
    hi += lo < add;
    const u64 y = reduce128(hi, lo, t);
    __stcs(dst + (u64)(l + e) * n + s, csub(shoup_lazy(y, t[6], t[7], t[0]), t[0]));
  }
}

// One CTA scales kTile slots of one tensor polynomial D over Q u Bsk (l + k + 1 limbs) by t/Q into Q (l limbs):
// phase 1 stages u'_i = [D_{q_i} t (Q/q_i)^-1]_{q_i}; phase 2 gives each warp one target m of Bsk, the fast floor
// w_m = [t Q^-1 D_m - Q^-1 FBC(u)_m]_m, and stages [w_{b_j} (B/b_j)^-1]_{b_j} (or w_{m_sk}); phase 3 forms alpha per
// slot; phase 4 gives each warp one target q_i: FBC(w_B)_{q_i} corrected by [B]_{q_i} times the centred alpha.
__global__ void __launch_bounds__(kThreads)
    bfv_scale_kernel(BfvOutputs out, const u64* tensor, u64 d_poly, u64 n, u64 tiles, unsigned l, unsigned k,
                     const u64* __restrict__ tab) {
  extern __shared__ __align__(16) u64 smem[];
  u64* u = smem;                 // [i][slot]
  u64* y = u + l * kTile;        // [j][slot]
  u64* wsk = y + k * kTile;      // [slot]
  u64* al = wsk + kTile;         // [slot]
  const u64 p = blockIdx.x / tiles, s0 = (blockIdx.x - p * tiles) * kTile;
  const unsigned width = (unsigned)min((u64)kTile, n - s0);
  const u64* src = tensor + p * d_poly + s0;
  u64* dst = (p == 0 ? out.p[0] : p == 1 ? out.p[1] : out.p[2]) + s0;  // constant indices keep out in parameters
  const unsigned kb = k + 1;
  const u64* tgt1 = tab + 3 * l;            // per m of Bsk: m, mu, 2^64 mod m, Shoup, [t Q^-1]_m, Shoup,
                                            //   [-Q^-1]_m, Shoup, [(B/b_j)^-1]_{b_j}, Shoup
  const u64* mat1 = tgt1 + 10 * kb;         // [e][i]: [Q/q_i]_m
  const u64* tgt2 = mat1 + (u64)kb * l;     // per q_i, then m_sk: q, mu, 2^64 mod q, Shoup, [B]_q
  const u64* mat2 = tgt2 + 5 * (l + 1);     // [i][j]: [B/b_j]_{q_i}, row l for m_sk
  const u64* binv = mat2 + (u64)(l + 1) * k;  // [B^-1]_{m_sk}, Shoup
  for (unsigned idx = threadIdx.x; idx < l * kTile; idx += kThreads) {
    const unsigned i = idx / kTile, s = idx - i * kTile;
    if (s >= width) continue;
    const u64* c = tab + 3 * i;  // q_i, [t (Q/q_i)^-1]_{q_i}, its Shoup factor
    u[i * kTile + s] = csub(shoup_lazy(__ldcs(src + i * n + s), c[1], c[2], c[0]), c[0]);
  }
  __syncthreads();
  for (unsigned idx = threadIdx.x; idx < kb * kTile; idx += kThreads) {
    const unsigned e = idx / kTile, s = idx - e * kTile;
    if (s >= width) continue;
    const u64* t = tgt1 + 10 * e;
    const u64 m = t[0];
    u64 hi, lo;
    dot128(u + s, mat1 + (u64)e * l, l, hi, lo);
    const u64 f = reduce128(hi, lo, t);
    const u64 dm = __ldcs(src + (u64)(l + e) * n + s);
    const u64 w = csub(csub(shoup_lazy(dm, t[4], t[5], m) + shoup_lazy(f, t[6], t[7], m), m << 1), m);
    if (e < k)
      y[e * kTile + s] = csub(shoup_lazy(w, t[8], t[9], m), m);
    else
      wsk[s] = w;
  }
  __syncthreads();
  const u64* tsk = tgt2 + 5 * l;
  const u64 msk = tsk[0];
  for (unsigned s = threadIdx.x; s < width; s += kThreads) {
    u64 hi, lo;
    dot128(y + s, mat2 + (u64)l * k, k, hi, lo);
    const u64 gamma = reduce128(hi, lo, tsk);
    const u64 diff = gamma >= wsk[s] ? gamma - wsk[s] : gamma + msk - wsk[s];
    al[s] = csub(shoup_lazy(diff, binv[0], binv[1], msk), msk);
  }
  __syncthreads();
  const u64 half = msk >> 1;
  for (unsigned idx = threadIdx.x; idx < l * kTile; idx += kThreads) {
    const unsigned i = idx / kTile, s = idx - i * kTile;
    if (s >= width) continue;
    const u64* t = tgt2 + 5 * i;
    const u64 q = t[0];
    u64 hi, lo;
    dot128(y + s, mat2 + (u64)i * k, k, hi, lo);
    const u64 c = reduce128(hi, lo, t);
    const u64 a = al[s];
    const bool neg = a > half;  // alpha stands for alpha - m_sk
    const u64 mag = neg ? msk - a : a;
    const u64 corr = reduce128(mulhi(t[4], mag), t[4] * mag, t);
    const u64 o = neg ? csub(c + corr, q) : (c >= corr ? c - corr : c + q - corr);
    __stcs(dst + (u64)i * n + s, o);
  }
}

}  // namespace

cudaError_t launch_bfv_extend(u64* result, u64 res_poly, const u64* operand, u64 op_poly, u64 n, u64 polys, u64 l,
                              u64 k, const u64* tab, cudaStream_t stream) {
  if (n == 0 || polys == 0) return cudaSuccess;
  const u64 tiles = (n + kTile - 1) / kTile;
  const size_t smem = (l + 1) * kTile * sizeof(u64);
  bfv_extend_kernel<<<(unsigned)(tiles * polys), kThreads, smem, stream>>>(result, res_poly, operand, op_poly, n,
                                                                          tiles, (unsigned)l, (unsigned)(k + 1), tab);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_bfv_scale(const BfvOutputs& out, const u64* tensor, u64 d_poly, u64 n, u64 polys, u64 l, u64 k,
                             const u64* tab, cudaStream_t stream) {
  if (n == 0 || polys == 0) return cudaSuccess;
  const u64 tiles = (n + kTile - 1) / kTile;
  const size_t smem = (l + k + 2) * kTile * sizeof(u64);
  bfv_scale_kernel<<<(unsigned)(tiles * polys), kThreads, smem, stream>>>(out, tensor, d_poly, n, tiles, (unsigned)l,
                                                                         (unsigned)k, tab);
  count_launch();
  return cudaGetLastError();
}

}  // namespace hexl_b200
