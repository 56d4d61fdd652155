// Fast base conversion between RNS bases (OpenFHE's ApproxSwitchCRTBasis, SEAL's BaseConverter::fast_convert_array):
// the mod-up and the mod-down of the hybrid key switch (capi_hybrid.cu), and hexl_b200_fast_base_convert.
#include "internal.h"

namespace hexl_b200 {
namespace {

constexpr int kThreads = 256;
constexpr unsigned kTile = 64;  // coefficient slots per CTA

// One CTA converts kTile slots of one polynomial.  Phase 1 reads each source limb of the tile once and stages
// y_i = [(x_i + add_i) (Q/q_i)^-1]_{q_i} in shared memory; phase 2 gives each warp one target at a time (kTile / VEC
// threads per target, so every constant read from the parameter table is uniform across the warp) and writes each
// target limb of the tile once: (from + to) words of traffic per slot.
// The per-target sum of from <= 64 products y_i [Q/q_i]_t, each below (2^61 - 1)^2, is below 64 (2^61 - 1)^2 < 2^128:
// it is added up unreduced in 128 bits, as ks_mac_kernel does, and reduced once.
template <int VEC>
__global__ void __launch_bounds__(kThreads)
    base_conv_kernel(u64* result, u64 res_limb, u64 res_poly, const u64* operand, u64 op_limb, u64 op_poly, u64 n,
                     u64 tiles, unsigned from, unsigned to, const __grid_constant__ BaseConvTable tab) {
  __shared__ __align__(16) u64 y[kParamBlock * kTile];
  constexpr unsigned kLanes = kTile / VEC;  // threads per limb of the tile
  const u64 p = blockIdx.x / tiles, s0 = (blockIdx.x - p * tiles) * kTile;
  const unsigned width = (unsigned)min((u64)kTile, n - s0);
  const u64* src = operand + p * op_poly + s0;
  for (unsigned idx = threadIdx.x; idx < from * kLanes; idx += kThreads) {
    const unsigned i = idx / kLanes, v = (idx - i * kLanes) * VEC;
    if (v >= width) continue;
    const u64* c = tab.w + 4 * i;  // q_i, (Q/q_i)^-1 mod q_i, its Shoup factor, add_i
    u64 x[VEC];
    if constexpr (VEC == 2) {
      const ulonglong2 t = ld_stream2(src + i * op_limb + v);
      x[0] = t.x;
      x[1] = t.y;
    } else {
      x[0] = __ldcs(src + i * op_limb + v);
    }
#pragma unroll
    for (int k = 0; k < VEC; ++k) y[i * kTile + v + k] = csub(shoup_lazy(x[k] + c[3], c[1], c[2], c[0]), c[0]);
  }
  __syncthreads();
  const u64* targets = tab.w + 4 * from;  // t, floor(2^64 / t), 2^64 mod t, its Shoup factor, sub
  const u64* matrix = targets + 5 * to;   // [e][i]: [Q/q_i]_{t_e}
  u64* dst = result + p * res_poly + s0;
  for (unsigned idx = threadIdx.x; idx < to * kLanes; idx += kThreads) {
    const unsigned e = idx / kLanes, v = (idx - e * kLanes) * VEC;
    if (v >= width) continue;
    const u64* m = matrix + (u64)e * from;
    u64 lo[VEC], hi[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) lo[k] = hi[k] = 0;
#pragma unroll 4
    for (unsigned i = 0; i < from; ++i) {
      const u64 b = m[i];
      u64 a[VEC];
      if constexpr (VEC == 2) {
        const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(y + i * kTile + v);
        a[0] = t.x;
        a[1] = t.y;
      } else {
        a[0] = y[i * kTile + v];
      }
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        const u64 plo = a[k] * b, phi = mulhi(a[k], b);
        lo[k] += plo;
        hi[k] += phi + (lo[k] < plo);
      }
    }
    const u64* t = targets + 5 * e;
    u64 out[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      u64 r = shoup_lazy(hi[k], t[2], t[3], t[0]) + barrett64_lazy(lo[k], t[0], t[1]);  // < 4t
      r = csub(csub(r, t[0] << 1), t[0]);
      out[k] = r >= t[4] ? r - t[4] : r + t[0] - t[4];
    }
    u64* o = dst + e * res_limb + v;
    if constexpr (VEC == 2) {
      st_stream2(o, make_ulonglong2(out[0], out[1]));
    } else {
      __stcs(o, out[0]);
    }
  }
}

// The t-corrected conversion (BGV's mod-down by P_T): phase 1 as above without the rounding offset, then
//   X~_tau = [sum_i y_i [P_T/q_i]_tau]_tau,  k = [-X~_tau P_T^-1]_tau          one pass per tile, into shared memory
//   delta_e = [X~_e + [P_T]_{t_e} k]_{t_e}                                    per target, after a __syncthreads
// The sums are those of base_conv_kernel (below 2^128); k [P_T]_{t_e} is added after the reduction, as a Shoup product
// (any 64-bit k) and one more conditional subtraction, so |T| = 64 sources never make a 65th 128-bit term.
template <int VEC>
__device__ __forceinline__ void conv_sum(const u64* y, const u64* m, unsigned from, unsigned v, u64 (&lo)[VEC],
                                         u64 (&hi)[VEC]) {
#pragma unroll
  for (int k = 0; k < VEC; ++k) lo[k] = hi[k] = 0;
#pragma unroll 4
  for (unsigned i = 0; i < from; ++i) {
    const u64 b = m[i];
    u64 a[VEC];
    if constexpr (VEC == 2) {
      const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(y + i * kTile + v);
      a[0] = t.x;
      a[1] = t.y;
    } else {
      a[0] = y[i * kTile + v];
    }
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      const u64 plo = a[k] * b, phi = mulhi(a[k], b);
      lo[k] += plo;
      hi[k] += phi + (lo[k] < plo);
    }
  }
}

template <int VEC>
__global__ void __launch_bounds__(kThreads)
    base_conv_t_kernel(u64* result, u64 res_limb, u64 res_poly, const u64* operand, u64 op_limb, u64 op_poly, u64 n,
                       u64 tiles, unsigned from, unsigned to, const __grid_constant__ BaseConvTable tab) {
  __shared__ __align__(16) u64 y[kParamBlock * kTile];
  __shared__ __align__(16) u64 corr[kTile];  // k of every slot of the tile
  constexpr unsigned kLanes = kTile / VEC;
  const u64 p = blockIdx.x / tiles, s0 = (blockIdx.x - p * tiles) * kTile;
  const unsigned width = (unsigned)min((u64)kTile, n - s0);
  const u64* src = operand + p * op_poly + s0;
  for (unsigned idx = threadIdx.x; idx < from * kLanes; idx += kThreads) {
    const unsigned i = idx / kLanes, v = (idx - i * kLanes) * VEC;
    if (v >= width) continue;
    const u64* c = tab.w + 3 * i;  // q_i, (P_T/q_i)^-1 mod q_i, its Shoup factor
    u64 x[VEC];
    if constexpr (VEC == 2) {
      const ulonglong2 t = ld_stream2(src + i * op_limb + v);
      x[0] = t.x;
      x[1] = t.y;
    } else {
      x[0] = __ldcs(src + i * op_limb + v);
    }
#pragma unroll
    for (int k = 0; k < VEC; ++k) y[i * kTile + v + k] = csub(shoup_lazy(x[k], c[1], c[2], c[0]), c[0]);
  }
  __syncthreads();
  const u64* tau = tab.w + 3 * from;  // tau, floor(2^64 / tau), 2^64 mod tau, its Shoup factor, [-P_T^-1]_tau, Shoup,
                                      // then [P_T/q_i]_tau for every source i
  if (threadIdx.x < kLanes) {
    const unsigned v = threadIdx.x * VEC;
    u64 lo[VEC], hi[VEC];
    conv_sum<VEC>(y, tau + 6, from, v, lo, hi);
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      u64 r = shoup_lazy(hi[k], tau[2], tau[3], tau[0]) + barrett64_lazy(lo[k], tau[0], tau[1]);  // < 4 tau
      r = csub(csub(r, tau[0] << 1), tau[0]);
      corr[v + k] = csub(shoup_lazy(r, tau[4], tau[5], tau[0]), tau[0]);
    }
  }
  __syncthreads();
  const u64* targets = tau + 6 + from;     // t, floor(2^64 / t), 2^64 mod t, its Shoup factor, [P_T]_t, its Shoup factor
  const u64* matrix = targets + 6 * to;    // [e][i]: [P_T/q_i]_{t_e}
  u64* dst = result + p * res_poly + s0;
  for (unsigned idx = threadIdx.x; idx < to * kLanes; idx += kThreads) {
    const unsigned e = idx / kLanes, v = (idx - e * kLanes) * VEC;
    if (v >= width) continue;
    u64 lo[VEC], hi[VEC];
    conv_sum<VEC>(y, matrix + (u64)e * from, from, v, lo, hi);
    const u64* t = targets + 6 * e;
    u64 out[VEC];
#pragma unroll
    for (int k = 0; k < VEC; ++k) {
      u64 r = shoup_lazy(hi[k], t[2], t[3], t[0]) + barrett64_lazy(lo[k], t[0], t[1]);  // < 4t
      r = csub(r, t[0] << 1) + shoup_lazy(corr[v + k], t[4], t[5], t[0]);               // < 2t + 2t
      out[k] = csub(csub(r, t[0] << 1), t[0]);
    }
    u64* o = dst + e * res_limb + v;
    if constexpr (VEC == 2) {
      st_stream2(o, make_ulonglong2(out[0], out[1]));
    } else {
      __stcs(o, out[0]);
    }
  }
}

}  // namespace

cudaError_t launch_base_conv_t(u64* result, u64 res_limb, u64 res_poly, const u64* operand, u64 op_limb, u64 op_poly,
                               u64 n, u64 polys, u64 from, u64 to, const BaseConvTable& tab, cudaStream_t stream) {
  if (n == 0 || polys == 0 || to == 0) return cudaSuccess;
  if (from < 1 || from > kParamBlock || to > base_conv_t_targets(from)) return cudaErrorInvalidValue;
  const u64 tiles = (n + kTile - 1) / kTile;
  const bool vec = ((n | res_limb | res_poly | op_limb | op_poly) & 1) == 0 &&
                   ((reinterpret_cast<uintptr_t>(result) | reinterpret_cast<uintptr_t>(operand)) & 15) == 0;
  auto kernel = vec ? base_conv_t_kernel<2> : base_conv_t_kernel<1>;
  kernel<<<(unsigned)(tiles * polys), kThreads, 0, stream>>>(result, res_limb, res_poly, operand, op_limb, op_poly,
                                                             n, tiles, (unsigned)from, (unsigned)to, tab);
  count_launch();
  return cudaGetLastError();
}

cudaError_t launch_base_conv(u64* result, u64 res_limb, u64 res_poly, const u64* operand, u64 op_limb, u64 op_poly,
                             u64 n, u64 polys, u64 from, u64 to, const BaseConvTable& tab, cudaStream_t stream) {
  if (n == 0 || polys == 0 || to == 0) return cudaSuccess;
  if (from < 1 || from > kParamBlock || 4 * from + to * (5 + from) > (u64)kBaseConvWords) return cudaErrorInvalidValue;
  const u64 tiles = (n + kTile - 1) / kTile;
  // 16-byte accesses: every limb and polynomial offset even, both buffers 16-byte aligned
  const bool vec = ((n | res_limb | res_poly | op_limb | op_poly) & 1) == 0 &&
                   ((reinterpret_cast<uintptr_t>(result) | reinterpret_cast<uintptr_t>(operand)) & 15) == 0;
  auto kernel = vec ? base_conv_kernel<2> : base_conv_kernel<1>;
  kernel<<<(unsigned)(tiles * polys), kThreads, 0, stream>>>(result, res_limb, res_poly, operand, op_limb, op_poly, n,
                                                             tiles, (unsigned)from, (unsigned)to, tab);
  count_launch();
  return cudaGetLastError();
}

}  // namespace hexl_b200
