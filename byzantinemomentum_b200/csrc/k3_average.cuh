// k3_average.cuh — the body of K3, the ordered-subset average (k3_average.cu), shared with the average of
// bz_coordinate_many above kMaxNCoordinate rows (k1_many.cu), whose kernel takes the 1024-pointer table.
#pragma once

#include "launch.cuh"

namespace bz {

constexpr int kK3Threads = 256;
constexpr int kK3Unroll = 8;

// FULL: the whole vector lies inside [0, d) and is naturally aligned (the common case, kept
// free of per-load branches so that kK3Unroll loads stay in flight); otherwise element-wise.
template <int VEC, bool FULL, class Rows>
__device__ __forceinline__ void average_body(const Rows& rows, const int64_t e0, const int64_t d,
                                             const int32_t* __restrict__ sel, const int count, const int zero_init,
                                             const float divisor, float* __restrict__ out) {
  float acc[VEC];
  {
    const int r0 = sel ? sel[0] : 0;
    float t[VEC];
    load_vec<VEC>(rows.p[r0], e0, d, FULL, t);
#pragma unroll
    for (int c = 0; c < VEC; ++c) acc[c] = zero_init ? __fadd_rn(0.f, t[c]) : t[c];
  }
  int k = 1;
  for (; k + kK3Unroll <= count; k += kK3Unroll) {
    float t[kK3Unroll][VEC];
#pragma unroll
    for (int u = 0; u < kK3Unroll; ++u) {
      const int r = sel ? sel[k + u] : k + u;
      load_vec<VEC>(rows.p[r], e0, d, FULL, t[u]);
    }
#pragma unroll
    for (int u = 0; u < kK3Unroll; ++u)
#pragma unroll
      for (int c = 0; c < VEC; ++c) acc[c] = __fadd_rn(acc[c], t[u][c]);
  }
  for (; k < count; ++k) {
    const int r = sel ? sel[k] : k;
    float t[VEC];
    load_vec<VEC>(rows.p[r], e0, d, FULL, t);
#pragma unroll
    for (int c = 0; c < VEC; ++c) acc[c] = __fadd_rn(acc[c], t[c]);
  }
#pragma unroll
  for (int c = 0; c < VEC; ++c) acc[c] = __fdiv_rn(acc[c], divisor);
  store_vec<VEC>(out, e0, d, FULL, acc);
}

template <int VEC, class Rows>
__device__ __forceinline__ void k3_average_body(const Rows& rows, const Geom& g, const int32_t* __restrict__ sel,
                                                const int count, const int zero_init, const float divisor,
                                                const int32_t* __restrict__ status, float* __restrict__ out) {
  const int64_t blk = g.reverse ? (int64_t)gridDim.x - 1 - blockIdx.x : (int64_t)blockIdx.x;
  const int64_t v = blk * kK3Threads + threadIdx.x;
  if (v >= g.nv) return;
  const int64_t e0 = v * VEC - g.shift;
  const bool full = e0 >= 0 && e0 + VEC <= g.d;
  pdl_wait();        // launched while the scoring step drains: the selection / status / rows are valid from here
  if (status != nullptr && *status != 0) {
    float nan[VEC];
#pragma unroll
    for (int c = 0; c < VEC; ++c) nan[c] = quiet_nan();
    store_vec<VEC>(out, e0, g.d, full, nan);
    return;
  }
  if (full) average_body<VEC, true>(rows, e0, g.d, sel, count, zero_init, divisor, out);
  else      average_body<VEC, false>(rows, e0, g.d, sel, count, zero_init, divisor, out);
}

}  // namespace bz
