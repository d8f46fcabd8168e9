// k3_average.cu — K3: ordered-subset average,
//   out[j] = (((z + g[s0][j]) + g[s1][j]) + ... + g[s(c-1)][j]) / divisor
// with z = 0.0f for Python `sum()` call sites (average.py:29, krum.py:80, brute.py:80,
// aksel.py:64) or the first row itself for cge.py:53-56; fp32 adds in the given order, one
// IEEE division — bit-exact with the reference given the same selection.
// The selection is read from DEVICE memory (written by the K5 scoring kernel), so the
// distance pass, the scoring and this pass chain on one stream with no host round trip.
// Roofline: HBM, (count + 1)·4 B per coordinate.
// bz_coordinate's average above kMaxN rows runs the same body over the 128-pointer WideRowTable
// (an overload of the kernel; the 64-pointer kernels are unchanged).
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

template <int VEC>
__global__ void __launch_bounds__(kK3Threads)
k3_average(const __grid_constant__ RowTable rows, const Geom g, const int32_t* __restrict__ sel,
           const int count, const int zero_init, const float divisor,
           const int32_t* __restrict__ status, float* __restrict__ out) {
  k3_average_body<VEC>(rows, g, sel, count, zero_init, divisor, status, out);
}
template <int VEC>
__global__ void __launch_bounds__(kK3Threads)
k3_average(const __grid_constant__ WideRowTable rows, const Geom g, const int32_t* __restrict__ sel,
           const int count, const int zero_init, const float divisor,
           const int32_t* __restrict__ status, float* __restrict__ out) {
  k3_average_body<VEC>(rows, g, sel, count, zero_init, divisor, status, out);
}

template <class Rows>
static void launch_average_rows(const Rows& rows, const Geom& g, const int32_t* sel, int count,
                                int zero_init, float divisor, const int32_t* status, float* out, cudaStream_t st) {
  typedef void (*Kernel)(Rows, Geom, const int32_t*, int, int, float, const int32_t*, float*);
  if (g.nv <= 0) return;
  const unsigned blocks = (unsigned)((g.nv + kK3Threads - 1) / kK3Threads);
  const Kernel kernel = (g.vec == 4) ? Kernel(k3_average<4>) : (g.vec == 2) ? Kernel(k3_average<2>) : Kernel(k3_average<1>);
  launch_after(kernel, blocks, kK3Threads, 0, st, rows, g, sel, count, zero_init, divisor, status, out);
}

void launch_average(const RowTable& rows, const Geom& g, const int32_t* sel, int count,
                    int zero_init, float divisor, const int32_t* status, float* out, cudaStream_t st) {
  launch_average_rows(rows, g, sel, count, zero_init, divisor, status, out, st);
}
void launch_average(const WideRowTable& rows, const Geom& g, const int32_t* sel, int count,
                    int zero_init, float divisor, const int32_t* status, float* out, cudaStream_t st) {
  launch_average_rows(rows, g, sel, count, zero_init, divisor, status, out, st);
}

}  // namespace bz
