// k3_average.cu — K3: ordered-subset average,
//   out[j] = (((z + g[s0][j]) + g[s1][j]) + ... + g[s(c-1)][j]) / divisor
// with z = 0.0f for Python `sum()` call sites (average.py:29, krum.py:80, brute.py:80,
// aksel.py:64) or the first row itself for cge.py:53-56; fp32 adds in the given order, one
// IEEE division — bit-exact with the reference given the same selection.
// The selection is read from DEVICE memory (written by the K5 scoring kernel), so the
// distance pass, the scoring and this pass chain on one stream with no host round trip.
// Roofline: HBM, (count + 1)·4 B per coordinate.
// bz_coordinate's average above kMaxN rows runs the same body over the 128-pointer WideRowTable
// (an overload of the kernel; the 64-pointer kernels are unchanged).  The body is in k3_average.cuh.
#include "k3_average.cuh"

namespace bz {

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
