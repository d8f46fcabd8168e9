// k8_candidate.cu — K8: the candidate row of the attacks' line search,
//   identical family (attacks/identical.py:70-72, :83-85):  byz = fl32(avg + fl32(fl32(s) * att))
//   empire-strict    (attacks/empire.py:54, :61):           byz = fl32(avg * fl32(-x))
// for the factor x the previous evaluation's score pass left in device memory (it is only known once that
// pass has run).  fp32 multiply and add, rounded separately as ATen's `mul` by a scalar and `add` are.
// Roofline: HBM, 3·4 B per coordinate (2·4 B for empire-strict).
#include "dist.cuh"
#include "launch.cuh"

namespace bz {

constexpr int kK8Threads = 256;

template <int VEC>
__global__ void __launch_bounds__(kK8Threads)
k8_candidate(const float* __restrict__ avg, const float* __restrict__ att, float* __restrict__ byz, const Geom g,
             SearchState* __restrict__ state, const int which, const int negative, const int empire) {
  const int64_t v = (int64_t)blockIdx.x * kK8Threads + threadIdx.x;
  if (v >= g.nv) return;
  const int64_t e0 = v * VEC - g.shift;
  const bool full = e0 >= 0 && e0 + VEC <= g.d;
  pdl_wait();        // the previous score pass has written the factor
  double x = 0.;     // line_maximize's start
  if (which == 1) x = state->next_x;
  else if (which == 2) x = state->best_x;
  else if (v == 0) { state->next_x = 0.; state->ticket = 0u; }
  // the factor the statement applies: -x (empire-strict, and the identical family's `negative` while
  // searching); the returned factor has no sign applied (identical.py:78-82 negates fixed factors only)
  const float s = (float)((empire || (negative && which != 2)) ? -x : x);
  float a[VEC], o[VEC];
  load_vec<VEC>(avg, e0, g.d, full, a);
  if (empire) {
#pragma unroll
    for (int c = 0; c < VEC; ++c) o[c] = __fmul_rn(a[c], s);
  } else {
    float t[VEC];
    load_vec<VEC>(att, e0, g.d, full, t);
#pragma unroll
    for (int c = 0; c < VEC; ++c) o[c] = __fadd_rn(a[c], __fmul_rn(s, t[c]));
  }
  store_vec<VEC>(byz, e0, g.d, full, o);
}

int launch_candidate(const float* avg, const float* att, float* byz, int64_t d, SearchState* state, int which,
                     int negative, int empire, cudaStream_t st) {
  const float* in[2] = {avg, empire ? avg : att};
  const Geom g = make_geom(in, 2, byz, nullptr, d, 4);
  const unsigned blocks = (unsigned)((g.nv + kK8Threads - 1) / kK8Threads);
  const cudaError_t err = g.vec == 4
      ? launch_after(k8_candidate<4>, blocks, kK8Threads, 0, st, avg, att, byz, g, state, which, negative, empire)
      : launch_after(k8_candidate<1>, blocks, kK8Threads, 0, st, avg, att, byz, g, state, which, negative, empire);
  return err == cudaSuccess ? 0 : -1;
}

}  // namespace bz
