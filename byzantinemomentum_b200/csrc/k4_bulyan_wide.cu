// k4_bulyan_wide.cu — K4 above 64 rows (bz_distance's Bulyan): the reduce pass of k4_bulyan<THETA> over the
// 128-pointer table, for theta = n - 2f - 2 in 33..126 (n = 65 with f = 15 gives the smallest, f = 0 at
// n = 128 the largest).  One kernel per bucket of 8 theta values instead of one per theta: the theta means
// are padded with keys that sort after every real key, NaN keys included (INT_MAX, the key of a NaN, so the
// first theta sorted keys are those of the theta means alone), and the median and the window of the beta
// closest values are then read from the sorted shared column at run-time positions.  Everything else is
// k4_bulyan's: one thread per coordinate, the m_max = n - f - 2 best-scored rows in score order in a shared
// column of max(m_max, theta) x kK4Threads floats (<= 126 x 512 B), the running means in the reference's
// order, the lower median, the last strict gain of the closest-beta window.  Only the window's sum differs: it is
// accumulated in fp64 and rounded to fp32 once before the division (see below).
#include "dist.cuh"
#include "launch.cuh"
#include "networks_gen.cuh"
#include "networks_wide_gen.cuh"
#include "reduce.cuh"

namespace bz {

constexpr int kK4WideThreads = 128;
constexpr int kK4WideBucket = 8;

template <int B>
__global__ void __launch_bounds__(kK4WideThreads, 1)
k4_bulyan_wide(const __grid_constant__ WideRowTable rows, const int64_t d, const int n, const int f, const int m, const int one,
               const int mone, const int32_t* __restrict__ order, const int32_t* __restrict__ status, float* __restrict__ out) {
  extern __shared__ float sm[];   // [max(m_max, theta)][kK4WideThreads]
  // reversed walk: the distance pass before this one went forward (see Geom::reverse)
  const int64_t e = ((int64_t)gridDim.x - 1 - blockIdx.x) * kK4WideThreads + threadIdx.x;
  if (e >= d) return;
  pdl_wait();        // PDL: order / status / rows are valid from here
  if (status != nullptr && *status != 0) { out[e] = quiet_nan(); return; }
  float* col = sm + threadIdx.x;
  const int m_max = n - f - 2, theta = n - 2 * f - 2;
  // The m_max best-scored rows of this coordinate, in score order
  int k = 0;
  for (; k + 8 <= m_max; k += 8) {
    float t[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) t[u] = __ldcs(rows.p[order[k + u]] + e);
#pragma unroll
    for (int u = 0; u < 8; ++u) col[(k + u) * kK4WideThreads] = t[u];
  }
  for (; k < m_max; ++k) col[k * kK4WideThreads] = __ldcs(rows.p[order[k]] + e);
  // Stage 1: selected[i] = sum(gradients at sorted positions i..i+m_i-1).div_(m_i)  (bulyan.py:66-70)
  int key[B];
  int mi = m;
#pragma unroll
  for (int it = 0; it < B; ++it) {
    key[it] = 0x7fffffff;
    if (it < theta) {
      mi = min(mi, m_max - it);
      float acc = __fadd_rn(0.f, col[it * kK4WideThreads]);
      for (int q = 1; q < mi; ++q) acc = __fadd_rn(acc, col[(it + q) * kK4WideThreads]);
      key[it] = float_to_key(__fdiv_rn(acc, (float)mi));
    }
  }
  // Stage 2 (bulyan.py:78-84): lower median over theta, beta closest to it, mean
  SortNet<B>::run(OpsKeyMix<MixFull<B>>{one, mone}, key);
#pragma unroll
  for (int it = 0; it < B; ++it)
    if (it < theta) col[it * kK4WideThreads] = key_to_float(key[it]);
  const float last = col[(theta - 1) * kK4WideThreads];
  const float med = (last != last) ? quiet_nan() : col[((theta - 1) / 2) * kK4WideThreads];
  // the window of the beta closest values starts right after the last strict gain (see k4_bulyan)
  const int beta = theta - 2 * f;
  const int R = theta - beta;
  int lstar = 0;
  for (int l = 0; l < R; ++l) {
    const int dlo = abs_key(__fsub_rn(col[l * kK4WideThreads], med));
    const int dhi = abs_key(__fsub_rn(col[(l + beta) * kK4WideThreads], med));
    lstar = (dlo > dhi) ? l + 1 : lstar;
  }
  // The window is added in fp64 and rounded once: beta reaches 124 here, and an ascending fp32 sum of that many
  // values (aliased rows repeat one value, so its rounding errors add up) drifts past 1e-6 of the exact mean.
  // The fp32 rounding of the sum keeps the reference's overflow to +-inf, the division stays fp32's.
  double acc = 0.;
  for (int q = 0; q < beta; ++q) acc += (double)col[(lstar + q) * kK4WideThreads];
  const float r = __fdiv_rn(__double2float_rn(acc), (float)beta);
  out[e] = (med != med) ? quiet_nan() : r;
}

template <int B>
static void launch_bucket(const WideRowTable& rows, int64_t d, int n, int f, int m, const int32_t* order,
                          const int32_t* status, float* out, cudaStream_t st) {
  const int m_max = n - f - 2, theta = n - 2 * f - 2;
  const size_t smem = (size_t)(m_max > theta ? m_max : theta) * kK4WideThreads * sizeof(float);
  static unsigned long long opted = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(opted & bit)) {
    cudaFuncSetAttribute(k4_bulyan_wide<B>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                         (int)((size_t)(kMaxNDistance - 2) * kK4WideThreads * sizeof(float)));
    opted |= bit;
  }
  launch_after(k4_bulyan_wide<B>, (unsigned)((d + kK4WideThreads - 1) / kK4WideThreads), kK4WideThreads, smem, st,
               rows, d, n, f, m, 1, -1, order, status, out);
}

bool launch_bulyan_reduce_wide(const WideRowTable& rows, int n, int f, int m, const int32_t* order, const int32_t* status,
                               int64_t d, float* out, cudaStream_t st) {
  if (d <= 0) return true;
  const int bucket = (n - 2 * f - 2 + kK4WideBucket - 1) / kK4WideBucket;     // theta 33..126: buckets 5..16
  switch (bucket) {
#define X(K) case K: launch_bucket<K * kK4WideBucket>(rows, d, n, f, m, order, status, out, st); return true;
    X(5) X(6) X(7) X(8) X(9) X(10) X(11) X(12) X(13) X(14) X(15) X(16)
#undef X
    default: return false;
  }
}

}  // namespace bz
