// k5_score_wide.cu — K5 above 64 rows: the scoring and selection of Multi-Krum and Bulyan on up to
// kMaxNDistance rows, one CTA, after the last distance pass (bz_distance).  The steps and their order are
// those of score_from_table (k5_device.cuh): fp32 norms with every non-finite distance mapped to +inf
// (krum.py:46-47) and +inf on the diagonal, each row sorted by ranking, CPython's compensated sum of the
// rule's count, the stable argsort, Bulyan's status rule.  The n x n tables are kept as float, where the
// 64-row kernel keeps doubles: every distance is an fp32 norm, so nothing is lost, and the two tables of 128
// rows take 128 KB instead of 256 KB of shared memory.
#include "k5_device.cuh"

namespace bz {

constexpr int kK5WideThreads = 1024;

// The squared distance of unique rows a <= b (the self distance when a == b) from the pass that holds it.
__device__ __forceinline__ double pass_sq(const PassTables& t, int a, int b) {
  int ba = 0;
  while (a >= t.start[ba + 1]) ++ba;
  int bb = ba;
  while (b >= t.start[bb + 1]) ++bb;
  const int p = t.pass[ba][bb], f = t.first[p], s = t.size[p];
  const int s0 = t.start[f + 1] - t.start[f];
  const int la = ba == f ? a - t.start[f] : s0 + a - t.start[ba];
  const int lb = bb == f ? b - t.start[f] : s0 + b - t.start[bb];
  return __ldcg(t.table + (size_t)p * kPassTable + (size_t)la * s + lb);
}

__global__ void __launch_bounds__(kK5WideThreads)
k5_score_select_wide(const __grid_constant__ PassTables t, int n, int count, int32_t* __restrict__ order,
                     int32_t* __restrict__ status, int f, int m, int bulyan) {
  extern __shared__ double sm_wide[];
  double* score = sm_wide;                                   // n
  float* dist = reinterpret_cast<float*>(sm_wide + n);      // n x n
  float* sorted = dist + n * n;                              // n x n
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e / n, j = e - i * n;
    float v = __int_as_float(0x7f800000);
    if (i != j) {
      // aliases (a == b) read the self distance: 0 for a finite row, NaN for a row holding NaN / inf
      const int a = t.to_unique[i], b = t.to_unique[j];
      v = fp32_norm(pass_sq(t, min(a, b), max(a, b)));
      if (!finite_d(v)) v = __int_as_float(0x7f800000);
    }
    dist[e] = v;
  }
  __syncthreads();
  sort_rows(dist, sorted, n);
  for (int i = threadIdx.x; i < n; i += blockDim.x) score[i] = py_sum(sorted + i * n, count);
  __syncthreads();
  stable_order(score, n, order);
  if (threadIdx.x == 0 && status != nullptr) *status = bulyan ? bulyan_status(score, n, f, m) : BZ_STATUS_OK;
}

constexpr size_t kScoreWideSmemMax = (size_t)kMaxNDistance * sizeof(double) + 2 * (size_t)kMaxNDistance * kMaxNDistance * sizeof(float);

void launch_select_wide(const PassTables& t, int n, int count, int32_t* order, int32_t* status, int f, int m, int bulyan,
                        cudaStream_t st) {
  static unsigned long long opted = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(opted & bit)) {
    cudaFuncSetAttribute(k5_score_select_wide, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kScoreWideSmemMax);
    opted |= bit;
  }
  const size_t smem = (size_t)n * sizeof(double) + 2 * (size_t)n * n * sizeof(float);
  k5_score_select_wide<<<1, kK5WideThreads, smem, st>>>(t, n, count, order, status, f, m, bulyan);
}

}  // namespace bz
