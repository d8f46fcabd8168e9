// k5_score_wide.cu — K5 above 64 rows: the scoring and selection of Multi-Krum and Bulyan on up to
// kMaxNDistance rows, one CTA, after the last distance pass (bz_distance).  The steps and their order are
// those of score_from_table (k5_device.cuh): fp32 norms with every non-finite distance mapped to +inf
// (krum.py:46-47) and +inf on the diagonal, each row sorted by ranking, CPython's compensated sum of the
// rule's count, the stable argsort, Bulyan's status rule.  The n x n tables are kept as float, where the
// 64-row kernel keeps doubles: every distance is an fp32 norm, so nothing is lost, and the two tables of 128
// rows take 128 KB instead of 256 KB of shared memory.
// Phase B of the d-sharded path (bz_distance_select) runs the same steps from the ranks' gathered blocks
// (k5_blocks_select_wide), and selects the rows of Aksel and CGE from their gathered sums (k5_rowkeys_select_wide).
#include "k5_wide.cuh"

namespace bz {

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
  score_from_floats(dist, sorted, score, n, count, order, status, f, m, bulyan);
}

// The same from `nparts` n x n blocks of phase A (entries i < j): the pair (i, j) is the entry (min, max) of
// every block, added in rank order, ((p0 + p1) + p2) + ...  With one block it is p0, the pass table's value.
__global__ void __launch_bounds__(kK5WideThreads)
k5_blocks_select_wide(const double* __restrict__ parts, int nparts, int n, int count, int32_t* __restrict__ order,
                      int32_t* __restrict__ status, int f, int m, int bulyan) {
  extern __shared__ double sm_wide[];
  double* score = sm_wide;                                   // n
  float* dist = reinterpret_cast<float*>(sm_wide + n);      // n x n
  float* sorted = dist + n * n;                              // n x n
  const size_t len = (size_t)n * n;
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e / n, j = e - i * n;
    float v = __int_as_float(0x7f800000);
    if (i != j) {
      const size_t k = (size_t)min(i, j) * n + max(i, j);
      double s = __ldcg(parts + k);
      for (int p = 1; p < nparts; ++p) s += __ldcg(parts + (size_t)p * len + k);
      v = fp32_norm(s);
      if (!finite_d(v)) v = __int_as_float(0x7f800000);
    }
    dist[e] = v;
  }
  score_from_floats(dist, sorted, score, n, count, order, status, f, m, bulyan);
}

// Aksel and CGE: the n sums of `nparts` blocks added in rank order, the keys of K2''s last CTA, the stable order.
constexpr int kRowKeysThreads = kMaxNDistance;
__global__ void __launch_bounds__(kRowKeysThreads)
k5_rowkeys_select_wide(const double* __restrict__ parts, int nparts, int n, int sqrt_norm, int32_t* __restrict__ order) {
  __shared__ double key[kMaxNDistance];
  block_sum_parts(StridedParts{parts, (size_t)n}, nparts, n, key);
  for (int i = threadIdx.x; i < n; i += blockDim.x) key[i] = row_key(key[i], sqrt_norm);
  __syncthreads();
  stable_order(key, n, order);
}

void launch_select_wide(const PassTables& t, int n, int count, int32_t* order, int32_t* status, int f, int m, int bulyan,
                        cudaStream_t st) {
  static unsigned long long opted = 0;
  opt_in_wide(k5_score_select_wide, opted);
  k5_score_select_wide<<<1, kK5WideThreads, score_wide_smem(n), st>>>(t, n, count, order, status, f, m, bulyan);
}

void launch_blocks_select_wide(const double* parts, int nparts, int n, int count, int32_t* order, int32_t* status, int f,
                               int m, int bulyan, cudaStream_t st) {
  static unsigned long long opted = 0;
  opt_in_wide(k5_blocks_select_wide, opted);
  k5_blocks_select_wide<<<1, kK5WideThreads, score_wide_smem(n), st>>>(parts, nparts, n, count, order, status, f, m, bulyan);
}

void launch_rowkeys_select_wide(const double* parts, int nparts, int n, int sqrt_norm, int32_t* order, cudaStream_t st) {
  k5_rowkeys_select_wide<<<1, kRowKeysThreads, 0, st>>>(parts, nparts, n, sqrt_norm, order);
}

}  // namespace bz
