// k5_many.cu — K5-many: the scoring and selection of Multi-Krum and Bulyan above kMaxNDistance rows
// (bz_distance_many), after K2-many.  The 128-row K5 keeps two n x n tables in one CTA's shared memory, which cannot
// reach 1024 rows (8 MB); here one warp takes one row, so the rows spread over n / 8 CTAs.  The steps are those of
// score_from_floats (k5_wide.cuh), and their order fixes the bits:
//   * the row's n distances through the alias map: fp32_norm of the summed squares (krum.py:46-47), every
//     non-finite norm mapped to +inf, +inf on the diagonal; an aliased pair reads the row's self distance (0, or NaN
//     and so +inf for a row holding NaN / inf);
//   * the row sorted (K1-many's warp bitonic sort on the bit patterns, which order as the values: every norm is
//     +0 .. +inf; the pads sort after +inf), and CPython's compensated sum of the rule's count (py_sum);
//   * in the last CTA (ticket): the stable order of the n scores and Bulyan's status word.
#include <climits>

#include "distance_many.cuh"
#include "bitonic.cuh"
#include "k5_device.cuh"

namespace bz {

constexpr int kSelThreads = 256;
constexpr int kSelWarps = kSelThreads / 32;

template <int P>
__global__ void __launch_bounds__(kSelThreads)
k5_select_many(const double* __restrict__ table, const __grid_constant__ ManyAliasMap map, const int n, const int u,
               const int count, double* __restrict__ scores, int32_t* __restrict__ order, int32_t* __restrict__ status,
               const int f, const int m, const int bulyan, unsigned* __restrict__ ticket) {
  constexpr int K = P / 32;
  __shared__ float sorted[kSelWarps][P];
  __shared__ double key[kMaxNMany];
  __shared__ bool last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int i = blockIdx.x * kSelWarps + warp;
  if (i < n) {
    const int a = map.to_unique[i];
    int v[K];
#pragma unroll
    for (int q = 0; q < K; ++q) {
      const int j = q * 32 + lane;
      int k = INT_MAX;
      if (j < n) {
        float x = __int_as_float(0x7f800000);
        if (j != i) {
          const int b = map.to_unique[j];
          x = fp32_norm(__ldcg(table + (size_t)min(a, b) * u + max(a, b)));
          if (!finite_d(x)) x = __int_as_float(0x7f800000);
        }
        k = __float_as_int(x);
      }
      v[q] = k;
    }
    warp_bitonic<K>(v, lane);
#pragma unroll
    for (int q = 0; q < K; ++q) sorted[warp][lane * K + q] = __int_as_float(v[q]);
    __syncwarp();
    if (lane == 0) scores[i] = py_sum(sorted[warp], count);
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int r = threadIdx.x; r < n; r += kSelThreads) key[r] = __ldcg(scores + r);
  __syncthreads();
  stable_order(key, n, order);
  if (threadIdx.x == 0) {
    if (status != nullptr) *status = bulyan ? bulyan_status(key, n, f, m) : BZ_STATUS_OK;
    *ticket = 0u;
  }
}

void launch_select_many(const double* table, const ManyAliasMap& map, int n, int u, int count, double* scores,
                        int32_t* order, int32_t* status, int f, int m, int bulyan, unsigned* ticket, cudaStream_t st) {
  const unsigned blocks = (unsigned)((n + kSelWarps - 1) / kSelWarps);
  if (n <= 256)
    k5_select_many<256><<<blocks, kSelThreads, 0, st>>>(table, map, n, u, count, scores, order, status, f, m, bulyan, ticket);
  else if (n <= 512)
    k5_select_many<512><<<blocks, kSelThreads, 0, st>>>(table, map, n, u, count, scores, order, status, f, m, bulyan, ticket);
  else
    k5_select_many<1024><<<blocks, kSelThreads, 0, st>>>(table, map, n, u, count, scores, order, status, f, m, bulyan, ticket);
}

}  // namespace bz
