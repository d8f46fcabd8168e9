// k5_wide.cuh — the scoring and selection steps of Multi-Krum and Bulyan above 64 rows, one CTA of
// kK5WideThreads threads, shared by K5-wide (k5_score_wide.cu, libbyzagg.so) and by the selection kernel that
// exchanges phase A's blocks over peer memory (k5_select_peers.cu, libbyzagg_peers.so): the n x n tables of fp32
// norms in dynamic shared memory, and the opt-in to more than 48 KB of it.
#pragma once

#include "k5_device.cuh"

namespace bz {

constexpr int kK5WideThreads = 1024;

// The steps after the n x n table `dist` of fp32 norms is filled: each row sorted into `sorted`, the rule's
// compensated sums into `score`, the stable order, the status word.
__device__ __forceinline__ void score_from_floats(const float* dist, float* sorted, double* score, int n, int count,
                                                  int32_t* __restrict__ order, int32_t* __restrict__ status, int f, int m,
                                                  int bulyan) {
  __syncthreads();
  sort_rows(dist, sorted, n);
  for (int i = threadIdx.x; i < n; i += blockDim.x) score[i] = py_sum(sorted + i * n, count);
  __syncthreads();
  stable_order(score, n, order);
  if (threadIdx.x == 0 && status != nullptr) *status = bulyan ? bulyan_status(score, n, f, m) : BZ_STATUS_OK;
}

constexpr size_t kScoreWideSmemMax = (size_t)kMaxNDistance * sizeof(double) + 2 * (size_t)kMaxNDistance * kMaxNDistance * sizeof(float);

// The scores (n doubles), then the table and its sorted rows (n x n floats each).
static inline size_t score_wide_smem(int n) { return (size_t)n * sizeof(double) + 2 * (size_t)n * n * sizeof(float); }

// Once per device and kernel (`opted`: one bit per device): the largest table's shared memory.
template <class K>
static void opt_in_wide(K kernel, unsigned long long& opted) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(opted & bit)) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kScoreWideSmemMax);
    opted |= bit;
  }
}

}  // namespace bz
