// k2_pairshare_wide.cu — phase A of Multi-Krum and Bulyan above 64 rows on a d-shard (bz_distance_partial): the
// n x n block of this shard's squared distances in the layout of the original rows, read from the pass tables
// that bz_distance's passes left (dist.cuh, PassTables).  Entry (i, j), i < j, is the pair of the unique rows
// i and j map to, the self distance when they alias; every other entry is 0 (bz_pairdist_partial's layout).
#include "dist.cuh"

namespace bz {

constexpr int kPairShareThreads = 256;

__global__ void __launch_bounds__(kPairShareThreads)
k2_pairshare_wide(const __grid_constant__ PassTables t, int n, double* __restrict__ block) {
  const int e = blockIdx.x * kPairShareThreads + threadIdx.x;
  if (e >= n * n) return;
  const int i = e / n, j = e - i * n;
  double v = 0.;
  if (i < j) {
    const int a = t.to_unique[i], b = t.to_unique[j];
    v = pass_sq(t, min(a, b), max(a, b));
  }
  block[e] = v;
}

void launch_pairshare_wide(const PassTables& t, int n, double* block, cudaStream_t st) {
  k2_pairshare_wide<<<(n * n + kPairShareThreads - 1) / kPairShareThreads, kPairShareThreads, 0, st>>>(t, n, block);
}

}  // namespace bz
