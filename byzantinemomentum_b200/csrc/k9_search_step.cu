// k9_search_step.cu — K9: the transition of the d-sharded line search.  Every rank's score pass leaves
// its fp64 share of sum_k fl32(out_k - avg_k)^2; once the R shares are all-gathered, one thread adds them
// in rank order, ((p0 + p1) + p2) + ..., rounds the sum to fp32 (y) and runs the transition — the same
// bits on every rank, hence the same next factor.  With R = 1 the sum is p0 itself: the y of the
// single-GPU score pass.
#include "search.cuh"

namespace bz {

__global__ void __launch_bounds__(32) k9_search_step(const double* __restrict__ partials, const int nparts, const SearchTail tail) {
  if (threadIdx.x != 0) return;
  double sum = partials[0];
  for (int p = 1; p < nparts; ++p) sum += partials[p];
  search_step(tail, (double)(float)sum);
}

int launch_search_step(const double* partials, int nparts, const SearchTail& tail, cudaStream_t st) {
  k9_search_step<<<1, 32, 0, st>>>(partials, nparts, tail);
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -1;
}

}  // namespace bz
