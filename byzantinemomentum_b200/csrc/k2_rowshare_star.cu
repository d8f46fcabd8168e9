// k2_rowshare_star.cu — K2'-star (libbyzagg_star.so, include/byzagg_rowshare_star.h): CGE's phase A of the d-sharded
// line search above 64 rows after its first evaluation.  The honest rows' sums of squares do not change from one
// evaluation to the next; only the candidate's does, and the candidate is one row repeated as rows [c0, n).  So this
// kernel reads that one row and writes part[c0, n) with the bits k2_rowshare_wide (bz_distance_partial, CGE) writes
// there, leaving part[0, c0) as it is.
//
// The bits follow rowdist_wide_body (k2_rowdist_wide.cu) step for step:
//   * the grid is rowdist_wide_grid's (at most 2 CTAs per SM and kMaxParts), the same warp-uniform walk over d;
//   * a chunk's 32 fp32 squares go through transpose_reduce (reduce.cuh) with 0 in the entries of the rows outside
//     [c0, n): an entry only ever meets the same entry of the other lanes, so a row's sum is the one K2'-share forms;
//   * the 8 warps are added in warp order, one fp64 block per CTA;
//   * the last CTA (ticket) sums the blocks in S = 256 / n interleaved classes, with the real n, then the classes in
//     class order.
// Roofline: HBM, 4 B per coordinate instead of K2'-share's n * 4 B.
#include "dist.cuh"
#include "reduce.cuh"

namespace bz {

constexpr int kStarThreads = 256;
constexpr int kStarWarps = kStarThreads / 32;
constexpr int kStarChunks = BZ_MAX_N_DISTANCE / 32;

__global__ void __launch_bounds__(kStarThreads, 2)
k2_rowshare_star(const float* __restrict__ cand, const int n, const int c0, const int64_t d, double* __restrict__ parts,
                 unsigned* __restrict__ ticket, double* __restrict__ sums) {
  __shared__ double warp_tot[kStarWarps][BZ_MAX_N_DISTANCE];
  __shared__ bool last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ch0 = c0 / 32, ch1 = (n - 1) / 32;                // the chunks that hold rows of [c0, n)
  double dr[kStarChunks];
#pragma unroll
  for (int c = 0; c < kStarChunks; ++c) dr[c] = 0.;
  const int64_t stride = (int64_t)gridDim.x * kStarThreads;
  const int64_t first = (int64_t)blockIdx.x * kStarThreads + warp * 32;
  for (int64_t vf = first; vf < d; vf += stride) {
    const int64_t e = vf + lane;
    const float x = e < d ? __ldcs(cand + e) : 0.f;
    const float sq = __fmul_rn(x, x);
#pragma unroll
    for (int ch = 0; ch < kStarChunks; ++ch) {
      if (ch < ch0 || ch > ch1) continue;                     // warp-uniform
      float v[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int r = ch * 32 + j;
        v[j] = (r >= c0 && r < n) ? sq : 0.f;
      }
      dr[ch] += (double)transpose_reduce(v, lane);
    }
  }
#pragma unroll
  for (int c = 0; c < kStarChunks; ++c) warp_tot[warp][c * 32 + lane] = dr[c];
  __syncthreads();
  if ((int)threadIdx.x >= c0 && (int)threadIdx.x < n) {
    double s = 0.;
#pragma unroll
    for (int w = 0; w < kStarWarps; ++w) s += warp_tot[w][threadIdx.x];
    parts[(size_t)blockIdx.x * n + threadIdx.x] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double* partial = &warp_tot[0][0];                          // S * n <= kStarThreads doubles
  const int S = kStarThreads / n;                             // 2 or 3
  const int c = threadIdx.x % n, cls = threadIdx.x / n;
  if (cls < S && c >= c0) {
    double s = 0.;
    for (int p = cls; p < (int)gridDim.x; p += S) s += __ldcg(parts + (size_t)p * n + c);
    partial[cls * n + c] = s;
  }
  __syncthreads();
  if ((int)threadIdx.x >= c0 && (int)threadIdx.x < n) {
    double sum = 0.;
    for (int k = 0; k < S; ++k) sum += partial[k * n + threadIdx.x];
    sums[threadIdx.x] = sum;
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

// rowdist_wide_grid's geometry for VEC = 1 (nv = d): at most two CTAs per SM and kMaxParts; the ticket is zeroed first.
int launch_rowshare_star(const float* cand, int n, int c0, int64_t d, int sms, double* parts, unsigned* ticket,
                         double* sums, cudaStream_t st) {
  int64_t grid = (d + kStarThreads - 1) / kStarThreads;
  if (grid > (int64_t)sms * 2) grid = (int64_t)sms * 2;
  if (grid > kMaxParts) grid = kMaxParts;
  if (grid < 1) grid = 1;
  cudaMemsetAsync(ticket, 0, sizeof(unsigned), st);
  k2_rowshare_star<<<(unsigned)grid, kStarThreads, 0, st>>>(cand, n, c0, d, parts, ticket, sums);
  return (int)grid;
}

}  // namespace bz
