// k2_star_many.cu — K2-star-many: the squared distances of one row, the candidate, to the u - 1 other unique rows
// (and to itself), above kMaxNDistance rows, with K2-many's bits (bz_distance_line_search_many).
//
// K2-many's contract per pair and slice: every 32-column chunk is an fp32 FFMA sum of its (x - y)^2 in column order,
// and the slice's fp64 sum takes the chunk sums in chunk order.  The fold within a slice is the only serial step, and
// the slices are few at large u (4 at u = 770), so the parallelism comes from rows and chunks inside a slice:
//   * a CTA takes kStarRows rows (two per warp) and one slice, and walks the slice 32 chunks (1024 columns) at a
//     time: every thread loads its columns of the next stage into registers while the current stage is summed;
//   * a stage is stored to shared memory with a row of 33 floats per chunk, so that lane k then reads chunk k's
//     columns in order without a bank conflict and computes the chunk's fp32 sum for both of its rows;
//   * the 32 chunk sums are added to the fp64 accumulator in chunk order, through shuffles;
//   * the candidate's stage is shared by the CTA's rows: it is read from L2 once per kStarRows rows.
// k2_starfold_many then adds the slices' sums in slice order into the table's column c.
// Roofline: HBM, (u - 1) * 4 B per column (the candidate comes from L2).
#include "distance_many.cuh"

namespace bz {

constexpr int kStarThreads = 256;
constexpr int kStarWarps = kStarThreads / 32;
constexpr int kStarRowsPerWarp = 2;
constexpr int kStarRows = kStarWarps * kStarRowsPerWarp;
constexpr int kStarLd = kPairChunk + 1;             // floats per staged chunk: lane k reads bank (k + j) % 32
constexpr int kStarStageFloats = 32 * kStarLd;      // 32 chunks, one per lane
constexpr int kStarStageCols = 32 * kPairChunk;
constexpr size_t kStarSmem = (size_t)(1 + kStarRows) * kStarStageFloats * sizeof(float);

__global__ void __launch_bounds__(kStarThreads, 2)
k2_star_many(const __grid_constant__ ManyRowTable uniq, const int u, const int64_t d, const int64_t slice_chunks,
             double* __restrict__ blocks) {
  extern __shared__ __align__(16) float sm_star[];
  float* cand_s = sm_star;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* rows_s = sm_star + (1 + warp * kStarRowsPerWarp) * kStarStageFloats;
  const int a0 = blockIdx.x * kStarRows + warp * kStarRowsPerWarp;
  const int64_t c_first = (int64_t)blockIdx.y * slice_chunks;
  const int64_t total = (d + kPairChunk - 1) / kPairChunk;
  const int nchunks = (int)((c_first + slice_chunks < total ? c_first + slice_chunks : total) - c_first);
  const int64_t col_first = c_first * kPairChunk;
  const int64_t col_end = col_first + (int64_t)nchunks * kPairChunk < d ? col_first + (int64_t)nchunks * kPairChunk : d;
  const float* y = uniq.p[u - 1];
  const float* x[kStarRowsPerWarp];
  bool live[kStarRowsPerWarp];
#pragma unroll
  for (int r = 0; r < kStarRowsPerWarp; ++r) {
    live[r] = a0 + r < u;
    x[r] = uniq.p[live[r] ? a0 + r : 0];
  }

  // Stage t: columns col_first + t * kStarStageCols + [0, kStarStageCols); columns past the slice or past d are 0.
  float xv[kStarRowsPerWarp][32], yv[kStarStageCols / kStarThreads];
  auto load = [&](int t) {
    const int64_t base = col_first + (int64_t)t * kStarStageCols;
#pragma unroll
    for (int r = 0; r < kStarRowsPerWarp; ++r)
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        const int64_t col = base + q * kPairChunk + lane;
        xv[r][q] = (live[r] && col < col_end) ? __ldcs(x[r] + col) : 0.f;
      }
#pragma unroll
    for (int q = 0; q < kStarStageCols / kStarThreads; ++q) {
      const int64_t col = base + q * kStarThreads + threadIdx.x;
      yv[q] = col < col_end ? __ldg(y + col) : 0.f;
    }
  };

  double acc[kStarRowsPerWarp];
#pragma unroll
  for (int r = 0; r < kStarRowsPerWarp; ++r) acc[r] = 0.;
  const int nstages = (nchunks + 31) / 32;
  load(0);
#pragma unroll 1
  for (int t = 0; t < nstages; ++t) {
#pragma unroll
    for (int r = 0; r < kStarRowsPerWarp; ++r)
#pragma unroll
      for (int q = 0; q < 32; ++q) rows_s[r * kStarStageFloats + q * kStarLd + lane] = xv[r][q];
#pragma unroll
    for (int q = 0; q < kStarStageCols / kStarThreads; ++q) {
      const int e = q * kStarThreads + threadIdx.x;
      cand_s[(e >> 5) * kStarLd + (e & 31)] = yv[q];
    }
    __syncthreads();                                  // stage t is in shared memory
    if (t + 1 < nstages) load(t + 1);
    float part[kStarRowsPerWarp];
#pragma unroll
    for (int r = 0; r < kStarRowsPerWarp; ++r) part[r] = 0.f;
#pragma unroll 8
    for (int j = 0; j < kPairChunk; ++j) {
      const float yj = cand_s[lane * kStarLd + j];
#pragma unroll
      for (int r = 0; r < kStarRowsPerWarp; ++r) {
        const float df = __fsub_rn(rows_s[r * kStarStageFloats + lane * kStarLd + j], yj);
        part[r] = __fmaf_rn(df, df, part[r]);
      }
    }
    const int valid = nchunks - t * 32 < 32 ? nchunks - t * 32 : 32;
#pragma unroll 1
    for (int k = 0; k < valid; ++k)
#pragma unroll
      for (int r = 0; r < kStarRowsPerWarp; ++r) acc[r] += (double)__shfl_sync(0xffffffffu, part[r], k);
    __syncthreads();                                  // every warp is done with stage t
  }
  if (lane == 0)
#pragma unroll
    for (int r = 0; r < kStarRowsPerWarp; ++r)
      if (live[r]) blocks[(size_t)blockIdx.y * u + a0 + r] = acc[r];
}

// table[a * u + c] (a <= c) = the row's slice sums added in slice order, ((s0 + s1) + s2) + ...
__global__ void __launch_bounds__(256)
k2_starfold_many(const double* __restrict__ blocks, const int u, const int slices, double* __restrict__ table) {
  const int a = blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= u) return;
  double v = __ldcg(blocks + a);
  for (int s = 1; s < slices; ++s) v += __ldcg(blocks + (size_t)s * u + a);
  table[(size_t)a * u + (u - 1)] = v;
}

void launch_star_many(const ManyRowTable& uniq, int u, int64_t d, const PairGrid& g, double* blocks, double* table,
                      cudaStream_t st) {
  if (d <= 0) return;
  static unsigned long long opted = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(opted & bit)) {
    cudaFuncSetAttribute(k2_star_many, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStarSmem);
    opted |= bit;
  }
  k2_star_many<<<dim3((u + kStarRows - 1) / kStarRows, g.slices), kStarThreads, kStarSmem, st>>>(uniq, u, d, g.slice_chunks,
                                                                                               blocks);
  k2_starfold_many<<<(u + 255) / 256, 256, 0, st>>>(blocks, u, g.slices, table);
}

}  // namespace bz
