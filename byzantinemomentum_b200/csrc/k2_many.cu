// k2_many.cu — the distance passes of Multi-Krum, Bulyan, Aksel and CGE above kMaxNDistance rows
// (bz_distance_many), over up to kMaxNMany rows.
//
// K2-many: the pairwise squared distances of the u unique rows.  The rows are cut into tiles of kPairTile; a CTA
// takes one pair of tiles I <= J (the upper triangle of the tile grid) and one slice of the columns, so that every
// row is read once per tile pair, not once per pair of rows:
//   * a ring of kPairStages stages, each one 32-column chunk of both tiles, staged by 4-byte cp.async (rows keep any
//     4-byte offset; thread t always copies 16 adjacent columns of the same row, so its row pointer is computed
//     once), column c of a tile at c * kPairLd: a thread's four rows of a column are one float4;
//   * each of the 16 x 16 threads keeps a 4 x 4 micro-tile of pairs: (a - b) in fp32, squared by FFMA into an fp32
//     sum of the chunk's at most 32 terms, flushed into fp64 after each chunk (K2's contract, DESIGN §4.2);
//   * the diagonal tile pair also gives the self distance of every row: 0, or NaN for a row holding NaN / inf;
//   * the slices (a function of u and d only, never of the device: as many as fit the tile pairs in 396 CTAs, one
//     wave of three CTAs on each of the H100's 132 SMs, so that no CTA runs in a second, nearly empty wave there) write
//     one fp64 block each, and
//     k2_pairsum_many adds a pair's blocks in slice order.  Deterministic: nothing depends on timing.
// Roofline: FP32, 2 lane operations per pair and coordinate; the diagonal tiles compute their pairs twice.
//
// K2'-many: Aksel's squared distance of every row to the centre and CGE's squared norm, K2''s arithmetic over the
// 1024-pointer table: a warp takes 32 adjacent coordinates of 32 rows, the squares go through the transposed warp
// reduction (an fp32 sum over the 32 coordinates) into one fp64 sum per row and lane; the 32-row chunks follow one
// another, the warps are added in warp order and the last CTA (ticket) adds the per-CTA blocks in CTA order and
// writes the stable order of the keys.  Roofline: HBM, n * 4 B per coordinate (+4 B of centre per 32 rows, from L2).
#include "distance_many.cuh"
#include "k5_device.cuh"
#include "reduce.cuh"

namespace bz {

constexpr int kPairThreads = 256;
constexpr int kPairStages = 3;
constexpr int kPairLd = kPairTile + 4;              // floats per staged column: float4 reads stay aligned
constexpr int kPairTileFloats = kPairChunk * kPairLd;
constexpr int kPairStageFloats = 2 * kPairTileFloats;
constexpr size_t kPairSmem = (size_t)kPairStages * kPairStageFloats * sizeof(float);

__global__ void __launch_bounds__(kPairThreads, 3)
k2_pairdist_many(const __grid_constant__ ManyRowTable uniq, const int u, const int64_t d, const int tiles,
                 const int npairs, const int64_t slice_chunks, double* __restrict__ parts) {
  extern __shared__ __align__(16) float sm_pair[];
  int p = blockIdx.x, I = 0;
  while (p >= tiles - I) { p -= tiles - I; ++I; }
  const int J = I + p;
  const int64_t c_first = (int64_t)blockIdx.y * slice_chunks;
  const int64_t total = (d + kPairChunk - 1) / kPairChunk;
  const int nchunks = (int)((c_first + slice_chunks < total ? c_first + slice_chunks : total) - c_first);
  const int tid = threadIdx.x;
  const int ty = tid >> 4, tx = tid & 15;

  // Stage chunk k (columns c_first + k of the slice) into stage s: thread t copies columns h .. h + 15 (h = 16 (t & 1))
  // of row t / 2 of the two tiles; a row past u is left as it is (its pairs are never written), columns past d are zero.
  const int cr = tid >> 1, ch = (tid & 1) * 16;
  const int crow = (cr < kPairTile ? I : J) * kPairTile + (cr & (kPairTile - 1));
  const float* src = uniq.p[crow < u ? crow : 0] + ch;
  const int dst0 = (cr >> 6) * kPairTileFloats + ch * kPairLd + (cr & (kPairTile - 1));
  auto issue = [&](int k, int s) {
    if (crow >= u) return;
    float* dst = sm_pair + s * kPairStageFloats + dst0;
    const int64_t col0 = (c_first + k) * kPairChunk;
    if (col0 + ch + 16 <= d) {
#pragma unroll
      for (int q = 0; q < 16; ++q) cp_async_vec<1>(dst + q * kPairLd, src + col0 + q);
    } else {
      for (int q = 0; q < 16; ++q) {
        if (col0 + ch + q < d) cp_async_vec<1>(dst + q * kPairLd, src + col0 + q);
        else                   dst[q * kPairLd] = 0.f;
      }
    }
  };

  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.;

#pragma unroll
  for (int s = 0; s < kPairStages - 1; ++s) {
    if (s < nchunks) issue(s, s);
    cp_async_commit();
  }
#pragma unroll 1
  for (int k = 0; k < nchunks; ++k) {
    cp_async_wait<kPairStages - 2>();
    __syncthreads();                                  // chunk k has landed, and every thread is done with k - 1
    const int ahead = k + kPairStages - 1;
    if (ahead < nchunks) issue(ahead, ahead % kPairStages);
    cp_async_commit();
    const float* a = sm_pair + (k % kPairStages) * kPairStageFloats + ty * 4;
    const float* b = sm_pair + (k % kPairStages) * kPairStageFloats + kPairTileFloats + tx * 4;
    float part[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) part[i][j] = 0.f;
#pragma unroll 8
    for (int c = 0; c < kPairChunk; ++c) {
      const float4 x = *reinterpret_cast<const float4*>(a + c * kPairLd);
      const float4 y = *reinterpret_cast<const float4*>(b + c * kPairLd);
      const float xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float df = __fsub_rn(xs[i], ys[j]);
          part[i][j] = __fmaf_rn(df, df, part[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] += (double)part[i][j];
  }
  cp_async_wait<0>();
  double* blk = parts + ((size_t)blockIdx.y * npairs + blockIdx.x) * kPairBlock;
  // 8-byte stores: the workspace is only required to be 8-byte aligned
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) blk[(ty * 4 + i) * kPairTile + tx * 4 + j] = acc[i][j];
}

// table[a * u + b] (a <= b) = the blocks of the pair's slices added in slice order, ((s0 + s1) + s2) + ...
__global__ void __launch_bounds__(256)
k2_pairsum_many(const double* __restrict__ parts, const int u, const int tiles, const int npairs, const int slices,
                double* __restrict__ table) {
  const int64_t len = (int64_t)u * u;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < len; e += (int64_t)gridDim.x * blockDim.x) {
    const int a = (int)(e / u), b = (int)(e - (int64_t)a * u);
    if (a > b) continue;
    const int I = a / kPairTile, J = b / kPairTile;
    const int pair = I * tiles - I * (I - 1) / 2 + (J - I);
    const double* src = parts + (size_t)pair * kPairBlock + (a % kPairTile) * kPairTile + b % kPairTile;
    double v = __ldcg(src);
    for (int s = 1; s < slices; ++s) v += __ldcg(src + (size_t)s * npairs * kPairBlock);
    table[e] = v;
  }
}

void launch_pairdist_many(const ManyRowTable& uniq, int u, int64_t d, const PairGrid& g, double* parts, double* table,
                          cudaStream_t st) {
  if (d <= 0) return;
  static unsigned long long opted = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(opted & bit)) {
    cudaFuncSetAttribute(k2_pairdist_many, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPairSmem);
    opted |= bit;
  }
  k2_pairdist_many<<<dim3(g.npairs, g.slices), kPairThreads, kPairSmem, st>>>(uniq, u, d, g.tiles, g.npairs,
                                                                               g.slice_chunks, parts);
  const int64_t len = (int64_t)u * u;
  const unsigned blocks = (unsigned)((len + 255) / 256 < 1024 ? (len + 255) / 256 : 1024);
  k2_pairsum_many<<<blocks, 256, 0, st>>>(parts, u, g.tiles, g.npairs, g.slices, table);
}

// ---- K2'-many -------------------------------------------------------------------------------------------------

constexpr int kRkThreads = 256;
constexpr int kRkWarps = kRkThreads / 32;

template <bool CENTER>
__global__ void __launch_bounds__(kRkThreads)
k2_rowkeys_many(const __grid_constant__ ManyRowTable rows, const int n, const float* __restrict__ center, const int64_t d,
                double* __restrict__ parts, int32_t* __restrict__ order, unsigned* __restrict__ ticket, const int sqrt_norm) {
  __shared__ double warp_tot[kRkWarps][32];
  __shared__ double key[kMaxNMany];
  __shared__ bool last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t stride = (int64_t)gridDim.x * kRkThreads;
  // warp-uniform trip count: lanes past the end contribute zeros and still join the shuffles
  const int64_t first = (int64_t)blockIdx.x * kRkThreads + warp * 32;
  const int chunks = (n + 31) / 32;
#pragma unroll 1
  for (int ch = 0; ch < chunks; ++ch) {
    double dr = 0.;
    for (int64_t vf = first; vf < d; vf += stride) {
      const int64_t e = vf + lane;
      const bool live = e < d;
      // out-of-range lanes and rows past n add exactly 0: they take the centre itself
      const float c = (CENTER && live) ? __ldg(center + e) : 0.f;
      float v[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int r = ch * 32 + j;
        v[j] = (live && r < n) ? __ldcs(rows.p[r] + e) : c;
      }
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        if (CENTER) {
          const float df = __fsub_rn(v[j], c);
          v[j] = __fmul_rn(df, df);                       // aksel.py:41: the square is rounded to fp32
        } else {
          v[j] = __fmul_rn(v[j], v[j]);
        }
      }
      dr += (double)transpose_reduce(v, lane);
    }
    warp_tot[warp][lane] = dr;
    __syncthreads();
    if (threadIdx.x < 32 && ch * 32 + (int)threadIdx.x < n) {
      double s = 0.;
#pragma unroll
      for (int w = 0; w < kRkWarps; ++w) s += warp_tot[w][threadIdx.x];
      parts[(size_t)blockIdx.x * n + ch * 32 + threadIdx.x] = s;
    }
    __syncthreads();
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  for (int i = threadIdx.x; i < n; i += kRkThreads) {
    double s = __ldcg(parts + i);
    for (int p = 1; p < (int)gridDim.x; ++p) s += __ldcg(parts + (size_t)p * n + i);
    key[i] = row_key(s, sqrt_norm);
  }
  __syncthreads();
  stable_order(key, n, order);
  if (threadIdx.x == 0) *ticket = 0u;
}

void launch_rowkeys_many(const ManyRowTable& rows, int n, const float* center, int64_t d, double* parts, int32_t* order,
                         unsigned* ticket, int sqrt_norm, cudaStream_t st) {
  int64_t grid = (d + kRkThreads - 1) / kRkThreads;
  if (grid > kMaxRowParts) grid = kMaxRowParts;
  if (grid < 1) grid = 1;
  if (center) k2_rowkeys_many<true><<<(unsigned)grid, kRkThreads, 0, st>>>(rows, n, center, d, parts, order, ticket, sqrt_norm);
  else        k2_rowkeys_many<false><<<(unsigned)grid, kRkThreads, 0, st>>>(rows, n, center, d, parts, order, ticket, sqrt_norm);
}

}  // namespace bz
