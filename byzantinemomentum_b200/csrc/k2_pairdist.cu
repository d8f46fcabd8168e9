// k2_pairdist.cu — K2 for rows the ring kernel (k2_ring.cu) does not take: all n(n-1)/2 squared
// pairwise distances in ONE pass over the rows (the reference makes n(n-1)/2 passes of
// `x.sub(y).norm().item()`, each with a host sync: krum.py:44-48, bulyan.py:49-54, brute.py:44-45).
// `launch_pairdist_auto` runs the ring and falls back to this kernel for rows that are not 16-byte
// aligned (e.g. views at odd offsets) or when the ring cannot launch.  Also the fixed-order sum of
// the per-CTA blocks (`launch_reduce_parts`).
//
// Layout: persistent CTAs (one per SM) walk tiles of T coordinates.  A tile of all n rows
// is staged in shared memory with cp.async (zero-filled past d), double buffered.  Rows are
// grouped by 5; a warp owns one group pair (A, B) — a 5x5 block of row pairs (10 pairs on
// the diagonal) — and sweeps the tile: each lane reads 4 adjacent coordinates of the 10 rows
// (LDS.128, conflict free) and feeds 25 accumulators, each a pair of coordinates updated with
// one FADD and one FFMA per coordinate (reduce.cuh).  No Gram trick: (a-b)^2 is formed
// directly, so aliased rows give an exact 0 and nothing cancels (SURVEY.md §7.2).
// Every tile (<= 1024 coordinates, i.e. <= 16 terms per fp32 accumulator half) the 25 lane
// partials are transposed-reduced over the warp (lane p ends with pair p) and added to a
// per-lane fp64 accumulator; per-CTA fp64 blocks are summed in fixed order by K5.
// Every pair walks the coordinates in the same lane/step pattern, so identical data (aliased
// rows) give bitwise identical sums.
// Roofline: HBM n·4 B per coordinate; secondary: FP32 pipe, n(n-1) lane-ops per coordinate.
#include "dist.cuh"
#include "reduce.cuh"

namespace bz {

constexpr int kG = 5;
constexpr int kK2Warps = 16;
constexpr int kK2Threads = kK2Warps * 32;
constexpr int kStep = 128;              // coordinates per warp step (4 per lane)
constexpr size_t kK2SmemBudget = 226 * 1024;

__device__ __forceinline__ void cp_async16(float* smem, const float* gmem, int src_bytes) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async4(float* smem, const float* gmem, int src_bytes) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(s), "l"(gmem), "r"(src_bytes) : "memory");
}

// Stage tile [base, base+T) of every row into buf[n][T]; zero fill past d.
__device__ __forceinline__ void stage_tile(float* buf, const RowTable& rows, int n, int T, int logq,
                                           int64_t base, int64_t d) {
  const int total = n << logq;            // 16-byte chunks: n * T/4
  for (int q = threadIdx.x; q < total; q += kK2Threads) {
    const int r = q >> logq, cq = q & ((1 << logq) - 1);
    const float* row = rows.p[r];
    const int64_t col = base + (int64_t)cq * 4;
    const int64_t remain = d - col;
    float* dst = buf + r * T + cq * 4;
    if ((((uintptr_t)row) & 15) == 0) {
      const int bytes = remain >= 4 ? 16 : (remain > 0 ? (int)remain * 4 : 0);
      cp_async16(dst, bytes ? row + col : row, bytes);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int bytes = remain > e ? 4 : 0;
        cp_async4(dst + e, bytes ? row + col + e : row, bytes);
      }
    }
  }
}

// DIAG: both groups are the same (pairs i < j only; with SELF also i == j: the "distance" of a
// row to itself, 0 for a finite row and NaN for a row holding NaN / inf — what the reference
// gets from x.sub(x).norm() for aliased rows; needed when aliases are de-duplicated).
template <bool DIAG, bool SELF = false>
__device__ __forceinline__ void sweep_tile(const float* buf, int T, const int (&oa)[kG], const int (&ob)[kG],
                                           int lane, u64 (&acc)[kG * kG]) {
  for (int c = lane * 4; c < T; c += kStep) {
    u64 a0[kG], a1[kG], b0[kG], b1[kG];
#pragma unroll
    for (int i = 0; i < kG; ++i) {
      const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(buf + oa[i] + c);
      a0[i] = t.x; a1[i] = t.y;
    }
    if (!DIAG) {
#pragma unroll
      for (int j = 0; j < kG; ++j) {
        const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(buf + ob[j] + c);
        b0[j] = t.x; b1[j] = t.y;
      }
#pragma unroll
      for (int i = 0; i < kG; ++i)
#pragma unroll
        for (int j = 0; j < kG; ++j) {
          const u64 d0 = sub2(a0[i], b0[j]), d1 = sub2(a1[i], b1[j]);
          acc[i * kG + j] = fma2(d0, d0, acc[i * kG + j]);
          acc[i * kG + j] = fma2(d1, d1, acc[i * kG + j]);
        }
    } else {
      int p = 0;
#pragma unroll
      for (int i = 0; i < kG; ++i)
#pragma unroll
        for (int j = i + (SELF ? 0 : 1); j < kG; ++j) {
          const u64 d0 = sub2(a0[i], a0[j]), d1 = sub2(a1[i], a1[j]);
          acc[p] = fma2(d0, d0, acc[p]);
          acc[p] = fma2(d1, d1, acc[p]);
          ++p;
        }
    }
  }
}

// lane p -> p-th pair of a diagonal task, row-major; i < j (10 pairs) or i <= j (15 pairs, SELF)
__device__ __forceinline__ void diag_pair(int lane, bool self, int& i, int& j, bool& valid) {
  if (self) {
    i = (lane >= 14) ? 4 : (lane >= 12) ? 3 : (lane >= 9) ? 2 : (lane >= 5) ? 1 : 0;
    const int first = (i == 0) ? 0 : (i == 1) ? 5 : (i == 2) ? 9 : (i == 3) ? 12 : 14;
    j = lane - first + i;
    valid = lane < 15;
  } else {
    i = (lane >= 9) ? 3 : (lane >= 7) ? 2 : (lane >= 4) ? 1 : 0;
    const int first = (i == 0) ? 0 : (i == 1) ? 4 : (i == 2) ? 7 : 9;
    j = lane - first + i + 1;
    valid = lane < 10;
  }
}

template <int NP>
__device__ __forceinline__ void flush(u64 (&acc)[kG * kG], int lane, double& dacc) {
  float v[32];
#pragma unroll
  for (int p = 0; p < 32; ++p) v[p] = (p < NP) ? half_sum(acc[p]) : 0.f;
#pragma unroll
  for (int p = 0; p < kG * kG; ++p) acc[p] = 0ull;
  dacc += (double)transpose_reduce(v, lane);
}

__global__ void __launch_bounds__(kK2Threads, 1)
k2_pairdist(const __grid_constant__ RowTable rows, const int n, const int T, const int logq, const int64_t d,
            const int64_t ntiles, const int self_pairs, double* __restrict__ parts) {
  extern __shared__ __align__(16) float smem[];   // [2][n][T]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ng = (n + kG - 1) / kG;
  const int ntasks = ng * (ng + 1) / 2;
  int task = blockIdx.y * kK2Warps + warp;
  const bool active = task < ntasks;
  int ga = 0, gb = 0;
  if (active) {
    int t = task;
    while (t >= ng - ga) { t -= ng - ga; ++ga; }
    gb = ga + t;
  }
  const bool diag = ga == gb;
  int oa[kG], ob[kG];
#pragma unroll
  for (int i = 0; i < kG; ++i) {
    oa[i] = min(ga * kG + i, n - 1) * T;
    ob[i] = min(gb * kG + i, n - 1) * T;
  }
  u64 acc[kG * kG];
#pragma unroll
  for (int p = 0; p < kG * kG; ++p) acc[p] = 0ull;
  double dacc = 0.;

  const int stage_floats = n * T;
  int64_t tile = blockIdx.x;
  if (tile < ntiles) stage_tile(smem, rows, n, T, logq, tile * T, d);
  cp_async_commit();
  int cur = 0;
  for (; tile < ntiles; tile += gridDim.x) {
    const int64_t next = tile + gridDim.x;
    if (next < ntiles) stage_tile(smem + (cur ^ 1) * stage_floats, rows, n, T, logq, next * T, d);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    if (active) {
      const float* buf = smem + cur * stage_floats;
      if (diag && self_pairs) { sweep_tile<true, true>(buf, T, oa, ob, lane, acc); flush<15>(acc, lane, dacc); }
      else if (diag)          { sweep_tile<true>(buf, T, oa, ob, lane, acc); flush<10>(acc, lane, dacc); }
      else                    { sweep_tile<false>(buf, T, oa, ob, lane, acc); flush<kG * kG>(acc, lane, dacc); }
    }
    __syncthreads();
    cur ^= 1;
  }
  cp_async_wait<0>();

  if (active) {
    int i, j;
    bool valid;
    if (diag) {
      diag_pair(lane, self_pairs != 0, i, j, valid);
    } else {
      i = lane / kG; j = lane % kG;
      valid = lane < kG * kG;
    }
    const int ri = ga * kG + i, rj = gb * kG + j;
    if (valid && ri < n && rj < n) parts[(size_t)blockIdx.x * n * n + (size_t)ri * n + rj] = dacc;
  }
}

// ---- fixed-order reduction of partial blocks --------------------------------------------------
// One CTA per 32 entries; warp w adds the blocks p = w, w + 8, ... (coalesced 256-byte rows of
// 32 entries), the 8 warp sums are then added in warp order: a fixed order, whatever the grid.
__global__ void __launch_bounds__(kReduceWarps * 32)
k_reduce_parts(const double* __restrict__ parts, int nparts, int len, int pair_n, double* __restrict__ block) {
  __shared__ double partial[kReduceWarps][32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e = blockIdx.x * 32 + lane;
  double s = 0.;
  if (e < len)
    for (int p = warp; p < nparts; p += kReduceWarps) s += parts[(size_t)p * len + e];
  partial[warp][lane] = s;
  __syncthreads();
  if (warp == 0 && e < len) {
    double total = 0.;
#pragma unroll
    for (int w = 0; w < kReduceWarps; ++w) total += partial[w][lane];
    if (pair_n > 0 && (e / pair_n) >= (e % pair_n)) total = 0.;
    block[e] = total;
  }
}

// ---- host side ---------------------------------------------------------------------------

// cp.async staging, any alignment.  Largest power-of-two tile whose two stages fit the shared
// memory of one CTA per SM.
static int launch_pairdist(const RowTable& rows, int n, int64_t d, double* parts, cudaStream_t st, int self_pairs) {
  const int ng = (n + kG - 1) / kG;
  const int ntasks = ng * (ng + 1) / 2;
  const int gy = (ntasks + kK2Warps - 1) / kK2Warps;
  int T = 1024;
  while (T > 128 && (size_t)2 * n * T * sizeof(float) > kK2SmemBudget) T >>= 1;
  int logq = 0;
  while ((1 << logq) < T / 4) ++logq;
  const size_t smem = (size_t)2 * n * T * sizeof(float);
  static unsigned long long opted = 0;
  {
    int dev = 0;
    cudaGetDevice(&dev);
    const unsigned long long bit = 1ull << (dev & 63);
    if (!(opted & bit)) {
      cudaFuncSetAttribute(k2_pairdist, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kK2SmemBudget);
      opted |= bit;
    }
  }
  const int64_t ntiles = (d + T - 1) / T;
  int gx = sm_count() / (gy > 0 ? gy : 1);
  if (gx < 1) gx = 1;
  if (gx > kMaxParts) gx = kMaxParts;
  if ((int64_t)gx > ntiles) gx = (int)(ntiles > 0 ? ntiles : 1);
  k2_pairdist<<<dim3(gx, gy > 0 ? gy : 1), kK2Threads, smem, st>>>(rows, n, T, logq, d, ntiles, self_pairs, parts);
  return gx;
}

int aliased_rows(const int* to_unique, int u, int n_orig, unsigned char* self_rows) {
  int nself = 0;
  if (to_unique != nullptr && u < n_orig) {
    int mult[kMaxN] = {0};
    for (int i = 0; i < n_orig; ++i) ++mult[to_unique[i]];
    for (int k = 0; k < u; ++k)
      if (mult[k] > 1) self_rows[nself++] = (unsigned char)k;
  }
  return nself;
}

int launch_pairdist_rows(const RowTable& rows, int u, int64_t d, double* parts, cudaStream_t st,
                         const unsigned char* self_rows, int nself, SelectTail* select) {
  const int nparts = launch_pairdist_ring(rows, u, d, parts, st, self_rows, nself, select);
  if (nparts > 0) return nparts;
  if (select != nullptr) select->fused = 0;
  return launch_pairdist(rows, u, d, parts, st, nself > 0 ? 1 : 0);
}

int launch_pairdist_auto(const RowTable& rows, int u, int64_t d, double* parts, cudaStream_t st,
                         const int* to_unique, int n_orig, SelectTail* select) {
  unsigned char self_rows[kMaxN];
  const int nself = aliased_rows(to_unique, u, n_orig, self_rows);
  return launch_pairdist_rows(rows, u, d, parts, st, self_rows, nself, select);
}

void launch_reduce_parts(const double* parts, int nparts, int len, int pair_n, double* block, cudaStream_t st) {
  k_reduce_parts<<<(len + 31) / 32, kReduceWarps * 32, 0, st>>>(parts, nparts, len, pair_n, block);
}

}  // namespace bz
