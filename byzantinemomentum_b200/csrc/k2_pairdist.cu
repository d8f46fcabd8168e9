// k2_pairdist.cu — K2: all n(n-1)/2 squared pairwise distances in ONE pass over the rows
// (the reference makes n(n-1)/2 passes of `x.sub(y).norm().item()`, each with a host sync:
// krum.py:44-48, bulyan.py:49-54, brute.py:44-45), and K2': squared distance of every row to
// a centre vector (cge.py:36, aksel.py:41).
//
// K2 layout: persistent CTAs (one per SM) walk tiles of T coordinates.  A tile of all n rows
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
#include <cstdlib>

#include "dist.cuh"
#include "reduce.cuh"
#include "tma.cuh"

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

// ---- K2 with TMA staging -------------------------------------------------------------------
// Same task layout and arithmetic as k2_pairdist, but full tiles are brought in by the TMA
// engine: ONE thread issues n bulk copies (cp.async.bulk, T·4 bytes each) per tile into a ring
// of kStages shared-memory stages, completion is signalled on an mbarrier (`full`), consumers
// release a stage through a second mbarrier (`empty`).  No block-wide barrier in the steady
// state and none of the per-thread address arithmetic of the cp.async loop (which cost ~25 %
// of the issue slots).  Needs 16-byte aligned rows; the ragged tail tile (and unaligned rows)
// take the cooperative path.  The producer is lane 0 of warp 0, whose own task is a diagonal
// (light) one, so waiting for the slowest warp before re-arming a stage costs it nothing.
// Tile width and minimum ring depth are build parameters for A/B runs (the bulk-copy issue loop is
// the measured bottleneck: `make VARIANT=t1024 EXTRA="-DBZ_K2_TMA_T=1024 -DBZ_K2_TMA_MIN_STAGES=2"`
// halves the copies per coordinate at n = 25).
#ifndef BZ_K2_TMA_T
#define BZ_K2_TMA_T 512
#endif
#ifndef BZ_K2_TMA_MIN_STAGES
#define BZ_K2_TMA_MIN_STAGES 3
#endif
constexpr int kTmaT = BZ_K2_TMA_T;  // coordinates per tile (a power of two, 256...1024)
constexpr int kTmaLogQ = (kTmaT == 256) ? 6 : (kTmaT == 512) ? 7 : 8;   // log2(kTmaT / 4)
// BZ_K2_FLUSH_SCALE (A/B builds): 2 = 32 fp32 terms per accumulator half between two flushes into
// fp64 instead of 16 (the transposed reduction is ~14 % of the executed instructions at n = 25).
#ifndef BZ_K2_FLUSH_SCALE
#define BZ_K2_FLUSH_SCALE 1
#endif
constexpr int kTmaFlush = (1024 / kTmaT) * BZ_K2_FLUSH_SCALE;   // tiles between flushes: <= 16 terms per accumulator half
static_assert(kTmaT == 256 || kTmaT == 512 || kTmaT == 1024, "BZ_K2_TMA_T");

template <int STAGES>
__global__ void __launch_bounds__(kK2Threads, 1)
k2_pairdist_tma(const __grid_constant__ RowTable rows, const int n, const int64_t d, const int64_t nfull,
                const int self_pairs, double* __restrict__ parts) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int T = kTmaT;
  float* stages = reinterpret_cast<float*>(smem_raw);
  const int stage_floats = n * T;
  unsigned long long* full = reinterpret_cast<unsigned long long*>(smem_raw + (size_t)STAGES * stage_floats * sizeof(float));
  unsigned long long* empty = full + STAGES;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ng = (n + kG - 1) / kG;
  const int ntasks = ng * (ng + 1) / 2;
  const int task = blockIdx.y * kK2Warps + warp;
  const bool active = task < ntasks;
  const int nactive = min(kK2Warps, ntasks - (int)blockIdx.y * kK2Warps);
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

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], nactive); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // Full tiles of this CTA: blockIdx.x, blockIdx.x + gridDim.x, ... < nfull
  const int64_t mine = (nfull > (int64_t)blockIdx.x) ? (nfull - 1 - blockIdx.x) / gridDim.x + 1 : 0;
  const unsigned tile_bytes = (unsigned)(n * T * sizeof(float));
  auto issue = [&](int64_t k) {      // producer thread only
    const int s = (int)(k % STAGES);
    float* dst = stages + (size_t)s * stage_floats;
    const int64_t base = (blockIdx.x + k * gridDim.x) * (int64_t)T;
    mbar_expect_tx(&full[s], tile_bytes);
    for (int r = 0; r < n; ++r) tma_load_1d(dst + r * T, rows.p[r] + base, T * sizeof(float), &full[s]);
  };
  if (threadIdx.x == 0)
    for (int64_t k = 0; k < mine && k < STAGES; ++k) issue(k);

  int pending = 0;
  for (int64_t k = 0; k < mine; ++k) {
    const int s = (int)(k % STAGES);
    const unsigned parity = (unsigned)((k / STAGES) & 1);
    if (active) {
      mbar_wait(&full[s], parity);
      const float* buf = stages + (size_t)s * stage_floats;
      if (diag && self_pairs) sweep_tile<true, true>(buf, T, oa, ob, lane, acc);
      else if (diag)          sweep_tile<true>(buf, T, oa, ob, lane, acc);
      else                    sweep_tile<false>(buf, T, oa, ob, lane, acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      if (++pending == kTmaFlush) {  // <= 16 terms per accumulator half between flushes
        pending = 0;
        if (diag) flush<15>(acc, lane, dacc); else flush<kG * kG>(acc, lane, dacc);
      }
    }
    if (threadIdx.x == 0 && k + STAGES < mine) {
      mbar_wait(&empty[s], parity);  // every consumer warp has released the stage
      issue(k + STAGES);
    }
  }
  // Ragged tail tile (d not a multiple of T): cooperative staging with zero fill, one CTA
  const int64_t ntiles = (d + T - 1) / T;
  if (ntiles > nfull && (nfull % gridDim.x) == blockIdx.x) {
    __syncthreads();                 // the ring is drained: stage 0 is free
    stage_tile(stages, rows, n, T, kTmaLogQ, nfull * T, d);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    if (active) {
      if (diag && self_pairs) sweep_tile<true, true>(stages, T, oa, ob, lane, acc);
      else if (diag)          sweep_tile<true>(stages, T, oa, ob, lane, acc);
      else                    sweep_tile<false>(stages, T, oa, ob, lane, acc);
      pending = 1;
    }
  }
  if (active && pending > 0) {
    if (diag) flush<15>(acc, lane, dacc); else flush<kG * kG>(acc, lane, dacc);
  }
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
constexpr int kReduceWarps = 8;
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

template <int STAGES>
static void launch_tma(const RowTable& rows, int n, int64_t d, int gx, int gy, int self_pairs, double* parts, cudaStream_t st) {
  const size_t smem = (size_t)STAGES * n * kTmaT * sizeof(float) + 2 * STAGES * sizeof(unsigned long long);
  static unsigned long long opted = 0;
  {
    int dev = 0;
    cudaGetDevice(&dev);
    const unsigned long long bit = 1ull << (dev & 63);
    if (!(opted & bit)) {
      cudaFuncSetAttribute(k2_pairdist_tma<STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kK2SmemBudget);
      opted |= bit;
    }
  }
  k2_pairdist_tma<STAGES><<<dim3(gx, gy), kK2Threads, smem, st>>>(rows, n, d, d / kTmaT, self_pairs, parts);
}

int launch_pairdist(const RowTable& rows, int n, int64_t d, double* parts, cudaStream_t st, int self_pairs) {
  const int ng = (n + kG - 1) / kG;
  const int ntasks = ng * (ng + 1) / 2;
  const int gy = (ntasks + kK2Warps - 1) / kK2Warps;
  // TMA path: every row 16-byte aligned and at least 3 ring stages of n x 512 floats fit
  bool aligned = true;
  for (int r = 0; r < n && aligned; ++r) aligned = (((uintptr_t)rows.p[r]) & 15) == 0;
  const size_t stage_bytes = (size_t)n * kTmaT * sizeof(float);
  const int stages_fit = (int)((kK2SmemBudget - 256) / stage_bytes);
  static const bool force_generic = getenv("BYZAGG_K2_GENERIC") != nullptr;
  if (aligned && stages_fit >= BZ_K2_TMA_MIN_STAGES && !force_generic) {   // with 2 stages the cp.async path measured faster (n > 36)
    const int64_t ntiles = (d + kTmaT - 1) / kTmaT;
    int gx = sm_count() / (gy > 0 ? gy : 1);
    if (gx < 1) gx = 1;
    if (gx > kMaxParts) gx = kMaxParts;
    if ((int64_t)gx > ntiles) gx = (int)(ntiles > 0 ? ntiles : 1);
    if (stages_fit >= 4)      launch_tma<4>(rows, n, d, gx, gy, self_pairs, parts, st);
    else if (stages_fit == 3) launch_tma<3>(rows, n, d, gx, gy, self_pairs, parts, st);
    else                      launch_tma<2>(rows, n, d, gx, gy, self_pairs, parts, st);
    return gx;
  }
  // Generic path: cp.async staging, any alignment.  Largest power-of-two tile whose two stages
  // fit the shared memory of one CTA per SM
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

int launch_pairdist_auto(const RowTable& rows, int u, int64_t d, double* parts, cudaStream_t st,
                         const int* to_unique, int n_orig, SelectTail* select) {
  unsigned char self_rows[kMaxN];
  int nself = 0;
  if (to_unique != nullptr && u < n_orig) {
    int mult[kMaxN] = {0};
    for (int i = 0; i < n_orig; ++i) ++mult[to_unique[i]];
    for (int k = 0; k < u; ++k)
      if (mult[k] > 1) self_rows[nself++] = (unsigned char)k;
  }
  const char* env = getenv("BYZAGG_K2_LEGACY");     // read per call: tools/k2_ab.py flips it between launches
  const bool legacy = env != nullptr && env[0] == '1';
  if (!legacy) {
    const int nparts = launch_pairdist_ring(rows, u, d, parts, st, self_rows, nself, select);
    if (nparts > 0) return nparts;
  }
  if (select != nullptr) select->fused = 0;
  return launch_pairdist(rows, u, d, parts, st, nself > 0 ? 1 : 0);
}

void launch_reduce_parts(const double* parts, int nparts, int len, int pair_n, double* block, cudaStream_t st) {
  k_reduce_parts<<<(len + 31) / 32, kReduceWarps * 32, 0, st>>>(parts, nparts, len, pair_n, block);
}

}  // namespace bz
