// k1_select.cuh — K1: coordinate-wise order statistics down the d axis.
//
// One thread owns VEC adjacent coordinates: it loads the n values of each coordinate with
// one coalesced vector load per row (a warp reads 128·VEC contiguous bytes of every row),
// keeps them in registers and runs a literal-index sorting network on them — no stack of the
// n rows (the `torch.stack` of median.py:39 / trmean.py:79 is gone), no shared memory on the
// default path, no block-level barrier.  Tiles of 128·VEC coordinates map one to one onto
// CTAs; ~4 CTAs are resident per SM, so while some warps sort others have their loads in
// flight (two alternative walks — persistent, and persistent with cp.async prefetch — are kept
// as build variants; they measured slower, see BZ_K1_VARIANT below).
//
//   k1_median<N, VEC>            median.py:31-39        FMNMX.NAN network, pruned to one rank
//   k1_sorted<N, VEC, F, MODE>   trmean.py:24-50,69-109 sort, then trmean / phocas / meamed
//
// F / MODE = -1 mean "run-time value": one generic kernel per (N, VEC) serves every f and the
// three epilogues after a full sort.  For n = 11, 25, 51 (BASELINE.json's configs and the
// reference's experiment grids) the trimmed mean is also instantiated for every f with F and
// MODE fixed: the compiler's dead-code elimination then prunes the network to the comparators
// ranks f..n-f-1 depend on.
//
// Roofline: HBM (n·4 B read + 4 B written per coordinate); secondary bound: the ALU pipe
// (FMNMX issues at 64 lanes/clk/SM): see DESIGN.md for the per-N operation counts.
#pragma once

#include "common.cuh"
#include "launch.cuh"
#include "networks_gen.cuh"

namespace bz {

// Threads per CTA (A/B builds: `make VARIANT=t64 EXTRA=-DBZ_K1_THREADS=64`; shorter CTAs shrink the
// ragged last wave at d ~ 1M, at the price of more CTA launches).
#ifndef BZ_K1_THREADS
#define BZ_K1_THREADS 128
#endif
constexpr int kK1Threads = BZ_K1_THREADS;

// How a thread walks the coordinates (A/B builds: `make VARIANT=v0 EXTRA=-DBZ_K1_VARIANT=0`):
//   2 (default)  one logical vector per thread, direct register loads, grid = all tiles.  The
//                hardware CTA scheduler balances the tail.
//   1            persistent grid-stride loop, direct loads.
//   0            persistent loop with cp.async staging of the next tile in a per-thread
//                shared-memory column while the current one is sorted.
#ifndef BZ_K1_VARIANT
#define BZ_K1_VARIANT 2
#endif

// Shared-memory staging of one tile: column of thread t = N slots of VEC floats,
// slot r at stage[(r * kK1Threads + t) * VEC] (a warp's slots of one row are contiguous).
template <int N, int VEC>
struct Stage {
  static constexpr int kFloats = (BZ_K1_VARIANT == 0) ? N * kK1Threads * VEC : 0;   // experiment variants stage nothing
  static constexpr int kColumnFloats = N * kK1Threads * VEC;
  static __device__ __forceinline__ void issue(const RowTable& rows, int64_t e0, float* col) {
#pragma unroll
    for (int r = 0; r < N; ++r) cp_async_vec<VEC>(col + r * kK1Threads * VEC, rows.p[r] + e0);
    cp_async_commit();
  }
  static __device__ __forceinline__ void fetch(const float* col, float (&x)[VEC][N]) {
    cp_async_wait<0>();
#pragma unroll
    for (int r = 0; r < N; ++r) {
      float t[VEC];
      lds_vec<VEC>(col + r * kK1Threads * VEC, t);
#pragma unroll
      for (int c = 0; c < VEC; ++c) x[c][r] = t[c];
    }
  }
};

// Walk this thread's tiles: `body(x, e0, full)` consumes the N x VEC values of one logical
// vector (sorting them in place is fine) and stores its result.
template <int N, int VEC, class Body>
__device__ __forceinline__ void k1_walk(const RowTable& rows, const Geom& g, float* stage, Body body) {
  const int64_t stride = (int64_t)gridDim.x * kK1Threads;
  int64_t v = (int64_t)blockIdx.x * kK1Threads + threadIdx.x;
  // Programmatic dependent launch on both sides: the NEXT kernel of the stream may be scheduled while this
  // grid drains, and this one was scheduled while its predecessor drained — the wait below returns once
  // that predecessor has completed and its writes (possibly these very rows) are visible.  Back-to-back
  // calls lose the launch gap (~1.5 us of a 24 us pass at d = 1.3M).
  pdl_trigger();
  if (v >= g.nv) return;
  pdl_wait();
#if BZ_K1_VARIANT == 0
  float* col = stage + threadIdx.x * VEC;
  int64_t e0 = v * VEC - g.shift;
  bool full = e0 >= 0 && e0 + VEC <= g.d;
  if (full) Stage<N, VEC>::issue(rows, e0, col);
  while (true) {
    float x[VEC][N];
    if (full) Stage<N, VEC>::fetch(col, x);
    else      load_rows<N, VEC>(rows, e0, g.d, false, x);      // first / last partial vector only
    // Prefetch the next tile into the (now free) column before the ALU phase
    const int64_t vn = v + stride;
    const bool more = vn < g.nv;
    const int64_t en = vn * VEC - g.shift;
    const bool fulln = more && en >= 0 && en + VEC <= g.d;
    if (fulln) Stage<N, VEC>::issue(rows, en, col);
    body(x, e0, full);
    if (!more) break;
    v = vn; e0 = en; full = fulln;
  }
#else
  // Experiment variants (A/B builds, `make VARIANT=...`): direct register loads, no prefetch;
  // 1 = persistent grid-stride loop, 2 = one tile per thread (the launcher sizes the grid).
  (void)stage;
  for (; v < g.nv; v += stride) {
    const int64_t e0 = v * VEC - g.shift;
    const bool full = e0 >= 0 && e0 + VEC <= g.d;
    float x[VEC][N];
    load_rows<N, VEC>(rows, e0, g.d, full, x);
    body(x, e0, full);
  }
#endif
}

// ---- median ---------------------------------------------------------------------------

// Register cap: 512 resident threads per SM (<= 128 registers) whenever the N x VEC values leave room.
#ifndef BZ_K1_CAP
#define BZ_K1_CAP 104
#endif
__host__ __device__ constexpr int k1_min_blocks(int n, int vec) { return (n * vec <= BZ_K1_CAP) ? 512 / kK1Threads : 1; }

template <int N, int VEC>
__global__ void __launch_bounds__(kK1Threads, k1_min_blocks(N, VEC))
k1_median(const __grid_constant__ RowTable rows, const Geom g, float* __restrict__ out) {
  extern __shared__ __align__(16) float smem[];
  k1_walk<N, VEC>(rows, g, smem, [&](float (&x)[VEC][N], int64_t e0, bool full) {
    float chk = 0.f;
#pragma unroll
    for (int r = 0; r < N; ++r)
#pragma unroll
      for (int c = 0; c < VEC; ++c) chk = fmaf(x[c][r], 0.f, chk);   // NaN iff a NaN / inf is present
    float res[VEC];
    if (chk == chk) {
      // all finite: comparators split over the ALU and FMA pipes
      const OpsMix<MixMedian<N>> ops{g.one, g.mone};
#pragma unroll
      for (int c = 0; c < VEC; ++c) {
        SortNet<N>::run(ops, x[c]);
        res[c] = x[c][(N - 1) / 2];   // lower median; every other output is dead code
      }
    } else {
#pragma unroll
      for (int c = 0; c < VEC; ++c) {
        SortNet<N>::run(OpsNaNProp{}, x[c]);
        res[c] = x[c][(N - 1) / 2];
      }
    }
    store_vec<VEC>(out, e0, g.d, full, res);
  });
}

// ---- trimmed mean of a sorted column (trmean.py:33) -----------------------------------------
// `values[f:-f].mean(dim=0)`: ATen sums rows in a cascade of 16-row blocks (sequential when
// R = n - 2f <= 16), then divides by R with one IEEE division.
template <int N>
__device__ __forceinline__ float trmean_sorted(const float (&s)[N], const int f) {
  const int R = N - 2 * f;
  const int hi = N - f;
  float acc0 = 0.f;
  if (N - 2 <= 16 || R <= 16) {
#pragma unroll
    for (int k = 0; k < N; ++k)
      if (k >= f && k < hi) acc0 = __fadd_rn(acc0, s[k]);
    return __fdiv_rn(acc0, (float)R);
  }
  float acc1 = 0.f;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    if (k >= f && k < hi) {
      acc0 = __fadd_rn(acc0, s[k]);
      if (((k - f) & 15) == 15) { acc1 = __fadd_rn(acc1, acc0); acc0 = 0.f; }
    }
  }
  return __fdiv_rn(__fadd_rn(acc0, acc1), (float)R);
}

// ---- mean of the m values closest to c (trmean.py:35-50) -------------------------------------
// In a sorted column the m closest values form a window [l, l+m).  It always holds the core
// [R, m) (R = N - m removals) when m >= R, and of each pair (s[l], s[l+m]), l < R, the closer
// one.  NaN distances count as largest (`topk(largest=False)`); a NaN centre gives NaN.
// The partner index l+m is run-time uniform, so the sorted column is staged in shared
// memory (`col`, stride `stride` floats between consecutive ranks).
template <int N>
__device__ __forceinline__ float closest_pairs(const float (&s)[N], int m, float c, float* col, int stride) {
  const int R = N - m;            // removals; requires m >= R (phocas/meamed: m = n-f > f)
#pragma unroll
  for (int k = 0; k < N; ++k) col[k * stride] = s[k];
  // (own column only: no barrier needed)
  float acc = 0.f;
  for (int l = 0; l < R; ++l) {
    const float lo = col[l * stride], hi = col[(l + m) * stride];
    const int dlo = abs_key(__fsub_rn(lo, c)), dhi = abs_key(__fsub_rn(hi, c));
    acc = __fadd_rn(acc, (dlo > dhi) ? hi : lo);
  }
  for (int k = R; k < m; ++k) acc = __fadd_rn(acc, col[k * stride]);
  const float r = __fdiv_rn(acc, (float)m);
  return (c != c) ? quiet_nan() : r;
}

// Compile-time f: the partner index l + m is a literal, no staging needed.
template <int N, int F>
__device__ __forceinline__ float closest_pairs_static(const float (&s)[N], float c) {
  constexpr int M = N - F;
  float acc = 0.f;
#pragma unroll
  for (int l = 0; l < F; ++l) {
    const int dlo = abs_key(__fsub_rn(s[l], c)), dhi = abs_key(__fsub_rn(s[l + M], c));
    acc = __fadd_rn(acc, (dlo > dhi) ? s[l + M] : s[l]);
  }
#pragma unroll
  for (int k = F; k < M; ++k) acc = __fadd_rn(acc, s[k]);
  const float r = __fdiv_rn(acc, (float)M);
  return (c != c) ? quiet_nan() : r;
}

// Mask of the mixed comparators: pruned for a compile-time trimmed mean, full sort otherwise.
template <int N, int F, int MODE> struct MixFor { typedef MixFull<N> mask; typedef OpsMix<mask> type; };
template <int N, int F> struct MixFor<N, F, kModeTrmean> { typedef MixTrim<N, F> mask; typedef OpsMix<mask> type; };

template <int N, int VEC, int F, int MODE>
__global__ void __launch_bounds__(kK1Threads, k1_min_blocks(N, VEC))
k1_sorted(const __grid_constant__ RowTable rows, const Geom g, const int mode_rt, const int f_rt,
          float* __restrict__ out) {
  extern __shared__ __align__(16) float smem[];   // [stage][+ sorted columns for the closest modes]
  const int mode = (MODE >= 0) ? MODE : mode_rt;
  const int f = (F >= 0) ? F : f_rt;
  float* sorted_cols = smem + Stage<N, VEC>::kFloats;
  k1_walk<N, VEC>(rows, g, smem, [&](float (&x)[VEC][N], int64_t e0, bool full) {
    float chk = 0.f;
#pragma unroll
    for (int r = 0; r < N; ++r)
#pragma unroll
      for (int c = 0; c < VEC; ++c)
        chk = fmaf(x[c][r], 0.f, chk);   // NaN iff some value is NaN or +-inf (FMA pipe, off the ALU pipe)
    float res[VEC];
    if (chk == chk) {
      // Fast path: all finite, FMNMX / IMAD network (for a compile-time trimmed mean the mask is
      // the one balanced for the ranks it reads)
      const typename MixFor<N, F, MODE>::type ops{g.one, g.mone};
#pragma unroll
      for (int c = 0; c < VEC; ++c) {
        SortNet<N>::run(ops, x[c]);
        if (MODE == kModeTrmean) res[c] = trmean_sorted<N>(x[c], f);
      }
    } else {
      // Non-finite values present: sort integer keys so that NaN sorts last and +-inf keep their place
#pragma unroll
      for (int c = 0; c < VEC; ++c) {
        int k[N];
#pragma unroll
        for (int r = 0; r < N; ++r) k[r] = float_to_key(x[c][r]);
        SortNet<N>::run(OpsKeyMix<typename MixFor<N, F, MODE>::mask>{g.one, g.mone}, k);
#pragma unroll
        for (int r = 0; r < N; ++r) x[c][r] = key_to_float(k[r]);
        if (MODE == kModeTrmean) res[c] = trmean_sorted<N>(x[c], f);
      }
    }
    if (MODE != kModeTrmean) {
#pragma unroll
      for (int c = 0; c < VEC; ++c) {
        if (mode == kModeTrmean) {
          res[c] = trmean_sorted<N>(x[c], f);
        } else {
          float center;
          if (mode == kModePhocas) {
            center = trmean_sorted<N>(x[c], f);
          } else {
            // lower median; NaN sorts last, so a NaN anywhere shows in the last rank (median.py:39)
            center = (x[c][N - 1] != x[c][N - 1]) ? quiet_nan() : x[c][(N - 1) / 2];
          }
          if (F >= 0) res[c] = closest_pairs_static<N, (F >= 0 ? F : 0)>(x[c], center);
          else        res[c] = closest_pairs<N>(x[c], N - f, center, sorted_cols + c * kK1Threads + threadIdx.x, VEC * kK1Threads);
        }
      }
    }
    store_vec<VEC>(out, e0, g.d, full, res);
  });
}

}  // namespace bz
