// k5_device.cuh — device-side building blocks of the scoring / selection step (K5), shared by
// the stand-alone kernels of k5_score.cu and by the tail of the distance pass (k2_ring.cu), which
// runs them in its last CTA instead of paying a launch (krum.py:49-62, bulyan.py:56-73,
// brute.py:47-68 are host-side Python in the reference).
#pragma once

#include <math_constants.h>

#include "dist.cuh"

namespace bz {

__device__ __forceinline__ bool finite_d(double x) { return fabs(x) <= 1.7976931348623157e308; }

// Where the partial blocks live: one strided buffer (per-CTA blocks of K2 / K2', or blocks gathered
// by a collective), or one pointer per peer GPU — the blocks are then read IN PLACE from the
// peers' memory over NVLink (ld.global on peer-mapped addresses): the exchange step of the
// d-sharded path is fused into the scoring kernel, no all-gather, no staging copy.
struct StridedParts {
  const double* base;
  size_t stride;
  __device__ __forceinline__ const double* block(int p) const { return base + (size_t)p * stride; }
};
constexpr int kMaxPeers = BZ_MAX_PEERS;
struct PeerParts {
  const double* ptr[kMaxPeers];
  __device__ __forceinline__ const double* block(int p) const { return ptr[p]; }
};

// Block-wide, deterministic sum of `nparts` partial blocks of `len` doubles into smem `out`.
// The parts are split in `slices` interleaved classes (p mod slices); thread (slice, t) walks
// entries t, t + T, ... and adds its class in ascending p; the classes are then added in
// ascending order.  The order depends only on (nparts, slices): bitwise reproducible, and the
// same on every rank of the sharded path.  All loads of a thread are independent across
// entries, so a thread keeps several in flight (a naive per-entry loop over one part per SM
// is pure latency).
template <class Parts>
__device__ void block_sum_parts(const Parts& parts, int nparts, int len, int slices,
                                double* __restrict__ scratch, double* __restrict__ out) {
  const int T = blockDim.x / slices;            // threads per slice
  const int slice = threadIdx.x / T, t = threadIdx.x - slice * T;
  constexpr int E = 8;                          // entries per thread in flight together
  if (slice < slices) {
    for (int e0 = t; e0 < len; e0 += T * E) {
      double s[E];
#pragma unroll
      for (int q = 0; q < E; ++q) s[q] = 0.;
#pragma unroll 4
      for (int p = slice; p < nparts; p += slices) {
        const double* __restrict__ row = parts.block(p);
#pragma unroll
        for (int q = 0; q < E; ++q) {
          const int e = e0 + q * T;
          if (e < len) s[q] += __ldcg(row + e);
        }
      }
#pragma unroll
      for (int q = 0; q < E; ++q) {
        const int e = e0 + q * T;
        if (e < len) scratch[slice * len + e] = s[q];
      }
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < len; e += blockDim.x) {
    double s = 0.;
    for (int k = 0; k < slices; ++k) s += scratch[k * len + e];
    out[e] = s;
  }
  __syncthreads();
}

// Aliased rows (the f Byzantine gradients are ONE tensor repeated, attacks/identical.py:86) are
// detected on the host by pointer equality; the distance pass then runs on the u unique rows only
// (with the self pairs i == i) and this map expands its u x u table to the n x n one.
struct RowMap {
  unsigned char to_unique[kMaxN];
  int u;          // number of unique rows (u == n: identity, no expansion)
};

// dist[i][j] = double(fl32(sqrt(sum_k (x_i - x_j)^2))) from the summed u x u table `sq`;
// diagonal = `diag`.  `sq` and `dist` must not overlap when map.u < n.
__device__ inline void finish_distances_mapped(const double* sq, const RowMap& map, int n, bool map_nonfinite, double diag, double* dist) {
  const int u = map.u;
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e / n, j = e - i * n;
    if (i < j) {
      // aliases (a == b) read the diagonal: 0 for a finite row, NaN for a row holding NaN / inf,
      // exactly what the reference's x.sub(x).norm() gives
      const int a = map.to_unique[i], b = map.to_unique[j];
      double v = (double)(float)sqrt(sq[min(a, b) * u + max(a, b)]);
      if (map_nonfinite && !finite_d(v)) v = CUDART_INF;
      dist[i * n + j] = v;
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e / n, j = e - i * n;
    if (i > j) dist[e] = dist[j * n + i];
    else if (i == j) dist[e] = diag;
  }
  __syncthreads();
}

// dist[i][j] = double(fl32(sqrt(sum_k (x_i - x_j)^2))) from the summed table `sq` (in place
// allowed); diagonal = `diag`.
__device__ inline void finish_distances(const double* sq, int n, bool map_nonfinite, double diag, double* dist) {
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e / n, j = e - i * n;
    if (i < j) {
      double v = (double)(float)sqrt(sq[e]);
      if (map_nonfinite && !finite_d(v)) v = CUDART_INF;
      dist[i * n + j] = v;
    }
  }
  __syncthreads();
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e / n, j = e - i * n;
    if (i > j) dist[e] = dist[j * n + i];
    else if (i == j) dist[e] = diag;
  }
  __syncthreads();
}

// CPython >= 3.12 `sum()` over floats (Objects/bltinmodule.c: Neumaier's compensated sum;
// the compensation is dropped when it is not finite).
__device__ inline double py_sum(const double* v, int count) {
  if (count <= 0) return 0.;
  double f = v[0], c = 0.;
  for (int k = 1; k < count; ++k) {
    const double x = v[k];
    const double t = f + x;
    if (fabs(f) >= fabs(x)) c += (f - t) + x;
    else                    c += (x - t) + f;
    f = t;
  }
  if (c != 0. && finite_d(c)) f += c;
  return f;
}

// Row-wise ascending sort by ranking: sorted[i][rank] = dist[i][j] (ties by column index).
__device__ inline void sort_rows(const double* dist, double* sorted, int n) {
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e / n, j = e - i * n;
    const double v = dist[e];
    int rank = 0;
    for (int k = 0; k < n; ++k) {
      const double w = dist[i * n + k];
      rank += (w < v || (w == v && k < j)) ? 1 : 0;
    }
    sorted[i * n + rank] = v;
  }
  __syncthreads();
}

// Stable ascending argsort of key[0..n): order[rank] = index.  NaN keys sort last.
__device__ inline void stable_order(const double* key, int n, int32_t* __restrict__ order) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = key[i];
    const bool vn = v != v;
    int rank = 0;
    for (int j = 0; j < n; ++j) {
      const double w = key[j];
      const bool wn = w != w;
      const bool less = vn ? (!wn) : (!wn && w < v);
      const bool same = vn ? wn : (w == v);
      rank += (less || (same && j < i)) ? 1 : 0;
    }
    order[rank] = i;
  }
}

// krum.py:52-62 (count = n-f-1, diagonal excluded) and bulyan.py:56-62 (count = m over the
// row INCLUDING its +inf diagonal).  Putting +inf on the diagonal serves both: the extra +inf
// can only be reached after every finite distance, where the sum is +inf either way.
// Block-wide, any blockDim.x that `slices` divides; `sm`: (2 n^2 + n + slices n^2) doubles of shared memory.
// Scoring from an already summed table of squared distances, left by the caller in shared memory:
// at `sm` (n x n) when map.u == n, else the u x u table at `sm + n*n`.  `sm`: (2 n^2 + n) doubles.
__device__ inline void score_from_table(const RowMap& map, int n, int count, int32_t* __restrict__ order, int32_t* __restrict__ status,
                                        int f, int m, int bulyan, double* sm) {
  double* dist = sm;
  double* sorted = sm + n * n;
  double* score = sm + 2 * n * n;
  if (map.u == n) finish_distances(dist, n, true, CUDART_INF, dist);
  else            finish_distances_mapped(sorted, map, n, true, CUDART_INF, dist);
  sort_rows(dist, sorted, n);
  for (int i = threadIdx.x; i < n; i += blockDim.x) score[i] = py_sum(sorted + i * n, count);
  __syncthreads();
  stable_order(score, n, order);
  if (threadIdx.x == 0 && status != nullptr) {
    int st = BZ_STATUS_OK;
    if (bulyan) {
      // bulyan.py:65-73: from the second iteration on, pruned `(inf, None)` entries precede every
      // +inf score (stable sort), so fewer than m_i finite scores left means gradients[None]
      int finite = 0;
      for (int i = 0; i < n; ++i) finite += finite_d(score[i]) ? 1 : 0;
      const int m_max = n - f - 2, theta = n - 2 * f - 2;
      int mi = m;
      for (int i = 0; i < theta; ++i) {
        mi = min(mi, m_max - i);
        if (i >= 1 && finite - i < mi) st = BZ_STATUS_DEGENERATE;
      }
    }
    *status = st;
  }
}

template <class Parts>
__device__ void score_select_body(const Parts& parts, const RowMap& map, int nparts, int n, int count,
                                  int32_t* __restrict__ order, int32_t* __restrict__ status, int f, int m, int bulyan, int slices,
                                  double* sm) {
  double* scratch = sm + 2 * n * n + n;
  if (map.u == n) block_sum_parts(parts, nparts, n * n, slices, scratch, sm);
  else            block_sum_parts(parts, nparts, map.u * map.u, slices, scratch, sm + n * n);   // u x u table, parked in `sorted`
  score_from_table(map, n, count, order, status, f, m, bulyan, sm);
}


// ---- brute: exhaustive minimum-diameter subset (brute.py:47-68) -----------------------------
// Thread t scans a contiguous range of lexicographic ranks; the first strict minimum wins,
// so the block-wide winner is the smallest (diameter, thread) pair.
__device__ __forceinline__ unsigned long long sat_add(unsigned long long a, unsigned long long b) {
  const unsigned long long s = a + b;
  return s < a ? ~0ull : s;
}

// Exhaustive search from an already summed table: at `sm` (n x n) when map.u == n, else the u x u
// table at `sm + n*n` (where the Pascal triangle goes next).  `sm`: n^2 + (n+1)^2 + 64 doubles.
__device__ inline void brute_from_table(const RowMap& map, int n, int f, unsigned long long total,
                                        int32_t* __restrict__ sel, int32_t* __restrict__ status, double* sm) {
  double* dist = sm;                                                  // n*n
  unsigned long long* binom = reinterpret_cast<unsigned long long*>(sm + n * n);   // (n+1)*(n+1)
  // per-warp winners (32 + 32 words)
  double* best_diam = sm + n * n + (n + 1) * (n + 1);
  unsigned long long* best_rank = reinterpret_cast<unsigned long long*>(best_diam + 32);
  const int k = n - f;
  const int W = n + 1;
  if (map.u == n) finish_distances(dist, n, false, 0., dist);
  else            finish_distances_mapped(reinterpret_cast<double*>(binom), map, n, false, 0., dist);
  // Pascal triangle, row by row
  for (int a = 0; a <= n; ++a) {
    for (int b = threadIdx.x; b <= n; b += blockDim.x) {
      unsigned long long v;
      if (b == 0) v = 1;
      else if (b > a) v = 0;
      else v = sat_add(binom[(a - 1) * W + b - 1], binom[(a - 1) * W + b]);
      binom[a * W + b] = v;
    }
    __syncthreads();
  }
  // This thread's rank range
  const unsigned long long per = (total + blockDim.x - 1) / blockDim.x;
  const unsigned long long lo = per * threadIdx.x;
  const unsigned long long hi = (lo + per < total) ? lo + per : total;
  double my_diam = CUDART_INF;
  unsigned long long my_rank = ~0ull;
  bool found = false;
  if (lo < hi) {
    int comb[kMaxN];
    {  // unrank `lo`
      unsigned long long r = lo;
      int x = 0;
      for (int pos = 0; pos < k; ++pos) {
        while (true) {
          const unsigned long long c = binom[(n - 1 - x) * W + (k - 1 - pos)];
          if (c > r) break;
          r -= c;
          ++x;
        }
        comb[pos] = x++;
      }
    }
    for (unsigned long long rank = lo; rank < hi; ++rank) {
      double diam = 0.;
      bool ok = true;
      for (int a = 0; a < k - 1 && ok; ++a) {
        const double* row = dist + comb[a] * n;
        for (int b = a + 1; b < k; ++b) {
          const double v = row[comb[b]];
          if (!finite_d(v)) { ok = false; break; }
          if (v > diam) diam = v;
        }
      }
      if (ok && (!found || diam < my_diam)) { found = true; my_diam = diam; my_rank = rank; }
      // next combination in lexicographic order
      int pos = k - 1;
      while (pos >= 0 && comb[pos] == n - k + pos) --pos;
      if (pos < 0) break;
      ++comb[pos];
      for (int q = pos + 1; q < k; ++q) comb[q] = comb[q - 1] + 1;
    }
  }
  // Block-wide minimum of (found ? diam : +inf-with-no-rank, rank)
  double dm = found ? my_diam : CUDART_INF;
  unsigned long long rk = found ? my_rank : ~0ull;
  for (int h = 16; h >= 1; h >>= 1) {
    const double od = __shfl_xor_sync(0xffffffffu, dm, h);
    const unsigned long long orank = __shfl_xor_sync(0xffffffffu, rk, h);
    if (orank != ~0ull && (rk == ~0ull || od < dm || (od == dm && orank < rk))) { dm = od; rk = orank; }
  }
  if ((threadIdx.x & 31) == 0) { best_diam[threadIdx.x >> 5] = dm; best_rank[threadIdx.x >> 5] = rk; }
  __syncthreads();
  if (threadIdx.x == 0) {
    dm = CUDART_INF; rk = ~0ull;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
      const double od = best_diam[w];
      const unsigned long long orank = best_rank[w];
      if (orank != ~0ull && (rk == ~0ull || od < dm || (od == dm && orank < rk))) { dm = od; rk = orank; }
    }
    if (rk == ~0ull) {
      if (status) *status = BZ_STATUS_NO_FINITE_SET;
      for (int pos = 0; pos < k; ++pos) sel[pos] = pos;
    } else {
      if (status) *status = BZ_STATUS_OK;
      unsigned long long r = rk;
      int x = 0;
      for (int pos = 0; pos < k; ++pos) {
        while (true) {
          const unsigned long long c = binom[(n - 1 - x) * W + (k - 1 - pos)];
          if (c > r) break;
          r -= c;
          ++x;
        }
        sel[pos] = x++;
      }
    }
  }
}


// Block-wide, any blockDim.x <= 1024 that `slices` divides; `sm`: n^2 + (n+1)^2 + 64 + slices n^2 doubles.
template <class Parts>
__device__ void brute_select_body(const Parts& parts, const RowMap& map, int nparts, int n, int f,
                                  unsigned long long total, int32_t* __restrict__ sel, int32_t* __restrict__ status, int slices,
                                  double* sm) {
  double* scratch = sm + n * n + (n + 1) * (n + 1) + 64;
  if (map.u == n) block_sum_parts(parts, nparts, n * n, slices, scratch, sm);
  else            block_sum_parts(parts, nparts, map.u * map.u, slices, scratch, sm + n * n);
  brute_from_table(map, n, f, total, sel, status, sm);
}

// Interleaved part classes for block_sum_parts: as many as fit `budget` bytes of scratch, at most 8,
// dividing `threads`.
inline int pick_slices(int n, int nparts, int threads, size_t budget = 48 * 1024) {
  int slices = (int)(budget / ((size_t)n * n * sizeof(double)));
  if (slices > 8) slices = 8;
  if (slices > nparts) slices = nparts;
  if (slices < 1) slices = 1;
  while (threads % slices) --slices;
  return slices;
}

inline RowMap identity_map(int n) {
  RowMap map;
  for (int i = 0; i < kMaxN; ++i) map.to_unique[i] = (unsigned char)(i < n ? i : 0);
  map.u = n;
  return map;
}

inline RowMap make_map(const int* to_unique, int n, int u) {
  if (to_unique == nullptr || u >= n) return identity_map(n);
  RowMap map;
  for (int i = 0; i < kMaxN; ++i) map.to_unique[i] = (unsigned char)(i < n ? to_unique[i] : 0);
  map.u = u;
  return map;
}

}  // namespace bz
