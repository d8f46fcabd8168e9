// k4_bulyan.cu — K4: Bulyan's reduce pass, fused per coordinate (bulyan.py:64-84).
//
// The reference materialises `selected[theta, d]` (theta = n-2f-2 Multi-Krum means, each a
// pass over up to m rows), then runs median / topk / take / mean over it.  Here one thread owns
// one coordinate: it reads the m_max = n-f-2 best-scored rows once (in score order, from the
// device-side `order` written by K5) into a shared-memory column, forms the theta running
// means in the reference's left-to-right order, sorts them in registers (NaN last), takes
// the lower median and averages the beta = theta-2f values closest to it.
// Scores are never updated between iterations (bulyan.py:74-76 is unreachable), so iteration i
// averages sorted positions i .. i+m_i-1 with m_i = min(m, m_max - i).
// Roofline: HBM, (m_max + 1)·4 B per coordinate.
#include "dist.cuh"
#include "launch.cuh"
#include "networks_gen.cuh"
#include "reduce.cuh"

namespace bz {

constexpr int kK4Threads = 128;

template <int THETA>
__global__ void __launch_bounds__(kK4Threads)
k4_bulyan(const __grid_constant__ RowTable rows, const int64_t d, const int n, const int f, const int m, const int one, const int mone,
          const int32_t* __restrict__ order, const int32_t* __restrict__ status, float* __restrict__ out) {
  extern __shared__ float sm[];   // [max(m_max, THETA)][kK4Threads]
  // reversed walk: the distance pass before this one went forward (see Geom::reverse)
  const int64_t i = ((int64_t)gridDim.x - 1 - blockIdx.x) * kK4Threads + threadIdx.x;
  if (i >= d) return;
  const int64_t e = i;
  pdl_wait();        // PDL: order / status / rows are valid from here
  if (status != nullptr && *status != 0) { out[e] = quiet_nan(); return; }
  float* col = sm + threadIdx.x;
  const int m_max = n - f - 2;
  // The m_max best-scored rows of this coordinate, in score order
  int k = 0;
  for (; k + 8 <= m_max; k += 8) {
    float t[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) t[u] = __ldcs(rows.p[order[k + u]] + e);
#pragma unroll
    for (int u = 0; u < 8; ++u) col[(k + u) * kK4Threads] = t[u];
  }
  for (; k < m_max; ++k) col[k * kK4Threads] = __ldcs(rows.p[order[k]] + e);
  // Stage 1: selected[i] = sum(gradients at sorted positions i..i+m_i-1).div_(m_i)  (bulyan.py:66-70)
  int key[THETA];
  int mi = m;
#pragma unroll
  for (int it = 0; it < THETA; ++it) {
    mi = min(mi, m_max - it);
    float acc = __fadd_rn(0.f, col[it * kK4Threads]);
    for (int q = 1; q < mi; ++q) acc = __fadd_rn(acc, col[(it + q) * kK4Threads]);
    key[it] = float_to_key(__fdiv_rn(acc, (float)mi));
  }
  // Stage 2 (bulyan.py:78-84): lower median over theta, beta closest to it, mean
  SortNet<THETA>::run(OpsKeyMix<MixFull<THETA>>{one, mone}, key);
  float last = key_to_float(key[THETA - 1]);
  const float med = (last != last) ? quiet_nan() : key_to_float(key[(THETA - 1) / 2]);
#pragma unroll
  for (int it = 0; it < THETA; ++it) col[it * kK4Threads] = key_to_float(key[it]);
  // In the sorted column the beta closest values are a window [l, l+beta).  Moving the window
  // from l to l+1 trades s[l] for s[l+beta]: a strict gain iff |s[l]-med| > |s[l+beta]-med|.  The
  // distance to med is valley shaped along the sorted column, so the best window starts right
  // after the LAST strict gain (a plateau of equal values longer than beta makes the gains
  // non-contiguous, hence "last", not "count").  NaN distances count as largest.
  const int beta = THETA - 2 * f;
  const int R = THETA - beta;
  int lstar = 0;
  for (int l = 0; l < R; ++l) {
    const int dlo = abs_key(__fsub_rn(col[l * kK4Threads], med));
    const int dhi = abs_key(__fsub_rn(col[(l + beta) * kK4Threads], med));
    lstar = (dlo > dhi) ? l + 1 : lstar;
  }
  float acc = 0.f;
  for (int q = 0; q < beta; ++q) acc = __fadd_rn(acc, col[(lstar + q) * kK4Threads]);
  const float r = __fdiv_rn(acc, (float)beta);
  out[e] = (med != med) ? quiet_nan() : r;
}

// ---- compile-time (n, f), default m = n-f-2: everything in registers ------------------------
// For the (n, f) of BASELINE.json's configs and of the reference's grids.  The m_max rows of a
// coordinate are m_max literal registers (all loads in flight at once), the theta running
// means are fully unrolled chains, the closest-beta window needs no shared memory because
// theta and beta are literals (only the window start is run-time: predicated adds).
template <int N, int F, int VEC>
__global__ void __launch_bounds__(kK4Threads)
k4_bulyan_static(const __grid_constant__ RowTable rows, const Geom g, const int32_t* __restrict__ order,
                 const int32_t* __restrict__ status, float* __restrict__ out) {
  constexpr int M_MAX = N - F - 2, THETA = N - 2 * F - 2, BETA = THETA - 2 * F, R = THETA - BETA;
  const int64_t blk = g.reverse ? (int64_t)gridDim.x - 1 - blockIdx.x : (int64_t)blockIdx.x;
  const int64_t v = blk * kK4Threads + threadIdx.x;
  if (v >= g.nv) return;
  const int64_t e0 = v * VEC - g.shift;
  const bool full = e0 >= 0 && e0 + VEC <= g.d;
  float res[VEC];
  pdl_wait();        // PDL: order / status / rows are valid from here
  if (status != nullptr && *status != 0) {
#pragma unroll
    for (int c = 0; c < VEC; ++c) res[c] = quiet_nan();
    store_vec<VEC>(out, e0, g.d, full, res);
    return;
  }
  // Stage 1 (bulyan.py:66-70, scores never updated): selected[i] = (0 + v[i] + ... + v[M_MAX-1]) / (M_MAX - i).
  // The THETA chains start at different rows, so no partial sum can be shared without changing the
  // rounding: sum(M_MAX - i) additions per coordinate (156 for n = 25, 625 for n = 51) and THETA
  // divisions make this kernel instruction bound.  With two coordinates per thread the additions go
  // through the pair helpers (`add2`: one IEEE addition per lane) and the divisions by the
  // compile-time row counts through `div_small2` (exact, reduce.cuh).
  float sel[VEC][THETA];
  if (VEC == 2) {
    u64 xp[M_MAX];
    if (full) {
#pragma unroll
      for (int k = 0; k < M_MAX; ++k) {
        float t[VEC];
        VecLoad<VEC>::load(rows.p[order[k]] + e0, t);
        xp[k] = pack2(t[0], t[VEC - 1]);
      }
    } else {
#pragma unroll
      for (int k = 0; k < M_MAX; ++k) {
        float t[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int64_t e = e0 + c;
          t[c] = (e >= 0 && e < g.d) ? __ldcs(rows.p[order[k]] + e) : 0.f;
        }
        xp[k] = pack2(t[0], t[1]);
      }
    }
    const u64 zero2 = pack2(0.f, 0.f);
#pragma unroll
    for (int it = 0; it < THETA; ++it) {
      u64 acc = add2(zero2, xp[it]);
#pragma unroll
      for (int q = it + 1; q < M_MAX; ++q) acc = add2(acc, xp[q]);
      unpack2(div_small2(acc, (float)(M_MAX - it)), sel[0][it], sel[VEC - 1][it]);
    }
  } else {
    float x[M_MAX];
#pragma unroll
    for (int k = 0; k < M_MAX; ++k) x[k] = (e0 >= 0 && e0 < g.d) ? __ldcs(rows.p[order[k]] + e0) : 0.f;
#pragma unroll
    for (int it = 0; it < THETA; ++it) {
      float acc = __fadd_rn(0.f, x[it]);
#pragma unroll
      for (int q = it + 1; q < M_MAX; ++q) acc = __fadd_rn(acc, x[q]);
      sel[0][it] = div_small(acc, (float)(M_MAX - it));
    }
  }
#pragma unroll
  for (int c = 0; c < VEC; ++c) {
    int key[THETA];
#pragma unroll
    for (int it = 0; it < THETA; ++it) key[it] = float_to_key(sel[c][it]);
    // Stage 2 (bulyan.py:78-84)
    SortNet<THETA>::run(OpsKeyMix<MixFull<THETA>>{g.one, g.mone}, key);
    float s[THETA];
#pragma unroll
    for (int it = 0; it < THETA; ++it) s[it] = key_to_float(key[it]);
    const float med = (s[THETA - 1] != s[THETA - 1]) ? quiet_nan() : s[(THETA - 1) / 2];
    int lstar = 0;
#pragma unroll
    for (int l = 0; l < R; ++l) {
      const int dlo = abs_key(__fsub_rn(s[l], med)), dhi = abs_key(__fsub_rn(s[l + BETA], med));
      lstar = (dlo > dhi) ? l + 1 : lstar;
    }
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < THETA; ++k) {
      const bool in = (unsigned)(k - lstar) < (unsigned)BETA;
      acc = in ? __fadd_rn(acc, s[k]) : acc;
    }
    const float r = div_small(acc, (float)BETA);
    res[c] = (med != med) ? quiet_nan() : r;
  }
  store_vec<VEC>(out, e0, g.d, full, res);
}

template <int N, int F>
static void launch_static(const RowTable& rows, const Geom& g, const int32_t* order, const int32_t* status, float* out, cudaStream_t st) {
  if (g.nv <= 0) return;
  const unsigned blocks = (unsigned)((g.nv + kK4Threads - 1) / kK4Threads);
  if (g.vec == 2) launch_after(k4_bulyan_static<N, F, 2>, blocks, kK4Threads, 0, st, rows, g, order, status, out);
  else            launch_after(k4_bulyan_static<N, F, 1>, blocks, kK4Threads, 0, st, rows, g, order, status, out);
}

bool launch_bulyan_reduce_static(const RowTable& rows, int n, int f, int m, const int32_t* order, const int32_t* status,
                                 const Geom& g, float* out, cudaStream_t st) {
  if (m != n - f - 2) return false;
#define Y(N, F) if (n == N && f == F) { launch_static<N, F>(rows, g, order, status, out, st); return true; }
  // the reference's grids (reproduce.py:109-209, reproduce-appendix.py: n = 11 / 25 / 51) and the
  // tightest configuration n = 4f + 3 of every f (bulyan.py:104-105)
  Y(11, 2) Y(25, 5) Y(51, 12)
  Y(7, 1) Y(15, 3) Y(19, 4) Y(23, 5) Y(27, 6) Y(31, 7) Y(35, 8) Y(39, 9) Y(43, 10) Y(47, 11)
#undef Y
  return false;
}

template <int THETA>
static void launch_theta(const RowTable& rows, int64_t d, int n, int f, int m, const int32_t* order,
                         const int32_t* status, float* out, cudaStream_t st) {
  const int64_t threads = d;
  if (threads <= 0) return;
  const int m_max = n - f - 2;
  const int rowsm = m_max > THETA ? m_max : THETA;
  const size_t smem = (size_t)rowsm * kK4Threads * sizeof(float);
  launch_after(k4_bulyan<THETA>, (unsigned)((threads + kK4Threads - 1) / kK4Threads), kK4Threads, smem, st,
               rows, d, n, f, m, 1, -1, order, status, out);
}

bool launch_bulyan_reduce(const RowTable& rows, int n, int f, int m, const int32_t* order, const int32_t* status,
                          int64_t d, float* out, cudaStream_t st) {
  const int theta = n - 2 * f - 2;
  switch (theta) {
#define X(T) case T: launch_theta<T>(rows, d, n, f, m, order, status, out, st); return true;
    X(1) X(2) X(3) X(4) X(5) X(6) X(7) X(8) X(9) X(10) X(11) X(12) X(13) X(14) X(15) X(16)
    X(17) X(18) X(19) X(20) X(21) X(22) X(23) X(24) X(25) X(26) X(27) X(28) X(29) X(30) X(31) X(32)
    X(33) X(34) X(35) X(36) X(37) X(38) X(39) X(40) X(41) X(42) X(43) X(44) X(45) X(46) X(47) X(48)
    X(49) X(50) X(51) X(52) X(53) X(54) X(55) X(56) X(57) X(58) X(59) X(60)
#undef X
    default: return false;
  }
}

}  // namespace bz
