// k2_rowdist.cu — K2': squared distance of every row to a centre vector, in one pass over
// the rows: the coordinate-wise median for Aksel (`(x - m).pow_(2).sum()`, aksel.py:41: the
// square is rounded to fp32 before it is summed) or the origin for CGE (`grad.norm()`,
// cge.py:36).  The reference makes n separate passes with a host sync each.
//
// One thread owns VEC adjacent coordinates and walks the rows in chunks of 8 (8 independent
// vector loads in flight), keeping one fp32 accumulator per row in registers (64 of them: the
// row index must be a literal).  Every 8 vectors (<= 32 terms per accumulator) the lane
// partials are transposed-reduced over the warp (lane r ends with row r and row r+32) into
// fp64; warps are combined through shared memory in fixed order; one fp64 block per CTA is
// summed by K5.  Deterministic; identical rows give identical sums.
// Roofline: HBM, n·4 B per coordinate (+4 B for the centre).
#include "dist.cuh"
#include "k5_device.cuh"
#include "launch.cuh"
#include "reduce.cuh"

namespace bz {

constexpr int kRdThreads = 256;
constexpr int kRdWarps = kRdThreads / 32;
constexpr int kRdChunk = 4;      // rows loaded together (4 x VEC values in flight per thread)
constexpr int kRdFlush = 8;      // vectors between two flushes

// One transition of `line_maximize` (tools/misc.py:468-513, start = 0, delta = 1, ratio = 0.8) after the
// evaluation of x = state->next_x scored y: the Python statements in the same order, in fp64 with
// explicit rounding (no contraction).  NaN never compares greater, as in Python.
__device__ void search_step(const SearchTail& s, const double y) {
  SearchState* st = s.state;
  const double x = st->next_x;
  s.trace[2 * s.k] = x;
  s.trace[2 * s.k + 1] = y;
  int32_t code = s.k == 0 ? 0 : *s.status;
  if (code == 0 && s.eval_status != nullptr) code = *s.eval_status;
  *s.status = code;
  double best_x, best_y, delta, prop_x = x;
  int phase;
  if (s.k == 0) {                       // best_x = start; best_y = scape(best_x)
    best_x = x; best_y = y; delta = 1.; phase = 1;
  } else {
    best_x = st->best_x; best_y = st->best_y; delta = st->delta; phase = st->phase;
    if (phase == 1) {                   // expansion
      if (y > best_y) { best_y = y; best_x = prop_x; delta = __dmul_rn(delta, 2.); }
      else            { delta = __dmul_rn(delta, 0.8); phase = 2; }
    } else {                            // contraction
      if (y > best_y) { best_y = y; best_x = prop_x; }
      delta = __dmul_rn(delta, 0.8);
    }
  }
  // the x the next evaluation (if any) takes
  if (phase == 1) {
    prop_x = __dadd_rn(best_x, delta);
  } else if (prop_x < best_x) {
    prop_x = __dadd_rn(prop_x, delta);
  } else {
    double t = __dsub_rn(prop_x, delta);
    while (t < 0.) t = __ddiv_rn(__dadd_rn(t, prop_x), 2.);
    prop_x = t;
  }
  st->best_x = best_x; st->best_y = best_y; st->delta = delta; st->prop_x = prop_x; st->phase = phase;
  st->next_x = prop_x;
  if (s.k == s.evals - 1) s.trace[2 * s.evals] = best_x;
}

// DOT: sum_k x_r[k] * c[k] instead of the squared distance (the dot products of the study step,
// attack.py:854-866: one vector against up to 64 others in one pass).
// SEARCH: the score of the attacks' line search (one row, `search` set): launched by PDL after the rule,
// the last CTA rounds the sum to fp32 and runs `search_step` instead of the selection.
template <bool CENTER, int VEC, bool DOT = false, bool SEARCH = false>
__global__ void __launch_bounds__(kRdThreads, 2)
k2_rowdist(const __grid_constant__ RowTable rows, const int n, const float* __restrict__ center, const Geom g,
           double* __restrict__ parts, int32_t* __restrict__ order, unsigned* __restrict__ ticket, const int sqrt_norm,
           const SearchTail search) {
  __shared__ double warp_tot[kRdWarps][kMaxN];
  if (SEARCH) pdl_wait();      // the rule's output is valid from here
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc[kMaxN];
#pragma unroll
  for (int r = 0; r < kMaxN; ++r) acc[r] = 0.f;
  double d0 = 0., d1 = 0.;      // rows `lane` and `lane + 32`
  const int64_t stride = (int64_t)gridDim.x * kRdThreads;
  // warp-uniform trip count: lanes past the end contribute zeros and still join the shuffles
  const int64_t first = (int64_t)blockIdx.x * kRdThreads + warp * 32;
  int pending = 0;
  for (int64_t vf = first; vf < g.nv; vf += stride) {
    // reversed walk (Geom::reverse): same warp-uniform trip count, mirrored base
    const int64_t vb = g.reverse ? ((g.nv - 1) / 32) * 32 - vf : vf;
    const int64_t v = vb + lane;
    const bool live = v < g.nv;
    const int64_t e0 = v * VEC - g.shift;
    const bool full = live && e0 >= 0 && e0 + VEC <= g.d;
    float c[VEC];
    if (CENTER) {
      if (full) VecLoad<VEC>::load(center + e0, c);
      else {
#pragma unroll
        for (int q = 0; q < VEC; ++q) { const int64_t e = e0 + q; c[q] = (live && e >= 0 && e < g.d) ? __ldcs(center + e) : 0.f; }
      }
    }
#pragma unroll
    for (int r0 = 0; r0 < kMaxN; r0 += kRdChunk) {
      if (r0 < n) {     // uniform; rows r >= n alias row 0 in the table, their sums are discarded
        float x[kRdChunk][VEC];
        if (full) {
#pragma unroll
          for (int u = 0; u < kRdChunk; ++u) VecLoad<VEC>::load(rows.p[r0 + u] + e0, x[u]);
        } else {
#pragma unroll
          for (int u = 0; u < kRdChunk; ++u)
#pragma unroll
            for (int q = 0; q < VEC; ++q) {
              const int64_t e = e0 + q;
              const bool ok = live && e >= 0 && e < g.d;
              // out-of-range lanes must add exactly 0: take the centre itself
              x[u][q] = ok ? __ldcs(rows.p[r0 + u] + e) : ((CENTER && !DOT) ? c[q] : 0.f);
            }
        }
#pragma unroll
        for (int u = 0; u < kRdChunk; ++u)
#pragma unroll
          for (int q = 0; q < VEC; ++q) {
            if (DOT) {
              acc[r0 + u] = fmaf(x[u][q], c[q], acc[r0 + u]);
            } else if (CENTER) {
              const float df = __fsub_rn(x[u][q], c[q]);
              acc[r0 + u] = __fadd_rn(acc[r0 + u], __fmul_rn(df, df));
            } else {
              acc[r0 + u] = fmaf(x[u][q], x[u][q], acc[r0 + u]);
            }
          }
      }
    }
    if (++pending == kRdFlush) {
      pending = 0;
      d0 += (double)transpose_reduce(*reinterpret_cast<float(*)[32]>(&acc[0]), lane);
      if (n > 32) d1 += (double)transpose_reduce(*reinterpret_cast<float(*)[32]>(&acc[32]), lane);
#pragma unroll
      for (int r = 0; r < kMaxN; ++r) acc[r] = 0.f;
    }
  }
  if (pending > 0) {
    d0 += (double)transpose_reduce(*reinterpret_cast<float(*)[32]>(&acc[0]), lane);
    if (n > 32) d1 += (double)transpose_reduce(*reinterpret_cast<float(*)[32]>(&acc[32]), lane);
  }
  warp_tot[warp][lane] = d0;
  warp_tot[warp][lane + 32] = d1;
  __syncthreads();
  if (threadIdx.x < n) {
    double s = 0.;
#pragma unroll
    for (int w = 0; w < kRdWarps; ++w) s += warp_tot[w][threadIdx.x];
    parts[(size_t)blockIdx.x * n + threadIdx.x] = s;
  }
  if (!SEARCH && order == nullptr) return;
  if (SEARCH) ticket = &search.state->ticket;
  // The selection step (aksel.py:49 / cge.py:38: stable order of the n keys) in the LAST CTA to
  // finish instead of a single-CTA launch: blocks summed in S interleaved classes with every load in
  // flight, class sums added in class order (fixed for a given grid), keys as in k5_rowdist_select.
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double* partial = &warp_tot[0][0];                // S * n <= 256 doubles
  double* key = partial + kRdThreads;               // n <= 64 doubles behind them (the table holds 512)
  const int S = kRdThreads / n;
  const int c = threadIdx.x % n, cls = threadIdx.x / n;
  if (cls < S) {
    double sum = 0.;
    int p = cls;
    for (; p + 7 * S < (int)gridDim.x; p += 8 * S) {
      double t[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) t[u] = __ldcg(parts + (size_t)(p + u * S) * n + c);
#pragma unroll
      for (int u = 0; u < 8; ++u) sum += t[u];
    }
    for (; p < (int)gridDim.x; p += S) sum += __ldcg(parts + (size_t)p * n + c);
    partial[cls * n + c] = sum;
  }
  __syncthreads();
  if (threadIdx.x < n) {
    double sum = 0.;
    for (int k = 0; k < S; ++k) sum += partial[k * n + threadIdx.x];
    double v;
    if (sqrt_norm) {
      v = (double)fp32_norm(sum);                    // cge.py:36-37: fp32 norm, non-finite -> +inf
      if (!finite_d(v)) v = CUDART_INF;
    } else {
      v = (double)(float)sum;                        // aksel.py:41 (and the search's `dot`): fp32 sum of squares
    }
    if (SEARCH) {
      search_step(search, v);
      *ticket = 0u;
    }
    key[threadIdx.x] = v;
  }
  if (SEARCH) return;
  __syncthreads();
  stable_order(key, n, order);
  if (threadIdx.x == 0) *ticket = 0u;
}


int launch_rowdist(const RowTable& rows, int n, const float* const* host_rows, const float* center, int64_t d,
                   double* parts, cudaStream_t st, int reverse, int32_t* order, unsigned* ticket, int sqrt_norm, int dot) {
  // The centre doubles as the alignment reference ("out") of the geometry
  Geom g = make_geom(host_rows, n, center ? (const void*)center : (const void*)host_rows[0], nullptr, d, 4);
  g.reverse = reverse;
  int64_t grid = (g.nv + kRdThreads - 1) / kRdThreads;
  const int64_t cap = (int64_t)sm_count() * 2;
  if (grid > cap) grid = cap;
  if (grid > kMaxParts) grid = kMaxParts;
  if (grid < 1) grid = 1;
  if (dot && center != nullptr) {
    if (g.vec == 4) k2_rowdist<true, 4, true><<<(unsigned)grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, nullptr, nullptr, 0, SearchTail{});
    else            k2_rowdist<true, 1, true><<<(unsigned)grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, nullptr, nullptr, 0, SearchTail{});
    return (int)grid;
  }
  if (order != nullptr) cudaMemsetAsync(ticket, 0, sizeof(unsigned), st);
  if (g.vec == 4) {
    if (center) k2_rowdist<true, 4><<<(unsigned)grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, SearchTail{});
    else        k2_rowdist<false, 4><<<(unsigned)grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, SearchTail{});
  } else {
    if (center) k2_rowdist<true, 1><<<(unsigned)grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, SearchTail{});
    else        k2_rowdist<false, 1><<<(unsigned)grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, SearchTail{});
  }
  return (int)grid;
}

int launch_rowdist_search(const float* out, const float* center, int64_t d, double* parts, const SearchTail& tail,
                          cudaStream_t st) {
  RowTable rows;
  for (int r = 0; r < kMaxN; ++r) rows.p[r] = out;
  const Geom g = make_geom(&out, 1, center, nullptr, d, 4);
  int64_t grid = (g.nv + kRdThreads - 1) / kRdThreads;
  const int64_t cap = (int64_t)sm_count() * 2;
  if (grid > cap) grid = cap;
  if (grid > kMaxParts) grid = kMaxParts;
  if (grid < 1) grid = 1;
  const cudaError_t err = g.vec == 4
      ? launch_after(k2_rowdist<true, 4, false, true>, (unsigned)grid, kRdThreads, 0, st, rows, 1, center, g, parts, nullptr, nullptr, 0, tail)
      : launch_after(k2_rowdist<true, 1, false, true>, (unsigned)grid, kRdThreads, 0, st, rows, 1, center, g, parts, nullptr, nullptr, 0, tail);
  return err == cudaSuccess ? (int)grid : -1;
}

}  // namespace bz
