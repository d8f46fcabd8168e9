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
#include "peers.cuh"
#include "reduce.cuh"
#include "search.cuh"

namespace bz {

constexpr int kRdThreads = 256;
constexpr int kRdWarps = kRdThreads / 32;
constexpr int kRdChunk = 4;      // rows loaded together (4 x VEC values in flight per thread)
constexpr int kRdFlush = 8;      // vectors between two flushes

// DOT: sum_k x_r[k] * c[k] instead of the squared distance (the dot products of the study step,
// attack.py:854-866: one vector against up to 64 others in one pass).
// SEARCH: the score of the attacks' line search (one row, `search` set): launched by PDL after the rule,
// the last CTA rounds the sum to fp32 and runs `search_step` (search.cuh) instead of the selection, or,
// with `search.partial` set (one rank of the d-sharded search), writes the fp64 sum there unrounded.
// PEERS (kernel k2_rowdist_peers): the last CTA exchanges its sum over peer memory first (`peers`,
// PeerTail): the selection, or the transition, then runs on the R ranks' sums added in rank order,
// bitwise the same on every rank.
// KEEP (kernel k2_anticge_norms, with PEERS): the last CTA also writes those R-summed sums to parts[0, n),
// once it has read every block there, for the attack against CGE (k10_anticge.cu) to take the key of σ_maxpos
// from after this rank's slot may have been rewritten by a peer.
template <bool CENTER, int VEC, bool DOT, bool SEARCH, bool PEERS, bool KEEP = false>
__device__ __forceinline__ void
rowdist_body(const RowTable& rows, const int n, const float* __restrict__ center, const Geom g,
             double* __restrict__ parts, int32_t* __restrict__ order, unsigned* __restrict__ ticket, const int sqrt_norm,
             const SearchTail search, const PeerTail& peers) {
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
  __shared__ int peer_timeout;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double* partial = &warp_tot[0][0];                // S * n <= 256 doubles (PEERS: kReduceWarps * n <= 512)
  double* key = partial + kRdThreads;               // n <= 64 doubles behind them (the table holds 512)
  double sum = 0.;                                  // thread c < n: the sum of entry c over the blocks
  if (PEERS && !SEARCH) {
    // the block bz_rowdist_partial gives (k_reduce_parts's order), so that every rank publishes what the
    // collective path all-gathers
    for (int idx = threadIdx.x; idx < kReduceWarps * n; idx += kRdThreads) {
      const int w = idx / n, c = idx - w * n;
      double s = 0.;
      for (int p = w; p < (int)gridDim.x; p += kReduceWarps) s += __ldcg(parts + (size_t)p * n + c);
      partial[idx] = s;
    }
    __syncthreads();
    if (threadIdx.x < n)
      for (int w = 0; w < kReduceWarps; ++w) sum += partial[w * n + threadIdx.x];
  } else {
    const int S = kRdThreads / n;
    const int c = threadIdx.x % n, cls = threadIdx.x / n;
    if (cls < S) {
      double s = 0.;
      int p = cls;
      for (; p + 7 * S < (int)gridDim.x; p += 8 * S) {
        double t[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) t[u] = __ldcg(parts + (size_t)(p + u * S) * n + c);
#pragma unroll
        for (int u = 0; u < 8; ++u) s += t[u];
      }
      for (; p < (int)gridDim.x; p += S) s += __ldcg(parts + (size_t)p * n + c);
      partial[cls * n + c] = s;
    }
    __syncthreads();
    if (threadIdx.x < n)
      for (int k = 0; k < S; ++k) sum += partial[k * n + threadIdx.x];
  }
  if (PEERS) {
    // the epoch and the slot: by value, or (`next`) from this rank's own flags, read by every thread that
    // needs them before the barrier below (SEARCH: after this kernel's pdl_wait); then publish, flag, wait
    // (peers.cuh), and ((p0 + p1) + p2) + ... over the R ranks
    unsigned epoch = peers.epoch;
    int slot = 0;
    if (peers.next && ((int)threadIdx.x < n || (int)threadIdx.x < peers.nranks)) {
      epoch = next_epoch(peers.flag[0][peers.rank] + peers.rank, peers.flag[1][peers.rank] + peers.rank);
      slot = (int)(epoch & 1u);
    }
    double* const* blocks = peers.block[slot];
    unsigned* const* flags = peers.flag[slot];
    if (threadIdx.x == 0) peer_timeout = 0;
    if (threadIdx.x < n) blocks[peers.rank][threadIdx.x] = sum;
    __threadfence_system();
    __syncthreads();
    if ((int)threadIdx.x < peers.nranks &&
        peer_signal_wait(flags[threadIdx.x] + peers.rank, flags[peers.rank] + threadIdx.x, epoch))
      peer_timeout = 1;
    __syncthreads();
    asm volatile("" ::: "memory");      // the block loads below stay below the flag wait
    if (threadIdx.x < n) {
      sum = ld_relaxed_sys_f64(blocks[0] + threadIdx.x);
      for (int r = 1; r < peers.nranks; ++r) sum += ld_relaxed_sys_f64(blocks[r] + threadIdx.x);
      if (KEEP) parts[threadIdx.x] = sum;           // every block was read before the barrier above
    }
  }
  if (threadIdx.x < n) {
    double v;
    if (sqrt_norm) {
      v = (double)fp32_norm(sum);                    // cge.py:36-37: fp32 norm, non-finite -> +inf
      if (!finite_d(v)) v = CUDART_INF;
    } else {
      v = (double)(float)sum;                        // aksel.py:41 (and the search's `dot`): fp32 sum of squares
    }
    if (SEARCH) {
      if (search.partial != nullptr) *search.partial = sum;
      else                           search_step(search, v);
      *ticket = 0u;
    }
    key[threadIdx.x] = v;
  }
  // the status word after the transition, which rewrites the search's
  if (PEERS && threadIdx.x == 0 && peers.status != nullptr && (peer_timeout || !SEARCH))
    *peers.status = peer_timeout ? BZ_STATUS_PEER_TIMEOUT : BZ_STATUS_OK;
  if (SEARCH) return;
  __syncthreads();
  stable_order(key, n, order);
  if (threadIdx.x == 0) *ticket = 0u;
}

template <bool CENTER, int VEC, bool DOT = false, bool SEARCH = false>
__global__ void __launch_bounds__(kRdThreads, 2)
k2_rowdist(const __grid_constant__ RowTable rows, const int n, const float* __restrict__ center, const Geom g,
           double* __restrict__ parts, int32_t* __restrict__ order, unsigned* __restrict__ ticket, const int sqrt_norm,
           const SearchTail search) {
  rowdist_body<CENTER, VEC, DOT, SEARCH, false>(rows, n, center, g, parts, order, ticket, sqrt_norm, search, PeerTail{});
}

template <bool CENTER, int VEC, bool SEARCH>
__global__ void __launch_bounds__(kRdThreads, 2)
k2_rowdist_peers(const __grid_constant__ RowTable rows, const int n, const float* __restrict__ center, const Geom g,
                 double* __restrict__ parts, int32_t* __restrict__ order, unsigned* __restrict__ ticket, const int sqrt_norm,
                 const SearchTail search, const __grid_constant__ PeerTail peers) {
  rowdist_body<CENTER, VEC, false, SEARCH, true>(rows, n, center, g, parts, order, ticket, sqrt_norm, search, peers);
}

// K2' in CGE mode with the peers tail, keeping the R-summed sums (bz_anticge_peers' first exchange).
template <int VEC>
__global__ void __launch_bounds__(kRdThreads, 2)
k2_anticge_norms(const __grid_constant__ RowTable rows, const int n, const Geom g, double* __restrict__ parts,
                 int32_t* __restrict__ order, unsigned* __restrict__ ticket, const __grid_constant__ PeerTail peers) {
  rowdist_body<false, VEC, false, false, true, true>(rows, n, nullptr, g, parts, order, ticket, 1, SearchTail{}, peers);
}

// Blocks of a K2' launch over the vectors of g: up to two per SM, at least one (an empty shard too).
static unsigned rowdist_grid(const Geom& g) {
  int64_t grid = (g.nv + kRdThreads - 1) / kRdThreads;
  const int64_t cap = (int64_t)sm_count() * 2;
  if (grid > cap) grid = cap;
  if (grid > kMaxParts) grid = kMaxParts;
  if (grid < 1) grid = 1;
  return (unsigned)grid;
}

int launch_rowdist(const RowTable& rows, int n, const float* const* host_rows, const float* center, int64_t d,
                   double* parts, cudaStream_t st, int reverse, int32_t* order, unsigned* ticket, int sqrt_norm, int dot) {
  // The centre doubles as the alignment reference ("out") of the geometry
  Geom g = make_geom(host_rows, n, center ? (const void*)center : (const void*)host_rows[0], nullptr, d, 4);
  g.reverse = reverse;
  const unsigned grid = rowdist_grid(g);
  if (dot && center != nullptr) {
    if (g.vec == 4) k2_rowdist<true, 4, true><<<grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, nullptr, nullptr, 0, SearchTail{});
    else            k2_rowdist<true, 1, true><<<grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, nullptr, nullptr, 0, SearchTail{});
    return (int)grid;
  }
  if (order != nullptr) cudaMemsetAsync(ticket, 0, sizeof(unsigned), st);
  if (g.vec == 4) {
    if (center) k2_rowdist<true, 4><<<grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, SearchTail{});
    else        k2_rowdist<false, 4><<<grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, SearchTail{});
  } else {
    if (center) k2_rowdist<true, 1><<<grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, SearchTail{});
    else        k2_rowdist<false, 1><<<grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, SearchTail{});
  }
  return (int)grid;
}

int launch_rowdist_peers(const RowTable& rows, int n, const float* const* host_rows, const float* center, int64_t d,
                         double* parts, cudaStream_t st, int32_t* order, unsigned* ticket, int sqrt_norm,
                         const PeerTail& peers) {
  // bz_rowdist_partial's geometry (forward walk), so that the blocks are the collective path's
  const Geom g = make_geom(host_rows, n, center ? (const void*)center : (const void*)host_rows[0], nullptr, d, 4);
  const unsigned grid = rowdist_grid(g);
  cudaMemsetAsync(ticket, 0, sizeof(unsigned), st);
  const SearchTail none = {};
  if (g.vec == 4) {
    if (center) k2_rowdist_peers<true, 4, false><<<grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, none, peers);
    else        k2_rowdist_peers<false, 4, false><<<grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, none, peers);
  } else {
    if (center) k2_rowdist_peers<true, 1, false><<<grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, none, peers);
    else        k2_rowdist_peers<false, 1, false><<<grid, kRdThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm, none, peers);
  }
  return (int)grid;
}

int launch_anticge_norms(const RowTable& rows, int n, const float* const* host_rows, int64_t d, double* parts, int32_t* order,
                         unsigned* ticket, const PeerTail& peers, cudaStream_t st) {
  // bz_distance_partial's geometry for CGE (bz_rowdist_partial's), as launch_rowdist_peers
  const Geom g = make_geom(host_rows, n, (const void*)host_rows[0], nullptr, d, 4);
  const unsigned grid = rowdist_grid(g);
  cudaMemsetAsync(ticket, 0, sizeof(unsigned), st);
  if (g.vec == 4) k2_anticge_norms<4><<<grid, kRdThreads, 0, st>>>(rows, n, g, parts, order, ticket, peers);
  else            k2_anticge_norms<1><<<grid, kRdThreads, 0, st>>>(rows, n, g, parts, order, ticket, peers);
  return (int)grid;
}

int launch_rowdist_search(const float* out, const float* center, int64_t d, double* parts, const SearchTail& tail,
                          cudaStream_t st, const PeerTail* peers) {
  RowTable rows;
  for (int r = 0; r < kMaxN; ++r) rows.p[r] = out;
  const Geom g = make_geom(&out, 1, center, nullptr, d, 4);
  const unsigned grid = rowdist_grid(g);
  cudaError_t err;
  if (peers != nullptr)
    err = g.vec == 4
        ? launch_after(k2_rowdist_peers<true, 4, true>, grid, kRdThreads, 0, st, rows, 1, center, g, parts, nullptr, nullptr, 0, tail, *peers)
        : launch_after(k2_rowdist_peers<true, 1, true>, grid, kRdThreads, 0, st, rows, 1, center, g, parts, nullptr, nullptr, 0, tail, *peers);
  else
    err = g.vec == 4
        ? launch_after(k2_rowdist<true, 4, false, true>, grid, kRdThreads, 0, st, rows, 1, center, g, parts, nullptr, nullptr, 0, tail)
        : launch_after(k2_rowdist<true, 1, false, true>, grid, kRdThreads, 0, st, rows, 1, center, g, parts, nullptr, nullptr, 0, tail);
  return err == cudaSuccess ? (int)grid : -1;
}

}  // namespace bz
