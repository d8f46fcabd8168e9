// k2_rowdist_wide.cu — K2' above 64 rows (bz_distance's Aksel and CGE): the squared distance of every row to
// the coordinate-wise median (aksel.py:41) or to the origin (cge.py:36) over the 128-pointer table, with the
// selection in the last CTA, as k2_rowdist does up to 64 rows.  K2'-share (k2_rowshare_wide, phase A of the
// d-sharded path, bz_distance_partial) is the same kernel with the last CTA writing the n sums instead.
//
// One fp32 accumulator per row and per thread, as k2_rowdist keeps, would take 128 registers; instead, as
// K6 does over the wide table (k6_study.cu), a thread takes one coordinate (VEC = 1) and folds its rows 32 at
// a time: the 32 squares of a chunk go through the transposed warp reduction (an fp32 sum over the warp's 32
// coordinates) and into fp64, so that lane L ends with rows L, L + 32, L + 64 and L + 96.  Warps are combined
// through shared memory in fixed order, one fp64 block per CTA; the last CTA (ticket) sums the blocks in S
// interleaved classes, the class sums in class order, and writes the stable order of the n keys.
// Deterministic; identical rows give identical sums.  Roofline: HBM, n·4 B per coordinate (+4 B for the centre).
// K2'-norms (k2_anticge_norms_wide, bz_anticge_peers' first exchange): CGE mode with the exchange over peer memory
// in the last CTA, as k2_rowdist's peers tail does up to 64 rows: it publishes the n sums K2'-share would write,
// adds the R ranks' sums in rank order, keeps them in parts[0, n) and writes the stable order of their keys.
#include "dist.cuh"
#include "k5_device.cuh"
#include "peers.cuh"
#include "reduce.cuh"

namespace bz {

constexpr int kRwThreads = 256;
constexpr int kRwWarps = kRwThreads / 32;
constexpr int kRwChunks = kMaxNDistance / 32;

// The last CTA of K2'-norms after the class sums are in `partial`: thread c < n forms the sum K2'-share writes,
// publishes it in this rank's slot, flags and waits (peers.cuh), adds the R ranks' sums in rank order,
// ((p0 + p1) + p2) + ..., keeps that in parts[c] (every block was read before the caller's barrier), and the stable
// order of the keys follows as in k2_rowdist_wide.  The epoch and the slot: by value, or (`next`) from this
// rank's own flags, read before the barrier that precedes the signal.
__device__ __forceinline__ void rowdist_wide_peers_tail(const PeerTail& peers, const double* partial, double* key, int S, int n,
                                                        double* __restrict__ parts, int32_t* __restrict__ order,
                                                        unsigned* __restrict__ ticket) {
  __shared__ int peer_timeout;
  double sum = 0.;
  if (threadIdx.x < n)
    for (int k = 0; k < S; ++k) sum += partial[k * n + threadIdx.x];
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
    parts[threadIdx.x] = sum;
    const double v = (double)fp32_norm(sum);           // cge.py:36-37: fp32 norm, non-finite -> +inf
    key[threadIdx.x] = finite_d(v) ? v : CUDART_INF;
  }
  if (threadIdx.x == 0 && peers.status != nullptr) *peers.status = peer_timeout ? BZ_STATUS_PEER_TIMEOUT : BZ_STATUS_OK;
  __syncthreads();
  stable_order(key, n, order);
  if (threadIdx.x == 0) *ticket = 0u;
}

// SUMS: the last CTA writes the n sums to `sums` (K2'-share); otherwise the stable order of their keys to `order`.
// PEERS (CGE, not SUMS): the sums are exchanged first (`peers`), and the R-summed sums are kept in parts[0, n).
template <bool CENTER, bool SUMS, bool PEERS = false>
__device__ __forceinline__ void rowdist_wide_body(const WideRowTable& rows, const int n, const float* __restrict__ center,
                                                  const Geom& g, double* __restrict__ parts, int32_t* __restrict__ order,
                                                  unsigned* __restrict__ ticket, const int sqrt_norm,
                                                  double* __restrict__ sums, const PeerTail* peers = nullptr) {
  __shared__ double warp_tot[kRwWarps][kMaxNDistance];
  __shared__ bool last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double dr[kRwChunks];
#pragma unroll
  for (int c = 0; c < kRwChunks; ++c) dr[c] = 0.;
  const int64_t stride = (int64_t)gridDim.x * kRwThreads;
  // warp-uniform trip count: lanes past the end contribute zeros and still join the shuffles
  const int64_t first = (int64_t)blockIdx.x * kRwThreads + warp * 32;
  for (int64_t vf = first; vf < g.nv; vf += stride) {
    // reversed walk (Geom::reverse): same warp-uniform trip count, mirrored base; VEC = 1: no shift
    const int64_t e = (g.reverse ? ((g.nv - 1) / 32) * 32 - vf : vf) + lane;
    const bool live = e < g.d;
    // out-of-range lanes and rows past n add exactly 0: they take the centre itself
    const float c = (CENTER && live) ? __ldcs(center + e) : 0.f;
#pragma unroll
    for (int ch = 0; ch < kRwChunks; ++ch) {
      if (ch * 32 >= n) break;                              // warp-uniform
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
          v[j] = __fmul_rn(df, df);                        // aksel.py:41: the square is rounded to fp32
        } else {
          v[j] = __fmul_rn(v[j], v[j]);
        }
      }
      dr[ch] += (double)transpose_reduce(v, lane);
    }
  }
#pragma unroll
  for (int c = 0; c < kRwChunks; ++c) warp_tot[warp][c * 32 + lane] = dr[c];
  __syncthreads();
  if (threadIdx.x < n) {
    double s = 0.;
#pragma unroll
    for (int w = 0; w < kRwWarps; ++w) s += warp_tot[w][threadIdx.x];
    parts[(size_t)blockIdx.x * n + threadIdx.x] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  double* partial = &warp_tot[0][0];                // S * n <= kRwThreads doubles
  double* key = partial + kRwThreads;               // n doubles behind them
  const int S = kRwThreads / n;                     // >= 2
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
  if (PEERS) {
    rowdist_wide_peers_tail(*peers, partial, key, S, n, parts, order, ticket);
    return;
  }
  if (threadIdx.x < n) {
    double sum = 0.;
    for (int k = 0; k < S; ++k) sum += partial[k * n + threadIdx.x];
    if (SUMS) {
      sums[threadIdx.x] = sum;
    } else {
      double v;
      if (sqrt_norm) {
        v = (double)fp32_norm(sum);                  // cge.py:36-37: fp32 norm, non-finite -> +inf
        if (!finite_d(v)) v = CUDART_INF;
      } else {
        v = (double)(float)sum;                      // aksel.py:41: fp32 sum of squares
      }
      key[threadIdx.x] = v;
    }
  }
  if (!SUMS) {
    __syncthreads();
    stable_order(key, n, order);
  }
  if (threadIdx.x == 0) *ticket = 0u;
}

template <bool CENTER>
__global__ void __launch_bounds__(kRwThreads, 2)
k2_rowdist_wide(const __grid_constant__ WideRowTable rows, const int n, const float* __restrict__ center, const Geom g,
                double* __restrict__ parts, int32_t* __restrict__ order, unsigned* __restrict__ ticket, const int sqrt_norm) {
  rowdist_wide_body<CENTER, false>(rows, n, center, g, parts, order, ticket, sqrt_norm, nullptr);
}

template <bool CENTER>
__global__ void __launch_bounds__(kRwThreads, 2)
k2_rowshare_wide(const __grid_constant__ WideRowTable rows, const int n, const float* __restrict__ center, const Geom g,
                 double* __restrict__ parts, unsigned* __restrict__ ticket, double* __restrict__ sums) {
  rowdist_wide_body<CENTER, true>(rows, n, center, g, parts, nullptr, ticket, 0, sums);
}

__global__ void __launch_bounds__(kRwThreads, 2)
k2_anticge_norms_wide(const __grid_constant__ WideRowTable rows, const int n, const Geom g, double* __restrict__ parts,
                      int32_t* __restrict__ order, unsigned* __restrict__ ticket, const __grid_constant__ PeerTail peers) {
  rowdist_wide_body<false, false, true>(rows, n, nullptr, g, parts, order, ticket, 1, nullptr, &peers);
}

// The geometry of the kernels: at most two CTAs per SM and kMaxParts blocks; the ticket is zeroed first.
static unsigned rowdist_wide_grid(const float* const* host_rows, int n, const float* center, int64_t d, int reverse,
                                  unsigned* ticket, cudaStream_t st, Geom& g) {
  g = make_geom(host_rows, n, center, nullptr, d, 1);
  g.reverse = reverse;
  int64_t grid = (g.nv + kRwThreads - 1) / kRwThreads;
  const int64_t cap = (int64_t)sm_count() * 2;
  if (grid > cap) grid = cap;
  if (grid > kMaxParts) grid = kMaxParts;
  if (grid < 1) grid = 1;
  cudaMemsetAsync(ticket, 0, sizeof(unsigned), st);
  return (unsigned)grid;
}

int launch_rowdist(const WideRowTable& rows, int n, const float* const* host_rows, const float* center, int64_t d,
                   double* parts, cudaStream_t st, int reverse, int32_t* order, unsigned* ticket, int sqrt_norm) {
  Geom g;
  const unsigned grid = rowdist_wide_grid(host_rows, n, center, d, reverse, ticket, st, g);
  if (center) k2_rowdist_wide<true><<<grid, kRwThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm);
  else        k2_rowdist_wide<false><<<grid, kRwThreads, 0, st>>>(rows, n, center, g, parts, order, ticket, sqrt_norm);
  return (int)grid;
}

int launch_rowshare(const WideRowTable& rows, int n, const float* const* host_rows, const float* center, int64_t d,
                    double* parts, cudaStream_t st, int reverse, unsigned* ticket, double* sums) {
  Geom g;
  const unsigned grid = rowdist_wide_grid(host_rows, n, center, d, reverse, ticket, st, g);
  if (center) k2_rowshare_wide<true><<<grid, kRwThreads, 0, st>>>(rows, n, center, g, parts, ticket, sums);
  else        k2_rowshare_wide<false><<<grid, kRwThreads, 0, st>>>(rows, n, center, g, parts, ticket, sums);
  return (int)grid;
}

int launch_anticge_norms(const WideRowTable& rows, int n, const float* const* host_rows, int64_t d, double* parts,
                         int32_t* order, unsigned* ticket, const PeerTail& peers, cudaStream_t st) {
  Geom g;
  // launch_rowshare's geometry for CGE (bz_distance_partial), so that the published sums are phase A's
  const unsigned grid = rowdist_wide_grid(host_rows, n, nullptr, d, 0, ticket, st, g);
  k2_anticge_norms_wide<<<grid, kRwThreads, 0, st>>>(rows, n, g, parts, order, ticket, peers);
  return (int)grid;
}

}  // namespace bz
