// k10_anticge.cu — the attack built against CGE (attacks/anticge.py) after K2' has ranked the honest rows by
// their fp32 norm (CGE mode, the stable order σ in device memory):
//   K10  attack = σ0 + σ0 + σ1 + ... + σ(maxpos-1), fp32 adds in that order (`clone(σ0)` then `add_` over
//        normed[:maxpos]), and Σ attack² in fp64.  The last CTA (ticket) forms the fp32 `attnorm`, the
//        bound `maxnorm = nextafter(norm[σ_maxpos], 0)` in double, and the decision: scale by
//        fl32(-maxnorm / attnorm) when attnorm > 0, else leave the row as it is.
//        Roofline: HBM, (maxpos + 1)·4 B read (σ0 is loaded once for both of its terms) + 4 B written per coordinate.
//   K11  attack[j] = fl32(attack[j] · s) when the decision says so (ATen's `mul_` by a Python float multiplies by
//        the fp32 rounding of the scalar).  Walks backwards, so the columns K10 wrote last are read first from L2.
//        Roofline: 4 B read + 4 B written per coordinate.
//   fill The row of NaN the attack returns when f_real > f_decl: one launch, nothing read.
// The d-sharded form (bz_anticge_partial, bz_anticge_scale): K10 writes this rank's unscaled shard and its fp64
// partial Σ attack² instead of deciding; K11 then forms the same decision in every CTA from the R partials and
// the gathered norm blocks, added in rank order, so the factor has the same bits on every rank.
// The d-sharded form over peer memory (bz_anticge_peers, kernel k10_anticge_peers): K10 as in bz_anticge_partial,
// then its last CTA exchanges the partial (peers.cuh), adds the R partials in rank order and decides from them and
// the R-summed norms K2'-norms kept, as K11 of bz_anticge_scale does; K11 then reads the decision.
#include "dist.cuh"
#include "k5_device.cuh"
#include "launch.cuh"
#include "peers.cuh"

namespace bz {

constexpr int kAcThreads = 256;
constexpr int kAcWarps = kAcThreads / 32;
constexpr int kAcUnroll = 8;        // row loads in flight per vector

// The key K2''s last CTA ranked row `r` by, from its `nparts` per-CTA blocks: the S = 256 / n interleaved
// classes, each summed from 0.0 in block order, then the class sums in class order (k2_rowdist.cu and
// k2_rowdist_wide.cu sum them so, both with 256 threads), rounded as CGE rounds its norm.
__device__ __forceinline__ double rowdist_key(const double* __restrict__ parts, int nparts, int n, int r) {
  const int S = 256 / n;
  double sum = 0.;
  for (int k = 0; k < S; ++k) {
    double s = 0.;
    for (int p = k; p < nparts; p += S) s += __ldcg(parts + (size_t)p * n + r);
    sum += s;
  }
  const double v = (double)fp32_norm(sum);
  return finite_d(v) ? v : CUDART_INF;
}

// cge.py's key of a row from the R gathered blocks of phase A, added in rank order (k5's block_sum_parts).
__device__ __forceinline__ double gathered_key(const double* __restrict__ blocks, int nparts, int n, int r) {
  double s = __ldcg(blocks + r);
  for (int p = 1; p < nparts; ++p) s += __ldcg(blocks + (size_t)p * n + r);
  const double v = (double)fp32_norm(s);
  return finite_d(v) ? v : CUDART_INF;
}

// anticge.py:74-76 from the sum of squares of the attack and the key of σ_maxpos.
__device__ __forceinline__ AntiCgeScale anticge_decision(double sum_sq, double key) {
  const double maxnorm = nextafter(key, 0.);                   // math.nextafter(normed[maxpos][0], 0)
  const double attnorm = (double)fp32_norm(sum_sq);            // attack.norm().item()
  AntiCgeScale s;
  s.apply = attnorm > 0. ? 1 : 0;                              // false for NaN
  s.factor = s.apply ? (float)(-maxnorm / attnorm) : 1.f;
  return s;
}

// Sum over the CTA of one fp64 value per thread, in a fixed order; the result in thread 0.
__device__ __forceinline__ double block_sum(double v, double* smem) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int h = 16; h >= 1; h >>= 1) v += __shfl_xor_sync(0xffffffffu, v, h);
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  double s = 0.;
  if (threadIdx.x == 0)
    for (int w = 0; w < kAcWarps; ++w) s += smem[w];
  return s;
}

template <int VEC, bool FULL>
__device__ __forceinline__ void attack_vector(const float* const* srow, int maxpos, int64_t e0, int64_t d, float* out,
                                              double& sq) {
  float acc[VEC];
  load_vec<VEC>(srow[0], e0, d, FULL, acc);
  if (maxpos > 0) {
#pragma unroll
    for (int c = 0; c < VEC; ++c) acc[c] = __fadd_rn(acc[c], acc[c]);      // clone(σ0).add_(σ0)
  }
  int k = 1;
  for (; k + kAcUnroll <= maxpos; k += kAcUnroll) {
    float t[kAcUnroll][VEC];
#pragma unroll
    for (int u = 0; u < kAcUnroll; ++u) load_vec<VEC>(srow[k + u], e0, d, FULL, t[u]);
#pragma unroll
    for (int u = 0; u < kAcUnroll; ++u)
#pragma unroll
      for (int c = 0; c < VEC; ++c) acc[c] = __fadd_rn(acc[c], t[u][c]);
  }
  for (; k < maxpos; ++k) {
    float t[VEC];
    load_vec<VEC>(srow[k], e0, d, FULL, t);
#pragma unroll
    for (int c = 0; c < VEC; ++c) acc[c] = __fadd_rn(acc[c], t[c]);
  }
  // plain stores: K11 reads the row back, from L2 where it can
  if (FULL && VEC == 4) {
    *reinterpret_cast<float4*>(out + e0) = make_float4(acc[0], acc[VEC > 1 ? 1 : 0], acc[VEC > 2 ? 2 : 0], acc[VEC > 3 ? 3 : 0]);
  } else if (FULL) {
    out[e0] = acc[0];
  } else {
#pragma unroll
    for (int c = 0; c < VEC; ++c)
      if (e0 + c >= 0 && e0 + c < d) out[e0 + c] = acc[c];
  }
  // out-of-range lanes loaded 0 and add 0; a square is exact in fp64
#pragma unroll
  for (int c = 0; c < VEC; ++c) sq += (double)acc[c] * (double)acc[c];
}

// K10's pass: this CTA's columns of the attack row into `out`, its fp64 block of Σ out² into parts[blockIdx.x];
// true in the last CTA to finish (the ticket), which may then read every block.
template <int VEC, class Rows>
__device__ __forceinline__ bool attack_pass(const Rows& rows, const int maxpos, const int32_t* __restrict__ order,
                                            const Geom& g, float* __restrict__ out, double* __restrict__ parts,
                                            unsigned* __restrict__ ticket) {
  __shared__ const float* srow[kMaxNDistance];
  __shared__ double warp_sum[kAcWarps];
  __shared__ bool last;
  pdl_wait();                                    // σ is K2''s (or phase B's) output: valid from here
  for (int k = threadIdx.x; k <= maxpos; k += kAcThreads) srow[k] = rows.p[order[k]];
  __syncthreads();
  double sq = 0.;
  const int64_t stride = (int64_t)gridDim.x * kAcThreads;
  for (int64_t v = (int64_t)blockIdx.x * kAcThreads + threadIdx.x; v < g.nv; v += stride) {
    const int64_t e0 = v * VEC - g.shift;
    if (e0 >= 0 && e0 + VEC <= g.d) attack_vector<VEC, true>(srow, maxpos, e0, g.d, out, sq);
    else                            attack_vector<VEC, false>(srow, maxpos, e0, g.d, out, sq);
  }
  const double block = block_sum(sq, warp_sum);
  if (threadIdx.x == 0) {
    parts[blockIdx.x] = block;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  return last;
}

// K10.  `nparts_k2` > 0: the single-GPU form, the last CTA writes the decision to `scale` from K2''s blocks `k2_parts`;
// otherwise (bz_anticge_partial) it writes the fp64 sum of squares to `partial`.  `ticket` is zero on entry and again
// on exit.
template <int VEC, class Rows>
__global__ void __launch_bounds__(kAcThreads)
k10_anticge_sum(const __grid_constant__ Rows rows, const int n, const int maxpos, const int32_t* __restrict__ order,
                const Geom g, float* __restrict__ out, double* __restrict__ parts, unsigned* __restrict__ ticket,
                const double* __restrict__ k2_parts, const int nparts_k2, AntiCgeScale* __restrict__ scale,
                double* __restrict__ partial) {
  if (!attack_pass<VEC>(rows, maxpos, order, g, out, parts, ticket) || threadIdx.x != 0) return;
  __threadfence();
  double sum = 0.;                               // the blocks in block order
  for (int p = 0; p < (int)gridDim.x; ++p) sum += __ldcg(parts + p);
  if (partial != nullptr) *partial = sum;
  else                    *scale = anticge_decision(sum, rowdist_key(k2_parts, nparts_k2, n, order[maxpos]));
  *ticket = 0u;
}

// K10 with the second exchange of bz_anticge_peers.  The last CTA forms bz_anticge_partial's sum, publishes it in
// this rank's slot, flags and waits (peers.cuh), adds the R partials in rank order, ((p0 + p1) + p2) + ..., and
// writes to `scale` the decision k11_anticge_scale forms from the gathered partials and blocks: the key of σ_maxpos
// comes from `sums`, the R-summed norm sums K2'-norms kept in this rank's workspace (the peers' slots of the first
// exchange may be rewritten once this rank has signalled).  A timeout sets *peers.status; it is never cleared here.
template <int VEC, class Rows>
__global__ void __launch_bounds__(kAcThreads)
k10_anticge_peers(const __grid_constant__ Rows rows, const int n, const int maxpos, const int32_t* __restrict__ order,
                  const Geom g, float* __restrict__ out, double* __restrict__ parts, unsigned* __restrict__ ticket,
                  const double* __restrict__ sums, AntiCgeScale* __restrict__ scale, const __grid_constant__ PeerTail peers) {
  __shared__ int peer_timeout;
  if (!attack_pass<VEC>(rows, maxpos, order, g, out, parts, ticket)) return;
  __threadfence();
  // the epoch and the slot: by value, or (`next`) from this rank's own flags, which K2'-norms raised before this
  // grid's pdl_wait; read by every thread that needs them before the barrier below
  unsigned epoch = peers.epoch;
  int slot = 0;
  if (peers.next && (int)threadIdx.x < peers.nranks) {
    epoch = next_epoch(peers.flag[0][peers.rank] + peers.rank, peers.flag[1][peers.rank] + peers.rank);
    slot = (int)(epoch & 1u);
  }
  double* const* blocks = peers.block[slot];
  unsigned* const* flags = peers.flag[slot];
  if (threadIdx.x == 0) {
    double sum = 0.;                             // the blocks in block order: bz_anticge_partial's sum
    for (int p = 0; p < (int)gridDim.x; ++p) sum += __ldcg(parts + p);
    blocks[peers.rank][0] = sum;
    peer_timeout = 0;
  }
  __threadfence_system();
  __syncthreads();
  if ((int)threadIdx.x < peers.nranks &&
      peer_signal_wait(flags[threadIdx.x] + peers.rank, flags[peers.rank] + threadIdx.x, epoch))
    peer_timeout = 1;
  __syncthreads();
  asm volatile("" ::: "memory");      // the partial loads below stay below the flag wait
  if (threadIdx.x != 0) return;
  double sum = ld_relaxed_sys_f64(blocks[0]);
  for (int r = 1; r < peers.nranks; ++r) sum += ld_relaxed_sys_f64(blocks[r]);
  *scale = anticge_decision(sum, gathered_key(sums, 1, n, order[maxpos]));
  if (peer_timeout && peers.status != nullptr) *peers.status = BZ_STATUS_PEER_TIMEOUT;
  *ticket = 0u;
}

// K11.  `blocks` == NULL: the decision is K10's, in `scale`; otherwise every CTA forms it from the `nparts` gathered
// partial sums of squares and the gathered norm blocks (bz_anticge_scale).
template <int VEC>
__global__ void __launch_bounds__(kAcThreads)
k11_anticge_scale(const Geom g, float* __restrict__ out, const AntiCgeScale* __restrict__ scale,
                  const double* __restrict__ blocks, const double* __restrict__ partials, const int nparts, const int n,
                  const int maxpos, const int32_t* __restrict__ order) {
  __shared__ AntiCgeScale s;
  const int64_t blk = (int64_t)gridDim.x - 1 - blockIdx.x;
  const int64_t v = blk * kAcThreads + threadIdx.x;
  pdl_wait();                                    // K10's row and decision are valid from here
  if (threadIdx.x == 0) {
    if (blocks == nullptr) {
      s = *scale;
    } else {
      double sum = __ldcg(partials);
      for (int p = 1; p < nparts; ++p) sum += __ldcg(partials + p);
      s = anticge_decision(sum, gathered_key(blocks, nparts, n, order[maxpos]));
    }
  }
  __syncthreads();
  if (!s.apply || v >= g.nv) return;
  const int64_t e0 = v * VEC - g.shift;
  const bool full = e0 >= 0 && e0 + VEC <= g.d;
  float x[VEC];
  load_vec<VEC>(out, e0, g.d, full, x);
#pragma unroll
  for (int c = 0; c < VEC; ++c) x[c] = __fmul_rn(x[c], s.factor);
  store_vec<VEC>(out, e0, g.d, full, x);
}

__global__ void __launch_bounds__(kAcThreads) k_nan_fill(float* __restrict__ out, const int64_t d) {
  const int64_t stride = (int64_t)gridDim.x * kAcThreads;
  for (int64_t j = (int64_t)blockIdx.x * kAcThreads + threadIdx.x; j < d; j += stride) out[j] = quiet_nan();
}

// K10's grid over the vectors of g: up to two CTAs per SM and kMaxParts blocks, at least one (an empty shard too).
static unsigned sum_grid(const Geom& g) {
  int64_t grid = (g.nv + kAcThreads - 1) / kAcThreads;
  const int64_t cap = (int64_t)sm_count() * 2;
  if (grid > cap) grid = cap;
  if (grid > kMaxParts) grid = kMaxParts;
  if (grid < 1) grid = 1;
  return (unsigned)grid;
}

template <class Rows>
static int launch_sum(const Rows& rows, int n, const float* const* host_rows, int maxpos, const int32_t* order, int64_t d,
                      float* out, double* parts, unsigned* ticket, const double* k2_parts, int nparts_k2,
                      AntiCgeScale* scale, double* partial, cudaStream_t st) {
  const Geom g = make_geom(host_rows, n, out, nullptr, d, 4);
  const unsigned grid = sum_grid(g);
  const cudaError_t err = g.vec == 4
      ? launch_after(k10_anticge_sum<4, Rows>, (unsigned)grid, kAcThreads, 0, st, rows, n, maxpos, order, g, out, parts, ticket,
                     k2_parts, nparts_k2, scale, partial)
      : launch_after(k10_anticge_sum<1, Rows>, (unsigned)grid, kAcThreads, 0, st, rows, n, maxpos, order, g, out, parts, ticket,
                     k2_parts, nparts_k2, scale, partial);
  return err == cudaSuccess ? 0 : -1;
}

int launch_anticge_sum(const RowTable& rows, int n, const float* const* host_rows, int maxpos, const int32_t* order, int64_t d,
                       float* out, double* parts, unsigned* ticket, const double* k2_parts, int nparts_k2,
                       AntiCgeScale* scale, double* partial, cudaStream_t st) {
  return launch_sum(rows, n, host_rows, maxpos, order, d, out, parts, ticket, k2_parts, nparts_k2, scale, partial, st);
}
int launch_anticge_sum(const WideRowTable& rows, int n, const float* const* host_rows, int maxpos, const int32_t* order,
                       int64_t d, float* out, double* parts, unsigned* ticket, const double* k2_parts, int nparts_k2,
                       AntiCgeScale* scale, double* partial, cudaStream_t st) {
  return launch_sum(rows, n, host_rows, maxpos, order, d, out, parts, ticket, k2_parts, nparts_k2, scale, partial, st);
}

template <class Rows>
static int launch_peers(const Rows& rows, int n, const float* const* host_rows, int maxpos, const int32_t* order, int64_t d,
                        float* out, double* parts, unsigned* ticket, const double* sums, AntiCgeScale* scale,
                        const PeerTail& peers, cudaStream_t st) {
  const Geom g = make_geom(host_rows, n, out, nullptr, d, 4);       // bz_anticge_partial's geometry and grid
  const unsigned grid = sum_grid(g);
  const cudaError_t err = g.vec == 4
      ? launch_after(k10_anticge_peers<4, Rows>, grid, kAcThreads, 0, st, rows, n, maxpos, order, g, out, parts, ticket, sums,
                     scale, peers)
      : launch_after(k10_anticge_peers<1, Rows>, grid, kAcThreads, 0, st, rows, n, maxpos, order, g, out, parts, ticket, sums,
                     scale, peers);
  return err == cudaSuccess ? 0 : -1;
}

int launch_anticge_peers(const RowTable& rows, int n, const float* const* host_rows, int maxpos, const int32_t* order, int64_t d,
                         float* out, double* parts, unsigned* ticket, const double* sums, AntiCgeScale* scale,
                         const PeerTail& peers, cudaStream_t st) {
  return launch_peers(rows, n, host_rows, maxpos, order, d, out, parts, ticket, sums, scale, peers, st);
}
int launch_anticge_peers(const WideRowTable& rows, int n, const float* const* host_rows, int maxpos, const int32_t* order,
                         int64_t d, float* out, double* parts, unsigned* ticket, const double* sums, AntiCgeScale* scale,
                         const PeerTail& peers, cudaStream_t st) {
  return launch_peers(rows, n, host_rows, maxpos, order, d, out, parts, ticket, sums, scale, peers, st);
}

int launch_anticge_scale(float* out, int64_t d, const AntiCgeScale* scale, const double* blocks, const double* partials,
                         int nparts, int n, int maxpos, const int32_t* order, cudaStream_t st) {
  const float* row = out;
  const Geom g = make_geom(&row, 1, out, nullptr, d, 4);
  if (g.nv <= 0) return 0;
  const unsigned grid = (unsigned)((g.nv + kAcThreads - 1) / kAcThreads);
  const cudaError_t err = g.vec == 4
      ? launch_after(k11_anticge_scale<4>, grid, kAcThreads, 0, st, g, out, scale, blocks, partials, nparts, n, maxpos, order)
      : launch_after(k11_anticge_scale<1>, grid, kAcThreads, 0, st, g, out, scale, blocks, partials, nparts, n, maxpos, order);
  return err == cudaSuccess ? 0 : -1;
}

int launch_nan_fill(float* out, int64_t d, cudaStream_t st) {
  int64_t grid = (d + kAcThreads - 1) / kAcThreads;
  const int64_t cap = (int64_t)sm_count() * 8;
  if (grid > cap) grid = cap;
  k_nan_fill<<<(unsigned)grid, kAcThreads, 0, st>>>(out, d);
  return cudaPeekAtLastError() == cudaSuccess ? 0 : -1;
}

}  // namespace bz
