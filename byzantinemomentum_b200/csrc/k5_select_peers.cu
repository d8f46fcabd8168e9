// k5_select_peers.cu — phase B of the d-sharded Multi-Krum, Bulyan, Aksel and CGE above 64 rows with the exchange
// over peer memory (bz_distance_select_peers, libbyzagg_peers.so): one CTA takes the exchange's epoch, copies this
// rank's phase-A block from the staging buffer into its slot, raises its flag on every rank and waits for theirs
// (peers.cuh), adds the R blocks in rank order, ((p0 + p1) + p2) + ..., and runs the steps of k5_blocks_select_wide
// (Multi-Krum, Bulyan) or k5_rowkeys_select_wide (Aksel, CGE) on the sum: the order and the status word are
// bz_distance_select's over the all-gathered blocks, bit for bit.
#include "k5_wide.cuh"
#include "peers.cuh"

namespace bz {

// The exchange up to the rank-order sum: the epoch (by value, or from this rank's own flags, read by thread 0
// before the barrier that precedes the signal) and its slot, the copy of `len` doubles of `staged` into this
// rank's slot, the signal and the bounded wait.  Returns the slot's blocks on every rank; *timeout is 1 when a
// peer did not show up.
__device__ __forceinline__ double* const* publish_and_wait(const PeerTail& peers, const double* __restrict__ staged, int len,
                                                           int* timeout) {
  __shared__ unsigned sh_epoch;
  __shared__ int sh_timeout;
  if (threadIdx.x == 0) {
    sh_epoch = peers.next ? next_epoch(peers.flag[0][peers.rank] + peers.rank, peers.flag[1][peers.rank] + peers.rank)
                          : peers.epoch;
    sh_timeout = 0;
  }
  __syncthreads();
  const unsigned epoch = sh_epoch;
  const int slot = peers.next ? (int)(epoch & 1u) : 0;
  double* const* blocks = peers.block[slot];
  unsigned* const* flags = peers.flag[slot];
  double* mine = blocks[peers.rank];
  for (int e = threadIdx.x; e < len; e += blockDim.x) mine[e] = staged[e];
  __threadfence_system();
  __syncthreads();
  if ((int)threadIdx.x < peers.nranks &&
      peer_signal_wait(flags[threadIdx.x] + peers.rank, flags[peers.rank] + threadIdx.x, epoch))
    sh_timeout = 1;
  __syncthreads();
  asm volatile("" ::: "memory");      // the block loads below stay below the flag wait
  *timeout = sh_timeout;
  return blocks;
}

// Entry k of the R blocks, added in rank order.
__device__ __forceinline__ double rank_sum(double* const* blocks, int nranks, size_t k) {
  double s = ld_relaxed_sys_f64(blocks[0] + k);
  for (int p = 1; p < nranks; ++p) s += ld_relaxed_sys_f64(blocks[p] + k);
  return s;
}

// Multi-Krum (bulyan = 0) and Bulyan: `part` is the n x n block of bz_distance_partial (entries i < j).  Each pair
// is read once from the R slots and written to both halves of the table; the diagonal is +inf.
__global__ void __launch_bounds__(kK5WideThreads)
k5_blocks_select_peers(const double* __restrict__ part, int n, int count, int32_t* __restrict__ order, int f, int m,
                       int bulyan, const __grid_constant__ PeerTail peers) {
  extern __shared__ double sm_wide[];
  double* score = sm_wide;                                   // n
  float* dist = reinterpret_cast<float*>(sm_wide + n);      // n x n
  float* sorted = dist + n * n;                              // n x n
  int timeout;
  double* const* blocks = publish_and_wait(peers, part, n * n, &timeout);
  for (int e = threadIdx.x; e < n * n; e += blockDim.x) {
    const int i = e / n, j = e - i * n;
    if (i == j) {
      dist[e] = __int_as_float(0x7f800000);
    } else if (i < j) {
      float v = fp32_norm(rank_sum(blocks, peers.nranks, (size_t)e));
      if (!finite_d(v)) v = __int_as_float(0x7f800000);
      dist[e] = v;
      dist[j * n + i] = v;
    }
  }
  score_from_floats(dist, sorted, score, n, count, order, peers.status, f, m, bulyan);
  if (threadIdx.x == 0 && timeout) *peers.status = BZ_STATUS_PEER_TIMEOUT;
}

// Aksel (sqrt_norm = 0) and CGE: `part` holds the n sums of bz_distance_partial.
constexpr int kKeysPeersThreads = kMaxNDistance;
__global__ void __launch_bounds__(kKeysPeersThreads)
k5_rowkeys_select_peers(const double* __restrict__ part, int n, int sqrt_norm, int32_t* __restrict__ order,
                        const __grid_constant__ PeerTail peers) {
  __shared__ double key[kMaxNDistance];
  int timeout;
  double* const* blocks = publish_and_wait(peers, part, n, &timeout);
  for (int i = threadIdx.x; i < n; i += blockDim.x) key[i] = row_key(rank_sum(blocks, peers.nranks, (size_t)i), sqrt_norm);
  __syncthreads();
  stable_order(key, n, order);
  if (threadIdx.x == 0) *peers.status = timeout ? BZ_STATUS_PEER_TIMEOUT : BZ_STATUS_OK;
}

void launch_blocks_select_peers(const double* part, int n, int count, int32_t* order, int f, int m, int bulyan,
                                const PeerTail& peers, cudaStream_t st) {
  static unsigned long long opted = 0;
  opt_in_wide(k5_blocks_select_peers, opted);
  k5_blocks_select_peers<<<1, kK5WideThreads, score_wide_smem(n), st>>>(part, n, count, order, f, m, bulyan, peers);
}

void launch_rowkeys_select_peers(const double* part, int n, int sqrt_norm, int32_t* order, const PeerTail& peers,
                                 cudaStream_t st) {
  k5_rowkeys_select_peers<<<1, kKeysPeersThreads, 0, st>>>(part, n, sqrt_norm, order, peers);
}

}  // namespace bz
