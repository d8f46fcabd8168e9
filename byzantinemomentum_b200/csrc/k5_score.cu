// k5_score.cu — K5: scoring and selection on the n x n distance table, one CTA, on device.
// The reference does this part in Python on the host after n(n-1)/2 `.item()` syncs
// (krum.py:49-62, bulyan.py:56-62, brute.py:47-68, aksel.py:49, cge.py:38); here it chains on
// the stream between the distance pass and the reduce pass, and must reproduce Python's
// behaviour exactly: distances are fp32 values widened to double, non-finite -> +inf
// (krum.py:46-47), `sum()` of floats is CPython's (>= 3.12: Neumaier-compensated), sorts are
// stable, brute enumerates `itertools.combinations` in lexicographic order with a strict `<`.
#include "k5_device.cuh"

namespace bz {

constexpr int kK5Threads = 1024;

template <class Parts>
__global__ void __launch_bounds__(kK5Threads)
k5_score_select(const __grid_constant__ Parts parts, const __grid_constant__ RowMap map, int nparts, int n, int count,
                int32_t* __restrict__ order, int32_t* __restrict__ status, int f, int m, int bulyan) {
  extern __shared__ double sm[];
  score_select_body(parts, map, nparts, n, count, order, status, f, m, bulyan, sm);
}

// aksel.py:39-49 / cge.py:28-38: stable order of n keys.
constexpr int kRowSelThreads = kMaxN;   // one per row
template <class Parts>
__global__ void __launch_bounds__(kRowSelThreads)
k5_rowdist_select(const __grid_constant__ Parts parts, int nparts, int n, int sqrt_norm, int32_t* __restrict__ order) {
  __shared__ double key[kMaxN];
  block_sum_parts(parts, nparts, n, key);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const double s = key[i];
    double v;
    if (sqrt_norm) {
      v = (double)fp32_norm(s);
      if (!finite_d(v)) v = CUDART_INF;
    } else {
      v = (double)(float)s;
    }
    key[i] = v;
  }
  __syncthreads();
  stable_order(key, n, order);
}

template <class Parts>
__global__ void __launch_bounds__(kK5Threads)
k5_brute_select(const __grid_constant__ Parts parts, const __grid_constant__ RowMap map, int nparts, int n, int f,
                unsigned long long total, int32_t* __restrict__ sel, int32_t* __restrict__ status) {
  extern __shared__ double sm[];
  brute_select_body(parts, map, nparts, n, f, total, sel, status, sm);
}

// ---- host side ---------------------------------------------------------------------------

template <class K>
static void opt_in_once(K kernel, size_t bytes, unsigned long long& mask) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(mask & bit)) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    mask |= bit;
  }
}

constexpr size_t kScoreSmemMax = (size_t)(2 * kMaxN * kMaxN + kMaxN) * sizeof(double);
constexpr size_t kBruteSmemMax = (size_t)kMaxN * kMaxN * sizeof(double) + (size_t)(kMaxN + 1) * (kMaxN + 1) * sizeof(unsigned long long) + 512;

// Brute (kind 3) runs k5_brute_select; Multi-Krum and Bulyan run k5_score_select, where only
// Bulyan's step reads the status word (as in the distance pass's tail).
template <class Parts>
static void rule_select(const Parts& parts, const RowMap& map, int nparts, const SelectTail& s, cudaStream_t st) {
  const int n = s.n;
  if (s.kind == 3) {
    const size_t smem = (size_t)n * n * sizeof(double) + (size_t)(n + 1) * (n + 1) * sizeof(unsigned long long) + 64 * sizeof(double);
    static unsigned long long opted = 0;
    opt_in_once(k5_brute_select<Parts>, kBruteSmemMax, opted);
    k5_brute_select<Parts><<<1, kK5Threads, smem, st>>>(parts, map, nparts, n, s.f, s.total, s.order, s.status);
  } else {
    const int bulyan = s.kind == 2;
    const size_t smem = (size_t)(2 * n * n + n) * sizeof(double);
    static unsigned long long opted = 0;
    opt_in_once(k5_score_select<Parts>, kScoreSmemMax, opted);
    k5_score_select<Parts><<<1, kK5Threads, smem, st>>>(parts, map, nparts, n, s.count, s.order, bulyan ? s.status : nullptr,
                                                        s.f, s.m, bulyan);
  }
}

static PeerParts make_peers(const double* const* ptrs, int npeers) {
  PeerParts p;
  for (int r = 0; r < kMaxPeers; ++r) p.ptr[r] = ptrs[r < npeers ? r : 0];
  return p;
}

void launch_select(const SelectTail& sel, const double* parts, int nparts, cudaStream_t st, int u) {
  const RowMap map = make_map(sel.to_unique, sel.n, u);
  rule_select(StridedParts{parts, (size_t)map.u * map.u}, map, nparts, sel, st);
}
void launch_rowdist_select(const double* parts, int nparts, int n, int sqrt_norm, int32_t* order, cudaStream_t st) {
  k5_rowdist_select<StridedParts><<<1, kRowSelThreads, 0, st>>>(StridedParts{parts, (size_t)n}, nparts, n, sqrt_norm, order);
}

// Peer variants: block p is read from peers[p] (NVLink peer memory)
void launch_select(const SelectTail& sel, const double* const* peers, int npeers, cudaStream_t st) {
  rule_select(make_peers(peers, npeers), identity_map(sel.n), npeers, sel, st);
}
void launch_rowdist_select_peers(const double* const* peers, int npeers, int n, int sqrt_norm, int32_t* order, cudaStream_t st) {
  k5_rowdist_select<PeerParts><<<1, kRowSelThreads, 0, st>>>(make_peers(peers, npeers), npeers, n, sqrt_norm, order);
}

}  // namespace bz
