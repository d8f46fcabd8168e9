// bitonic.cuh — the warp-wide bitonic sort of K1-many (k1_many.cu), shared with the scoring and the Bulyan reduce
// above kMaxNDistance rows (k5_many.cu, k4_many.cu): 32·K integer keys per warp, K per lane, in registers.
#pragma once

namespace bz {

// Where rank r of a sorted column is kept: a lane's K consecutive ranks then fall in distinct banks.
__device__ __forceinline__ int skew(int r) { return r + (r >> 5); }

// Ascending bitonic sort of the 32·K keys of a warp; lane l holds ranks l*K .. l*K + K-1 on return.
template <int K>
__device__ __forceinline__ void warp_bitonic(int (&v)[K], const int lane) {
  constexpr int LOGP = (K == 8) ? 8 : (K == 16) ? 9 : 10;
#pragma unroll
  for (int lk = 1; lk <= LOGP; ++lk) {
    const int k = 1 << lk;
#pragma unroll
    for (int lj = lk - 1; lj >= 0; --lj) {
      const int j = 1 << lj;
      if (j >= K) {
        // partner: the same register of lane ^ (j / K); this lane is the upper one when rank bit j is set
        const int lm = j / K;
        const bool upper = (lane & lm) != 0;
        const bool desc = ((lane * K) & k) != 0;    // k > j >= K: the direction depends on the lane only
        const bool keep_min = (upper == desc);
#pragma unroll
        for (int q = 0; q < K; ++q) {
          const int o = __shfl_xor_sync(0xffffffffu, v[q], lm);
          v[q] = keep_min ? min(v[q], o) : max(v[q], o);
        }
      } else {
#pragma unroll
        for (int q = 0; q < K; ++q) {
          if ((q & j) == 0) {
            const int p = q | j;
            const bool desc = (k < K) ? ((q & k) != 0) : (((lane * K) & k) != 0);
            const int lo = min(v[q], v[p]), hi = max(v[q], v[p]);
            v[q] = desc ? hi : lo;
            v[p] = desc ? lo : hi;
          }
        }
      }
    }
  }
}

}  // namespace bz
