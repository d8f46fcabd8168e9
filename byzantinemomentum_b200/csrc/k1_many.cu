// k1_many.cu — K1-many: the coordinate-wise rules over kMaxNCoordinate < n <= kMaxNMany rows (bz_coordinate_many).
//
// Above 128 rows a column no longer fits one thread's registers, so the column is ordered by a warp:
//   * a persistent CTA (one per SM) walks tiles of TC adjacent columns.  Each tile of all n rows is staged in
//     shared memory by 4-byte cp.async (rows need only be 4-byte aligned, each at its own offset) into a ring of
//     kManyStages stages; every thread's copies complete on the stage's mbarrier (cp.async.mbarrier.arrive.noinc),
//     so the next tiles stream in from HBM while the current one is sorted;
//   * one warp sorts one staged column: lane l takes rows l, l + 32, ... as K1's integer keys (NaN last, -0 before
//     +0), padded with INT_MAX up to P = 256, 512 or 1024 (one kernel per bucket of n), bitonic-sorts the P keys in
//     registers (lane l holds ranks l*K .. l*K + K-1; partners K or more ranks apart are exchanged by shuffles) and
//     writes the sorted column back over the staged one, rank r at r + r/32 so that no two lanes share a bank;
//   * one lane per column then runs the epilogue K1 runs (k1_select.cuh) on the sorted column, in the order the
//     NumPy oracle restates: the lower median (NaN when the column holds a NaN); the trimmed mean summed in
//     ascending rank order in ATen's 16-row cascade (levels of 16 and 256 rows), then divided by n - 2f; Phocas /
//     MeaMed: of each pair (s[l], s[l + m]), l < f, the one closer to the centre, then the core s[f .. m-1], summed
//     from +0 in that order and divided by m (K1's closest_pairs).
// The average above 128 rows is K3's ordered sum over the 1024-pointer table (k3_many_average).
// Shared memory: three stages of TC x (P + P/32 + 1) floats, ~199 KB, so one CTA of 8 warps per SM.
#include <climits>

#include "launch.cuh"
#include "tma.cuh"
#include "k3_average.cuh"
#include "bitonic.cuh"

namespace bz {

constexpr int kManyThreads = 256;
constexpr int kManyWarps = kManyThreads / 32;
constexpr int kManyStages = 3;
constexpr int kManyTileFloats = 16384;           // TC x P: every bucket stages the same bytes per tile

template <int P>
struct ManyTile {
  static constexpr int K = P / 32;                  // keys per lane
  static constexpr int TC = kManyTileFloats / P;    // columns per tile: 64, 32, 16
  static constexpr int LD = P + P / 32 + 1;         // floats per staged column: room for the skewed ranks, odd so
                                                    // that the copies of adjacent columns land in distinct banks
  static constexpr int kStageFloats = TC * LD;
  static constexpr int kBarrierBytes = 64;
  static constexpr size_t kSmemBytes = kBarrierBytes + (size_t)kManyStages * kStageFloats * sizeof(float);
  static_assert(TC % kManyWarps == 0, "whole columns per warp");
};

__device__ __forceinline__ void cp_async_arrive_noinc(unsigned long long* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ---- epilogues on a sorted column: rank r at col[skew(r)] ----------------------------------------

__device__ __forceinline__ float many_median(const float* col, int n) {
  const float top = col[skew(n - 1)];        // NaN sorts last
  return (top != top) ? quiet_nan() : col[skew((n - 1) / 2)];
}

// `values[f:-f].mean(dim=0)` for R = n - 2f <= 1024 kept ranks: ATen's cascade (the oracle's aten_mean_dim0)
// folds a level of 16 rows into the next every 16 rows, that one into a third every 256, and adds the
// partial levels as ((acc0 + acc1) + acc2) + acc3 (acc3, the 4096-row level, is +0 here).
__device__ __forceinline__ float many_trmean(const float* col, int n, int f) {
  const int R = n - 2 * f;
  float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f;
  int k = 0;
  for (; k + 16 <= R; k += 16) {
    float b = 0.f;
#pragma unroll
    for (int t = 0; t < 16; ++t) b = __fadd_rn(b, col[skew(f + k + t)]);
    acc1 = __fadd_rn(acc1, b);
    if (((k + 16) & 255) == 0) {
      acc2 = __fadd_rn(acc2, acc1);
      acc1 = 0.f;
    }
  }
  for (; k < R; ++k) acc0 = __fadd_rn(acc0, col[skew(f + k)]);
  return __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(acc0, acc1), acc2), 0.f), (float)R);
}

// The mean of the m = n - f values closest to c (K1's closest_pairs, in its order).
__device__ __forceinline__ float many_closest(const float* col, int n, int f, float c) {
  const int m = n - f;
  float acc = 0.f;
  for (int l = 0; l < f; ++l) {
    const float lo = col[skew(l)], hi = col[skew(l + m)];
    acc = __fadd_rn(acc, (abs_key(__fsub_rn(lo, c)) > abs_key(__fsub_rn(hi, c))) ? hi : lo);
  }
  for (int k = f; k < m; ++k) acc = __fadd_rn(acc, col[skew(k)]);
  const float r = __fdiv_rn(acc, (float)m);
  return (c != c) ? quiet_nan() : r;
}

__device__ __forceinline__ float many_epilogue(const float* col, int n, int rule, int f) {
  if (rule == BZ_RULE_MEDIAN) return many_median(col, n);
  if (rule == BZ_RULE_TRMEAN) return many_trmean(col, n, f);
  const float c = (rule == BZ_RULE_PHOCAS) ? many_trmean(col, n, f) : many_median(col, n);
  return many_closest(col, n, f, c);
}

// ---- the kernel ----------------------------------------------------------------------------------

template <int P>
__global__ void __launch_bounds__(kManyThreads, 1)
k1_many(const __grid_constant__ ManyRowTable rows, const int n, const int64_t d, const int rule, const int f,
        float* __restrict__ out) {
  using T = ManyTile<P>;
  constexpr int TC = T::TC, K = T::K;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* full = reinterpret_cast<unsigned long long*>(smem_raw);
  float* stages = reinterpret_cast<float*>(smem_raw + T::kBarrierBytes);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t ntiles = (d + TC - 1) / TC;

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kManyStages; ++s) mbar_init(&full[s], kManyThreads);
  }
  __syncthreads();
  pdl_wait();        // the rows are valid from here

  // Stage tile t (columns [t*TC, t*TC + TC) of all n rows) into stage s; column c at stages + s*kStageFloats + c*LD,
  // row r at offset r.  Every thread arrives on the stage's barrier once its own copies have landed.
  auto issue = [&](int64_t t, int s) {
    const int64_t e0 = t * TC;
    float* st = stages + s * T::kStageFloats;
    for (int q = threadIdx.x; q < n * TC; q += kManyThreads) {
      const int r = q / TC, c = q % TC;
      if (e0 + c < d) cp_async_vec<1>(st + c * T::LD + r, rows.p[r] + e0 + c);
    }
    cp_async_arrive_noinc(&full[s]);
  };

#pragma unroll
  for (int s = 0; s < kManyStages - 1; ++s) {
    const int64_t t = blockIdx.x + (int64_t)s * gridDim.x;
    if (t < ntiles) issue(t, s);
  }
  int it = 0;
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
    // the stage of tile it + kManyStages - 1 held tile it - 1, which every thread is done with (barrier below)
    const int64_t ahead = t + (int64_t)(kManyStages - 1) * gridDim.x;
    if (ahead < ntiles) issue(ahead, (it + kManyStages - 1) % kManyStages);
    const int s = it % kManyStages;
    mbar_wait(&full[s], (unsigned)(it / kManyStages) & 1u);
    float* st = stages + s * T::kStageFloats;
    const int64_t e0 = t * TC;
    // each warp sorts its columns warp, warp + 8, ... one after the other
#pragma unroll 1
    for (int j = 0; j < TC / kManyWarps; ++j) {
      const int c = warp + kManyWarps * j;
      if (e0 + c >= d) break;
      float* col = st + c * T::LD;
      int v[K];
#pragma unroll
      for (int q = 0; q < K; ++q) {
        const int r = q * 32 + lane;
        v[q] = (r < n) ? float_to_key(col[r]) : INT_MAX;
      }
      __syncwarp();
      warp_bitonic<K>(v, lane);
#pragma unroll
      for (int q = 0; q < K; ++q) col[skew(lane * K + q)] = key_to_float(v[q]);
    }
    __syncwarp();
    if (lane < TC / kManyWarps) {
      const int c = warp + kManyWarps * lane;
      if (e0 + c < d) __stcs(out + e0 + c, many_epilogue(st + c * T::LD, n, rule, f));
    }
    __syncthreads();
  }
}

template <int VEC>
__global__ void __launch_bounds__(kK3Threads)
k3_many_average(const __grid_constant__ ManyRowTable rows, const Geom g, const int count, const float divisor,
                float* __restrict__ out) {
  k3_average_body<VEC>(rows, g, nullptr, count, 1, divisor, nullptr, out);
}

template <int P>
static void launch_bucket(const ManyRowTable& rows, int n, int64_t d, int rule, int f, int sms, float* out, cudaStream_t st) {
  using T = ManyTile<P>;
  const int64_t ntiles = (d + T::TC - 1) / T::TC;
  const unsigned blocks = (unsigned)(ntiles < sms ? ntiles : sms);
  cudaFuncSetAttribute(k1_many<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T::kSmemBytes);
  launch_after(k1_many<P>, blocks, kManyThreads, T::kSmemBytes, st, rows, n, d, rule, f, out);
}

void launch_many_sorted(const ManyRowTable& rows, int n, int64_t d, int rule, int f, int sms, float* out, cudaStream_t st) {
  if (d <= 0) return;
  if (n <= 256)      launch_bucket<256>(rows, n, d, rule, f, sms, out, st);
  else if (n <= 512) launch_bucket<512>(rows, n, d, rule, f, sms, out, st);
  else               launch_bucket<1024>(rows, n, d, rule, f, sms, out, st);
}

void launch_many_average(const ManyRowTable& rows, const Geom& g, int n, float* out, cudaStream_t st) {
  typedef void (*Kernel)(ManyRowTable, Geom, int, float, float*);
  if (g.nv <= 0) return;
  const unsigned blocks = (unsigned)((g.nv + kK3Threads - 1) / kK3Threads);
  const Kernel kernel = (g.vec == 4) ? Kernel(k3_many_average<4>) : (g.vec == 2) ? Kernel(k3_many_average<2>) : Kernel(k3_many_average<1>);
  launch_after(kernel, blocks, kK3Threads, 0, st, rows, g, n, (float)n, out);
}

}  // namespace bz
