// k6_many.cu — K6-many: the study metrics of bz_avg_dev_max (tools/pytorch.py:97-125 `compute_avg_dev_max`) over
// kMaxNCoordinate < n <= kMaxNMany rows (bz_avg_dev_max_many, libbyzagg_many_tools.so), in one pass over HBM:
// (n + 1)·4 bytes per coordinate.
//
// A column of 129..1024 values no longer fits one thread's registers, and the deviations need the finished
// average, so a persistent CTA (one per SM) stages column tiles of all n rows in shared memory, as K1-many does:
// 4-byte cp.async (rows need only be 4-byte aligned) into a ring of kStStages stages, each completing on its
// mbarrier (cp.async.mbarrier.arrive.noinc).  The warps have two roles, so that the sums of one tile overlap the
// deviations of the one before:
//   * the sum warps (the first kSumWarps): one thread per column forms the average in the reference's order
//     (clone, add_ in list order, one division: K3's and K6's bits), stores it, keeps it in a shared buffer for
//     the other warps, and accumulates avg^2 (fp64) and max |avg| (bit patterns; a NaN pattern is largest);
//   * the deviation warps (the rest): they issue the copies of every tile, and fold the squared deviations of
//     the previous tile into per-row fp64 accumulators, each thread owning rows dt, dt + DT, ... and summing
//     (g_i[k] - avg[k])^2 in fp32 over the tile's columns first.
// Iteration `it` of a CTA: the sum warps sum tile it, the deviation warps issue tile it + 1 and fold tile it - 1;
// three stages hold those three tiles.
// The ordered sum is a chain of n dependent fp32 adds per column, so the tile's columns (TC = 64 / 32 / 16 for
// the buckets P = 256 / 512 / 1024) are the chains in flight per SM; each thread loads the next 8 rows of its
// column while it adds the current 8, so a chain advances one add per FADD latency.
// Each CTA writes one block of n + 2 doubles (sum avg^2, its max |avg| pattern, the n row sums); the LAST CTA to
// finish (ticket) adds the blocks in index order: deterministic, and no second launch.
// Shared memory: three stages of TC x (P + 1) floats (~197 KB), so one CTA of 8 warps per SM.
#include "tma.cuh"

namespace bz {

constexpr int kStManyThreads = 256;
constexpr int kStStages = 3;
constexpr int kStTileFloats = 16384;              // TC x P: every bucket stages the same bytes per tile
constexpr int kStManyBlocks = 256;                // most CTAs of a launch: the workspace holds that many blocks

template <int P>
struct StudyTile {
  static constexpr int TC = kStTileFloats / P;    // columns per tile: 64, 32, 16
  static constexpr int LD = P + 1;                // floats per staged column, odd: the sum warps' lanes (one column
                                                  // each) read distinct banks
  static constexpr int kSumWarps = (TC + 31) / 32;
  static constexpr int DT = kStManyThreads - 32 * kSumWarps;    // deviation threads: 192, 224, 224
  static constexpr int RPT = (P + DT - 1) / DT;                 // rows per deviation thread: 2, 3, 5
  static constexpr int kStageFloats = TC * LD;
  static constexpr int kBarrierBytes = 64;
  static constexpr size_t kSmemBytes = kBarrierBytes + (size_t)kStStages * kStageFloats * sizeof(float);
};

// The same instruction as k1_many.cu's helper of that name (that file is kept as it is).
__device__ __forceinline__ void cp_async_arrive_noinc(unsigned long long* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

template <int P>
__global__ void __launch_bounds__(kStManyThreads, 1)
k6_many(const __grid_constant__ ManyRowTable rows, const int n, const int64_t d, const float divisor,
        float* __restrict__ avg, double* __restrict__ parts, unsigned* __restrict__ ticket, double* __restrict__ stats) {
  using T = StudyTile<P>;
  constexpr int TC = T::TC, LD = T::LD, DT = T::DT, RPT = T::RPT;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* full = reinterpret_cast<unsigned long long*>(smem_raw);
  float* stages = reinterpret_cast<float*>(smem_raw + T::kBarrierBytes);
  __shared__ float avg_s[2][TC];                  // the averages of the last two tiles
  __shared__ double warp_sq[T::kSumWarps];
  __shared__ unsigned warp_max[T::kSumWarps];
  __shared__ bool last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool summer = warp < T::kSumWarps;
  const int dt = threadIdx.x - 32 * T::kSumWarps;                         // deviation thread index
  const int64_t ntiles = (d + TC - 1) / TC;
  const int mine = (int)((ntiles - blockIdx.x + gridDim.x - 1) / gridDim.x);   // >= 1: the grid is <= ntiles

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kStStages; ++s) mbar_init(&full[s], DT);
  }
  __syncthreads();

  auto first_col = [&](int j) { return ((int64_t)blockIdx.x + (int64_t)j * gridDim.x) * TC; };
  // Local tile j (columns [e0, e0 + TC) of all n rows) into stage j % kStStages: column c at c * LD, row r at
  // offset r.  Every deviation thread arrives on the stage's barrier once its own copies have landed.
  auto issue = [&](int j) {
    const int64_t e0 = first_col(j);
    float* st = stages + (j % kStStages) * T::kStageFloats;
    for (int q = dt; q < n * TC; q += DT) {
      const int r = q / TC, c = q % TC;
      if (e0 + c < d) cp_async_vec<1>(st + c * LD + r, rows.p[r] + e0 + c);
    }
    cp_async_arrive_noinc(&full[j % kStStages]);
  };

  double dc = 0., acc[RPT];
#pragma unroll
  for (int q = 0; q < RPT; ++q) acc[q] = 0.;
  unsigned cm = 0;
  if (!summer) issue(0);
  for (int it = 0; it <= mine; ++it) {
    if (summer) {
      const int c = threadIdx.x;
      if (it < mine) {
        const int s = it % kStStages;
        mbar_wait(&full[s], (unsigned)(it / kStStages) & 1u);
        const int64_t e = first_col(it) + c;
        if (c < TC && e < d) {
          const float* col = stages + s * T::kStageFloats + c * LD;
          float sum = col[0];                                   // clone()            :108
          float cur[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) cur[u] = col[min(1 + u, n - 1)];
          int r = 1;
          for (; r + 8 <= n; r += 8) {
            float next[8];
#pragma unroll
            for (int u = 0; u < 8; ++u) next[u] = col[min(r + 8 + u, n - 1)];
#pragma unroll
            for (int u = 0; u < 8; ++u) sum = __fadd_rn(sum, cur[u]);   // add_ in list order  :109-110
#pragma unroll
            for (int u = 0; u < 8; ++u) cur[u] = next[u];
          }
#pragma unroll
          for (int u = 0; u < 8; ++u)
            if (r + u < n) sum = __fadd_rn(sum, cur[u]);
          const float a = __fdiv_rn(sum, divisor);              // div_(len(samples))  :111
          avg_s[it & 1][c] = a;
          __stcs(avg + e, a);
          const double a2 = (double)a * (double)a;             // exact; a square fp32 cannot see (<= 2^-150)
          dc += a2 <= 0x1p-150 ? 0. : a2;                        // counts 0, as in the reference's fp32 norm
          cm = max(cm, __float_as_uint(a) & 0x7fffffffu);
        }
      }
    } else {
      if (it + 1 < mine) issue(it + 1);       // its stage held tile it - 2, folded before the last barrier
      if (it >= 1) {
        const int j = it - 1, s = j % kStStages;
        mbar_wait(&full[s], (unsigned)(j / kStStages) & 1u);
        const float* st = stages + s * T::kStageFloats;
        const int64_t left = d - first_col(j);
        const int cols = left < TC ? (int)left : TC;
        float part[RPT];
#pragma unroll
        for (int q = 0; q < RPT; ++q) part[q] = 0.f;
#pragma unroll
        for (int c = 0; c < TC; ++c) {
          if (c < cols) {
            const float a = avg_s[j & 1][c];
#pragma unroll
            for (int q = 0; q < RPT; ++q) {
              const int r = dt + q * DT;
              if (r < n) {
                const float df = __fsub_rn(st[c * LD + r], a);  // grad.sub(grad_avg)  :118
                part[q] = fmaf(df, df, part[q]);                  // grad.dot(grad)      :119
              }
            }
          }
        }
#pragma unroll
        for (int q = 0; q < RPT; ++q) acc[q] += (double)part[q];
      }
    }
    __syncthreads();
  }

  // this CTA's block: [sum avg^2, max |avg| pattern, row sums]
  double* block = parts + (size_t)blockIdx.x * (n + 2);
  if (summer) {
#pragma unroll
    for (int h = 16; h >= 1; h >>= 1) {
      dc += __shfl_xor_sync(0xffffffffu, dc, h);
      cm = max(cm, __shfl_xor_sync(0xffffffffu, cm, h));
    }
    if (lane == 0) { warp_sq[warp] = dc; warp_max[warp] = cm; }
  } else {
#pragma unroll
    for (int q = 0; q < RPT; ++q) {
      const int r = dt + q * DT;
      if (r < n) block[2 + r] = acc[q];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.;
    unsigned m = 0;
#pragma unroll
    for (int w = 0; w < T::kSumWarps; ++w) { s += warp_sq[w]; m = max(m, warp_max[w]); }
    block[0] = s;
    block[1] = (double)m;                        // exact: a 32-bit pattern
  }
  // publish this CTA's block, take a ticket; the holder of the last ticket sees every block
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  // Entry j of the blocks, added in block order (entry 1: their largest pattern), eight loads in flight.
  const int width = n + 2, nb = (int)gridDim.x;
  for (int j = threadIdx.x; j < width; j += kStManyThreads) {
    double sum = 0., top = 0.;
    int p = 0;
    for (; p + 8 <= nb; p += 8) {
      double t[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) t[u] = __ldcg(parts + (size_t)(p + u) * width + j);
#pragma unroll
      for (int u = 0; u < 8; ++u) { sum += t[u]; top = fmax(top, t[u]); }
    }
    for (; p < nb; ++p) {
      const double t = __ldcg(parts + (size_t)p * width + j);
      sum += t;
      top = fmax(top, t);
    }
    stats[j] = j == 1 ? (double)__uint_as_float((unsigned)top) : sum;
  }
}

template <int P>
static void launch_bucket(const ManyRowTable& rows, int n, int64_t d, float* avg, double* parts, unsigned* ticket,
                          double* stats, int sms, cudaStream_t st) {
  using T = StudyTile<P>;
  const int64_t ntiles = (d + T::TC - 1) / T::TC;
  int64_t blocks = ntiles < sms ? ntiles : sms;
  if (blocks > kStManyBlocks) blocks = kStManyBlocks;
  cudaFuncSetAttribute(k6_many<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T::kSmemBytes);
  cudaMemsetAsync(ticket, 0, sizeof(unsigned), st);
  k6_many<P><<<(unsigned)blocks, kStManyThreads, T::kSmemBytes, st>>>(rows, n, d, (float)n, avg, parts, ticket, stats);
}

// Bytes of the per-CTA blocks of a launch over n rows (the ticket goes in front of them).
size_t study_many_parts_bytes(int n) { return (size_t)kStManyBlocks * (n + 2) * sizeof(double); }

// K6-many over kMaxNCoordinate < n <= kMaxNMany rows, d >= 1; `parts` holds study_many_parts_bytes(n) bytes.
void launch_study_many(const ManyRowTable& rows, int n, int64_t d, float* avg, double* stats, double* parts,
                       unsigned* ticket, int sms, cudaStream_t st) {
  if (n <= 256)      launch_bucket<256>(rows, n, d, avg, parts, ticket, stats, sms, st);
  else if (n <= 512) launch_bucket<512>(rows, n, d, avg, parts, ticket, stats, sms, st);
  else               launch_bucket<1024>(rows, n, d, avg, parts, ticket, stats, sms, st);
}

}  // namespace bz
