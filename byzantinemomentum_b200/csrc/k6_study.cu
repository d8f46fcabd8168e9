// k6_study.cu — K6: the study metrics of tools/pytorch.py:97-125 (`compute_avg_dev_max`, called
// three times per step by attack.py:846-848) in ONE pass over the rows.
//
// Everything the function returns is separable per coordinate: avg[k] needs column k only, and
// (g_i[k] - avg[k])^2 needs column k and avg[k].  So a thread that owns VEC adjacent coordinates
// loads its n x VEC values once, keeps them in registers, forms the average in the reference's
// order (clone, add_ in list order, one division), stores it, and accumulates per row the squared
// deviations, plus avg^2 and max |avg|.  The reference reads the rows n+... times: once for the
// average, once per `grad.sub(grad_avg)` (which also writes and re-reads a d-vector per row).
// Roofline: HBM, (n + 1)·4 B per coordinate.
//
// Accumulation: fp32 per thread over <= kStFlush vectors, then the transposed warp reduction into
// fp64 (lane r ends with row r and row r + 32), warps combined through shared memory in fixed
// order, one fp64 block per CTA; the LAST CTA to finish (ticket counter) sums the blocks in index
// order into `stats`: deterministic whichever CTA that is, and no second launch.
// max |avg| is order independent, so an atomicMax on the |x| bit patterns is deterministic too
// (a NaN pattern is larger than +inf: it propagates like torch's max()).
// Above kMaxN rows (bz_avg_dev_max up to kMaxNCoordinate) the kernel takes the 128-pointer WideRowTable,
// with VEC = 1 and the deviations folded at every vector (see that overload).
#include "dist.cuh"
#include "reduce.cuh"

namespace bz {

constexpr int kStThreads = 256;
constexpr int kStWarps = kStThreads / 32;
constexpr int kStFlush = 8;      // vectors between two flushes (<= 32 terms per fp32 accumulator)

// The end of the K6 kernels over the 128-pointer table (SLOTS = kMaxNCoordinate), once each warp has written
// its fp64 row sums to warp_tot[warp][0, n), its sum of avg^2 to warp_tot[warp][SLOTS] and its max |avg|
// pattern to warp_max[warp]: the CTA's block of n + 1 doubles, the ticket, and the final sum of the blocks
// by the last CTA, for CTAs of THREADS > SLOTS + 1 threads.  The same steps as the end of the 64-row kernel
// below, which keeps its own copy:
// calling this helper there permutes its register allocation, and its SASS is kept as it was.
template <int SLOTS, int THREADS>
__device__ __forceinline__ void study_blocks(double (&warp_tot)[THREADS / 32][SLOTS + 1], const unsigned (&warp_max)[THREADS / 32],
                                             bool& last, const int n, double* parts, unsigned* absmax_bits,
                                             unsigned* tickets, double* stats) {
  __syncthreads();
  double* mine = parts + (size_t)blockIdx.x * (n + 1);
  if (threadIdx.x < n) {
    double s = 0.;
#pragma unroll
    for (int w = 0; w < THREADS / 32; ++w) s += warp_tot[w][threadIdx.x];
    mine[1 + threadIdx.x] = s;
  } else if (threadIdx.x == SLOTS) {
    double s = 0.;
    unsigned m = 0;
#pragma unroll
    for (int w = 0; w < THREADS / 32; ++w) { s += warp_tot[w][SLOTS]; m = max(m, warp_max[w]); }
    mine[0] = s;
    if (m != 0) atomicMax(absmax_bits, m);
  }
  // publish this CTA's block, take a ticket; the holder of the last ticket sees every block
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(tickets, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  // Final sum of the gridDim.x blocks by the last CTA.  One thread per entry walking all blocks was a
  // chain of ~gridDim.x / 8 dependent L2 round trips (~20 us at 296 blocks: half of the kernel at
  // d = 1.3M); instead the blocks are split in S interleaved classes, thread (class s, entry c) adds
  // its class in ascending order with all loads in flight, and the S class sums are added in class
  // order: a fixed order for a given grid, every load independent.
  {
    const int width = n + 1;                        // entry 0: sum avg^2; entry 1 + i: deviations of row i
    const int S = THREADS / width;                  // >= 1 (THREADS > n + 1)
    const int c = threadIdx.x % width, cls = threadIdx.x / width;
    double* partial = &warp_tot[0][0];              // S * width <= THREADS doubles of the (now free) warp table
    if (cls < S) {
      double sum = 0.;
      int p = cls;
      for (; p + 7 * S < (int)gridDim.x; p += 8 * S) {
        double t[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) t[u] = __ldcg(parts + (size_t)(p + u * S) * width + c);
#pragma unroll
        for (int u = 0; u < 8; ++u) sum += t[u];
      }
      for (; p < (int)gridDim.x; p += S) sum += __ldcg(parts + (size_t)p * width + c);
      partial[cls * width + c] = sum;
    }
    __syncthreads();
    if (threadIdx.x < width) {
      double sum = 0.;
      for (int k = 0; k < S; ++k) sum += partial[k * width + threadIdx.x];
      stats[threadIdx.x == 0 ? 0 : 1 + threadIdx.x] = sum;
    } else if (threadIdx.x == SLOTS + 1) {
      stats[1] = (double)__uint_as_float(atomicMax(absmax_bits, 0u));
    }
  }
}

template <int NMAX, int VEC>
__global__ void __launch_bounds__(kStThreads, (NMAX * VEC + (NMAX <= 32 ? 32 : 64) > 100) ? 1 : 2)
k6_study(const __grid_constant__ RowTable rows, const int n, const Geom g, const float divisor,
         float* __restrict__ avg, double* __restrict__ parts, unsigned* __restrict__ scratch,
         double* __restrict__ stats) {
  unsigned* const absmax_bits = scratch;      // both zeroed by the launcher
  unsigned* const tickets = scratch + 1;
  constexpr int NACC = NMAX <= 32 ? 32 : 64;
  __shared__ double warp_tot[kStWarps][kMaxN + 1];
  __shared__ unsigned warp_max[kStWarps];
  __shared__ bool last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float acc[NACC];
#pragma unroll
  for (int r = 0; r < NACC; ++r) acc[r] = 0.f;
  float cs = 0.f;               // avg^2 of this thread since the last flush
  unsigned cm = 0;              // max |avg| bit pattern of this thread
  double d0 = 0., d1 = 0., dc = 0.;
  const int64_t stride = (int64_t)gridDim.x * kStThreads;
  // warp-uniform trip count: lanes past the end contribute zeros and still join the shuffles
  const int64_t first = (int64_t)blockIdx.x * kStThreads + warp * 32;
  int pending = 0;
  for (int64_t vf = first; vf < g.nv; vf += stride) {
    const int64_t v = vf + lane;
    const bool live = v < g.nv;
    const int64_t e0 = v * VEC - g.shift;
    const bool full = live && e0 >= 0 && e0 + VEC <= g.d;
    float x[NMAX][VEC];
    if (full) {
#pragma unroll
      for (int r = 0; r < NMAX; ++r)
        if (r < n) VecLoad<VEC>::load(rows.p[r] + e0, x[r]);
    } else {
#pragma unroll
      for (int r = 0; r < NMAX; ++r)
#pragma unroll
        for (int q = 0; q < VEC; ++q) {
          const int64_t e = e0 + q;
          x[r][q] = (r < n && live && e >= 0 && e < g.d) ? __ldcs(rows.p[r] + e) : 0.f;   // out of range: exactly 0
        }
    }
    float a[VEC];
#pragma unroll
    for (int q = 0; q < VEC; ++q) {
      float s = x[0][q];                                     // clone()            :108
#pragma unroll
      for (int r = 1; r < NMAX; ++r)
        if (r < n) s = __fadd_rn(s, x[r][q]);                // add_ in list order  :109-110
      a[q] = __fdiv_rn(s, divisor);                          // div_(len(samples))  :111
      cs = fmaf(a[q], a[q], cs);
      cm = max(cm, __float_as_uint(a[q]) & 0x7fffffffu);
    }
    if (full) VecLoad<VEC>::store(avg + e0, a);
    else {
#pragma unroll
      for (int q = 0; q < VEC; ++q) {
        const int64_t e = e0 + q;
        if (live && e >= 0 && e < g.d) avg[e] = a[q];
      }
    }
#pragma unroll
    for (int r = 0; r < NMAX; ++r)
      if (r < n) {
#pragma unroll
        for (int q = 0; q < VEC; ++q) {
          const float df = __fsub_rn(x[r][q], a[q]);         // grad.sub(grad_avg)  :118
          acc[r] = fmaf(df, df, acc[r]);                     // grad.dot(grad)      :119
        }
      }
    if (++pending == kStFlush) {
      pending = 0;
      d0 += (double)transpose_reduce(*reinterpret_cast<float(*)[32]>(&acc[0]), lane);
      if (NACC > 32) d1 += (double)transpose_reduce(*reinterpret_cast<float(*)[32]>(&acc[NACC - 32]), lane);
      dc += (double)cs;
      cs = 0.f;
#pragma unroll
      for (int r = 0; r < NACC; ++r) acc[r] = 0.f;
    }
  }
  if (pending > 0) {
    d0 += (double)transpose_reduce(*reinterpret_cast<float(*)[32]>(&acc[0]), lane);
    if (NACC > 32) d1 += (double)transpose_reduce(*reinterpret_cast<float(*)[32]>(&acc[NACC - 32]), lane);
    dc += (double)cs;
  }
#pragma unroll
  for (int h = 16; h >= 1; h >>= 1) {
    dc += __shfl_xor_sync(0xffffffffu, dc, h);
    cm = max(cm, __shfl_xor_sync(0xffffffffu, cm, h));
  }
  warp_tot[warp][lane] = d0;
  warp_tot[warp][lane + 32] = d1;
  if (lane == 0) { warp_tot[warp][kMaxN] = dc; warp_max[warp] = cm; }
  __syncthreads();
  double* mine = parts + (size_t)blockIdx.x * (n + 1);
  if (threadIdx.x < n) {
    double s = 0.;
#pragma unroll
    for (int w = 0; w < kStWarps; ++w) s += warp_tot[w][threadIdx.x];
    mine[1 + threadIdx.x] = s;
  } else if (threadIdx.x == kMaxN) {
    double s = 0.;
    unsigned m = 0;
#pragma unroll
    for (int w = 0; w < kStWarps; ++w) { s += warp_tot[w][kMaxN]; m = max(m, warp_max[w]); }
    mine[0] = s;
    if (m != 0) atomicMax(absmax_bits, m);
  }
  // publish this CTA's block, take a ticket; the holder of the last ticket sees every block
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(tickets, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  // Final sum of the gridDim.x blocks by the last CTA.  One thread per entry walking all blocks was a
  // chain of ~gridDim.x / 8 dependent L2 round trips (~20 us at 296 blocks: half of the kernel at
  // d = 1.3M); instead the blocks are split in S interleaved classes, thread (class s, entry c) adds
  // its class in ascending order with all loads in flight, and the S class sums are added in class
  // order: a fixed order for a given grid, every load independent.
  {
    const int width = n + 1;                        // entry 0: sum avg^2; entry 1 + i: deviations of row i
    const int S = kStThreads / width;               // >= 3 (n <= 64)
    const int c = threadIdx.x % width, cls = threadIdx.x / width;
    double* partial = &warp_tot[0][0];              // S * width <= 256 doubles of the (now free) warp table
    if (cls < S) {
      double sum = 0.;
      int p = cls;
      for (; p + 7 * S < (int)gridDim.x; p += 8 * S) {
        double t[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) t[u] = __ldcg(parts + (size_t)(p + u * S) * width + c);
#pragma unroll
        for (int u = 0; u < 8; ++u) sum += t[u];
      }
      for (; p < (int)gridDim.x; p += S) sum += __ldcg(parts + (size_t)p * width + c);
      partial[cls * width + c] = sum;
    }
    __syncthreads();
    if (threadIdx.x < width) {
      double sum = 0.;
      for (int k = 0; k < S; ++k) sum += partial[k * width + threadIdx.x];
      stats[threadIdx.x == 0 ? 0 : 1 + threadIdx.x] = sum;
    } else if (threadIdx.x == kMaxN + 1) {
      stats[1] = (double)__uint_as_float(atomicMax(absmax_bits, 0u));
    }
  }
}

// kMaxN < n <= kMaxNCoordinate (the 128-pointer table), VEC = 1.  A thread keeps its column of up to 128
// values in registers, as k1_sorted<128> does; per-row fp32 accumulators across vectors would need another
// 128 registers, so the squared deviations are instead folded right away, 32 rows at a time: chunk c's
// 32 values go through the transposed warp reduction (an fp32 sum over the warp's 32 coordinates) and
// into fp64, so that lane L ends with rows L, L + 32, L + 64 and L + 96.  avg^2 goes straight into fp64.
// Occupancy by register count (ptxas): up to n = 96 (<= 128 registers) two 256-thread CTAs per SM, above
// (147 / 163 registers) one CTA of 384 threads, 12 warps where 256-thread CTAs would leave 8.
template <int NMAX> __host__ __device__ constexpr int wide_threads() { return NMAX <= 96 ? 256 : 384; }
template <int NMAX> __host__ __device__ constexpr int wide_ctas_per_sm() { return NMAX <= 96 ? 2 : 1; }

template <int NMAX, int VEC>
__global__ void __launch_bounds__(wide_threads<NMAX>(), wide_ctas_per_sm<NMAX>())
k6_study(const __grid_constant__ WideRowTable rows, const int n, const Geom g, const float divisor,
         float* __restrict__ avg, double* __restrict__ parts, unsigned* __restrict__ scratch,
         double* __restrict__ stats) {
  static_assert(VEC == 1 && NMAX > kMaxN && NMAX <= kMaxNCoordinate, "K6 over the wide table: VEC = 1, 64 < NMAX <= 128");
  constexpr int NCH = (NMAX + 31) / 32;
  constexpr int THREADS = wide_threads<NMAX>(), WARPS = THREADS / 32;
  unsigned* const absmax_bits = scratch;      // both zeroed by the launcher
  unsigned* const tickets = scratch + 1;
  __shared__ double warp_tot[WARPS][kMaxNCoordinate + 1];
  __shared__ unsigned warp_max[WARPS];
  __shared__ bool last;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double dr[NCH];
#pragma unroll
  for (int c = 0; c < NCH; ++c) dr[c] = 0.;
  double dc = 0.;
  unsigned cm = 0;
  const int64_t stride = (int64_t)gridDim.x * THREADS;
  // warp-uniform trip count: lanes past the end contribute zeros and still join the shuffles
  const int64_t first = (int64_t)blockIdx.x * THREADS + warp * 32;
  for (int64_t vf = first; vf < g.nv; vf += stride) {
    const int64_t e = vf + lane;                // VEC = 1: no shift
    const bool live = e < g.d;
    float x[NMAX];
#pragma unroll
    for (int r = 0; r < NMAX; ++r) x[r] = (r < n && live) ? __ldcs(rows.p[r] + e) : 0.f;   // out of range: exactly 0
    float s = x[0];                                        // clone()            :108
#pragma unroll
    for (int r = 1; r < NMAX; ++r)
      if (r < n) s = __fadd_rn(s, x[r]);                   // add_ in list order  :109-110
    const float a = __fdiv_rn(s, divisor);                 // div_(len(samples))  :111
    if (live) __stcs(avg + e, a);
    dc = fma((double)a, (double)a, dc);
    cm = max(cm, __float_as_uint(a) & 0x7fffffffu);
    // rows r >= n get values here that nobody reads (study_blocks reads rows [0, n) only)
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      if (c * 32 >= n) continue;                           // warp-uniform
      float v[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        if (c * 32 + j < NMAX) {
          const float df = __fsub_rn(x[c * 32 + j], a);    // grad.sub(grad_avg)  :118
          v[j] = __fmul_rn(df, df);                        // grad.dot(grad)      :119
        } else {
          v[j] = 0.f;
        }
      }
      dr[c] += (double)transpose_reduce(v, lane);
    }
  }
#pragma unroll
  for (int h = 16; h >= 1; h >>= 1) {
    dc += __shfl_xor_sync(0xffffffffu, dc, h);
    cm = max(cm, __shfl_xor_sync(0xffffffffu, cm, h));
  }
#pragma unroll
  for (int c = 0; c < NCH; ++c) warp_tot[warp][c * 32 + lane] = dr[c];
  if (lane == 0) { warp_tot[warp][kMaxNCoordinate] = dc; warp_max[warp] = cm; }
  study_blocks<kMaxNCoordinate, THREADS>(warp_tot, warp_max, last, n, parts, absmax_bits, tickets, stats);
}

template <int NMAX, int VEC>
static void launch_one(const RowTable& rows, int n, const Geom& g, float* avg, double* parts, unsigned* bits,
                       double* stats, unsigned grid, cudaStream_t st) {
  k6_study<NMAX, VEC><<<grid, kStThreads, 0, st>>>(rows, n, g, (float)n, avg, parts, bits, stats);
}

template <int NMAX, int WIDE>
static void launch_bucket(const RowTable& rows, int n, const Geom& g, float* avg, double* parts, unsigned* bits,
                          double* stats, unsigned grid, cudaStream_t st) {
  if (g.vec == WIDE) launch_one<NMAX, WIDE>(rows, n, g, avg, parts, bits, stats, grid, st);
  else               launch_one<NMAX, 1>(rows, n, g, avg, parts, bits, stats, grid, st);
}

void launch_study(const RowTable& rows, int n, const float* const* host_rows, int64_t d, float* avg,
                  double* stats, double* parts, unsigned* bits, cudaStream_t st) {
  // widest vector that keeps the n x VEC values plus the accumulators in registers (on sm_90,
  // 8 < n <= 16 with VEC = 4 spills under the two-CTAs-per-SM bound)
  const int want = n <= 8 ? 4 : n <= 32 ? 2 : 1;
  const Geom g = make_geom(host_rows, n, avg, nullptr, d, want);
  int64_t grid = (g.nv + kStThreads - 1) / kStThreads;
  const int64_t cap = (int64_t)sm_count() * 2;
  if (grid > cap) grid = cap;
  // the partial blocks are n + 1 doubles wide in a buffer sized kMaxParts * n * n
  const int64_t room = n >= 2 ? kMaxParts : kMaxParts / 2;
  if (grid > room) grid = room;
  if (grid < 1) grid = 1;
  cudaMemsetAsync(bits, 0, 2 * sizeof(unsigned), st);      // max |avg| pattern, ticket counter
  const unsigned gr = (unsigned)grid;
  if (n <= 8)       launch_bucket<8, 4>(rows, n, g, avg, parts, bits, stats, gr, st);
  else if (n <= 16) launch_bucket<16, 2>(rows, n, g, avg, parts, bits, stats, gr, st);
  else if (n <= 24) launch_bucket<24, 2>(rows, n, g, avg, parts, bits, stats, gr, st);
  else if (n <= 32) launch_bucket<32, 2>(rows, n, g, avg, parts, bits, stats, gr, st);
  else if (n <= 48) launch_bucket<48, 1>(rows, n, g, avg, parts, bits, stats, gr, st);
  else              launch_bucket<64, 1>(rows, n, g, avg, parts, bits, stats, gr, st);
}

template <int NMAX>
static void launch_wide(const WideRowTable& rows, int n, const Geom& g, float* avg, double* parts, unsigned* bits,
                        double* stats, cudaStream_t st) {
  // as many CTAs as fit at once (the register bound of the bucket).  grid * (n + 1) doubles fit the parts
  // of workspace_bytes(kMaxN) (kMaxParts * kMaxN * kMaxN doubles) many times over.
  constexpr int threads = wide_threads<NMAX>();
  int64_t grid = (g.nv + threads - 1) / threads;
  const int64_t cap = (int64_t)sm_count() * wide_ctas_per_sm<NMAX>();
  if (grid > cap) grid = cap;
  if (grid > kMaxParts) grid = kMaxParts;
  if (grid < 1) grid = 1;
  cudaMemsetAsync(bits, 0, 2 * sizeof(unsigned), st);      // max |avg| pattern, ticket counter
  k6_study<NMAX, 1><<<(unsigned)grid, threads, 0, st>>>(rows, n, g, (float)n, avg, parts, bits, stats);
}

void launch_study(const WideRowTable& rows, int n, const float* const* host_rows, int64_t d, float* avg,
                  double* stats, double* parts, unsigned* bits, cudaStream_t st) {
  const Geom g = make_geom(host_rows, n, avg, nullptr, d, 1);
  if (n <= 80)       launch_wide<80>(rows, n, g, avg, parts, bits, stats, st);
  else if (n <= 96)  launch_wide<96>(rows, n, g, avg, parts, bits, stats, st);
  else if (n <= 112) launch_wide<112>(rows, n, g, avg, parts, bits, stats, st);
  else               launch_wide<128>(rows, n, g, avg, parts, bits, stats, st);
}

}  // namespace bz
