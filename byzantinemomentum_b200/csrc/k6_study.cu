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
#include "dist.cuh"
#include "reduce.cuh"

namespace bz {

constexpr int kStThreads = 256;
constexpr int kStWarps = kStThreads / 32;
constexpr int kStFlush = 8;      // vectors between two flushes (<= 32 terms per fp32 accumulator)

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

}  // namespace bz
