// k4_many.cu — the reduces of the distance rules above kMaxNDistance rows (bz_distance_many), over the 1024-pointer
// table of the n original rows.
//
// K3-many: K3's ordered-subset average (k3_average.cuh) taking an order array: Multi-Krum's and Aksel's
// ((0 + g0) + g1) + ... / count, CGE's clone-then-add form.
//
// K4-many: Bulyan's reduce with k4_bulyan_wide's per-column contract, which tests/bulyan_columns.py restates:
//   * the m_max = n - f - 2 best-scored rows in score order, staged for kBmCols adjacent columns in shared memory;
//   * the theta = n - 2f - 2 window means in the reference's order (bulyan.py:66-70): window i summed from its own
//     first row, (0 + s[i]) + s[i + 1] + ..., then divided by m_i = min(m, m_max - i).  A thread takes kBmWindows
//     adjacent windows of one column and adds each staged value it reads into every window that holds it, each
//     window still in its own order, so that one shared-memory load feeds up to kBmWindows adds.  Bit parity with
//     those per-window sums rules out prefix sums: a column costs sum_i m_i fp32 adds (261,888 at n = 1024,
//     f = 255), the FP32 floor of this kernel;
//   * the theta keys of a column sorted by one warp with K1-many's bitonic sort (buckets of 256, 512 and 1024 keys,
//     padded with INT_MAX, which sorts after every real key, NaN included);
//   * the lower median (NaN when the column holds a NaN), the window of the beta = theta - 2f closest values that
//     starts right after the last strict gain, its sum in fp64 rounded once to fp32, one fp32 division by beta.
// A non-zero status word (Bulyan's degenerate case) makes the output NaN.
#include <climits>

#include "distance_many.cuh"
#include "bitonic.cuh"
#include "k3_average.cuh"

namespace bz {

template <int VEC>
__global__ void __launch_bounds__(kK3Threads)
k3_average_many(const __grid_constant__ ManyRowTable rows, const Geom g, const int32_t* __restrict__ sel, const int count,
                const int zero_init, const float divisor, float* __restrict__ out) {
  k3_average_body<VEC>(rows, g, sel, count, zero_init, divisor, nullptr, out);
}

void launch_average_many(const ManyRowTable& rows, const Geom& g, const int32_t* sel, int count, int zero_init,
                         float divisor, float* out, cudaStream_t st) {
  typedef void (*Kernel)(ManyRowTable, Geom, const int32_t*, int, int, float, float*);
  if (g.nv <= 0) return;
  const unsigned blocks = (unsigned)((g.nv + kK3Threads - 1) / kK3Threads);
  const Kernel kernel = (g.vec == 4) ? Kernel(k3_average_many<4>) : (g.vec == 2) ? Kernel(k3_average_many<2>)
                                                                                 : Kernel(k3_average_many<1>);
  kernel<<<blocks, kK3Threads, 0, st>>>(rows, g, sel, count, zero_init, divisor, out);
}

// ---- K4-many ---------------------------------------------------------------------------------------------------

constexpr int kBmThreads = 256;
constexpr int kBmWarps = kBmThreads / 32;
constexpr int kBmCols = 16;                          // columns per CTA
constexpr int kBmLd = 18;                            // floats per staged row: the two half-warps, kBmWindows rows
                                                     // apart, read distinct banks
constexpr int kBmWindows = 8;                        // windows per thread

// Shared memory of bucket P for m_max staged rows: the order, the rows [m_max][kBmLd], the keys [kBmCols][LD]
// (room for the skewed ranks; odd, so that the columns start in distinct banks).
template <int P>
struct BulyanTile {
  static constexpr int K = P / 32;
  static constexpr int LD = P + P / 32 + 1;
  static size_t smem(int m_max) {
    return (size_t)kMaxNMany * sizeof(int) + (size_t)m_max * kBmLd * sizeof(float) + (size_t)kBmCols * LD * sizeof(int);
  }
};

template <int P>
__global__ void __launch_bounds__(kBmThreads, 1)
k4_bulyan_many(const __grid_constant__ ManyRowTable rows, const int64_t d, const int n, const int f, const int m,
               const int32_t* __restrict__ order, const int32_t* __restrict__ status, float* __restrict__ out) {
  using T = BulyanTile<P>;
  extern __shared__ __align__(16) unsigned char sm_bm[];
  const int m_max = n - f - 2, theta = n - 2 * f - 2, beta = theta - 2 * f;
  int* sel = reinterpret_cast<int*>(sm_bm);
  float* col = reinterpret_cast<float*>(sm_bm + kMaxNMany * sizeof(int));
  int* keys = reinterpret_cast<int*>(col + m_max * kBmLd);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t e0 = (int64_t)blockIdx.x * kBmCols;
  if (status != nullptr && *status != 0) {
    if (tid < kBmCols && e0 + tid < d) out[e0 + tid] = quiet_nan();
    return;
  }
  for (int k = tid; k < m_max; k += kBmThreads) sel[k] = order[k];
  __syncthreads();
  // The m_max best-scored rows of these columns, in score order: row k, column c at col[k * kBmLd + c]
  for (int q = tid; q < m_max * kBmCols; q += kBmThreads) {
    const int k = q / kBmCols, c = q % kBmCols;
    col[k * kBmLd + c] = (e0 + c < d) ? __ldcs(rows.p[sel[k]] + e0 + c) : 0.f;
  }
  __syncthreads();
  // Stage 1: selected[i] = sum(gradients at sorted positions i .. i + m_i - 1).div_(m_i)  (bulyan.py:66-70).  Window
  // it0 + w holds the rows [it0 + w, end[w]), end[w] = min(it0 + w + m, m_max): non-decreasing in w, so from row
  // it0 + kBmWindows - 1 to end[0] every window takes the row, before and after only some do.
  const int groups = (theta + kBmWindows - 1) / kBmWindows;
  for (int t = tid; t < groups * kBmCols; t += kBmThreads) {
    const int it0 = (t / kBmCols) * kBmWindows, c = t % kBmCols;
    const float* x = col + c;
    int end[kBmWindows];
    float acc[kBmWindows];
#pragma unroll
    for (int w = 0; w < kBmWindows; ++w) {
      end[w] = min(it0 + w + m, m_max);
      acc[w] = 0.f;                                    // (0 + s[i]) + s[i + 1] + ...
    }
    const int all = it0 + kBmWindows - 1, last = end[kBmWindows - 1];
    for (int k = it0; k < min(all, last); ++k) {
      const float v = x[k * kBmLd];
#pragma unroll
      for (int w = 0; w < kBmWindows; ++w)
        if (k >= it0 + w && k < end[w]) acc[w] = __fadd_rn(acc[w], v);
    }
#pragma unroll 4
    for (int k = all; k < end[0]; ++k) {
      const float v = x[k * kBmLd];
#pragma unroll
      for (int w = 0; w < kBmWindows; ++w) acc[w] = __fadd_rn(acc[w], v);
    }
    for (int k = max(all, end[0]); k < last; ++k) {
      const float v = x[k * kBmLd];
#pragma unroll
      for (int w = 0; w < kBmWindows; ++w)
        if (k < end[w]) acc[w] = __fadd_rn(acc[w], v);
    }
#pragma unroll
    for (int w = 0; w < kBmWindows; ++w)
      if (it0 + w < theta) keys[c * T::LD + it0 + w] = float_to_key(__fdiv_rn(acc[w], (float)(end[w] - it0 - w)));
  }
  __syncthreads();
  // Stage 2 (bulyan.py:78-84): each warp takes the columns warp and warp + kBmWarps.  It sorts a column's theta keys
  // (rank r written at skew(r)), takes the lower median, and finds the window of the beta closest values, which
  // starts right after the last strict gain (see k4_bulyan): every lane scans its share of the theta - beta
  // candidate starts and the warp keeps the largest.  Lane j then adds column j's window in fp64, in ascending
  // order, and rounds the sum once, as K4-wide does; the fp32 rounding keeps the reference's overflow to +-inf.
  static_assert(kBmCols == 2 * kBmWarps, "two columns per warp");
  float med0 = 0.f, med1 = 0.f;                        // scalars, not arrays: a runtime index would need a stack
  int lstar0 = 0, lstar1 = 0;
#pragma unroll 1
  for (int j = 0; j < 2; ++j) {
    int* kc = keys + (warp + kBmWarps * j) * T::LD;
    int v[T::K];
#pragma unroll
    for (int q = 0; q < T::K; ++q) {
      const int r = q * 32 + lane;
      v[q] = (r < theta) ? kc[r] : INT_MAX;
    }
    __syncwarp();
    warp_bitonic<T::K>(v, lane);
#pragma unroll
    for (int q = 0; q < T::K; ++q) kc[skew(lane * T::K + q)] = v[q];
    __syncwarp();
    const float last = key_to_float(kc[skew(theta - 1)]);
    const float mj = (last != last) ? quiet_nan() : key_to_float(kc[skew((theta - 1) / 2)]);
    int gain = 0;
    for (int l = lane; l < theta - beta; l += 32) {
      const int dlo = abs_key(__fsub_rn(key_to_float(kc[skew(l)]), mj));
      const int dhi = abs_key(__fsub_rn(key_to_float(kc[skew(l + beta)]), mj));
      if (dlo > dhi) gain = l + 1;
    }
    const int lj = __reduce_max_sync(0xffffffffu, gain);
    if (j == 0) { med0 = mj; lstar0 = lj; }
    else        { med1 = mj; lstar1 = lj; }
  }
  if (lane < 2) {
    const int c = warp + kBmWarps * lane;
    if (e0 + c < d) {
      const int* kc = keys + c * T::LD;
      const float mj = lane ? med1 : med0;
      const int lj = lane ? lstar1 : lstar0;
      double acc = 0.;
      for (int q = 0; q < beta; ++q) acc += (double)key_to_float(kc[skew(lj + q)]);
      const float r = __fdiv_rn(__double2float_rn(acc), (float)beta);
      out[e0 + c] = (mj != mj) ? quiet_nan() : r;
    }
  }
}

template <int P>
static void launch_bulyan_bucket(const ManyRowTable& rows, int n, int f, int m, const int32_t* order,
                                 const int32_t* status, int64_t d, float* out, cudaStream_t st) {
  using T = BulyanTile<P>;
  static unsigned long long opted = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(opted & bit)) {
    cudaFuncSetAttribute(k4_bulyan_many<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T::smem(kMaxNMany - 2));
    opted |= bit;
  }
  const unsigned blocks = (unsigned)((d + kBmCols - 1) / kBmCols);
  k4_bulyan_many<P><<<blocks, kBmThreads, T::smem(n - f - 2), st>>>(rows, d, n, f, m, order, status, out);
}

void launch_bulyan_many(const ManyRowTable& rows, int n, int f, int m, const int32_t* order, const int32_t* status,
                        int64_t d, float* out, cudaStream_t st) {
  if (d <= 0) return;
  const int theta = n - 2 * f - 2;
  if (theta <= 256)      launch_bulyan_bucket<256>(rows, n, f, m, order, status, d, out, st);
  else if (theta <= 512) launch_bulyan_bucket<512>(rows, n, f, m, order, status, d, out, st);
  else                   launch_bulyan_bucket<1024>(rows, n, f, m, order, status, d, out, st);
}

}  // namespace bz
