// k1_inst.cu — instantiations of the K1 kernels for a range of n, compiled once per part
// (`-DBZ_PART=<0..26>`) so that the kernels build in parallel.  Parts 0-3: k1_median for n in
// 1-16 / 17-32 / 33-48 / 49-64; parts 4-7: generic k1_sorted for the same ranges; parts 8-10:
// trimmed mean / phocas / meamed with (n, f) fixed at compile time for n = 11, 25, 51.
// Parts 11-26 (bz_coordinate above 64 rows, VEC = 1): k1_median (11-18) and generic k1_sorted
// (19-26) for n in 65-72 / 73-80 / ... / 121-128.
#include "k1_select.cuh"

#ifndef BZ_PART
#error "compile with -DBZ_PART=<0..26>"
#endif

#if BZ_PART >= 11
#include "networks_wide_gen.cuh"
#define BZ_WIDE_BASE (65 + 8 * ((BZ_PART - 11) % 8))
#define BZ_N_LIST X(BZ_WIDE_BASE) X(BZ_WIDE_BASE + 1) X(BZ_WIDE_BASE + 2) X(BZ_WIDE_BASE + 3) \
                  X(BZ_WIDE_BASE + 4) X(BZ_WIDE_BASE + 5) X(BZ_WIDE_BASE + 6) X(BZ_WIDE_BASE + 7)
#elif (BZ_PART % 4) == 0
#define BZ_N_LIST X(1) X(2) X(3) X(4) X(5) X(6) X(7) X(8) X(9) X(10) X(11) X(12) X(13) X(14) X(15) X(16)
#elif (BZ_PART % 4) == 1
#define BZ_N_LIST X(17) X(18) X(19) X(20) X(21) X(22) X(23) X(24) X(25) X(26) X(27) X(28) X(29) X(30) X(31) X(32)
#elif (BZ_PART % 4) == 2
#define BZ_N_LIST X(33) X(34) X(35) X(36) X(37) X(38) X(39) X(40) X(41) X(42) X(43) X(44) X(45) X(46) X(47) X(48)
#else
#define BZ_N_LIST X(49) X(50) X(51) X(52) X(53) X(54) X(55) X(56) X(57) X(58) X(59) X(60) X(61) X(62) X(63) X(64)
#endif

namespace bz {

// One CTA per tile of kK1Threads vectors.  The closest modes' sorted columns may need more than
// 48 KB of shared memory: opted in once per kernel instantiation and device.
template <class K>
static unsigned tile_grid(K kernel, size_t smem, int64_t nv, unsigned long long& opted) {
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (smem > 48 * 1024 && !(opted & bit)) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    opted |= bit;
  }
  return (unsigned)((nv + kK1Threads - 1) / kK1Threads);
}

#if BZ_PART >= 19

template <int N>
static void launch_sorted_wide_n(const WideRowTable& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  if (g.nv <= 0) return;
  // the closest modes stage the sorted columns in shared memory (64 KB per CTA at n = 128)
  static unsigned long long opted = 0;
  const size_t smem = (mode == kModeTrmean) ? 0 : Stage<N, 1>::kColumnFloats * sizeof(float);
  const auto kernel = k1_sorted_fn<N, 1, -1, -1>();
  launch_after(kernel, tile_grid(kernel, smem, g.nv, opted), kK1Threads, smem, st, rows, g, mode, f, out);
}

#define BZ_FN2(p) launch_sorted_wide_part##p
#define BZ_FN(p) BZ_FN2(p)
bool BZ_FN(BZ_PART)(int n, const WideRowTable& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  switch (n) {
#define X(N) case N: launch_sorted_wide_n<N>(rows, g, mode, f, out, st); return true;
    BZ_N_LIST
#undef X
    default: return false;
  }
}

#elif BZ_PART >= 11

template <int N>
static void launch_median_wide_n(const WideRowTable& rows, const Geom& g, float* out, cudaStream_t st) {
  if (g.nv <= 0) return;
  static unsigned long long opted = 0;
  const auto kernel = k1_median_fn<N, 1>();
  launch_after(kernel, tile_grid(kernel, 0, g.nv, opted), kK1Threads, 0, st, rows, g, out);
}

#define BZ_FN2(p) launch_median_wide_part##p
#define BZ_FN(p) BZ_FN2(p)
bool BZ_FN(BZ_PART)(int n, const WideRowTable& rows, const Geom& g, float* out, cudaStream_t st) {
  switch (n) {
#define X(N) case N: launch_median_wide_n<N>(rows, g, out, st); return true;
    BZ_N_LIST
#undef X
    default: return false;
  }
}

#elif BZ_PART < 4

template <int N>
static void launch_median_n(const RowTable& rows, const Geom& g, float* out, cudaStream_t st) {
  if (g.nv <= 0) return;
  static unsigned long long opted = 0;
  if (g.vec == 1)
    launch_after(k1_median_fn<N, 1>(), tile_grid(k1_median_fn<N, 1>(), 0, g.nv, opted), kK1Threads, 0, st, rows, g, out);
  else
    launch_after(k1_median_fn<N, body_vec(N)>(), tile_grid(k1_median_fn<N, body_vec(N)>(), 0, g.nv, opted), kK1Threads, 0, st, rows, g, out);
}

#define BZ_FN2(p) launch_median_part##p
#define BZ_FN(p) BZ_FN2(p)
bool BZ_FN(BZ_PART)(int n, const RowTable& rows, const Geom& g, float* out, cudaStream_t st) {
  switch (n) {
#define X(N) case N: launch_median_n<N>(rows, g, out, st); return true;
    BZ_N_LIST
#undef X
    default: return false;
  }
}

#elif BZ_PART < 8

template <int N, int VEC>
static void launch_sorted_nv(const RowTable& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  if (g.nv <= 0) return;
  // the closest modes stage the sorted columns in shared memory
  static unsigned long long opted = 0;
  const size_t smem = (mode == kModeTrmean) ? 0 : Stage<N, VEC>::kColumnFloats * sizeof(float);
  launch_after(k1_sorted_fn<N, VEC, -1, -1>(), tile_grid(k1_sorted_fn<N, VEC, -1, -1>(), smem, g.nv, opted), kK1Threads, smem, st, rows, g, mode, f, out);
}

template <int N>
static void launch_sorted_n(const RowTable& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  if (g.vec == 1) launch_sorted_nv<N, 1>(rows, g, mode, f, out, st);
  else            launch_sorted_nv<N, body_vec(N)>(rows, g, mode, f, out, st);
}

#define BZ_FN2(p) launch_sorted_part##p
#define BZ_FN(p) BZ_FN2(p)
bool BZ_FN(BZ_PART)(int n, const RowTable& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  switch (n) {
#define X(N) case N: launch_sorted_n<N>(rows, g, mode, f, out, st); return true;
    BZ_N_LIST
#undef X
    default: return false;
  }
}

#else

// n of BASELINE.json's configs and of the reference's grids (reproduce.py:122-209,
// reproduce-appendix.py:122-158), every valid f: trimmed mean with the network pruned at compile time.
#define BZ_NF_LIST \
  Y(11, 1) Y(11, 2) Y(11, 3) Y(11, 4) Y(11, 5) \
  Y(25, 1) Y(25, 2) Y(25, 3) Y(25, 4) Y(25, 5) Y(25, 6) Y(25, 7) Y(25, 8) Y(25, 9) Y(25, 10) Y(25, 11) Y(25, 12) \
  Y(51, 1) Y(51, 2) Y(51, 3) Y(51, 4) Y(51, 5) Y(51, 6) Y(51, 7) Y(51, 8) Y(51, 9) Y(51, 10) Y(51, 11) Y(51, 12) Y(51, 13) \
  Y(51, 14) Y(51, 15) Y(51, 16) Y(51, 17) Y(51, 18) Y(51, 19) Y(51, 20) Y(51, 21) Y(51, 22) Y(51, 23) Y(51, 24) Y(51, 25)

#if BZ_PART == 8
#define BZ_SPECIAL_MODE kModeTrmean
#define BZ_SPECIAL_FN launch_trmean_special
#elif BZ_PART == 9
#define BZ_SPECIAL_MODE kModePhocas
#define BZ_SPECIAL_FN launch_phocas_special
#else
#define BZ_SPECIAL_MODE kModeMeamed
#define BZ_SPECIAL_FN launch_meamed_special
#endif

template <int N, int F>
static void launch_special_nf(const RowTable& rows, const Geom& g, float* out, cudaStream_t st) {
  if (g.nv <= 0) return;
  static unsigned long long opted = 0;
  launch_after(k1_sorted_fn<N, body_vec(N), F, BZ_SPECIAL_MODE>(), tile_grid(k1_sorted_fn<N, body_vec(N), F, BZ_SPECIAL_MODE>(), 0, g.nv, opted), kK1Threads, 0, st, rows, g, BZ_SPECIAL_MODE, F, out);
}

bool BZ_SPECIAL_FN(int n, int f, const RowTable& rows, const Geom& g, float* out, cudaStream_t st) {
  if (g.vec == 1) return false;   // unaligned rows take the generic scalar kernel
#define Y(N, F) if (n == N && f == F) { launch_special_nf<N, F>(rows, g, out, st); return true; }
  BZ_NF_LIST
#undef Y
  return false;
}

#endif

}  // namespace bz
