// k1_inst.cu — instantiations of the K1 kernels, compiled once per family and range of n so that
// the kernels build in parallel (the Makefile names each object after what it holds):
//   -DBZ_MEDIAN_FROM=<first n>   k1_median for every n of the range
//   -DBZ_SORTED_FROM=<first n>   generic k1_sorted for every n of the range
//   -DBZ_SPECIAL=<0..2>          trimmed mean / phocas / meamed with (n, f) fixed at compile time for n = 11, 25, 51
// A range is 16 sizes up to kMaxN rows and 8 above (VEC = 1, networks_wide_gen.cuh).
#include "k1_select.cuh"

#if defined(BZ_MEDIAN_FROM)
#define BZ_FIRST BZ_MEDIAN_FROM
#elif defined(BZ_SORTED_FROM)
#define BZ_FIRST BZ_SORTED_FROM
#elif !defined(BZ_SPECIAL)
#error "compile with -DBZ_MEDIAN_FROM=<first n>, -DBZ_SORTED_FROM=<first n> or -DBZ_SPECIAL=<0..2>"
#endif

#ifdef BZ_FIRST
#define BZ_N8(b) X((b)) X((b) + 1) X((b) + 2) X((b) + 3) X((b) + 4) X((b) + 5) X((b) + 6) X((b) + 7)
#if BZ_FIRST > BZ_MAX_N
#include "networks_wide_gen.cuh"
#define BZ_N_LIST BZ_N8(BZ_FIRST)
#else
#define BZ_N_LIST BZ_N8(BZ_FIRST) BZ_N8(BZ_FIRST + 8)
#endif
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

#if defined(BZ_MEDIAN_FROM)

template <int N>
static void launch_median_n(const RowsOf<N>& rows, const Geom& g, float* out, cudaStream_t st) {
  if (g.nv <= 0) return;
  static unsigned long long opted = 0;
  if (g.vec == 1)
    launch_after(k1_median_fn<N, 1>(), tile_grid(k1_median_fn<N, 1>(), 0, g.nv, opted), kK1Threads, 0, st, rows, g, out);
  else
    launch_after(k1_median_fn<N, body_vec(N)>(), tile_grid(k1_median_fn<N, body_vec(N)>(), 0, g.nv, opted), kK1Threads, 0, st, rows, g, out);
}

template <int FIRST>
bool launch_median_range(int n, const RowsOf<FIRST>& rows, const Geom& g, float* out, cudaStream_t st) {
  switch (n) {
#define X(N) case N: launch_median_n<N>(rows, g, out, st); return true;
    BZ_N_LIST
#undef X
    default: return false;
  }
}
template bool launch_median_range<BZ_FIRST>(int, const RowsOf<BZ_FIRST>&, const Geom&, float*, cudaStream_t);

#elif defined(BZ_SORTED_FROM)

template <int N, int VEC>
static void launch_sorted_nv(const RowsOf<N>& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  if (g.nv <= 0) return;
  // the closest modes stage the sorted columns in shared memory (64 KB per CTA at n = 128)
  static unsigned long long opted = 0;
  const size_t smem = (mode == kModeTrmean) ? 0 : Stage<N, VEC>::kColumnFloats * sizeof(float);
  launch_after(k1_sorted_fn<N, VEC, -1, -1>(), tile_grid(k1_sorted_fn<N, VEC, -1, -1>(), smem, g.nv, opted), kK1Threads, smem, st, rows, g, mode, f, out);
}

template <int N>
static void launch_sorted_n(const RowsOf<N>& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  if (g.vec == 1) launch_sorted_nv<N, 1>(rows, g, mode, f, out, st);
  else            launch_sorted_nv<N, body_vec(N)>(rows, g, mode, f, out, st);
}

template <int FIRST>
bool launch_sorted_range(int n, const RowsOf<FIRST>& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st) {
  switch (n) {
#define X(N) case N: launch_sorted_n<N>(rows, g, mode, f, out, st); return true;
    BZ_N_LIST
#undef X
    default: return false;
  }
}
template bool launch_sorted_range<BZ_FIRST>(int, const RowsOf<BZ_FIRST>&, const Geom&, int, int, float*, cudaStream_t);

#else

// n of BASELINE.json's configs and of the reference's grids (reproduce.py:122-209,
// reproduce-appendix.py:122-158), every valid f: trimmed mean with the network pruned at compile time.
#define BZ_NF_LIST \
  Y(11, 1) Y(11, 2) Y(11, 3) Y(11, 4) Y(11, 5) \
  Y(25, 1) Y(25, 2) Y(25, 3) Y(25, 4) Y(25, 5) Y(25, 6) Y(25, 7) Y(25, 8) Y(25, 9) Y(25, 10) Y(25, 11) Y(25, 12) \
  Y(51, 1) Y(51, 2) Y(51, 3) Y(51, 4) Y(51, 5) Y(51, 6) Y(51, 7) Y(51, 8) Y(51, 9) Y(51, 10) Y(51, 11) Y(51, 12) Y(51, 13) \
  Y(51, 14) Y(51, 15) Y(51, 16) Y(51, 17) Y(51, 18) Y(51, 19) Y(51, 20) Y(51, 21) Y(51, 22) Y(51, 23) Y(51, 24) Y(51, 25)

#if BZ_SPECIAL == 0
#define BZ_SPECIAL_MODE kModeTrmean
#define BZ_SPECIAL_FN launch_trmean_special
#elif BZ_SPECIAL == 1
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
