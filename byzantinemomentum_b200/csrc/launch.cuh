// launch.cuh — internal launch entry points shared between the kernel translation units
// and api.cu.
#pragma once

#include "common.cuh"

namespace bz {

// Programmatic dependent launch (PDL): the kernel may be scheduled as soon as the CTAs of the
// previous kernel of the stream have exited or triggered, instead of after the whole grid has
// drained and the launch latency has been paid again; it MUST execute pdl_wait() before it
// reads or writes anything global (the wait returns once the previous grid has completed and its
// writes are visible).  Used for the second pass of the distance rules (K3 / K4 after K2 + scoring).
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// In the PRIMARY kernel, at its start: dependents launched with `launch_after` may be scheduled as soon as
// SM resources free up (they still block in pdl_wait() until this whole grid has completed and flushed).
// Used by K1 (back-to-back calls of the coordinate-wise rules); the distance pass does not trigger early.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif
template <class... Params, class... Args>
inline cudaError_t launch_after(void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, Params(args)...);
}

// Elements per thread in the aligned body of a K1 launch: 4 (LDG.128) while 4n values fit
// the register file comfortably, else 2 (LDG.64).  The scalar variant (1) serves the
// unaligned head/tail and rows whose alignments disagree.
__host__ __device__ constexpr int body_vec(int n) { return n <= 28 ? 4 : 2; }

// Epilogue of k1_sorted.
enum SortedMode { kModeTrmean = 0, kModePhocas = 1, kModeMeamed = 2 };

// K1 (k1_inst.cu, 9 parts).  Parts 0-7 return false when n is outside the part's range;
// launch_trmean_special returns false when (n, f) has no compile-time specialisation.
bool launch_median_part0(int n, const RowTable& rows, const Geom& g, float* out, cudaStream_t st);
bool launch_median_part1(int n, const RowTable& rows, const Geom& g, float* out, cudaStream_t st);
bool launch_median_part2(int n, const RowTable& rows, const Geom& g, float* out, cudaStream_t st);
bool launch_median_part3(int n, const RowTable& rows, const Geom& g, float* out, cudaStream_t st);
bool launch_sorted_part4(int n, const RowTable& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st);
bool launch_sorted_part5(int n, const RowTable& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st);
bool launch_sorted_part6(int n, const RowTable& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st);
bool launch_sorted_part7(int n, const RowTable& rows, const Geom& g, int mode, int f, float* out, cudaStream_t st);
bool launch_trmean_special(int n, int f, const RowTable& rows, const Geom& g, float* out, cudaStream_t st);
bool launch_phocas_special(int n, int f, const RowTable& rows, const Geom& g, float* out, cudaStream_t st);
bool launch_meamed_special(int n, int f, const RowTable& rows, const Geom& g, float* out, cudaStream_t st);

// K3 (k3_average.cu): ordered-subset average.
void launch_average(const RowTable& rows, const Geom& g, const int32_t* sel, int count,
                    int zero_init, float divisor, const int32_t* status, float* out, cudaStream_t st);

}  // namespace bz
