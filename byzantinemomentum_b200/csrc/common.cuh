// common.cuh — shared device/host helpers of libbyzagg (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>

#include "../../include/byzagg.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libbyzagg is written for sm_90a (H100) only"
#endif

namespace bz {

constexpr int kMaxN = BZ_MAX_N;

// Host array of n device row pointers, passed BY VALUE as a kernel parameter (512 B in the
// constant bank): no torch.stack, no H2D copy of a pointer table (SURVEY.md §7.2).
struct RowTable {
  const float* p[kMaxN];
};

// Geometry of a launch over d coordinates with VEC per thread.  All rows (and the output)
// share the same misalignment, so shifting the element index by `shift` (0..VEC-1) makes every
// interior vector naturally aligned: logical vector v covers elements [v*VEC - shift,
// v*VEC - shift + VEC) clipped to [0, d).  Only the first and the last vector can be partial;
// they take a scalar load/store path inside the SAME launch (no separate edge kernel).
struct Geom {
  int64_t d;       // coordinates
  int64_t nv;      // logical vectors = ceil((d + shift) / VEC)
  int     shift;   // leading pad, in elements
  int     vec;     // VEC of the launch (host side bookkeeping)
  int     one;     // = 1 and
  int     mone;    // = -1, opaque to the compiler (OpsMix)
  int     reverse; // walk the vectors from the end: the previous pass over the same rows went
                   // forward, so its last ~L2-size bytes are still cached (K3 / K4 / K2' after K2)
};

// Widest usable vector (want_vec, else 1) for these rows / output / optional extra pointer.
Geom make_geom(const float* const* rows, int n, const void* out, const void* extra, int64_t d, int want_vec);

// SM count of the CURRENT device (cached per device; api.cu)
int  sm_count();

// Error plumbing (api.cu)
int  fail(int code, const char* fmt, ...);
int  check_launch(const char* what);

// ---- device helpers ---------------------------------------------------------------------

#ifdef __CUDACC__

template <int VEC> struct VecLoad;
template <> struct VecLoad<4> {
  static __device__ __forceinline__ void load(const float* p, float (&o)[4]) {
    const float4 t = __ldcs(reinterpret_cast<const float4*>(p));
    o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w;
  }
  static __device__ __forceinline__ void store(float* p, const float (&o)[4]) {
    __stcs(reinterpret_cast<float4*>(p), make_float4(o[0], o[1], o[2], o[3]));
  }
};
template <> struct VecLoad<2> {
  static __device__ __forceinline__ void load(const float* p, float (&o)[2]) {
    const float2 t = __ldcs(reinterpret_cast<const float2*>(p));
    o[0] = t.x; o[1] = t.y;
  }
  static __device__ __forceinline__ void store(float* p, const float (&o)[2]) {
    __stcs(reinterpret_cast<float2*>(p), make_float2(o[0], o[1]));
  }
};
template <> struct VecLoad<1> {
  static __device__ __forceinline__ void load(const float* p, float (&o)[1]) { o[0] = __ldcs(p); }
  static __device__ __forceinline__ void store(float* p, const float (&o)[1]) { __stcs(p, o[0]); }
};

// Load the N x VEC values of the logical vector starting at element e0 of every row.  The
// full / partial decision is taken ONCE around the whole batch so that the N loads of the
// common (full) case stay back to back in the instruction stream (one branch, N independent
// LDG in flight).  Partial vectors (e0 < 0 or e0 + VEC > d) read out-of-range lanes as 0.
template <int N, int VEC>
__device__ __forceinline__ void load_rows(const RowTable& rows, int64_t e0, int64_t d, bool full, float (&x)[VEC][N]) {
  if (full) {
#pragma unroll
    for (int r = 0; r < N; ++r) {
      float t[VEC];
      VecLoad<VEC>::load(rows.p[r] + e0, t);
#pragma unroll
      for (int c = 0; c < VEC; ++c) x[c][r] = t[c];
    }
  } else {
#pragma unroll
    for (int r = 0; r < N; ++r) {
#pragma unroll
      for (int c = 0; c < VEC; ++c) {
        const int64_t e = e0 + c;
        x[c][r] = (e >= 0 && e < d) ? __ldcs(rows.p[r] + e) : 0.f;
      }
    }
  }
}

// Single-row variant (K3): same semantics.
template <int VEC>
__device__ __forceinline__ void load_vec(const float* row, int64_t e0, int64_t d, bool full, float (&o)[VEC]) {
  if (full) {
    VecLoad<VEC>::load(row + e0, o);
  } else {
#pragma unroll
    for (int c = 0; c < VEC; ++c) {
      const int64_t e = e0 + c;
      o[c] = (e >= 0 && e < d) ? __ldcs(row + e) : 0.f;
    }
  }
}
template <int VEC>
__device__ __forceinline__ void store_vec(float* out, int64_t e0, int64_t d, bool full, const float (&o)[VEC]) {
  if (full) {
    VecLoad<VEC>::store(out + e0, o);
  } else {
#pragma unroll
    for (int c = 0; c < VEC; ++c) {
      const int64_t e = e0 + c;
      if (e >= 0 && e < d) __stcs(out + e, o[c]);
    }
  }
}

// ---- cp.async (LDGSTS) helpers -------------------------------------------------------------
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int K> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(K) : "memory"); }

// Copy VEC floats global -> shared (both naturally aligned to 4·VEC bytes).
template <int VEC>
__device__ __forceinline__ void cp_async_vec(float* smem, const float* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  if (VEC == 4)      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem) : "memory");
  else if (VEC == 2) asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(s), "l"(gmem) : "memory");
  else               asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gmem) : "memory");
}
template <int VEC>
__device__ __forceinline__ void lds_vec(const float* smem, float (&o)[VEC]) {
  if (VEC == 4) {
    const float4 t = *reinterpret_cast<const float4*>(smem);
    o[0] = t.x; o[1] = t.y; o[VEC > 2 ? 2 : 0] = t.z; o[VEC > 3 ? 3 : 0] = t.w;
  } else if (VEC == 2) {
    const float2 t = *reinterpret_cast<const float2*>(smem);
    o[0] = t.x; o[VEC > 1 ? 1 : 0] = t.y;
  } else {
    o[0] = *smem;
  }
}

// Compare-exchange policies for SortNet<N>::run(ops, v): ops.ce<K>(a, b) leaves min in a, max in b
// (K = index of the comparator in the generated network).
// Fast: inputs hold no NaN (plain FMNMX).
struct OpsFast {
  template <int K> __device__ __forceinline__ void ce(float& a, float& b) const {
    const float lo = fminf(a, b), hi = fmaxf(a, b);
    a = lo; b = hi;
  }
};
// Mixed pipes, finite inputs only.  FMNMX issues on the ALU pipe at one warp instruction every
// two cycles; a comparator is two of them.  For the comparators selected by `Mask` the max half
// is instead computed on the bit patterns as a + b - min (exact: min is bitwise one of the two
// inputs, so the other one comes out) with two IMADs, which issue on the FMA pipe at the same
// rate.  `one` / `mone` are 1 and -1 passed as kernel parameters so that ptxas cannot fold
// the multiply-adds back into an ALU-pipe IADD3 (tools/ub/ce_pipes.cu compares the mixes).
// NOT valid with NaN inputs (FMNMX then returns neither input) nor under flush-to-zero.
template <class Mask>
struct OpsMix {
  int one, mone;
  template <int K> __device__ __forceinline__ void ce(float& a, float& b) const {
    const float lo = fminf(a, b);
    if constexpr (Mask::mix(K)) {
      int s, h;
      asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(s) : "r"(__float_as_int(a)), "r"(one), "r"(__float_as_int(b)));
      asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(h) : "r"(__float_as_int(lo)), "r"(mone), "r"(s));
      b = __int_as_float(h);
    } else {
      b = fmaxf(a, b);
    }
    a = lo;
  }
};
// NaN-propagating (FMNMX.NAN): a NaN input poisons every output that depends on it, which
// is exactly torch's `median(dim)` semantics (median.py:39 with torch >= 1.7).
struct OpsNaNProp {
  template <int K> __device__ __forceinline__ void ce(float& a, float& b) const {
    float lo, hi;
    asm("min.NaN.f32 %0, %1, %2;" : "=f"(lo) : "f"(a), "f"(b));
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(hi) : "f"(a), "f"(b));
    a = lo; b = hi;
  }
};
// Total order on keys: signed-int image of the float order with every NaN mapped to INT_MAX
// (NaN sorts last, like `Tensor.sort` / `topk(largest=False)`).
struct OpsKey {
  template <int K> __device__ __forceinline__ void ce(int& a, int& b) const {
    const int lo = min(a, b), hi = max(a, b);
    a = lo; b = hi;
  }
};
// Same pipe split as OpsMix, on integer keys (exact for every input: no NaN caveat).
template <class Mask>
struct OpsKeyMix {
  int one, mone;
  template <int K> __device__ __forceinline__ void ce(int& a, int& b) const {
    const int lo = min(a, b);
    if constexpr (Mask::mix(K)) {
      int s, h;
      asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(s) : "r"(a), "r"(one), "r"(b));
      asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(h) : "r"(lo), "r"(mone), "r"(s));
      b = h;
    } else {
      b = max(a, b);
    }
    a = lo;
  }
};
__device__ __forceinline__ int float_to_key(float x) {
  int k = __float_as_int(x);
  k ^= (k >> 31) & 0x7fffffff;
  return (x != x) ? 0x7fffffff : k;
}
__device__ __forceinline__ float key_to_float(int k) {
  k ^= (k >> 31) & 0x7fffffff;
  return __int_as_float(k);   // INT_MAX -> 0x7fffffff, a quiet NaN
}
// |x| as an integer whose order is the order of |x| with NaN largest.
__device__ __forceinline__ int abs_key(float x) { return __float_as_int(x) & 0x7fffffff; }

__device__ __forceinline__ float quiet_nan() { return __int_as_float(0x7fc00000); }

#endif  // __CUDACC__

}  // namespace bz
