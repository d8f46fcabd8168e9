// reduce.cuh — warp-level helpers shared by K2 and K2'.
#pragma once

#include "common.cuh"

namespace bz {

typedef unsigned long long u64;

// fp32 pairs: two coordinates in one 64-bit register pair.  sm_90 has no packed fp32 arithmetic
// (f32x2), so each helper issues one IEEE-rounded scalar FADD / FMUL / FFMA per lane; the scalar
// pipe already retires 128 fp32 lanes per clock per SM, so nothing is lost against the pair form.
__device__ __forceinline__ u64 pack2(float lo, float hi) {
  return (u64)__float_as_uint(lo) | ((u64)__float_as_uint(hi) << 32);
}
__device__ __forceinline__ void unpack2(u64 v, float& lo, float& hi) {
  lo = __uint_as_float((unsigned)v);
  hi = __uint_as_float((unsigned)(v >> 32));
}
__device__ __forceinline__ u64 sub2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1); unpack2(b, b0, b1);
  return pack2(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
  float a0, a1, b0, b1, c0, c1;
  unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
  return pack2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1); unpack2(b, b0, b1);
  return pack2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  unpack2(a, a0, a1); unpack2(b, b0, b1);
  return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}

// IEEE division of two lanes by a small positive integer m known at compile time (after unrolling),
// without the generic division's reciprocal, range check and slow-path call per lane:
//   y = RN(1/m),  q0 = RN(a*y),  r = a - q0*m (one FMA: exact),  q = RN(q0 + r*y)
// is the correctly rounded a/m for EVERY float a with 2^-100 <= |a| <= FLT_MAX and every m in 1..64:
// checked exhaustively, all 2^32 operands for each m (tools/divcheck.c; what fails outside that range:
// +-inf -> NaN, -0 -> +0, and for even m that are not powers of two the operands below 2^-122, whose
// remainder underflows).  Everything else — zeros, subnormals, inf, NaN — takes the generic division.
constexpr float kDivTiny = 7.888609052210118e-31f;      // 2^-100
__device__ __forceinline__ bool div_fast_ok(float a) {
  return fabsf(a) >= kDivTiny && fabsf(a) <= 3.402823466e+38f;
}
__device__ __forceinline__ float div_small(float a, float m) {
  const float y = 1.f / m;                    // m is a literal after unrolling: folded at compile time (IEEE division, no fast-math)
  const float q0 = __fmul_rn(a, y);
  const float r = __fmaf_rn(-q0, m, a);
  const float q = __fmaf_rn(r, y, q0);
  return div_fast_ok(a) ? q : __fdiv_rn(a, m);
}
__device__ __forceinline__ u64 div_small2(u64 a, float m) {
  const float y = 1.f / m;                    // m is a literal after unrolling: folded at compile time (IEEE division, no fast-math)
  const u64 y2 = pack2(y, y);
  const u64 q0 = mul2(a, y2);
  const u64 r = fma2(q0, pack2(-m, -m), a);
  u64 q = fma2(r, y2, q0);
  float lo, hi;
  unpack2(a, lo, hi);
  if (!(div_fast_ok(lo) && div_fast_ok(hi))) q = pack2(__fdiv_rn(lo, m), __fdiv_rn(hi, m));
  return q;
}
__device__ __forceinline__ float half_sum(u64 v) {
  return __fadd_rn(__uint_as_float((unsigned)(v & 0xffffffffull)), __uint_as_float((unsigned)(v >> 32)));
}


// Transposed warp reduction: on return, lane L holds sum over lanes of v[L] (v has 32 slots).
// The halving step is a template parameter so that every loop below has a constant trip count
// and unrolls fully: a `for (h = 16; h >= 1; h >>= 1)` loop is not always unrolled for sm_90,
// and v[] then lives in local memory.
template <int H>
__device__ __forceinline__ void transpose_step(float (&v)[32], int lane) {
  const bool up = (lane & H) != 0;
#pragma unroll
  for (int j = 0; j < H; ++j) {
    const float send = up ? v[j] : v[j + H];
    const float keep = up ? v[j + H] : v[j];
    v[j] = __fadd_rn(keep, __shfl_xor_sync(0xffffffffu, send, H));
  }
  if constexpr (H > 1) transpose_step<H / 2>(v, lane);
}
__device__ __forceinline__ float transpose_reduce(float (&v)[32], int lane) {
  transpose_step<16>(v, lane);
  return v[0];
}

}  // namespace bz
