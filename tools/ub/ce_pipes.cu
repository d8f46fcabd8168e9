// Microbenchmark: compare-exchange throughput on H100 when the max half of a comparator is
// (a) FMNMX (ALU pipe, like the min), or (b) computed as a + b - min with two IMADs whose
// multipliers live in registers (FMA pipe), for different mixing ratios.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o ce_pipes ce_pipes.cu && ./ce_pipes
#include <cstdio>
#include <cuda_runtime.h>

template <int MODE>
__device__ __forceinline__ void ce(float& a, float& b, int one, int mone, int idx) {
  const float lo = fminf(a, b);
  bool mix = (MODE == 1) || (MODE == 2 && (idx % 3) != 0) || (MODE == 3 && (idx % 2) != 0);
  if (mix) {
    int s, h;
    asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(s) : "r"(__float_as_int(a)), "r"(one), "r"(__float_as_int(b)));
    asm("mad.lo.s32 %0, %1, %2, %3;" : "=r"(h) : "r"(__float_as_int(lo)), "r"(mone), "r"(s));
    b = __int_as_float(h);
  } else {
    b = fmaxf(a, b);
  }
  a = lo;
}

template <int MODE>
__global__ void __launch_bounds__(128) bench(const float* in, float* out, int iters, int one, int mone) {
  float v[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] = in[(blockIdx.x * 128 + threadIdx.x) * 16 + i];
  for (int it = 0; it < iters; ++it) {
    // odd-even transposition rounds on 16 wires: 15 comparators per 2 rounds
    int idx = 0;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
#pragma unroll
      for (int i = 0; i + 1 < 16; i += 2) ce<MODE>(v[i], v[i + 1], one, mone, idx++);
#pragma unroll
      for (int i = 1; i + 1 < 16; i += 2) ce<MODE>(v[i], v[i + 1], one, mone, idx++);
    }
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) out[(blockIdx.x * 128 + threadIdx.x) * 16 + i] = v[i];
}

template <int MODE>
float run(const float* in, float* out, int iters) {
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  bench<MODE><<<132 * 8, 128>>>(in, out, 10, 1, -1);
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  bench<MODE><<<132 * 8, 128>>>(in, out, iters, 1, -1);
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms;
  cudaEventElapsedTime(&ms, a, b);
  return ms;
}

int main() {
  const size_t n = (size_t)132 * 8 * 128 * 16;
  float *in, *out;
  cudaMalloc(&in, n * 4); cudaMalloc(&out, n * 4);
  cudaMemset(in, 0, n * 4);
  const int iters = 2000;
  const double ces = (double)132 * 8 * 128 * iters * 8 * 15;
  const float t0 = run<0>(in, out, iters), t1 = run<1>(in, out, iters), t2 = run<2>(in, out, iters), t3 = run<3>(in, out, iters);
  printf("all FMNMX      : %.3f ms  %.1f G CE/s\n", t0, ces / t0 / 1e6);
  printf("all IMAD max   : %.3f ms  %.1f G CE/s\n", t1, ces / t1 / 1e6);
  printf("2/3 IMAD max   : %.3f ms  %.1f G CE/s\n", t2, ces / t2 / 1e6);
  printf("1/2 IMAD max   : %.3f ms  %.1f G CE/s\n", t3, ces / t3 / 1e6);
  return 0;
}
