// k7_gradient.cu — K7: the per-worker gradient production of attack.py:776-780 / 791-795 (clip,
// clone) and :799-810 (momentum placement) in ONE pass per gradient, written straight into the rows
// the aggregation rules read (SURVEY.md §8(f) row 2).
//
// The reference, per worker: `grad.norm().item()` (a pass + a host sync), `grad.mul_(clip / norm)`
// (read + write), `grad.clone()` (read + write), then for worker-side momentum
// `gmtm.mul_(mu).add_(grad, alpha=1 - dampening)` (two more read-modify-write passes) — 7 vector
// passes and a synchronisation.  Here: [clip only] one read for the squared norm (fp64 partials,
// last-CTA ticket, the scale factor stays on the device), then one kernel that reads the gradient
// (and the momentum vector) once and writes the sampled row and the momentum / honest row.
//
// Arithmetic (fp32, exactly the ATen operator sequence; `fl` = round to fp32):
//   scale  = norm > clip ? fl(clip / norm) : (no multiplication)      attack.py:777-779 (Python double division)
//   g'     = fl(g * scale)                                            grad.mul_(scalar)
//   worker: m <- fma(fl(alpha), g', fl(m * fl(mu)))                   gmtm.mul_(mu).add_(grad, alpha=1-dampening)  :802
//   server: h  = fma(fl(mu), s, fl(g' * fl(alpha)))                   grad.mul(1-dampening).add_(server, alpha=mu) :807
// (`a + alpha * b` is one fused multiply-add in ATen's CPU and CUDA add kernels alike.)
// The norm is the fp32 rounding of the square root of an fp64 sum: ATen's own fp32 reduction order
// differs between builds, so `scale` may differ from the reference's by 1 ulp when clipping occurs.
// A sum past FLT_MAX gives norm = +inf as ATen's fp32 accumulator does, hence scale = 0 (a zero row).
//
// k7_scatter is the same clip + clone for a d-sharded trainer (bz_gradient_scatter, byzagg_shards.h):
// instead of one sampled row it writes column range [lo_r, hi_r) of the clipped gradient into rank r's
// slot, for every rank r, with the bits of k7_produce's sampled row.
#include "dist.cuh"
#include "launch.cuh"

namespace bz {

constexpr int kGrThreads = 256;

__global__ void __launch_bounds__(kGrThreads)
k7_sqnorm(const float* __restrict__ g, const int64_t d, const double clip, double* __restrict__ parts,
          unsigned* __restrict__ ticket, float* __restrict__ scale_out) {
  __shared__ double warp_sum[kGrThreads / 32];
  __shared__ bool last;
  double s = 0.;
  for (int64_t i = (int64_t)blockIdx.x * kGrThreads + threadIdx.x; i < d; i += (int64_t)gridDim.x * kGrThreads) {
    const double x = (double)__ldg(g + i);
    s = fma(x, x, s);
  }
#pragma unroll
  for (int h = 16; h >= 1; h >>= 1) s += __shfl_xor_sync(0xffffffffu, s, h);
  if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.;
#pragma unroll
    for (int w = 0; w < kGrThreads / 32; ++w) t += warp_sum[w];
    parts[blockIdx.x] = t;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x != 0) return;
  __threadfence();
  double total = 0.;
  for (int p = 0; p < (int)gridDim.x; ++p) total += __ldcg(parts + p);      // index order: deterministic
  const float norm = fp32_norm(total);                                      // Tensor.norm() is an fp32 value (+inf on overflow: scale 0)
  // attack.py:778-779: `if grad_norm > clip: grad.mul_(clip / grad_norm)` — the quotient is a Python double
  // handed to mul_ as a scalar, i.e. rounded to fp32; NaN norms compare false: no scaling
  *scale_out = ((double)norm > clip) ? (float)(clip / (double)norm) : 1.f;
  *ticket = 0u;
}

// mode 0: sampled only; 1: worker-side momentum (m in/out); 2: server-side momentum (m = server vector, read only)
template <int MODE>
__global__ void __launch_bounds__(kGrThreads)
k7_produce(const float* __restrict__ g, const int64_t d, const float* __restrict__ scale_ptr, float* __restrict__ sampled,
           float* __restrict__ m, const float mu, const float alpha, float* __restrict__ honest) {
  const int64_t i = (int64_t)blockIdx.x * kGrThreads + threadIdx.x;
  if (i >= d) return;
  pdl_wait();
  float x = __ldcs(g + i);
  if (scale_ptr != nullptr) {
    const float sc = *scale_ptr;
    if (sc != 1.f) x = __fmul_rn(x, sc);           // the reference does not multiply at all when it does not clip
  }
  if (sampled != nullptr) __stcs(sampled + i, x);
  if (MODE == 1) {
    const float t = __fmul_rn(m[i], mu);
    m[i] = __fmaf_rn(alpha, x, t);
  } else if (MODE == 2) {
    const float t = __fmul_rn(x, alpha);
    honest[i] = __fmaf_rn(mu, __ldg(m + i), t);
  }
}

// The destination slot of each rank, passed BY VALUE as a kernel parameter (like RowTable).
struct SlotTable {
  float* p[BZ_MAX_PEERS];
};

// Grid: x strides over the ceil(per / 4) vectors of 4 columns of a shard, y is the rank.  Rank r's
// shard is [lo, lo + len) with lo = min(d, r * per), len = min(d, lo + per) - lo (sharded.shard_bounds).
// The slot starts 16-byte aligned; the shard's first column generally does not (lo is not a multiple
// of 4, or the gradient itself is only 4-byte aligned), so a misaligned shard and the partial last
// vector read their columns one by one (L1-cached: the warp's four loads share the same lines).
__global__ void __launch_bounds__(kGrThreads)
k7_scatter(const float* __restrict__ g, const int64_t d, const int64_t per, const float* __restrict__ scale_ptr,
           const __grid_constant__ SlotTable dest) {             // indexed in place in the parameter bank, no local copy
  const int r = blockIdx.y;
  const int64_t lo = min(d, (int64_t)r * per);
  const int64_t len = min(d, lo + per) - lo;
  const float* src = g + lo;
  float* out = dest.p[r];
  const bool aligned = (reinterpret_cast<uintptr_t>(src) & 15) == 0;
  pdl_wait();
  float sc = 1.f;
  if (scale_ptr != nullptr && len > 0) sc = *scale_ptr;
  for (int64_t k = ((int64_t)blockIdx.x * kGrThreads + threadIdx.x) * 4; k < len; k += (int64_t)gridDim.x * kGrThreads * 4) {
    const bool full = k + 4 <= len;
    float x[4];
    if (full && aligned) {
      const float4 t = __ldcs(reinterpret_cast<const float4*>(src + k));
      x[0] = t.x; x[1] = t.y; x[2] = t.z; x[3] = t.w;
    } else {
#pragma unroll
      for (int c = 0; c < 4; ++c) x[c] = (k + c < len) ? __ldg(src + k + c) : 0.f;
    }
    if (sc != 1.f) {                                // the reference does not multiply at all when it does not clip
#pragma unroll
      for (int c = 0; c < 4; ++c) x[c] = __fmul_rn(x[c], sc);
    }
    if (full) {
      *reinterpret_cast<float4*>(out + k) = make_float4(x[0], x[1], x[2], x[3]);
    } else {
#pragma unroll
      for (int c = 0; c < 4; ++c)
        if (k + c < len) out[k + c] = x[c];
    }
  }
  // the slots may be another GPU's memory: order this CTA's stores before whatever the stream does next
  // (a barrier that tells the owner its rows have arrived)
  __syncthreads();
  if (threadIdx.x == 0) __threadfence_system();
}

// Row tables of k7_momentum, passed BY VALUE and read in place (__grid_constant__).
struct MomentumTables {
  const float* rows[kMaxN];     // the clipped rows
  float* mom[kMaxN];            // MODE 1: the momentum vectors, updated in place
  float* honest[kMaxN];         // MODE 2: the honest rows written
};

// The momentum placement of k7_produce (MODE 1 / 2, the same per-coordinate arithmetic) for n rows
// in ONE launch: grid y is the row, x strides over the d coordinates, four at a time with 16-byte
// accesses when the row's vectors (and `server`, MODE 2) are all 16-byte aligned, else one at a time.
template <int MODE>
__device__ __forceinline__ float momentum_step(const float x, float* __restrict__ m_or_h, const float* __restrict__ server,
                                               const int64_t i, const float mu, const float alpha) {
  if (MODE == 1) {
    const float u = __fmul_rn(m_or_h[i], mu);
    return __fmaf_rn(alpha, x, u);
  }
  const float u = __fmul_rn(x, alpha);
  return __fmaf_rn(mu, __ldg(server + i), u);
}

template <int MODE>
__global__ void __launch_bounds__(kGrThreads)
k7_momentum(const int64_t d, const float* __restrict__ server, const float mu, const float alpha,
            const __grid_constant__ MomentumTables t) {
  const int r = blockIdx.y;
  const float* __restrict__ g = t.rows[r];
  float* __restrict__ out = MODE == 1 ? t.mom[r] : t.honest[r];
  const bool vec = ((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(out) |
                     (MODE == 2 ? reinterpret_cast<uintptr_t>(server) : 0)) & 15) == 0;
  const int64_t stride = (int64_t)gridDim.x * kGrThreads;
  int64_t head = 0;                                // coordinates done by the vector loop
  pdl_wait();
  if (vec) {
    const int64_t nv = d / 4;
    for (int64_t v = (int64_t)blockIdx.x * kGrThreads + threadIdx.x; v < nv; v += stride) {
      const float4 x = __ldcs(reinterpret_cast<const float4*>(g) + v);
      float4 y;
      if (MODE == 1) {
        const float4 m = reinterpret_cast<const float4*>(out)[v];
        y = make_float4(__fmaf_rn(alpha, x.x, __fmul_rn(m.x, mu)), __fmaf_rn(alpha, x.y, __fmul_rn(m.y, mu)),
                        __fmaf_rn(alpha, x.z, __fmul_rn(m.z, mu)), __fmaf_rn(alpha, x.w, __fmul_rn(m.w, mu)));
      } else {
        const float4 c = __ldg(reinterpret_cast<const float4*>(server) + v);
        y = make_float4(__fmaf_rn(mu, c.x, __fmul_rn(x.x, alpha)), __fmaf_rn(mu, c.y, __fmul_rn(x.y, alpha)),
                        __fmaf_rn(mu, c.z, __fmul_rn(x.z, alpha)), __fmaf_rn(mu, c.w, __fmul_rn(x.w, alpha)));
      }
      reinterpret_cast<float4*>(out)[v] = y;
    }
    head = nv * 4;
  }
  for (int64_t i = head + (int64_t)blockIdx.x * kGrThreads + threadIdx.x; i < d; i += stride)
    out[i] = momentum_step<MODE>(__ldcs(g + i), out, server, i, mu, alpha);
}

}  // namespace bz

using namespace bz;

// The clip scale of a gradient on the device (k7_sqnorm into the workspace): *scale = NULL when
// clip <= 0, i.e. no multiplication.
static int launch_clip_scale(const float* grad, int64_t d, double clip, void* ws, size_t ws_bytes, cudaStream_t st,
                             const char* who, const float** scale) {
  *scale = nullptr;
  if (!(clip > 0.)) return BZ_OK;
  Workspace w;
  if (!carve_workspace(ws, ws_bytes, 1, w)) return fail(BZ_EWORKSPACE, "%s: workspace too small or misaligned", who);
  int64_t grid = (d + (int64_t)kGrThreads * 8 - 1) / ((int64_t)kGrThreads * 8);
  const int64_t cap = (int64_t)sm_count() * 4;
  if (grid > cap) grid = cap;
  if (grid > kMaxParts) grid = kMaxParts;
  if (grid < 1) grid = 1;
  float* scale_dev = reinterpret_cast<float*>(w.status);
  cudaMemsetAsync(w.ticket, 0, sizeof(unsigned), st);
  k7_sqnorm<<<(unsigned)grid, kGrThreads, 0, st>>>(grad, d, clip, w.parts, w.ticket, scale_dev);
  if (int rc = check_launch("k7_sqnorm")) return rc;
  *scale = scale_dev;
  return BZ_OK;
}

extern "C" int bz_gradient_row(const float* grad, int64_t d, double clip, float* sampled, int mode, float* momentum,
                               double mu, double alpha, float* honest, void* ws, size_t ws_bytes, void* stream) {
  if (grad == nullptr || d < 0) return fail(BZ_EINVAL, "bz_gradient_row: grad is NULL or d < 0");
  if (mode < 0 || mode > 2) return fail(BZ_EINVAL, "bz_gradient_row: mode = %d", mode);
  if (mode != 0 && momentum == nullptr) return fail(BZ_EINVAL, "bz_gradient_row: momentum is NULL");
  if (mode == 2 && honest == nullptr) return fail(BZ_EINVAL, "bz_gradient_row: honest is NULL");
  if (mode == 0 && sampled == nullptr) return fail(BZ_EINVAL, "bz_gradient_row: nothing to write");
  if (d == 0) return BZ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const float* scale;
  if (int rc = launch_clip_scale(grad, d, clip, ws, ws_bytes, st, "bz_gradient_row", &scale)) return rc;
  const unsigned blocks = (unsigned)((d + kGrThreads - 1) / kGrThreads);
  const float fmu = (float)mu, falpha = (float)alpha;
  cudaError_t err;
  if (mode == 1)      err = launch_after(k7_produce<1>, blocks, kGrThreads, 0, st, grad, d, scale, sampled, momentum, fmu, falpha, honest);
  else if (mode == 2) err = launch_after(k7_produce<2>, blocks, kGrThreads, 0, st, grad, d, scale, sampled, momentum, fmu, falpha, honest);
  else                err = launch_after(k7_produce<0>, blocks, kGrThreads, 0, st, grad, d, scale, sampled, momentum, fmu, falpha, honest);
  (void)err;
  return check_launch("k7_produce");
}

extern "C" int bz_gradient_scatter(const float* grad, int64_t d, double clip, int nranks, float* const* dest,
                                   void* ws, size_t ws_bytes, void* stream) {
  if (grad == nullptr || d < 0) return fail(BZ_EINVAL, "bz_gradient_scatter: grad is NULL or d < 0");
  if (nranks < 1 || nranks > BZ_MAX_PEERS) return fail(BZ_EINVAL, "bz_gradient_scatter: nranks = %d, expected 1..%d", nranks, BZ_MAX_PEERS);
  if (dest == nullptr) return fail(BZ_EINVAL, "bz_gradient_scatter: dest is NULL");
  const int64_t per = (d + nranks - 1) / nranks;
  SlotTable slots = {};
  for (int r = 0; r < nranks; ++r) {
    const int64_t lo = d < r * per ? d : r * per;
    const int64_t hi = d < lo + per ? d : lo + per;
    if (hi > lo && dest[r] == nullptr) return fail(BZ_EINVAL, "bz_gradient_scatter: dest[%d] is NULL", r);
    if (hi > lo && (uintptr_t)dest[r] % 16 != 0) return fail(BZ_EINVAL, "bz_gradient_scatter: dest[%d] is not 16-byte aligned", r);
    slots.p[r] = dest[r];
  }
  if (d == 0) return BZ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const float* scale;
  if (int rc = launch_clip_scale(grad, d, clip, ws, ws_bytes, st, "bz_gradient_scatter", &scale)) return rc;
  // a few waves of CTAs over all the ranks, each striding over its shard: one system fence per CTA
  int64_t blocks = (per + (int64_t)kGrThreads * 4 - 1) / ((int64_t)kGrThreads * 4);
  const int64_t cap = ((int64_t)sm_count() * 8 + nranks - 1) / nranks;
  if (blocks > cap) blocks = cap;
  cudaError_t err = launch_after(k7_scatter, dim3((unsigned)blocks, (unsigned)nranks), kGrThreads, 0, st, grad, d, per, scale, slots);
  (void)err;
  return check_launch("k7_scatter");
}

extern "C" int bz_gradient_momentum(const float* const* rows, int n, int64_t d, int mode, float* const* momentum,
                                    const float* server, double mu, double alpha, float* const* honest, void* stream) {
  if (rows == nullptr || d < 0) return fail(BZ_EINVAL, "bz_gradient_momentum: rows is NULL or d < 0");
  if (n < 1 || n > BZ_MAX_N) return fail(BZ_EINVAL, "bz_gradient_momentum: n = %d, expected 1..%d", n, BZ_MAX_N);
  if (mode != 1 && mode != 2) return fail(BZ_EINVAL, "bz_gradient_momentum: mode = %d, expected 1 or 2", mode);
  if (mode == 1 && momentum == nullptr) return fail(BZ_EINVAL, "bz_gradient_momentum: momentum is NULL");
  if (mode == 2 && honest == nullptr) return fail(BZ_EINVAL, "bz_gradient_momentum: honest is NULL");
  if (d == 0) return BZ_OK;                        // an empty shard: its vectors may all be at address 0
  if (mode == 2 && server == nullptr) return fail(BZ_EINVAL, "bz_gradient_momentum: server is NULL");
  MomentumTables t = {};
  for (int i = 0; i < n; ++i) {
    if (rows[i] == nullptr) return fail(BZ_EINVAL, "bz_gradient_momentum: rows[%d] is NULL", i);
    t.rows[i] = rows[i];
    if (mode == 1) {
      if (momentum[i] == nullptr) return fail(BZ_EINVAL, "bz_gradient_momentum: momentum[%d] is NULL", i);
      for (int j = 0; j < i; ++j)                  // updated in place: one vector twice would race with itself
        if (momentum[j] == momentum[i]) return fail(BZ_EINVAL, "bz_gradient_momentum: momentum[%d] and momentum[%d] are the same vector", j, i);
      t.mom[i] = momentum[i];
    } else {
      if (honest[i] == nullptr) return fail(BZ_EINVAL, "bz_gradient_momentum: honest[%d] is NULL", i);
      t.honest[i] = honest[i];
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  int64_t blocks = (d + 4 * kGrThreads - 1) / (4 * kGrThreads);
  const int64_t cap = ((int64_t)sm_count() * 16 + n - 1) / n;       // two waves of 8 CTAs per SM over all rows
  if (blocks > cap) blocks = cap;
  const dim3 grid((unsigned)blocks, (unsigned)n);
  const float fmu = (float)mu, falpha = (float)alpha;
  cudaError_t err = mode == 1 ? launch_after(k7_momentum<1>, grid, kGrThreads, 0, st, d, server, fmu, falpha, t)
                              : launch_after(k7_momentum<2>, grid, kGrThreads, 0, st, d, server, fmu, falpha, t);
  (void)err;
  return check_launch("k7_momentum");
}
