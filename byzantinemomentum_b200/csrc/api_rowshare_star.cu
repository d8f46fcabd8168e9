// api_rowshare_star.cu — the C ABI of libbyzagg_star.so (include/byzagg_rowshare_star.h): CGE's candidate-only phase
// A of the d-sharded line search above 64 rows (k2_rowshare_star.cu).  Its error string is its own.  Nothing here
// links against libbyzagg.so or libbyzagg_peers.so: a caller composes the libraries through their C ABIs.
#include <cstdarg>
#include <cstdio>

#include "dist.cuh"
#include "../../include/byzagg_rowshare_star.h"

namespace bz {

int launch_rowshare_star(const float* cand, int n, int c0, int64_t d, int sms, double* parts, unsigned* ticket,
                         double* sums, cudaStream_t st);

static thread_local char g_error[512] = "";

static int star_fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
  return code;
}

// The ticket, then the per-CTA blocks of n doubles (at most kMaxParts of them).
constexpr size_t kStarHeader = 256;
static size_t star_workspace_bytes(int n) {
  if (n < 1) n = 1;
  if (n > kMaxNDistance) n = kMaxNDistance;
  return (kStarHeader + (size_t)kMaxParts * n * sizeof(double) + 255) / 256 * 256;
}

}  // namespace bz

extern "C" {

const char* bz_rowshare_star_last_error(void) { return bz::g_error; }

size_t bz_rowshare_star_workspace_bytes(int n) { return bz::star_workspace_bytes(n); }

int bz_rowshare_star(const float* const* rows, int n, int c0, int64_t d, double* part, void* ws, size_t ws_bytes,
                     void* stream) {
  using namespace bz;
  static const char* who = "bz_rowshare_star";
  if (rows == nullptr) return star_fail(BZ_EINVAL, "%s: rows is NULL", who);
  if (n < 1) return star_fail(BZ_EINVAL, "%s: n = %d, expected n >= 1", who, n);
  if (n <= kMaxN || n > kMaxNDistance)
    return star_fail(BZ_EUNSUPPORTED, "%s: n = %d, expected BZ_MAX_N < n <= BZ_MAX_N_DISTANCE = %d", who, n, kMaxNDistance);
  if (c0 < 1 || c0 >= n) return star_fail(BZ_EINVAL, "%s: c0 = %d, expected 0 < c0 < n = %d", who, c0, n);
  if (d < 0) return star_fail(BZ_EINVAL, "%s: d = %lld < 0", who, (long long)d);
  // an empty shard reads no row: its rows may share any address (every empty tensor may have the same one)
  if (d > 0) {
    for (int r = c0 + 1; r < n; ++r)
      if (rows[r] != rows[c0])
        return star_fail(BZ_EINVAL, "%s: rows[%d] differs from rows[%d]: rows [c0, n) must be one row", who, r, c0);
    for (int r = 0; r < c0; ++r)
      if (rows[r] == rows[c0]) return star_fail(BZ_EINVAL, "%s: rows[%d] is the candidate rows[%d]", who, r, c0);
    for (int r = 0; r < n; ++r) {
      if (rows[r] == nullptr) return star_fail(BZ_EINVAL, "%s: rows[%d] is NULL", who, r);
      if (((uintptr_t)rows[r] % sizeof(float)) != 0) return star_fail(BZ_EINVAL, "%s: rows[%d] is not 4-byte aligned", who, r);
    }
  }
  if (part == nullptr || ((uintptr_t)part % 8) != 0) return star_fail(BZ_EINVAL, "%s: part is NULL or not 8-byte aligned", who);
  const size_t need = star_workspace_bytes(n);
  if (ws == nullptr || ((uintptr_t)ws % 8) != 0 || ws_bytes < need)
    return star_fail(BZ_EWORKSPACE, "%s: workspace of %zu bytes at %p is too small or misaligned (need %zu, 8-byte aligned)",
                     who, ws_bytes, ws, need);
  cudaStream_t st = (cudaStream_t)stream;
  if (d == 0) {
    cudaMemsetAsync(part + c0, 0, (size_t)(n - c0) * sizeof(double), st);
  } else {
    int dev = 0, sms = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    char* base = static_cast<char*>(ws);
    launch_rowshare_star(rows[c0], n, c0, d, sms > 0 ? sms : 132, reinterpret_cast<double*>(base + kStarHeader),
                         reinterpret_cast<unsigned*>(base), part, st);
  }
  const cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return star_fail(BZ_ECUDA, "%s: %s", who, cudaGetErrorString(err));
  return BZ_OK;
}

}  // extern "C"
