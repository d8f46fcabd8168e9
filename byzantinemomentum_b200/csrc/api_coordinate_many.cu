// api_coordinate_many.cu — the C ABI of libbyzagg_many.so (include/byzagg_coordinate_many.h): the coordinate-wise
// rules for up to 1024 rows.  Above 128 rows it launches the kernels of k1_many.cu; up to 128 it calls libbyzagg.so's
// bz_coordinate (this library links against it), so those calls are bz_coordinate's launches.  libbyzagg.so keeps
// exactly its own kernels, and this library keeps its own error string.
#include <cstdarg>
#include <cstdio>

#include "launch.cuh"

namespace bz {

// k1_many.cu
void launch_many_sorted(const ManyRowTable& rows, int n, int64_t d, int rule, int f, int sms, float* out, cudaStream_t st);
void launch_many_average(const ManyRowTable& rows, const Geom& g, int n, float* out, cudaStream_t st);

static thread_local char g_error[512] = "";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
  return code;
}

int check_launch(const char* what) {
  const cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return fail(BZ_ECUDA, "%s: %s", what, cudaGetErrorString(err));
  return BZ_OK;
}

static int many_sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  int& c = cached[dev & 63];
  if (c == 0) cudaDeviceGetAttribute(&c, cudaDevAttrMultiProcessorCount, dev);
  return c > 0 ? c : 132;
}

// The vector width of the average and the alignment shift all rows and the output share (api.cu's make_geom, whose
// definition lives in libbyzagg.so).
Geom make_geom(const float* const* rows, int n, const void* out, const void* extra, int64_t d, int want_vec) {
  Geom g{d, d, 0, 1, 1, -1, 0};
  if (want_vec <= 1 || d < 1) return g;
  const uintptr_t bytes = (uintptr_t)want_vec * sizeof(float);
  const uintptr_t mis = (uintptr_t)rows[0] % bytes;
  bool same = ((uintptr_t)out % bytes) == mis;
  if (extra != nullptr) same = same && ((uintptr_t)extra % bytes) == mis;
  for (int r = 1; r < n && same; ++r) same = ((uintptr_t)rows[r] % bytes) == mis;
  if (!same) return g;
  g.vec = want_vec;
  g.shift = (int)(mis / sizeof(float));
  g.nv = (d + g.shift + want_vec - 1) / want_vec;
  return g;
}

// bz_coordinate's checks, with the limit BZ_MAX_N_MANY.
static int check_many(int rule, const float* const* rows, int n, int f, int64_t d, const void* out) {
  const char* who = "bz_coordinate_many";
  if (rule < BZ_RULE_AVERAGE || rule > BZ_RULE_MEAMED) return fail(BZ_EINVAL, "%s: unknown rule %d", who, rule);
  if (rows == nullptr) return fail(BZ_EINVAL, "%s: rows is NULL", who);
  if (n < 1) return fail(BZ_EINVAL, "%s: n = %d, expected n >= 1", who, n);
  if (n > kMaxNMany) return fail(BZ_EUNSUPPORTED, "%s: n = %d exceeds BZ_MAX_N_MANY = %d", who, n, kMaxNMany);
  if (d < 0) return fail(BZ_EINVAL, "%s: d = %lld < 0", who, (long long)d);
  if (d > 0) {
    if (out == nullptr) return fail(BZ_EINVAL, "%s: output pointer is NULL", who);
    for (int r = 0; r < n; ++r) {
      if (rows[r] == nullptr) return fail(BZ_EINVAL, "%s: rows[%d] is NULL", who, r);
      if (((uintptr_t)rows[r] % sizeof(float)) != 0) return fail(BZ_EINVAL, "%s: rows[%d] is not 4-byte aligned", who, r);
    }
    if (((uintptr_t)out % sizeof(float)) != 0) return fail(BZ_EINVAL, "%s: output is not 4-byte aligned", who);
  }
  if (rule >= BZ_RULE_TRMEAN && (f < 0 || n - 2 * f < 1))
    return fail(BZ_EINVAL, "%s: f = %d not executable with n = %d (need n - 2f >= 1)", who, f, n);
  return BZ_OK;
}

}  // namespace bz

using namespace bz;

extern "C" {

const char* bz_coordinate_many_last_error(void) { return g_error; }

int bz_coordinate_many(int rule, const float* const* rows, int n, int f, int64_t d, float* out, void* stream) {
  if (int rc = check_many(rule, rows, n, f, d, out)) return rc;
  if (d == 0) return BZ_OK;
  if (n <= kMaxNCoordinate) {
    const int rc = bz_coordinate(rule, rows, n, f, d, out, stream);
    if (rc != BZ_OK) fail(rc, "%s", bz_last_error());
    return rc;
  }
  ManyRowTable t;
  for (int r = 0; r < kMaxNMany; ++r) t.p[r] = rows[r < n ? r : 0];
  const cudaStream_t st = (cudaStream_t)stream;
  if (rule == BZ_RULE_AVERAGE) {
    launch_many_average(t, make_geom(rows, n, out, nullptr, d, 4), n, out, st);
    return check_launch("k3_many_average");
  }
  launch_many_sorted(t, n, d, rule, f, many_sm_count(), out, st);
  return check_launch("k1_many");
}

}  // extern "C"
