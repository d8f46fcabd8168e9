// api_distance_many.cu — the C ABI of libbyzagg_many_distance.so (include/byzagg_distance_many.h): Multi-Krum,
// Bulyan, Aksel and CGE for up to 1024 rows.  Up to kMaxNDistance rows it calls libbyzagg.so's bz_distance; above,
// the kernels of k2_many.cu, k5_many.cu and k4_many.cu, and for Aksel's centre libbyzagg_many.so's
// bz_coordinate_many.  This library links against both and keeps its own error string; they keep exactly their
// kernels.
#include <cstdarg>
#include <cstdio>

#include "distance_many.cuh"
#include "../../include/byzagg_distance_many.h"
#include "../../include/byzagg_distance_many_table.h"

namespace bz {

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

// A failed call of the other libraries: its code, with its message copied here.
static int forward(int rc, const char* message) {
  if (rc != BZ_OK) fail(rc, "%s", message);
  return rc;
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

static size_t round256(size_t bytes) { return (bytes + 255) / 256 * 256; }

// The workspace above kMaxNDistance rows: the tickets and the status word in the first 256 bytes, the order and the
// scores of the rows, the u x u table of squared distances, then the blocks of K2-many (whose share K2'-many's
// kMaxRowParts x n sums also fit in).  Never less than bz_distance's at kMaxNDistance rows, so that the size at
// kMaxNMany serves every n.
constexpr size_t kOffStatus = 128;
constexpr size_t kOffOrder = 256;
constexpr size_t kOffScores = kOffOrder + kMaxNMany * sizeof(int32_t);
constexpr size_t kOffTable = kOffScores + kMaxNMany * sizeof(double);
static_assert(kOffTable % 256 == 0, "the table starts 256-byte aligned");
static_assert(kOffTable == BZ_DISTANCE_MANY_TABLE_OFFSET, "byzagg_distance_many_table.h states the table's offset");
static_assert((size_t)kMaxRowParts * kMaxNMany <= (size_t)kMaxPairBlocks * kPairBlock, "K2'-many's blocks fit");

static size_t many_distance_bytes(int n) {
  if (n <= BZ_MAX_N_DISTANCE) return bz_distance_workspace_bytes(n);
  const size_t own = round256(kOffTable + (size_t)n * n * sizeof(double)) + (size_t)kMaxPairBlocks * kPairBlock * sizeof(double);
  const size_t below = bz_distance_workspace_bytes(BZ_MAX_N_DISTANCE);
  return own > below ? own : below;
}

// The rule, the row count, the rows and the output: bz_distance's checks with the limit BZ_MAX_N_MANY, and `out` must
// not overlap a row.
static int check_call(int rule, const float* const* rows, int n, int64_t d, const float* out, const char* who) {
  if (rule < BZ_RULE_KRUM || rule > BZ_RULE_CGE) return fail(BZ_EINVAL, "%s: unknown rule %d", who, rule);
  if (n < 1) return fail(BZ_EINVAL, "%s: n = %d, expected n >= 1", who, n);
  if (n > kMaxNMany) return fail(BZ_EUNSUPPORTED, "%s: n = %d exceeds BZ_MAX_N_MANY = %d", who, n, kMaxNMany);
  if (rule == BZ_RULE_BRUTE && n > BZ_MAX_N)
    return fail(BZ_EUNSUPPORTED, "%s: brute takes n <= BZ_MAX_N = %d rows, got %d", who, BZ_MAX_N, n);
  if (rows == nullptr) return fail(BZ_EINVAL, "%s: rows is NULL", who);
  if (d < 0) return fail(BZ_EINVAL, "%s: d = %lld < 0", who, (long long)d);
  if (d == 0) return BZ_OK;
  if (out == nullptr) return fail(BZ_EINVAL, "%s: output pointer is NULL", who);
  for (int r = 0; r < n; ++r) {
    if (rows[r] == nullptr) return fail(BZ_EINVAL, "%s: rows[%d] is NULL", who, r);
    if (((uintptr_t)rows[r] % sizeof(float)) != 0) return fail(BZ_EINVAL, "%s: rows[%d] is not 4-byte aligned", who, r);
  }
  if (((uintptr_t)out % sizeof(float)) != 0) return fail(BZ_EINVAL, "%s: output is not 4-byte aligned", who);
  for (int r = 0; r < n; ++r)
    if (out < rows[r] + d && rows[r] < out + d) return fail(BZ_EINVAL, "%s: the output overlaps rows[%d]", who, r);
  return BZ_OK;
}

// bz_distance's verdicts on f, m and mode above kMaxNDistance rows (api_shared.cuh's rule_tail and aksel_count):
// `count` is the rule's scoring count (Multi-Krum n - f - 1, Bulyan m) or Aksel's number of averaged rows.
static int check_rule(int rule, int n, int f, int m, int mode, int& count, const char* who) {
  count = 0;
  if (rule == BZ_RULE_KRUM) {
    if (f < 0 || n - f - 1 < 1) return fail(BZ_EINVAL, "%s: f = %d not executable with n = %d (need n - f - 1 >= 1)", who, f, n);
    if (m < 1 || m > n) return fail(BZ_EINVAL, "%s: m = %d, expected 1..%d", who, m, n);
    count = n - f - 1;
  } else if (rule == BZ_RULE_BULYAN) {
    const int theta = n - 2 * f - 2, beta = theta - 2 * f, m_max = n - f - 2;
    if (f < 0 || theta < 1 || beta < 1) return fail(BZ_EINVAL, "%s: f = %d not executable with n = %d (need n >= 4f + 3)", who, f, n);
    if (m < 1 || m > m_max) return fail(BZ_EINVAL, "%s: m = %d, expected 1..%d", who, m, m_max);
    count = m;
  } else if (rule == BZ_RULE_AKSEL) {
    if (mode != BZ_AKSEL_MID && mode != BZ_AKSEL_NF) return fail(BZ_EINVAL, "%s: mode = %d", who, mode);
    count = (mode == BZ_AKSEL_MID) ? (n + 1) / 2 : n - f;
    if (count < 1 || count > n) return fail(BZ_EINVAL, "%s: f = %d not executable with n = %d", who, f, n);
  }
  return BZ_OK;
}

// The rows CGE sums (api_dist.inc's cge_count; cge.py:59-70 does not validate f, `normed[1:m]` with m = n - f <= 0 is
// a Python slice), divided by n - f.
static int cge_count(int n, int f) {
  const int m = n - f;
  int count = m;
  if (m == 0) count = 1;
  else if (m < 0) count = n + m;
  if (count > n) count = n;
  if (count < 1) count = 1;
  return count;
}

// The unique rows of the call (dedupe_many) and the map of the original rows to them.
static int alias_map(const float* const* rows, int n, ManyRowTable& ut, ManyAliasMap& map) {
  const float* uniq[kMaxNMany];
  const int u = dedupe_many(rows, n, uniq, map.to_unique);
  for (int i = n; i < kMaxNMany; ++i) map.to_unique[i] = 0;
  for (int k = 0; k < kMaxNMany; ++k) ut.p[k] = uniq[k < u ? k : 0];
  return u;
}

// "Select" of Multi-Krum or Bulyan above kMaxNDistance rows: K5-many from the u x u table the workspace holds, then
// the average of the m selected rows or K4-many.  The ticket is zero on entry.
static int run_select(int rule, const float* const* rows, int n, int f, int m, int count, int64_t d, float* out,
                      int32_t* order, int32_t* status, char* ws, const ManyAliasMap& map, int u, cudaStream_t st) {
  const bool bulyan = rule == BZ_RULE_BULYAN;
  unsigned* ticket = reinterpret_cast<unsigned*>(ws);
  int32_t* ord = order != nullptr ? order : reinterpret_cast<int32_t*>(ws + kOffOrder);
  int32_t* stat = !bulyan ? nullptr : status != nullptr ? status : reinterpret_cast<int32_t*>(ws + kOffStatus);
  double* scores = reinterpret_cast<double*>(ws + kOffScores);
  const double* table = reinterpret_cast<const double*>(ws + kOffTable);
  launch_select_many(table, map, n, u, count, scores, ord, stat, f, m, bulyan ? 1 : 0, ticket, st);
  if (int rc = check_launch("k5_select_many")) return rc;
  ManyRowTable t;
  for (int r = 0; r < kMaxNMany; ++r) t.p[r] = rows[r < n ? r : 0];
  if (bulyan) {
    launch_bulyan_many(t, n, f, m, ord, stat, d, out, st);
    return check_launch("k4_bulyan_many");
  }
  launch_average_many(t, make_geom(rows, n, out, nullptr, d, 4), ord, m, 1, (float)m, out, st);
  return check_launch("k3_average_many");
}

// Multi-Krum or Bulyan above kMaxNDistance rows, after the checks: "pairs" (K2-many over the unique rows into the
// table), then "select".
static int run_pairwise(int rule, const float* const* rows, int n, int f, int m, int count, int64_t d, float* out,
                        int32_t* order, int32_t* status, char* ws, cudaStream_t st) {
  ManyRowTable ut;
  ManyAliasMap map;
  const int u = alias_map(rows, n, ut, map);
  unsigned* ticket = reinterpret_cast<unsigned*>(ws);
  double* table = reinterpret_cast<double*>(ws + kOffTable);
  double* parts = reinterpret_cast<double*>(ws + round256(kOffTable + (size_t)n * n * sizeof(double)));   // 16-byte stores
  cudaMemsetAsync(ticket, 0, sizeof(unsigned), st);
  if (int rc = check_launch("memset")) return rc;
  launch_pairdist_many(ut, u, d, pair_grid(u, d), parts, table, st);
  if (int rc = check_launch("k2_pairdist_many")) return rc;
  return run_select(rule, rows, n, f, m, count, d, out, order, status, ws, map, u, st);
}

// Aksel or CGE above kMaxNDistance rows, after the checks: Aksel's centre is bz_coordinate_many's median written into
// `out` (aksel.py:39; the average overwrites it later, in stream order), K2'-many with the selection in its last
// CTA, the average of the `count` rows (Aksel) or CGE's sum divided by n - f.
static int run_rowkeys(int rule, const float* const* rows, int n, int f, int count, int64_t d, float* out,
                       int32_t* order, char* ws, cudaStream_t st) {
  const bool aksel = rule == BZ_RULE_AKSEL;
  if (aksel)
    if (int rc = bz_coordinate_many(BZ_RULE_MEDIAN, rows, n, 0, d, out, st)) return forward(rc, bz_coordinate_many_last_error());
  unsigned* ticket = reinterpret_cast<unsigned*>(ws);
  int32_t* ord = order != nullptr ? order : reinterpret_cast<int32_t*>(ws + kOffOrder);
  double* parts = reinterpret_cast<double*>(ws + kOffTable);
  ManyRowTable t;
  for (int r = 0; r < kMaxNMany; ++r) t.p[r] = rows[r < n ? r : 0];
  cudaMemsetAsync(ticket, 0, sizeof(unsigned), st);
  if (int rc = check_launch("memset")) return rc;
  launch_rowkeys_many(t, n, aksel ? out : nullptr, d, parts, ord, ticket, aksel ? 0 : 1, st);
  if (int rc = check_launch("k2_rowkeys_many")) return rc;
  const Geom g = make_geom(rows, n, out, nullptr, d, 4);
  if (aksel) launch_average_many(t, g, ord, count, 1, (float)count, out, st);
  else       launch_average_many(t, g, ord, cge_count(n, f), 0, (float)(n - f), out, st);
  return check_launch("k3_average_many");
}

}  // namespace bz

using namespace bz;

extern "C" {

const char* bz_distance_many_last_error(void) { return g_error; }

size_t bz_distance_many_workspace_bytes(int n) { return many_distance_bytes(n < 1 ? 1 : n > kMaxNMany ? kMaxNMany : n); }

int bz_distance_many(int rule, const float* const* rows, int n, int f, int m, int mode, int64_t d,
                     float* out, int32_t* order, int32_t* status, void* ws, size_t ws_bytes, void* stream) {
  static const char* who = "bz_distance_many";
  if (int rc = check_call(rule, rows, n, d, out, who)) return rc;
  if (n <= BZ_MAX_N_DISTANCE)
    return forward(bz_distance(rule, rows, n, f, m, mode, d, out, order, status, ws, ws_bytes, stream), bz_last_error());
  int count;
  if (int rc = check_rule(rule, n, f, m, mode, count, who)) return rc;
  const size_t need = many_distance_bytes(n);
  if (ws == nullptr || ((uintptr_t)ws % 8) != 0 || ws_bytes < need)
    return fail(BZ_EWORKSPACE, "%s: workspace of %zu bytes at %p is too small or misaligned (need %zu, 8-byte aligned)",
                who, ws_bytes, ws, need);
  if (d == 0) return BZ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  char* base = static_cast<char*>(ws);
  if (rule == BZ_RULE_KRUM || rule == BZ_RULE_BULYAN)
    return run_pairwise(rule, rows, n, f, m, count, d, out, order, status, base, st);
  return run_rowkeys(rule, rows, n, f, count, d, out, order, base, st);
}

int bz_distance_many_select(int rule, const float* const* rows, int n, int f, int m, int64_t d, float* out,
                            int32_t* order, int32_t* status, void* ws, size_t ws_bytes, void* stream) {
  static const char* who = "bz_distance_many_select";
  if (rule != BZ_RULE_KRUM && rule != BZ_RULE_BULYAN)
    return fail(BZ_EINVAL, "%s: rule %d, expected BZ_RULE_KRUM or BZ_RULE_BULYAN", who, rule);
  if (int rc = check_call(rule, rows, n, d, out, who)) return rc;
  if (n <= BZ_MAX_N_DISTANCE)
    return fail(BZ_EUNSUPPORTED, "%s: n = %d, expected BZ_MAX_N_DISTANCE < n <= BZ_MAX_N_MANY", who, n);
  int count;
  if (int rc = check_rule(rule, n, f, m, BZ_AKSEL_MID, count, who)) return rc;
  const size_t need = many_distance_bytes(n);
  if (ws == nullptr || ((uintptr_t)ws % 8) != 0 || ws_bytes < need)
    return fail(BZ_EWORKSPACE, "%s: workspace of %zu bytes at %p is too small or misaligned (need %zu, 8-byte aligned)",
                who, ws_bytes, ws, need);
  if (d == 0) return BZ_OK;
  cudaStream_t st = (cudaStream_t)stream;
  char* base = static_cast<char*>(ws);
  ManyRowTable ut;
  ManyAliasMap map;
  const int u = alias_map(rows, n, ut, map);
  cudaMemsetAsync(base, 0, sizeof(unsigned), st);
  if (int rc = check_launch("memset")) return rc;
  return run_select(rule, rows, n, f, m, count, d, out, order, status, base, map, u, st);
}

}  // extern "C"
