// api_many_tools.cu — the C ABI of libbyzagg_many_tools.so (include/byzagg_many_tools.h): the study metrics and the
// line search against the coordinate-wise rules for up to 1024 rows.  Up to 128 rows it calls libbyzagg.so's
// bz_avg_dev_max and bz_line_search; above, K6-many (k6_many.cu) and, per evaluation of the search, the one-rank
// form of byzagg_search_shards.h with libbyzagg_many.so's bz_coordinate_many.  This library links against both and
// keeps its own error string; libbyzagg.so and libbyzagg_many.so keep exactly their kernels.
#include <cstdarg>
#include <cstdio>

#include "common.cuh"
#include "../../include/byzagg_attack.h"
#include "../../include/byzagg_search_shards.h"
#include "../../include/byzagg_many_tools.h"

namespace bz {

// k6_many.cu
size_t study_many_parts_bytes(int n);
void launch_study_many(const ManyRowTable& rows, int n, int64_t d, float* avg, double* stats, double* parts,
                       unsigned* ticket, int sms, cudaStream_t st);

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

static int tools_sm_count() {
  static int cached[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  int& c = cached[dev & 63];
  if (c == 0) cudaDeviceGetAttribute(&c, cudaDevAttrMultiProcessorCount, dev);
  return c > 0 ? c : 132;
}

static size_t round256(size_t bytes) { return (bytes + 255) / 256 * 256; }

// Above kMaxNCoordinate rows: the ticket in the first 256 bytes, then the per-CTA blocks; never less than
// bz_avg_dev_max's workspace at kMaxNCoordinate rows, so that the size at kMaxNMany serves every n.
constexpr size_t kHead = 256;
static size_t avg_dev_max_many_bytes(int n) {
  if (n <= kMaxNCoordinate) return bz_workspace_bytes(n);
  const size_t blocks = round256(kHead + study_many_parts_bytes(n > kMaxNMany ? kMaxNMany : n));
  const size_t below = bz_workspace_bytes(kMaxNCoordinate);
  return blocks > below ? blocks : below;
}

// Above kMaxNCoordinate rows: the search state and the score's share in the first 256 bytes, then the workspace
// of bz_search_score_partial.
static size_t line_search_many_bytes(int n) {
  if (n <= kMaxNCoordinate) return bz_line_search_workspace_bytes(n);
  return round256(kHead + bz_workspace_bytes(1));
}

static int check_ws(const void* ws, size_t bytes, size_t need, const char* who) {
  if (ws == nullptr || ((uintptr_t)ws % 8) != 0 || bytes < need)
    return fail(BZ_EWORKSPACE, "%s: workspace of %zu bytes at %p is too small or misaligned (need %zu, 8-byte aligned)",
                who, bytes, ws, need);
  return BZ_OK;
}

// bz_avg_dev_max's checks of the rows, with the limit BZ_MAX_N_MANY.
static int check_rows(const float* const* rows, int n, int64_t d, const void* out, const char* who) {
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
  return BZ_OK;
}

// bz_line_search's checks (api_search.inc's check_search_args) with the limit BZ_MAX_N_MANY: rows[0, n) receives
// honest + [byz] * f_real.
static int check_search(const char* who, int rule, const float* const* honest, int nh, int f_real, int f_decl, int kind,
                        const float* avg, const float* att, int64_t d, int evals, const float* byz, const float* out,
                        const double* trace, const int32_t* status, const float** rows) {
  if (rule >= BZ_RULE_KRUM && rule <= BZ_RULE_CGE)
    return fail(BZ_EINVAL, "%s: rule %d is a distance rule: bz_line_search takes it up to BZ_MAX_N rows, "
                "bz_distance_line_search up to BZ_MAX_N_DISTANCE", who, rule);
  if (rule < BZ_RULE_AVERAGE || rule > BZ_RULE_MEAMED) return fail(BZ_EINVAL, "%s: unknown rule %d", who, rule);
  if (honest == nullptr) return fail(BZ_EINVAL, "%s: honest is NULL", who);
  if (nh < 1 || f_real < 1) return fail(BZ_EINVAL, "%s: nh = %d, f_real = %d, expected both >= 1", who, nh, f_real);
  const int n = nh + f_real;
  if (n > kMaxNMany) return fail(BZ_EUNSUPPORTED, "%s: nh + f_real = %d exceeds BZ_MAX_N_MANY = %d", who, n, kMaxNMany);
  if (d < 1) return fail(BZ_EINVAL, "%s: d = %lld, expected d >= 1", who, (long long)d);
  if (evals < 1) return fail(BZ_EINVAL, "%s: evals = %d, expected evals >= 1", who, evals);
  if (kind != BZ_ATTACK_IDENTICAL && kind != BZ_ATTACK_EMPIRE_STRICT) return fail(BZ_EINVAL, "%s: unknown kind %d", who, kind);
  const bool empire = kind == BZ_ATTACK_EMPIRE_STRICT;
  if (avg == nullptr || (att == nullptr && !empire) || byz == nullptr || out == nullptr || trace == nullptr || status == nullptr)
    return fail(BZ_EINVAL, "%s: avg, att, byz, out, trace or status is NULL", who);
  const void* vectors[4] = {avg, empire ? avg : att, byz, out};
  for (const void* p : vectors)
    if (((uintptr_t)p % sizeof(float)) != 0) return fail(BZ_EINVAL, "%s: avg, att, byz and out must be 4-byte aligned", who);
  if (byz == avg || byz == att || out == avg || out == att || out == byz)
    return fail(BZ_EINVAL, "%s: byz and out must be distinct from avg, att and each other", who);
  for (int i = 0; i < n; ++i) {
    rows[i] = i < nh ? honest[i] : byz;
    if (i < nh && (honest[i] == byz || honest[i] == out)) return fail(BZ_EINVAL, "%s: honest[%d] is byz or out", who, i);
  }
  if (int rc = check_rows(rows, n, d, out, who)) return rc;
  if (rule >= BZ_RULE_TRMEAN && (f_decl < 0 || n - 2 * f_decl < 1))
    return fail(BZ_EINVAL, "%s: f = %d not executable with n = %d (need n - 2f >= 1)", who, f_decl, n);
  return BZ_OK;
}

}  // namespace bz

using namespace bz;

extern "C" {

const char* bz_many_tools_last_error(void) { return g_error; }

size_t bz_avg_dev_max_many_workspace_bytes(int n) { return avg_dev_max_many_bytes(n < 1 ? 1 : n); }

int bz_avg_dev_max_many(const float* const* rows, int n, int64_t d, float* avg, double* stats,
                        void* ws, size_t ws_bytes, void* stream) {
  static const char* who = "bz_avg_dev_max_many";
  if (int rc = check_rows(rows, n, d, avg, who)) return rc;
  if (stats == nullptr) return fail(BZ_EINVAL, "%s: stats is NULL", who);
  if (int rc = check_ws(ws, ws_bytes, avg_dev_max_many_bytes(n), who)) return rc;
  if (n <= kMaxNCoordinate) return forward(bz_avg_dev_max(rows, n, d, avg, stats, ws, ws_bytes, stream), bz_last_error());
  cudaStream_t st = (cudaStream_t)stream;
  if (d == 0) {
    cudaMemsetAsync(stats, 0, (size_t)(2 + n) * sizeof(double), st);
    return check_launch("memset");
  }
  ManyRowTable t;
  for (int r = 0; r < kMaxNMany; ++r) t.p[r] = rows[r < n ? r : 0];
  char* base = static_cast<char*>(ws);
  launch_study_many(t, n, d, avg, stats, reinterpret_cast<double*>(base + kHead), reinterpret_cast<unsigned*>(base),
                    tools_sm_count(), st);
  return check_launch("k6_many");
}

size_t bz_line_search_many_workspace_bytes(int n) { return line_search_many_bytes(n < 1 ? 1 : n); }

int bz_line_search_many(int rule, const float* const* honest, int nh, int f_real, int f_decl, int kind, int negative,
                        const float* avg, const float* att, int64_t d, int evals, float* byz, float* out,
                        double* trace, int32_t* status, void* ws, size_t ws_bytes, void* stream) {
  static const char* who = "bz_line_search_many";
  const float* rows[kMaxNMany];
  if (int rc = check_search(who, rule, honest, nh, f_real, f_decl, kind, avg, att, d, evals, byz, out, trace, status, rows))
    return rc;
  const int n = nh + f_real;
  if (int rc = check_ws(ws, ws_bytes, line_search_many_bytes(n), who)) return rc;
  if (n <= kMaxNCoordinate)
    return forward(bz_line_search(rule, honest, nh, f_real, f_decl, kind, negative, avg, att, d, evals, byz, out, trace,
                                  status, ws, ws_bytes, stream), bz_last_error());
  // the one-rank form of byzagg_search_shards.h: the state and the score's share in the head, the score's workspace after
  char* base = static_cast<char*>(ws);
  void* state = base;
  double* share = reinterpret_cast<double*>(base + BZ_SEARCH_STATE_BYTES);
  void* score_ws = base + kHead;
  const size_t score_bytes = ws_bytes - kHead;
  for (int k = 0; k < evals; ++k) {
    if (int rc = bz_search_candidate(avg, att, byz, d, state, k == 0 ? BZ_CANDIDATE_FIRST : BZ_CANDIDATE_NEXT, negative,
                                     kind, stream))
      return forward(rc, bz_last_error());
    if (int rc = bz_coordinate_many(rule, rows, n, f_decl, d, out, stream)) return forward(rc, bz_coordinate_many_last_error());
    if (int rc = bz_search_score_partial(out, avg, d, state, share, score_ws, score_bytes, stream))
      return forward(rc, bz_last_error());
    if (int rc = bz_search_step(share, 1, state, trace, nullptr, status, k, evals, stream)) return forward(rc, bz_last_error());
  }
  return forward(bz_search_candidate(avg, att, byz, d, state, BZ_CANDIDATE_FINAL, negative, kind, stream), bz_last_error());
}

}  // extern "C"
