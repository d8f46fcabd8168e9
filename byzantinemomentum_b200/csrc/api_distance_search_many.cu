// api_distance_search_many.cu — the C ABI of libbyzagg_many_search.so (include/byzagg_distance_search_many.h): the
// attacks' line search against Multi-Krum, Bulyan, Aksel and CGE for up to 1024 rows.  Up to 128 rows it calls
// libbyzagg.so's bz_distance_line_search; above, per evaluation, the one-rank form of byzagg_search_shards.h around
// libbyzagg_many_distance.so's bz_distance_many, whose distance table Multi-Krum and Bulyan keep from one evaluation
// to the next: from the second on, K2-star-many (k2_star_many.cu) writes the candidate's column of it and
// bz_distance_many_select scores, selects and reduces.  This library keeps its own error string; the others keep
// exactly their kernels.
#include <cstdarg>
#include <cstdio>

#include "distance_many.cuh"
#include "../../include/byzagg_attack.h"
#include "../../include/byzagg_distance_search.h"
#include "../../include/byzagg_distance_many.h"
#include "../../include/byzagg_distance_many_table.h"
#include "../../include/byzagg_distance_search_many.h"

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

static size_t round256(size_t bytes) { return (bytes + 255) / 256 * 256; }

// Above BZ_MAX_N_DISTANCE rows: bz_distance_many's workspace, then the tail: the search state, the score's share and the
// evaluation's status word in its first 256 bytes, the workspace of bz_search_score_partial, K2-star-many's blocks.
// Never less than bz_distance_line_search's at BZ_MAX_N_DISTANCE rows, so that the sizes grow with n.
constexpr size_t kHead = 256;
constexpr size_t kOffShare = BZ_SEARCH_STATE_BYTES;
constexpr size_t kOffEvalStatus = 128;
static_assert(kOffShare + sizeof(double) <= kOffEvalStatus && kOffEvalStatus + sizeof(int32_t) <= kHead, "the head holds them");

static size_t score_bytes() { return round256(bz_workspace_bytes(1)); }

static size_t search_many_bytes(int n) {
  if (n <= BZ_MAX_N_DISTANCE) return bz_distance_line_search_workspace_bytes(n);
  const size_t own = bz_distance_many_workspace_bytes(n) + kHead + score_bytes() + round256((size_t)kStarBlocks * sizeof(double));
  const size_t below = bz_distance_line_search_workspace_bytes(BZ_MAX_N_DISTANCE);
  return own > below ? own : below;
}

// bz_distance_line_search's checks with the limit BZ_MAX_N_MANY, up to the verdicts on f, which bz_distance_many
// gives: rows[0, n) receives honest + [byz] * f_real.
static int check_search(const char* who, const float* const* honest, int nh, int f_real, int kind, const float* avg,
                        const float* att, int64_t d, int evals, const float* byz, const float* out, const double* trace,
                        const int32_t* status, const float** rows) {
  const int n = nh + f_real;
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
    if (i < nh && honest[i] == nullptr) return fail(BZ_EINVAL, "%s: honest[%d] is NULL", who, i);
    if (i < nh && ((uintptr_t)honest[i] % sizeof(float)) != 0) return fail(BZ_EINVAL, "%s: honest[%d] is not 4-byte aligned", who, i);
    if (i < nh && (honest[i] == byz || honest[i] == out)) return fail(BZ_EINVAL, "%s: honest[%d] is byz or out", who, i);
  }
  for (int i = 0; i < nh; ++i)
    if (out < honest[i] + d && honest[i] < out + d) return fail(BZ_EINVAL, "%s: out overlaps honest[%d]", who, i);
  return BZ_OK;
}

// The search above BZ_MAX_N_DISTANCE rows, after the checks.
static int run_search_many(int rule, const float* const* rows, int n, int f_decl, int kind, int negative,
                           const float* avg, const float* att, int64_t d, int evals, float* byz, float* out,
                           double* trace, int32_t* status, void* ws, void* stream) {
  const size_t rule_bytes = bz_distance_many_workspace_bytes(n);
  char* tail = static_cast<char*>(ws) + rule_bytes;
  void* state = tail;
  double* share = reinterpret_cast<double*>(tail + kOffShare);
  int32_t* eval_status = reinterpret_cast<int32_t*>(tail + kOffEvalStatus);
  void* score_ws = tail + kHead;
  double* blocks = reinterpret_cast<double*>(tail + kHead + score_bytes());
  const bool pairwise = rule == BZ_RULE_KRUM || rule == BZ_RULE_BULYAN;
  int32_t* rule_status = rule == BZ_RULE_BULYAN ? eval_status : nullptr;
  const int m = n - f_decl - 2;
  // the unique rows: the honest rows first, the candidate (new content at the same address every time) last
  const float* uniq[kMaxNMany];
  unsigned short to_unique[kMaxNMany];
  const int u = dedupe_many(rows, n, uniq, to_unique);
  ManyRowTable ut;
  for (int k = 0; k < kMaxNMany; ++k) ut.p[k] = uniq[k < u ? k : 0];
  const PairGrid g = pair_grid(u, d);
  cudaStream_t st = (cudaStream_t)stream;
  for (int k = 0; k < evals; ++k) {
    if (int rc = bz_search_candidate(avg, att, byz, d, state, k == 0 ? BZ_CANDIDATE_FIRST : BZ_CANDIDATE_NEXT, negative,
                                     kind, stream))
      return forward(rc, bz_last_error());
    if (k == 0 || !pairwise) {
      if (int rc = bz_distance_many(rule, rows, n, f_decl, m, BZ_AKSEL_MID, d, out, nullptr, rule_status, ws, rule_bytes, stream))
        return forward(rc, bz_distance_many_last_error());
    } else {
      launch_star_many(ut, u, d, g, blocks, BZ_DISTANCE_MANY_TABLE(ws), st);
      if (int rc = check_launch("k2_star_many")) return rc;
      if (int rc = bz_distance_many_select(rule, rows, n, f_decl, m, d, out, nullptr, rule_status, ws, rule_bytes, stream))
        return forward(rc, bz_distance_many_last_error());
    }
    if (int rc = bz_search_score_partial(out, avg, d, state, share, score_ws, score_bytes(), stream))
      return forward(rc, bz_last_error());
    if (int rc = bz_search_step(share, 1, state, trace, rule_status, status, k, evals, stream)) return forward(rc, bz_last_error());
  }
  return forward(bz_search_candidate(avg, att, byz, d, state, BZ_CANDIDATE_FINAL, negative, kind, stream), bz_last_error());
}

}  // namespace bz

using namespace bz;

extern "C" {

const char* bz_distance_line_search_many_last_error(void) { return g_error; }

size_t bz_distance_line_search_many_workspace_bytes(int n) { return search_many_bytes(n < 1 ? 1 : n > kMaxNMany ? kMaxNMany : n); }

int bz_distance_line_search_many(int rule, const float* const* honest, int nh, int f_real, int f_decl, int kind, int negative,
                                 const float* avg, const float* att, int64_t d, int evals, float* byz, float* out,
                                 double* trace, int32_t* status, void* ws, size_t ws_bytes, void* stream) {
  static const char* who = "bz_distance_line_search_many";
  if (rule >= BZ_RULE_AVERAGE && rule <= BZ_RULE_MEAMED)
    return fail(BZ_EINVAL, "%s: rule %d is coordinate-wise: bz_line_search_many takes it up to BZ_MAX_N_MANY rows", who, rule);
  if (rule < BZ_RULE_KRUM || rule > BZ_RULE_CGE) return fail(BZ_EINVAL, "%s: unknown rule %d", who, rule);
  if (honest == nullptr) return fail(BZ_EINVAL, "%s: honest is NULL", who);
  if (nh < 1 || f_real < 1) return fail(BZ_EINVAL, "%s: nh = %d, f_real = %d, expected both >= 1", who, nh, f_real);
  if (nh > kMaxNMany || f_real > kMaxNMany || nh + f_real > kMaxNMany)
    return fail(BZ_EUNSUPPORTED, "%s: nh + f_real = %lld exceeds BZ_MAX_N_MANY = %d", who, (long long)nh + f_real, kMaxNMany);
  const int n = nh + f_real;
  if (rule == BZ_RULE_BRUTE && n > BZ_MAX_N)
    return fail(BZ_EUNSUPPORTED, "%s: brute takes nh + f_real <= BZ_MAX_N = %d rows, got %d", who, BZ_MAX_N, n);
  if (n <= BZ_MAX_N_DISTANCE)
    return forward(bz_distance_line_search(rule, honest, nh, f_real, f_decl, kind, negative, avg, att, d, evals, byz, out,
                                           trace, status, ws, ws_bytes, stream), bz_last_error());
  const float* rows[kMaxNMany];
  if (int rc = check_search(who, honest, nh, f_real, kind, avg, att, d, evals, byz, out, trace, status, rows)) return rc;
  const size_t need = search_many_bytes(n);
  if (ws == nullptr || ((uintptr_t)ws % 8) != 0 || ws_bytes < need)
    return fail(BZ_EWORKSPACE, "%s: workspace of %zu bytes at %p is too small or misaligned (need %zu, 8-byte aligned)",
                who, ws_bytes, ws, need);
  // bz_distance_many's verdicts on f and m, with d = 0: its checks, and no CUDA call
  if (int rc = bz_distance_many(rule, rows, n, f_decl, n - f_decl - 2, BZ_AKSEL_MID, 0, out, nullptr, nullptr, ws,
                                bz_distance_many_workspace_bytes(n), stream))
    return fail(rc, "%s: %s", who, bz_distance_many_last_error());
  return run_search_many(rule, rows, n, f_decl, kind, negative, avg, att, d, evals, byz, out, trace, status, ws, stream);
}

}  // extern "C"
