/* byzagg_many_tools.h — C ABI of libbyzagg: the study metrics and the attacks' line search against the
 * coordinate-wise rules for up to 1024 gradients.  Not included by byzagg.h (include it after it); its
 * conventions apply, except for the bound on n and the error string.  The calls live in the fifth library,
 * libbyzagg_many_tools.so, which links against libbyzagg_many.so and libbyzagg.so (those keep exactly their
 * own kernels); its failures are reported by bz_many_tools_last_error.
 *
 * bz_avg_dev_max and bz_line_search stop at BZ_MAX_N_COORDINATE (128) rows.  Up to 128 rows the calls below
 * are those two calls (same launches, same bits).  Above, the study metrics run K6-many: a persistent CTA
 * per SM stages column tiles of all n rows in shared memory and reads every row once; and each evaluation of
 * the search is the one-rank form of byzagg_search_shards.h (bz_search_candidate, bz_coordinate_many,
 * bz_search_score_partial, bz_search_step with nparts = 1), whose trace is bz_line_search's.
 */
#ifndef BYZAGG_MANY_TOOLS_H
#define BYZAGG_MANY_TOOLS_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The message of this library's last failure (thread-local), as bz_last_error is libbyzagg.so's. */
BZ_API const char* bz_many_tools_last_error(void);

/* Bytes of device scratch bz_avg_dev_max_many needs for n rows (multiple of 256): bz_workspace_bytes(n) up
 * to BZ_MAX_N_COORDINATE, and above it one block of n + 2 doubles per CTA, but never less than at
 * BZ_MAX_N_COORDINATE: the size at BZ_MAX_N_MANY serves every n. */
BZ_API size_t bz_avg_dev_max_many_workspace_bytes(int n);

/* bz_avg_dev_max's contract (byzagg.h) for 1 <= n <= BZ_MAX_N_MANY rows: avg is the ordered sum divided by
 * n, bit for bit; stats[0] = sum_k avg[k]^2, stats[1] = max_k |avg[k]| (a NaN wins), stats[2+i] = sum_k
 * (g_i[k] - avg[k])^2, sums kept in fp64 and deterministic.  Every argument is checked before any CUDA call.
 *   n <= BZ_MAX_N_COORDINATE: exactly bz_avg_dev_max's launches;  n > BZ_MAX_N_MANY: BZ_EUNSUPPORTED.
 *   ws  bz_avg_dev_max_many_workspace_bytes(n) bytes, 8-byte aligned */
BZ_API int bz_avg_dev_max_many(const float* const* rows, int n, int64_t d, float* avg, double* stats,
                               void* ws, size_t ws_bytes, void* stream);

/* Bytes of device scratch bz_line_search_many needs for n = nh + f_real rows (multiple of 256):
 * bz_line_search_workspace_bytes(n) up to BZ_MAX_N_COORDINATE, above it the search state and the score's. */
BZ_API size_t bz_line_search_many_workspace_bytes(int n);

/* bz_line_search's arguments, checks, record and semantics (byzagg_attack.h) for rules BZ_RULE_AVERAGE ..
 * BZ_RULE_MEAMED with nh + f_real <= BZ_MAX_N_MANY (BZ_EUNSUPPORTED above); the distance rules are BZ_EINVAL
 * (bz_line_search and bz_distance_line_search take them).
 *   n <= BZ_MAX_N_COORDINATE: exactly bz_line_search's launches;
 *   ws  DEVICE scratch of bz_line_search_many_workspace_bytes(nh + f_real) bytes, 8-byte aligned
 * No allocation and no host synchronisation: a CUDA graph can capture the call. */
BZ_API int bz_line_search_many(int rule, const float* const* honest, int nh, int f_real, int f_decl, int kind, int negative,
                               const float* avg, const float* att, int64_t d, int evals, float* byz, float* out,
                               double* trace, int32_t* status, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_MANY_TOOLS_H */
