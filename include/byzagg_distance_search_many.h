/* byzagg_distance_search_many.h — C ABI of libbyzagg_many_search.so, the seventh library: the attacks' line search
 * (byzagg_attack.h) against Multi-Krum, Bulyan, Aksel and CGE for up to BZ_MAX_N_MANY (1024) rows.  Include it
 * after byzagg.h and byzagg_coordinate_many.h (BZ_MAX_N_MANY); their conventions apply, except for the bound on n
 * and the error string, bz_distance_line_search_many_last_error.  The library links against libbyzagg.so,
 * libbyzagg_many.so and libbyzagg_many_distance.so, which keep exactly their kernels.
 *
 * bz_distance_line_search stops at BZ_MAX_N_DISTANCE (128) rows.  Up to 128 rows bz_distance_line_search_many is
 * that call (same checks, launches, workspace size and bits).  Above, every evaluation k writes the candidate row
 * (bz_search_candidate), runs the rule as bz_distance_many runs it over honest + [byz] * f_real with f = f_decl
 * and the attack's defaults (Multi-Krum and Bulyan m = n - f - 2, Aksel "mid"), takes its share of the score
 * (bz_search_score_partial) and the search's step (bz_search_step with one share); a last bz_search_candidate
 * writes the Byzantine gradient.  For Multi-Krum and Bulyan, the evaluation k = 0 is the full bz_distance_many
 * call; from k = 1 on only the candidate's column of bz_distance_many's table is computed (K2-star-many, with the
 * full pass's bits) before bz_distance_many_select: every distance, and every output, has the bits of the plain
 * bz_distance_many call.  Aksel and CGE run the full bz_distance_many call at every evaluation.
 */
#ifndef BYZAGG_DISTANCE_SEARCH_MANY_H
#define BYZAGG_DISTANCE_SEARCH_MANY_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The message of this library's last failure (thread-local), as bz_last_error is libbyzagg.so's. */
BZ_API const char* bz_distance_line_search_many_last_error(void);

/* Bytes of device scratch bz_distance_line_search_many needs for n = nh + f_real rows (multiple of 256):
 * bz_distance_line_search_workspace_bytes(n) up to BZ_MAX_N_DISTANCE; above it bz_distance_many's workspace for n
 * rows plus the search's state, its score share, the evaluation's status word and K2-star-many's per-slice sums,
 * a size that depends on n alone (never on d) and grows with n. */
BZ_API size_t bz_distance_line_search_many_workspace_bytes(int n);

/* bz_distance_line_search's arguments, checks, record and semantics, with these limits:
 *   rule   BZ_RULE_KRUM, BZ_RULE_BULYAN, BZ_RULE_AKSEL, BZ_RULE_CGE (nh + f_real <= BZ_MAX_N_MANY) or BZ_RULE_BRUTE
 *          (nh + f_real <= BZ_MAX_N): BZ_EUNSUPPORTED above.  A coordinate-wise rule is BZ_EINVAL:
 *          bz_line_search_many takes those
 *   ws     DEVICE scratch of bz_distance_line_search_many_workspace_bytes(nh + f_real) bytes, 8-byte aligned
 * Every argument is checked before any CUDA call.  A Bulyan evaluation that fails writes its status word, and its
 * NaN output never wins the search.  No allocation and no host synchronisation: a CUDA graph can capture the call. */
BZ_API int bz_distance_line_search_many(int rule, const float* const* honest, int nh, int f_real, int f_decl, int kind,
                                        int negative, const float* avg, const float* att, int64_t d, int evals,
                                        float* byz, float* out, double* trace, int32_t* status,
                                        void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_DISTANCE_SEARCH_MANY_H */
