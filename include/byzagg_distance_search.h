/* byzagg_distance_search.h — C ABI of libbyzagg: the attacks' line search (byzagg_attack.h) against Multi-Krum,
 * Bulyan, Aksel and CGE for up to BZ_MAX_N_DISTANCE (128) rows.  This header includes byzagg.h and
 * byzagg_distance.h for their conventions; byzagg.h does not include it.
 *
 * bz_line_search stops at BZ_MAX_N (64) rows against a distance rule.  bz_distance_line_search runs the same
 * search over the rules bz_distance takes, with bz_distance's limits: Multi-Krum, Bulyan, Aksel and CGE up to
 * BZ_MAX_N_DISTANCE rows, brute up to BZ_MAX_N.
 *
 * Up to BZ_MAX_N rows it issues exactly the launches of bz_line_search (same kernels, same bits).  Above, every
 * evaluation writes the candidate row, runs the rule as bz_distance runs it over honest + [byz] * f_real with
 * f = f_decl and the attack's defaults (Multi-Krum and Bulyan m = n - f - 2, Aksel "mid"), then scores it.
 * Multi-Krum and Bulyan compute every pass of pairwise distances at the first evaluation only.  From the second
 * on, a pass that does not hold the candidate row launches nothing, and a pass that holds it computes the
 * candidate's pairs alone, in the full pass's launch shape.  So every distance, and every output, has the bits
 * of the plain bz_distance call.  Aksel and CGE run bz_distance's chain at every evaluation.
 */
#ifndef BYZAGG_DISTANCE_SEARCH_H
#define BYZAGG_DISTANCE_SEARCH_H

#include "byzagg.h"
#include "byzagg_distance.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of device scratch bz_distance_line_search needs for n = nh + f_real rows (multiple of 256):
 * bz_line_search_workspace_bytes(n) up to BZ_MAX_N, and above it bz_distance_workspace_bytes(n) plus the
 * search's state (one size for every n above BZ_MAX_N). */
BZ_API size_t bz_distance_line_search_workspace_bytes(int n);

/* bz_line_search's arguments, checks, record and semantics (byzagg_attack.h), with these differences:
 *   rule   BZ_RULE_KRUM, BZ_RULE_BULYAN, BZ_RULE_AKSEL, BZ_RULE_CGE (nh + f_real <= BZ_MAX_N_DISTANCE) or
 *          BZ_RULE_BRUTE (nh + f_real <= BZ_MAX_N): BZ_EUNSUPPORTED above, as bz_distance.  A coordinate-wise
 *          rule is BZ_EINVAL: bz_line_search takes those up to BZ_MAX_N_COORDINATE rows
 *   ws     DEVICE scratch of bz_distance_line_search_workspace_bytes(nh + f_real) bytes, 8-byte aligned
 * A Bulyan evaluation that fails writes its status word as bz_line_search does, and its NaN output never wins
 * the search.  No allocation, no host synchronisation and no memset the rules do not already issue: a CUDA graph
 * can capture the call. */
BZ_API int bz_distance_line_search(int rule, const float* const* honest, int nh, int f_real, int f_decl, int kind,
                                   int negative, const float* avg, const float* att, int64_t d, int evals,
                                   float* byz, float* out, double* trace, int32_t* status,
                                   void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_DISTANCE_SEARCH_H */
