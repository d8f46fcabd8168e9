/* byzagg_search_shards.h — C ABI of libbyzagg for the attacks' line search on a d-sharded trainer.
 * Included at the end of byzagg.h; its conventions apply.
 *
 * Rank r holds columns [lo_r, hi_r) (byzagg_shards.h) of the honest rows, of the honest average `avg` and
 * of the attack direction `att`.  A score is a sum over all d columns, so every evaluation of
 * bz_line_search is cut at its exchanges, which the caller runs (all-gathers, rank order):
 *   1. bz_search_candidate       this rank's columns of the candidate row
 *   2. the rule on honest + [byz] * f_real:
 *        average .. meamed       bz_<rule> on the shard, no exchange
 *        krum, bulyan, brute     bz_pairdist_partial_reuse, all-gather of the n x n blocks,
 *                                bz_<rule>_select, the reduce (bz_average_selected / bz_bulyan_reduce)
 *        aksel, cge              bz_median into a centre (aksel), bz_rowdist_partial, all-gather of the
 *                                n-entry blocks, bz_rowdist_select, bz_average_selected
 *   3. bz_search_score_partial   this rank's fp64 share of the score
 *   4. all-gather of the R shares (one double each)
 *   5. bz_search_step            y and the next factor: bitwise the same on every rank
 * and a last bz_search_candidate (BZ_CANDIDATE_FINAL) writes the Byzantine gradient's shard.  `evals` is
 * fixed in advance, so every rank issues the same launches and collectives; a rank with an empty shard
 * (d = 0) joins every exchange.  With one rank the trace is bz_line_search's, bit for bit.
 * byzagg_search_peers.h runs the same evaluation with every exchange inside the kernels, over peer memory.
 */
#ifndef BYZAGG_SEARCH_SHARDS_H
#define BYZAGG_SEARCH_SHARDS_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of the DEVICE search state (8-byte aligned, caller-owned) that the calls below carry from one
 * evaluation to the next. */
#define BZ_SEARCH_STATE_BYTES 64

/* Which factor bz_search_candidate applies */
#define BZ_CANDIDATE_FIRST 0   /* x = 0 (line_maximize's start); also resets the state */
#define BZ_CANDIDATE_NEXT  1   /* the x the last bz_search_step chose */
#define BZ_CANDIDATE_FINAL 2   /* the best x: the attack's Byzantine gradient (no sign applied) */

/* Phase A (bz_pairdist_partial) with distance reuse across the evaluations of the search.  The rows are
 * deduplicated by address (the f_real copies of the candidate are one row), the pass computes only the
 * pairs of the rows that are not in a previous table (the star pass of bz_krum_reuse), and the block is
 * published in the n x n layout of the ORIGINAL rows: part[i*n+j], i < j, is the shard's sum of squared
 * differences of rows i and j (for two aliases of one tensor, its alias flag: 0, or NaN when the row holds
 * NaN / inf), every other entry 0.
 *   old_index, cache_in, u_old, cache_out, mode_out   as in bz_krum_reuse (cache_out receives the u x u
 *              table over the unique rows; mode_out 1 = only the new rows' pairs, 0 = full pass,
 *              -1 = rows not 16-byte aligned: the full pass of bz_pairdist_partial, no table written)
 * The block is bit-identical with and without a cache.  d == 0 writes the zero block. */
BZ_API int bz_pairdist_partial_reuse(const float* const* rows, int n, int64_t d, double* part,
                                     const int32_t* old_index, const double* cache_in, int u_old, double* cache_out,
                                     int* mode_out, void* ws, size_t ws_bytes, void* stream);

/* K8 on this rank's columns: byz <- the candidate row of the factor `which` (BZ_CANDIDATE_*) reads from
 * `state`, kind BZ_ATTACK_* (byzagg_attack.h; negative applies to BZ_ATTACK_IDENTICAL while searching).
 *   state    DEVICE, BZ_SEARCH_STATE_BYTES, 8-byte aligned
 *   d == 0   nothing but the state reset of BZ_CANDIDATE_FIRST (the pointers may then be NULL) */
BZ_API int bz_search_candidate(const float* avg, const float* att, float* byz, int64_t d, void* state, int which,
                               int negative, int kind, void* stream);

/* This rank's share of the score: *partial = sum_k fl32(out_k - avg_k)^2 in fp64, summed in the order of
 * bz_line_search's score pass and not rounded.  `state` (the search's) lends its election word.
 *   partial  DEVICE double; d == 0 writes 0.0
 *   ws       bz_workspace_bytes(1) bytes suffice */
BZ_API int bz_search_score_partial(const float* out, const float* avg, int64_t d, void* state, double* partial,
                                   void* ws, size_t ws_bytes, void* stream);

/* One CTA: y = fl32(((partials[0] + partials[1]) + partials[2]) + ...) over the nparts gathered shares, then
 * the transition of evaluation k of `evals` (bz_line_search's): trace[2k], trace[2k+1] = (x_k, y_k), the
 * chosen factor at trace[2 * evals] after the last one, *status = the first non-zero *eval_status so far
 * (eval_status: the rule's status word, or NULL), and the state's next x.
 *   partials  DEVICE double[nparts], nparts >= 1 (rank order)
 *   trace     DEVICE double[2 * evals + 1];  status  DEVICE int32 */
BZ_API int bz_search_step(const double* partials, int nparts, void* state, double* trace, const int32_t* eval_status,
                          int32_t* status, int k, int evals, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_SEARCH_SHARDS_H */
