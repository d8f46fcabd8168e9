/* byzagg_distance_search_shards.h — C ABI of libbyzagg: phase A of the d-sharded line search against Multi-Krum and
 * Bulyan above BZ_MAX_N (64) rows, with the honest rows' distances kept from one evaluation to the next.  This header
 * includes byzagg.h and byzagg_distance_shards.h for their conventions; byzagg.h does not include it.
 *
 * bz_pairdist_partial_reuse is that phase up to BZ_MAX_N rows.  Above, a search evaluation's rows are the honest rows,
 * which do not change, and one candidate row repeated f_real times, which does.  bz_distance_partial_reuse computes
 * bz_distance_partial's block of those rows and keeps bz_distance's pass tables (byzagg_distance.h) in a buffer of
 * the caller's, so that the next evaluation computes only the candidate's pairs:
 *   star  when the previous tables are given (tables_in), every row that old_index marks as new (-1) is one unique
 *         row that comes last among the unique rows (the rows are deduplicated by address, in row order), every
 *         other row keeps its unique row of the previous call, and the unique row count is u_old: the pass plan is
 *         the previous one.  Then only the passes that hold the candidate run, each over its rows in the full pass's
 *         launch shape with the candidate as its one star row; their candidate column goes into tables_out, every
 *         other entry is tables_in's.
 *   full  otherwise: every pass runs, as bz_distance_partial runs them, into tables_out.
 * Either way the block is then laid out from tables_out as bz_distance_partial lays it out, so `part` has
 * bz_distance_partial's bits for the same rows.
 * The tables are bound to the row addresses and contents of the call that wrote them: old_index is taken on trust.
 * A caller that passes other kept rows, or rows whose contents changed, with the same deduplication shape gets that
 * call's stale distances, with mode_out = 1.  Pass tables_in = NULL (or old_index = NULL) whenever a kept row changed.
 * A star pass that cannot run (rows not 16-byte aligned) runs the full pass instead, with the same bits.
 */
#ifndef BYZAGG_DISTANCE_SEARCH_SHARDS_H
#define BYZAGG_DISTANCE_SEARCH_SHARDS_H

#include "byzagg.h"
#include "byzagg_distance_shards.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of one set of pass tables (tables_in, tables_out below): the same for every n, 8-byte aligned. */
BZ_API size_t bz_distance_pass_tables_bytes(void);

/* Phase A of Multi-Krum (BZ_RULE_KRUM) or Bulyan (BZ_RULE_BULYAN) on BZ_MAX_N < n <= BZ_MAX_N_DISTANCE rows.
 *   rows, n, d, part  as bz_distance_partial takes them: part is DEVICE double[n * n], written as it writes it
 *   old_index         HOST int32[n] or NULL: row i was unique row old_index[i] of the call that wrote tables_in,
 *                     -1 for a new row; NULL runs the full passes
 *   tables_in         DEVICE, bz_distance_pass_tables_bytes() bytes, or NULL: the tables_out of the previous call
 *   u_old             that call's unique row count (1..BZ_MAX_N_DISTANCE when tables_in is given)
 *   tables_out        DEVICE, bz_distance_pass_tables_bytes() bytes, 8-byte aligned; may equal tables_in
 *   mode_out          HOST int: 1 when every pass of the candidate ran as a star pass, 0 when the full passes ran,
 *                     -1 when d = 0 (the block is set to zeros and nothing else runs)
 *   ws                bz_distance_workspace_bytes(n) bytes, 8-byte aligned
 * Every argument is checked before any CUDA call.  n <= BZ_MAX_N is BZ_EUNSUPPORTED: bz_pairdist_partial_reuse takes
 * those rows.  No allocation and no host synchronisation: a CUDA graph can capture the call (its mode is then the one
 * the capture took). */
BZ_API int bz_distance_partial_reuse(int rule, const float* const* rows, int n, int64_t d, double* part,
                                     const int32_t* old_index, const double* tables_in, int u_old, double* tables_out,
                                     int* mode_out, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_DISTANCE_SEARCH_SHARDS_H */
