/* byzagg_anticge.h — C ABI of libbyzagg: the attack built against CGE (attacks/anticge.py), generated on the device
 * for 1 <= nh <= BZ_MAX_N_DISTANCE honest rows.  Included at the end of byzagg.h; its conventions apply.
 *
 * With maxpos = nh - f_decl, the attack ranks the honest rows by their fp32 norm (σ: the stable order of bz_cge),
 * sums attack = σ0 + σ0 + σ1 + ... + σ(maxpos-1) in fp32 in that order, and scales it by
 * fl32(-maxnorm / attnorm) when attnorm = ||attack|| > 0, where maxnorm is the double just below the norm of
 * σ_maxpos.  When f_real > f_decl the attack is instead a row of NaN.  Norms are the fp32 rounding of fp64 sums of
 * squares (+inf once the sum passes FLT_MAX), as bz_cge computes them.
 *
 * Every call checks every argument before any CUDA call, with 0 <= maxpos < nh (1 <= f_decl <= nh) and f_real >= 0;
 * the reference's behaviour outside that range (negative indexing, IndexError) is not reproduced.  No call reads
 * device memory from the host, allocates or synchronises: a CUDA graph can capture each of them.
 */
#ifndef BYZAGG_ANTICGE_H
#define BYZAGG_ANTICGE_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of device workspace bz_anticge and bz_anticge_partial need for nh rows. */
BZ_API size_t bz_anticge_workspace_bytes(int nh);

/* The attack row into out (device fp32[d], not overlapping a row); the caller returns it f_real times.
 *   rows    nh device fp32 rows, 4-byte aligned (aliases allowed)
 *   ws      bz_anticge_workspace_bytes(nh) bytes, 8-byte aligned
 *   f_real > f_decl: out is filled with NaN, nothing else runs.  d = 0: a no-op.
 * Launches: K2' in CGE mode (the order and the norms), K10 (the ordered sum and its squares), K11 (the scale). */
BZ_API int bz_anticge(const float* const* rows, int nh, int f_decl, int f_real, int64_t d, float* out, void* ws,
                      size_t ws_bytes, void* stream);

/* The d-sharded form.  Each rank holds the same nh rows cut to its own columns.  A step is, on every rank:
 *   A  bz_distance_partial(BZ_RULE_CGE, ...): this shard's sums of squares (nh doubles); the caller all-gathers
 *      the R blocks in rank order into `blocks` (double[R][nh]);
 *   B  bz_distance_select(BZ_RULE_CGE, blocks, R, ...): the order σ, the same on every rank;
 *   C  bz_anticge_partial: this shard of the unscaled attack into out, and its fp64 sum of squares into
 *      *partial; the caller all-gathers the R partials in rank order into `partials` (double[R]);
 *   D  bz_anticge_scale: the R partials added in rank order give attnorm, the blocks of A added in rank order the
 *      norm of σ_maxpos, hence the same factor on every rank; this shard is scaled by it.
 * Every rank gets the same σ and the same factor.  Against bz_anticge on the whole rows, the norms' fp64 sums are
 * added in another order (per rank, then in rank order), so the factor may differ in its last bit.  The NaN fill
 * (f_real > f_decl) needs no exchange: bz_anticge on the shard gives it. */

/* C: order (device int32[nh], phase B's), partial (device double, required), ws as bz_anticge's.  d = 0 (an empty
 * shard) still writes *partial = 0. */
BZ_API int bz_anticge_partial(const float* const* rows, int nh, int f_decl, const int32_t* order, int64_t d, float* out,
                              double* partial, void* ws, size_t ws_bytes, void* stream);

/* D: blocks (device double[nparts][nh], phase A's gathered), order (phase B's), partials (device double[nparts],
 * phase C's gathered); out: this rank's shard from phase C, scaled in place.  d = 0: a no-op. */
BZ_API int bz_anticge_scale(const double* blocks, const int32_t* order, const double* partials, int nparts, int nh,
                            int f_decl, int64_t d, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_ANTICGE_H */
