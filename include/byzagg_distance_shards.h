/* byzagg_distance_shards.h — C ABI of libbyzagg: the phases of the d-sharded path for the distance-based rules,
 * up to BZ_MAX_N_DISTANCE rows.  Included at the end of byzagg.h; its conventions apply, except for the bound on n.
 *
 * Each rank holds the same n rows cut to its own columns.  A step is, on every rank:
 *   A  bz_distance_partial: this shard's fp64 partial sums (an n x n block for Multi-Krum, Bulyan and brute, n sums
 *      for Aksel and CGE);
 *      the caller all-gathers the R blocks in rank order (one collective, or a copy on one rank);
 *   B  bz_distance_select: the R blocks added in rank order, ((p0 + p1) + p2) + ..., then the rule's selection:
 *      the same bits on every rank, so every rank selects the same rows;
 *   C  bz_distance_reduce: the rule's reduce of this shard over that selection.
 * With one rank (nparts = 1) the three calls give bz_distance's output, order and status bit for bit.
 * Up to BZ_MAX_N rows each call issues exactly the launches of its 64-row phase call (bz_pairdist_partial /
 * bz_rowdist_partial, bz_<rule>_select / bz_rowdist_select, bz_average_selected / bz_bulyan_reduce), so one
 * dispatch serves 1 to BZ_MAX_N_DISTANCE rows.  Brute stays at BZ_MAX_N rows: above, BZ_EUNSUPPORTED.
 *
 * Every call takes `rule` (BZ_RULE_KRUM / _BULYAN / _BRUTE / _AKSEL / _CGE, byzagg_attack.h) and
 * 1 <= n <= BZ_MAX_N_DISTANCE, and checks every argument before any CUDA call, like bz_distance.
 */
#ifndef BYZAGG_DISTANCE_SHARDS_H
#define BYZAGG_DISTANCE_SHARDS_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* A: this shard's partial block.  part: device double[n * n] (Multi-Krum, Bulyan, brute) or double[n] (Aksel, CGE).
 *   pairs  part[i * n + j], i < j: sum over the shard of (x_i - x_j)^2, in the layout of the ORIGINAL rows whichever
 *          rows alias (an aliased pair holds the self distance: 0, or NaN for a row holding NaN / inf); every
 *          other entry 0.  The layout of bz_pairdist_partial, so a rank with an empty shard publishes zeros.
 *   rows   part[i]: sum over the shard of (x_i - center)^2 for Aksel (`center`: device fp32[d], this shard of the
 *          coordinate-wise median of the rows, required when d > 0), of x_i^2 for CGE (`center` ignored).
 *   ws     bz_distance_workspace_bytes(n) bytes, 8-byte aligned.
 *   d = 0  the block is set to zeros (an empty shard still publishes its block); nothing else is launched
 *          above BZ_MAX_N rows. */
BZ_API int bz_distance_partial(int rule, const float* const* rows, int n, const float* center, int64_t d, double* part,
                               void* ws, size_t ws_bytes, void* stream);

/* B: the selection from `nparts` >= 1 gathered blocks, parts: device double[nparts][n * n] or [nparts][n] (phase
 *    A's layout), added in rank order.  f, m and mode as bz_distance takes them (m: Multi-Krum 1..n, Bulyan
 *    1..n - f - 2, ignored by the others; mode: Aksel's, ignored by the others).
 *   order   device int32[n] (brute: the n - f subset), required: what bz_distance writes there
 *   status  device int32 or NULL: Bulyan's and brute's status word, as bz_distance writes it; untouched otherwise */
BZ_API int bz_distance_select(int rule, const double* parts, int nparts, int n, int f, int m, int mode, int32_t* order,
                              int32_t* status, void* stream);

/* C: the rule's reduce of this shard over the selection of phase B, into out (device fp32[d]): the average of the
 *    first m (Multi-Krum), n - f (brute) or c (Aksel, by `mode`) rows of `order`, CGE's sum of its n - f rows
 *    divided by n - f, or Bulyan's reduce; counts, first terms and divisors are those of bz_distance.
 *   order   device int32 (required); status: device int32 or NULL, Bulyan's and brute's (non-zero: NaN fill)
 *   d = 0   a no-op. */
BZ_API int bz_distance_reduce(int rule, const float* const* rows, int n, int f, int m, int mode, const int32_t* order,
                              const int32_t* status, int64_t d, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_DISTANCE_SHARDS_H */
