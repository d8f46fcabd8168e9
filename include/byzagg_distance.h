/* byzagg_distance.h — C ABI of libbyzagg: the distance-based rules for up to 128 gradients.
 * Included at the end of byzagg.h; its conventions apply, except for the bound on n.
 *
 * bz_krum, bz_bulyan, bz_aksel and bz_cge stop at BZ_MAX_N (= 64) rows.  bz_distance runs Multi-Krum,
 * Bulyan, Aksel and CGE up to BZ_MAX_N_DISTANCE rows on one GPU: the pairwise distances of more than 64
 * rows come from several passes of the 64-row distance kernels over pairs of row blocks, the scoring,
 * the row distances and Bulyan's reduce from kernels that take 128 rows.  Brute stays at BZ_MAX_N: its
 * C(n, n - f) subsets are out of reach above 64 rows for all but tiny f.
 */
#ifndef BYZAGG_DISTANCE_H
#define BYZAGG_DISTANCE_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

#define BZ_MAX_N_DISTANCE 128

/* Bytes of device workspace bz_distance needs for n rows: bz_workspace_bytes(n) up to BZ_MAX_N, and
 * one size for every n above (the distance tables of up to six passes of at most 64 rows each). */
BZ_API size_t bz_distance_workspace_bytes(int n);

/* One distance-based rule over 1 <= n <= BZ_MAX_N_DISTANCE rows: the contract of bz_<rule> (rows
 * 4-byte aligned, aliases allowed, `out` not overlapping a row, d = 0 a no-op, order / status
 * optional, every argument checked before any CUDA call).
 *   rule   BZ_RULE_KRUM / _BULYAN / _BRUTE / _AKSEL / _CGE
 *   m      the selection size of Multi-Krum (1..n) and Bulyan (1..n - f - 2); ignored by the others
 *   mode   BZ_AKSEL_MID / BZ_AKSEL_NF for Aksel; ignored by the others
 *   order  n entries (brute: n - f), as bz_<rule> writes them; status: Bulyan and brute only
 *   ws     bz_distance_workspace_bytes(n) bytes, 8-byte aligned
 *   n <= BZ_MAX_N: exactly the launches of bz_<rule> (same kernels, same bits);
 *   n > BZ_MAX_N_DISTANCE, and brute above BZ_MAX_N: BZ_EUNSUPPORTED. */
BZ_API int bz_distance(int rule, const float* const* rows, int n, int f, int m, int mode, int64_t d,
                       float* out, int32_t* order, int32_t* status, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_DISTANCE_H */
