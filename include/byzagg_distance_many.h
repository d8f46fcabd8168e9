/* byzagg_distance_many.h — C ABI of libbyzagg: Multi-Krum, Bulyan, Aksel and CGE for up to 1024 gradients.
 * Not included by byzagg.h (include it after byzagg.h and byzagg_coordinate_many.h, whose BZ_MAX_N_MANY it
 * uses); their conventions apply, except for the bound on n and the error string.  The calls live in the sixth
 * library, libbyzagg_many_distance.so, which links against libbyzagg.so and libbyzagg_many.so (those keep
 * exactly their own kernels); its failures are reported by bz_distance_many_last_error.
 *
 * bz_distance stops at BZ_MAX_N_DISTANCE (128) rows.  Up to 128 rows bz_distance_many is that call (same
 * launches, same bits).  Above, the u unique rows (found by address) go through K2-many, a tiled pairwise
 * distance kernel that reads every row once per pair of 64-row tiles; K5-many scores and selects with one
 * warp per row; the reduce is K3's ordered average over a 1024-pointer table, or K4-many for Bulyan.  Aksel's
 * and CGE's row keys come from K2'-many, Aksel's centre from bz_coordinate_many's median.
 */
#ifndef BYZAGG_DISTANCE_MANY_H
#define BYZAGG_DISTANCE_MANY_H

#include "byzagg.h"
#include "byzagg_coordinate_many.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The message of this library's last failure (thread-local), as bz_last_error is libbyzagg.so's. */
BZ_API const char* bz_distance_many_last_error(void);

/* Bytes of device workspace bz_distance_many needs for n rows (multiple of 256): bz_distance_workspace_bytes(n)
 * up to BZ_MAX_N_DISTANCE; above it a size that depends on n alone (never on d) and is never less than at
 * BZ_MAX_N_DISTANCE, so that the size at BZ_MAX_N_MANY serves every n. */
BZ_API size_t bz_distance_many_workspace_bytes(int n);

/* bz_distance's arguments and contract (byzagg_distance.h) for 1 <= n <= BZ_MAX_N_MANY rows: rows 4-byte
 * aligned, aliases allowed, `out` not overlapping a row, d = 0 a no-op, order / status optional, every
 * argument checked before any CUDA call.
 *   rule   BZ_RULE_KRUM / _BULYAN / _AKSEL / _CGE; BZ_RULE_BRUTE up to BZ_MAX_N only
 *   n <= BZ_MAX_N_DISTANCE: exactly bz_distance's launches (same kernels, same bits);
 *   n > BZ_MAX_N_MANY, and brute above BZ_MAX_N: BZ_EUNSUPPORTED.
 *   ws     bz_distance_many_workspace_bytes(n) bytes, 8-byte aligned
 * No allocation and no host synchronisation: a CUDA graph can capture the call. */
BZ_API int bz_distance_many(int rule, const float* const* rows, int n, int f, int m, int mode, int64_t d,
                            float* out, int32_t* order, int32_t* status, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_DISTANCE_MANY_H */
