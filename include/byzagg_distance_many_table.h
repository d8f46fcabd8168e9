/* byzagg_distance_many_table.h — C ABI of libbyzagg_many_distance.so, the sixth library: the table of squared
 * distances that bz_distance_many leaves in its workspace for Multi-Krum and Bulyan above BZ_MAX_N_DISTANCE
 * rows, and the call that selects and reduces from it.  Include it after the header of bz_distance_many, whose
 * conventions and error string (bz_distance_many_last_error) apply.
 *
 * The table.  Above BZ_MAX_N_DISTANCE rows, a bz_distance_many call for Multi-Krum or Bulyan finds the u unique
 * rows of `rows` (by address, numbered in order of first appearance), writes the squared distance of unique rows
 * a <= b, in fp64, to entry a * u + b of a u x u table at BZ_DISTANCE_MANY_TABLE(ws), and leaves it there when it
 * returns.  The diagonal entry (a, a) is 0, or NaN when row a holds NaN or inf; entries a > b are not written.
 * A caller that changes rows in place may rewrite their entries and then call bz_distance_many_select, which
 * reads the table instead of computing it.
 */
#ifndef BYZAGG_DISTANCE_MANY_TABLE_H
#define BYZAGG_DISTANCE_MANY_TABLE_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Byte offset of the table in bz_distance_many's workspace (a multiple of 256), and the table itself. */
#define BZ_DISTANCE_MANY_TABLE_OFFSET 12544
#define BZ_DISTANCE_MANY_TABLE(ws) ((double*)((char*)(ws) + BZ_DISTANCE_MANY_TABLE_OFFSET))

/* bz_distance_many for Multi-Krum or Bulyan above BZ_MAX_N_DISTANCE rows without its distance pass: the scores
 * and the selection from the table the workspace holds, then the reduce, with bz_distance_many's bits when the
 * table holds what bz_distance_many would write for these rows.
 *   rule   BZ_RULE_KRUM or BZ_RULE_BULYAN (else BZ_EINVAL)
 *   n      BZ_MAX_N_DISTANCE < n <= BZ_MAX_N_MANY (else BZ_EUNSUPPORTED)
 *   f, m, d, out, order, status, ws, ws_bytes, stream   as in bz_distance_many (mode is Aksel's only)
 * Every argument checked before any CUDA call; no allocation, no host synchronisation. */
BZ_API int bz_distance_many_select(int rule, const float* const* rows, int n, int f, int m, int64_t d, float* out,
                                   int32_t* order, int32_t* status, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_DISTANCE_MANY_TABLE_H */
