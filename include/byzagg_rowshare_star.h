/* byzagg_rowshare_star.h — C ABI of libbyzagg_star: CGE's phase A of the d-sharded line search above BZ_MAX_N (64)
 * rows after its first evaluation.  The calls live in a third library, libbyzagg_star.so, built next to libbyzagg.so
 * and libbyzagg_peers.so by the same Makefile with the same flags and linked against neither; callers compose the
 * libraries through their C ABIs.  This header includes byzagg.h for its conventions (return codes); byzagg.h does not
 * include it.
 *
 * A search evaluation's rows are the honest rows, which do not change, and one candidate row repeated f_real times,
 * placed last.  bz_distance_partial(BZ_RULE_CGE, ...) writes part[i] = the sum over this shard of x_i^2 for every row.
 * After the first evaluation only the candidate's entries change, so bz_rowshare_star reads the candidate row once and
 * writes part[c0, n) with exactly the fp64 sums bz_distance_partial writes there for the same rows (its launch
 * geometry, its fp32 chunk sums and its fixed-order fp64 sums); part[0, c0) is left as it is.  It reads 4 bytes per
 * coordinate where bz_distance_partial reads n * 4.
 */
#ifndef BYZAGG_ROWSHARE_STAR_H
#define BYZAGG_ROWSHARE_STAR_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The message of the last failed call of libbyzagg_star in this thread (libbyzagg's bz_last_error() does not see it). */
BZ_API const char* bz_rowshare_star_last_error(void);

/* Bytes of device scratch bz_rowshare_star needs for n rows (a multiple of 256). */
BZ_API size_t bz_rowshare_star_workspace_bytes(int n);

/* rows   HOST array of n DEVICE pointers, BZ_MAX_N < n <= BZ_MAX_N_DISTANCE: the table bz_distance_partial took.  Rows
 *        [c0, n) are one pointer (the candidate), distinct from every row of [0, c0); 0 < c0 < n.  Only the candidate
 *        is read.  When d > 0 every pointer must be non-NULL and 4-byte aligned; when d = 0 no pointer is read and
 *        none is checked (the rows of an empty shard may share one address)
 * d      this shard's coordinates (>= 0); d = 0 writes zeros to part[c0, n)
 * part   DEVICE double[n], 8-byte aligned: entries [c0, n) are written, [0, c0) untouched
 * ws     DEVICE scratch of bz_rowshare_star_workspace_bytes(n) bytes, 8-byte aligned
 * Every argument is checked before any CUDA call (BZ_EINVAL, BZ_EUNSUPPORTED, BZ_EWORKSPACE).  No allocation and no
 * host synchronisation: a CUDA graph can capture the call. */
BZ_API int bz_rowshare_star(const float* const* rows, int n, int c0, int64_t d, double* part, void* ws, size_t ws_bytes,
                            void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_ROWSHARE_STAR_H */
