/* byzagg_coordinate_many.h — C ABI of libbyzagg: the coordinate-wise rules for up to 1024 gradients.
 * Included by byzagg.h, after byzagg_coordinate.h; its conventions apply, except for the bound on n and the
 * error string.  The calls live in the fourth library, libbyzagg_many.so, which links against libbyzagg.so
 * (libbyzagg.so keeps exactly its own kernels); its failures are reported by bz_coordinate_many_last_error.
 *
 * bz_coordinate keeps one column per thread in registers, which stops at BZ_MAX_N_COORDINATE (= 128)
 * rows.  Above that, a CTA stages column tiles of all n rows in shared memory through an mbarrier
 * ring, and each column is sorted by one warp (a bitonic sort of its integer keys in registers, n
 * padded to 256, 512 or 1024); the average is the same ordered sum as below 128 rows.  The row
 * pointer table (8 KB) is a kernel parameter: no host-to-device copy per call, and a call can be
 * captured in a CUDA graph as it is.
 */
#ifndef BYZAGG_COORDINATE_MANY_H
#define BYZAGG_COORDINATE_MANY_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

#define BZ_MAX_N_MANY 1024

/* One coordinate-wise rule over 1 <= n <= BZ_MAX_N_MANY rows: the contract of bz_coordinate
 * (rows 4-byte aligned, aliases allowed, `out` not overlapping a row, d = 0 a no-op, every argument
 * checked before any CUDA call).
 *   rule   BZ_RULE_AVERAGE / _MEDIAN / _TRMEAN / _PHOCAS / _MEAMED; f is ignored by AVERAGE / MEDIAN,
 *          BZ_EINVAL when n - 2f < 1 for the others
 *   n <= BZ_MAX_N_COORDINATE: exactly the launches of bz_coordinate (same kernels, same bits);
 *   n > BZ_MAX_N_MANY: BZ_EUNSUPPORTED.
 * Results are those of the reference: the median is the lower median (NaN when the column holds a
 * NaN), the trimmed mean sums the kept ranks in ascending order in ATen's 16-row cascade, Phocas and
 * MeaMed average the n - f values closest to their centre (NaN distances farthest), the average adds
 * the rows in order from 0. */
/* The message of this library's last failure (thread-local), as bz_last_error is libbyzagg.so's. */
BZ_API const char* bz_coordinate_many_last_error(void);

BZ_API int bz_coordinate_many(int rule, const float* const* rows, int n, int f, int64_t d, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_COORDINATE_MANY_H */
