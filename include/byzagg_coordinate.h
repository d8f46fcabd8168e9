/* byzagg_coordinate.h — C ABI of libbyzagg: the coordinate-wise rules for up to 128 gradients.
 * Included at the end of byzagg.h; its conventions apply, except for the bound on n.
 *
 * The distance-based rules stop at BZ_MAX_N (= 64) rows; average, median, trimmed mean, Phocas and
 * MeaMed work on each coordinate alone, and one thread still holds a column of up to 128 values in
 * registers.  bz_coordinate takes them up to BZ_MAX_N_COORDINATE rows.
 */
#ifndef BYZAGG_COORDINATE_H
#define BYZAGG_COORDINATE_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

#define BZ_MAX_N_COORDINATE 128

/* One coordinate-wise rule over 1 <= n <= BZ_MAX_N_COORDINATE rows: the contract of bz_<rule>
 * (rows 4-byte aligned, aliases allowed, `out` not overlapping a row, d = 0 a no-op).
 *   rule   BZ_RULE_AVERAGE / _MEDIAN / _TRMEAN / _PHOCAS / _MEAMED; f is ignored by AVERAGE / MEDIAN,
 *          BZ_EINVAL when n - 2f < 1 for the others
 *   n <= BZ_MAX_N: exactly the launches of bz_<rule> (same kernels, same bits);
 *   n > BZ_MAX_N_COORDINATE: BZ_EUNSUPPORTED.
 * Results are those of the reference at every n (the trimmed mean keeps ATen's summation cascade). */
BZ_API int bz_coordinate(int rule, const float* const* rows, int n, int f, int64_t d, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_COORDINATE_H */
