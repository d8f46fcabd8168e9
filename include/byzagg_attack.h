/* byzagg_attack.h — C ABI of libbyzagg for the attacks' line search.  Included at the end of byzagg.h;
 * its conventions apply.
 *
 * The identical-family attacks (attacks/identical.py:67-77: little, empire, bulyan) and empire-strict
 * (attacks/empire.py:51-59) pick their factor with `tools.line_maximize` (tools/misc.py:468-513) when
 * it is negative: `evals` evaluations of the rule, each scored by the squared distance of its output
 * to the honest average, each followed by a host read that decides the next factor.  bz_line_search
 * enqueues the whole search: every evaluation writes the candidate row, runs the rule, scores it and
 * computes the next factor on the device, so the caller reads the outcome once.
 */
#ifndef BYZAGG_ATTACK_H
#define BYZAGG_ATTACK_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Rule codes: BZ_RULE_AVERAGE .. BZ_RULE_MEAMED of byzagg.h (0..4), continued here */
#define BZ_RULE_KRUM   5
#define BZ_RULE_BULYAN 6
#define BZ_RULE_BRUTE  7
#define BZ_RULE_AKSEL  8
#define BZ_RULE_CGE    9

/* Candidate rows */
#define BZ_ATTACK_IDENTICAL     0   /* byz = fl32(avg + fl32(fl32(s) * att)), s = -x when negative, else x */
#define BZ_ATTACK_EMPIRE_STRICT 1   /* byz = fl32(avg * fl32(-x)); att is not read */

/* Bytes of device scratch bz_line_search needs for n = nh + f_real rows (multiple of 256). */
BZ_API size_t bz_line_search_workspace_bytes(int n);

/* `line_maximize(scape, evals, start=0., delta=1., ratio=0.8)` over the rule `rule` (defaults: Multi-Krum
 * and Bulyan m = n - f - 2, Aksel "mid") applied to honest + [byz] * f_real with f = f_decl, where the
 * scape of x is
 *   y(x) = fl32(sum_k fl32(out_k - avg_k)^2)     out = the rule's output with byz the candidate row of x
 * The search state is fp64 and follows tools/misc.py:468-513 operation for operation (NaN scores never
 * win a comparison), so the same y values give the same x sequence, bit for bit.  The score is K2''s
 * deterministic fp32-then-fp64 sum, not ATen's `dot` order.
 *   honest      HOST array of nh DEVICE pointers (fp32[d], 4-byte aligned), 1 <= nh, nh + f_real <= BZ_MAX_N
 *   f_real      copies of the candidate row in the rule's input, >= 1
 *   kind        BZ_ATTACK_*; negative applies to BZ_ATTACK_IDENTICAL only
 *   avg, att    DEVICE fp32[d]: honest average and attack direction (att unused by empire-strict)
 *   d >= 1, evals >= 1
 *   byz         DEVICE fp32[d]: the candidate row; after the call, the Byzantine gradient the attack
 *               returns: avg + best * att (identical; the reference applies no sign to the returned
 *               factor) or avg * -best (empire-strict)
 *   out         DEVICE fp32[d] scratch: the rule's output
 *   trace       DEVICE double[2 * evals + 1]: (x_k, y_k) of every evaluation, then the chosen factor
 *   status      DEVICE int32: the first non-zero status word of an evaluation (Bulyan's degenerate data,
 *               brute's "no finite subset"), else 0
 *   ws          DEVICE scratch of bz_line_search_workspace_bytes(nh + f_real) bytes, 8-byte aligned
 * Multi-Krum, Bulyan and brute compute all distances at the first evaluation and only the candidate
 * row's afterwards (the star pass of bz_*_reuse), with the bits of the plain call.  No allocation and no
 * host synchronisation: a CUDA graph can capture the call.  byz and out must not be any row, avg or att. */
BZ_API int bz_line_search(int rule, const float* const* honest, int nh, int f_real, int f_decl, int kind, int negative,
                          const float* avg, const float* att, int64_t d, int evals, float* byz, float* out,
                          double* trace, int32_t* status, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_ATTACK_H */
