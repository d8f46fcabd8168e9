/* byzagg_shards.h — C ABI of libbyzagg for a d-sharded trainer: delivery of the worker gradients to
 * the GPUs that own their columns.  Included at the end of byzagg.h; its conventions apply.
 *
 * On R GPUs with one process each, rank r owns columns [lo_r, hi_r) of every vector, where
 * per = ceil(d / R), lo_r = min(d, r * per) and hi_r = min(d, lo_r + per) (the last shards may be
 * shorter, and are empty wherever r * per >= d: when d < R, but also e.g. rank 3 for d = 9, R = 4).  A trainer backprops worker i on ONE rank; the aggregation rules
 * need columns [lo_r, hi_r) of all n workers on every rank r.  bz_gradient_scatter writes them there;
 * bz_gradient_momentum places the momentum of the owner's rows on its columns.
 */
#ifndef BYZAGG_SHARDS_H
#define BYZAGG_SHARDS_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* attack.py:776-780 / 791-795 for ONE worker gradient on a d-sharded trainer: clip, then write columns
 * [lo_r, hi_r) of the result to dest[r] for r = 0..nranks-1.
 *   grad    device fp32[d], 4-byte aligned, read only
 *   clip    > 0: scale as bz_gradient_row (fp64 norm, fl32(clip / norm), on the device, no host sync);
 *           <= 0: no clipping
 *   dest    HOST array of nranks DEVICE pointers, 1 <= nranks <= BZ_MAX_PEERS: this row's slot on each
 *           rank (hi_r - lo_r floats, 16-byte aligned; may be peer-mapped memory of another GPU).  The
 *           slot of an empty shard is not touched and may be NULL.  Nothing past hi_r - lo_r is written.
 *   ws      needed only with clip > 0 (bz_workspace_bytes(1) suffices)
 *   Bits: dest[r][k] == the sampled row bz_gradient_row writes, at column lo_r + k.
 * Every CTA ends its stores with a system-scope fence, so a stream-ordered barrier after the call
 * (e.g. torch symmetric memory's) publishes the stores that went to peer memory. */
BZ_API int bz_gradient_scatter(const float* grad, int64_t d, double clip, int nranks, float* const* dest,
                               void* ws, size_t ws_bytes, void* stream);

/* attack.py:799-810, the momentum placement, for n rows that are already clipped, in ONE launch: what
 * bz_gradient_row does after the clip (mode 1 / 2, the same per-coordinate arithmetic, hence the same
 * bits), so that the owner of a shard places the momentum of all its rows at once.
 *   rows      HOST array of n DEVICE pointers, 1 <= n <= BZ_MAX_N: the clipped rows, fp32[d] each (read only)
 *   mode 1    worker side: momentum[i] <- momentum[i] * mu + alpha * rows[i], in place; `momentum` is a HOST
 *             array of n DEVICE pointers to n distinct vectors (server and honest are not used)
 *   mode 2    server side: honest[i] <- rows[i] * alpha + mu * server; `honest` is a HOST array of n DEVICE
 *             pointers, `server` a DEVICE fp32[d] (momentum is not used)
 *   alpha = 1 - dampening.  d == 0 (an empty shard) is a no-op whatever the vectors' addresses. */
BZ_API int bz_gradient_momentum(const float* const* rows, int n, int64_t d, int mode, float* const* momentum,
                                const float* server, double mu, double alpha, float* const* honest, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_SHARDS_H */
