/* byzagg_anticge_peers.h — C ABI of libbyzagg: the d-sharded attack against CGE (byzagg_anticge.h) with both of its
 * exchanges over peer memory, inside its kernels: no collective, no host decision.  Included at the end of byzagg.h;
 * its conventions apply.
 *
 * A step is the collective path of byzagg_anticge.h (phases A to D) with each all-gather replaced by the protocol of
 * bz_krum_peers: the last CTA of a kernel writes this rank's block into its slot of a buffer mapped on every GPU
 * (peer memory over NVLink / NVSwitch, e.g. torch symmetric memory), raises its flag in every rank's flag array,
 * waits for every rank's flag, and adds the R blocks in rank order, ((p0 + p1) + p2) + ...:
 *   1. K2' in CGE mode over this shard, whose last CTA publishes the nh sums of squares of bz_distance_partial
 *      (BZ_RULE_CGE), exchanges them (exchange 1), keeps their R-summed values in the workspace and writes the
 *      stable order of bz_distance_select;
 *   2. K10, chained by programmatic dependent launch: this shard of the unscaled attack and its fp64 sum of squares
 *      (bz_anticge_partial's), whose last CTA exchanges that sum (exchange 2) and decides the factor from the R
 *      partials and the kept sums, as bz_anticge_scale does;
 *   3. K11: the shard scaled by that factor.
 * The order, the shard and the factor are the collective path's, bit for bit, on every rank.  The kept sums are
 * what makes this hold: once a rank has signalled exchange 2, a peer may finish it and start the next exchange,
 * which rewrites the slot of exchange 1.
 *
 * Arguments besides bz_anticge's (rows of any alignment, 1 <= nh <= BZ_MAX_N_DISTANCE, ws of
 * bz_anticge_workspace_bytes(nh) bytes; the order is left in the workspace's first nh int32):
 *   status         DEVICE int32, required: 0, or BZ_STATUS_PEER_TIMEOUT when a peer did not show up within ~2 s
 *   rank, nranks   this process; 1 <= nranks <= BZ_MAX_PEERS, 0 <= rank < nranks
 *   peer_blocks    HOST array of 2 * nranks DEVICE pointers: slot 0 on every rank, then slot 1 on every rank
 *                  ([rank] is the local one), 8-byte aligned, nh doubles each at least
 *   peer_flags     HOST array of 2 * nranks DEVICE pointers: the flag arrays (nranks uint32) of those slots, in the
 *                  same layout; zero before the first exchange
 *   epoch          bz_anticge_peers: the epoch of exchange 1, on slot epoch % 2; exchange 2 is epoch + 1, on the
 *                  other slot.  Strictly increasing from one exchange to the next over the same buffer (any
 *                  exchange, bz_krum_peers' and the line search's included), the same on every rank; wraps at 2^32
 * A call uses two epochs, so the next exchange over the buffer is epoch + 2.  bz_anticge_peers_next takes the epoch
 * of exchange 1 from the flags instead (next_epoch, as the bz_*_peers_next calls), so that a CUDA graph can capture it.
 * d == 0 (an empty shard) is a full participant: it publishes a zero block and a 0.0 sum, signals, waits and writes
 * the order and the status like every other rank.  f_real > f_decl: out is filled with NaN and nothing else runs, no
 * exchange and no epoch; every rank has the same f_decl and f_real, so every rank skips the exchanges alike.
 * Every argument is checked before any CUDA call.
 */
#ifndef BYZAGG_ANTICGE_PEERS_H
#define BYZAGG_ANTICGE_PEERS_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

BZ_API int bz_anticge_peers(const float* const* rows, int nh, int f_decl, int f_real, int64_t d, float* out, int32_t* status,
                            int rank, int nranks, double* const* peer_blocks, unsigned* const* peer_flags, unsigned epoch,
                            void* ws, size_t ws_bytes, void* stream);

BZ_API int bz_anticge_peers_next(const float* const* rows, int nh, int f_decl, int f_real, int64_t d, float* out,
                                 int32_t* status, int rank, int nranks, double* const* peer_blocks,
                                 unsigned* const* peer_flags, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_ANTICGE_PEERS_H */
