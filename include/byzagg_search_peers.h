/* byzagg_search_peers.h — C ABI of libbyzagg for the attacks' line search on a d-sharded trainer with its
 * exchanges over peer memory.  Included at the end of byzagg.h; its conventions apply.
 *
 * The same search as byzagg_search_shards.h, but no exchange is a collective: each runs inside the kernel
 * that needs it, with the protocol of bz_krum_peers (byzagg.h).  The last CTA writes this rank's block into
 * its slot of a buffer mapped on every GPU (peer memory over NVLink / NVSwitch, e.g. torch symmetric
 * memory), raises its flag in every rank's flag array, waits for every rank's flag, and adds the R blocks
 * in rank order, ((p0 + p1) + p2) + ...: bitwise the same on every rank.  One evaluation is
 *   1. bz_search_candidate            this rank's columns of the candidate row
 *   2. the rule on honest + [byz] * f_real:
 *        average .. meamed            bz_<rule> on the shard, no exchange
 *        krum, bulyan, brute          bz_pairdist_reuse_peers (distances with reuse, exchange, scoring, reduce)
 *        aksel, cge                   [aksel: bz_median into `out`, the centre] bz_rowdist_peers
 *   3. bz_search_score_peers          this rank's share of the score, exchange, the transition
 * and a last bz_search_candidate (BZ_CANDIDATE_FINAL) writes the Byzantine gradient's shard: two launches
 * of exchange per evaluation for a distance rule, one for the others, no collective and no host decision.
 * The blocks and shares every rank publishes are those the collective path all-gathers, and the R of them
 * are added in the order of its bz_*_select / bz_search_step, so the trace, the factor and the outputs are
 * the collective path's, bit for bit.
 *
 * Common arguments of the exchange (as bz_krum_peers):
 *   rank, nranks   this process; 1 <= nranks <= BZ_MAX_PEERS, 0 <= rank < nranks
 *   peer_blocks    HOST array of nranks DEVICE pointers: this exchange's slot on every rank, 8-byte aligned
 *                  ([rank] is the local one); n*n doubles (bz_pairdist_reuse_peers), n (bz_rowdist_peers), 1
 *                  (bz_search_score_peers).  Alternate between two slots from one exchange to the next.
 *   peer_flags     HOST array of nranks DEVICE pointers: the flag array (nranks uint32) of that slot on every
 *                  rank; zero before the first exchange
 *   epoch          strictly increasing from one exchange to the next (any exchange over the same slots,
 *                  bz_krum_peers' included), the same on every rank for the same exchange; wraps at 2^32
 *   status         DEVICE int32, required: BZ_STATUS_PEER_TIMEOUT when a peer did not show up within ~2 s
 * The epoch is passed by value: a CUDA graph that captured these calls would replay old epochs, so they
 * are not meant for capture.  d == 0 (an empty shard) is a full participant: the rank launches, publishes
 * a zero block (or a 0.0 share), signals, waits and writes the selection, the status and the trace like
 * every other rank; only the reduce pass is skipped.  Its rows and vectors are not read.
 */
#ifndef BYZAGG_SEARCH_PEERS_H
#define BYZAGG_SEARCH_PEERS_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Multi-Krum, Bulyan or brute (rule: BZ_RULE_KRUM, BZ_RULE_BULYAN or BZ_RULE_BRUTE of byzagg_attack.h; m
 * is ignored by brute) on this rank's shard, one evaluation of the search: the distance pass over the
 * unique rows with distance reuse (old_index, cache_in, u_old, cache_out, mode_out as in bz_krum_reuse:
 * cache_out receives THIS rank's u x u table, which the next evaluation's star pass reuses; mode_out 1 =
 * only the new rows' pairs, 0 = full pass), whose last CTA publishes the block in the n x n layout of
 * bz_pairdist_partial_reuse, exchanges it, scores the summed table and writes order / status (as
 * bz_krum_peers: Multi-Krum's status is 0 or BZ_STATUS_PEER_TIMEOUT); the reduce pass of the local shard
 * into `out` follows by programmatic dependent launch.  Rows must be 16-byte aligned (the ring kernel),
 * else BZ_EINVAL before anything is launched.  BZ_EUNSUPPORTED when the scoring step does not fit the
 * ring's shared memory (very few distinct rows among n > 43), after the distance pass was launched. */
BZ_API int bz_pairdist_reuse_peers(int rule, const float* const* rows, int n, int f, int m, int64_t d, float* out,
                                   int32_t* order, int32_t* status, const int32_t* old_index, const double* cache_in,
                                   int u_old, double* cache_out, int* mode_out, int rank, int nranks,
                                   double* const* peer_blocks, unsigned* const* peer_flags, unsigned epoch,
                                   void* ws, size_t ws_bytes, void* stream);

/* Aksel (rule BZ_RULE_AKSEL, mode BZ_AKSEL_*, center = the coordinate-wise median of this rank's rows, which
 * may be `out` itself as in bz_aksel) or CGE (BZ_RULE_CGE, center NULL) on this rank's shard: K2' over the
 * rows, whose last CTA publishes the n-entry block of bz_rowdist_partial, exchanges it, and writes the
 * stable order of the summed keys (bz_rowdist_select's), then the average of the selected rows of the
 * local shard into `out` (bz_aksel's / bz_cge's).  status: 0, or BZ_STATUS_PEER_TIMEOUT.  Any alignment. */
BZ_API int bz_rowdist_peers(int rule, const float* const* rows, int n, int f, int mode, const float* center, int64_t d,
                            float* out, int32_t* order, int32_t* status, int rank, int nranks,
                            double* const* peer_blocks, unsigned* const* peer_flags, unsigned epoch,
                            void* ws, size_t ws_bytes, void* stream);

/* The score pass of evaluation k (bz_search_score_partial's share of sum_k fl32(out_k - avg_k)^2), chained
 * by programmatic dependent launch after the rule, whose last CTA exchanges the share and runs the transition
 * of bz_search_step on the R shares: trace, *status and the state's next x are bz_search_step's, bit for
 * bit.  `status` is the search's status word; a peer timeout sets it to BZ_STATUS_PEER_TIMEOUT after the
 * transition.  eval_status: the rule's status word, or NULL.  ws: bz_workspace_bytes(1) bytes suffice. */
BZ_API int bz_search_score_peers(const float* out, const float* avg, int64_t d, void* state, double* trace,
                                 const int32_t* eval_status, int32_t* status, int k, int evals, int rank, int nranks,
                                 double* const* peer_blocks, unsigned* const* peer_flags, unsigned epoch,
                                 void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_SEARCH_PEERS_H */
