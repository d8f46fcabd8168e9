/* byzagg_distance_peers.h — C ABI of libbyzagg_peers: phase B of the d-sharded Multi-Krum, Bulyan, Aksel and CGE
 * above BZ_MAX_N rows (byzagg_distance_shards.h) with the exchange of phase A's blocks over peer memory, inside the
 * selection kernel: no collective, no host decision, so a step can be captured in a CUDA graph on any number of
 * ranks.  The calls live in a second library, libbyzagg_peers.so, built next to libbyzagg.so by the same Makefile;
 * the two are composed through their C ABIs.  This header includes byzagg.h for its conventions (return codes,
 * status words, rule codes of byzagg_attack.h); byzagg.h does not include it.
 *
 * A step on every rank is
 *   A  bz_distance_partial (libbyzagg) into a fixed staging buffer `part`: this shard's n x n block (Multi-Krum,
 *      Bulyan; original-row layout, entries i < j) or n sums (Aksel against this shard's median, CGE);
 *   B  bz_distance_select_peers (here): ONE single-CTA kernel copies `part` into this rank's slot of a buffer
 *      mapped on every GPU (peer memory over NVLink / NVSwitch, e.g. torch symmetric memory), raises its flag in
 *      every rank's flag array, waits for every rank's flag (bounded: BZ_STATUS_PEER_TIMEOUT after ~2 s), adds the
 *      R blocks in rank order, ((p0 + p1) + p2) + ..., and runs bz_distance_select's selection on the sum;
 *   C  bz_distance_reduce (libbyzagg) over that selection.
 * The order and the status word are those of bz_distance_select over the all-gathered blocks, bit for bit, on
 * every rank.  The copy into the slot is done here rather than by phase A because a captured phase A has one fixed
 * output pointer, while the slot alternates from one exchange to the next.
 *
 * Arguments:
 *   rule           BZ_RULE_KRUM, BZ_RULE_BULYAN, BZ_RULE_AKSEL or BZ_RULE_CGE; BZ_MAX_N < n <= BZ_MAX_N_DISTANCE.
 *                  Up to BZ_MAX_N rows the exchange runs inside the distance pass instead (bz_krum_peers,
 *                  bz_bulyan_peers, bz_rowdist_peers): BZ_EUNSUPPORTED here
 *   part           DEVICE double[n * n] (Multi-Krum, Bulyan) or double[n] (Aksel, CGE): phase A's block, 8-byte
 *                  aligned; read only
 *   f, m, mode     as bz_distance_select takes them, with its checks
 *   order          DEVICE int32[n], required: bz_distance_select's order
 *   status         DEVICE int32, required: Bulyan's status word as bz_distance_select writes it, 0 for the other
 *                  rules; BZ_STATUS_PEER_TIMEOUT, written after the rule's, when a peer did not show up
 *   rank, nranks   this process; 1 <= nranks <= BZ_MAX_PEERS, 0 <= rank < nranks
 *   peer_blocks    HOST array of nranks DEVICE pointers: this exchange's slot on every rank ([rank] is the local
 *                  one), 8-byte aligned, n * n (pairs) or n (sums) doubles
 *   peer_flags     HOST array of nranks DEVICE pointers: the flag array (nranks uint32) of that slot on every rank;
 *                  zero before the first exchange
 *   epoch          this exchange's number, strictly increasing from one exchange to the next over the same buffer
 *                  (any exchange of bz_krum_peers' protocol), the same on every rank; the caller passes slot
 *                  epoch % 2; wraps at 2^32
 * Every argument is checked before any CUDA call (BZ_EINVAL, BZ_EUNSUPPORTED).
 *
 * bz_distance_select_peers_next takes no epoch and the tables of both slots (2 * nranks entries each: slot 0 on
 * every rank, then slot 1), and derives the epoch from this rank's own flags as byzagg_peers_next.h describes, so
 * that a captured call replays correctly.
 *
 * The slots' lifetime: a rank rewrites slot s at epoch e + 2 only inside a kernel that starts after its kernel of
 * e + 1 (stream order), which waited for every peer's flag of e + 1; a peer raises that flag only after its kernel of
 * e has finished reading s.
 */
#ifndef BYZAGG_DISTANCE_PEERS_H
#define BYZAGG_DISTANCE_PEERS_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The message of the last failed call of libbyzagg_peers in this thread (libbyzagg's bz_last_error() does not see
 * it). */
BZ_API const char* bz_distance_peers_last_error(void);

BZ_API int bz_distance_select_peers(int rule, const double* part, int n, int f, int m, int mode, int32_t* order,
                                    int32_t* status, int rank, int nranks, double* const* peer_blocks,
                                    unsigned* const* peer_flags, unsigned epoch, void* stream);
BZ_API int bz_distance_select_peers_next(int rule, const double* part, int n, int f, int m, int mode, int32_t* order,
                                         int32_t* status, int rank, int nranks, double* const* peer_blocks,
                                         unsigned* const* peer_flags, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_DISTANCE_PEERS_H */
