/* byzagg_peers_next.h — C ABI of libbyzagg: the exchanges over peer memory with the epoch taken from the
 * exchange buffer, for CUDA-graph capture.  Included at the end of byzagg.h; its conventions apply.
 *
 * bz_krum_peers, bz_bulyan_peers (byzagg.h), bz_pairdist_reuse_peers, bz_rowdist_peers and
 * bz_search_score_peers (byzagg_search_peers.h) take the exchange's epoch by value, and the caller picks the
 * slot as epoch % 2: a graph that captured them would replay old epochs.  Their _next twins take no epoch.
 * The kernel that runs the exchange derives it from the buffer instead: the epoch is one past the last epoch
 * this rank raised, i.e. the later, wrap-aware as the flag wait compares them, of this rank's own entries
 * ([rank]) in its own flag arrays of the two slots.  A zeroed buffer gives epoch 1.  The slot is that epoch
 * modulo 2.  The kernel reads these flags once every exchanging kernel issued before it on the stream has
 * completed.  From there the exchange is the by-value one: publish the block, raise the flag on every rank,
 * the bounded wait (BZ_STATUS_PEER_TIMEOUT), the rank-order sum; the results are those of the by-value call
 * at the derived epoch, bit for bit.  A captured sequence of _next calls therefore replays correctly, as
 * long as every rank replays the same sequence at the same point of its stream order.
 *
 * Arguments: those of the by-value twin without `epoch`, except
 *   peer_blocks    HOST array of 2 * nranks DEVICE pointers: [s * nranks + r] is slot s on rank r (8-byte
 *                  aligned; [s * nranks + rank] is local), s = 0, 1
 *   peer_flags     HOST array of 2 * nranks DEVICE pointers: [s * nranks + r] is the flag array (nranks uint32)
 *                  of slot s on rank r; zero before the first exchange
 * Bad arguments (rank, NULL or misaligned table entries in either slot, a NULL status word, rows that are not
 * 16-byte aligned for the ring kernel, ...) return BZ_EINVAL with the by-value call's checks, before any CUDA
 * call.
 *
 * By-value and _next calls may be mixed on one buffer, in any order, as long as the by-value epochs continue
 * the flags' sequence: a by-value call after k exchanges from a zeroed buffer passes epoch k + 1 (slot
 * (k + 1) % 2), which is what the _next call would have derived.  That is what a host-side epoch counter
 * does when it adds, after each graph replay, the number of exchanges the graph holds.
 */
#ifndef BYZAGG_PEERS_NEXT_H
#define BYZAGG_PEERS_NEXT_H

#include "byzagg.h"

#ifdef __cplusplus
extern "C" {
#endif

BZ_API int bz_krum_peers_next(const float* const* rows, int n, int f, int m, int64_t d, float* out, int32_t* order,
                              int32_t* status, int rank, int nranks, double* const* peer_blocks,
                              unsigned* const* peer_flags, void* ws, size_t ws_bytes, void* stream);
BZ_API int bz_bulyan_peers_next(const float* const* rows, int n, int f, int m, int64_t d, float* out, int32_t* order,
                                int32_t* status, int rank, int nranks, double* const* peer_blocks,
                                unsigned* const* peer_flags, void* ws, size_t ws_bytes, void* stream);
BZ_API int bz_pairdist_reuse_peers_next(int rule, const float* const* rows, int n, int f, int m, int64_t d, float* out,
                                        int32_t* order, int32_t* status, const int32_t* old_index, const double* cache_in,
                                        int u_old, double* cache_out, int* mode_out, int rank, int nranks,
                                        double* const* peer_blocks, unsigned* const* peer_flags,
                                        void* ws, size_t ws_bytes, void* stream);
BZ_API int bz_rowdist_peers_next(int rule, const float* const* rows, int n, int f, int mode, const float* center, int64_t d,
                                 float* out, int32_t* order, int32_t* status, int rank, int nranks,
                                 double* const* peer_blocks, unsigned* const* peer_flags,
                                 void* ws, size_t ws_bytes, void* stream);
BZ_API int bz_search_score_peers_next(const float* out, const float* avg, int64_t d, void* state, double* trace,
                                      const int32_t* eval_status, int32_t* status, int k, int evals, int rank, int nranks,
                                      double* const* peer_blocks, unsigned* const* peer_flags,
                                      void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BYZAGG_PEERS_NEXT_H */
