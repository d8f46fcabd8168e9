/* byzagg.h — C ABI of libbyzagg (H100 / sm_90a Byzantine-robust gradient aggregation).
 *
 * Drop-in boundary for the aggregation rules (GARs) of LPD-EPFL/ByzantineMomentum.
 * Each entry point replaces one Python/ATen implementation in the reference (citations
 * are relative to the reference root) and is what the reference's optional `native`
 * hook (`native.<gar>.aggregate`, aggregators/median.py:41-49, krum.py:82-96,
 * bulyan.py:86-100, brute.py:82-91) or an `aggregators.register(...)` plugin binds.
 * The entry points of a d-sharded trainer that are not aggregation rules (delivery of the worker
 * gradients to the GPUs that own their columns, and the owners' momentum placement) are declared in
 * byzagg_shards.h, included at the end.
 *
 * Conventions
 *   - `rows` is a HOST array of n DEVICE pointers; row i is a contiguous fp32 vector of
 *     d elements (the list `gradients` of aggregators/__init__.py:17-21).  Rows may alias
 *     (the f Byzantine entries are one tensor repeated, attacks/identical.py:86) and only
 *     need 4-byte alignment (d-shard views); they are never written.
 *   - `out` is a DEVICE fp32 vector of d elements owned by the caller; it must not overlap
 *     any row (aggregators/__init__.py:21).
 *   - `ws` is a caller-owned DEVICE scratch buffer of at least bz_workspace_bytes(n) bytes,
 *     8-byte aligned; the library allocates no device memory.  One workspace per stream.
 *   - `stream` is a `cudaStream_t` passed as `void*` (NULL = legacy default stream).  All
 *     work is enqueued on it; no entry point synchronises the host.
 *   - `sel` / `order` outputs are DEVICE int32 arrays (may be NULL where stated) so that a
 *     following kernel can consume them without a host round trip.
 *   - `status` is a DEVICE int32 (may be NULL): set to 0 on success or to a BZ_STATUS_* code
 *     when the DATA makes the rule undefined (the reference raises there); `out` is then
 *     filled with NaN.
 *   - Return value: 0 on success, a negative BZ_E* code otherwise; bz_last_error() returns
 *     a thread-local message for the last failure.
 *   - 1 <= n <= bz_max_n() (= 64), d >= 0 (d = 0 is a no-op).  The coordinate-wise rules take up
 *     to 128 rows through bz_coordinate (byzagg_coordinate.h, included at the end), and to 1024 through
 *     bz_coordinate_many (byzagg_coordinate_many.h); up to 128 rows so do
 *     bz_avg_dev_max and bz_line_search with a coordinate-wise rule.  Multi-Krum, Bulyan, Aksel
 *     and CGE take up to 128 rows through bz_distance (byzagg_distance.h, included at the end).
 *   - Parameter validity (f, m ranges) is the caller's job, exactly like the reference's
 *     `check()` functions; the library only rejects what it cannot execute.
 */
#ifndef BYZAGG_H
#define BYZAGG_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define BZ_API __attribute__((visibility("default")))
#else
#define BZ_API
#endif

#define BZ_MAX_N 64
#define BZ_MAX_PEERS 16   /* ranks whose partial blocks one selection kernel can read in place */
#define BZ_CACHE_DOUBLES (BZ_MAX_N * BZ_MAX_N)   /* doubles in a distance-table buffer of the bz_*_reuse calls */

#define BZ_OK            0
#define BZ_EINVAL       -1   /* bad argument (null pointer, n/f/m out of executable range) */
#define BZ_EUNSUPPORTED -2   /* valid for the reference, not executable here (n > BZ_MAX_N, too many subsets) */
#define BZ_ECUDA        -3   /* CUDA runtime error; message in bz_last_error() */
#define BZ_EWORKSPACE   -4   /* workspace too small or misaligned */

#define BZ_STATUS_OK            0
#define BZ_STATUS_NO_FINITE_SET 1  /* brute: every subset holds a non-finite distance (brute.py:67 assert) */
#define BZ_STATUS_DEGENERATE    2  /* bulyan: too few finite scores (bulyan.py:70 fails on gradients[None]) */
#define BZ_STATUS_PEER_TIMEOUT  3  /* bz_*_peers: a peer's block did not arrive within ~2 s (the result is garbage) */

/* Aksel modes (aggregators/aksel.py:43-48) */
#define BZ_AKSEL_MID 0   /* c = (n + 1) / 2 */
#define BZ_AKSEL_NF  1   /* c = n - f       */

BZ_API int         bz_version(void);
BZ_API int         bz_max_n(void);
BZ_API const char* bz_last_error(void);
/* Bytes of device scratch the distance-based rules need for n rows (multiple of 256). */
BZ_API size_t      bz_workspace_bytes(int n);

/* ---- Coordinate-wise rules (shard along d with no collective) ---------------------- */

/* aggregators/average.py:21-29 — ((0 + g0) + g1) + ... then / n, fp32, IEEE division. */
BZ_API int bz_average(const float* const* rows, int n, int64_t d, float* out, void* stream);
/* aggregators/median.py:31-39 — lower median per coordinate, NaN-propagating. */
BZ_API int bz_median(const float* const* rows, int n, int64_t d, float* out, void* stream);
/* aggregators/trmean.py:24-33,69-79 — mean of ranks f..n-f-1 (NaN sorts last), ATen order. */
BZ_API int bz_trmean(const float* const* rows, int n, int f, int64_t d, float* out, void* stream);
/* aggregators/trmean.py:35-50,81-94 — mean of the n-f values closest to the trimmed mean. */
BZ_API int bz_phocas(const float* const* rows, int n, int f, int64_t d, float* out, void* stream);
/* aggregators/trmean.py:35-50,96-109 — mean of the n-f values closest to the median. */
BZ_API int bz_meamed(const float* const* rows, int n, int f, int64_t d, float* out, void* stream);

/* ---- Host buffers in, host buffer out (the reference's `--device-gar` hop, attack.py:811-815 and
 * :824-827: `[g.to(device_gar) for g in gradients]` ... `grad_defense.to(device)`), coordinate-wise rules.
 * The vector is cut into `chunks` column ranges: chunk c+1 is copied host->device on `in_stream` while chunk c
 * is reduced on `stream` and chunk c-1 returns device->host on `out_stream`, so a step costs the H2D time of the
 * rows plus the kernel and the D2H of ONE chunk.  Same result as the whole-vector call (coordinates are
 * independent).  Asynchronous: the result is complete once `stream` is synchronised.
 *   rule        BZ_RULE_*; f is ignored by AVERAGE / MEDIAN
 *   host_rows   n HOST pointers (pinned memory for full PCIe rate; equal pointers are staged once)
 *   host_out    HOST fp32[d]
 *   staging     DEVICE fp32[n][pitch] scratch (pitch >= d, multiple of 4; 64 keeps 256-byte row alignment)
 *   dev_out     DEVICE fp32[d] scratch
 *   in_stream / out_stream  copy streams (may equal `stream`: then everything is serial) */
/* Staging alone (any rule; the same `--device-gar` hop, attack.py:811-815): n HOST rows -> DEVICE staging[k][pitch], as one batched copy when the driver
 * has cudaMemcpyBatchAsync and `stream` is not the legacy default stream, else n cudaMemcpyAsync. */
BZ_API int bz_stage_rows(const float* const* host_rows, int n, int64_t d, float* staging, int64_t pitch, void* stream);
#define BZ_RULE_AVERAGE 0
#define BZ_RULE_MEDIAN  1
#define BZ_RULE_TRMEAN  2
#define BZ_RULE_PHOCAS  3
#define BZ_RULE_MEAMED  4
#define BZ_MAX_HOST_CHUNKS 32
BZ_API int bz_coordinate_host(int rule, const float* const* host_rows, int n, int f, int64_t d, float* host_out,
                              float* staging, int64_t pitch, float* dev_out, int chunks,
                              void* stream, void* in_stream, void* out_stream);

/* ---- Distance-based rules, whole vector on this device ------------------------------ */

/* aggregators/krum.py:31-80 — Multi-Krum.  order (n entries, may be NULL) receives all row
 * indices by increasing score (stable); the first m are the averaged selection. */
BZ_API int bz_krum(const float* const* rows, int n, int f, int m, int64_t d, float* out,
            int32_t* order, void* ws, size_t ws_bytes, void* stream);
/* aggregators/bulyan.py:31-84 — Bulyan over Multi-Krum (scores never updated, :74-76). */
BZ_API int bz_bulyan(const float* const* rows, int n, int f, int m, int64_t d, float* out,
              int32_t* order, int32_t* status, void* ws, size_t ws_bytes, void* stream);
/* aggregators/brute.py:32-80 — minimum-diameter subset of size n-f, then its average.
 * sel (n-f entries, may be NULL) receives the subset, ascending. */
BZ_API int bz_brute(const float* const* rows, int n, int f, int64_t d, float* out,
             int32_t* sel, int32_t* status, void* ws, size_t ws_bytes, void* stream);
/* aggregators/aksel.py:24-64 — average of the c rows closest to the median (squared L2). */
BZ_API int bz_aksel(const float* const* rows, int n, int f, int mode, int64_t d, float* out,
             int32_t* order, void* ws, size_t ws_bytes, void* stream);
/* aggregators/cge.py:28-57 — average of the n-f smallest-norm rows (clone + add_ + div_). */
BZ_API int bz_cge(const float* const* rows, int n, int f, int64_t d, float* out,
           int32_t* order, void* ws, size_t ws_bytes, void* stream);

/* ---- Multi-Krum / Bulyan / brute with distance reuse (SURVEY.md §8(f) row 1) ----------------------
 * attacks/identical.py:68-77 (the attacks' line search) calls the rule up to 16 times per step with
 * the SAME honest tensors and one new Byzantine tensor per evaluation: every honest-honest distance
 * is invariant.  These variants take the table of squared distances a previous call left behind:
 *   old_index  HOST int32[n]: position of rows[i] in that table — the caller vouches that the
 *              row's content is unchanged since — or -1 for a row that was not in it; NULL = no reuse
 *   cache_in   that table, DEVICE double[u_old * u_old] (NULL = none)
 *   cache_out  DEVICE double[BZ_CACHE_DOUBLES], different from cache_in: receives this call's
 *              u x u table over the unique rows (pointer equality, first-appearance order)
 *   mode_out   HOST int: 1 = only the pairs of the new rows were computed (1..4 new unique rows
 *              and the launch geometry of the cached call), 0 = full pass, table written,
 *              -1 = full pass and NO table written (unaligned rows, or the fused tail does not fit)
 * Results are bit-identical to the plain calls: a reused pair has exactly the bits the full pass
 * gives it (same coordinate-to-lane mapping, same summation order). */
BZ_API int bz_krum_reuse(const float* const* rows, int n, int f, int m, int64_t d, float* out, int32_t* order,
                         const int32_t* old_index, const double* cache_in, int u_old, double* cache_out,
                         int* mode_out, void* ws, size_t ws_bytes, void* stream);
BZ_API int bz_bulyan_reuse(const float* const* rows, int n, int f, int m, int64_t d, float* out, int32_t* order,
                           int32_t* status, const int32_t* old_index, const double* cache_in, int u_old,
                           double* cache_out, int* mode_out, void* ws, size_t ws_bytes, void* stream);
BZ_API int bz_brute_reuse(const float* const* rows, int n, int f, int64_t d, float* out, int32_t* sel,
                          int32_t* status, const int32_t* old_index, const double* cache_in, int u_old,
                          double* cache_out, int* mode_out, void* ws, size_t ws_bytes, void* stream);

/* ---- Whole distance rules on a d-shard with the exchange INSIDE the distance pass (one process per GPU)
 * The rank's n x n block of partial squared distances is written by the last CTA of the distance pass
 * straight into this rank's slot of a buffer that is mapped on every GPU (peer memory over NVLink /
 * NVSwitch, e.g. torch symmetric memory); the same CTA raises a flag in every peer's flag array, waits for
 * the peers' flags and adds the R blocks in place from the R GPUs (rank order: bitwise the same table,
 * hence the same selection, on every rank), scores, selects; the reduce pass over the local shard
 * follows by programmatic dependent launch.  Two launches per step, no collective call, no host sync.
 *   rank, nranks   this process; 1 <= nranks <= BZ_MAX_PEERS
 *   peer_blocks    HOST array of nranks DEVICE pointers: the slot of THIS step on every rank (n*n doubles
 *                  each; [rank] is the local one).  Alternate between two slots from step to step.
 *   peer_flags     HOST array of nranks DEVICE pointers: the flag array (nranks uint32) of this step's
 *                  slot on every rank; zero before the first step
 *   epoch          step number: strictly increasing, the same on every rank for the same step (the
 *                  exchanges of byzagg_search_peers.h over the same slots count in the same sequence)
 *   status         DEVICE int32, required: BZ_STATUS_PEER_TIMEOUT when a peer did not show up
 * Rows must be 16-byte aligned (the ring kernel); otherwise BZ_EUNSUPPORTED: use the phases below.
 * The published block is n x n: entry (i, j), i < j, is this shard's sum of squared differences of
 * rows i and j (the same layout on every rank, whichever rows alias), every other entry 0.
 * d == 0 (an empty shard, e.g. the last ranks when d < nranks) is a full participant: the rank
 * publishes a zero block, signals, waits, and writes `order` and `status` like every other rank; only
 * the reduce pass is skipped.  Its rows are not read: neither their addresses nor their aliasing matter. */
BZ_API int bz_krum_peers(const float* const* rows, int n, int f, int m, int64_t d, float* out, int32_t* order,
                         int32_t* status, int rank, int nranks, double* const* peer_blocks,
                         unsigned* const* peer_flags, unsigned epoch, void* ws, size_t ws_bytes, void* stream);
BZ_API int bz_bulyan_peers(const float* const* rows, int n, int f, int m, int64_t d, float* out, int32_t* order,
                           int32_t* status, int rank, int nranks, double* const* peer_blocks,
                           unsigned* const* peer_flags, unsigned epoch, void* ws, size_t ws_bytes, void* stream);

/* ---- Phases for the d-sharded multi-GPU path (SURVEY.md §8(e)) ------------------------
 * Each rank runs phase A on its shard, the R partial blocks are all-gathered (one small
 * collective, done by the host side with torch.distributed/NCCL), phase B sums them in
 * rank order — bitwise identical on every rank — and derives the selection, phase C
 * reduces the local shard. */

/* A: partial squared pairwise distances of the shard: part[i*n+j] (i<j) = sum_k (x_i-x_j)^2,
 *    fp64, other entries 0.  part: device double[n*n]. */
BZ_API int bz_pairdist_partial(const float* const* rows, int n, int64_t d, double* part,
                        void* ws, size_t ws_bytes, void* stream);
/* A': partial squared distance of every row to `center` (device fp32[d], or NULL for the
 *    origin: squared norms).  part: device double[n]. */
BZ_API int bz_rowdist_partial(const float* const* rows, int n, const float* center, int64_t d,
                       double* part, void* ws, size_t ws_bytes, void* stream);
/* B: selections from `nparts` gathered blocks (parts: device double[nparts][n*n] or [nparts][n]).
 *    The blocks are added in rank order, ((p0 + p1) + p2) + ..., for any nparts: the same table, bit
 *    for bit, as the exchange fused into bz_krum_peers / bz_bulyan_peers, hence the same selection. */
BZ_API int bz_krum_select(const double* parts, int nparts, int n, int f, int32_t* order, void* stream);
BZ_API int bz_bulyan_select(const double* parts, int nparts, int n, int f, int m, int32_t* order,
                     int32_t* status, void* stream);
BZ_API int bz_brute_select(const double* parts, int nparts, int n, int f, int32_t* sel,
                    int32_t* status, void* stream);
/* sqrt_norm != 0: keys are fl32(sqrt(sum)) with non-finite -> +inf (cge.py:36-37);
 * sqrt_norm == 0: keys are fl32(sum) (aksel.py:41).  Stable ascending order of the n keys. */
BZ_API int bz_rowdist_select(const double* parts, int nparts, int n, int sqrt_norm, int32_t* order,
                      void* stream);
/* B over PEER MEMORY: same selections (same rank-order sum), but block p is read in place from peers[p], a device
 *    pointer into rank p's memory mapped over NVLink (e.g. torch symmetric memory): the exchange
 *    step is fused into the selection kernel, no all-gather.  peers: HOST array of npeers device
 *    pointers (double[n*n] or double[n] each), npeers <= BZ_MAX_PEERS; the caller orders the
 *    ranks' writes before the reads (a barrier) and the reads before the next overwrite. */
BZ_API int bz_krum_select_peers(const double* const* peers, int npeers, int n, int f, int32_t* order,
                                void* stream);
BZ_API int bz_bulyan_select_peers(const double* const* peers, int npeers, int n, int f, int m,
                                  int32_t* order, int32_t* status, void* stream);
BZ_API int bz_brute_select_peers(const double* const* peers, int npeers, int n, int f, int32_t* sel,
                                 int32_t* status, void* stream);
BZ_API int bz_rowdist_select_peers(const double* const* peers, int npeers, int n, int sqrt_norm,
                                   int32_t* order, void* stream);
/* C: out = (((z + g[sel[0]]) + g[sel[1]]) + ...) / divisor over the local shard; z = 0.0f when
 *    zero_init (Python sum(), krum.py:80) else the first row itself (cge.py:53).  sel: device
 *    int32[count], or NULL for 0..count-1; divisor is rounded to fp32 (normally = count).
 *    status (device, may be NULL): non-zero -> NaN fill. */
BZ_API int bz_average_selected(const float* const* rows, int n, const int32_t* sel, int count,
                        int zero_init, double divisor, const int32_t* status, int64_t d,
                        float* out, void* stream);
/* C (bulyan): stage 1 means over `order` + coordinate-wise averaged median (bulyan.py:64-84). */
BZ_API int bz_bulyan_reduce(const float* const* rows, int n, int f, int m, const int32_t* order,
                     const int32_t* status, int64_t d, float* out, void* stream);

/* ---- Study metrics on the same [n, d] data (tools/pytorch.py:97-125 `compute_avg_dev_max`,
 * called three times per step by attack.py:846-848): avg = (g0 + g1 + ...)/n (clone, add_, div_),
 * stats[0] = sum_k avg[k]^2, stats[1] = max_k |avg[k]|, stats[2+i] = sum_k (g_i[k] - avg[k])^2.
 * avg: device fp32[d]; stats: device double[2+n].  One pass over the rows instead of n+2 with
 * n+2 host syncs; the caller derives norm_avg = sqrt(stats[0]) and
 * norm_dev = sqrt(sum_i stats[2+i] / (n-1)).  1 <= n <= BZ_MAX_N_COORDINATE (128); above 128,
 * BZ_EUNSUPPORTED.  ws: bz_workspace_bytes(n) bytes, which is the same for every n >= 64. */
BZ_API int bz_avg_dev_max(const float* const* rows, int n, int64_t d, float* avg, double* stats,
                          void* ws, size_t ws_bytes, void* stream);

/* ---- Dot products of the study step (attack.py:854-866: 6 cosines + up to 20 dot products with past
 * gradients, each a `torch.dot(...).item()` with its own pass and host sync): out[i] = sum_k rows[i][k] *
 * center[k] for all n rows in ONE pass (fp32 products accumulated in fp32 over <= 32 terms, then fp64;
 * deterministic).  out: device double[n].  The caller reads the results with one copy.  d = 0 writes
 * zeros (center may then be NULL). */
BZ_API int bz_rowdots(const float* const* rows, int n, const float* center, int64_t d, double* out,
                      void* ws, size_t ws_bytes, void* stream);

/* ---- Gradient production (SURVEY.md §8(f) row 2): attack.py:776-780 / 791-795 (clip + clone per
 * worker) and :799-810 (momentum placement) for ONE worker gradient, in one pass.
 *   grad      device fp32[d], the model's flat gradient (read only)
 *   clip      > 0: `if norm > clip: g *= clip / norm` (the norm and the scale stay on the device,
 *             no host sync); <= 0: no clipping
 *   sampled   device fp32[d] or NULL: receives the (clipped) gradient — `grad.clone()`, a row of
 *             the caller's preallocated [n, d] buffer
 *   mode 0    nothing else
 *   mode 1    worker-side momentum: momentum[d] <- momentum * mu + alpha * g'   (in place; the
 *             momentum vector IS the honest gradient the rule reads, attack.py:802-803)
 *   mode 2    server-side momentum: honest[d] <- g' * alpha + mu * momentum     (attack.py:807)
 *   alpha = 1 - dampening.  Bit-exact with the ATen operator sequence (the clip scale to 1 ulp).
 *   ws        needed only with clip > 0 (bz_workspace_bytes(1) suffices). */
BZ_API int bz_gradient_row(const float* grad, int64_t d, double clip, float* sampled, int mode, float* momentum,
                           double mu, double alpha, float* honest, void* ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif

/* Gradient delivery for a d-sharded trainer: bz_gradient_scatter clips one worker gradient and writes
 * each rank's columns into that rank's memory in one pass; bz_gradient_momentum places the momentum
 * of an owner's rows in one launch. */
#include "byzagg_shards.h"

/* The attacks' line search on the device: every evaluation of the rule, its score and the choice of the
 * next factor enqueued back to back, one host read for the outcome. */
#include "byzagg_attack.h"

/* The same search on a d-sharded trainer: each evaluation cut at its exchanges (the rule's partial block,
 * the score's R shares), which the caller all-gathers; every rank then takes the same next factor. */
#include "byzagg_search_shards.h"

/* The same search with every exchange over peer memory inside the kernel that needs it: no collective. */
#include "byzagg_search_peers.h"

/* The coordinate-wise rules (average, median, trimmed mean, Phocas, MeaMed) for up to
 * BZ_MAX_N_COORDINATE = 128 rows: bz_coordinate. */
#include "byzagg_coordinate.h"

/* The same rules for up to BZ_MAX_N_MANY = 1024 rows, each column sorted by a warp: bz_coordinate_many. */
#include "byzagg_coordinate_many.h"

/* The exchanges over peer memory (bz_krum_peers ... bz_search_score_peers) with the epoch taken from the
 * exchange buffer instead of an argument, so that a CUDA graph can capture them: the _next calls. */
#include "byzagg_peers_next.h"

/* Multi-Krum, Bulyan, Aksel and CGE for up to BZ_MAX_N_DISTANCE = 128 rows on one GPU: bz_distance. */
#include "byzagg_distance.h"

/* The phases of the d-sharded path for Multi-Krum, Bulyan, Aksel and CGE up to BZ_MAX_N_DISTANCE rows:
 * bz_distance_partial, bz_distance_select, bz_distance_reduce. */
#include "byzagg_distance_shards.h"

/* The attack against CGE generated on the device for up to BZ_MAX_N_DISTANCE honest rows, on one GPU and on the
 * d-sharded path: bz_anticge, bz_anticge_partial, bz_anticge_scale. */
#include "byzagg_anticge.h"

/* The d-sharded attack against CGE with both of its exchanges over peer memory inside its kernels, and its _next
 * twin for CUDA graphs: bz_anticge_peers, bz_anticge_peers_next. */
#include "byzagg_anticge_peers.h"

#endif /* BYZAGG_H */
