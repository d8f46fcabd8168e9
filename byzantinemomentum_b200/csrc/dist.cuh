// dist.cuh — internal interface of the distance-based rules: K2 (pairwise squared
// distances), K2' (row-to-centre squared distances), K5 (scoring / selection) and K4
// (Bulyan reduce).  Workspace layout is private to the library.
#pragma once

#include "common.cuh"

namespace bz {

// ---- workspace ---------------------------------------------------------------------------
// [0, kWsHeader)                       : int32 scratch (order / selection / status when the
//                                        caller passes NULL for them)
// [kWsHeader, kWsHeader + n*n*8)       : reduced block (double[n*n] or double[n])
// [.., + kMaxParts * n*n*8)            : per-CTA partial blocks of K2 / K2'
constexpr size_t kWsHeader = 1024;
constexpr int    kMaxParts = 336;     // >= number of CTAs K2 / K2' ever launch along x (2 per SM) + the group blocks of the fused reduction
size_t workspace_bytes(int n);

// The reference's fp32 `norm()` from the fp64 sum of squares the kernels accumulate: ATen sums in
// fp32, so once the sum passes FLT_MAX the norm is +inf, not the (finite) root of the fp64 sum.
// Otherwise the fp32 rounding of the root.  A NaN sum stays NaN.
__device__ __forceinline__ float fp32_norm(double sum_sq) {
  return isinf((float)sum_sq) ? __int_as_float(0x7f800000) : (float)sqrt(sum_sq);
}

struct Workspace {
  int32_t* order;     // n entries
  int32_t* status;    // 1 entry
  unsigned* ticket;   // 1 entry (last-CTA election of the fused scoring step)
  double*  block;     // n*n
  double*  parts;     // kMaxParts * n*n
};
bool carve_workspace(void* ws, size_t bytes, int n, Workspace& out);

// ---- K2: partial squared pairwise distances -------------------------------------------------
// parts[x*n*n + i*n + j] (i < j) = the share of block x of sum_k (rows[i][k] - rows[j][k])^2, and
// the diagonal entries i == j (sum of (x_i - x_i)^2: 0 or NaN) of the rows the alias map of K5 reads.
// The ring kernel (k2_ring.cu): balanced tasks, distributed TMA issue, clusters + multicast for
// n > 25.  Returns the number of blocks written, <= kMaxParts, or -1 when it cannot run (rows not
// 16-byte aligned, or a launch / occupancy failure).
// Optional scoring / selection step to run inside the distance pass (its last CTA): what the
// caller would otherwise launch as K5.  `fused` is set when the pass did run it; it does not when
// the step's tables do not fit the ring's shared memory.
struct SelectTail {
  int kind;                 // 1 = Multi-Krum order, 2 = Bulyan order + status, 3 = brute subset,
                            // 4 = the reduced block only (phase A of the sharded path): `order` is a double[n*n]
  int n, f, m, count;       // n = ORIGINAL row count
  unsigned long long total; // brute: C(n, n - f)
  const int* to_unique;     // original row -> unique row (NULL: identity)
  int32_t* order;
  int32_t* status;
  unsigned* ticket;         // 128 bytes of device scratch
  int fused;                // out: the pass ran the step
  // distance reuse (optional): old_index[i] = position of ORIGINAL row i in the table of squared
  // distances a previous call left in `cache_in` (u_old x u_old doubles), or -1; the table of this
  // call is written to `cache_out` (u x u).  `reused` is set when only the new rows' pairs were computed.
  const int32_t* old_index;
  const double* cache_in;
  int u_old;
  double* cache_out;
  int reused;
  // fused exchange over peer memory (bz_*_peers): nranks > 0.  By value: the tables hold nranks pointers
  // (this step's slot); `next` (bz_*_peers_next): 2 * nranks, slot 0's then slot 1's, and the kernel takes
  // the epoch and the slot from the flags (peers.cuh, next_epoch); `epoch` is unused
  int nranks, rank;
  unsigned epoch;
  int next;
  double* const* peer_blocks;
  unsigned* const* peer_flags;
};
// star_row >= 0 (no `select`): a star pass without a tail, in the full pass's shape, grid and cluster size: only the
// pairs of row star_row (and the self distances of `self_rows`) are written to the per-cluster blocks, with the bits
// the full pass gives them; every other entry of the blocks is left as it was.  -1 where the star pass cannot run
// (the caller then runs the full pass).
int launch_pairdist_ring(const RowTable& rows, int n, int64_t d, double* parts, cudaStream_t st,
                         const unsigned char* self_rows, int nself, SelectTail* select = nullptr, int star_row = -1);
// Dispatcher used by the rules: `rows` are the u unique rows, `to_unique` (or NULL) maps the n_orig
// original rows to them; the self distance is produced for the unique rows that are aliased.
// Runs the ring, or the cp.async kernel of k2_pairdist.cu when the ring returns -1.
int launch_pairdist_auto(const RowTable& rows, int u, int64_t d, double* parts, cudaStream_t st,
                         const int* to_unique, int n_orig, SelectTail* select = nullptr);
// The unique rows whose self distance is needed (more than one original row maps to them); returns their count.
int aliased_rows(const int* to_unique, int u, int n_orig, unsigned char* self_rows);

// K2': parts[x*n + i] = share of sum_k (rows[i][k] - center[k])^2 (center NULL: the origin).
// order != NULL: the last CTA also sums the blocks and writes the stable order of the n keys
// (sqrt_norm as in bz_rowdist_select) — the selection step without its launch; `ticket`: one zeroed word.
int launch_rowdist(const RowTable& rows, int n, const float* const* host_rows, const float* center, int64_t d,
                   double* parts, cudaStream_t st, int reverse = 0, int32_t* order = nullptr, unsigned* ticket = nullptr,
                   int sqrt_norm = 0, int dot = 0);

// The exchange of K2''s last CTA over peer memory (bz_rowdist_peers, bz_search_score_peers; protocol in
// peers.cuh): this rank's fp64 block (n doubles, or the one score share) goes to block[rank], the flags of
// `epoch` are raised and awaited, and the R blocks are added in rank order, ((p0 + p1) + p2) + ...
struct PeerTail {
  int nranks, rank;
  unsigned epoch;
  int next;                        // 1 (bz_*_peers_next): epoch and slot from the flags (next_epoch), `epoch` unused
  int32_t* status;                 // rowdist: 0, or BZ_STATUS_PEER_TIMEOUT; search: the search's status word,
                                   // set to BZ_STATUS_PEER_TIMEOUT on a timeout after the transition
  double* block[2][BZ_MAX_PEERS];  // [slot][rank]: the slot on every rank ([rank] is local); by value, [0] is
                                   // this step's slot and [1] is unused
  unsigned* flag[2][BZ_MAX_PEERS]; // the same for the flag arrays (nranks words each)
};
// K2' over the rows against `center` (NULL: the origin) in bz_rowdist_partial's geometry, its last CTA
// summing the blocks in k_reduce_parts's order (the block the collective path all-gathers), exchanging
// it, and writing the stable order of the n keys (sqrt_norm as in bz_rowdist_select).  Any d >= 0.
int launch_rowdist_peers(const RowTable& rows, int n, const float* const* host_rows, const float* center, int64_t d,
                         double* parts, cudaStream_t st, int32_t* order, unsigned* ticket, int sqrt_norm,
                         const PeerTail& peers);

// ---- The attacks' line search (bz_line_search, api_search.inc) -------------------------------------
// State of `line_maximize` (tools/misc.py:468-513) in device memory, carried from one evaluation to the next.
struct SearchState {
  double next_x;     // x of the next evaluation (= prop_x after the first)
  double best_x, best_y, delta, prop_x;
  int phase;         // 1 = expansion, 2 = contraction
  unsigned ticket;   // last-CTA election of the score pass; 0 between passes
};
// What the score pass's last CTA does after summing evaluation k's score y.
struct SearchTail {
  SearchState* state;
  double* trace;               // (x_k, y_k) at [2k], [2k + 1]; the chosen factor at [2 * evals]
  const int32_t* eval_status;  // this evaluation's status word (NULL: the rule has none)
  int32_t* status;             // first non-zero status word of the search
  int k, evals;
  double* partial;             // non-NULL (d-sharded search): the score pass writes its fp64 sum here instead
                               // of running the transition (bz_search_step adds the ranks' sums first)
};
// K2' over the one row `out` against `center`, chained by PDL after the rule, its last CTA rounding the
// sum to fp32 (y) and running one transition of the search.  `peers` (d-sharded search, any d >= 0): the
// share is exchanged first and y is fl32 of the R shares added in rank order, as in K9.
int launch_rowdist_search(const float* out, const float* center, int64_t d, double* parts, const SearchTail& tail,
                          cudaStream_t st, const PeerTail* peers = nullptr);
// K8 (k8_candidate.cu): byz <- the candidate row of x (which: 0 = start 0.0, also resets the state's ticket;
// 1 = state->next_x; 2 = state->best_x, the attack's result), chained by PDL.
int launch_candidate(const float* avg, const float* att, float* byz, int64_t d, SearchState* state, int which,
                     int negative, int empire, cudaStream_t st);
// K9 (k9_search_step.cu): one CTA adds the R score partials in rank order, rounds the sum to fp32 (y) and
// runs the transition of evaluation tail.k.
int launch_search_step(const double* partials, int nparts, const SearchTail& tail, cudaStream_t st);

// ---- K6: study metrics in one pass (k6_study.cu) -------------------------------------------------
// avg = (rows[0] + rows[1] + ...)/n; stats[0] = sum avg^2, stats[1] = max |avg|,
// stats[2+i] = sum_k (rows[i][k] - avg[k])^2.  `parts` needs kMaxParts*(n+1) doubles (n >= 2) and
// `bits`: two device scratch words.  The 128-pointer table: kMaxN < n <= kMaxNCoordinate.
void launch_study(const RowTable& rows, int n, const float* const* host_rows, int64_t d, float* avg,
                  double* stats, double* parts, unsigned* bits, cudaStream_t st);
void launch_study(const WideRowTable& rows, int n, const float* const* host_rows, int64_t d, float* avg,
                  double* stats, double* parts, unsigned* bits, cudaStream_t st);

// Sum `nparts` blocks of `len` doubles in index order into `block` (fixed order: deterministic).
// pair_n > 0: the block is a pair_n x pair_n table of which only entries i < j are defined; the
// others are written as 0.  The order: class w = the blocks p = w mod kReduceWarps, each summed in p
// order from 0.0, then the class sums in class order from 0.0 (K2' in peers mode sums its blocks so too).
constexpr int kReduceWarps = 8;
void launch_reduce_parts(const double* parts, int nparts, int len, int pair_n, double* block, cudaStream_t st);

// C(n, n - f), saturating at 2^64 - 1.
inline unsigned long long brute_total(int n, int f) {
  const int k = n - f;
  unsigned long long total = 1;
  for (int i = 1; i <= (k < n - k ? k : n - k); ++i) {
    const unsigned long long num = (unsigned long long)(n - i + 1);
    if (total > (~0ull) / num) return ~0ull;
    total = total * num / i;
  }
  return total;
}

// ---- K5: scoring / selection (single CTA each) --------------------------------------------------
// The scoring step of rule `sel` (kinds 1-3, the fields the distance pass would read) on `nparts`
// blocks; brute's subset limit is the caller's to check.  sel.to_unique / u: optional alias map
// (rows i, j with to_unique[i] == to_unique[j] are the same tensor); the blocks are then u x u
// tables over the unique rows.
void launch_select(const SelectTail& sel, const double* parts, int nparts, cudaStream_t st, int u = 0);
void launch_rowdist_select(const double* parts, int nparts, int n, int sqrt_norm, int32_t* order, cudaStream_t st);

// Same, reading block p IN PLACE from peers[p] (peer GPU memory over NVLink): fused exchange.
void launch_select(const SelectTail& sel, const double* const* peers, int npeers, cudaStream_t st);
void launch_rowdist_select_peers(const double* const* peers, int npeers, int n, int sqrt_norm, int32_t* order, cudaStream_t st);

// ---- K4: Bulyan stage 1 means + coordinate-wise averaged median ----------------------------------
bool launch_bulyan_reduce(const RowTable& rows, int n, int f, int m, const int32_t* order, const int32_t* status,
                          int64_t d, float* out, cudaStream_t st);

// (n, f) with a compile-time specialisation and the default m; false otherwise.
bool launch_bulyan_reduce_static(const RowTable& rows, int n, int f, int m, const int32_t* order, const int32_t* status,
                                 const Geom& g, float* out, cudaStream_t st);

// ---- Above kMaxN rows (bz_distance, api_distance.inc) ----------------------------------------------
// The pairwise distances of u <= kMaxNDistance unique rows come from passes of the 64-row K2: up to kMaxN
// rows one pass over all of them, above that the rows are cut into K = ceil(u / 32) blocks of consecutive
// unique rows (3 or 4, sizes differing by at most one) and every block pair I < J gets one pass over the
// rows of I then J.  A pair across blocks comes from its pass; a pair inside block I, and the self distance
// of an aliased row of I, from the pass (0, 1) for I = 0 and (0, I) otherwise.
constexpr int kMaxNDistance = BZ_MAX_N_DISTANCE;
constexpr int kMaxBlocks = 4;
constexpr int kMaxPasses = kMaxBlocks * (kMaxBlocks - 1) / 2;
constexpr size_t kPassTable = (size_t)kMaxN * kMaxN;     // doubles between two pass tables
struct PassTables {
  const double* table;                        // pass p: size[p] x size[p] squared distances at table + p * kPassTable
  int nblocks, npasses;
  int start[kMaxBlocks + 1];                  // block b: unique rows [start[b], start[b + 1])
  int first[kMaxPasses], size[kMaxPasses];    // pass p: its first block (rows 0 ..) and its row count
  signed char pass[kMaxBlocks][kMaxBlocks];   // the pass that holds the pairs of blocks (a, b)
  unsigned char to_unique[kMaxNDistance];     // original row -> unique row
};
size_t distance_workspace_bytes(int n);

// The squared distance of unique rows a <= b (the self distance when a == b) from the pass that holds it.
__device__ __forceinline__ double pass_sq(const PassTables& t, int a, int b) {
  int ba = 0;
  while (a >= t.start[ba + 1]) ++ba;
  int bb = ba;
  while (b >= t.start[bb + 1]) ++bb;
  const int p = t.pass[ba][bb], f = t.first[p], s = t.size[p];
  const int s0 = t.start[f + 1] - t.start[f];
  const int la = ba == f ? a - t.start[f] : s0 + a - t.start[ba];
  const int lb = bb == f ? b - t.start[f] : s0 + b - t.start[bb];
  return __ldcg(t.table + (size_t)p * kPassTable + (size_t)la * s + lb);
}

// K2 over `u` rows as given, the diagonal entries (self distance) of the rows in self_rows[0, nself) included:
// the ring, or the cp.async kernel when the ring cannot run.  Returns the number of blocks written.
int launch_pairdist_rows(const RowTable& rows, int u, int64_t d, double* parts, cudaStream_t st,
                         const unsigned char* self_rows, int nself, SelectTail* select = nullptr);
// K5 of Multi-Krum (bulyan = 0) or Bulyan on n <= kMaxNDistance rows, reading the pass tables.
void launch_select_wide(const PassTables& t, int n, int count, int32_t* order, int32_t* status, int f, int m, int bulyan,
                        cudaStream_t st);
// K2' over the 128-pointer table with the selection of launch_rowdist (order and ticket required).
int launch_rowdist(const WideRowTable& rows, int n, const float* const* host_rows, const float* center, int64_t d,
                   double* parts, cudaStream_t st, int reverse, int32_t* order, unsigned* ticket, int sqrt_norm);
// K4 over the 128-pointer table, kMaxN < n <= kMaxNDistance; false when theta is outside 33..128.
bool launch_bulyan_reduce_wide(const WideRowTable& rows, int n, int f, int m, const int32_t* order, const int32_t* status,
                               int64_t d, float* out, cudaStream_t st);

// ---- The d-sharded phases above kMaxN rows (bz_distance_partial / _select, api_distance_shards.inc) ----------------
// K2-share: the n x n block of the original rows from the pass tables (entries i < j, the self distance for an
// aliased pair, 0 elsewhere).
void launch_pairshare_wide(const PassTables& t, int n, double* block, cudaStream_t st);
// K2'-share: K2' over the 128-pointer table in launch_rowdist's geometry, its last CTA writing the n sums to `sums`
// (the sums K2' forms its keys from) instead of the order.
int launch_rowshare(const WideRowTable& rows, int n, const float* const* host_rows, const float* center, int64_t d,
                    double* parts, cudaStream_t st, int reverse, unsigned* ticket, double* sums);
// K5 of Multi-Krum (bulyan = 0) or Bulyan from `nparts` gathered n x n blocks, added in rank order.
void launch_blocks_select_wide(const double* parts, int nparts, int n, int count, int32_t* order, int32_t* status, int f,
                               int m, int bulyan, cudaStream_t st);
// The stable order of the n row keys from `nparts` gathered blocks of n sums, added in rank order (sqrt_norm as in
// bz_rowdist_select).
void launch_rowkeys_select_wide(const double* parts, int nparts, int n, int sqrt_norm, int32_t* order, cudaStream_t st);

// ---- The attack against CGE (bz_anticge, api_anticge.inc; k10_anticge.cu) ----------------------------------------
// What K11 does to the attack row: multiply by `factor` when `apply` (anticge.py:75-76).
struct AntiCgeScale {
  float factor;
  int apply;
};
// K10, chained by PDL: out = σ0 + σ0 + σ1 + ... + σ(maxpos-1) (σ = order, device) and the fp64 Σ out² in one pass;
// per-CTA blocks in `parts` (kMaxParts doubles), `ticket` zero on entry and left zero.  nparts_k2 > 0: K2''s
// `nparts_k2` blocks of n sums in `k2_parts` give the key of σ_maxpos and the last CTA writes the decision to `scale`;
// otherwise it writes the sum to `partial`.  Returns 0, or -1 when the launch fails.
int launch_anticge_sum(const RowTable& rows, int n, const float* const* host_rows, int maxpos, const int32_t* order, int64_t d,
                       float* out, double* parts, unsigned* ticket, const double* k2_parts, int nparts_k2,
                       AntiCgeScale* scale, double* partial, cudaStream_t st);
int launch_anticge_sum(const WideRowTable& rows, int n, const float* const* host_rows, int maxpos, const int32_t* order,
                       int64_t d, float* out, double* parts, unsigned* ticket, const double* k2_parts, int nparts_k2,
                       AntiCgeScale* scale, double* partial, cudaStream_t st);
// K11, chained by PDL: out *= factor when the decision says so; the decision is `scale`'s, or (blocks != NULL) formed
// from the `nparts` gathered sums `partials` and the gathered norm blocks `blocks` (nparts x n) by every CTA.
int launch_anticge_scale(float* out, int64_t d, const AntiCgeScale* scale, const double* blocks, const double* partials,
                         int nparts, int n, int maxpos, const int32_t* order, cudaStream_t st);
// out[0, d) = NaN (0x7fc00000).
int launch_nan_fill(float* out, int64_t d, cudaStream_t st);

// ---- libbyzagg_peers.so: phase B above kMaxN rows with the exchange over peer memory (k5_select_peers.cu) ----------
// One CTA: this rank's phase-A block `part` (n x n, entries i < j) copied into its slot, the exchange (`peers`),
// the R blocks added in rank order, then launch_blocks_select_wide's steps; status: the rule's word, then
// BZ_STATUS_PEER_TIMEOUT on a timeout.
void launch_blocks_select_peers(const double* part, int n, int count, int32_t* order, int f, int m, int bulyan,
                                const PeerTail& peers, cudaStream_t st);
// The same from the n sums of Aksel (sqrt_norm = 0) or CGE, with launch_rowkeys_select_wide's steps; status: 0 or
// BZ_STATUS_PEER_TIMEOUT.
void launch_rowkeys_select_peers(const double* part, int n, int sqrt_norm, int32_t* order, const PeerTail& peers,
                                 cudaStream_t st);
// The d-sharded form over peer memory (bz_anticge_peers).  K2'-norms: K2' in CGE mode in bz_distance_partial's
// geometry, its last CTA exchanging phase A's n sums (PeerTail), keeping their R-summed values in parts[0, n) and
// writing the stable order of the keys (bz_distance_select's); `ticket`: one word, zeroed here, left zero.
int launch_anticge_norms(const RowTable& rows, int n, const float* const* host_rows, int64_t d, double* parts, int32_t* order,
                         unsigned* ticket, const PeerTail& peers, cudaStream_t st);
int launch_anticge_norms(const WideRowTable& rows, int n, const float* const* host_rows, int64_t d, double* parts,
                         int32_t* order, unsigned* ticket, const PeerTail& peers, cudaStream_t st);
// K10 as launch_anticge_sum's sharded form, chained by PDL, its last CTA exchanging the partial sum of squares and
// writing the decision to `scale` from the R partials and the kept sums `sums` (n doubles).
int launch_anticge_peers(const RowTable& rows, int n, const float* const* host_rows, int maxpos, const int32_t* order, int64_t d,
                         float* out, double* parts, unsigned* ticket, const double* sums, AntiCgeScale* scale,
                         const PeerTail& peers, cudaStream_t st);
int launch_anticge_peers(const WideRowTable& rows, int n, const float* const* host_rows, int maxpos, const int32_t* order,
                         int64_t d, float* out, double* parts, unsigned* ticket, const double* sums, AntiCgeScale* scale,
                         const PeerTail& peers, cudaStream_t st);

}  // namespace bz
