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
  // fused exchange over peer memory (bz_*_peers): nranks > 0
  int nranks, rank;
  unsigned epoch;
  double* const* peer_blocks;
  unsigned* const* peer_flags;
};
int launch_pairdist_ring(const RowTable& rows, int n, int64_t d, double* parts, cudaStream_t st,
                         const unsigned char* self_rows, int nself, SelectTail* select = nullptr);
// Dispatcher used by the rules: `rows` are the u unique rows, `to_unique` (or NULL) maps the n_orig
// original rows to them; the self distance is produced for the unique rows that are aliased.
// Runs the ring, or the cp.async kernel of k2_pairdist.cu when the ring returns -1.
int launch_pairdist_auto(const RowTable& rows, int u, int64_t d, double* parts, cudaStream_t st,
                         const int* to_unique, int n_orig, SelectTail* select = nullptr);

// K2': parts[x*n + i] = share of sum_k (rows[i][k] - center[k])^2 (center NULL: the origin).
// order != NULL: the last CTA also sums the blocks and writes the stable order of the n keys
// (sqrt_norm as in bz_rowdist_select) — the selection step without its launch; `ticket`: one zeroed word.
int launch_rowdist(const RowTable& rows, int n, const float* const* host_rows, const float* center, int64_t d,
                   double* parts, cudaStream_t st, int reverse = 0, int32_t* order = nullptr, unsigned* ticket = nullptr,
                   int sqrt_norm = 0, int dot = 0);

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
};
// K2' over the one row `out` against `center`, chained by PDL after the rule, its last CTA rounding the
// sum to fp32 (y) and running one transition of the search.
int launch_rowdist_search(const float* out, const float* center, int64_t d, double* parts, const SearchTail& tail,
                          cudaStream_t st);
// K8 (k8_candidate.cu): byz <- the candidate row of x (which: 0 = start 0.0, also resets the state's ticket;
// 1 = state->next_x; 2 = state->best_x, the attack's result), chained by PDL.
int launch_candidate(const float* avg, const float* att, float* byz, int64_t d, SearchState* state, int which,
                     int negative, int empire, cudaStream_t st);

// ---- K6: study metrics in one pass (k6_study.cu) -------------------------------------------------
// avg = (rows[0] + rows[1] + ...)/n; stats[0] = sum avg^2, stats[1] = max |avg|,
// stats[2+i] = sum_k (rows[i][k] - avg[k])^2.  `parts` needs kMaxParts*(n+1) doubles (n >= 2) and
// `bits`: two device scratch words.
void launch_study(const RowTable& rows, int n, const float* const* host_rows, int64_t d, float* avg,
                  double* stats, double* parts, unsigned* bits, cudaStream_t st);

// Sum `nparts` blocks of `len` doubles in index order into `block` (fixed order: deterministic).
// pair_n > 0: the block is a pair_n x pair_n table of which only entries i < j are defined; the
// others are written as 0.
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

}  // namespace bz
