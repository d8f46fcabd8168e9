// distance_many.cuh — internal interface of libbyzagg_many_distance.so (api_distance_many.cu): the kernels of
// Multi-Krum, Bulyan, Aksel and CGE above kMaxNDistance rows, up to kMaxNMany.
#pragma once

#include "common.cuh"

namespace bz {

// Original row i is unique row to_unique[i] (rows found by address, as dedupe_rows does): a __grid_constant__
// parameter of 2 KB, like the 8 KB ManyRowTable, so that a call copies and allocates nothing.
struct ManyAliasMap {
  unsigned short to_unique[kMaxNMany];
};

// ---- K2-many (k2_many.cu): the pairwise squared distances of u <= kMaxNMany unique rows ---------------------
// Tiles of kPairTile unique rows; CTA (pair p of tiles I <= J, slice s) adds the columns of slice s for every
// (row of I, row of J) and writes one fp64 kPairTile x kPairTile block to parts + (s * npairs + p) * kPairBlock.
constexpr int kPairTile = 64;
constexpr int kPairBlock = kPairTile * kPairTile;
// The most blocks a pass writes at any u <= kMaxNMany (slices x tile pairs, at most one wave or one block per pair):
// the workspace's share of them.
constexpr int kPairTargetCtas = 396;                // three CTAs on each of the H100's 132 SMs; a constant, so
                                                    // that the slices, and with them the bits, do not depend on
                                                    // the device
constexpr int kMaxPairTiles = kMaxNMany / kPairTile;
constexpr int kMaxPairBlocks = kMaxPairTiles * (kMaxPairTiles + 1) / 2 > kPairTargetCtas
                               ? kMaxPairTiles * (kMaxPairTiles + 1) / 2 : kPairTargetCtas;
constexpr int kPairChunk = 32;                      // columns per stage: every fp32 sum holds at most 32 squares
constexpr int kMinSliceChunks = 8;                  // a slice keeps the ring busy for at least 8 chunks
struct PairGrid {
  int tiles, npairs, slices;
  int64_t slice_chunks;                             // 32-column chunks per slice (the last may have fewer)
};
// The slices of K2-many over u unique rows: part of the bit contract (a pair's sum is added slice by slice), so that
// every pass over these rows, K2-star-many's included, takes them from here.
inline PairGrid pair_grid(int u, int64_t d) {
  PairGrid g;
  g.tiles = (u + kPairTile - 1) / kPairTile;
  g.npairs = g.tiles * (g.tiles + 1) / 2;
  const int64_t chunks = (d + kPairChunk - 1) / kPairChunk;
  int64_t slices = kPairTargetCtas / g.npairs;
  const int64_t most = (chunks + kMinSliceChunks - 1) / kMinSliceChunks;
  if (slices > most) slices = most;
  if (slices < 1) slices = 1;
  g.slice_chunks = (chunks + slices - 1) / slices;
  if (g.slice_chunks < 1) g.slice_chunks = 1;
  g.slices = (int)((chunks + g.slice_chunks - 1) / g.slice_chunks);
  if (g.slices < 1) g.slices = 1;
  return g;
}

// Unique rows by address, in order of first appearance (dedupe_rows' numbering), through an open-addressing table.
inline int dedupe_many(const float* const* rows, int n, const float** uniq, unsigned short* to_unique) {
  constexpr int kSlots = 2 * kMaxNMany;
  int slot[kSlots];
  for (int s = 0; s < kSlots; ++s) slot[s] = -1;
  int u = 0;
  for (int i = 0; i < n; ++i) {
    int h = (int)((((uintptr_t)rows[i] >> 2) * 0x9E3779B97F4A7C15ull) >> 53);     // 11 bits
    while (slot[h] >= 0 && uniq[slot[h]] != rows[i]) h = (h + 1) & (kSlots - 1);
    if (slot[h] < 0) {
      slot[h] = u;
      uniq[u++] = rows[i];
    }
    to_unique[i] = (unsigned short)slot[h];
  }
  return u;
}
// K2-many, then the sum of each pair's slices in slice order into table[a * u + b] (a <= b, the diagonal is the
// self distance: 0, or NaN for a row holding NaN / inf).
void launch_pairdist_many(const ManyRowTable& uniq, int u, int64_t d, const PairGrid& g, double* parts, double* table,
                          cudaStream_t st);

// ---- K2-star-many (k2_star_many.cu, in libbyzagg_many_search.so) --------------------------------------------
// Column c = u - 1 of the table over the same u unique rows, the candidate last: table[a * u + c] for a <= c, with
// the bits launch_pairdist_many writes there (the slices of pair_grid(u, d), each slice's chunk sums added in chunk
// order, the slices in slice order).  `blocks` takes one fp64 sum per (slice, row): g.slices * u <= kStarBlocks.
constexpr int kStarBlocks = kPairTargetCtas * kPairTile;
void launch_star_many(const ManyRowTable& uniq, int u, int64_t d, const PairGrid& g, double* blocks, double* table,
                      cudaStream_t st);

// ---- K2'-many (k2_many.cu): one fp64 sum per row over the 1024-pointer table --------------------------------
// Aksel (center != NULL): sum_k (x_i[k] - center[k])^2; CGE: sum_k x_i[k]^2.  Per-CTA blocks of n sums in `parts`
// (kMaxRowParts x n doubles); the last CTA (ticket: one word, zero on entry and left zero) adds them in CTA order
// and writes the stable order of the keys (row_key, sqrt_norm for CGE) to `order`.
constexpr int kMaxRowParts = 264;                   // the grid: two CTAs on each of 132 SMs, whatever the device
void launch_rowkeys_many(const ManyRowTable& rows, int n, const float* center, int64_t d, double* parts, int32_t* order,
                         unsigned* ticket, int sqrt_norm, cudaStream_t st);

// ---- K5-many (k5_many.cu): scoring and selection of Multi-Krum (bulyan = 0) and Bulyan -----------------------
// One warp per row: its n distances through the alias map from the u x u `table`, the rule's compensated sum of
// the `count` smallest into scores[i]; the last CTA (ticket as above) writes the stable order and the status.
void launch_select_many(const double* table, const ManyAliasMap& map, int n, int u, int count, double* scores,
                        int32_t* order, int32_t* status, int f, int m, int bulyan, unsigned* ticket, cudaStream_t st);

// ---- The reduces (k4_many.cu) over the 1024-pointer table of the n original rows ---------------------------
// K3's ordered-subset average: out = (((0 +) r[sel[0]] + r[sel[1]]) + ...) / divisor over `count` rows.
void launch_average_many(const ManyRowTable& rows, const Geom& g, const int32_t* sel, int count, int zero_init,
                         float divisor, float* out, cudaStream_t st);
// K4-many: Bulyan's reduce for m_max = n - f - 2 and theta = n - 2f - 2 up to kMaxNMany - 2.
void launch_bulyan_many(const ManyRowTable& rows, int n, int f, int m, const int32_t* order, const int32_t* status,
                        int64_t d, float* out, cudaStream_t st);

}  // namespace bz
