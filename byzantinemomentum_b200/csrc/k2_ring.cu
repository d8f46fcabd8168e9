// k2_ring.cu — K2, second generation: all n(n-1)/2 squared pairwise distances in ONE pass over
// the rows, every input byte fetched from HBM/L2 exactly once for any n <= 64
// (krum.py:44-48, bulyan.py:49-54, brute.py:44-45: one pass PER PAIR plus a host sync each).
//
// What changed against the round-1 kernel (k2_pairdist.cu's layout with one thread issuing every
// bulk copy; that file now holds only the cp.async variant, for rows that are not 16-byte aligned):
//  * Balanced tasks.  Pairs are cut in tasks of 25 accumulator slots: the 5x5 block of two row
//    groups (OFF), or a composite of diagonal blocks (COMP: two whole 5-row blocks, 10 pairs each,
//    plus one 5-cycle of a third block; K5 = two edge-disjoint 5-cycles, so a block split over
//    two composites costs no extra slot).  n = 25: 10 OFF + 2 COMP = 12 equal warps, 3 per SM
//    sub-partition (was 10 heavy + 5 light warps).
//  * Distributed bulk-copy issue.  One thread issuing the n copies of a tile serialises them
//    (dependent constant-bank pointer load, 64-bit add, UBLKCP per copy).  Now row r
//    belongs to one warp which keeps its pointer in a register and issues <= 3 copies per tile,
//    one tile late (the stage freed in the PREVIOUS iteration), so that the `empty` wait before
//    the refill never blocks in steady state.
//  * Thread-block clusters + TMA multicast for n > 25.  12 warps hold 12 tasks of accumulators;
//    n = 51 has 60 tasks.  Instead of several independent CTAs each staging the whole tile
//    (every row read once per CTA), C = ceil(tasks / 12) CTAs of one cluster
//    work on the SAME tile: every row is fetched once per cluster by one CTA and written into the
//    shared memory of all C CTAs by the copy itself (cp.async.bulk ... .multicast::cluster); a
//    consumer releases a stage by arriving on the `empty` barrier of every CTA of the cluster.
//  * Alias flags instead of self pairs: the distance of an aliased row to itself is 0 or NaN
//    (x.sub(x).norm() of a row holding NaN/inf); fma(x, 0, acc) over the row gives the same
//    0 / NaN for 1 operation per coordinate, only for the rows that ARE aliased.
// Arithmetic is unchanged: (a-b)^2 formed directly (no Gram trick), coordinate pairs updated with
// one FADD and one FFMA per coordinate (reduce.cuh), a bounded number of fp32 terms per accumulator
// half, then a transposed warp reduction into fp64.
#include "dist.cuh"
#include "k5_device.cuh"
#include "launch.cuh"
#include "peers.cuh"
#include "reduce.cuh"
#include "tma.cuh"

namespace bz {

constexpr int kG = 5;
constexpr int kRWarps = 12;             // warps (= tasks) per CTA ...
constexpr int kRWarpsSmall = 6;         // ... or 6, two CTAs per SM, when all tasks fit 6 warps (n <= 15): a warp's 25-slot
                                        // task takes the same time per tile whatever n, so small n is bound by tiles per
                                        // SM per unit time, and two resident CTAs walk two tile streams at once
constexpr int kRWarpsWide = 16;         // ... or 16 (four per scheduler, 128 registers) in the clusters of n > 35: the same 60 tasks of
                                        // n = 51 then need 4 CTAs instead of 5
constexpr int kRThreads = kRWarps * 32;
constexpr int kRSlots = kG * kG;
constexpr size_t kRSmemBudget = 226 * 1024;
constexpr int kRMaxCluster = 8;
constexpr int kSelfPerWarp = 3;
constexpr int kTailGroup = 16;           // clusters per first-level group of the fused reduction
constexpr int kTailTickets = 32;         // words of ticket scratch (1 + number of groups)
// fp32 terms per accumulator half between two flushes into fp64.  32: worst-case relative error
// 32 * 2^-24 = 1.9e-6 on one lane partial if every rounding went the same way; the distance tests
// hold the summed distance to rtol = 5e-7 against fp64 (test_cuda_abi.py, test_cuda_depth.py).
// It decides the bits of every distance, which the reuse cache relies on: not a tuning knob.
constexpr int kFlushTerms = 32;

// Unique rows whose distance to themselves is needed (multiplicity > 1), spread over the warps.
struct SelfList {
  unsigned char row[kRWarpsWide * kRMaxCluster * kSelfPerWarp];
  int count;
};

// Scoring / selection run by the LAST CTA to finish (ticket), in the shared memory the ring no
// longer needs: the rule's K5 step without its launch (k5_device.cuh).
struct RingTail {
  int kind;                 // 0 = none, 1 = Multi-Krum order, 2 = Bulyan order + status, 3 = brute subset,
                            // 4 = only the reduced block, in the N x N layout of the original rows, written to
                            //     `order` (a double*)
  int n, f, m, count, slices;
  unsigned long long total; // brute: C(n, n - f)
  int32_t* order;
  int32_t* status;
  unsigned* ticket;         // kTailTickets words, zero before the launch; left at zero
  RowMap map;               // original rows -> unique rows
  // Distance reuse (the attacks' line search, attacks/identical.py:68-77: the same honest rows with a
  // new Byzantine row at every evaluation): `old_index[k]` >= 0 places unique row k in the table of
  // a previous call (`cache_in`, u_old x u_old); pairs of two such rows are taken from it, the pass
  // only computes the pairs of the NEW rows (star tasks).  The assembled table goes to `cache_out`.
  const double* cache_in;
  double* cache_out;
  int u_old;
  signed char old_index[kMaxN];
  // Exchange fused into this launch (d-sharded path, one process per GPU): the last CTA writes the rank's
  // reduced block (from its own table, reuse included) into its slot of a buffer mapped on every GPU (peer
  // memory over NVLink), raises its flag in every peer's flag array, waits for the peers' flags, then adds
  // the R blocks IN PLACE from the R GPUs (plain loads on peer addresses, rank order: bitwise the same
  // table on every rank) and scores.
  int nranks, rank;                       // nranks == 0: single GPU
  unsigned epoch;                         // step number, > the previous step's
  int next;                               // 1 (bz_*_peers_next): epoch and slot from the flags (next_epoch)
  double* peer_block[2][BZ_MAX_PEERS];    // [slot][rank]: the slot on every rank ([rank] is local); by value,
                                          // [0] is this step's slot and [1] is unused
  unsigned* peer_flag[2][BZ_MAX_PEERS];   // the same for the flag arrays (nranks words each)
};

// New rows of a reuse call: star task = one new row against 25 consecutive rows.
constexpr int kStarMax = 4;
struct StarList {
  unsigned char row[kStarMax];
  int count;                // 0: the ordinary pass over all pairs
  int slots;                // rows per star task: 3 or 25
};

// ---- cluster helpers -------------------------------------------------------------------------
__device__ __forceinline__ unsigned cluster_ctarank() {
  unsigned r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// Arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster.
__device__ __forceinline__ void mbar_arrive_remote(unsigned long long* bar, unsigned rank) {
  asm volatile(
      "{\n\t.reg .b32 ra;\n\t"
      "mapa.shared::cluster.u32 ra, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [ra];\n\t}"
      ::"r"(smem_u32(bar)), "r"(rank) : "memory");
}
// ---- tasks -----------------------------------------------------------------------------------
// Task t of ntasks(ng): first the ng(ng-1)/2 OFF blocks (ga < gb, row-major), then the composites:
// composite 2k covers diagonal blocks 5k, 5k+1 (whole) and the identity 5-cycle of 5k+2,
// composite 2k+1 covers 5k+3, 5k+4 (whole) and the second 5-cycle of 5k+2.
struct Task {
  int kind;        // 0 = none, 1 = OFF, 2 = COMP, 3 = STAR
  int g0, g1, g2;  // OFF: (ga, gb, -); COMP: (X, Y, Z) group indices, -1 = absent; STAR: (pivot row, first group, -)
  int perm;        // COMP: Z rows walked in the order 0,2,4,1,3
};
__host__ __device__ inline int ring_ncomp(int ng) {
  const int r = ng % 5;
  return 2 * (ng / 5) + (r == 0 ? 0 : r <= 2 ? 1 : 2);
}
__host__ __device__ inline int ring_ntasks(int ng) { return ng * (ng - 1) / 2 + ring_ncomp(ng); }

__device__ __forceinline__ Task make_task(int t, int ng) {
  Task k{0, -1, -1, -1, 0};
  const int noff = ng * (ng - 1) / 2;
  if (t < noff) {
    int ga = 0, r = t;
    while (r >= ng - 1 - ga) { r -= ng - 1 - ga; ++ga; }
    k.kind = 1; k.g0 = ga; k.g1 = ga + 1 + r;
  } else if (t < noff + ring_ncomp(ng)) {
    const int c = t - noff, base = 5 * (c >> 1);
    k.kind = 2;
    k.perm = c & 1;
    const int x = base + (k.perm ? 3 : 0), y = base + (k.perm ? 4 : 1), z = base + 2;
    k.g0 = x < ng ? x : -1;
    k.g1 = y < ng ? y : -1;
    k.g2 = z < ng ? z : -1;
  }
  return k;
}
// The 5-cycle 0-1-2-3-4-0: slot e pairs local rows (cyc_a[e], cyc_b[e]) of the walked order.
__device__ __forceinline__ int zperm(int i, int perm) { return perm ? ((2 * i) % 5) : i; }   // 0,2,4,1,3

// ---- sweeps: one staged tile, this warp's task -------------------------------------------------
template <int T>
__device__ __forceinline__ void sweep_off(const float* a_base, const float* b_base, int lane, u64 (&acc)[kRSlots]) {
#pragma unroll
  for (int c = 0; c < T; c += 128) {
    u64 a0[kG], a1[kG], b0[kG], b1[kG];
#pragma unroll
    for (int i = 0; i < kG; ++i) {
      const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(a_base + i * T + c + lane * 4);
      a0[i] = t.x; a1[i] = t.y;
    }
#pragma unroll
    for (int j = 0; j < kG; ++j) {
      const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(b_base + j * T + c + lane * 4);
      b0[j] = t.x; b1[j] = t.y;
    }
#pragma unroll
    for (int i = 0; i < kG; ++i)
#pragma unroll
      for (int j = 0; j < kG; ++j) {
        const u64 d0 = sub2(a0[i], b0[j]), d1 = sub2(a1[i], b1[j]);
        acc[i * kG + j] = fma2(d0, d0, acc[i * kG + j]);
        acc[i * kG + j] = fma2(d1, d1, acc[i * kG + j]);
      }
  }
}

template <int T>
__device__ __forceinline__ void sweep_comp(const float* x_base, const float* y_base, const float* z_base, int perm, int lane,
                                           u64 (&acc)[kRSlots]) {
  const int z1 = zperm(1, perm) * T, z2 = zperm(2, perm) * T, z3 = zperm(3, perm) * T, z4 = zperm(4, perm) * T;
#pragma unroll
  for (int c = 0; c < T; c += 128) {
    const int o = c + lane * 4;
    {
      u64 a0[kG], a1[kG];
#pragma unroll
      for (int i = 0; i < kG; ++i) {
        const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(x_base + i * T + o);
        a0[i] = t.x; a1[i] = t.y;
      }
      int p = 0;
#pragma unroll
      for (int i = 0; i < kG; ++i)
#pragma unroll
        for (int j = i + 1; j < kG; ++j) {
          const u64 d0 = sub2(a0[i], a0[j]), d1 = sub2(a1[i], a1[j]);
          acc[p] = fma2(d0, d0, acc[p]);
          acc[p] = fma2(d1, d1, acc[p]);
          ++p;
        }
    }
    {
      u64 a0[kG], a1[kG];
#pragma unroll
      for (int i = 0; i < kG; ++i) {
        const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(y_base + i * T + o);
        a0[i] = t.x; a1[i] = t.y;
      }
      int p = 10;
#pragma unroll
      for (int i = 0; i < kG; ++i)
#pragma unroll
        for (int j = i + 1; j < kG; ++j) {
          const u64 d0 = sub2(a0[i], a0[j]), d1 = sub2(a1[i], a1[j]);
          acc[p] = fma2(d0, d0, acc[p]);
          acc[p] = fma2(d1, d1, acc[p]);
          ++p;
        }
    }
    {
      u64 a0[kG], a1[kG];
      const int zo[kG] = {0, z1, z2, z3, z4};
#pragma unroll
      for (int i = 0; i < kG; ++i) {
        const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(z_base + zo[i] + o);
        a0[i] = t.x; a1[i] = t.y;
      }
#pragma unroll
      for (int e = 0; e < kG; ++e) {
        const int i = (e < 4) ? e : 0, j = (e < 4) ? e + 1 : 4;
        const u64 d0 = sub2(a0[i], a0[j]), d1 = sub2(a1[i], a1[j]);
        acc[20 + e] = fma2(d0, d0, acc[20 + e]);
        acc[20 + e] = fma2(d1, d1, acc[20 + e]);
      }
    }
  }
}

// STAR: the pivot row against NS consecutive rows (NS = 3: a new row's pairs spread over many warps, so
// that a reuse pass is bound by the staging of the rows, not by one warp's 25 pairs; NS = 25 when there
// are too few warps for that).  Each pair goes through exactly the operations it goes through in an
// OFF / COMP task — same lane, same steps, (a-b)^2 = (b-a)^2 bit for bit — so a distance computed here
// equals the one the full pass would produce.  Slots past `valid` re-read the first row (in bounds).
template <int T, int NS>
__device__ __forceinline__ void sweep_star(const float* x_base, const float* r_base, int valid, int lane, u64 (&acc)[kRSlots]) {
#pragma unroll
  for (int c = 0; c < T; c += 128) {
    const int o = c + lane * 4;
    const ulonglong2 x = *reinterpret_cast<const ulonglong2*>(x_base + o);
#pragma unroll
    for (int p = 0; p < NS; ++p) {
      const ulonglong2 r = *reinterpret_cast<const ulonglong2*>(r_base + (p < valid ? p : 0) * T + o);
      const u64 d0 = sub2(x.x, r.x), d1 = sub2(x.y, r.y);
      acc[p] = fma2(d0, d0, acc[p]);
      acc[p] = fma2(d1, d1, acc[p]);
    }
  }
}

template <int T>
__device__ __forceinline__ void sweep_self(const float* stage, const int (&srow)[kSelfPerWarp], int nself, int lane, u64 (&facc)[kSelfPerWarp]) {
#pragma unroll
  for (int q = 0; q < kSelfPerWarp; ++q) {
    if (q < nself) {
      const float* row = stage + srow[q] * T + lane * 4;
#pragma unroll
      for (int c = 0; c < T; c += 128) {
        const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(row + c);
        facc[q] = fma2(t.x, 0ull, facc[q]);       // x * 0 + acc: 0 for finite x, NaN for NaN / inf
        facc[q] = fma2(t.y, 0ull, facc[q]);
      }
    }
  }
}

__device__ __forceinline__ void ring_flush(u64 (&acc)[kRSlots], int lane, double& dacc) {
  float v[32];
#pragma unroll
  for (int p = 0; p < 32; ++p) v[p] = (p < kRSlots) ? half_sum(acc[p]) : 0.f;
#pragma unroll
  for (int p = 0; p < kRSlots; ++p) acc[p] = 0ull;
  dacc += (double)transpose_reduce(v, lane);
}

// Cooperative staging of one (ragged) tile with cp.async, zero fill past d (rows 16-byte aligned).
template <int T, int THREADS>
__device__ __forceinline__ void ring_stage_tail(float* buf, const RowTable& rows, int n, int64_t base, int64_t d) {
  constexpr int Q = T / 4;
  for (int q = threadIdx.x; q < n * Q; q += THREADS) {
    const int r = q / Q, cq = q - r * Q;
    const float* row = rows.p[r];
    const int64_t col = base + (int64_t)cq * 4;
    const int64_t remain = d - col;
    const int bytes = remain >= 4 ? 16 : (remain > 0 ? (int)remain * 4 : 0);
    const unsigned s = smem_u32(buf + r * T + cq * 4);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(bytes ? row + col : row), "r"(bytes) : "memory");
  }
}

// One CTA = 12 warps = 12 tasks; a cluster of C CTAs covers tasks [0, 12 C) of the same tiles.
// parts[cluster * n * n + i * n + j] (i < j; i == j for the rows of `self`).
template <int T, int STAGES, bool SELF, bool CLUSTER, int W>
__global__ void __launch_bounds__(W * 32, W == kRWarpsSmall ? 2 : 1)
k2_ring(const __grid_constant__ RowTable rows, const __grid_constant__ SelfList self, const __grid_constant__ RingTail tail,
        const __grid_constant__ StarList star, const int n, const int csize, const int64_t d, const int64_t nfull,
        double* __restrict__ parts) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr int kThreads = W * 32;
  // (No early `pdl_trigger()` here: A/B on one box, krum n = 25: 71.0 us with it, 65.9 without, 1394 vs 1296 us at
  // d = 36.5M — the reduce pass's CTAs scheduled on the SMs that finish first only get in the way.  K3 / K4 are still
  // launched with the programmatic attribute: they start when the last CTA of this grid exits.)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ng = (n + kG - 1) / kG;
  const int rows_alloc = ng * kG;
  const int stage_floats = rows_alloc * T;
  float* stages = reinterpret_cast<float*>(smem_raw);
  unsigned long long* full = reinterpret_cast<unsigned long long*>(smem_raw + (size_t)STAGES * stage_floats * sizeof(float));
  unsigned long long* empty = full + STAGES;
  const int rank = CLUSTER ? (int)cluster_ctarank() : 0;
  const int C = CLUSTER ? csize : 1;
  const int cluster_id = CLUSTER ? (int)(blockIdx.x / C) : (int)blockIdx.x;
  const int nclusters = CLUSTER ? (int)(gridDim.x / C) : (int)gridDim.x;

  Task task;
  if (star.count == 0) {
    task = make_task(rank * W + warp, ng);
  } else {
    // reuse call: star task t = (new row t / chunks, rows [slots (t % chunks), + slots)); g1 = first ROW here
    const int chunks = (n + star.slots - 1) / star.slots, t = rank * W + warp;
    task = Task{0, -1, -1, -1, 0};
    if (t < star.count * chunks) { task.kind = 3; task.g0 = star.row[t / chunks]; task.g1 = (t % chunks) * star.slots; }
  }
  // Rows this warp brings in: global issue slot q = r mod (12 C) -> CTA q mod C, warp q / C
  const int slot = warp * C + rank;
  const int stride = W * C;
  const float* my_row[3];
  int my_idx[3];
  int nmine = 0;
#pragma unroll
  for (int q = 0; q < 3; ++q) {
    const int r = slot + q * stride;
    my_idx[q] = r;
    my_row[q] = rows.p[r < n ? r : 0];
    if (r < n) nmine = q + 1;
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full[s], 1);            // ONE arrival (thread 0) carrying the expected bytes of the whole tile; the copies
                                         // are issued by the warps that own the rows, in this CTA and in its peers, and may
                                         // complete before that arrival (the transaction count is signed)
      mbar_init(&empty[s], W * C);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (CLUSTER) cluster_sync_all(); else __syncthreads();

  // Loop bookkeeping in 32-bit counters (the 64-bit `k % STAGES` of the first version cost ~10 % of
  // the issue slots): stage / parity advance incrementally, source pointers advance by one stride.
  const int mine = (nfull > (int64_t)cluster_id) ? (int)((nfull - 1 - cluster_id) / nclusters) + 1 : 0;
  constexpr unsigned row_bytes = T * sizeof(float);
  const unsigned short mask = (unsigned short)((1u << C) - 1u);
  const size_t tile_stride = (size_t)nclusters * T;
  const float* src0 = my_row[0] + (size_t)cluster_id * T;
  const float* src1 = my_row[1] + (size_t)cluster_id * T;
  const float* src2 = my_row[2] + (size_t)cluster_id * T;
  const unsigned stage_bytes = (unsigned)stage_floats * sizeof(float);
  const unsigned smem0 = smem_u32(stages), full0 = smem_u32(full), empty0 = smem_u32(empty);
  const unsigned dst0 = (unsigned)my_idx[0] * row_bytes, dst1 = (unsigned)my_idx[1] * row_bytes, dst2 = (unsigned)my_idx[2] * row_bytes;
  auto copy_row = [&](unsigned dst, const float* src, unsigned bar) {
    if (CLUSTER)
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
                   ::"r"(dst), "l"(src), "r"(row_bytes), "r"(bar), "h"(mask) : "memory");
    else
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                   ::"r"(dst), "l"(src), "r"(row_bytes), "r"(bar) : "memory");
  };
  auto refill = [&](int s) {         // lane 0: announce (warp 0) and bring this warp's rows of the next tile into stage s
    const unsigned bar = full0 + 8u * (unsigned)s, base = smem0 + (unsigned)s * stage_bytes;
    if (warp == 0)
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"((unsigned)n * row_bytes) : "memory");
    if (nmine > 0) { copy_row(base + dst0, src0, bar); src0 += tile_stride; }
    if (nmine > 1) { copy_row(base + dst1, src1, bar); src1 += tile_stride; }
    if (nmine > 2) { copy_row(base + dst2, src2, bar); src2 += tile_stride; }
  };
  const bool refiller = lane == 0 && (nmine > 0 || warp == 0);
  int issued = mine < STAGES ? mine : STAGES;
  if (refiller)
    for (int k = 0; k < issued; ++k) refill(k);

  u64 acc[kRSlots];
#pragma unroll
  for (int p = 0; p < kRSlots; ++p) acc[p] = 0ull;
  double dacc = 0.;
  u64 facc[kSelfPerWarp] = {0ull, 0ull, 0ull};
  int srow[kSelfPerWarp] = {0, 0, 0};
  int nself = 0;
  if (SELF) {
    const int gw = rank * W + warp;     // entry e of the list belongs to warp e mod (12 C)
#pragma unroll
    for (int q = 0; q < kSelfPerWarp; ++q)
      if (gw + q * W * C < self.count) { srow[q] = self.row[gw + q * W * C]; nself = q + 1; }
  }
  // shared-memory offsets of the task's row groups (absent groups read group 0: discarded)
  const int o0 = task.kind == 3 ? task.g0 * T : (task.g0 >= 0 ? task.g0 : 0) * kG * T;
  const int o1 = task.kind == 3 ? task.g1 * T : (task.g1 >= 0 ? task.g1 : 0) * kG * T;
  const int star_valid = task.kind == 3 ? min(star.slots, n - task.g1) : 0;
  const int o2 = (task.g2 >= 0 ? task.g2 : 0) * kG * T;
  // fp32 terms per accumulator half between two flushes into fp64 (a tile adds T / 64 of them)
  constexpr int kFlushTiles = (kFlushTerms * 64) / T;
  static_assert(kFlushTiles >= 1, "kFlushTerms");

  int pending = 0;
  int s = 0, sp = 0;
  unsigned parity = 0, pp = 0;
  // (Two tiles per loop iteration with a blocking refill — half the bookkeeping — was measured SLOWER:
  // 62 vs 52 us at n = 25, d = 1.31M: every iteration then waits for the slowest warp of the CTA.)
  for (int k = 0; k < mine; ++k) {
    mbar_wait(&full[s], parity);
    const float* buf = stages + (size_t)s * stage_floats;
    if (task.kind == 1)      sweep_off<T>(buf + o0, buf + o1, lane, acc);
    else if (task.kind == 2) sweep_comp<T>(buf + o0, buf + o1, buf + o2, task.perm, lane, acc);
    else if (task.kind == 3) {
      if (star.slots == 3) sweep_star<T, 3>(buf + o0, buf + o1, star_valid, lane, acc);
      else                 sweep_star<T, kRSlots>(buf + o0, buf + o1, star_valid, lane, acc);
    }
    if (SELF && nself > 0) sweep_self<T>(buf, srow, nself, lane, facc);
    __syncwarp();
    if (lane == 0) {
      // the values read from the stage have been consumed by the arithmetic above: a plain
      // (relaxed) arrive is enough to hand the stage back; `.release.cluster` here would add a
      // fence (MEMBAR) per arrive
      if (!CLUSTER) mbar_arrive(&empty[s]);
      else
        for (int r = 0; r < C; ++r) mbar_arrive_remote(&empty[s], (unsigned)r);
    }
    if (task.kind != 0 && ++pending == kFlushTiles) { pending = 0; ring_flush(acc, lane, dacc); }
    // refill the stage released one iteration ago (every warp of the cluster is past it by now)
    if (refiller && k >= 1 && issued < mine) {
      mbar_wait(&empty[sp], pp);
      refill(sp);
      ++issued;
    }
    sp = s; pp = parity;
    if (++s == STAGES) { s = 0; parity ^= 1u; }
  }
  // Ragged tail tile (d not a multiple of T): cooperative staging with zero fill; every CTA of the
  // owning cluster stages it for itself (its own tasks)
  const int64_t ntiles = (d + T - 1) / T;
  if (ntiles > nfull && (nfull % nclusters) == cluster_id) {
    __syncthreads();                 // this CTA's ring is drained: every tile issued (here or by a peer) was awaited above
    ring_stage_tail<T, kThreads>(stages, rows, n, nfull * T, d);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    if (task.kind == 1)      sweep_off<T>(stages + o0, stages + o1, lane, acc);
    else if (task.kind == 2) sweep_comp<T>(stages + o0, stages + o1, stages + o2, task.perm, lane, acc);
    else if (task.kind == 3) {
      if (star.slots == 3) sweep_star<T, 3>(stages + o0, stages + o1, star_valid, lane, acc);
      else                 sweep_star<T, kRSlots>(stages + o0, stages + o1, star_valid, lane, acc);
    }
    if (SELF && nself > 0) sweep_self<T>(stages, srow, nself, lane, facc);
    pending = 1;
  }
  if (task.kind != 0 && pending > 0) ring_flush(acc, lane, dacc);

  double* block = parts + (size_t)cluster_id * n * n;
  if (task.kind == 1) {
    const int i = lane / kG, j = lane % kG;
    const int ri = task.g0 * kG + i, rj = task.g1 * kG + j;
    if (lane < kRSlots && ri < n && rj < n) block[(size_t)ri * n + rj] = dacc;
  } else if (task.kind == 2) {
    int g = -1, i = 0, j = 0;
    if (lane < 20) {
      const int p = lane < 10 ? lane : lane - 10;
      g = lane < 10 ? task.g0 : task.g1;
      i = (p >= 9) ? 3 : (p >= 7) ? 2 : (p >= 4) ? 1 : 0;
      const int first = (i == 0) ? 0 : (i == 1) ? 4 : (i == 2) ? 7 : 9;
      j = p - first + i + 1;
    } else if (lane < kRSlots) {
      const int e = lane - 20;
      g = task.g2;
      const int a = zperm((e < 4) ? e : 0, task.perm), b = zperm((e < 4) ? e + 1 : 4, task.perm);
      i = min(a, b); j = max(a, b);
    }
    if (g >= 0) {
      const int ri = g * kG + i, rj = g * kG + j;
      if (ri < n && rj < n) block[(size_t)ri * n + rj] = dacc;
    }
  }
  else if (task.kind == 3) {
    const int r = task.g1 + lane;
    if (lane < star_valid && r != task.g0) block[(size_t)min(r, task.g0) * n + max(r, task.g0)] = dacc;
  }
  if (SELF) {
#pragma unroll
    for (int q = 0; q < kSelfPerWarp; ++q) {
      if (q < nself) {
        float v = half_sum(facc[q]);
#pragma unroll
        for (int h = 16; h >= 1; h >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, h));
        if (lane == 0) block[(size_t)srow[q] * n + srow[q]] = (double)v;
      }
    }
  }
  if (tail.kind != 0) {
    // Two-level, fixed-order reduction of the per-cluster blocks followed by the scoring step, all
    // inside this launch.  One CTA pulling one block per cluster alone is bandwidth-starved
    // (a single SM pulls ~740 KB at n = 25), so the blocks are first summed by groups of kTailGroup clusters
    // — by whichever CTA of the group finishes last, but always in index order: deterministic —
    // and the last group to finish sums the <= 10 group blocks and runs the selection in the
    // shared memory the ring no longer needs (every other CTA is past its ring by then).
    __shared__ int elected;
    __shared__ int peer_timeout;
    if (threadIdx.x == 0) peer_timeout = 0;
    const int len = n * n;
    const int ngroups = (nclusters + kTailGroup - 1) / kTailGroup;
    const int group = cluster_id / kTailGroup;
    const int first = group * kTailGroup;
    const int members = min(kTailGroup, nclusters - first);
    double* gblocks = parts + (size_t)nclusters * len;            // behind the per-cluster blocks
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) elected = (atomicAdd(tail.ticket + 1 + group, 1u) == (unsigned)(members * C) - 1u) ? 1 : 0;
    __syncthreads();
    if (elected) {
      __threadfence();
      for (int e = threadIdx.x; e < len; e += kThreads) {
        double v[kTailGroup];
#pragma unroll
        for (int p = 0; p < kTailGroup; ++p) v[p] = (p < members) ? __ldcg(parts + (size_t)(first + p) * len + e) : 0.;
        double sum = v[0];
#pragma unroll
        for (int p = 1; p < kTailGroup; ++p) sum += v[p];          // + 0.0 past `members`: exact
        gblocks[(size_t)group * len + e] = sum;
      }
      __threadfence();
      __syncthreads();
      if (threadIdx.x == 0) elected = (atomicAdd(tail.ticket, 1u) == (unsigned)ngroups - 1u) ? 1 : 0;
      __syncthreads();
      if (elected) {
        __threadfence();
        double* sm = reinterpret_cast<double*>(smem_raw);
        if (tail.kind == 4) {
          // Phase A of the d-sharded path: this rank's reduced block.  The u x u table over the unique rows
          // first (pairs of two rows of a previous table from `cache_in`, every other pair and the alias
          // flags on the diagonal from this pass, group blocks added in index order), kept in `cache_out`
          // when asked; then the block in the N x N layout of the original rows, as the exchange below
          // publishes it: entry (i, j), i < j, is the pair of their distinct rows (the alias flag when both
          // are one tensor), every other entry 0.
          const int N = tail.n;
          const RowMap& map = tail.map;
          for (int e = threadIdx.x; e < len; e += kThreads) {
            const int i = e / n, j = e - i * n;
            double v = 0.;
            if (i <= j) {
              const int oi = tail.old_index[i], oj = tail.old_index[j];
              if (i < j && tail.cache_in != nullptr && oi >= 0 && oj >= 0) {
                v = __ldcg(tail.cache_in + (size_t)min(oi, oj) * tail.u_old + max(oi, oj));
              } else {
                for (int g = 0; g < ngroups; ++g) v += __ldcg(gblocks + (size_t)g * len + e);
              }
            }
            sm[e] = v;
            if (tail.cache_out != nullptr) tail.cache_out[e] = v;
          }
          __syncthreads();
          double* out_block = reinterpret_cast<double*>(tail.order);
          for (int e = threadIdx.x; e < N * N; e += kThreads) {
            const int i = e / N, j = e - i * N;
            double v = 0.;
            if (i < j) {
              const int a = map.to_unique[i], b = map.to_unique[j];
              v = sm[min(a, b) * n + max(a, b)];
            }
            out_block[e] = v;
          }
        } else {
          // The summed u x u table, group blocks added in index order (canonical: a pair has the same
          // bits whether it comes out of a full pass, a star pass or the cache), assembled where the
          // scoring code expects it; diagonal entries (alias flags) always come from this pass.
          const int N = tail.n;
          const bool exchange = tail.nranks > 0;
          double* table = sm + (n == N || exchange ? 0 : (size_t)N * N);
          RowMap map = tail.map;
          if (exchange) {
            // ---- exchange over peer memory, inside this launch ----
            // The block is published in the N x N layout of the original rows: entry (i, j), i < j, is the
            // pair of their distinct rows (the alias flag when both are one tensor), every other entry 0.
            // That layout is the same on every rank whatever its rows alias — a rank with an empty shard
            // cannot tell, an empty tensor has no address — and holds nothing the workspace left behind.
            // This rank's u x u table first, as the plain pass below builds it (reuse included), kept in
            // `cache_out` when asked: this rank's own pairs, which the next call's star pass reuses.
            const int NN = N * N;
            double* local = sm + NN;            // behind the N x N table the exchange sums into
            for (int e = threadIdx.x; e < len; e += kThreads) {
              const int i = e / n, j = e - i * n;
              double v = 0.;
              if (i <= j) {
                const int oi = tail.old_index[i], oj = tail.old_index[j];
                if (i < j && tail.cache_in != nullptr && oi >= 0 && oj >= 0) {
                  v = __ldcg(tail.cache_in + (size_t)min(oi, oj) * tail.u_old + max(oi, oj));
                } else {
                  for (int g = 0; g < ngroups; ++g) v += __ldcg(gblocks + (size_t)g * len + e);
                }
              }
              local[e] = v;
              if (tail.cache_out != nullptr) tail.cache_out[e] = v;
            }
            // the epoch and the slot: by value, or (`next`) from this rank's own flags, read by every thread
            // before the barrier that precedes the signal
            unsigned epoch = tail.epoch;
            int slot = 0;
            if (tail.next) {
              epoch = next_epoch(tail.peer_flag[0][tail.rank] + tail.rank, tail.peer_flag[1][tail.rank] + tail.rank);
              slot = (int)(epoch & 1u);
            }
            double* const* blocks = tail.peer_block[slot];
            unsigned* const* flags = tail.peer_flag[slot];
            __syncthreads();
            double* mine = blocks[tail.rank];
            for (int e = threadIdx.x; e < NN; e += kThreads) {
              const int i = e / N, j = e - i * N;
              double v = 0.;
              if (i < j) {
                const int a = map.to_unique[i], b = map.to_unique[j];
                v = local[min(a, b) * n + max(a, b)];
              }
              mine[e] = v;
            }
            map.u = N;                          // the summed table below is N x N already
            __threadfence_system();
            __syncthreads();
            // flag, bounded wait (peers.cuh): a peer that never shows up sets the status word
            if ((int)threadIdx.x < tail.nranks &&
                peer_signal_wait(flags[threadIdx.x] + tail.rank, flags[tail.rank] + threadIdx.x, epoch))
              peer_timeout = 1;
            __syncthreads();
            asm volatile("" ::: "memory");      // the block loads below stay below the flag wait
            for (int e = threadIdx.x; e < NN; e += kThreads) {
              double part[BZ_MAX_PEERS];
#pragma unroll
              for (int r = 0; r < BZ_MAX_PEERS; ++r) part[r] = (r < tail.nranks) ? ld_relaxed_sys_f64(blocks[r] + e) : 0.;
              double v = part[0];
#pragma unroll
              for (int r = 1; r < BZ_MAX_PEERS; ++r) v += part[r];      // rank order; + 0.0 past nranks is exact
              table[e] = v;
            }
            __syncthreads();
          } else
          for (int e = threadIdx.x; e < len; e += kThreads) {
            const int i = e / n, j = e - i * n;
            double v = 0.;
            if (i <= j) {
              const int oi = tail.old_index[i], oj = tail.old_index[j];
              if (i < j && tail.cache_in != nullptr && oi >= 0 && oj >= 0) {
                v = __ldcg(tail.cache_in + (size_t)min(oi, oj) * tail.u_old + max(oi, oj));
              } else {
                for (int g = 0; g < ngroups; ++g) v += __ldcg(gblocks + (size_t)g * len + e);
              }
            }
            table[e] = v;
            if (tail.cache_out != nullptr) tail.cache_out[e] = v;
          }
          __syncthreads();
          if (tail.kind == 3) brute_from_table(map, N, tail.f, tail.total, tail.order, tail.status, sm);
          else                score_from_table(map, N, tail.count, tail.order, tail.kind == 2 ? tail.status : nullptr,
                                               tail.f, tail.m, tail.kind == 2 ? 1 : 0, sm);
          __syncthreads();
          if (threadIdx.x == 0 && peer_timeout && tail.status != nullptr) *tail.status = BZ_STATUS_PEER_TIMEOUT;
        }
        if (threadIdx.x <= ngroups) tail.ticket[threadIdx.x] = 0u;
      }
    }
  }
  if (CLUSTER) cluster_sync_all();   // no CTA leaves while a peer may still arrive on its barriers
}

// ---- host side -------------------------------------------------------------------------------

// The launch shapes: warps per CTA, tile width, ring depth, and whether C > 1 CTAs of a cluster share
// each tile (multicast).
struct RingShape { int W, T, stages; bool cluster; };
enum { kShapeSmall, kShapeOne, kShapeCluster, kShapeWide };
constexpr RingShape kShapes[] = {
    {kRWarpsSmall, 512, 3, false},   // n <= 15 (all tasks fit 6 warps): two CTAs per SM
    {kRWarps, 512, 4, false},        // n <= 25: one CTA per tile
    {kRWarps, 512, 3, true},         // n <= 35: clusters of 12-warp CTAs
    {kRWarpsWide, 256, 3, true},     // n >  35: clusters of 16-warp CTAs (512-column tiles with 2 stages
                                     // measured 20 % slower at n = 40...51)
};

// The shape for n rows and its cluster size C (1 when all tasks fit one CTA).  Returns false when
// the kernel does not support n.
static bool ring_shape(int n, int& shape, int& C) {
  const int ng = (n + kG - 1) / kG, tasks = ring_ntasks(ng);
  if (tasks <= kRWarpsSmall && n <= 3 * kRWarpsSmall) shape = kShapeSmall;
  else if (ng * kG > 35)                              shape = kShapeWide;
  else                                                shape = tasks <= kRWarps ? kShapeOne : kShapeCluster;
  const int W = kShapes[shape].W;
  C = (tasks + W - 1) / W;
  return C <= kRMaxCluster;
}

// Whether the scoring step's tables fit the ring's stage area, where it works once the ring is drained
// (the barriers behind the stages stay untouched).  Kind 4 keeps only the u x u table there, which the
// stages of u rows always hold (u * u * 8 bytes <= 3 stages of u rows of 256 floats).
static bool tail_fits(const SelectTail& sel, size_t stage_area) {
  if (sel.kind == 4) return true;
  const size_t nn = (size_t)sel.n * sel.n * sizeof(double);
  const size_t need = sel.kind == 3 ? nn + (size_t)(sel.n + 1) * (sel.n + 1) * sizeof(unsigned long long) + 64 * sizeof(double)
                                    : 2 * nn + (size_t)sel.n * sizeof(double);
  return stage_area >= need;
}

template <int S, bool SELF>
static int launch_ring_cfg(const RowTable& rows, const SelfList& self, const RingTail& tail, const StarList& star, int n, int C,
                           int64_t d, double* parts, cudaStream_t st) {
  constexpr int T = kShapes[S].T, STAGES = kShapes[S].stages, W = kShapes[S].W;
  constexpr bool CLUSTER = kShapes[S].cluster;
  const int ng = (n + kG - 1) / kG;
  const size_t smem = (size_t)STAGES * ng * kG * T * sizeof(float) + 2 * STAGES * sizeof(unsigned long long);
  auto kernel = k2_ring<T, STAGES, SELF, CLUSTER, W>;
  static unsigned long long opted = 0;
  static int max_clusters[64][kRMaxCluster + 1] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = 1ull << (dev & 63);
  if (!(opted & bit)) {
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRSmemBudget);
    opted |= bit;
  }
  const int64_t nfull = d / T, ntiles = (d + T - 1) / T;
  cudaLaunchConfig_t cfg = {};
  cfg.blockDim = dim3(W * 32);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  int nclusters = sm_count() * (W == kRWarpsSmall ? 2 : 1) / C;
  if (CLUSTER) {
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)C;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int& cached = max_clusters[dev & 63][C];
    if (cached == 0) {
      cfg.gridDim = dim3((unsigned)(nclusters * C));
      int active = 0;
      if (cudaOccupancyMaxActiveClusters(&active, kernel, &cfg) != cudaSuccess || active < 1) { cudaGetLastError(); active = -1; }
      cached = active;
    }
    if (cached < 1) return -1;                 // this cluster size cannot be scheduled here
    if (nclusters > cached) nclusters = cached;  // persistent kernel: only co-resident clusters
  }
  if (nclusters > kMaxParts - kTailTickets) nclusters = kMaxParts - kTailTickets;   // room for the group blocks behind
  if ((int64_t)nclusters > ntiles) nclusters = (int)(ntiles > 0 ? ntiles : 1);
  if (nclusters < 1) nclusters = 1;
  cfg.gridDim = dim3((unsigned)(nclusters * C));
  if (tail.kind != 0) cudaMemsetAsync(tail.ticket, 0, kTailTickets * sizeof(unsigned), st);
  if (cudaLaunchKernelEx(&cfg, kernel, rows, self, tail, star, n, C, d, nfull, parts) != cudaSuccess) return -1;
  return nclusters;
}

template <bool SELF>
static int launch_ring(int shape, const RowTable& rows, const SelfList& self, const RingTail& tail, const StarList& star, int n, int C,
                       int64_t d, double* parts, cudaStream_t st) {
  switch (shape) {
    case kShapeSmall:   return launch_ring_cfg<kShapeSmall, SELF>(rows, self, tail, star, n, C, d, parts, st);
    case kShapeOne:     return launch_ring_cfg<kShapeOne, SELF>(rows, self, tail, star, n, C, d, parts, st);
    case kShapeCluster: return launch_ring_cfg<kShapeCluster, SELF>(rows, self, tail, star, n, C, d, parts, st);
    default:            return launch_ring_cfg<kShapeWide, SELF>(rows, self, tail, star, n, C, d, parts, st);
  }
}

// Returns the number of partial blocks written, or -1 when the rows are not 16-byte aligned or the
// launch fails (the caller falls back to k2_pairdist).  `self_rows`: unique rows whose self distance K5 reads.
int launch_pairdist_ring(const RowTable& rows, int n, int64_t d, double* parts, cudaStream_t st,
                         const unsigned char* self_rows, int nself, SelectTail* select, int star_row) {
  int shape, C;
  if (!ring_shape(n, shape, C)) return -1;
  const int W = kShapes[shape].W;
  if (nself > W * C * kSelfPerWarp) return -1;
  for (int r = 0; r < n && d > 0; ++r)           // an empty shard reads nothing: any address will do
    if ((((uintptr_t)rows.p[r]) & 15) != 0) return -1;
  SelfList self;
  self.count = nself;
  for (int q = 0; q < nself; ++q) self.row[q] = self_rows[q];
  const int ng = (n + kG - 1) / kG;
  const size_t stage_area = (size_t)kShapes[shape].stages * ng * kG * kShapes[shape].T * sizeof(float);
  RingTail tail = {};
  StarList star = {};
  for (int k = 0; k < kMaxN; ++k) tail.old_index[k] = -1;
  // The scoring step is fused only when it fits; otherwise the caller launches K5, and no star pass is
  // prepared, so that a reuse call runs exactly the pass of the plain call.
  if (select != nullptr && select->kind != 0 && tail_fits(*select, stage_area)) {
    tail.kind = select->kind; tail.n = select->n; tail.f = select->f; tail.m = select->m; tail.count = select->count;
    tail.total = select->total; tail.order = select->order; tail.status = select->status; tail.ticket = select->ticket;
    tail.map = make_map(select->to_unique, select->n, n);
    tail.cache_out = select->cache_out;
    tail.u_old = select->u_old;
    select->reused = 0;
    if (select->nranks > 0) {
      tail.nranks = select->nranks; tail.rank = select->rank; tail.epoch = select->epoch; tail.next = select->next;
      for (int s = 0; s < (select->next ? 2 : 1); ++s)
        for (int r = 0; r < BZ_MAX_PEERS; ++r) {
          tail.peer_block[s][r] = select->peer_blocks[s * select->nranks + (r < select->nranks ? r : 0)];
          tail.peer_flag[s][r] = select->peer_flags[s * select->nranks + (r < select->nranks ? r : 0)];
        }
    }
    // Distance reuse: unique row k was row old_index[k] of the table in `cache_in`.  A star pass is
    // taken when 1..kStarMax unique rows are new, every other one is in the table, and that table
    // came out of the same launch shape and cluster size (functions of the row count) — then every
    // pair has the bits the full pass would give it.
    if (select->cache_in != nullptr && select->old_index != nullptr && select->u_old >= 1) {
      int fresh[kMaxN], nfresh = 0;
      bool ok = true;
      for (int k = 0; k < n; ++k) {
        int oi = -1;
        for (int i = 0; i < select->n; ++i)
          if ((select->to_unique ? select->to_unique[i] : i) == k) { oi = select->old_index[i]; break; }
        if (oi >= select->u_old) ok = false;
        tail.old_index[k] = (signed char)oi;
        if (oi < 0) fresh[nfresh++] = k;
      }
      // 3 rows per star task when the cluster has the warps for it, else 25
      int slots = 3;
      if (nfresh * ((n + slots - 1) / slots) > W * C) slots = kRSlots;
      const int chunks = (n + slots - 1) / slots;
      int old_shape = 0, old_C = 0;
      ok = ok && nfresh >= 1 && nfresh <= kStarMax && nfresh * chunks <= W * C && nfresh < n
              && ring_shape(select->u_old, old_shape, old_C) && old_shape == shape && old_C == C;
      if (ok) {
        star.count = nfresh;
        star.slots = slots;
        for (int q = 0; q < nfresh; ++q) star.row[q] = (unsigned char)fresh[q];
        tail.cache_in = select->cache_in;
        select->reused = 1;
      } else {
        for (int k = 0; k < kMaxN; ++k) tail.old_index[k] = -1;
      }
    }
  }
  if (star_row >= 0) {
    // the star pass of bz_distance_line_search: one fresh row, its slots picked as above
    const int slots = (n + 2) / 3 > W * C ? kRSlots : 3;
    if (select != nullptr || star_row >= n || n < 2 || (n + slots - 1) / slots > W * C) return -1;
    star.count = 1;
    star.slots = slots;
    star.row[0] = (unsigned char)star_row;
  }
  const int nparts = nself > 0 ? launch_ring<true>(shape, rows, self, tail, star, n, C, d, parts, st)
                               : launch_ring<false>(shape, rows, self, tail, star, n, C, d, parts, st);
  if (select != nullptr) {
    select->fused = (nparts > 0 && tail.kind != 0) ? 1 : 0;
    if (!select->fused) select->reused = 0;
  }
  return nparts;
}

}  // namespace bz
