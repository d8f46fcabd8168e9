// api_shared.cuh — host code of the C ABI that libbyzagg.so (api.cu) and libbyzagg_peers.so (api_distance_peers.cu)
// both run: the rule and count checks of the distance-based rules, the checks of the exchange tables over peer
// memory, and the PeerTail a kernel of that exchange takes.  Each library defines its own `fail`.
#pragma once

#include <cstdio>

#include "dist.cuh"

namespace bz {

// The rule and the row count, the first checks of bz_distance and of the phases of byzagg_distance_shards.h.
static int check_distance_rule(int rule, int n, const char* who) {
  if (rule < BZ_RULE_KRUM || rule > BZ_RULE_CGE) return fail(BZ_EINVAL, "%s: unknown rule %d", who, rule);
  if (n < 1) return fail(BZ_EINVAL, "%s: n = %d, expected n >= 1", who, n);
  if (n > kMaxNDistance) return fail(BZ_EUNSUPPORTED, "%s: n = %d exceeds BZ_MAX_N_DISTANCE = %d", who, n, kMaxNDistance);
  if (rule == BZ_RULE_BRUTE && n > kMaxN)
    return fail(BZ_EUNSUPPORTED, "%s: brute takes n <= BZ_MAX_N = %d rows, got %d", who, kMaxN, n);
  return BZ_OK;
}

// The reduce step of Multi-Krum and brute: the average of `count` selected rows, divided by `count`;
// brute's skips the rows when the status word says so.  Bulyan has its own (run_bulyan_reduce).
struct AverageStep {
  int count;
  bool status;
};

// Checks Multi-Krum (kind 1), Bulyan (2) or brute (3) at (n, f, m) and fills the fields of `sel` its
// scoring step reads: Multi-Krum scores each row over its n - f - 1 nearest (and passes m = 0),
// Bulyan selects m rows, brute searches the C(n, n - f) subsets.  `avg`, if given, gets the reduce step.
static int rule_tail(int kind, int n, int f, int m, const char* who, SelectTail& sel, AverageStep* avg = nullptr) {
  sel.kind = kind; sel.n = n; sel.f = f; sel.m = 0; sel.count = 0; sel.total = 0;
  if (kind == 1) {
    if (f < 0 || n - f - 1 < 1) return fail(BZ_EINVAL, "%s: f = %d not executable with n = %d (need n - f - 1 >= 1)", who, f, n);
    if (m < 1 || m > n) return fail(BZ_EINVAL, "%s: m = %d, expected 1..%d", who, m, n);
    sel.count = n - f - 1;
    if (avg != nullptr) *avg = {m, false};
  } else if (kind == 2) {
    const int theta = n - 2 * f - 2, beta = theta - 2 * f, m_max = n - f - 2;
    if (f < 0 || theta < 1 || beta < 1) return fail(BZ_EINVAL, "%s: f = %d not executable with n = %d (need n >= 4f + 3)", who, f, n);
    if (m < 1 || m > m_max) return fail(BZ_EINVAL, "%s: m = %d, expected 1..%d", who, m, m_max);
    sel.m = m; sel.count = m;
  } else {
    if (f < 0 || n - f < 1) return fail(BZ_EINVAL, "%s: f = %d not executable with n = %d", who, f, n);
    sel.total = brute_total(n, f);
    if (avg != nullptr) *avg = {n - f, true};
  }
  return BZ_OK;
}

// The rows Aksel averages (aksel.py:43-48), after checking mode and f.
static int aksel_count(int n, int f, int mode, int& c, const char* who) {
  if (mode != BZ_AKSEL_MID && mode != BZ_AKSEL_NF) return fail(BZ_EINVAL, "%s: mode = %d", who, mode);
  c = (mode == BZ_AKSEL_MID) ? (n + 1) / 2 : n - f;
  if (c < 1 || c > n) return fail(BZ_EINVAL, "%s: f = %d not executable with n = %d", who, f, n);
  return BZ_OK;
}

// The exchange arguments of the calls over peer memory; the status word is required: a peer timeout is
// reported there.  `who` + `suffix` names the call.
static int check_peers(int rank, int nranks, double* const* blocks, unsigned* const* flags, const int32_t* status,
                       const char* who, const char* suffix = "") {
  if (nranks < 1 || nranks > BZ_MAX_PEERS || rank < 0 || rank >= nranks) return fail(BZ_EINVAL, "%s%s: rank %d of %d", who, suffix, rank, nranks);
  if (blocks == nullptr || flags == nullptr || status == nullptr) return fail(BZ_EINVAL, "%s%s: NULL peer table or status", who, suffix);
  for (int r = 0; r < nranks; ++r)
    if (blocks[r] == nullptr || flags[r] == nullptr || ((uintptr_t)blocks[r] % 8) != 0 || ((uintptr_t)flags[r] % 4) != 0)
      return fail(BZ_EINVAL, "%s%s: peer %d: NULL or misaligned block / flag pointer", who, suffix, r);
  return BZ_OK;
}

// The same for the bz_*_peers_next calls: the tables of both slots, 2 * nranks pointers each (slot 0's, then
// slot 1's).
static int check_peers_next(int rank, int nranks, double* const* blocks, unsigned* const* flags, const int32_t* status,
                            const char* who, const char* suffix = "") {
  if (int rc = check_peers(rank, nranks, blocks, flags, status, who, suffix)) return rc;
  char slot1[64];
  snprintf(slot1, sizeof(slot1), "%s (slot 1)", suffix);
  return check_peers(rank, nranks, blocks + nranks, flags + nranks, status, who, slot1);
}

static PeerTail make_peer_tail(int rank, int nranks, unsigned epoch, int next, int32_t* status, double* const* blocks,
                               unsigned* const* flags) {
  PeerTail p = {};
  p.nranks = nranks; p.rank = rank; p.epoch = epoch; p.next = next; p.status = status;
  for (int s = 0; s < (next ? 2 : 1); ++s)
    for (int r = 0; r < BZ_MAX_PEERS; ++r) {
      p.block[s][r] = blocks[s * nranks + (r < nranks ? r : 0)];
      p.flag[s][r] = flags[s * nranks + (r < nranks ? r : 0)];
    }
  return p;
}

}  // namespace bz
