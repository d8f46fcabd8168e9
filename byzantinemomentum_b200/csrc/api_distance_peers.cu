// api_distance_peers.cu — the C ABI of libbyzagg_peers.so (include/byzagg_distance_peers.h): phase B of the d-sharded
// Multi-Krum, Bulyan, Aksel and CGE above 64 rows with the exchange over peer memory (k5_select_peers.cu).  Its
// argument checks are libbyzagg's (api_shared.cuh); its error string is its own.  Nothing here links against
// libbyzagg.so: a caller composes the two libraries through their C ABIs.
#include <cstdarg>
#include <cstdio>

#include "dist.cuh"
#include "api_shared.cuh"
#include "../../include/byzagg_distance_peers.h"

namespace bz {

static thread_local char g_error[512] = "";

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
  return code;
}

int check_launch(const char* what) {
  const cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return fail(BZ_ECUDA, "%s: %s", what, cudaGetErrorString(err));
  return BZ_OK;
}

// bz_distance_select_peers (next == 0, `epoch` by value) and bz_distance_select_peers_next: every check, then one
// launch.
static int distance_select_peers(int rule, const double* part, int n, int f, int m, int mode, int32_t* order,
                                 int32_t* status, int rank, int nranks, double* const* blocks, unsigned* const* flags,
                                 unsigned epoch, int next, void* stream, const char* who) {
  if (int rc = check_distance_rule(rule, n, who)) return rc;
  if (n <= kMaxN)
    return fail(BZ_EUNSUPPORTED, "%s: n = %d: up to BZ_MAX_N = %d rows the exchange runs inside the distance pass "
                "(bz_krum_peers, bz_bulyan_peers, bz_rowdist_peers)", who, n, kMaxN);
  if (part == nullptr || order == nullptr) return fail(BZ_EINVAL, "%s: part / order is NULL", who);
  if (((uintptr_t)part % 8) != 0) return fail(BZ_EINVAL, "%s: part is not 8-byte aligned", who);
  const bool pair = rule == BZ_RULE_KRUM || rule == BZ_RULE_BULYAN;
  SelectTail sel = {};
  if (rule == BZ_RULE_AKSEL) {
    int c;
    if (int rc = aksel_count(n, f, mode, c, who)) return rc;
  } else if (pair) {
    if (int rc = rule_tail(rule - BZ_RULE_KRUM + 1, n, f, m, who, sel)) return rc;
  }
  if (int rc = next ? check_peers_next(rank, nranks, blocks, flags, status, who) : check_peers(rank, nranks, blocks, flags, status, who))
    return rc;
  const PeerTail peers = make_peer_tail(rank, nranks, epoch, next, status, blocks, flags);
  cudaStream_t st = (cudaStream_t)stream;
  if (pair) {
    launch_blocks_select_peers(part, n, sel.count, order, f, m, rule == BZ_RULE_BULYAN ? 1 : 0, peers, st);
    return check_launch("k5_blocks_select_peers");
  }
  launch_rowkeys_select_peers(part, n, rule == BZ_RULE_CGE ? 1 : 0, order, peers, st);
  return check_launch("k5_rowkeys_select_peers");
}

}  // namespace bz

extern "C" {

const char* bz_distance_peers_last_error(void) { return bz::g_error; }

int bz_distance_select_peers(int rule, const double* part, int n, int f, int m, int mode, int32_t* order, int32_t* status,
                             int rank, int nranks, double* const* peer_blocks, unsigned* const* peer_flags, unsigned epoch,
                             void* stream) {
  return bz::distance_select_peers(rule, part, n, f, m, mode, order, status, rank, nranks, peer_blocks, peer_flags, epoch, 0,
                                   stream, "bz_distance_select_peers");
}

int bz_distance_select_peers_next(int rule, const double* part, int n, int f, int m, int mode, int32_t* order,
                                  int32_t* status, int rank, int nranks, double* const* peer_blocks,
                                  unsigned* const* peer_flags, void* stream) {
  return bz::distance_select_peers(rule, part, n, f, m, mode, order, status, rank, nranks, peer_blocks, peer_flags, 0u, 1,
                                   stream, "bz_distance_select_peers_next");
}

}  // extern "C"
