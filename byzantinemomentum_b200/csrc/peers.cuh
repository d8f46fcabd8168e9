// peers.cuh — the flag protocol of the exchanges that run inside a kernel over peer memory (one process
// per GPU, buffers mapped on every GPU over NVLink / NVSwitch): the tail of the distance pass
// (k2_ring.cu, bz_*_peers) and the last CTA of K2' (k2_rowdist.cu, bz_rowdist_peers / bz_search_score_peers).
// A rank writes its block into its slot, raises its flag for `epoch` in every rank's flag array, waits for
// every rank's flag in its own array, then reads the R slots in place.
#pragma once

#include "common.cuh"

namespace bz {

__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// Coherent at system scope, never from a stale L1 line (the slot is rewritten every other step); NOT
// `volatile` asm, so that the R loads of a table entry are issued together (a volatile load per rank made
// the entry cost R NVLink round trips).
__device__ __forceinline__ double ld_relaxed_sys_f64(const double* p) {
  double v;
  asm("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}

// The epoch of an exchange that takes it from the buffer (bz_*_peers_next): one past the last epoch this rank
// raised, i.e. the later, compared wrap-aware as below, of its own entries in its own flag arrays of the two
// slots (`own0`, `own1`: flag[s][rank] + rank).  A zeroed buffer gives 1; the slot is the epoch modulo 2.
// Only this rank writes those entries, and only in the signal below: read them before the barrier that
// precedes it, once every earlier exchanging kernel has completed (stream order, or pdl_wait).
__device__ __forceinline__ unsigned next_epoch(const unsigned* own0, const unsigned* own1) {
  const unsigned e0 = ld_acquire_sys(own0), e1 = ld_acquire_sys(own1);
  return ((int)(e1 - e0) > 0 ? e1 : e0) + 1u;
}

// One thread per rank t of the exchange: raise this rank's flag for `epoch` in rank t's flag array
// (`signal`) and wait for rank t's flag in this rank's array (`wait_on`).  The caller has made its block
// visible (__threadfence_system + __syncthreads) before, and synchronises the block after.  The wait is
// bounded (~2 s): a peer that never shows up must not hang the GPU.  Returns true when it did not show up.
__device__ __forceinline__ bool peer_signal_wait(unsigned* signal, const unsigned* wait_on, unsigned epoch) {
  st_release_sys(signal, epoch);                          // "this rank's block of step `epoch` is there"
  unsigned spins = 0;
  while ((int)(ld_acquire_sys(wait_on) - epoch) < 0) {
    __nanosleep(100);
    if (++spins > (1u << 24)) return true;
  }
  return false;
}

}  // namespace bz
