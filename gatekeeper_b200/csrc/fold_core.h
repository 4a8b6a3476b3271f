// The fold of an expanded batch (GK_F_EXPAND): each resultant's violation and error rows ORed into its parent's rows.  One parent per
// call, so that no two callers write one row: the CUDA backend runs it one thread per parent (kernels.cu gk_fold_kernel), the host
// emulation in a loop.
#pragma once
#include <stdint.h>

#include "program.h"

namespace gk {

typedef struct {
  const uint32_t* par;           // [m] the parents that have resultants, ascending
  const uint32_t* off;           // [m + 1] parent j's resultants are rows off[j] .. off[j + 1] - 1 of the resultant planes
  uint32_t m, words, nconstraints;
  const uint32_t* cviol;         // the resultants' planes [resultants * words]
  const uint32_t* cerr;
  const uint32_t* sviol;         // the parents' unfolded planes [parents * words]
  const uint32_t* serr;
  uint32_t* dviol;               // where the folded rows go (may be null: the peers only) -- may equal sviol / serr
  uint32_t* derr;
  uint32_t* peer_viol[GK_MAX_PEERS];   // the fused exchange: this rank's shard in every peer's receive buffer
  unsigned long long* peer_tot[GK_MAX_PEERS];
  uint32_t npeers, tot_stride;
  unsigned long long* totals;    // [nconstraints] the newly set bits are added here
  unsigned long long* err_totals;
} GkFoldArgs;

GK_HD uint32_t gk_ctz32(uint32_t b) {
#ifdef __CUDA_ARCH__
  return (uint32_t)__ffs((int)b) - 1u;
#else
  return (uint32_t)__builtin_ctz(b);
#endif
}

// parent j: its folded rows stored to every destination; count(c, plane) for every bit the fold set (plane 0: violations, 1: errors)
template <class Count>
GK_HD void gk_fold_parent(const GkFoldArgs& a, uint32_t j, Count&& count) {
  const uint32_t p = a.par[j], lo = a.off[j], hi = a.off[j + 1], W = a.words;
  for (uint32_t w = 0; w < W; ++w) {
    const size_t at = (size_t)p * W + w;
    const uint32_t v0 = a.sviol[at], e0 = a.serr[at];
    uint32_t v = v0, e = e0;
    for (uint32_t k = lo; k < hi; ++k) {
      v |= a.cviol[(size_t)k * W + w];
      e |= a.cerr[(size_t)k * W + w];
    }
    for (uint32_t b = v & ~v0; b; b &= b - 1) count(w * 32u + gk_ctz32(b), 0u);
    for (uint32_t b = e & ~e0; b; b &= b - 1) count(w * 32u + gk_ctz32(b), 1u);
    if (a.dviol) a.dviol[at] = v;
    for (uint32_t q = 0; q < a.npeers; ++q) a.peer_viol[q][at] = v;
    a.derr[at] = e;
  }
}

// The audit of an expanded batch (gk_audit_add_batch(_ordered)): the resultants' flagged pairs sorted into those the run counts and
// those the host renders.  The CUDA backend runs it one thread per resultant (kernels.cu gk_res_classify_kernel), the host in loops.
typedef struct {
  const uint32_t* viol;          // the resultants' planes [resultants * words]
  const uint32_t* err;
  const uint32_t* amb;           // the resultants' ambiguity plane (bit clear: at most one result for the pair), or null: none
  const uint8_t* single;         // [nconstraints] 1: one result for every pair of the constraint
  uint32_t words, nconstraints;
} GkResClassArgs;

// resultant r, whose parent passes cand(c) when it can still enter constraint c's list: a matcher-error pair is emitted (emit(c, 1)); a
// violation pair is emitted (emit(c, 0)) when its parent is a candidate or it may have several results, and counted (count(c)) otherwise
template <class Cand, class Count, class Emit>
GK_HD void gk_classify_resultant(const GkResClassArgs& a, uint32_t r, Cand&& cand, Count&& count, Emit&& emit) {
  const uint32_t W = a.words;
  for (uint32_t w = 0; w < W; ++w) {
    const size_t at = (size_t)r * W + w;
    const uint32_t v = a.viol[at], e = a.err[at], am = a.amb ? a.amb[at] : ~0u;
    for (uint32_t b = v | e; b; b &= b - 1) {
      const uint32_t k = gk_ctz32(b), c = w * 32u + k;
      if (c >= a.nconstraints) continue;
      if (e >> k & 1u) emit(c, 1u);
      else if (cand(c) || !(a.single[c] || !(am >> k & 1u))) emit(c, 0u);
      else count(c);
    }
  }
}

}  // namespace gk
