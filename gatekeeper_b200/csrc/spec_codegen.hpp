// The constraint netlist as generated CUDA C++ (the "specialised" evaluation kernel).
//
// gk_eval_kernel (tile_kernel.cuh) INTERPRETS the netlist: every node is a bit column of a 512-object tile in shared memory, every
// op a work item some warp decodes, ~400 warp-instructions per object at the benchmark's 50 constraints.  The netlist is known when
// the constraint set is compiled, so the engine also writes it out as straight-line code, constants as immediates, in two phases per
// tile.  Phase 1, one thread per ROW: the row's atoms and every gate that reads that row alone, of which only the bits something
// else reads (exports) are stored, as bit planes of 32-row blocks.  Phase 2, one thread per OBJECT: every remaining node a 32-bit mask
// register (bit j = row j of THIS object in the node's scope), an export one 32-bit window of its plane from the object's first row,
// EXISTS a `!= 0`, the object-major bitmap words assembled in registers without a transpose.  NVRTC compiles that text for
// sm_90a when the first large batch is evaluated (kernels.cu).  Objects with more than 32 rows in some scope do not fit the mask registers: they are
// handed to the interpreter one by one, or with their whole tile when a tile holds more than GK_HANDOVER_MAX (GkKParams::units):
// gk_spec_plan_kernel lists them from the CSR offsets before the rows are evaluated, and the interpreter runs beside the two kernels.
#pragma once
#include <string>
#include <vector>

#include "engine.hpp"
#include "eval_layout.h"

namespace gk {

struct SpecSource {
  std::string src;        // one self-contained translation unit: program.h + vm_core.h + gk_spec_row_<g>() + gk_spec_rows_kernel + gk_spec_stage()
                          // + gk_spec_wide() + gk_spec_object() + gk_spec_kernel + gk_spec_plan_kernel
  uint32_t words = 1;     // bitmap words per object
  size_t smem = 0;        // fixed dynamic shared memory of a launch (column / scope tables, enforcement-point mask, totals)
  size_t n_fast = 0, n_generic = 0;   // atoms emitted as immediates / as calls of the generic gk_atom()
  // the per-tile staging area behind the fixed part: `hdr` words, then one region per entry of `stage` (the first `ngroups` are the
  // row loops' export planes, in row-loop order; the rest the nested scopes' offsets)
  struct StageRegion {
    // a row loop: `planes` export planes (its exports rounded up to 4), one word per plane per block of 32 rows of `scope`; a
    // nested scope's offsets: one 16-bit value per row of `scope` (its parent) + 1 (planes = 0)
    uint32_t scope, planes;
  };
  std::vector<StageRegion> stage;
  uint32_t stage_hdr = 0;
  uint32_t ngroups = 0;
  std::vector<uint32_t> nested;   // the used nested scopes, whose offsets are staged: stage[ngroups + j] is nested[j]'s
  // The offset image (gk_spec_plan_kernel writes it once per batch and text, gk_spec_stage copies a tile's run verbatim): per tile,
  // the offsets regions of the staging area back to back, every nested scope's tile-relative CSR offsets as 16-bit values, the run
  // padded to 16 bytes; tile t's run at t * image_stride(cap) values.  The stride bounds every tile's run from the largest tile's
  // rows per scope (cap), as stage_bytes() bounds the staging area.
  uint32_t image_stride(const std::vector<uint32_t>& cap) const {
    uint64_t v = 0;
    for (size_t i = ngroups; i < stage.size(); ++i) v += (uint64_t)(stage[i].scope < cap.size() ? cap[stage[i].scope] : 0u) + 1u;
    return (uint32_t)((v + 7) / 8 * 8);
  }
  // A tile-relative offset of scope s is at most the tile's rows of s: the image holds them when no tile has more than 65535 rows
  // in a nested scope.  A batch with such a tile (only objects far too wide for the mask registers make one) is interpreted.
  bool image_fits(const std::vector<uint32_t>& cap) const {
    for (uint32_t s : nested)
      if (s < cap.size() && cap[s] > 0xffffu) return false;
    return true;
  }
  // per scope with atoms: what a row evaluates (atoms, row-local gates) and what it exports (by read form; on scope 0 the mask-form
  // exports include the match and error bits of the spec.match blocks), in `words` words per row
  struct Fold {
    uint32_t scope, atoms, gates, any, mask, words;
  };
  std::vector<Fold> fold;
  // the type words the rows read (gk_tw_layout of the constraint set's columns): a batch evaluated with this text must have them
  // laid out alike
  GkTwLayout tw;
  // "folded: scope S: A atoms + G gates -> X any + Y mask in W words; ..." (the first line of `src`, and the backend's trace)
  std::string fold_text() const {
    std::string t = "folded:";
    for (size_t i = 0; i < fold.size(); ++i) {
      const Fold& f = fold[i];
      t += std::string(i ? ";" : "") + " scope " + std::to_string(f.scope) + ": " + std::to_string(f.atoms) + " atoms + " + std::to_string(f.gates) + " gates -> " +
           std::to_string(f.any) + " any + " + std::to_string(f.mask) + " mask in " + std::to_string(f.words) + " words";
    }
    return t;
  }
  // bytes of the staging area for a batch whose largest tile has cap[s] rows in scope s: a tile's rows of a scope start anywhere in
  // a block of 32, so they span at most ceil(cap / 32) + 1 blocks, and the region holds one more (gk_spec_stage); then one run of
  // the offset image.  (Every region is a multiple of 16 bytes, so the offsets start 16-byte aligned.)
  size_t stage_bytes(const std::vector<uint32_t>& cap) const {
    size_t w = stage_hdr;
    for (size_t i = 0; i < ngroups; ++i) w += (((size_t)(stage[i].scope < cap.size() ? cap[stage[i].scope] : 0u) + 31) / 32 + 2) * stage[i].planes;
    return w * 4 + (size_t)image_stride(cap) * 2;
  }
  // bytes of the export planes (gk_spec_rows_kernel -> gk_spec_kernel) of a batch with rows[s] rows in scope s (rows[0] = objects):
  // per row loop, `planes` words per block of 32 rows and one guard block (a window's high word past the last block)
  size_t export_bytes(const std::vector<uint32_t>& rows) const {
    size_t w = 0;
    for (uint32_t g = 0; g < ngroups; ++g) w += (((stage[g].scope < rows.size() ? rows[stage[g].scope] : 0u) + (size_t)31) / 32 + 1) * stage[g].planes;
    return w * 4;
  }
  // blocks of gk_spec_rows_kernel over such a batch at `threads` per block
  uint32_t rows_blocks(const std::vector<uint32_t>& rows, uint32_t threads) const {
    uint64_t b = 0;
    for (uint32_t g = 0; g < ngroups; ++g) b += ((stage[g].scope < rows.size() ? rows[stage[g].scope] : 0u) + (uint64_t)threads - 1) / threads;
    return (uint32_t)b;
  }
};

SpecSource spec_codegen(const Compiled& c);

}  // namespace gk
