// Shared-memory sizing of the netlist interpreter (gk_eval_kernel, tile_kernel.cuh): the layout of its dynamic shared memory,
// the slot area of a tile, and the tile size of a batch.  The kernel carves its shared memory with gk_eval_layout and the
// CUDA backend sizes every launch and every tile with the same functions, so the two cannot disagree.
#pragma once
#include <algorithm>
#include <vector>

#include "program.h"

// Byte offset of every region of gk_eval_kernel's dynamic shared memory, in the kernel's order; each region is padded to 16
// bytes (the tables are staged with 16-byte copies), so a region ends where the next one starts and the last one at `end`.
struct GkEvalLayout {
  size_t s_tot, s_err, s_act, s_lo, s_cnt, s_poff, slots, outs, ops, items, match, cols, scopes, pool, cbytes, end;
  size_t total;   // bytes a launch needs: `end` plus 64 bytes of tail (resident CTAs per SM are computed from this total)
};

// C constraints, NS scopes, NP dependency phases, a slot area of slot_words words; the rest are the lengths of the program and
// schema tables staged in shared memory (ops, work items, match blocks, columns, scopes, pool words, constant bytes).
GK_HD GkEvalLayout gk_eval_layout(uint32_t C, uint32_t NS, uint32_t NP, uint32_t slot_words, uint32_t nops, uint32_t nitems, uint32_t nmatch,
                                  uint32_t ncols, uint32_t npool, uint32_t ncbytes) {
  GkEvalLayout L;
  size_t off = 0;
  auto take = [&off](size_t bytes) {
    const size_t o = off;
    off += (bytes + 15) / 16 * 16;
    return o;
  };
  L.s_tot = take((size_t)C * 4);
  L.s_err = take((size_t)C * 4);
  L.s_act = take((size_t)C * 4);
  L.s_lo = take((size_t)NS * 4);
  L.s_cnt = take((size_t)NS * 4);
  L.s_poff = take((size_t)(NP + 1) * 4);
  L.slots = take((size_t)slot_words * 4);
  L.outs = take((size_t)C * sizeof(GkOutEnt));
  L.ops = take((size_t)nops * sizeof(GkOp));
  L.items = take((size_t)nitems * 4);
  L.match = take((size_t)nmatch * sizeof(GkMatch));
  L.cols = take((size_t)ncols * sizeof(GkColumn));
  L.scopes = take((size_t)NS * sizeof(GkScope));
  L.pool = take((size_t)npool * 4);
  L.cbytes = take((size_t)ncbytes);
  L.end = off;
  L.total = off + 64;
  return L;
}

// Slot area of a tile: slot i holds one bit per row of its scope (cap[slot_level[i]] rows; cap[0] is the tile) plus one word,
// rounded up to 4 words -- 16-byte aligned, padded: atoms store 4 words at a time.  Fills `off` (if not null) with the word offset
// of every slot and returns the total words.
inline uint64_t gk_slot_layout(const std::vector<uint8_t>& slot_level, const std::vector<uint32_t>& cap, std::vector<uint32_t>* off) {
  if (off) off->resize(slot_level.size());
  uint64_t words = 0;
  for (size_t i = 0; i < slot_level.size(); ++i) {
    if (off) (*off)[i] = (uint32_t)words;
    words += ((cap[slot_level[i]] + 31) / 32 + 1 + 3) & ~3u;
  }
  return words;
}

// The type words of a batch (program.h): which scopes have them, which column is which nibble, and where each scope's words lie
// in the batch's one type-word allocation.  Computed from the column table alone, so the backend's allocation and pack pass, the
// code generator and the generated text's host build all take it from here.
struct GkTwLayout {
  std::vector<uint32_t> words;                // per scope: W_s, words per row (0: no type words)
  std::vector<std::vector<uint32_t>> vtcols;  // per scope with words: its VT columns in nibble order (column-index order)
  std::vector<uint32_t> nibble;               // per column: its nibble in its scope's row, or GK_NONE (no VT, or no words in the scope)
  bool operator==(const GkTwLayout& o) const { return words == o.words && vtcols == o.vtcols; }
  // the allocation of a batch with rows[s] rows in scope s: the per-scope pointer table (nscopes pointers), then each scope's
  // words, every region 16-byte aligned; `at` (if not null) gets every scope's byte offset (0: no words)
  size_t bytes(const std::vector<uint32_t>& rows, std::vector<size_t>* at) const {
    auto r16 = [](size_t b) { return (b + 15) / 16 * 16; };
    size_t off = r16(words.size() * 8);
    if (at) at->assign(words.size(), 0);
    for (size_t s = 0; s < words.size(); ++s) {
      if (!words[s]) continue;
      if (at) (*at)[s] = off;
      off += r16((s < rows.size() ? rows[s] : 0u) * (size_t)words[s] * 4);
    }
    return off;
  }
  bool any() const {
    for (uint32_t w : words)
      if (w) return true;
    return false;
  }
};
// cols: the batch's column table, anything with `scope` and `enc` (GkColumn, the schema's column definitions)
template <class Col>
inline GkTwLayout gk_tw_layout(const std::vector<Col>& cols, size_t nscopes) {
  GkTwLayout L;
  L.words.assign(nscopes, 0);
  L.vtcols.assign(nscopes, {});
  L.nibble.assign(cols.size(), GK_NONE);
  for (size_t ci = 0; ci < cols.size(); ++ci)
    if ((cols[ci].enc & GK_ENC_VT) && (size_t)cols[ci].scope < nscopes) L.vtcols[(size_t)cols[ci].scope].push_back((uint32_t)ci);
  for (size_t s = 0; s < nscopes; ++s) {
    L.words[s] = gk_tw_words((uint32_t)L.vtcols[s].size());
    if (!L.words[s]) {
      L.vtcols[s].clear();
      continue;
    }
    for (size_t k = 0; k < L.vtcols[s].size(); ++k) L.nibble[L.vtcols[s][k]] = (uint32_t)k;
  }
  return L;
}

// What one netlist needs in shared memory besides the tile: the table counts gk_eval_layout takes and the scope of every slot.
struct GkNetSize {
  uint32_t C, NS, NP, nops, nitems, nmatch, ncols, npool, ncbytes;
  std::vector<uint8_t> slot_level;
};

// Whether tiles of `tile` objects whose largest tile has cap[s] rows in scope s fit one launch: slot offsets must fit the netlist's
// 16-bit fields and the whole layout the per-CTA shared-memory limit.
inline bool gk_tile_fits(const GkNetSize& n, std::vector<uint32_t> cap, uint32_t tile, size_t max_smem) {
  cap[0] = tile;
  const uint64_t sw = gk_slot_layout(n.slot_level, cap, nullptr);
  return sw <= 0xffffu && gk_eval_layout(n.C, n.NS, n.NP, (uint32_t)sw, n.nops, n.nitems, n.nmatch, n.ncols, n.npool, n.ncbytes).total <= max_smem;
}

// Objects per tile: every bit column of a tile lives in the CTA's shared memory, so a page whose objects iterate very many rows
// needs smaller tiles, not a refusal.  Starts at `first` and halves (keeping a multiple of 32) until every netlist of `nets` fits,
// but not below 32 objects; a 32-object tile that still does not fit is refused at launch.  caps_of(tile) lays the batch out in
// tiles of that size and returns the rows of its largest tile per scope; its last call is for the tile returned.
template <class CapsOf>
inline uint32_t gk_choose_tile(uint32_t first, const std::vector<GkNetSize>& nets, size_t max_smem, CapsOf&& caps_of) {
  for (uint32_t tile = first;; tile = std::max(32u, tile / 2 / 32 * 32)) {
    const std::vector<uint32_t>& cap = caps_of(tile);
    bool fits = true;
    for (const GkNetSize& n : nets) fits = fits && gk_tile_fits(n, cap, tile, max_smem);
    if (fits || tile <= 32) return tile;
  }
}
