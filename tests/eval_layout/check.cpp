// Prints what eval_layout.h decides, for tests/test_eval_layout.py.  One request per line on stdin, one answer line per request:
//
//   layout C NS NP slot_words nops nitems nmatch ncols npool ncbytes
//       -> layout <s_tot> <s_err> ... <cbytes> <end> <total>
//   slots ncap cap... nslots level...
//       -> slots <total words> <offset of every slot>...
//   tile max_smem first nnets {C NS NP nops nitems nmatch ncols npool ncbytes nslots level...}... ntiles {tile ncap cap...}...
//       -> tile <chosen> fits <0|1> tried <tile sizes passed to the caps callback, in order>...
//   sizes
//       -> sizes <sizeof GkOutEnt> <GkOp> <GkMatch> <GkColumn> <GkScope>
#include <cstdio>
#include <iostream>
#include <map>
#include <sstream>
#include <string>

#include "eval_layout.h"

static std::vector<uint32_t> read_vec(std::istream& in) {
  size_t n = 0;
  in >> n;
  std::vector<uint32_t> v(n);
  for (auto& x : v) in >> x;
  return v;
}

int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string cmd;
    if (!(in >> cmd)) continue;
    if (cmd == "layout") {
      uint32_t a[10];
      for (auto& x : a) in >> x;
      const GkEvalLayout L = gk_eval_layout(a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7], a[8], a[9]);
      const size_t r[] = {L.s_tot, L.s_err, L.s_act, L.s_lo, L.s_cnt, L.s_poff, L.slots, L.outs, L.ops,
                          L.items, L.match, L.cols,  L.scopes, L.pool, L.cbytes, L.end,   L.total};
      std::printf("layout");
      for (size_t x : r) std::printf(" %zu", x);
    } else if (cmd == "slots") {
      const std::vector<uint32_t> cap = read_vec(in), lv = read_vec(in);
      std::vector<uint32_t> off;
      const uint64_t words = gk_slot_layout(std::vector<uint8_t>(lv.begin(), lv.end()), cap, &off);
      std::printf("slots %llu", (unsigned long long)words);
      for (uint32_t o : off) std::printf(" %u", o);
    } else if (cmd == "tile") {
      size_t max_smem = 0;
      uint32_t first = 0, nnets = 0, ntiles = 0;
      in >> max_smem >> first >> nnets;
      std::vector<GkNetSize> nets(nnets);
      for (auto& n : nets) {
        in >> n.C >> n.NS >> n.NP >> n.nops >> n.nitems >> n.nmatch >> n.ncols >> n.npool >> n.ncbytes;
        const std::vector<uint32_t> lv = read_vec(in);
        n.slot_level.assign(lv.begin(), lv.end());
      }
      std::map<uint32_t, std::vector<uint32_t>> caps;   // tile size -> rows of the largest tile per scope
      in >> ntiles;
      for (uint32_t i = 0; i < ntiles; ++i) {
        uint32_t t = 0;
        in >> t;
        caps[t] = read_vec(in);
      }
      std::vector<uint32_t> tried;
      const uint32_t tile = gk_choose_tile(first, nets, max_smem, [&](uint32_t t) -> const std::vector<uint32_t>& {
        tried.push_back(t);
        return caps.at(t);
      });
      bool fits = true;
      for (const GkNetSize& n : nets) fits = fits && gk_tile_fits(n, caps.at(tile), tile, max_smem);
      std::printf("tile %u fits %d tried", tile, fits ? 1 : 0);
      for (uint32_t t : tried) std::printf(" %u", t);
    } else if (cmd == "sizes") {
      std::printf("sizes %zu %zu %zu %zu %zu", sizeof(GkOutEnt), sizeof(GkOp), sizeof(GkMatch), sizeof(GkColumn), sizeof(GkScope));
    } else {
      std::fprintf(stderr, "unknown request: %s\n", cmd.c_str());
      return 2;
    }
    std::printf("\n");
  }
  return 0;
}
