// Netlist -> CUDA C++ text (see spec_codegen.hpp).  The semantics of every op are those of the interpreter (tile_kernel.cuh) and of
// the test-only host emulation; tests/_hostemu compiles the SAME text with g++ (-DGK_SPEC_HOST) and compares it object by object
// with the interpreted netlist (GK_SPEC_CHECK=1), which is how the generator is verified in a container without a GPU.
#include "spec_codegen.hpp"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <map>
#include <set>
#include <sstream>
#include <tuple>

#include "spec_headers.inc"   // kSpecHdrProgram / kSpecHdrVmCore: the text of program.h and vm_core.h (written by build.py)

namespace gk {

namespace {

std::string strip_includes(const char* text) {
  std::istringstream in(text);
  std::string line, out;
  while (std::getline(in, line)) {
    if (line.rfind("#pragma once", 0) == 0 || line.rfind("#include \"program.h\"", 0) == 0) continue;
    out += line;
    out += '\n';
  }
  return out;
}

std::string hx(uint32_t v) {
  char b[24];
  snprintf(b, sizeof b, "0x%xu", v);
  return b;
}

// the fixed part: launch wrapper (device) / per-object entry point (host test build)
const char* kWrapper = R"GKSRC(
#ifndef GK_SPEC_HOST
// xs: the export planes (gk_spec_rows_kernel); img: the offset image, a run of img_stride values per tile (gk_spec_plan_kernel)
extern "C" __global__ void __launch_bounds__(GK_SPEC_THREADS, GK_SPEC_MINB) gk_spec_kernel(const __grid_constant__ GkKParams p, const uint32_t* __restrict__ xs,
                                                                                          const uint16_t* __restrict__ img, const uint32_t img_stride) {
  extern __shared__ uint4 gk_smem4[];
  unsigned char* smem = reinterpret_cast<unsigned char*>(gk_smem4);
  const uint32_t NC = p.batch.ncols, NS = p.batch.nscopes;
  GkColumn* cols = reinterpret_cast<GkColumn*>(smem);
  GkScope* scopes = reinterpret_cast<GkScope*>(smem + (size_t)NC * sizeof(GkColumn));
  uint32_t* act = reinterpret_cast<uint32_t*>(smem + (size_t)NC * sizeof(GkColumn) + (size_t)NS * sizeof(GkScope));
  uint32_t* s_tot = act + GK_SPEC_W * 32u;
  uint32_t* s_err = s_tot + GK_SPEC_W * 32u;
  uint32_t* actw = s_err + GK_SPEC_W * 32u;   // the enforcement-point mask packed: bit c of word c / 32
  uint32_t* stg = reinterpret_cast<uint32_t*>(smem + GK_SPEC_STAGE_AT);   // the tile's staged export bits and offsets (gk_spec_stage)
  {
    const uint4* a = reinterpret_cast<const uint4*>(p.batch.cols);
    uint4* d = reinterpret_cast<uint4*>(cols);
    for (uint32_t i = threadIdx.x; i < NC * (uint32_t)(sizeof(GkColumn) / 16); i += blockDim.x) d[i] = a[i];
    const uint4* b = reinterpret_cast<const uint4*>(p.batch.scopes);
    uint4* e = reinterpret_cast<uint4*>(scopes);
    for (uint32_t i = threadIdx.x; i < NS * (uint32_t)(sizeof(GkScope) / 16); i += blockDim.x) e[i] = b[i];
    for (uint32_t i = threadIdx.x; i < GK_SPEC_W * 32u; i += blockDim.x) {
      act[i] = i < GK_SPEC_C ? p.active[i] : 0u;
      s_tot[i] = 0u;
      s_err[i] = 0u;
    }
  }
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u;
  for (uint32_t i = threadIdx.x; i < GK_SPEC_W * 32u; i += blockDim.x) {   // (whole warps: both bounds are multiples of 32)
    const uint32_t bits = __ballot_sync(0xffffffffu, act[i] != 0u);
    if (lane == 0u) actw[i >> 5] = bits;
  }
  __syncthreads();
  uint32_t tv[GK_SPEC_W], te[GK_SPEC_W];
#pragma unroll
  for (uint32_t w = 0; w < GK_SPEC_W; ++w) tv[w] = te[w] = 0u;
  for (uint32_t t = blockIdx.x; t < p.ntiles; t += gridDim.x) {
    // a tile handed over whole (gk_spec_plan_kernel) is the interpreter's: its words and its totals (uniform across the CTA)
    if (__ldg(p.whole + t)) continue;
    const uint32_t obj0 = t * p.tile, nobj = min(p.tile, p.batch.n - obj0);
    // phase 1: the copy of the tile's exports and offsets, every thread of the CTA; phase 2: its objects, one per thread.  (The
    // barrier at the end of the tile keeps the next tile's copy from overwriting what the last objects of this one still read.)
    const uint32_t* tl = p.tile_lo + (size_t)t * NS;
    gk_spec_stage(p.batch, scopes, xs, img + (size_t)t * img_stride, tl, tl + NS, stg, threadIdx.x, blockDim.x);
    __syncthreads();
#ifdef GK_SPEC_X_STAGEONLY   /* (measurement only: the staging of every tile without the object walk; results differ) */
    for (uint32_t base = nobj; base < nobj; base += blockDim.x) {
#else
    for (uint32_t base = 0; base < nobj; base += blockDim.x) {
#endif
      const uint32_t o = base + threadIdx.x;
      uint32_t vw[GK_SPEC_W], ew[GK_SPEC_W];
#pragma unroll
      for (uint32_t w = 0; w < GK_SPEC_W; ++w) vw[w] = ew[w] = 0u;
      if (o < nobj) {
        // A wide object (gk_spec_object() returns true) is a unit of the interpreter's, which may be storing its words right now:
        // nothing of it is stored here, and it is out of the totals.
        const bool wide = gk_spec_object(p.batch, stg, p.prog.pool, p.prog.cbytes, actw, p.out, obj0 + o, o, vw, ew);
        if (wide) {
#pragma unroll
          for (uint32_t w = 0; w < GK_SPEC_W; ++w) vw[w] = ew[w] = 0u;
        } else {
          const size_t at = (size_t)(obj0 + o) * GK_SPEC_W;
#if GK_SPEC_W == 2
          const uint2 v2 = make_uint2(vw[0], vw[1]);
          if (p.npeers) {
            for (uint32_t q = 0; q < p.npeers; ++q) *reinterpret_cast<uint2*>(p.peer_viol[q] + at) = v2;   // this rank is one of the peers
          } else {
            *reinterpret_cast<uint2*>(p.out.viol + at) = v2;
          }
          *reinterpret_cast<uint2*>(p.out.err + at) = make_uint2(ew[0], ew[1]);
#else
#pragma unroll
          for (uint32_t w = 0; w < GK_SPEC_W; ++w) {
            if (p.npeers) {
              for (uint32_t q = 0; q < p.npeers; ++q) p.peer_viol[q][at + w] = vw[w];
            } else {
              p.out.viol[at + w] = vw[w];
            }
            p.out.err[at + w] = ew[w];
          }
#endif
        }
      }
      // totals: after the transpose lane c holds the bit of constraint (32 w + c) for the warp's 32 objects
      uint32_t anye = 0u;
#pragma unroll
      for (uint32_t w = 0; w < GK_SPEC_W; ++w) {
        tv[w] += (uint32_t)__popc(gk_tr32(vw[w], lane));
        anye |= ew[w];
      }
      if (__any_sync(0xffffffffu, anye != 0u)) {
#pragma unroll
        for (uint32_t w = 0; w < GK_SPEC_W; ++w) te[w] += (uint32_t)__popc(gk_tr32(ew[w], lane));
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (uint32_t w = 0; w < GK_SPEC_W; ++w) {
    if (tv[w]) atomicAdd(&s_tot[w * 32u + lane], tv[w]);
    if (te[w]) atomicAdd(&s_err[w * 32u + lane], te[w]);
  }
  __syncthreads();
  for (uint32_t c = threadIdx.x; c < GK_SPEC_C; c += blockDim.x) {
    if (s_tot[c]) atomicAdd(p.out.totals + c, (unsigned long long)s_tot[c]);
    if (s_err[c]) atomicAdd(p.out.err_totals + c, (unsigned long long)s_err[c]);
  }
  if (p.npeers) gk_publish_totals(p, GK_SPEC_C, act);   // (act is free by now)
}

// The hand-over plan, before any row is evaluated: one CTA per tile finds the tile's wide objects from the CSR offsets
// (gk_spec_wide) and lists them for the interpreter -- each alone, or the whole tile when it has more than GK_HANDOVER_MAX
// (gk_spec_tile_whole) -- and sets the tile's whole flag, which gk_spec_kernel reads.  It also writes the tile's run of the offset
// image (gk_spec_offsets), which gk_spec_kernel stages.
extern "C" __global__ void gk_spec_plan_kernel(const __grid_constant__ GkKParams p, uint16_t* __restrict__ img, const uint32_t img_stride) {
  const uint32_t t = blockIdx.x, obj0 = t * p.tile, nobj = min(p.tile, p.batch.n - obj0);
  const uint32_t* tl = p.tile_lo + (size_t)t * p.batch.nscopes;
  gk_spec_offsets(p.batch.scopes, tl, tl + p.batch.nscopes, img + (size_t)t * img_stride, threadIdx.x, blockDim.x);
  uint32_t nwide = 0u;
  for (uint32_t base = 0; base < nobj; base += blockDim.x) {
    const uint32_t o = base + threadIdx.x;
    nwide += (uint32_t)__syncthreads_count(o < nobj && gk_spec_wide(p.batch.scopes, obj0 + o));
  }
  const bool whole = gk_spec_tile_whole(nwide);
  if (threadIdx.x == 0) {
    p.whole[t] = whole ? 1u : 0u;
    if (whole) {
      const uint32_t u = atomicAdd(p.unit_count, 1u);
      p.units[2 * u] = obj0;
      p.units[2 * u + 1] = nobj;
    }
  }
  if (nwide && !whole)
    for (uint32_t o = threadIdx.x; o < nobj; o += blockDim.x)
      if (gk_spec_wide(p.batch.scopes, obj0 + o)) {
        const uint32_t u = atomicAdd(p.unit_count, 1u);
        p.units[2 * u] = obj0 + o;
        p.units[2 * u + 1] = 1u;
      }
}
#else
#include <vector>
#include <cstdio>
#include <cstdlib>
#include <string>
// TEST-ONLY host build: the hand-over plan of gk_spec_plan_kernel for tiles of `tile` objects, tile after tile and a tile's
// objects in order (the kernel appends them in any order).  Fills units (capacity: 2 per object) and whole (one per tile); returns
// the units.  Also, into `im`, the offset image of those tiles as the kernel writes it: `stride` values per tile
// (gk_spec_image_stride of the largest tile's rows per scope, the tile itself in scope 0, as the backend sizes it), a value no run
// covers poisoned; `fits` as the backend decides whether the batch may run the generated kernel (gk_spec_image_fits).
#ifndef GK_SPEC_HOST_PLAN_TILE
#define GK_SPEC_HOST_PLAN_TILE 512u   /* the device's tile (tile_kernel.cuh GK_TILE) */
#endif
struct GkSpecHostImage {
  std::vector<uint16_t> img;
  std::vector<uint32_t> lo, hi;   // [tiles * GK_SPEC_NS] each tile's first row and end per scope (the nested scopes and scope 0)
  uint32_t stride = 0u;
  bool fits = true;
};
static uint32_t gk_spec_host_plan(const GkBatch& B, uint32_t tile, std::vector<uint32_t>& units, std::vector<uint32_t>& whole, GkSpecHostImage& im) {
  units.clear();
  whole.assign((B.n + tile - 1u) / tile, 0u);
  const size_t NT = whole.size();
  im.lo.assign(NT * GK_SPEC_NS, 0u);
  im.hi.assign(NT * GK_SPEC_NS, 0u);
  std::vector<uint32_t> cap(GK_SPEC_NS, 0u);
  for (size_t t = 0; t < NT; ++t) {
    uint32_t* lo = im.lo.data() + t * GK_SPEC_NS;
    uint32_t* hi = im.hi.data() + t * GK_SPEC_NS;
    lo[0] = (uint32_t)t * tile;
    hi[0] = B.n - lo[0] < tile ? B.n : lo[0] + tile;
    gk_spec_tile_rows(B.scopes, lo, hi);
    for (uint32_t s = 0; s < GK_SPEC_NS; ++s) cap[s] = hi[s] - lo[s] > cap[s] ? hi[s] - lo[s] : cap[s];
  }
  cap[0] = tile;
  im.stride = gk_spec_image_stride(cap.data());
  im.fits = gk_spec_image_fits(cap.data());
  im.img.assign(NT * im.stride, 0xbeefu);
  for (size_t t = 0; t < NT; ++t)
    gk_spec_offsets(B.scopes, im.lo.data() + t * GK_SPEC_NS, im.hi.data() + t * GK_SPEC_NS, im.img.data() + t * im.stride, 0u, 1u);
  for (uint32_t t = 0; t < whole.size(); ++t) {
    const uint32_t obj0 = t * tile, nobj = B.n - obj0 < tile ? B.n - obj0 : tile;
    uint32_t nwide = 0u;
    for (uint32_t o = 0; o < nobj; ++o) nwide += gk_spec_wide(B.scopes, obj0 + o) ? 1u : 0u;
    whole[t] = gk_spec_tile_whole(nwide) ? 1u : 0u;
    if (whole[t]) {
      units.insert(units.end(), {obj0, nobj});
    } else {
      for (uint32_t o = 0; o < nobj; ++o)
        if (gk_spec_wide(B.scopes, obj0 + o)) units.insert(units.end(), {obj0 + o, 1u});
    }
  }
  return (uint32_t)(units.size() / 2);
}
// TEST-ONLY host build (tests/_hostemu, GK_SPEC_CHECK=1): one object; returns 1 when the object does not fit the mask registers.
// The rows of the object's tile (GK_SPEC_HOST_TILE objects; its rows found through the CSR offsets) are evaluated by the same
// gk_spec_row_<g>() the rows kernel runs into a poisoned export buffer, which the same gk_spec_stage() the tile kernel runs copies
// with three "threads" striding over it; both again only when `obj` leaves the tile (or starts it again).
// The objects are checked in order: at the last one the hand-over plan of the batch is made, and every object the plan's test
// (gk_spec_wide) decides otherwise than the object walk did is counted.  GK_SPEC_TRACE=1 prints the plan and that count:
//   [spec plan] tiles of T: U units: <first object>+<objects> ...; whole tiles: <tile> ...; disagreements: D
#ifndef GK_SPEC_HOST_TILE
#define GK_SPEC_HOST_TILE 96u
#endif
extern "C" int gk_spec_host(const GkKParams* p, uint32_t obj, uint32_t* vw, uint32_t* ew) {
  // the batch's type words, packed again at its first object (the backend packs them where the batch becomes resident)
  struct Types {
    const void* flags = nullptr;
    uint32_t n = 0;
    std::vector<std::vector<uint32_t>> words;
    std::vector<const uint32_t*> ptrs;
  };
  static thread_local Types ty;
  if (obj == 0u || ty.flags != (const void*)p->batch.flags || ty.n != p->batch.n) {
    gk_spec_host_types(p->batch, ty.words, ty.ptrs);
    ty.flags = p->batch.flags;
    ty.n = p->batch.n;
  }
  GkKParams pt = *p;
  pt.batch.tw = ty.ptrs.data();
  p = &pt;
  uint32_t actw[GK_SPEC_W];
  for (uint32_t w = 0; w < GK_SPEC_W; ++w) vw[w] = ew[w] = actw[w] = 0u;
  for (uint32_t c = 0; c < GK_SPEC_C; ++c)
    if (p->active[c]) actw[c >> 5] |= 1u << (c & 31u);
  // the batch's offset image for the tiles below, made again at its first object (the plan kernel writes it once per batch); a batch
  // whose tile rows do not fit it is the interpreter's: every object is handed over
  struct Image {
    const void* flags = nullptr;
    uint32_t n = 0;
    GkSpecHostImage im;
  };
  static thread_local Image ki;
  if (obj == 0u || ki.flags != (const void*)p->batch.flags || ki.n != p->batch.n) {
    std::vector<uint32_t> u, wh;
    gk_spec_host_plan(p->batch, GK_SPEC_HOST_TILE, u, wh, ki.im);
    ki.flags = p->batch.flags;
    ki.n = p->batch.n;
  }
  if (!ki.im.fits) return 1;
  struct Tile {
    const void* flags = nullptr;
    uint32_t n = 0, t = 0xffffffffu;
    std::vector<uint32_t> lo, hi, stg, x;
    std::vector<uint8_t> walk_wide;   // what gk_spec_object() returned, per object of the batch so far
  };
  static thread_local Tile k;
  const GkBatch& B = p->batch;
  const uint32_t T = GK_SPEC_HOST_TILE, t = obj / T;
  if (t != k.t || k.flags != (const void*)B.flags || k.n != B.n || obj % T == 0u) {
    k.lo.assign(GK_SPEC_NS, 0u);
    k.hi.assign(GK_SPEC_NS, 0u);
    k.lo[0] = t * T;
    k.hi[0] = B.n - t * T < T ? B.n : (t + 1u) * T;
    gk_spec_tile_rows(B.scopes, k.lo.data(), k.hi.data());
    k.stg.assign(gk_spec_stage_words(k.lo.data(), k.hi.data()), 0xdeadbeefu);   // (poisoned: a word the staging misses shows)
    k.x.assign(gk_spec_export_words(B), 0xdeadbeefu);
    gk_spec_host_rows(p, k.lo.data(), k.hi.data(), k.x.data());
    for (uint32_t tid = 0; tid < 3u; ++tid)
      gk_spec_stage(B, B.scopes, k.x.data(), ki.im.img.data() + (size_t)t * ki.im.stride, k.lo.data(), k.hi.data(), k.stg.data(), tid, 3u);
    k.flags = B.flags;
    k.n = B.n;
    k.t = t;
  }
  const int wide = gk_spec_object(B, k.stg.data(), p->prog.pool, p->prog.cbytes, actw, p->out, obj, obj - t * T, vw, ew) ? 1 : 0;
  if (obj == 0u) {
    k.walk_wide.assign(B.n, 2u);   // (2: not walked)
    if (getenv("GK_SPEC_TRACE")) gk_spec_trace_planes(B);
  }
  if (obj < k.walk_wide.size()) k.walk_wide[obj] = (uint8_t)wide;
  if (obj + 1u == B.n && k.walk_wide.size() == B.n) {
    uint32_t disagree = 0u;
    for (uint32_t o = 0; o < B.n; ++o) disagree += k.walk_wide[o] != (gk_spec_wide(B.scopes, o) ? 1u : 0u);
    std::vector<uint32_t> units, whole;
    GkSpecHostImage im;
    const uint32_t nu = gk_spec_host_plan(B, GK_SPEC_HOST_PLAN_TILE, units, whole, im);
    if (getenv("GK_SPEC_TRACE")) {
      // "[spec offsets] tiles of T: scopes <s>/<parent> ...; rows <the tile's rows of each parent> | ...; stride <S> bytes; runs <R>
      // bytes; image <I> bytes" (a run: the values gk_spec_stage() copies, padded to 16 bytes)
      std::string ol = "[spec offsets] tiles of " + std::to_string(GK_SPEC_HOST_PLAN_TILE) + ": scopes";
      size_t runs = 0;
      for (uint32_t s = 1; s < GK_SPEC_NS; ++s)
        if (gk_spec_parent(s) < GK_SPEC_NS) ol += " " + std::to_string(s) + "/" + std::to_string(gk_spec_parent(s));
      ol += "; rows";
      for (size_t t = 0; t < whole.size(); ++t) {
        uint32_t ni = 0u;
        ol += t ? " |" : "";
        for (uint32_t s = 1; s < GK_SPEC_NS; ++s) {
          const uint32_t P = gk_spec_parent(s);
          if (P >= GK_SPEC_NS) continue;
          const uint32_t c = im.hi[t * GK_SPEC_NS + P] - im.lo[t * GK_SPEC_NS + P];
          ol += " " + std::to_string(c);
          ni += c + 1u;
        }
        runs += (ni + 7u) / 8u * 16u;
      }
      ol += "; stride " + std::to_string(2u * im.stride) + " bytes; runs " + std::to_string(runs) + " bytes; image " + std::to_string(im.img.size() * 2) + " bytes";
      fprintf(stderr, "%s\n", ol.c_str());
      std::string line = "[spec plan] tiles of " + std::to_string(GK_SPEC_HOST_PLAN_TILE) + ": " + std::to_string(nu) + " units:";
      for (uint32_t u = 0; u < nu; ++u) line += " " + std::to_string(units[2 * u]) + "+" + std::to_string(units[2 * u + 1]);
      line += "; whole tiles:";
      for (uint32_t w = 0; w < whole.size(); ++w)
        if (whole[w]) line += " " + std::to_string(w);
      line += "; disagreements: " + std::to_string(disagree);
      fprintf(stderr, "%s\n", line.c_str());
    }
  }
  return wide;
}
#endif
)GKSRC";

// ---- one spec.match block written out as gk_spec_match_<mid>(): the same eight criteria in the same order as gk_match_row() /
// gk_match() (vm_core.h; reference pkg/mutation/match/match.go:32-65, pkg/target/matcher.go:21-71), with everything the block fixes
// folded in.  Returns false (nothing written) when the block's tables do not lie inside the pool: the caller then keeps the generic form.
// a wildcard pattern (wildcard.go:17-41) against the bytes s[0, sl): the pattern's bytes are immediates
std::string wild_expr(const Compiled& c, uint32_t mode, uint32_t off, uint32_t len, const std::string& s, const std::string& sl, bool generate_name) {
  const std::string L = std::to_string(len) + "u";
  if (generate_name && mode != GK_W_PREFIX && mode != GK_W_CONTAINS) return "false";   // exact and "*x" never match a generateName
  const std::string generic = std::string(generate_name ? "gk_wild_gen(" : "gk_wild(") + std::to_string(mode) + "u, cbytes + " + std::to_string(off) + "u, " + L + ", " + s + ", " + sl + ")";
  if ((size_t)off + len > c.cbytes.size() || len > 24u) return generic;
  if (mode == GK_W_CONTAINS) return len == 0 ? "true" : generic;
  std::string e = "(" + sl + (mode == GK_W_EXACT ? " == " : " >= ") + L;
  for (uint32_t i = 0; i < len; ++i) {
    const std::string at = mode == GK_W_SUFFIX ? s + " + (" + sl + " - " + L + ") + " + std::to_string(i) + "u" : s + " + " + std::to_string(i) + "u";
    e += " && GK_LD(" + at + ") == " + hx(c.cbytes[off + i]);
  }
  return e + ")";
}

// labels.Selector.Matches over the (key, value) run [lo, hi) of `kv`: one walk of the run fetches the value of every key the
// selector names (backwards, so that the first entry of a key is the one that stays, as in gk_label()); statements that `return 0`
bool selector_code(std::ostringstream& o, const Compiled& c, uint32_t off, uint32_t nreq, const std::string& kv, const std::string& lo, const std::string& hi,
                   const std::string& tag) {
  struct Req {
    uint32_t key, op;
    std::vector<uint32_t> vals;
  };
  std::vector<Req> reqs;
  std::vector<uint32_t> keys;
  for (uint32_t r = 0; r < nreq; ++r) {
    if ((size_t)off + 3 > c.pool.size()) return false;
    Req q{c.pool[off], c.pool[off + 1], {}};
    const uint32_t nv = c.pool[off + 2];
    if ((size_t)off + 3 + nv > c.pool.size() || nv > 64u) return false;
    q.vals.assign(c.pool.begin() + off + 3, c.pool.begin() + off + 3 + nv);
    off += 3 + nv;
    if (std::find(keys.begin(), keys.end(), q.key) == keys.end()) keys.push_back(q.key);
    reqs.push_back(std::move(q));
  }
  if (reqs.empty()) return true;
  o << "  {\n    uint32_t";
  for (size_t k = 0; k < keys.size(); ++k) o << (k ? ", " : " ") << tag << k << " = GK_NONE";
  o << ";\n    _Pragma(\"unroll 1\") for (uint32_t i = " << hi << "; i-- > " << lo << ";) {\n      const uint32_t k = GK_LD(" << kv << " + 2u * i), v = GK_LD(" << kv
    << " + 2u * i + 1u);\n";
  for (size_t k = 0; k < keys.size(); ++k) o << "      if (k == " << hx(keys[k]) << ") " << tag << k << " = v;\n";
  o << "    }\n";
  for (const Req& q : reqs) {
    const std::string x = tag + std::to_string(std::find(keys.begin(), keys.end(), q.key) - keys.begin());
    const std::string has = "(" + x + " != GK_NONE)";
    std::string in = "false";
    if (!q.vals.empty()) {
      in = "(" + has + " && (";
      for (size_t j = 0; j < q.vals.size(); ++j) in += (j ? " || " : "") + x + " == " + hx(q.vals[j]);
      in += "))";
    }
    const std::string ok = q.op == GK_SEL_IN ? in : q.op == GK_SEL_NOTIN ? "!" + in : q.op == GK_SEL_EXISTS ? has : "!" + has;
    o << "    if (!(" << ok << ")) return 0;\n";
  }
  o << "  }\n";
  return true;
}

bool emit_match(std::ostringstream& out, const Compiled& c, uint32_t mid) {
  const GkMatch& m = c.match[mid];
  const std::string M = std::to_string(mid);
  const char* sig_tail = "(const GkBatch& B, const uint32_t* __restrict__ pool, const uint8_t* __restrict__ cbytes, ";
  std::ostringstream o;
  if (!(m.flags & GK_M_HAS_MATCH)) {   // matcher.go:22-25: no spec.match matches everything
    out << "GK_SPEC_FN int gk_spec_match_" << M << sig_tail << "const uint32_t obj) {\n  (void)B; (void)pool; (void)cbytes; (void)obj;\n  return 1;\n}\n";
    return true;
  }
  o << "GK_SPEC_FN int gk_spec_mrow_" << M << sig_tail << "const uint32_t row, const uint32_t obj) {\n  (void)pool; (void)cbytes; (void)obj;\n";
  o << "  const uint32_t fl = GK_LD(B.flags + row);\n  const bool is_ns = (fl & GK_F_IS_NS) != 0u;\n  (void)is_ns;\n";
  // 1 kinds -- match.go:181-201
  if (m.kinds_n) {
    std::string any;
    uint32_t off = m.kinds_off;
    bool always = false;
    for (uint32_t e = 0; e < m.kinds_n; ++e) {
      if ((size_t)off + 3 > c.pool.size()) return false;
      const uint32_t nk = c.pool[off], ng = c.pool[off + 1], wild = c.pool[off + 2];
      if ((size_t)off + 3 + nk + ng > c.pool.size() || nk > 64u || ng > 64u) return false;
      std::string km, gm;
      if (!(nk == 0 || (wild & 1u))) {
        for (uint32_t j = 0; j < nk; ++j) km += (j ? " || kind == " : "kind == ") + hx(c.pool[off + 3 + j]);
        km = "(" + km + ")";
      }
      if (!(ng == 0 || (wild & 2u))) {
        for (uint32_t j = 0; j < ng; ++j) gm += (j ? " || group == " : "group == ") + hx(c.pool[off + 3 + nk + j]);
        gm = "(" + gm + ")";
      }
      const std::string both = km.empty() && gm.empty() ? "" : km.empty() ? gm : gm.empty() ? km : "(" + km + " && " + gm + ")";
      if (both.empty()) always = true;
      else any += (any.empty() ? "" : " || ") + both;
      off += 3 + nk + ng;
    }
    if (!always) o << "  {\n    const uint32_t kind = GK_LD(B.kind_sid + row), group = GK_LD(B.group_sid + row);\n    (void)kind; (void)group;\n    if (!(" << any << ")) return 0;\n  }\n";
  }
  // 2 scope -- match.go:214-227
  if (m.flags & (GK_M_SCOPE_CLUSTER | GK_M_SCOPE_NAMESPACED)) {
    o << "  {\n    const bool has_ns = (fl & (GK_F_HAS_NS | GK_F_NS_OBJ)) != 0u;\n";
    if (m.flags & GK_M_SCOPE_CLUSTER) o << "    if (!(is_ns || !has_ns)) return 0;\n";
    if (m.flags & GK_M_SCOPE_NAMESPACED) o << "    if (!(!is_ns && has_ns)) return 0;\n";
    o << "  }\n";
  }
  // 3/4 namespaces, excludedNamespaces -- match.go:118-179
  if (m.ns_n || m.exns_n) {
    if ((size_t)m.ns_off + 3 * (size_t)m.ns_n > c.pool.size() || (size_t)m.exns_off + 3 * (size_t)m.exns_n > c.pool.size() || m.ns_n > 64u || m.exns_n > 64u) return false;
    o << "  if (fl & GK_F_NSNAME) {\n    const uint32_t s0 = GK_LD(B.nsn_off + row), sl = GK_LD(B.nsn_off + row + 1u) - s0;\n    const uint8_t* s = B.nsn_bytes + s0;\n    (void)s; (void)sl;\n";
    if (m.ns_n) {
      o << "    if (!(";
      for (uint32_t j = 0; j < m.ns_n; ++j) {
        const uint32_t* e = &c.pool[m.ns_off + 3 * j];
        o << (j ? "\n          || " : "") << wild_expr(c, e[0], e[1], e[2], "s", "sl", false);
      }
      o << ")) return 0;\n";
    }
    for (uint32_t j = 0; j < m.exns_n; ++j) {
      const uint32_t* e = &c.pool[m.exns_off + 3 * j];
      o << "    if (" << wild_expr(c, e[0], e[1], e[2], "s", "sl", false) << ") return 0;\n";
    }
    o << "  }\n";
  }
  // 5 labelSelector -- match.go:103-116
  if (m.flags & GK_M_HAS_LSEL) {
    if (m.flags & GK_M_LSEL_INVALID) {
      o << "  return -GK_E_LSEL_INVALID;\n}\n";
      goto wrapper;
    }
    o << "  {\n    const uint32_t l0 = GK_LD(B.lbl_off + row), l1 = GK_LD(B.lbl_off + row + 1u);\n";
    if (!selector_code(o, c, m.lsel_off, m.lsel_n, "B.lbl_kv", "l0", "l1", "lv")) return false;
    o << "  }\n";
  }
  // 6 namespaceSelector -- match.go:73-101
  if (m.flags & GK_M_HAS_NSSEL) {
    o << "  {\n    const bool ns_obj = (fl & GK_F_NS_OBJ) != 0u, obj_ns = (fl & GK_F_HAS_NS) != 0u;\n    if (is_ns || ns_obj || obj_ns) {\n";
    if (m.flags & GK_M_NSSEL_INVALID) {
      o << "      return -GK_E_NSSEL_INVALID;\n    }\n  }\n";
    } else {
      o << "      if (is_ns) {\n        const uint32_t l0 = GK_LD(B.lbl_off + row), l1 = GK_LD(B.lbl_off + row + 1u);\n";
      if (!selector_code(o, c, m.nssel_off, m.nssel_n, "B.lbl_kv", "l0", "l1", "sv")) return false;
      o << "      } else {\n        if (!ns_obj) return -GK_E_NS_MISSING;\n        const uint32_t nr = GK_LD(B.nsrow + obj);\n        const uint32_t l0 = GK_LD(B.nsl_off + nr), l1 = GK_LD(B.nsl_off + nr + 1u);\n";
      if (!selector_code(o, c, m.nssel_off, m.nssel_n, "B.nsl_kv", "l0", "l1", "nv")) return false;
      o << "      }\n    }\n  }\n";
    }
  }
  // 7 name -- match.go:203-212
  if (m.flags & GK_M_HAS_NAME) {
    o << "  {\n    const uint32_t a = GK_LD(B.name_off + row), al = GK_LD(B.name_off + row + 1u) - a;\n    const uint8_t* nm = B.name_bytes + a;\n    (void)nm; (void)al;\n";
    o << "    bool ok = " << wild_expr(c, m.name_mode, m.name_boff, m.name_len, "nm", "al", false) << ";\n";
    const std::string ge = wild_expr(c, m.name_mode, m.name_boff, m.name_len, "gn", "gl", true);
    if (ge != "false")
      o << "    if (!ok) {\n      const uint32_t g = GK_LD(B.gen_off + row), gl = GK_LD(B.gen_off + row + 1u) - g;\n      const uint8_t* gn = B.gen_bytes + g;\n      (void)gn; (void)gl;\n      ok = " << ge
        << ";\n    }\n";
    o << "    if (!ok) return 0;\n  }\n";
  }
  // 8 source -- match.go:229-253
  {
    if (m.flags & GK_M_SRC_INVALID) {
      o << "  return -GK_E_SRC_INVALID_MATCH;\n}\n";
      goto wrapper;
    }
    const uint32_t msrc = (m.flags >> GK_M_SRC_SHIFT) & 7u;
    if (msrc != GK_SRC_ALL) {
      o << "  {\n    const uint32_t tsrc = (fl & GK_F_SRC_MASK) >> GK_F_SRC_SHIFT;\n    if (tsrc == GK_SRC_EMPTY) return -GK_E_SRC_UNSPECIFIED;\n    if (tsrc == GK_SRC_INVALID) return -GK_E_SRC_INVALID_OBJ;\n    if (tsrc != "
        << msrc << "u) return 0;\n  }\n";
    }
  }
  o << "  return 1;\n}\n";
wrapper:
  // Matcher.Match: the object, then the old object (matcher.go:21-71); one copy of the row code for both
  o << "GK_SPEC_FN int gk_spec_match_" << M << sig_tail << "const uint32_t obj) {\n  int nil = 0;\n"
    << "  _Pragma(\"unroll 1\") for (uint32_t pass = 0u; pass < 2u; ++pass) {\n"
    << "    if (pass && !B.has_old) {\n      ++nil;\n      break;\n    }\n"
    << "    const uint32_t row = pass ? B.n + obj : obj;\n"
    << "    if (!(GK_LD(B.flags + row) & GK_F_HAS_OBJ)) {\n      ++nil;\n      continue;\n    }\n"
    << "    const int r = gk_spec_mrow_" << M << "(B, pool, cbytes, row, obj);\n"
    << "    if (r < 0) return pass ? r - GK_E_FROM_OLD : r;   // the error text names the object that failed: here the old one\n"
    << "    if (r) return r;\n  }\n  return nil == 2 ? -GK_E_NO_OBJECT : 0;\n}\n";
  out << o.str();
  return true;
}

// One netlist op after SSA renaming (slots are reused by liveness; every write gets a fresh variable): its text, what it
// reads and what it defines.  Nodes are emitted depth-first from the constraint results (see spec_codegen()), not in netlist
// order, which keeps the live values of one scope subtree together instead of all ~300 at once.
struct SpecNode {
  std::string code;
  std::vector<uint32_t> deps;
  bool done = false;
  // what the row-local classification (spec_codegen()) reads: the op's kind and scope; of a gate its inputs (variable, or -1 for a
  // slot never written = 0; negated?) and flags, so that phase 1 can write it as a boolean expression; of a constant its value
  uint32_t kind = GK_N_END, level = 0;
  std::vector<std::pair<int, bool>> in;
  bool is_or = false, neg_out = false, one = false;
};

struct Gen {
  const Compiled& c;
  std::vector<SpecNode> nodes;
  std::vector<int> producer;               // variable -> node, or -(scope + 1) for an atom of that scope's row loop
  struct AtomRec {
    uint32_t var, scope;
    std::string expr;                              // boolean expression over the row's loaded values
    std::map<uint32_t, uint32_t> need;             // column -> encodings the expression reads
    int group = -1;                                // row loop it is computed in (see spec_codegen())
  };
  std::vector<AtomRec> atoms;
  std::vector<int> atom_of;                        // variable -> atom record, or -1
  std::map<uint32_t, uint32_t>* need_now = nullptr;
  std::vector<uint8_t> scope_used;
  std::vector<int> cur;                    // slot -> variable holding its current value (-1: never written)
  uint32_t nvar = 0;
  size_t n_fast = 0, n_generic = 0;
  std::set<uint32_t> match_used;
  struct MatchRec {
    uint32_t vm, ve, mid;                  // match bit, error bit, block
  };
  std::vector<MatchRec> matches;
  std::ostringstream body;                 // the node being built
  std::vector<uint32_t> deps;

  explicit Gen(const Compiled& cc) : c(cc) {
    const size_t NS = c.schema.scopes.size();
    scope_used.assign(NS, 0);
    cur.assign(c.slot_level.size() + 1, -1);
  }
  void use_scope(uint32_t s) {
    while (!scope_used[s]) {
      scope_used[s] = 1;
      if (s == 0) break;
      s = (uint32_t)c.schema.scopes[s].parent;
    }
  }
  std::string rd(uint32_t slot) {
    if (slot >= cur.size() || cur[slot] < 0) return "0u";
    deps.push_back((uint32_t)cur[slot]);
    return "v" + std::to_string(cur[slot]);
  }
  uint32_t fresh(uint32_t slot, int prod) {
    if (slot >= cur.size()) cur.resize(slot + 1, -1);
    cur[slot] = (int)nvar;
    producer.push_back(prod);
    atom_of.push_back(-1);
    return nvar++;
  }
  uint32_t fresh(uint32_t slot) { return fresh(slot, (int)nodes.size()); }   // defined by the node being built
  SpecNode cur_node;                       // (its structured part, filled in by op())
  void finish_node() {
    cur_node.code = body.str();
    cur_node.deps = deps;
    nodes.push_back(std::move(cur_node));
    cur_node = SpecNode();
    body.str("");
    deps.clear();
  }

  // a boolean C expression for one atom on `row` of column ci; the loads it needs are recorded in col_need
  std::string atom_expr(uint32_t level, uint32_t ci, uint32_t aop, uint32_t a, uint32_t b) {
    const std::string K = std::to_string(ci);
    (void)level;
    auto need = [&](uint32_t enc) { (*need_now)[ci] |= enc; };
    const std::string t = "t" + K, i = "i" + K, n = "n" + K;
    switch (aop) {
      case GK_OP_TRUTHY: need(GK_ENC_VT); ++n_fast; return "(" + t + " != 0u && " + t + " != 2u)";
      case GK_OP_DEFINED: need(GK_ENC_VT); ++n_fast; return "(" + t + " != 0u)";
      case GK_OP_VTMASK: need(GK_ENC_VT); ++n_fast; return "(((" + hx(a) + " >> " + t + ") & 1u) != 0u)";
      case GK_OP_SID_EQ: need(GK_ENC_SID); ++n_fast; return "(" + i + " == " + hx(a) + ")";
      case GK_OP_SID_IN:
        if (b <= 16u && (size_t)a + b <= c.pool.size()) {
          need(GK_ENC_SID);
          ++n_fast;
          if (b == 0) return "false";
          std::string e = "(";
          for (uint32_t j = 0; j < b; ++j) e += (j ? " || " : "") + i + " == " + hx(c.pool[a + j]);
          return e + ")";
        }
        break;
      case GK_OP_NUM_CMP: {
        if ((size_t)a + 1 >= c.pool.size()) break;
        const int64_t k = (int64_t)(((uint64_t)c.pool[a + 1] << 32) | c.pool[a]);
        if (k == INT64_MIN || k == INT64_MAX) break;   // the sentinels of non-numbers: the generic path orders by type rank
        // (a defined non-number holds INT64_MIN / INT64_MAX by its type rank, so one signed compare is OPA's order: tile_kernel.cuh)
        need(GK_ENC_VT | GK_ENC_NUM);
        ++n_fast;
        const char* opn = b == GK_CMP_LT ? "<" : b == GK_CMP_LE ? "<=" : b == GK_CMP_GT ? ">" : b == GK_CMP_GE ? ">=" : b == GK_CMP_EQ ? "==" : "!=";
        return "(" + t + " != 0u && " + n + " " + opn + " " + std::to_string((long long)k) + "LL)";
      }
      case GK_OP_ANYPREFIX: {
        bool all_short = (size_t)a + (size_t)b * GK_PREFIX_ENT <= c.pool.size();
        for (uint32_t j = 0; all_short && j < b; ++j) all_short = c.pool[a + j * GK_PREFIX_ENT] <= GK_HEAD_BYTES;
        if (!all_short) break;
        need(GK_ENC_VT | GK_ENC_HEAD);
        ++n_fast;
        if (b == 0) return "false";
        const std::string h = "h" + K;
        static const char* comp[8] = {"a.x", "a.y", "a.z", "a.w", "b.x", "b.y", "b.z", "b.w"};
        std::string e = "(" + t + " == 5u && (";
        for (uint32_t j = 0; j < b; ++j) {
          const uint32_t* ent = &c.pool[a + j * GK_PREFIX_ENT];
          std::string one = "((" + h + "b.w >> 24) >= " + std::to_string(ent[0]) + "u";
          for (uint32_t w = 0; w < GK_HEAD_WORDS; ++w) {
            const uint32_t m = ent[2 + GK_HEAD_WORDS + w], v = ent[2 + w] & m;
            if (!m) continue;
            if (m == 0xffffffffu) one += " && " + h + comp[w] + " == " + hx(v);
            else one += " && (" + h + comp[w] + " & " + hx(m) + ") == " + hx(v);
          }
          e += (j ? " || " : "") + one + ")";
        }
        return e + "))";
      }
      default: break;
    }
    ++n_generic;
    return "gk_atom(cols[" + K + "], (uint32_t)row, " + std::to_string(aop) + "u, " + hx(a) + ", " + hx(b) + ", pool, cbytes)";
  }

  void atom(uint32_t level, uint32_t out_slot, uint32_t ci, uint32_t aop, uint32_t a, uint32_t b) {
    use_scope(level);
    AtomRec r;
    r.var = fresh(out_slot, -1);
    r.scope = level;
    need_now = &r.need;
    r.expr = atom_expr(level, ci, aop, a, b);
    need_now = nullptr;
    atom_of[r.var] = (int)atoms.size();
    atoms.push_back(std::move(r));
  }

  // `rm` = the mask of the children of parent row pj inside the object's rows of scope L, `pb` = the parent row's own bit.  The CSR
  // offsets are monotone, so rm = (rows below the END of pj) & ~(rows below its START), and the start of pj is the end of pj - 1: one
  // load and one mask per turn, carried.  (lo<L> is by definition the offset at lo<P>: the first parent's children start at bit 0.)
  // q<L> is the tile's slice of the offsets in shared memory, tile-relative 16-bit values (gk_spec_stage).
  // Not unrolled: parents have one to three rows here, the unrolled-by-four body the compiler makes is text that never runs.
  std::string range_loop_head(uint32_t L) {
    const uint32_t P = (uint32_t)c.schema.scopes[L].parent;
    const std::string l = std::to_string(L), p = std::to_string(P);
    return "  {\n  uint32_t lmp = 0u;\n  _Pragma(\"unroll 1\") for (uint32_t pj = 0; pj < n" + p + "; ++pj) {\n    const uint32_t rb = (uint32_t)q" + l + "[lo" + p + " + pj + 1u] - lo" + l +
           ";\n    const uint32_t lm = rb >= 32u ? 0xffffffffu : ((1u << rb) - 1u), rm = lm & ~lmp, pb = 1u << pj;\n    lmp = lm;\n    (void)pb;\n";
  }

  void op(const GkOp& op) {
    const uint32_t kind = op.w0 & 0xffu, level = (op.w0 >> 8) & 0xffu, out = op.w0 >> 16;
    const std::string L = std::to_string(level);
    cur_node.kind = kind;
    cur_node.level = level;
    switch (kind) {
      case GK_N_ATOM: atom(level, out, op.w1 >> 8, op.w1 & 0xffu, op.w2, op.w3); break;
      case GK_N_ATOMS:
        for (uint32_t j = 0; j < op.w3; ++j) {
          const uint32_t* e = &c.pool[op.w2 + j * GK_ATOMS_ENT];
          atom(level, e[0] >> 16, op.w1 >> 8, e[0] & 0xffu, e[1], e[2]);
        }
        break;
      case GK_N_CONST: {
        use_scope(level);
        const uint32_t v = fresh(out);
        cur_node.one = (op.w1 & 1u) != 0u;
        body << "  const uint32_t v" << v << " = " << ((op.w1 & 1u) ? "f" + L : std::string("0u")) << ";\n";
        break;
      }
      case GK_N_GATE: {
        use_scope(level);
        const bool is_or = (op.w2 & GK_G_OR) != 0u, neg_out = (op.w2 & GK_G_NEG_OUT) != 0u;
        std::string e;
        bool any_neg = neg_out;
        for (uint32_t j = 0; j < op.w3; ++j) {
          const uint32_t in = c.pool[op.w1 + j];
          const bool neg = (in >> 31) != 0u;
          any_neg = any_neg || neg;
          const uint32_t slot = in & 0xffffu;
          cur_node.in.emplace_back(slot < cur.size() ? cur[slot] : -1, neg);
          e += (j ? (is_or ? " | " : " & ") : "") + std::string(neg ? "~" : "") + rd(slot);
        }
        cur_node.is_or = is_or;
        cur_node.neg_out = neg_out;
        if (op.w3 == 0) e = is_or ? "0u" : "0xffffffffu", any_neg = true;
        if (neg_out) e = "~(" + e + ")";
        if (any_neg) e = "(" + e + ") & f" + L;
        const uint32_t v = fresh(out);
        body << "  const uint32_t v" << v << " = " << e << ";\n";
        break;
      }
      case GK_N_BCAST: {   // parent-level values -> the rows of the child scope `level`
        use_scope(level);
        const uint32_t P = (uint32_t)c.schema.scopes[level].parent;
        std::vector<std::pair<std::string, uint32_t>> pr;
        for (uint32_t j = 0; j < op.w3; ++j) {
          const uint32_t e = c.pool[op.w1 + j];
          const std::string in = rd(e & 0xffffu);
          pr.emplace_back(in, fresh(e >> 16));
        }
        if (P == 0) {
          for (auto& q : pr) body << "  const uint32_t v" << q.second << " = (0u - (" << q.first << " & 1u)) & f" << L << ";\n";
        } else {
          for (auto& q : pr) body << "  uint32_t v" << q.second << " = 0u;\n";
          body << range_loop_head(level);
          for (auto& q : pr) body << "    if (" << q.first << " & pb) v" << q.second << " |= rm;\n";
          body << "  }\n  }\n";
        }
        break;
      }
      case GK_N_ACC:
      case GK_N_ACC2: {    // EXISTS (at least one / at least two rows of the child scope `level`) per parent row
        use_scope(level);
        const uint32_t P = (uint32_t)c.schema.scopes[level].parent;
        const bool two = kind == GK_N_ACC2;
        std::vector<std::pair<std::string, uint32_t>> pr;
        for (uint32_t j = 0; j < op.w3; ++j) {
          const uint32_t e = c.pool[op.w1 + j];
          const std::string in = rd(e & 0xffffu);
          pr.emplace_back(in, fresh(e >> 16));
        }
        auto test = [&](const std::string& x) { return two ? "(GK_SPEC_POPC(" + x + ") >= 2)" : "((" + x + ") != 0u)"; };
        if (P == 0) {
          for (auto& q : pr) body << "  const uint32_t v" << q.second << " = " << test(q.first) << " ? 1u : 0u;\n";
        } else {
          for (auto& q : pr) body << "  uint32_t v" << q.second << " = 0u;\n";
          body << range_loop_head(level);
          for (auto& q : pr) body << "    if (" << test(q.first + " & rm") << ") v" << q.second << " |= pb;\n";
          body << "  }\n  }\n";
        }
        break;
      }
      case GK_N_MATCH: {
        const uint32_t mid = op.w2;
        match_used.insert(mid);
        // (no text here: the block is evaluated on the object's scope-0 row, and its two bits are exports of that row)
        const uint32_t vm = fresh(out), ve = fresh(op.w1 & 0xffffu);
        matches.push_back({vm, ve, mid});
        break;
      }
      default: break;
    }
    if (kind != GK_N_ATOM && kind != GK_N_ATOMS) finish_node();
  }
};

}  // namespace

SpecSource spec_codegen(const Compiled& c) {
  SpecSource out;
  const uint32_t C = (uint32_t)c.cons_match.size(), W = std::max<uint32_t>(1, (C + 31) / 32);
  const size_t NS = c.schema.scopes.size();
  Gen g(c);
  g.use_scope(0);
  out.tw = gk_tw_layout(c.schema.cols, NS);
  for (const GkOp& op : c.ops) {
    const uint32_t kind = op.w0 & 0xffu;
    if (kind == GK_N_END) break;
    g.op(op);
  }
  std::ostringstream o;
  o << "// generated by spec_codegen.cpp for constraint-set version " << c.version << ": " << C << " constraints, " << c.ops.size() << " netlist ops\n";
  o << "#define GK_SPEC_C " << C << "u\n#define GK_SPEC_W " << W << "\n";
  o << "#ifndef GK_SPEC_THREADS\n#define GK_SPEC_THREADS 256\n#endif\n#ifndef GK_SPEC_MINB\n#define GK_SPEC_MINB 3\n#endif\n";
  o << "#ifndef GK_SPEC_ROWS_THREADS\n#define GK_SPEC_ROWS_THREADS 256\n#endif\n#ifndef GK_SPEC_ROWS_MINB\n#define GK_SPEC_ROWS_MINB 6\n#endif\n";
  o << "#ifndef GK_SPEC_HOST\n#define GK_LD(p) __ldg(p)   /* pool, cbytes and every batch array are global and read-only here */\n#endif\n";
  o << strip_includes(kSpecHdrProgram) << strip_includes(kSpecHdrVmCore);
  o << R"GKSRC(
#ifdef GK_SPEC_X_NOMATCH   /* (measurement only: what the spec.match pre-filter costs) */
#define GK_SPEC_MATCH(MID, B, pool, cbytes, obj) 1
#else
#define GK_SPEC_MATCH(MID, B, pool, cbytes, obj) gk_spec_match_##MID(B, pool, cbytes, obj)
#endif
#ifdef GK_SPEC_HOST
#define GK_SPEC_FN static inline
#define GK_SPEC_LD(p) (*(p))
#define GK_SPEC_POPC(x) __builtin_popcount(x)
#define GK_SPEC_ERR(o, mid, code)                                    \
  {                                                                  \
    const uint32_t sl_ = (*out.errcount)++;                          \
    if (sl_ < out.errcap) {                                          \
      out.errlist[3 * sl_] = (o);                                    \
      out.errlist[3 * sl_ + 1] = (mid);                              \
      out.errlist[3 * sl_ + 2] = (code);                             \
    }                                                                \
  }
struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; };
#define GK_SPEC_CP16(d, s) (*(d) = *(s))
#define GK_SPEC_CP_WAIT()
static inline uint32_t gk_spec_funnel(uint32_t lo, uint32_t hi, uint32_t sh) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (sh & 31u)); }
#define GK_SPEC_FUNNEL(lo, hi, sh) gk_spec_funnel(lo, hi, sh)
#else
#define GK_SPEC_FN __device__ __forceinline__
#define GK_SPEC_LD(p) __ldg(p)      /* every array of a resident batch is read-only while it is evaluated */
#define GK_SPEC_POPC(x) __popc(x)
/* one 16-byte global -> shared copy in flight (export planes and their regions are 16-byte aligned); GK_SPEC_CP_WAIT() lands this thread's */
#define GK_SPEC_CP16(d, s) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"((uint32_t)__cvta_generic_to_shared(d)), "l"(s) : "memory")
#define GK_SPEC_CP_WAIT() asm volatile("cp.async.wait_all;\n" ::: "memory")
/* bits [sh, sh + 32) of the 64-bit word hi:lo */
#define GK_SPEC_FUNNEL(lo, hi, sh) __funnelshift_r(lo, hi, sh)
__device__ __forceinline__ uint32_t gk_tr_step(uint32_t x, uint32_t lane, uint32_t j, uint32_t m) {
  const uint32_t y = __shfl_xor_sync(0xffffffffu, x, j);
  return (lane & j) ? ((x & ~m) | ((y & ~m) >> j)) : ((x & m) | ((y & m) << j));
}
// 32 x 32 bit transpose across the warp: lane i gives row i and receives column i
__device__ __forceinline__ uint32_t gk_tr32(uint32_t x, uint32_t lane) {
  x = gk_tr_step(x, lane, 16u, 0x0000ffffu);
  x = gk_tr_step(x, lane, 8u, 0x00ff00ffu);
  x = gk_tr_step(x, lane, 4u, 0x0f0f0f0fu);
  x = gk_tr_step(x, lane, 2u, 0x33333333u);
  x = gk_tr_step(x, lane, 1u, 0x55555555u);
  return x;
}
#define GK_SPEC_ERR(o, mid, code)                                    \
  {                                                                  \
    const uint32_t sl_ = atomicAdd(out.errcount, 1u);                \
    if (sl_ < out.errcap) {                                          \
      out.errlist[3 * sl_] = (o);                                    \
      out.errlist[3 * sl_ + 1] = (mid);                              \
      out.errlist[3 * sl_ + 2] = (code);                             \
    }                                                                \
  }
#endif
)GKSRC";
  // ---- the spec.match pre-filter of every block the netlist uses, written out (emit_match below): criteria the block does not have are
  // not emitted, kind / group / label ids and the bytes of the wildcard patterns are immediates, the labels are walked once per selector.
  // GK_SPEC_MATCHGEN=0: the block as a GkMatch literal through the shared gk_match() (vm_core.h) instead -- the form the first
  // generated kernels had; the pool / cbytes reads of that form are what the written-out one removes.
  const bool matchgen = !(getenv("GK_SPEC_MATCHGEN") && atoi(getenv("GK_SPEC_MATCHGEN")) == 0);
  for (uint32_t mid : g.match_used) {
    const GkMatch& m = c.match[mid];
    if (matchgen && emit_match(o, c, mid)) continue;
    o << "#define M" << mid << " (GkMatch{" << hx(m.flags) << ", " << m.kinds_off << "u, " << m.kinds_n << "u, " << m.ns_off << "u, " << m.ns_n << "u, " << m.exns_off << "u, "
      << m.exns_n << "u, " << m.lsel_off << "u, " << m.lsel_n << "u, " << m.nssel_off << "u, " << m.nssel_n << "u, " << m.name_mode << "u, " << m.name_boff << "u, "
      << m.name_len << "u, 0u, 0u})\n";
    o << "GK_SPEC_FN int gk_spec_match_" << mid << "(const GkBatch& B, const uint32_t* __restrict__ pool, const uint8_t* __restrict__ cbytes, const uint32_t obj) {\n"
      << "  return gk_match(B, pool, cbytes, M" << mid << ", obj);\n}\n";
  }
  // ---- emission order of the constraints: by template kind, then by the scopes their cones touch
  std::vector<std::vector<uint32_t>> cone_atoms(g.nvar);   // variable -> atoms in its cone (memoised)
  std::vector<uint8_t> cone_done(g.nvar, 0);
  std::function<const std::vector<uint32_t>&(uint32_t)> cone = [&](uint32_t v) -> const std::vector<uint32_t>& {
    if (cone_done[v]) return cone_atoms[v];
    cone_done[v] = 1;
    std::set<uint32_t> acc;
    if (g.atom_of[v] >= 0) {
      acc.insert((uint32_t)g.atom_of[v]);
    } else if (g.producer[v] >= 0) {
      for (uint32_t d : g.nodes[(size_t)g.producer[v]].deps) {
        const std::vector<uint32_t>& sub = cone(d);
        acc.insert(sub.begin(), sub.end());
      }
    }
    cone_atoms[v].assign(acc.begin(), acc.end());
    return cone_atoms[v];
  };
  auto var_of = [&](uint32_t slot) -> int { return slot < g.cur.size() ? g.cur[slot] : -1; };
  struct Ord {
    std::string kind;
    std::vector<int> sig;
    uint32_t cix;
    bool operator<(const Ord& x) const { return std::tie(kind, sig, cix) < std::tie(x.kind, x.sig, x.cix); }
  };
  std::vector<Ord> order;
  for (uint32_t cix = 0; cix < C; ++cix) {
    const GkOutEnt& oe = c.outs[cix];
    Ord e;
    e.cix = cix;
    e.kind = cix < c.order.size() && c.order[cix] ? c.order[cix]->kind : std::string();
    if (!(oe.flags & 3u) && var_of(oe.prog_slot) >= 0) {
      std::set<int> sc;
      for (uint32_t ai : cone((uint32_t)var_of(oe.prog_slot))) sc.insert((int)g.atoms[ai].scope);
      e.sig.assign(sc.rbegin(), sc.rend());
    }
    order.push_back(std::move(e));
  }
  std::sort(order.begin(), order.end());
  // ---- atom groups: ONE row loop per scope computes every atom of that scope.  A loop per (scope, template kind) measured no
  // better: every extra loop is one more exposed memory latency per object.
  std::map<uint32_t, int> group_ix;   // scope -> row loop
  std::vector<std::vector<uint32_t>> groups;
  std::vector<uint32_t> gscope;       // row loop -> its scope
  auto add_group = [&](uint32_t s) {
    auto it = group_ix.find(s);
    if (it != group_ix.end()) return it->second;
    group_ix.emplace(s, (int)groups.size());
    groups.emplace_back();
    gscope.push_back(s);
    return (int)groups.size() - 1;
  };
  for (const Ord& e : order) {
    const GkOutEnt& oe = c.outs[e.cix];
    if ((oe.flags & 3u) || var_of(oe.prog_slot) < 0) continue;
    for (uint32_t ai : cone((uint32_t)var_of(oe.prog_slot))) {
      Gen::AtomRec& r = g.atoms[ai];
      if (r.group >= 0) continue;
      r.group = add_group(r.scope);
      groups[(size_t)r.group].push_back(ai);
    }
  }
  if (!g.matches.empty()) add_group(0);   // the match blocks are evaluated on the scope-0 row, with or without atoms there
  auto parent_of = [&](uint32_t s) { return (uint32_t)c.schema.scopes[s].parent; };
  // ---- row-local values and exports.  A variable of scope L is ROW-LOCAL when it is a function of one row of L alone: an atom of L,
  // or a gate of L whose inputs are row-local values and constants (and at least one of the former).  Phase 1 has every atom of a
  // row in a register, so it evaluates those gates there and stages only the EXPORTS: the row-local values that something else
  // reads -- an EXISTS, a broadcast, a gate with an input that is not row-local, a constraint's result.  An export that only
  // object-level EXISTS read is in ANY form (phase 2 tests the object's window of its plane against 0); every other export is in MASK
  // form (phase 2 takes the window as the per-row mask).  Constants, and gates of nothing but constants,
  // are literals in phase 1 and stay the nodes they were in phase 2.
  enum : uint8_t { kNotExported = 0, kAny = 1, kMask = 2 };
  std::vector<int> local(g.nvar, -1);      // variable -> the scope it is row-local in
  std::vector<int8_t> konst(g.nvar, -1);   // variable -> its value in a row that exists, when it is a constant
  std::vector<uint8_t> is_match(g.nvar, 0);   // the match / error bit of a spec.match block: row-local in scope 0
  for (const Gen::MatchRec& m : g.matches) is_match[m.vm] = is_match[m.ve] = 1;
  for (uint32_t v = 0; v < g.nvar; ++v) {
    if (g.atom_of[v] >= 0) {
      local[v] = (int)g.atoms[(size_t)g.atom_of[v]].scope;
      continue;
    }
    if (is_match[v]) {
      local[v] = 0;
      continue;
    }
    if (g.producer[v] < 0) continue;
    const SpecNode& n = g.nodes[(size_t)g.producer[v]];
    if (n.kind == GK_N_CONST) konst[v] = n.one ? 1 : 0;
    if (n.kind != GK_N_GATE) continue;
    bool all = true, some = false, val = !n.is_or;
    for (const auto& in : n.in) {
      const bool k = in.first < 0 || konst[(size_t)in.first] >= 0, l = !k && local[(size_t)in.first] == (int)n.level;
      all = all && (k || l);
      some = some || l;
      if (k) {
        const bool x = (in.first >= 0 && konst[(size_t)in.first] == 1) != in.second;
        val = n.is_or ? (val || x) : (val && x);
      }
    }
    if (all && some) local[v] = (int)n.level;
    else if (all) konst[v] = (val != n.neg_out) ? 1 : 0;
  }
  auto folded = [&](uint32_t v) { return local[v] >= 0 && g.atom_of[v] < 0 && !is_match[v]; };   // a gate phase 1 evaluates
  std::vector<uint8_t> form(g.nvar, kNotExported), live(g.nvar, 0);
  {
    std::vector<uint32_t> todo;
    auto reach = [&](uint32_t v) {
      if (!live[v]) live[v] = 1, todo.push_back(v);
    };
    for (uint32_t cix = 0; cix < C; ++cix) {
      const GkOutEnt& oe = c.outs[cix];
      for (int v : {(oe.flags & 3u) ? -1 : var_of(oe.prog_slot), var_of(oe.match_slot), var_of(oe.err_slot)}) {
        if (v < 0) continue;
        reach((uint32_t)v);
        if (local[(size_t)v] >= 0) form[(size_t)v] = kMask;
      }
    }
    while (!todo.empty()) {
      const uint32_t v = todo.back();
      todo.pop_back();
      if (g.producer[v] < 0) continue;
      const SpecNode& n = g.nodes[(size_t)g.producer[v]];
      // (GK_N_ACC2 exists only in the audit's ambiguity netlist, which is interpreted; the generator is handed the decision netlist.
      // Were one to reach it, its input would be exported in mask form, which the count needs.)
      const bool any = n.kind == GK_N_ACC && parent_of(n.level) == 0u;
      for (uint32_t d : n.deps) {
        reach(d);
        if (local[d] >= 0 && !folded(v)) form[d] = std::max<uint8_t>(form[d], any ? kAny : kMask);
      }
    }
  }
  // per row loop: its exports (any form first), and the gates phase 1 evaluates for them, in netlist order
  std::vector<std::vector<uint32_t>> exports(groups.size()), gates(groups.size());
  std::vector<uint32_t> nany(groups.size(), 0);
  for (uint8_t f : {kAny, kMask})
    for (uint32_t v = 0; v < g.nvar; ++v) {
      if (!live[v] || form[v] != f) continue;
      const size_t gi = (size_t)group_ix.at((uint32_t)local[v]);
      exports[gi].push_back(v);
      if (f == kAny) ++nany[gi];
    }
  for (uint32_t v = 0; v < g.nvar; ++v)
    if (live[v] && folded(v)) gates[(size_t)group_ix.at((uint32_t)local[v])].push_back(v);
  // ---- the rows, gk_spec_row_<g>() run by gk_spec_rows_kernel: one thread per row of a row loop's scope over the whole batch evaluates
  // the loop's atoms and row-local gates (on a scope-0 row also the spec.match blocks, listing their errors) and returns the loop's
  // exports as packed bits (ceil(exports / 32) words; bit k of word k / 32 = the loop's k-th export).  The kernel stores them as BIT
  // PLANES: a warp is 32 consecutive rows of one scope, aligned to 32, so a 32 x 32 bit transpose across the warp turns the warp's
  // words into plane words, bit j = row 32 * blk + j.  Row loop g's planes are P<g> = its exports rounded up to 4 (the padding planes are 0), and
  // word (blk, k) lies at X<g> + blk * P<g> + k: a block's planes are one 16-byte aligned run.  One guard block past the last keeps
  // every window's high word (below) in bounds.  The loops' planes lie back to back in one scratch buffer, in row-loop order
  // (SpecSource::export_bytes).
  // ---- the tile, gk_spec_stage(): the CTA copies the tile's blocks of every row loop's planes (16-byte copies) and every used nested
  // scope's CSR offsets (tile-relative) into shared memory.  The per-tile layout follows from the rows of every scope in the tile
  // (tile_lo): a header of region offsets and of each row loop's first bit (b<s> & 31: the tile's first row of the scope within its
  // block), then the regions.  SpecSource::stage lists them so the launch can size the area.
  std::vector<uint32_t> nested;   // used nested scopes: their offsets are staged
  for (size_t s = 1; s < NS; ++s)
    if (g.scope_used[s]) nested.push_back((uint32_t)s);
  const uint32_t NG = (uint32_t)groups.size(), NR = NG + (uint32_t)nested.size(), data0 = (NR + NG + 3u) & ~3u;
  auto group_scope = [&](size_t gi) { return gscope[gi]; };
  auto group_words = [&](size_t gi) { return (uint32_t)((exports[gi].size() + 31) / 32); };
  auto group_planes = [&](size_t gi) { return (uint32_t)((exports[gi].size() + 3) / 4 * 4); };
  for (size_t gi = 0; gi < NG; ++gi) {
    out.stage.push_back({group_scope(gi), group_planes(gi)});
    if (!groups[gi].empty())
      out.fold.push_back({group_scope(gi), (uint32_t)groups[gi].size(), (uint32_t)gates[gi].size(), nany[gi], (uint32_t)exports[gi].size() - nany[gi], group_words(gi)});
  }
  for (uint32_t s : nested) out.stage.push_back({parent_of(s), 0u});
  out.stage_hdr = data0;
  out.ngroups = NG;
  out.nested = nested;
  // the per-tile layout: b<s> / c<s> = first row / rows of scope s in the tile, R<g> = region offsets.  Row loop g's region is
  // ceil(c / 32) + 2 blocks, at least ((b & 31) + c) / 32 + 2: the ceil(((b & 31) + c) / 32) + 1 the copy fills (the tile's rows and
  // the block after them) and, when (b & 31) + c is a multiple of 32, one more that only the window of an object with no rows there
  // reads (masked to 0).  Then, at word QA, the tile's run of the offset image (SpecSource::image_stride): nested scope s's offsets
  // at 16-bit value I<s> of the run, c<parent> + 1 of them; NI values in all, padded to 16 bytes.
  std::ostringstream tiles, img;
  tiles << "  const uint32_t b0 = GK_SPEC_LD(tlo), c0 = GK_SPEC_LD(thi) - b0;\n  (void)b0; (void)c0;\n";
  for (uint32_t s : nested)
    tiles << "  const uint32_t b" << s << " = GK_SPEC_LD(tlo + " << s << "), c" << s << " = GK_SPEC_LD(thi + " << s << ") - b" << s << ";\n  (void)c" << s << ";\n";
  img << "  uint32_t NI = 0u;\n";
  for (uint32_t s : nested) img << "  const uint32_t I" << s << " = NI;\n  NI += c" << parent_of(s) << " + 1u;\n";
  std::ostringstream lay;
  lay << tiles.str() << "  uint32_t at = " << data0 << "u;\n";
  for (size_t gi = 0; gi < NG; ++gi) {
    const std::string s = std::to_string(group_scope(gi));
    lay << "  const uint32_t R" << gi << " = at;\n";
    if (group_planes(gi)) lay << "  at += ((c" << s << " + 31u) / 32u + 2u) * " << group_planes(gi) << "u;\n";
  }
  lay << "  const uint32_t QA = at;\n" << img.str() << "  at += (NI + 7u) / 8u * 4u;\n";
  // X<g> = the word offset of row loop g's planes in the scratch buffer; X<NG> = the buffer's words
  std::ostringstream xbase;
  // (32-bit words: the planes are under one bit per row per export, and a scope's rows fit 32 bits)
  xbase << "  const uint32_t X0 = 0u;\n";
  for (size_t gi = 0; gi < NG; ++gi) {
    const uint32_t s = group_scope(gi);
    xbase << "  const uint32_t X" << gi + 1 << " = X" << gi << " + ((" << (s ? "scopes[" + std::to_string(s) + "].rows" : std::string("B.n")) << " + 31u) / 32u + 1u) * "
          << group_planes(gi) << "u;\n";
  }
  xbase << "  (void)scopes;";
  for (size_t gi = 0; gi <= NG; ++gi) xbase << " (void)X" << gi << ";";
  xbase << "\n";
  std::map<uint32_t, std::vector<const Gen::MatchRec*>> match_at;   // (only the blocks whose bits something reads)
  for (const Gen::MatchRec& m : g.matches)
    if (live[m.vm] || live[m.ve]) match_at[0].push_back(&m);
  for (size_t gi = 0; gi < NG; ++gi) {
    const std::vector<uint32_t>& members = groups[gi];
    const uint32_t s = group_scope(gi), AW = group_words(gi);
    std::map<uint32_t, uint32_t> need;
    for (uint32_t ai : members)
      for (auto& kv : g.atoms[ai].need) need[kv.first] |= kv.second;
    o << "\n// atoms, row-local gates" << (s == 0 && !match_at[0].empty() ? ", spec.match blocks" : "") << " and exports of one row of scope " << s << " (row loop " << gi << ")\n";
    o << "GK_SPEC_FN void gk_spec_row_" << gi << "(const GkBatch& B, const GkColumn* cols, const uint32_t* __restrict__ pool, const uint8_t* __restrict__ cbytes, const GkOut& out,\n"
      << "                              const size_t row, uint32_t* __restrict__ a) {\n  (void)B; (void)cols; (void)pool; (void)cbytes; (void)out; (void)a;\n";
    // the row's type words, when its scope has them (gk_tw_layout) and an atom reads a type: one aligned 4- or 8-byte load, or one
    // 16-byte load per 4 words, and every tK a nibble of them instead of a byte load of its own
    const uint32_t TW = s < out.tw.words.size() ? out.tw.words[s] : 0u;
    auto packed = [&](uint32_t ci) { return TW && ci < out.tw.nibble.size() && out.tw.nibble[ci] != GK_NONE && (uint32_t)c.schema.cols[ci].scope == s; };
    bool any_packed = false;
    for (auto& kv : need) any_packed = any_packed || ((kv.second & GK_ENC_VT) && packed(kv.first));
    if (any_packed) {
      o << "  const uint32_t* __restrict__ tws = B.tw[" << s << "];\n";
      if (TW == 1) {
        o << "  const uint32_t tw0 = GK_SPEC_LD(tws + row);\n";
      } else if (TW == 2) {
        o << "  const uint2 twv = GK_SPEC_LD(reinterpret_cast<const uint2*>(tws) + row);\n  const uint32_t tw0 = twv.x, tw1 = twv.y;\n";
      } else {
        for (uint32_t j = 0; j < TW / 4; ++j) {
          const std::string J = std::to_string(j), q = std::to_string(4 * j);
          o << "  const uint4 twv" << J << " = GK_SPEC_LD(reinterpret_cast<const uint4*>(tws) + row * " << TW / 4 << "u + " << j << "u);\n";
          o << "  const uint32_t tw" << q << " = twv" << J << ".x, tw" << 4 * j + 1 << " = twv" << J << ".y, tw" << 4 * j + 2 << " = twv" << J << ".z, tw" << 4 * j + 3 << " = twv"
            << J << ".w;\n";
        }
      }
      for (uint32_t w = 0; w < TW; ++w) o << (w ? " " : "  ") << "(void)tw" << w << ";";
      o << "\n";
    }
    for (auto& kv : need) {
      const uint32_t ci = kv.first, enc = kv.second;
      const std::string K = std::to_string(ci);
      if ((enc & GK_ENC_VT) && packed(ci)) {
        const uint32_t k = out.tw.nibble[ci];
        o << "  const uint32_t t" << K << " = (tw" << k / 8 << " >> " << 4 * (k % 8) << "u) & 15u;\n";
      } else if (enc & GK_ENC_VT) {
        o << "  const uint32_t t" << K << " = GK_SPEC_LD(cols[" << K << "].vt + row);\n";
      }
      if (enc & GK_ENC_SID) o << "  const uint32_t i" << K << " = GK_SPEC_LD(cols[" << K << "].sid + row);\n";
      if (enc & GK_ENC_NUM) o << "  const long long n" << K << " = GK_SPEC_LD(reinterpret_cast<const long long*>(cols[" << K << "].num) + row);\n";
      if (enc & GK_ENC_HEAD)
        o << "  const uint4* __restrict__ ph" << K << " = reinterpret_cast<const uint4*>(cols[" << K << "].head);\n  const uint4 h" << K << "a = GK_SPEC_LD(ph" << K
          << " + 2 * row), h" << K << "b = GK_SPEC_LD(ph" << K << " + 2 * row + 1);\n";
    }
    if (s == 0 && !match_at[0].empty()) {
      // a skipped object (review-level error) evaluates no block and lists no error: both of its bits are 0
      o << "  const uint32_t obj = (uint32_t)row;\n  const bool skip = (GK_SPEC_LD(B.flags + obj) & GK_F_SKIP) != 0u;\n";
      for (const Gen::MatchRec* m : match_at[0]) {
        const std::string M = std::to_string(m->vm);
        o << "  const int m" << M << " = skip ? 0 : GK_SPEC_MATCH(" << m->mid << ", B, pool, cbytes, obj);\n";
        o << "  if (m" << M << " < 0) GK_SPEC_ERR(obj, " << m->mid << "u, (uint32_t)(-m" << M << "));\n";
        o << "  const bool v" << M << " = m" << M << " > 0, v" << m->ve << " = m" << M << " < 0;\n  (void)v" << M << "; (void)v" << m->ve << ";\n";
      }
    }
    for (uint32_t ai : members) o << "  const bool v" << g.atoms[ai].var << " = " << g.atoms[ai].expr << ";\n";
    for (uint32_t v : gates[gi]) {
      const SpecNode& n = g.nodes[(size_t)g.producer[v]];
      std::string e;
      for (const auto& in : n.in) {
        const bool k = in.first < 0 || konst[(size_t)in.first] >= 0;
        const std::string x = k ? ((in.first >= 0 && konst[(size_t)in.first] == 1) ? "true" : "false") : "v" + std::to_string(in.first);
        e += (e.empty() ? "" : n.is_or ? " | " : " & ") + std::string(in.second ? "!" : "") + x;
      }
      o << "  const bool v" << v << " = " << (n.neg_out ? "!(" + e + ")" : e) << ";   // row-local gate\n";
    }
    o << "  uint32_t";
    for (uint32_t w = 0; w < AW; ++w) o << (w ? ", a" : " a") << w << " = 0u";
    o << ";\n";
    for (size_t m = 0; m < exports[gi].size(); ++m) o << "  if (v" << exports[gi][m] << ") a" << m / 32 << " |= " << hx(1u << (m % 32)) << ";\n";
    for (uint32_t w = 0; w < AW; ++w) o << "  a[" << w << "] = a" << w << ";\n";
    o << "}\n";
  }
  o << "\n#ifdef GK_SPEC_HOST\n";
  o << "static uint32_t gk_spec_stage_words(const uint32_t* tlo, const uint32_t* thi) {\n" << lay.str() << "  return at;\n}\n";
  // SpecSource::image_stride and image_fits, over the tiles the host build makes
  o << "static uint32_t gk_spec_image_stride(const uint32_t* cap) {\n  uint32_t v = 0u;\n";
  for (uint32_t s : nested) o << "  v += cap[" << parent_of(s) << "] + 1u;\n";
  o << "  return (v + 7u) / 8u * 8u;\n}\n";
  o << "static bool gk_spec_image_fits(const uint32_t* cap) {\n  (void)cap;\n  return true";
  for (uint32_t s : nested) o << " && cap[" << s << "] <= 0xffffu";
  o << ";\n}\n";
  o << "// the parent of a nested scope whose offsets are staged, ~0u for any other scope\nstatic uint32_t gk_spec_parent(uint32_t s) {\n  switch (s) {\n";
  for (uint32_t s : nested) o << "    case " << s << "u: return " << parent_of(s) << "u;\n";
  o << "    default: return 0xffffffffu;\n  }\n}\n";
  o << "static void gk_spec_tile_rows(const GkScope* scopes, uint32_t* tlo, uint32_t* thi) {\n";
  for (uint32_t s : nested)
    o << "  tlo[" << s << "] = scopes[" << s << "].off[tlo[" << parent_of(s) << "]];\n  thi[" << s << "] = scopes[" << s << "].off[thi[" << parent_of(s) << "]];\n";
  o << "}\n";
  o << "static size_t gk_spec_export_words(const GkBatch& B) {\n  const GkScope* scopes = B.scopes;\n" << xbase.str() << "  return X" << NG << ";\n}\n";
  // GK_SPEC_TRACE: "[spec planes] loop <g>: scope <s>, <exports> exports, <rows> rows; ...; <words> export words" (once per batch)
  o << "#include <cstdio>\n#include <vector>\nstatic void gk_spec_trace_planes(const GkBatch& B) {\n  fprintf(stderr, \"[spec planes]\");\n";
  for (size_t gi = 0; gi < NG; ++gi) {
    const uint32_t s = group_scope(gi);
    o << "  fprintf(stderr, \" loop " << gi << ": scope " << s << ", " << exports[gi].size() << " exports, %u rows;\", " << (s ? "B.scopes[" + std::to_string(s) + "].rows" : std::string("B.n")) << ");\n";
  }
  o << "  fprintf(stderr, \" %zu export words\\n\", gk_spec_export_words(B));\n";
  // "[spec types] scope <s>: <vt columns> vt columns in <W> words, <rows> rows; ...; <bytes> type-word bytes" (the scopes with type words)
  o << "  size_t twb = 0;\n  fprintf(stderr, \"[spec types]\");\n";
  for (size_t s = 0; s < NS; ++s) {
    if (!out.tw.words[s]) continue;
    const std::string R = s ? "B.scopes[" + std::to_string(s) + "].rows" : std::string("B.n");
    o << "  fprintf(stderr, \" scope " << s << ": " << out.tw.vtcols[s].size() << " vt columns in " << out.tw.words[s] << " words, %u rows;\", " << R << ");\n  twb += (size_t)"
      << R << " * " << out.tw.words[s] * 4 << "u;\n";
  }
  o << "  fprintf(stderr, \" %zu type-word bytes\\n\", twb);\n}\n";
  // the type words of the whole batch, as the backend's pack pass makes them (gk_tw_pack_row over the same layout), into `words`;
  // returns the per-scope pointer table for GkBatch::tw
  o << "static const uint32_t* const* gk_spec_host_types(const GkBatch& B, std::vector<std::vector<uint32_t>>& words, std::vector<const uint32_t*>& ptrs) {\n"
    << "  words.assign(" << NS << "u, std::vector<uint32_t>());\n  ptrs.assign(" << NS << "u, nullptr);\n";
  for (size_t s = 0; s < NS; ++s) {
    if (!out.tw.words[s]) continue;
    const std::vector<uint32_t>& vc = out.tw.vtcols[s];
    o << "  {\n    static const uint32_t vc[" << vc.size() << "] = {";
    for (size_t k = 0; k < vc.size(); ++k) o << (k ? ", " : "") << vc[k] << "u";
    o << "};\n    const uint32_t rows = " << (s ? "B.scopes[" + std::to_string(s) + "].rows" : std::string("B.n")) << ";\n    words[" << s << "].assign((size_t)rows * "
      << out.tw.words[s] << "u + 1u, 0xdeadbeefu);\n    for (size_t row = 0; row < rows; ++row) gk_tw_pack_row(B.cols, vc, " << vc.size() << "u, " << out.tw.words[s]
      << "u, row, words[" << s << "].data());\n    ptrs[" << s << "] = words[" << s << "].data();\n  }\n";
  }
  o << "  return ptrs.data();\n}\n";
  // (the rows of the tile [tlo, thi) only, and of those only their own bits of the plane words: a copy, or a window, that reads a row
  // outside them finds the caller's poison)
  o << "static void gk_spec_host_rows(const GkKParams* p, const uint32_t* tlo, const uint32_t* thi, uint32_t* xs) {\n  const GkBatch& B = p->batch;\n  const GkScope* scopes = B.scopes;\n"
    << xbase.str();
  for (size_t gi = 0; gi < NG; ++gi) {
    const uint32_t s = group_scope(gi);
    o << "  for (size_t row = tlo[" << s << "]; row < thi[" << s << "]; ++row) {\n    uint32_t a[" << std::max<uint32_t>(1, group_words(gi)) << "] = {0u};\n    gk_spec_row_" << gi
      << "(B, B.cols, p->prog.pool, p->prog.cbytes, p->out, row, a);\n    uint32_t* x = xs + X" << gi << " + (row >> 5) * " << group_planes(gi) << "u;\n    const uint32_t r = 1u << (row & 31u);\n"
      << "    for (uint32_t k = 0; k < " << exports[gi].size() << "u; ++k) x[k] = ((a[k >> 5] >> (k & 31u)) & 1u) ? (x[k] | r) : (x[k] & ~r);\n    (void)x; (void)r;\n  }\n";
  }
  o << "}\n#else\n";
  // one thread per row; blocks [first, first + ceil(rows / threads)) of the grid are row loop g's, so a block never mixes scopes and
  // a warp is one block of 32 rows.  Every lane reaches the transpose (a row past the scope's end contributes zeros); a warp past the
  // scope's last block stores nothing.  The 32 x 32 transpose of word i (five shuffles, fewer instructions than a ballot per export
  // from about eight exports up) leaves plane word 32 i + j of the block in lane j.
  o << "static_assert(GK_SPEC_ROWS_THREADS % 32 == 0, \"a warp of gk_spec_rows_kernel is one block of 32 rows\");\n";
  o << "extern \"C\" __global__ void __launch_bounds__(GK_SPEC_ROWS_THREADS, GK_SPEC_ROWS_MINB) gk_spec_rows_kernel(const __grid_constant__ GkKParams p, uint32_t* __restrict__ xs) {\n"
    << "  const GkBatch& B = p.batch;\n  const GkScope* scopes = B.scopes;\n  const uint32_t lane = threadIdx.x & 31u;\n  (void)lane;\n"
    << xbase.str() << "  uint32_t blk = blockIdx.x;\n";
  // the block's row loop runs its row function and names its planes; the transpose and the store are one tail for every loop
  uint32_t AWM = 1;
  for (size_t gi = 0; gi < NG; ++gi) AWM = std::max(AWM, group_words(gi));
  o << "  uint32_t nr = 0u, row = 0u, np = 0u";
  for (uint32_t i = 0; i < AWM; ++i) o << ", a" << i << " = 0u";
  o << ";\n  uint32_t xo = 0u;\n  do {\n";
  for (size_t gi = 0; gi < NG; ++gi) {
    const uint32_t s = group_scope(gi);
    o << "    {\n      nr = " << (s ? "scopes[" + std::to_string(s) + "].rows" : std::string("B.n")) << ";\n      const uint32_t nb = (nr + GK_SPEC_ROWS_THREADS - 1u) / GK_SPEC_ROWS_THREADS;\n"
      << "      if (blk < nb) {\n        row = blk * GK_SPEC_ROWS_THREADS + threadIdx.x;\n        if (row < nr) {\n          uint32_t w[" << std::max<uint32_t>(1, group_words(gi)) << "];\n          gk_spec_row_" << gi
      << "(B, B.cols, p.prog.pool, p.prog.cbytes, p.out, row, w);\n";
    for (uint32_t i = 0; i < group_words(gi); ++i) o << "          a" << i << " = w[" << i << "];\n";
    o << "        }\n        np = " << group_planes(gi) << "u;\n        xo = X" << gi << ";\n        break;\n      }\n      blk -= nb;\n    }\n";
  }
  o << "    return;\n  } while (0);\n";
  o << "  if ((row & ~31u) < nr) {\n    uint32_t* __restrict__ x = xs + xo + (size_t)(row >> 5) * np;\n";
  for (uint32_t i = 0; i < AWM; ++i) {
    o << "    " << (i ? "if (np > " + std::to_string(32 * i) + "u) " : std::string()) << "{\n      const uint32_t w = gk_tr32(a" << i << ", lane);\n      if (" << 32 * i
      << "u + lane < np) x[" << 32 * i << "u + lane] = w;\n    }\n";
  }
  o << "  }\n";
  o << "}\n#endif\n";
  // the copy: every 16-byte copy of the tile's plane blocks and of its run of the offset image (`img`) in flight together (cp.async),
  // one wait.  The header's offsets entries are 16-bit indices from stg.
  o << "GK_SPEC_FN void gk_spec_stage(const GkBatch& B, const GkScope* scopes, const uint32_t* __restrict__ xs, const uint16_t* __restrict__ img, const uint32_t* tlo,\n"
       "                              const uint32_t* thi, uint32_t* stg, const uint32_t tid, const uint32_t nthr) {\n  (void)B; (void)xs; (void)img;\n";
  o << lay.str() << xbase.str();
  o << "  if (tid == 0u) {\n";
  for (size_t gi = 0; gi < NG; ++gi) o << "    stg[" << gi << "] = R" << gi << ";\n";
  for (size_t j = 0; j < nested.size(); ++j) o << "    stg[" << NG + j << "] = 2u * QA + I" << nested[j] << ";\n";
  for (size_t gi = 0; gi < NG; ++gi) o << "    stg[" << NR + gi << "] = b" << group_scope(gi) << " & 31u;\n";
  o << "  }\n";
  for (size_t gi = 0; gi < NG; ++gi) {
    const uint32_t s = group_scope(gi), P = group_planes(gi);
    if (!P) continue;
    o << "  {   // planes of scope " << s << " (row loop " << gi << "): blocks b / 32 to ceil((b + c) / 32), the last for the windows' high words\n"
      << "    const uint4* __restrict__ src = reinterpret_cast<const uint4*>(xs + X" << gi << " + (size_t)(b" << s << " >> 5) * " << P << "u);\n"
      << "    uint4* dst = reinterpret_cast<uint4*>(stg + R" << gi << ");\n"
      << "    const uint32_t n = (((b" << s << " & 31u) + c" << s << " + 31u) / 32u + 1u) * " << P / 4 << "u;\n"
      << "    for (uint32_t i = tid; i < n; i += nthr) GK_SPEC_CP16(dst + i, src + i);\n  }\n";
  }
  if (!nested.empty())
    o << "  {   // the offsets: the tile's run of the offset image, verbatim\n    const uint4* __restrict__ src = reinterpret_cast<const uint4*>(img);\n"
      << "    uint4* dst = reinterpret_cast<uint4*>(stg + QA);\n    const uint32_t n = (NI + 7u) / 8u;\n"
      << "    for (uint32_t i = tid; i < n; i += nthr) GK_SPEC_CP16(dst + i, src + i);\n  }\n";
  o << "  GK_SPEC_CP_WAIT();\n}\n";
  // ---- the offset image of one tile (gk_spec_plan_kernel, gk_spec_host_plan): from the batch's CSR offsets, tile-relative, in the
  // layout gk_spec_stage() copies.  The offsets of sibling scopes are read at the same parent rows: one item writes all of a parent's
  // children.
  o << "GK_SPEC_FN void gk_spec_offsets(const GkScope* __restrict__ scopes, const uint32_t* tlo, const uint32_t* thi, uint16_t* img, const uint32_t tid,\n"
       "                                const uint32_t nthr) {\n  (void)scopes; (void)img; (void)tid; (void)nthr;\n";
  o << tiles.str() << img.str() << "  (void)NI;\n";
  std::map<uint32_t, std::vector<uint32_t>> children;
  for (uint32_t s : nested) children[parent_of(s)].push_back(s);
  for (auto& ch : children) {
    const uint32_t P = ch.first;
    o << "  for (uint32_t k = tid; k <= c" << P << "; k += nthr) {   // offsets of the children of scope " << P << "\n";
    for (uint32_t s : ch.second) o << "    img[I" << s << " + k] = (uint16_t)(GK_SPEC_LD(scopes[" << s << "].off + b" << P << " + k) - b" << s << ");\n";
    o << "  }\n";
  }
  o << "}\n";
  // ---- which objects are WIDE: more rows in some used nested scope than a mask register holds.  The object's row range in scope s,
  // [lo<s>, hi<s>), from its parent's through s's CSR offsets, read by `off(s, row)`.  A scope with more rows than a mask holds
  // counts as EMPTY from there on and raises `big`: no branch.  gk_spec_object() reads the tile's staged offsets, gk_spec_wide()
  // (the hand-over plan) the batch's own: one text, so that the two decide every object alike.
  auto scope_extent = [&](uint32_t s, const std::function<std::string(const std::string&)>& off) {
    const uint32_t P = parent_of(s);
    o << "  const uint32_t lo" << s << " = " << off("lo" + std::to_string(P)) << ", r" << s << " = " << off("hi" + std::to_string(P)) << " - lo" << s << ";\n";
    o << "  const uint32_t n" << s << " = r" << s << " > GK_SPEC_MASK_ROWS ? 0u : r" << s << ", hi" << s << " = lo" << s << " + n" << s << ";\n";
    o << "  big = big || r" << s << " > GK_SPEC_MASK_ROWS;\n";
  };
  o << "\n#define GK_SPEC_MASK_ROWS 32u\n";
  o << "GK_SPEC_FN bool gk_spec_wide(const GkScope* __restrict__ scopes, const uint32_t obj) {\n";
  o << "  const uint32_t lo0 = obj, hi0 = obj + 1u;\n  (void)scopes; (void)lo0; (void)hi0;\n  bool big = false;\n";
  for (uint32_t s : nested) {
    scope_extent(s, [&](const std::string& row) { return "GK_SPEC_LD(scopes[" + std::to_string(s) + "].off + " + row + ")"; });
    o << "  (void)hi" << s << ";\n";
  }
  o << "  return big;\n}\n";
  o << "// the hand-over rule per tile: a tile with more wide objects than this goes to the interpreter whole (program.h)\n";
  o << "GK_SPEC_FN bool gk_spec_tile_whole(const uint32_t nwide) { return nwide > GK_HANDOVER_MAX; }\n";
  // ---- phase 2, gk_spec_object(): one thread per object, from shared memory.  Returns true when the object is wide: its words are
  // then meaningless (the interpreter evaluates it, gk_spec_wide() having listed it; a matcher error may be listed twice, with the
  // same code).  `o` is the object's index in the tile, `obj` its index in the batch.
  o << "\nGK_SPEC_FN bool gk_spec_object(const GkBatch& B, const uint32_t* stg, const uint32_t* __restrict__ pool, const uint8_t* __restrict__ cbytes,\n"
       "                               const uint32_t* actw, const GkOut& out, const uint32_t obj, const uint32_t o, uint32_t* vw, uint32_t* ew) {\n";
  o << "  const uint32_t lo0 = o, hi0 = o + 1u, n0 = 1u, f0 = 1u;\n  (void)lo0; (void)hi0; (void)n0; (void)f0; (void)out; (void)pool; (void)cbytes; (void)stg;\n";
  o << "  bool big = false;\n";
  for (size_t j = 0; j < nested.size(); ++j) {
    const uint32_t s = nested[j];
    o << "  const uint16_t* __restrict__ q" << s << " = reinterpret_cast<const uint16_t*>(stg) + stg[" << NG + j << "];\n";
    scope_extent(s, [&](const std::string& row) { return "(uint32_t)q" + std::to_string(s) + "[" + row + "]"; });
    o << "  const uint32_t f" << s << " = n" << s << " >= 32u ? 0xffffffffu : ((1u << n" << s << ") - 1u);\n  (void)hi" << s << "; (void)f" << s << ";\n";
  }
  // the object's rows of scope s start at bit e<g> of row loop g's staged planes: plane k's 32-bit window there, bit j = row j of the
  // object, is the mask of export k (masked to the object's rows, f<s>); an export only object-level EXISTS read is that mask != 0.
  // On the object's own row (f0 = 1) the window is one bit of the low word.  Each window is taken where the walk first reads it.
  std::vector<uint8_t> group_done(groups.size(), 0), window_done(g.nvar, 0);
  std::vector<int> plane_of(g.nvar, -1);
  for (size_t gi = 0; gi < NG; ++gi)
    for (size_t k = 0; k < exports[gi].size(); ++k) plane_of[exports[gi][k]] = (int)k;
  auto emit_window = [&](size_t gi, uint32_t v) {
    const std::string G = std::to_string(gi), S = std::to_string(group_scope(gi));
    const uint32_t P = group_planes(gi), k = (uint32_t)plane_of[v];
    if (!group_done[gi]) {
      group_done[gi] = 1;
      o << "  // ---- exports of scope " << S << " (row loop " << gi << "): windows of the planes gk_spec_stage() left, from the object's first row\n";
      o << "  const uint32_t e" << G << " = lo" << S << " + stg[" << NR + gi << "], sh" << G << " = e" << G << " & 31u;\n";
      o << "  const uint32_t* __restrict__ pl" << G << " = stg + stg[" << gi << "] + (e" << G << " >> 5) * " << P << "u;\n";
    }
    if (group_scope(gi) == 0) {
      o << "  const uint32_t v" << v << " = (pl" << G << "[" << k << "] >> sh" << G << ") & 1u;\n";
    } else {
      const std::string win = "GK_SPEC_FUNNEL(pl" + G + "[" + std::to_string(k) + "], pl" + G + "[" + std::to_string(P + k) + "], sh" + G + ") & f" + S;
      o << "  const uint32_t v" << v << " = " << (form[v] == kAny ? "(" + win + ") != 0u ? 1u : 0u" : win) << ";\n";
    }
  };
  // ---- everything else depth-first from the results: a node right after what it reads.  The gates phase 1 evaluated are not nodes
  // here: the walk ends at the exports.
  std::function<void(uint32_t)> emit_var = [&](uint32_t v) {
    if (local[v] >= 0) {
      if (!window_done[v]) {
        window_done[v] = 1;
        emit_window((size_t)group_ix.at((uint32_t)local[v]), v);
      }
      return;
    }
    const int pr = g.producer[v];
    if (pr < 0) return;
    SpecNode& n = g.nodes[(size_t)pr];
    if (n.done) return;
    n.done = true;
    for (uint32_t d : n.deps) emit_var(d);
    o << n.code;
  };
  for (const Ord& ent : order) {
    const uint32_t cix = ent.cix;
    const GkOutEnt& oe = c.outs[cix];
    g.deps.clear();
    const std::string pv = (oe.flags & 1u) ? "1u" : (oe.flags & 2u) ? "0u" : "(" + g.rd(oe.prog_slot) + " & 1u)";
    const std::string mt = g.rd(oe.match_slot), er = g.rd(oe.err_slot);
    for (uint32_t d : g.deps) emit_var(d);
    o << "  vw[" << (cix >> 5) << "] |= (" << pv << " & " << mt << ") << " << (cix & 31u) << ";   // constraint " << cix << " (" << ent.kind << ")\n  ew[" << (cix >> 5) << "] |= (" << er
      << " & 1u) << " << (cix & 31u) << ";\n";
  }
  // the enforcement-point filter: one packed word per 32 constraints (actw), not a test per constraint
  for (uint32_t w = 0; w < W; ++w) o << "  vw[" << w << "] &= actw[" << w << "];\n  ew[" << w << "] &= actw[" << w << "];\n";
  o << "  return big;\n}\n";
  auto r16 = [](size_t x) { return (x + 15) / 16 * 16; };
  out.smem = r16(c.schema.cols.size() * sizeof(GkColumn) + NS * sizeof(GkScope) + 3 * (size_t)W * 32 * 4 + (size_t)W * 4) + 16;
  o << "#define GK_SPEC_NS " << NS << "u\n#define GK_SPEC_STAGE_AT " << out.smem << "u   /* the staging area's byte offset in dynamic shared memory */\n";
  o << kWrapper;
  // (the folding as the text's first line: a dumped text says what it stages)
  out.src = "// " + out.fold_text() + "\n" + o.str();
  out.words = W;
  out.n_fast = g.n_fast;
  out.n_generic = g.n_generic;
  return out;
}

}  // namespace gk
