// The evaluation kernel for sm_90a: a tile-at-a-time columnar bitmap engine.
//
//   * ALL constraints are one netlist of bit-column ops (program.h GkOp).  A CTA owns a tile of kTile consecutive
//     objects; every node of the netlist is a packed bit column of the tile held in shared memory (32 rows/word).
//   * ATOM  : one warp streams the tile's slice of one feature column -- unit-stride, coalesced loads of 32 rows per
//             instruction -- compares against the constant and packs the 32 verdicts with one __ballot_sync.
//             Prefix tests read a fixed 32-byte HEAD record per row with two 128-bit loads and do masked word compares.
//   * GATE  : n-ary AND/OR on whole words: 32 rows per instruction, operands broadcast from shared memory.
//   * ACC / BCAST : EXISTS and loop-invariant hoisting as segmented OR / range fill over the CSR child ranges; all
//             reductions over the same scope in a phase share one pass over the ranges.
//   * MATCH : the spec.match pre-filter, once per DISTINCT match block per object, ballot-packed like an atom.
//   * gather: after the last phase a 32x32 bit transpose per warp (32 ballots) turns the per-constraint result columns
//             into the object-major bitmap rows, which are contiguous in HBM: coalesced stores; totals via popc.
//   * ops of one dependency phase are independent; warps pull work items (an op, or a row slice of a heavy op,
//     heaviest first) from a shared-memory counter, and one __syncthreads separates phases.
// This is integer / byte work bounded by instruction issue and HBM traffic -- nothing here belongs on tensor cores.
#pragma once
#include <cuda_runtime.h>

#include "eval_layout.h"
#include "program.h"
#include "vm_core.h"

// the EXISTS walk shared by GK_N_ACC and GK_N_ACC2 (GK_ACC_TEST decides a parent row from its window of child bits)
#define GK_ACC_WALK \
          { \
            const uint32_t par = (uint32_t)scopes[level].parent, npair = op.w3; \
            const uint32_t* pairs = pool + op.w1; \
            const uint32_t* coff = scopes[level].off + s_lo[par]; \
            const uint32_t clo = s_lo[level], pcnt = s_cnt[par]; \
            const uint32_t pw = (pcnt + 31u) >> 5, cw = (s_cnt[level] + 31u) >> 5; \
            const uint32_t g0 = pw * part / nparts, g1 = pw * (part + 1u) / nparts; \
            for (uint32_t g = g0; g < g1; g += 4u) { \
              uint32_t ra[4], rb[4]; \
_Pragma("unroll") \
              for (int u = 0; u < 4; ++u) { \
                const uint32_t r = (g + u) * 32u + lane; \
                ra[u] = rb[u] = 0u; \
                if (g + u < g1 && r < pcnt) { \
                  ra[u] = coff[r] - clo; \
                  rb[u] = coff[r + 1] - clo; \
                } \
              } \
_Pragma("unroll") \
              for (int u = 0; u < 4; ++u) { \
                if (g + u >= g1) break; \
                const uint32_t a = ra[u], b = rb[u]; \
                const uint32_t nb = b - a, sh = a & 31u; \
                const uint32_t m = nb >= 32u ? FULL : ((1u << nb) - 1u); \
                const uint32_t wl = cw ? min(a >> 5, cw - 1u) : 0u, wh = cw ? min((a >> 5) + 1u, cw - 1u) : 0u; \
                const bool wide = nb > 32u; \
                const bool any_wide = __any_sync(FULL, wide); \
                for (uint32_t j = 0; j < npair; ++j) { \
                  const uint32_t e = pairs[j]; \
                  const uint32_t* in = slots + (e & 0xffffu); \
                  const uint32_t win = __funnelshift_r(in[wl], in[wh], sh) & m; \
                  bool any; \
                  GK_ACC_TEST \
                  const uint32_t wd = __ballot_sync(FULL, any); \
                  if (lane == 0) slots[(e >> 16) + g + u] = wd; \
                } \
              } \
            } \
          }

namespace gk {

using KParams = GkKParams;

#ifndef GK_THREADS
#define GK_THREADS 256
#endif
#ifndef GK_TILE
#define GK_TILE 512
#endif
constexpr int kThreads = GK_THREADS;
constexpr int kWarps = kThreads / 32;
constexpr uint32_t kTile = GK_TILE;
constexpr uint32_t kMaxPhases = 64;

__device__ __forceinline__ void stage(void* dst, const void* src, size_t bytes) {
  // 16-byte vector copies; sizes/offsets are padded to 16 on the host
  const uint4* s = reinterpret_cast<const uint4*>(src);
  uint4* d = reinterpret_cast<uint4*>(dst);
  for (size_t i = threadIdx.x; i < bytes / 16; i += blockDim.x) d[i] = s[i];
}

__device__ __forceinline__ uint32_t range_mask(uint32_t w, uint32_t a, uint32_t b) {
  // bits of word w that lie in the row range [a, b)
  const uint32_t lo = w * 32u, hi = lo + 32u;
  const uint32_t x = a > lo ? a : lo, y = b < hi ? b : hi;
  if (x >= y) return 0u;
  const uint32_t nb = y - x;
  return (nb == 32u ? 0xffffffffu : ((1u << nb) - 1u)) << (x - lo);
}

// words [w0, w1) of one column's tile slice, one ballot-packed word per 32 rows.  The op switch is OUTSIDE the row loop:
// every loop body is a straight load-compare-ballot sequence over FOUR 32-row groups -- four independent loads per lane
// in flight, no per-group bounds branch (rows past the tile's count evaluate to 0; slots are padded to 4 words), and
// lane 0 stores the four result words with one 128-bit shared-memory store.  w0 is a multiple of 4.
#ifndef GK_ATOM_UNROLL
#define GK_ATOM_UNROLL 4      /* measured: 8 or 16 groups per trip cost registers (resident CTAs) and buy nothing */
#endif
#define GK_ATOM_LOOP(EXPR)                                                        \
  for (uint32_t w = w0; w < w1; w += GK_ATOM_UNROLL) {                            \
    const uint32_t r0 = w * 32u + lane;                                           \
    const size_t row0 = (size_t)lo + r0;                                          \
    bool v4[GK_ATOM_UNROLL];                                                      \
    _Pragma("unroll") for (int u = 0; u < GK_ATOM_UNROLL; ++u) {                  \
      const size_t row = row0 + 32u * u;                                          \
      v4[u] = (r0 + 32u * u < cnt) && (EXPR);                                     \
    }                                                                             \
    _Pragma("unroll") for (int u = 0; u < GK_ATOM_UNROLL; u += 4) {               \
      uint4 wd;                                                                   \
      wd.x = __ballot_sync(0xffffffffu, v4[u]);                                   \
      wd.y = __ballot_sync(0xffffffffu, v4[u + 1]);                               \
      wd.z = __ballot_sync(0xffffffffu, v4[u + 2]);                               \
      wd.w = __ballot_sync(0xffffffffu, v4[u + 3]);                               \
      if (lane == 0 && w + u < wcap) *reinterpret_cast<uint4*>(out + w + u) = wd; \
    }                                                                             \
  }

// The same loop with the row's loads separated from the test: LOAD fills A[u] (32-bit) / B[u] (64-bit) for the four groups
// unconditionally -- a test written `vt[row] != UNDEF && num[row] < k` makes the second load wait for the first -- and
// TEST then runs on registers (a, b).
#ifdef GK_EXP_NOLOAD   /* latency experiment: atoms test a function of the row index instead of loaded data */
#define GK_EXP_LOAD(L) A[u] = (uint32_t)row & 7u; B[u] = (long long)row
#else
#define GK_EXP_LOAD(L) L
#endif
#define GK_ATOM_LOOP2(LOAD, TEST)                                                 \
  for (uint32_t w = w0; w < w1; w += GK_ATOM_UNROLL) {                            \
    const uint32_t r0 = w * 32u + lane;                                           \
    const size_t row0 = (size_t)lo + r0;                                          \
    uint32_t A[GK_ATOM_UNROLL];                                                   \
    long long B[GK_ATOM_UNROLL];                                                  \
    bool v4[GK_ATOM_UNROLL];                                                      \
    if ((w + GK_ATOM_UNROLL) * 32u <= cnt) { /* interior trip (warp-uniform): no bounds predicates at all */ \
      _Pragma("unroll") for (int u = 0; u < GK_ATOM_UNROLL; ++u) {                \
        const size_t row = row0 + 32u * u;                                        \
        A[u] = 0u;                                                                \
        B[u] = 0ll;                                                               \
        GK_EXP_LOAD(LOAD);                                                        \
      }                                                                           \
      _Pragma("unroll") for (int u = 0; u < GK_ATOM_UNROLL; ++u) {                \
        const uint32_t a = A[u];                                                  \
        const long long b = B[u];                                                 \
        (void)a; (void)b;                                                         \
        v4[u] = (TEST);                                                           \
      }                                                                           \
    } else {                                                                      \
      _Pragma("unroll") for (int u = 0; u < GK_ATOM_UNROLL; ++u) {                \
        const size_t row = row0 + 32u * u;                                        \
        A[u] = 0u;                                                                \
        B[u] = 0ll;                                                               \
        if (r0 + 32u * u < cnt) { GK_EXP_LOAD(LOAD); }                            \
      }                                                                           \
      _Pragma("unroll") for (int u = 0; u < GK_ATOM_UNROLL; ++u) {                \
        const uint32_t a = A[u];                                                  \
        const long long b = B[u];                                                 \
        (void)a; (void)b;                                                         \
        v4[u] = (r0 + 32u * u < cnt) && (TEST);                                   \
      }                                                                           \
    }                                                                             \
    _Pragma("unroll") for (int u = 0; u < GK_ATOM_UNROLL; u += 4) {               \
      uint4 wd;                                                                   \
      wd.x = __ballot_sync(0xffffffffu, v4[u]);                                   \
      wd.y = __ballot_sync(0xffffffffu, v4[u + 1]);                               \
      wd.z = __ballot_sync(0xffffffffu, v4[u + 2]);                               \
      wd.w = __ballot_sync(0xffffffffu, v4[u + 3]);                               \
      if (lane == 0 && w + u < wcap) *reinterpret_cast<uint4*>(out + w + u) = wd; \
    }                                                                             \
  }

__device__ __forceinline__ bool sid_in_small(const uint32_t* pool, uint32_t a, uint32_t b, uint32_t v) {
  bool hit = false;
  for (uint32_t j = 0; j < b; ++j) hit = hit || pool[a + j] == v;
  return hit;
}

__device__ __forceinline__ bool num_cmp_row(const uint8_t* vt, const int64_t* num, size_t row, int64_t k, uint32_t cmp) {
  const uint32_t t = vt[row];
  if (t == GK_VT_NUM) {
    const int64_t v = num[row];
    return gk_cmp_apply(cmp, v < k ? -1 : (v > k ? 1 : 0));
  }
  if (t == GK_VT_UNDEF || t == GK_VT_NUM_INEXACT) return false;
  return gk_cmp_apply(cmp, gk_vt_rank(t) < 2 ? -1 : 1);
}

__device__ __forceinline__ void atom_rows(const GkColumn& c, uint32_t aop, uint32_t a, uint32_t b, const uint32_t* pool, const uint8_t* cbytes,
                                          uint32_t lo, uint32_t cnt, uint32_t w0, uint32_t w1, uint32_t lane, uint32_t* out) {
  const uint32_t wcap = (((cnt + 31u) >> 5) + 3u) & ~3u;   // words of the slot that may be written (slots are padded to 4 words)
  switch (aop) {
    case GK_OP_TRUTHY: {
      const uint8_t* vt = c.vt;
      GK_ATOM_LOOP2(A[u] = vt[row], a != GK_VT_UNDEF && a != GK_VT_FALSE)
      break;
    }
    case GK_OP_DEFINED: {
      const uint8_t* vt = c.vt;
      GK_ATOM_LOOP2(A[u] = vt[row], a != GK_VT_UNDEF)
      break;
    }
    case GK_OP_VTMASK: {
      const uint8_t* vt = c.vt;
      const uint32_t mask = a;
      GK_ATOM_LOOP2(A[u] = vt[row], ((1u << a) & mask) != 0u)
      break;
    }
    case GK_OP_SID_EQ: {
      const uint32_t* sid = c.sid;
      const uint32_t want = a;
      GK_ATOM_LOOP2(A[u] = sid[row], a == want)
      break;
    }
    case GK_OP_SID_IN: {
      const uint32_t* sid = c.sid;
      if (b <= 8u) {   // small sets: a broadcast linear scan beats the binary search
        const uint32_t pa = a, pn = b;
        GK_ATOM_LOOP2(A[u] = sid[row], sid_in_small(pool, pa, pn, a))
      } else {
        GK_ATOM_LOOP(gk_atom(c, row, aop, a, b, pool, cbytes))
      }
      break;
    }
    case GK_OP_NUM_CMP: {
      const uint8_t* vt = c.vt;
      const int64_t* num = c.num;
      const int64_t k = (int64_t)(((uint64_t)pool[a + 1] << 32) | pool[a]);
      if (k == INT64_MIN || k == INT64_MAX) {   // the sentinels of non-numbers (see Flattener::encode): generic path
        GK_ATOM_LOOP(num_cmp_row(vt, num, row, k, b))
        break;
      }
      // a defined non-number holds INT64_MIN / INT64_MAX according to its type rank, so one signed compare is OPA's order
      switch (b) {
        case GK_CMP_LT: GK_ATOM_LOOP2(A[u] = vt[row]; B[u] = num[row], a != GK_VT_UNDEF && b < k) break;
        case GK_CMP_LE: GK_ATOM_LOOP2(A[u] = vt[row]; B[u] = num[row], a != GK_VT_UNDEF && b <= k) break;
        case GK_CMP_GT: GK_ATOM_LOOP2(A[u] = vt[row]; B[u] = num[row], a != GK_VT_UNDEF && b > k) break;
        case GK_CMP_GE: GK_ATOM_LOOP2(A[u] = vt[row]; B[u] = num[row], a != GK_VT_UNDEF && b >= k) break;
        case GK_CMP_EQ: GK_ATOM_LOOP2(A[u] = vt[row]; B[u] = num[row], a != GK_VT_UNDEF && b == k) break;
        default: GK_ATOM_LOOP2(A[u] = vt[row]; B[u] = num[row], a != GK_VT_UNDEF && b != k) break;
      }
      break;
    }
    case GK_OP_ANYPREFIX: {
      // two 128-bit loads fetch the row's 32-byte HEAD record (coalesced: 1 KB per warp); every prefix of the list is
      // then tested with masked word compares against constants broadcast from shared memory
      const uint8_t* vt = c.vt;
      const uint4* head = reinterpret_cast<const uint4*>(c.head);
      const uint32_t* ent = pool + a;
      bool all_short = true;
      for (uint32_t j = 0; j < b; ++j) all_short = all_short && ent[j * GK_PREFIX_ENT] <= GK_HEAD_BYTES;
      if (!all_short) {
        GK_ATOM_LOOP(gk_atom(c, row, aop, a, b, pool, cbytes))
        break;
      }
      const uint32_t wend = min(w1, (cnt + 31u) >> 5);
      for (uint32_t r = w0 * 32u + lane; r < wend * 32u; r += 32u) {
        bool v = false;
        // the type byte and the 32-byte record are fetched together (independent loads), then tested
        uint32_t t = GK_VT_UNDEF;
        uint4 h0 = make_uint4(0, 0, 0, 0), h1 = make_uint4(0, 0, 0, 0);
        if (r < cnt) {
          t = vt[lo + r];
          h0 = head[2 * (size_t)(lo + r)];
          h1 = head[2 * (size_t)(lo + r) + 1];
        }
        if (t == GK_VT_STR) {
          const uint32_t lenb = h1.w >> 24;
          for (uint32_t j = 0; j < b && !v; ++j) {
            const uint32_t* e = ent + j * GK_PREFIX_ENT;
            const uint32_t* m = e + 2 + GK_HEAD_WORDS;
            const uint32_t diff = ((h0.x ^ e[2]) & m[0]) | ((h0.y ^ e[3]) & m[1]) | ((h0.z ^ e[4]) & m[2]) | ((h0.w ^ e[5]) & m[3]) |
                                  ((h1.x ^ e[6]) & m[4]) | ((h1.y ^ e[7]) & m[5]) | ((h1.z ^ e[8]) & m[6]) | ((h1.w ^ e[9]) & m[7]);
            v = diff == 0u && lenb >= e[0];
          }
        }
        const uint32_t wd = __ballot_sync(0xffffffffu, v);
        if (lane == 0) out[r >> 5] = wd;
      }
      break;
    }
    default: {
      GK_ATOM_LOOP(gk_atom(c, row, aop, a, b, pool, cbytes))
      break;
    }
  }
}

// ---- every register-testable atom of one column in one pass (GK_N_ATOMS): the row's type byte / sid / number are loaded once
// per trip -- four 32-row groups, all loads in flight together -- and each atom of the column is then a compare + ballot on
// registers, its four result words stored with one 128-bit shared-memory store.
#define GK_RUN_ATOM(EXPR)                                                            \
  {                                                                                  \
    bool v4[4];                                                                      \
    _Pragma("unroll") for (int u = 0; u < 4; ++u) v4[u] = ok[u] && (EXPR);           \
    uint4 wd;                                                                        \
    wd.x = __ballot_sync(0xffffffffu, v4[0]);                                        \
    wd.y = __ballot_sync(0xffffffffu, v4[1]);                                        \
    wd.z = __ballot_sync(0xffffffffu, v4[2]);                                        \
    wd.w = __ballot_sync(0xffffffffu, v4[3]);                                        \
    if (lane == 0) *reinterpret_cast<uint4*>(slots + (e.x >> 16) + w) = wd;          \
  }
__device__ __noinline__ void atoms_rows(const GkColumn& c, const uint32_t* ent, uint32_t nent, const uint32_t* pool, uint32_t lo, uint32_t cnt, uint32_t w0,
                                        uint32_t w1, uint32_t lane, uint32_t* slots) {
  const bool has_vt = (c.enc & GK_ENC_VT) != 0u, has_sid = (c.enc & GK_ENC_SID) != 0u, has_num = (c.enc & GK_ENC_NUM) != 0u;
  const uint8_t* __restrict__ pvt = c.vt;
  const uint32_t* __restrict__ psid = c.sid;
  const long long* __restrict__ pnum = reinterpret_cast<const long long*>(c.num);
  for (uint32_t w = w0; w < w1; w += 4u) {
    const uint32_t r0 = w * 32u + lane;
    const size_t row0 = (size_t)lo + r0;
    uint32_t vt[4], sid[4];
    long long num[4];
    bool ok[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      ok[u] = r0 + 32u * u < cnt;
      vt[u] = (uint32_t)GK_VT_UNDEF;
      sid[u] = (uint32_t)GK_SID_UNDEF;
      num[u] = 0ll;
    }
    if (has_vt) {
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (ok[u]) vt[u] = pvt[row0 + 32u * u];
    }
    if (has_sid) {
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (ok[u]) sid[u] = psid[row0 + 32u * u];
    }
    if (has_num) {
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (ok[u]) num[u] = pnum[row0 + 32u * u];
    }
    for (uint32_t j = 0; j < nent; ++j) {
      const uint4 e = *reinterpret_cast<const uint4*>(ent + j * GK_ATOMS_ENT);
      switch (e.x & 0xffu) {
        case GK_OP_TRUTHY: GK_RUN_ATOM(vt[u] != GK_VT_UNDEF && vt[u] != GK_VT_FALSE) break;
        case GK_OP_DEFINED: GK_RUN_ATOM(vt[u] != GK_VT_UNDEF) break;
        case GK_OP_VTMASK: GK_RUN_ATOM(((1u << vt[u]) & e.y) != 0u) break;
        case GK_OP_SID_EQ: GK_RUN_ATOM(sid[u] == e.y) break;
        case GK_OP_SID_IN: GK_RUN_ATOM(sid_in_small(pool, e.y, e.z, sid[u])) break;
        default: {   // GK_OP_NUM_CMP: non-numbers hold INT64_MIN / INT64_MAX by their type rank, so one signed compare is OPA's order
          const long long k = (long long)(((uint64_t)pool[e.y + 1] << 32) | pool[e.y]);
          switch (e.z) {
            case GK_CMP_LT: GK_RUN_ATOM(vt[u] != GK_VT_UNDEF && num[u] < k) break;
            case GK_CMP_LE: GK_RUN_ATOM(vt[u] != GK_VT_UNDEF && num[u] <= k) break;
            case GK_CMP_GT: GK_RUN_ATOM(vt[u] != GK_VT_UNDEF && num[u] > k) break;
            case GK_CMP_GE: GK_RUN_ATOM(vt[u] != GK_VT_UNDEF && num[u] >= k) break;
            case GK_CMP_EQ: GK_RUN_ATOM(vt[u] != GK_VT_UNDEF && num[u] == k) break;
            default: GK_RUN_ATOM(vt[u] != GK_VT_UNDEF && num[u] != k) break;
          }
          break;
        }
      }
    }
  }
}

// One CTA = one tile of consecutive objects at a time; all intermediate bit columns live in shared memory.
#ifndef GK_MIN_CTAS
#define GK_MIN_CTAS 4         /* 4 resident CTAs per SM = 64 registers per thread: room for the fused atom runs */
#endif
__global__ void __launch_bounds__(kThreads, GK_MIN_CTAS) gk_eval_kernel(const KParams p) {
  extern __shared__ __align__(16) unsigned char smem[];
  const uint32_t C = p.prog.nconstraints, W = p.out.words, NS = p.batch.nscopes, NP = p.prog.nphases;
  // ---- shared-memory layout (the launch is sized with the same call: CudaBackend::prepare)
  const GkEvalLayout L = gk_eval_layout(p.prog.nconstraints, p.batch.nscopes, p.prog.nphases, p.slot_words, p.prog.nops, p.prog.nitems, p.prog.nmatch,
                                        p.batch.ncols, p.prog.npool, p.prog.ncbytes);
  uint32_t* s_tot = reinterpret_cast<uint32_t*>(smem + L.s_tot);
  uint32_t* s_err = reinterpret_cast<uint32_t*>(smem + L.s_err);
  uint32_t* s_act = reinterpret_cast<uint32_t*>(smem + L.s_act);
  uint32_t* s_lo = reinterpret_cast<uint32_t*>(smem + L.s_lo);
  uint32_t* s_cnt = reinterpret_cast<uint32_t*>(smem + L.s_cnt);
  uint32_t* s_poff = reinterpret_cast<uint32_t*>(smem + L.s_poff);
  uint32_t* slots = reinterpret_cast<uint32_t*>(smem + L.slots);
  GkOutEnt* outs = reinterpret_cast<GkOutEnt*>(smem + L.outs);
  GkOp* ops = reinterpret_cast<GkOp*>(smem + L.ops);
  uint32_t* items = reinterpret_cast<uint32_t*>(smem + L.items);
  GkMatch* match = reinterpret_cast<GkMatch*>(smem + L.match);
  GkColumn* cols = reinterpret_cast<GkColumn*>(smem + L.cols);
  GkScope* scopes = reinterpret_cast<GkScope*>(smem + L.scopes);
  uint32_t* pool = reinterpret_cast<uint32_t*>(smem + L.pool);
  uint8_t* cbytes = reinterpret_cast<uint8_t*>(smem + L.cbytes);

  // list mode (beside gk_spec_kernel): only the object ranges gk_spec_plan_kernel listed; a CTA without one stages nothing
  const uint32_t nunits = p.list_mode ? *p.unit_count : p.ntiles;
  for (uint32_t i = threadIdx.x; i < C; i += blockDim.x) {
    s_tot[i] = 0;
    s_err[i] = 0;
    s_act[i] = p.active[i];
  }
  for (uint32_t i = threadIdx.x; i <= NP; i += blockDim.x) s_poff[i] = p.prog.phase_off[i];
  if (blockIdx.x < nunits) {   // the program and schema tables, each its whole padded region
    stage(outs, p.prog.outs, L.ops - L.outs);
    stage(ops, p.prog.ops, L.items - L.ops);
    stage(items, p.prog.items, L.match - L.items);
    stage(match, p.prog.match, L.cols - L.match);
    stage(cols, p.batch.cols, L.scopes - L.cols);
    stage(scopes, p.batch.scopes, L.pool - L.scopes);
    stage(pool, p.prog.pool, L.cbytes - L.pool);
    stage(cbytes, p.prog.cbytes, L.end - L.cbytes);
  }
  __syncthreads();

  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t FULL = 0xffffffffu;

  for (uint32_t ti = blockIdx.x; ti < nunits; ti += gridDim.x) {
    // ---- the unit's row ranges (rows of consecutive objects are contiguous at every scope): a tile's from the precomputed table;
    // a listed object range's through the CSR offsets, parents before children (any such range lies inside one tile, so the slot
    // area sized for the largest tile holds it)
    if (p.list_mode) {
      if (threadIdx.x == 0) {
        const uint32_t a = p.units[2 * ti];
        uint32_t* s_hi = s_cnt;   // (the range ends first, turned into counts below)
        s_lo[0] = a;
        s_hi[0] = a + p.units[2 * ti + 1];
        for (uint32_t s = 1; s < NS; ++s) {
          const uint32_t par = (uint32_t)scopes[s].parent;
          s_lo[s] = scopes[s].off[s_lo[par]];
          s_hi[s] = scopes[s].off[s_hi[par]];
        }
        for (uint32_t s = 0; s < NS; ++s) s_cnt[s] -= s_lo[s];
      }
    } else {
      for (uint32_t s = threadIdx.x; s < NS; s += blockDim.x) {
        const uint32_t a = p.tile_lo[(size_t)ti * NS + s], b = p.tile_lo[(size_t)(ti + 1) * NS + s];
        s_lo[s] = a;
        s_cnt[s] = b - a;
      }
    }
    __syncthreads();
    const uint32_t nobj = s_cnt[0], obj0 = s_lo[0];

    for (uint32_t ph = 0; ph < NP; ++ph) {
      const uint32_t ibase = s_poff[ph], icnt = s_poff[ph + 1] - ibase;
#ifdef GK_PHASE_TIMING
      const long long tp0 = clock64();
#endif
      // items are sorted heaviest first: dealing them round-robin to the warps is a longest-processing-time schedule
      for (uint32_t k = warp; k < icnt; k += kWarps) {
        const uint32_t item = items[ibase + k];
        const GkOp op = ops[item & 0xfffffu];
        const uint32_t part = (item >> 20) & 0x3fu, nparts = item >> 26;
        const uint32_t kind = op.w0 & 0xffu, level = (op.w0 >> 8) & 0xffu;
        uint32_t* out = slots + (op.w0 >> 16);
#ifdef GK_PHASE_TIMING
        const long long ti0 = clock64();
#endif
        switch (kind) {
          case GK_N_ATOM: {
            const uint32_t cnt = s_cnt[level], words = (cnt + 31u) >> 5;
            const uint32_t amask = ~(uint32_t)(GK_ATOM_UNROLL - 1);
            const uint32_t pw0 = (words * part / nparts) & amask, pw1 = part + 1u == nparts ? words : ((words * (part + 1u) / nparts) & amask);
            atom_rows(cols[op.w1 >> 8], op.w1 & 0xffu, op.w2, op.w3, pool, cbytes, s_lo[level], cnt, pw0, pw1, lane, out);
            break;
          }
          case GK_N_ATOMS: {
            const uint32_t cnt = s_cnt[level], words = (cnt + 31u) >> 5;
            const uint32_t pw0 = (words * part / nparts) & ~3u, pw1 = part + 1u == nparts ? words : ((words * (part + 1u) / nparts) & ~3u);
            atoms_rows(cols[op.w1 >> 8], pool + op.w2, op.w3, pool, s_lo[level], cnt, pw0, pw1, lane, slots);
            break;
          }
          case GK_N_GATE: {
            const uint32_t f = op.w2, words = (s_cnt[level] + 31u) >> 5, nin = op.w3;
            const uint32_t* in = pool + op.w1;
            const uint32_t no = (f & GK_G_NEG_OUT) ? FULL : 0u;
            const bool is_or = (f & GK_G_OR) != 0u;
            for (uint32_t i = lane; i < words; i += 32u) {
              uint32_t acc = is_or ? 0u : FULL;
              for (uint32_t j = 0; j < nin; ++j) {
                const uint32_t e = in[j];
                const uint32_t x = slots[(e & 0xffffu) + i] ^ (uint32_t)((int32_t)e >> 31);
                acc = is_or ? (acc | x) : (acc & x);
              }
              out[i] = acc ^ no;
            }
            break;
          }
          case GK_N_CONST: {
            const uint32_t v = (op.w1 & 1u) ? FULL : 0u, words = (s_cnt[level] + 31u) >> 5;
            for (uint32_t i = lane; i < words; i += 32u) out[i] = v;
            break;
          }
          case GK_N_BCAST: {   // parent-level columns -> rows of the child scope `level`, for every (in, out) pair of the group
            const uint32_t par = (uint32_t)scopes[level].parent, npair = op.w3;
            const uint32_t* pairs = pool + op.w1;
            const uint32_t* coff = scopes[level].off + s_lo[par];
            const uint32_t clo = s_lo[level], pcnt = s_cnt[par], words = (s_cnt[level] + 31u) >> 5;
            for (uint32_t j = 0; j < npair; ++j) {
              uint32_t* dst = slots + (pairs[j] >> 16);
              for (uint32_t i = lane; i < words; i += 32u) dst[i] = 0u;
            }
            __syncwarp();
            // the CSR offsets are the only global loads here: fetch them for four 32-row groups before touching any, so the
            // op pays one memory latency per 128 parent rows instead of one per 32
            for (uint32_t r0 = lane; r0 < pcnt; r0 += 128u) {
              uint32_t ra[4], rb[4];
#pragma unroll
              for (int u = 0; u < 4; ++u) {
                const uint32_t r = r0 + 32u * u;
                ra[u] = rb[u] = 0u;
                if (r < pcnt) {
                  ra[u] = coff[r] - clo;
                  rb[u] = coff[r + 1] - clo;
                }
              }
#pragma unroll
              for (int u = 0; u < 4; ++u) {
                const uint32_t r = r0 + 32u * u, a = ra[u], b = rb[u];
                if (b <= a) continue;
                for (uint32_t j = 0; j < npair; ++j) {
                  const uint32_t e = pairs[j];
                  if ((slots[(e & 0xffffu) + (r >> 5)] >> (r & 31u)) & 1u) {
                    uint32_t* dst = slots + (e >> 16);
                    for (uint32_t w = a >> 5; w <= (b - 1u) >> 5; ++w) atomicOr(&dst[w], range_mask(w, a, b));
                  }
                }
              }
            }
            break;
          }
          // EXISTS: OR over each parent's child range; ranges + masks computed once for the whole group.  The CSR offsets of four
          // parent-row groups are fetched first (the only global loads of the op): one memory latency per 128 parent rows.  A range
          // of up to 32 children is a 32-bit window of the child bit column starting at bit a: one funnel shift over two adjacent
          // words, branch-free for every lane; longer ranges (rare) add a tail loop.  (m == 0 for a parent without children.)
          case GK_N_ACC: {
#define GK_ACC_TEST                                                                                                                   \
  any = win != 0u;                                                                                                                    \
  if (any_wide)                                                                                                                       \
    if (wide && !any)                                                                                                                 \
      for (uint32_t w = (a + 32u) >> 5; w <= (b - 1u) >> 5 && !any; ++w) any = (in[w] & range_mask(w, a + 32u, b)) != 0u;
            GK_ACC_WALK
#undef GK_ACC_TEST
            break;
          }
          case GK_N_ACC2: {    // "at least two children" (the audit's ambiguity netlist): the same walk, counting -- its own copy so
                               // that the decision netlist's EXISTS carries no extra branch
#define GK_ACC_TEST                                                                                                                   \
  {                                                                                                                                   \
    uint32_t cnt = (uint32_t)__popc(win);                                                                                             \
    if (any_wide)                                                                                                                     \
      if (wide)                                                                                                                       \
        for (uint32_t w = (a + 32u) >> 5; w <= (b - 1u) >> 5 && cnt < 2u; ++w) cnt += (uint32_t)__popc(in[w] & range_mask(w, a + 32u, b)); \
    any = cnt >= 2u;                                                                                                                  \
  }
            GK_ACC_WALK
#undef GK_ACC_TEST
            break;
          }
          case GK_N_MATCH: {
            uint32_t* err = slots + (op.w1 & 0xffffu);
            const GkMatch& m = match[op.w2];
            const uint32_t words = (nobj + 31u) >> 5;
            for (uint32_t r = (words * part / nparts) * 32u + lane; r < (words * (part + 1u) / nparts) * 32u; r += 32u) {
              int res = 0;
              if (r < nobj && !(p.batch.flags[obj0 + r] & GK_F_SKIP)) res = gk_match(p.batch, pool, cbytes, m, obj0 + r);
              if (res < 0) {
                const uint32_t slot = atomicAdd(p.out.errcount, 1u);
                if (slot < p.out.errcap) {
                  p.out.errlist[3 * slot] = obj0 + r;
                  p.out.errlist[3 * slot + 1] = op.w2;
                  p.out.errlist[3 * slot + 2] = (uint32_t)(-res);
                }
              }
              const uint32_t wm = __ballot_sync(FULL, res > 0), we = __ballot_sync(FULL, res < 0);
              if (lane == 0) {
                out[r >> 5] = wm;
                err[r >> 5] = we;
              }
            }
            break;
          }
          default: break;
        }
#ifdef GK_PHASE_TIMING
        if (lane == 0) {
          const uint32_t tk = kind;
          atomicAdd(p.timing + 2 * (kMaxPhases + 2) + 2 * tk, (unsigned long long)(clock64() - ti0));
          atomicAdd(p.timing + 2 * (kMaxPhases + 2) + 2 * tk + 1, 1ull);
        }
#endif
      }
#ifdef GK_PHASE_TIMING
      if (lane == 0) atomicAdd(p.timing + 2 * ph + 1, (unsigned long long)(clock64() - tp0));
      __syncthreads();
      if (threadIdx.x == 0) atomicAdd(p.timing + 2 * ph, (unsigned long long)(clock64() - tp0));
#else
      __syncthreads();
#endif
    }
#ifdef GK_PHASE_TIMING
    const long long tg0 = clock64();
#endif
    // ---- gather: lane l of a warp holds the result word of constraint (32 w + l) for one group of 32 objects; 32 ballots
    // transpose that 32x32 bit block so that lane o ends up with the bitmap word of object o.  The 32 objects of a group
    // are consecutive rows of the object-major output: the stores are contiguous.
    const uint32_t owords = (nobj + 31u) >> 5;
    if (W == 2u) {
      // two constraint words per object (33..64 constraints): one warp produces BOTH words of a group of 32 objects and stores
      // them as one 8-byte word per object -- whole sectors, and half as many stores per peer over NVLink
      for (uint32_t ow = warp; ow < owords; ow += kWarps) {
        uint32_t yv[2] = {0u, 0u}, ye[2] = {0u, 0u};
#pragma unroll
        for (uint32_t wi = 0; wi < 2u; ++wi) {
          const uint32_t c = wi * 32u + lane;
          uint32_t xv = 0, xe = 0;
          if (c < C && s_act[c]) {
            const GkOutEnt oe = outs[c];
            const uint32_t pv = (oe.flags & 1u) ? FULL : (oe.flags & 2u) ? 0u : slots[(oe.prog_slot) + ow];
            xv = pv & slots[(oe.match_slot) + ow];
            xe = slots[(oe.err_slot) + ow];
          }
#pragma unroll
          for (uint32_t o = 0; o < 32u; ++o) {
            const uint32_t bv = __ballot_sync(FULL, (xv >> o) & 1u);
            if (lane == o) yv[wi] = bv;
          }
          if (__any_sync(FULL, xe != 0u)) {
#pragma unroll
            for (uint32_t o = 0; o < 32u; ++o) {
              const uint32_t be = __ballot_sync(FULL, (xe >> o) & 1u);
              if (lane == o) ye[wi] = be;
            }
          }
          const uint32_t valid = range_mask(ow, 0u, nobj);
          const uint32_t nv = __popc(xv & valid), ne = __popc(xe & valid);
          if (c < C) {
            if (nv) atomicAdd(&s_tot[c], nv);
            if (ne) atomicAdd(&s_err[c], ne);
          }
        }
        const uint32_t obj = ow * 32u + lane;
        if (obj < nobj) {
          const size_t at = (size_t)(obj0 + obj) * 2u;
          const uint2 v2 = make_uint2(yv[0], yv[1]);
          if (p.npeers) {
            for (uint32_t q = 0; q < p.npeers; ++q) *reinterpret_cast<uint2*>(p.peer_viol[q] + at) = v2;   // this rank is one of the peers
          } else {
            *reinterpret_cast<uint2*>(p.out.viol + at) = v2;
          }
          *reinterpret_cast<uint2*>(p.out.err + at) = make_uint2(ye[0], ye[1]);
        }
      }
    } else
    for (uint32_t g = warp; g < owords * W; g += kWarps) {
      const uint32_t wi = g % W, ow = g / W;          // constraint word, object word
      const uint32_t c = wi * 32u + lane;
      uint32_t xv = 0, xe = 0;
      if (c < C && s_act[c]) {
        const GkOutEnt oe = outs[c];
        const uint32_t pv = (oe.flags & 1u) ? FULL : (oe.flags & 2u) ? 0u : slots[(oe.prog_slot) + ow];
        xv = pv & slots[(oe.match_slot) + ow];
        xe = slots[(oe.err_slot) + ow];
      }
      uint32_t yv = 0, ye = 0;
#pragma unroll
      for (uint32_t o = 0; o < 32u; ++o) {
        const uint32_t bv = __ballot_sync(FULL, (xv >> o) & 1u);
        if (lane == o) yv = bv;
      }
      if (__any_sync(FULL, xe != 0u)) {   // matcher errors are rare: the second transpose only where one occurred
#pragma unroll
        for (uint32_t o = 0; o < 32u; ++o) {
          const uint32_t be = __ballot_sync(FULL, (xe >> o) & 1u);
          if (lane == o) ye = be;
        }
      }
      const uint32_t obj = ow * 32u + lane;
      if (obj < nobj) {
        const size_t at = (size_t)(obj0 + obj) * W + wi;
        if (p.npeers) {
          for (uint32_t q = 0; q < p.npeers; ++q) p.peer_viol[q][at] = yv;   // this rank is one of the peers
        } else {
          p.out.viol[at] = yv;
        }
        p.out.err[at] = ye;
      }
      // totals: every lane's column word covers 32 objects of ITS constraint
      const uint32_t valid = range_mask(ow, 0u, nobj);
      const uint32_t nv = __popc(xv & valid), ne = __popc(xe & valid);
      if (c < C) {
        if (nv) atomicAdd(&s_tot[c], nv);
        if (ne) atomicAdd(&s_err[c], ne);
      }
    }
#ifdef GK_PHASE_TIMING
    if (lane == 0) atomicAdd(p.timing + 2 * NP + 1, (unsigned long long)(clock64() - tg0));
    __syncthreads();
    if (threadIdx.x == 0) atomicAdd(p.timing + 2 * NP, (unsigned long long)(clock64() - tg0));
#else
    __syncthreads();
#endif
  }
  for (uint32_t c = threadIdx.x; c < C; c += blockDim.x) {
    if (s_tot[c]) atomicAdd(p.out.totals + c, (unsigned long long)s_tot[c]);
    if (s_err[c]) atomicAdd(p.out.err_totals + c, (unsigned long long)s_err[c]);
  }
  // (the flag lives in the dynamic shared-memory area -- s_lo is free by now -- so the kernel keeps zero static shared bytes)
  if (p.npeers) gk_publish_totals(p, C, s_lo);
}

}  // namespace gk
