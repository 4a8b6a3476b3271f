// Device-visible layout of (a) a flattened object batch and (b) the lowered constraint table.
// Plain C structs shared by the host builder (C++), the CUDA kernels and the test-only host emulation.
//
//   batch  : column-wise (SoA) -- header columns one row per object, CSR label table, CSR "scopes" (one
//            row per iterated element, e.g. spec.containers[_]) with fixed-width feature columns.
//   program: DISTINCT match blocks (the spec.match pre-filter, pkg/mutation/match/match.go:32-65) and one
//            netlist of bit-column ops shared by all constraints (see GkOp).
#pragma once
#ifdef __CUDACC_RTC__   /* NVRTC (the specialised kernel, spec_codegen.cpp) has no system headers */
typedef unsigned char uint8_t;
typedef unsigned short uint16_t;
typedef unsigned int uint32_t;
typedef int int32_t;
typedef long long int64_t;
typedef unsigned long long uint64_t;
typedef unsigned long size_t;
typedef unsigned long uintptr_t;
#else
#include <stdint.h>
#include <stddef.h>
#endif

#ifdef __CUDACC__
#define GK_HD __host__ __device__ __forceinline__
#else
#define GK_HD inline
#endif
// loads of batch / program arrays in the shared per-object code (vm_core.h).  The generated kernel (spec_codegen.cpp) defines
// GK_LD as __ldg: there every such array is in global memory and read-only for the whole evaluation, so the loads take the
// non-coherent path and survive the stores of the error list.  The interpreter stages pool / cbytes in SHARED memory: plain loads.
#ifndef GK_LD
#define GK_LD(p) (*(p))
#endif

// ---- value-type codes stored in VT columns (== gk::VT)
enum { GK_VT_UNDEF = 0, GK_VT_NULL = 1, GK_VT_FALSE = 2, GK_VT_TRUE = 3, GK_VT_NUM = 4, GK_VT_STR = 5,
       GK_VT_ARR = 6, GK_VT_OBJ = 7, GK_VT_SET = 8, GK_VT_NUM_INEXACT = 9 /* number not representable as i64 */ };

// ---- column encodings (bitmask)
enum { GK_ENC_VT = 1, GK_ENC_SID = 2, GK_ENC_NUM = 4, GK_ENC_BYTES = 8,
       GK_ENC_HEAD = 16 /* fixed 32-byte record per row: the first 31 bytes of the string (zero padded) + min(len, 255) */ };
#define GK_HEAD_WORDS 8
#define GK_HEAD_BYTES 31
#define GK_PREFIX_ENT (2 + 2 * GK_HEAD_WORDS)

#define GK_SID_UNDEF 0u          /* intern id 0 is reserved: "no value" */
#define GK_SID_OTHER 1u          /* a defined value that equals none of the constants the program mentions */
#define GK_NONE 0xFFFFFFFFu
#define GK_MAX_LOOP_DEPTH 4
#define GK_MAX_SCOPES 250        /* scope ids fit one byte */
#define GK_MAX_SLOTS 65535

typedef struct {
  int32_t scope;           // 0 = root (one row per object)
  uint32_t enc;
  const uint8_t* vt;       // [rows]
  const uint32_t* sid;     // [rows]
  const int64_t* num;      // [rows]
  const uint32_t* boff;    // [rows+1]
  const uint8_t* bytes;
  const uint32_t* head;    // [rows * GK_HEAD_WORDS]
  const void* pad_;        // keeps the struct a multiple of 16 bytes (it is staged with 16-byte copies)
} GkColumn;

typedef struct {
  int32_t parent;          // parent scope id (0 = root)
  uint32_t rows;
  const uint32_t* off;     // [parent_rows+1]
} GkScope;

// header flags (per object)
enum { GK_F_HAS_OBJ = 1, GK_F_IS_NS = 2, GK_F_HAS_NS = 4 /* metadata.namespace != "" */,
       GK_F_NS_OBJ = 8 /* a Namespace object is known for the review */, GK_F_SRC_SHIFT = 4, GK_F_SRC_MASK = 0x70,
       GK_F_SKIP = 128 /* review-level error (bad JSON, ...): the kernel skips the object */,
       GK_F_NSNAME = 256 /* the row has a namespace NAME for namespaces / excludedNamespaces (nsn_off / nsn_bytes) */ };
enum { GK_SRC_EMPTY = 0, GK_SRC_ORIGINAL = 1, GK_SRC_GENERATED = 2, GK_SRC_ALL = 3, GK_SRC_INVALID = 4 };

typedef struct {
  uint32_t n;                    // objects in the batch
  uint32_t has_old;              // 1: header arrays carry 2n rows, rows [n,2n) describe OldObject
  const uint32_t* flags;         // [n or 2n]
  const uint32_t* kind_sid;      // [..]
  const uint32_t* group_sid;
  const uint32_t* nsn_off;       // [rows+1] namespace NAME used by namespaces/excludedNamespaces (match.go:118-179); valid with GK_F_NSNAME
  const uint8_t* nsn_bytes;
  const uint32_t* name_off;      // [rows+1] metadata.name bytes
  const uint8_t* name_bytes;
  const uint32_t* gen_off;       // [rows+1] metadata.generateName bytes
  const uint8_t* gen_bytes;
  const uint32_t* lbl_off;       // [rows+1]
  const uint32_t* lbl_kv;        // 2 * nlabels: (key sid, value sid)
  const uint32_t* nsrow;         // [n] row in the namespace table or GK_NONE   (shared by obj and old)
  const uint32_t* nsl_off;       // namespace table: [nsrows+1]
  const uint32_t* nsl_kv;
  // interned-string dictionary (engine-global, append-only): bytes of sid i are dict_bytes[dict_off[i], dict_off[i+1])
  const uint32_t* dict_off;
  const uint8_t* dict_bytes;
  uint32_t dict_n;
  const GkColumn* cols;
  const GkScope* scopes;
  uint32_t ncols, nscopes;
  // [nscopes] the type words of every scope (gk_tw_layout, eval_layout.h): tw[s][row * W_s + w], null for a scope without them.
  // A derived copy of the VT columns, made where the batch becomes resident; only the generated kernel's rows read it.
  const uint32_t* const* tw;
} GkBatch;

// ---- type words: the VT values of one row of a scope, 4 bits each (GK_VT_* < 16), 8 per 32-bit word.  A row's words are one
// aligned load where its VT columns are one byte load each.  Nibble k of a row is the k-th VT column of the scope in column order;
// its value is (tw[row * W + k / 8] >> 4 * (k % 8)) & 15.  gk_tw_layout (eval_layout.h) decides which scopes have them.
#define GK_TW_MIN 4u   /* VT columns a scope needs for type words: below that its byte loads cost no more */
// words per row of a scope with nvt VT columns: none below GK_TW_MIN, else ceil(nvt / 8) rounded up to 1, 2 or a multiple of 4,
// so that a row is one 4- or 8-byte load or whole 16-byte loads
GK_HD uint32_t gk_tw_words(uint32_t nvt) {
  const uint32_t w = (nvt + 7u) / 8u;
  return nvt < GK_TW_MIN ? 0u : w <= 2u ? w : (w + 3u) & ~3u;
}
// one row of one scope: its nvt VT columns (column indices in nibble order) into its W words
GK_HD void gk_tw_pack_row(const GkColumn* cols, const uint32_t* vtcols, uint32_t nvt, uint32_t W, size_t row, uint32_t* dst) {
  for (uint32_t w = 0; w < W; ++w) {
    uint32_t x = 0u;
    for (uint32_t k = 8u * w; k < nvt && k < 8u * w + 8u; ++k) x |= ((uint32_t)GK_LD(cols[vtcols[k]].vt + row) & 15u) << (4u * (k & 7u));
    dst[(size_t)row * W + w] = x;
  }
}

// ---- match block
enum { GK_M_HAS_MATCH = 1, GK_M_SCOPE_CLUSTER = 2, GK_M_SCOPE_NAMESPACED = 4, GK_M_HAS_LSEL = 8, GK_M_HAS_NSSEL = 16,
       GK_M_LSEL_INVALID = 32, GK_M_NSSEL_INVALID = 64, GK_M_SRC_INVALID = 128, GK_M_HAS_NAME = 256,
       GK_M_SRC_SHIFT = 12 /* 3 bits: GK_SRC_* of the matcher (EMPTY => All) */ };
enum { GK_W_EXACT = 0, GK_W_PREFIX = 1, GK_W_SUFFIX = 2, GK_W_CONTAINS = 3 };
enum { GK_SEL_IN = 0, GK_SEL_NOTIN = 1, GK_SEL_EXISTS = 2, GK_SEL_NOTEXISTS = 3 };

// error codes written to the error list (host renders the reference's error text from them)
enum { GK_E_NONE = 0, GK_E_LSEL_INVALID = 1, GK_E_NSSEL_INVALID = 2, GK_E_NS_MISSING = 3, GK_E_SRC_INVALID_MATCH = 4,
       GK_E_SRC_UNSPECIFIED = 5, GK_E_SRC_INVALID_OBJ = 6, GK_E_NO_OBJECT = 7, GK_E_NUM_RANGE = 8,
       GK_E_FROM_OLD = 256 /* added to the code when the failing object was OldObject */ };

typedef struct {
  uint32_t flags;
  uint32_t kinds_off, kinds_n;    // pool: per entry [nk, ng, wild(bit0 kind '*', bit1 group '*'), nk kind sids, ng group sids]
  uint32_t ns_off, ns_n;          // pool: per pattern [mode, byte_off, len]
  uint32_t exns_off, exns_n;
  uint32_t lsel_off, lsel_n;      // pool: per requirement [key sid, op, nvals, vals...]
  uint32_t nssel_off, nssel_n;
  uint32_t name_mode, name_boff, name_len;
  uint32_t pad0, pad1;
} GkMatch;

// ---- the constraint netlist.
// ALL constraints are compiled jointly into one DAG whose nodes are BIT COLUMNS: one bit per object (root
// level) or per iterated element (scope level).  A CTA owns a tile of consecutive objects; every node of the
// tile lives in shared memory as packed 32-bit words (32 rows per word):
//   ATOM   column value <op> constant          one bit per row, assembled with warp ballots (coalesced loads)
//   GATE   AND/OR of two columns (negations folded into flags)   bitwise on words: 32 rows per instruction
//   BCAST  parent-level column -> child-level rows   (loop-invariant sub-formulas hoisted out of an EXISTS)
//   ACC    EXISTS: child-level column -> parent level by OR over each parent's CSR child range
//   MATCH  the spec.match pre-filter of one DISTINCT match block -> match column + error column
//   OUT    constraint result = program column AND match column -> result area, per-constraint totals
// Ops are sorted into dependency phases; inside a phase the warps of the CTA pull work items (an op, or a row
// slice of a heavy op) from a shared counter; a __syncthreads separates phases.  Identical sub-formulas of
// different constraints are one node.
typedef struct {
  uint32_t w0;   // kind | level<<8 | out_slot<<16     (level = scope id of the rows the op iterates)
  uint32_t w1;
  uint32_t w2;
  uint32_t w3;
} GkOp;

enum {
  GK_N_END = 0,
  GK_N_PHASE = 1,   // (unused marker)
  GK_N_ATOM = 2,    // w1 = atom op | col<<8 ; w2, w3 = operands (see GK_OP_*)
  GK_N_GATE = 3,    // n-ary: pool[w1 .. w1+w3) = input slots (bit 31: negate that input); w2 = flags: 1 OR (else AND), 8 negate out
  GK_N_CONST = 4,   // w1 = 0 / 1
  GK_N_BCAST = 5,   // level = child scope; pool[w1 .. w1+w3) = (input slot at the parent level | output slot << 16)
  GK_N_ACC = 6,     // level = child scope; pool[w1 .. w1+w3) = (input slot at the child level | output slot at the parent level << 16)
  GK_N_MATCH = 7,   // w1 = error-column slot ; w2 = match block id
  GK_N_ACC2 = 9,    // like ACC, but "at least TWO children have the bit" (the audit's ambiguity netlist: may a pair have > 1 result?)
  GK_N_ATOMS = 8,   // every atom of ONE column (same phase): w1 = col<<8 ; pool[w2 ..]: w3 entries of GK_ATOMS_ENT words
                    //   [atom op | out_slot<<16, operand a, operand b, 0] -- the column is loaded once per row for all of them
};
#define GK_ATOMS_ENT 4

// per constraint: where its result comes from.  After the last phase one pass over the tile's objects gathers bit c of
// every constraint into the object-major bitmap words and writes them straight to HBM (coalesced).
typedef struct {
  uint16_t prog_slot, match_slot, err_slot;
  uint16_t flags;            // 1 = program is constant TRUE, 2 = constant FALSE (prog_slot ignored)
} GkOutEnt;

// atom ops (w1 low byte of an ATOM)
enum {
  GK_OP_TRUTHY = 1,     // vt != undef && vt != false
  GK_OP_DEFINED = 2,    // vt != undef
  GK_OP_VTMASK = 3,     // (1 << vt) & w2
  GK_OP_SID_EQ = 4,     // sid == w2
  GK_OP_SID_IN = 5,     // sid in pool[w2 .. w2+w3) (sorted)
  GK_OP_NUM_CMP = 6,    // w3 = GK_CMP_*; i64 constant at pool[w2], pool[w2+1] (lo, hi); OPA cross-type ordering
  GK_OP_PREFIX = 7,     // (lowered as ANYPREFIX with one entry)
  GK_OP_SUFFIX = 8,
  GK_OP_CONTAINS = 9,
  GK_OP_ANYPREFIX = 10, // pool[w2 ..]: w3 entries of GK_PREFIX_ENT words [len, byte_off, 8 words = first 32 bytes, 8 byte-mask words]
  GK_OP_ANYSUFFIX = 11, // pool[w2 ..]: w3 entries of [byte_off, len]
};
enum { GK_CMP_LT = 0, GK_CMP_LE = 1, GK_CMP_GT = 2, GK_CMP_GE = 3, GK_CMP_EQ = 4, GK_CMP_NE = 5 };
enum { GK_G_OR = 1, GK_G_NEG_A = 2, GK_G_NEG_B = 4, GK_G_NEG_OUT = 8 };

typedef struct {
  uint32_t nconstraints;
  uint32_t nmatch;
  uint32_t nops;
  uint32_t nslots;
  uint32_t npool;
  uint32_t ncbytes;
  uint32_t nphases;
  uint32_t nitems;
  const GkOp* ops;           // [nops]
  const uint32_t* items;     // [nitems] work items: op index | part<<20 | nparts<<26, heaviest first inside a phase
  const uint32_t* phase_off; // [nphases + 1] item ranges of the phases
  const GkOutEnt* outs;      // [nconstraints]
  const uint8_t* slot_level; // [nslots] scope id of each slot
  const uint32_t* cons_match;// [nconstraints] match block id
  const GkMatch* match;      // [nmatch]
  const uint32_t* pool;      // u32 constant pool
  const uint8_t* cbytes;     // constant byte strings (wildcard literals, prefixes)
} GkProgram;

typedef struct {
  uint32_t* viol;            // [n * words]   bit c%32 of word c/32 set: object violates constraint c
  uint32_t* err;             // [n * words]   matcher error ("autoreject") plane
  unsigned long long* totals;     // [nconstraints] violating pairs
  unsigned long long* err_totals; // [nconstraints]
  uint32_t* errlist;         // [errcap * 3]  (object, match block, code)
  uint32_t* errcount;        // [1]
  uint32_t errcap;
  uint32_t words;            // ceil(nconstraints / 32)
} GkOut;

// ---- launch parameters shared by the netlist interpreter (tile_kernel.cuh: gk_eval_kernel) and the kernel generated for one
// constraint set (spec_codegen.cpp: gk_spec_kernel, compiled at run time by NVRTC)
#define GK_MAX_PEERS 8
typedef struct {
  GkBatch batch;
  GkProgram prog;
  GkOut out;
  const uint32_t* active;     // [nconstraints] enforcement-point filter
  const uint32_t* tile_lo;    // [(ntiles + 1) * nscopes] first row of every scope for every tile (row ranges are contiguous)
  uint32_t ntiles;
  uint32_t tile;              // objects per tile (multiple of 32)
  uint32_t slot_words;        // words in the slot area
  // Fused exchange (multi-GPU sweep): with npeers > 0 the gather epilogue stores every bitmap word straight into each
  // peer's receive buffer over NVLink (peer_viol[q] already points at THIS rank's shard inside peer q's buffer), and the
  // last CTA to finish publishes the per-constraint totals the same way.  A device-side barrier on the caller's stream
  // then replaces the all-gather collective.
  uint32_t* peer_viol[GK_MAX_PEERS];
  unsigned long long* peer_tot[GK_MAX_PEERS];   // [2 * tot_stride]: violations, then matcher errors
  uint32_t npeers;
  uint32_t tot_stride;
  uint32_t* done_ctr;
  uint32_t done_target;       // CTAs that count themselves in done_ctr: the last of them publishes (every CTA of both kernels
                              // when the generated kernel and the interpreter's units run side by side)
  unsigned long long* timing; // GK_PHASE_TIMING builds: [kMaxPhases + 2][2] = (CTA cycles between barriers, summed warp busy cycles)
  // Hand-over list.  gk_spec_kernel keeps one mask word per netlist node and object, so an object may have at most 32 rows in a
  // scope.  gk_spec_plan_kernel finds those wide objects from the CSR offsets alone, before any row is evaluated: a tile with up
  // to GK_HANDOVER_MAX of them appends each as a unit (object, 1); a tile with more appends itself whole, (first object,
  // objects), and sets its whole flag.  gk_eval_kernel with list_mode = 1 evaluates exactly those units, while gk_spec_kernel
  // does every other object and stores nothing for the units' objects.
  uint32_t* units;            // [2 * unit capacity]: (first object, objects) pairs, each inside one tile
  uint32_t* unit_count;
  uint32_t* whole;            // [ntiles]: 1 = the tile is one unit of the list
  uint32_t list_mode;
} GkKParams;
#ifdef __CUDACC__
// Fused exchange, the end of a CTA whose totals are in p.out: the last of the done_target CTAs to arrive (of whichever kernel)
// sees every contribution and publishes the totals to all peers.  No CTA waits for another.  `s_last`: one word of shared memory.
__device__ __forceinline__ void gk_publish_totals(const GkKParams& p, uint32_t nconstraints, volatile uint32_t* s_last) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) *s_last = atomicAdd(p.done_ctr, 1u) == p.done_target - 1u ? 1u : 0u;
  __syncthreads();
  if (*s_last) {
    __threadfence();
    for (uint32_t c = threadIdx.x; c < nconstraints; c += blockDim.x) {
      const unsigned long long tv = atomicAdd(p.out.totals + c, 0ull), te = atomicAdd(p.out.err_totals + c, 0ull);
      for (uint32_t q = 0; q < p.npeers; ++q) {
        p.peer_tot[q][c] = tv;
        p.peer_tot[q][p.tot_stride + c] = te;
      }
    }
    __threadfence_system();
  }
}
#endif
// More wide objects than this in one tile hand the whole tile over.  A one-object unit pays the interpreter's per-phase barriers and
// latencies for 1/512 of a tile's work.  Measured on an H100 over 1 M config-2 Pods with a wide object every 512 / 256 / 128 / 100
// objects (1, 2, 4, ~5 per tile), one by one against whole tiles: 0.58 / 0.89 / 1.43 / 1.72 ms against 1.35 / 1.43 / 1.48 / 1.47.
// So up to 4 go one by one.  (Defined from outside only to measure another value: tools/spec_probe.py --handover; 0 is the
// whole-tile hand-over alone.)
#ifndef GK_HANDOVER_MAX
#define GK_HANDOVER_MAX 4u
#endif
