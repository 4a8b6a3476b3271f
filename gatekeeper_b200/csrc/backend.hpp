// Execution backend interface.  The product library links exactly one implementation: the CUDA backend
// (kernels.cu).  tests/_hostemu links the CPU emulation of the same per-object core (vm_core.h) so the
// lowering/flattening logic can be unit-tested in a container without a GPU; it is never part of the
// product library and the product has no CPU fallback.
#pragma once
#include <atomic>
#include <thread>
#include <cstdint>
#include <cstring>
#include <functional>
#include <memory>
#include <new>
#include <utility>
#include <string>
#include <unordered_map>
#include <vector>

#include "engine.hpp"
#include "fold_core.h"
#include "program.h"

namespace gk {

struct BackendError {
  std::string msg;
};

// Result bitmaps land in page-locked host memory when the backend has any (the CUDA backend installs the hooks): a device->host
// copy into pageable memory runs at a fraction of the link rate.  Blocks are recycled through a small size-bucketed pool
// (page-locking is expensive: ~1 ms per 8 MB).
struct HostBlockHooks {
  void* (*alloc)(size_t) = nullptr;   // null: plain malloc / free
  void (*release)(void*) = nullptr;
};
HostBlockHooks& host_block_hooks();
void* host_block_take(size_t bytes);
void host_block_give(void* p, size_t bytes);
template <class T>
struct HostBlockAlloc {
  using value_type = T;
  HostBlockAlloc() = default;
  template <class U>
  HostBlockAlloc(const HostBlockAlloc<U>&) {}
  T* allocate(size_t n) { return static_cast<T*>(host_block_take(n * sizeof(T))); }
  void deallocate(T* p, size_t n) { host_block_give(p, n * sizeof(T)); }
  template <class U>
  void construct(U* p) noexcept { ::new (static_cast<void*>(p)) U; }   // resize() leaves the words unset: the copy-back overwrites all of them
  template <class U, class... A>
  void construct(U* p, A&&... a) { ::new (static_cast<void*>(p)) U(std::forward<A>(a)...); }
  template <class U>
  bool operator==(const HostBlockAlloc<U>&) const { return true; }
  template <class U>
  bool operator!=(const HostBlockAlloc<U>&) const { return false; }
};
using BitPlane = std::vector<uint32_t, HostBlockAlloc<uint32_t>>;

struct EvalOut {
  uint32_t n = 0, nconstraints = 0, words = 0;
  BitPlane viol, err;                       // [n * words]  (filled when copy_back)
  std::vector<uint64_t> totals, err_totals; // [nconstraints]
  std::vector<uint32_t> errlist;            // triples (object, constraint, code)
  float kernel_ms = 0.f;
  uint64_t launches = 0;
};

struct DevOutPtrs {          // caller-owned device buffers (e.g. torch tensors) -- used by the multi-GPU path
  void* viol = nullptr;      // u32 [n * words]
  void* err = nullptr;       // u32 [n * words]
  void* totals = nullptr;    // u64 [nconstraints]
  void* err_totals = nullptr;
  void* stream = nullptr;    // cudaStream_t
  // fused exchange: device addresses, on every peer GPU, of the place THIS rank's bitmap shard / totals go
  uint64_t peer_viol[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  uint64_t peer_tot[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  uint32_t npeers = 0, tot_stride = 0;
  uint32_t rank = 0;         // which of the peers this rank is (its own slot holds its unfolded rows: Backend::fold_into)
};

// What orders audit results besides the message: group / version / kind, namespace, name (pkg/audit/manager.go:161-202).  Read
// back from the batch's header arrays; `uniform_gvk`: every object that was not skipped has the same apiVersion and kind.
struct BatchIdentity {
  bool uniform_gvk = false;
  std::vector<uint32_t> flags, ns_off, name_off;
  std::vector<uint8_t> ns_bytes, name_bytes;
};

// The ranking of one audit_candidates call, kept for audit_resultants: rank[o], the rank of object o's identity (equal identities share
// one), and thr[c], the rank of constraint c's limit-th flagged object (~0u: fewer than `limit` are flagged).  The CUDA backend keeps
// both on the device, in `dev`; the host default keeps them in the vectors.
struct AuditRanks {
  std::vector<uint32_t> rank, thr;
  std::shared_ptr<void> dev;
};

// An expanded batch's resultants as the audit sorts their pairs (fold_core.h gk_classify_resultant).
struct ResultantSplit {
  std::vector<uint64_t> counted;   // [classes * nconstraints] pairs counted, per action class (ResultantClasses::cls) and constraint
  std::vector<uint32_t> render;    // the pairs to render, (resultant, constraint | is_err << 31) each, in no particular order
};
struct ResultantClasses {
  const uint8_t* single = nullptr;   // [nconstraints] Compiled::single_result
  const uint8_t* cls = nullptr;      // [resultants] action class: 0 = the constraint's own action, k = the k-th template override
  uint32_t classes = 1, nconstraints = 0, parents = 0;
  const uint8_t* dead = nullptr;     // [parents] 1: the parent's own review failed, its resultants take no part (null: none)
};

class Backend {
 public:
  virtual ~Backend() {}
  virtual const char* name() const = 0;
  // which kernel decided the last evaluation: "gk_spec_kernel" (generated for the constraint set, spec_codegen.hpp) or "gk_eval_kernel"
  virtual const char* last_kernel() const { return "gk_eval_kernel"; }
  virtual void set_program(const Compiled& c) = 0;                       // upload tables when the version changed
  virtual void sync_strings(const StringTable& st) = 0;                  // (re)upload the dictionary if it grew
  virtual void* upload(const HostBatch& hb, const Compiled& c, double* h2d_ms, uint64_t* h2d_bytes) = 0;
  virtual void release(void* batch) = 0;
  virtual void eval(void* batch, const std::vector<uint32_t>& active, EvalOut& out, bool copy_back) = 0;
  virtual void eval_into(void* batch, const std::vector<uint32_t>& active, const DevOutPtrs& dst) = 0;
  // Device ingest (ingest_core.h): raw JSON blob -> resident columnar batch without a host parse.  `status` receives one
  // GK_ING_* code per object (the caller renders the error text of the rare non-OK ones with the host parser).
  virtual void* ingest(const IngestReq& rq, IngestStats* st, std::vector<uint32_t>* status) = 0;
  // Keeping a page's source for a refresh after a constraint change (gk_batch_refresh, GK_F_KEEP_SOURCE).  ingest_keep() is ingest()
  // that also hands the caller the page's source in *keep; reextract() builds a new batch from it for the program of rq.c without
  // reading the caller's page (rq.blob / rq.ooff are not read) -- `status` (may be null) receives its objects' GK_ING_* codes;
  // release_source() frees it.  The CUDA backend keeps the page's device
  // JSON, offsets and token tape and re-runs only the extraction passes.  These defaults, for a backend whose pages do not stay on a
  // device (the test-only host emulation), keep a host copy of the page and ingest it again.
  virtual void* ingest_keep(const IngestReq& rq, IngestStats* st, std::vector<uint32_t>* status, void** keep);
  virtual void* reextract(void* source, const IngestReq& rq, IngestStats* st, std::vector<uint32_t>* status);
  virtual void release_source(void* source);
  // A new page source for gk_batch_patch: objects `keep` of `source` (ascending, each at most once), then the n_add documents of
  // blob / ooff (object k at blob[ooff[k], ooff[k+1])), as a source kept by ingest_keep() of that page would be.  `source` stays
  // as it was; the caller's page is not read after the call.  The CUDA backend moves the staying objects' JSON and token tape on the
  // device and copies and tokenises only the added documents; this default concatenates host copies.
  virtual void* patch_source(void* source, const std::vector<uint32_t>& keep, const uint8_t* blob, const unsigned long long* ooff, size_t n_add,
                             IngestStats* st);
  // The JSON of objects `idx` of a kept page source, back to back into `bytes`, object k at [off[k], off[k+1]) (an expanded batch's
  // refresh, which does not read the caller's page).  The CUDA backend gathers them from the page's device copy.
  virtual void source_bytes(void* source, const std::vector<uint32_t>& idx, std::string& bytes, std::vector<uint64_t>& off);
  virtual void identity(void* batch, BatchIdentity& out) = 0;
  // The audit's candidates of a reviewed batch for any mix of kinds (gk_audit_add_batch_ordered).  Objects are ordered by (group,
  // version, kind, namespace, name) as sv_less orders results (namespace and name as BatchIdentity holds them); for constraint c the
  // candidates are the objects whose bit c is set in `viol` [n * words] and whose identity is at or below the `limit`-th smallest
  // such identity, ties included (all of them when fewer than `limit` are set).  `cand` receives that bitmap [n * words].  `gvk_of`
  // decodes the (group, version, kind) of one object from its JSON: the backend asks for one object of each distinct apiVersion /
  // kind it holds.  The CUDA backend ranks and selects on the device; this default does it on the host from identity().  `keep` (may be
  // null) receives the ranking for audit_resultants.
  using GvkOf = std::function<void(uint32_t object, std::string& group, std::string& version, std::string& kind)>;
  virtual void audit_candidates(void* batch, const uint32_t* viol, uint32_t words, uint32_t nconstraints, uint32_t limit, const GvkOf& gvk_of,
                                std::vector<uint32_t>& cand, float* device_ms, AuditRanks* keep = nullptr);
  // The audit of an expanded batch's resultants against their parents' ranking `ranks` (audit_candidates of the parent batch): pair
  // (r, c) is counted when it is a violation with one result (`cls.single`, or a clear bit of the ambiguity plane) and r's parent p
  // is above c's threshold (rank[p] > thr[c]); every other flagged pair is listed in `out.render`.  `res` is the resultant batch as
  // its last eval() left it, `amb` its ambiguity fork as its last eval() left it (may be null), with the CSR (par, off) of set_parents.
  // The CUDA backend reads the planes the evaluations left on the device; this default reads the host planes of `rev` / `ramb`.
  virtual void audit_resultants(void* res, void* amb, const EvalOut& rev, const EvalOut* ramb, const std::vector<uint32_t>& par,
                                const std::vector<uint32_t>& off, const AuditRanks& ranks, const ResultantClasses& cls, ResultantSplit& out,
                                float* device_ms);
  // ---- expanded batches (GK_F_EXPAND, gk_engine.h).  The defaults run on the host: for a backend whose batches are host memory and
  // whose "device" output buffers are host memory too (the test-only host emulation).
  // Generator selection: the objects of `batch` that may have resultants, ascending, into `sel`: those whose (group, version, kind)
  // -- decoded by `gvk_of` -- `wanted` keeps.  `kinds`: how many distinct kinds were decoded.  The CUDA backend decodes one object per
  // distinct apiVersion / kind hash of the batch, marks and compacts the objects on the device, and selects every object without a
  // hash (skipped by the excluder, no object, the old object of a DELETE) as well; this default decodes every object.
  using GvkWanted = std::function<bool(const std::string& group, const std::string& version, const std::string& kind)>;
  virtual void select_generators(void* batch, const GvkOf& gvk_of, const GvkWanted& wanted, std::vector<uint32_t>& sel, uint32_t* kinds,
                                 float* device_ms);
  // The parents of resultant batch `res`, a CSR over the parents that have resultants: par[j] has resultants off[j] .. off[j+1]-1.
  // The same vectors are passed to eval_expanded / fold_into; a backend that keeps its own copy (the CUDA backend: in device memory)
  // takes it here.  The default keeps nothing.
  virtual void set_parents(void* res, const std::vector<uint32_t>& par, const std::vector<uint32_t>& off) { (void)res, (void)par, (void)off; }
  // gk_batch_eval of an expanded batch: `batch`, then its resultant batch `res`, then every resultant's rows ORed into its parent's;
  // `out` receives the folded planes (when copy_back), the parents' matcher-error list, and totals / kernel time that include the
  // resultants and the fold.  `own` (may be null): the parents' unfolded planes; `rout` (may be null): the resultants' evaluation.
  virtual void eval_expanded(void* batch, void* res, const std::vector<uint32_t>& par, const std::vector<uint32_t>& off,
                             const std::vector<uint32_t>& active, EvalOut& out, bool copy_back, EvalOut* own, EvalOut* rout);
  // After eval_into(batch, active, dst): evaluates `res` into its own planes and folds them into every destination of `dst` (the
  // unfolded rows are read from dst.viol, or from this rank's slot dst.peer_viol[dst.rank]; dst.err), on dst.stream, unsynchronised.
  virtual void fold_into(void* res, const std::vector<uint32_t>& par, const std::vector<uint32_t>& off, const std::vector<uint32_t>& active,
                         const DevOutPtrs& dst);
  // A second view of a resident batch for ANOTHER netlist over the same schema (Compiled::amb): shares the columns, owns its
  // own slot-resolved netlist and output planes.  Evaluate it with eval() while the backend holds `other`; release() it before
  // the batch it was forked from.
  virtual void* fork_batch(void* batch, const Compiled& other) = 0;
  // Start moving a blob to the device ahead of its ingest() (copy + tokenise on the copy / front streams, into the idle one of
  // two front buffers) and return at once: the next page of an audit sweep streams in while the current one is being extracted
  // and evaluated.  ingest() of the same (blob, n) picks the prefetched copy up; anything else is ingested from scratch.
  virtual void prefetch(const uint8_t* blob, const unsigned long long* ooff, size_t n) { (void)blob, (void)ooff, (void)n; }
  // page-lock (or release) a caller-owned host buffer so that the blob copy is a direct DMA at link speed
  virtual void pin_host(const void* p, size_t bytes, bool pin) { (void)p, (void)bytes, (void)pin; }
};

Backend* make_backend(int device);   // defined by whichever backend the library links

// the default page source of Backend::ingest_keep: a host copy of the page
struct HostPageCopy {
  std::vector<uint8_t> blob;
  std::vector<unsigned long long> ooff;
};
inline void* Backend::ingest_keep(const IngestReq& rq, IngestStats* st, std::vector<uint32_t>* status, void** keep) {
  auto src = std::make_unique<HostPageCopy>();
  src->blob.assign(rq.blob, rq.blob + rq.ooff[rq.n]);
  src->blob.resize(src->blob.size() + 16, 0);
  src->ooff.assign(rq.ooff, rq.ooff + rq.n + 1);
  void* b = ingest(rq, st, status);
  *keep = src.release();
  return b;
}
inline void* Backend::reextract(void* source, const IngestReq& rq, IngestStats* st, std::vector<uint32_t>* status) {
  auto* src = static_cast<HostPageCopy*>(source);
  if (!src || src->ooff.size() != rq.n + 1) throw BackendError{"device ingest: the kept source is of another page"};
  IngestReq r = rq;
  r.blob = src->blob.data();
  r.ooff = src->ooff.data();
  r.lut_fill = [&rq, src](const GkMiss* m, size_t k, std::vector<GkLutVal>& out) { rq.lut_fill_from(src->blob.data(), m, k, out); };
  std::vector<uint32_t> own;
  return ingest(r, st, status ? status : &own);
}
inline void Backend::release_source(void* source) { delete static_cast<HostPageCopy*>(source); }
inline void* Backend::patch_source(void* source, const std::vector<uint32_t>& keep, const uint8_t* blob, const unsigned long long* ooff, size_t n_add,
                                   IngestStats* st) {
  auto* old = static_cast<HostPageCopy*>(source);
  if (!old) throw BackendError{"kept source: none"};
  auto src = std::make_unique<HostPageCopy>();
  src->ooff.assign(1, 0);
  for (uint32_t i : keep) {
    if ((size_t)i + 1 >= old->ooff.size()) throw BackendError{"kept source: object index out of range"};
    src->blob.insert(src->blob.end(), old->blob.begin() + old->ooff[i], old->blob.begin() + old->ooff[i + 1]);
    src->ooff.push_back(src->blob.size());
  }
  for (size_t k = 0; k < n_add; ++k) {
    src->blob.insert(src->blob.end(), blob + ooff[k], blob + ooff[k + 1]);
    src->ooff.push_back(src->blob.size());
  }
  src->blob.resize(src->blob.size() + 16, 0);
  if (st) *st = IngestStats{};
  return src.release();
}
inline void Backend::source_bytes(void* source, const std::vector<uint32_t>& idx, std::string& bytes, std::vector<uint64_t>& off) {
  auto* src = static_cast<HostPageCopy*>(source);
  bytes.clear();
  off.assign(1, 0);
  for (uint32_t i : idx) {
    if (!src || (size_t)i + 1 >= src->ooff.size()) throw BackendError{"kept source: object index out of range"};
    bytes.append(reinterpret_cast<const char*>(src->blob.data()) + src->ooff[i], (size_t)(src->ooff[i + 1] - src->ooff[i]));
    off.push_back(bytes.size());
  }
}

// the fold of resultant planes `cviol` / `cerr` into parents by the CSR (par, off), on host arrays; the caller fills in the rest
inline GkFoldArgs fold_args_host(const std::vector<uint32_t>& par, const std::vector<uint32_t>& off, const EvalOut& res, uint32_t words,
                                 uint32_t nconstraints) {
  if (off.size() != par.size() + 1) throw BackendError{"fold: the offsets must have one entry more than the parents"};
  if (!off.empty() && (size_t)off.back() * words > res.viol.size()) throw BackendError{"fold: more resultants than the resultant batch holds"};
  GkFoldArgs a{};
  a.par = par.data();
  a.off = off.data();
  a.m = (uint32_t)par.size();
  a.words = words;
  a.nconstraints = nconstraints;
  a.cviol = res.viol.data();
  a.cerr = res.err.data();
  return a;
}

// every parent of `a` in turn (the rule gk_fold_kernel runs one thread per parent), then the totals of the fused exchange
// published to every peer
inline void fold_host(const GkFoldArgs& a) {
  for (uint32_t j = 0; j < a.m; ++j)
    gk_fold_parent(a, j, [&](uint32_t c, uint32_t plane) {
      if (c < a.nconstraints) ++(plane ? a.err_totals : a.totals)[c];
    });
  for (uint32_t q = 0; q < a.npeers; ++q)
    for (uint32_t c = 0; c < a.nconstraints; ++c) {
      a.peer_tot[q][c] = a.totals[c];
      a.peer_tot[q][a.tot_stride + c] = a.err_totals[c];
    }
}

// gk_classify_resultant over every resultant of the CSR (par, off) on host planes; `cand(p, c)`: parent p can still enter constraint c's list
template <class Cand>
inline void classify_resultants_host(const GkResClassArgs& a, const std::vector<uint32_t>& par, const std::vector<uint32_t>& off,
                                     const ResultantClasses& cls, Cand&& cand, ResultantSplit& out) {
  if (off.size() != par.size() + 1) throw BackendError{"audit resultants: the offsets must have one entry more than the parents"};
  const uint32_t C = cls.nconstraints;
  out.counted.assign((size_t)cls.classes * C, 0);
  out.render.clear();
  for (size_t j = 0; j < par.size(); ++j) {
    const uint32_t p = par[j];
    if (cls.dead && cls.dead[p]) continue;
    for (uint32_t r = off[j]; r < off[j + 1]; ++r)
      gk_classify_resultant(
          a, r, [&](uint32_t c) { return cand(p, c); }, [&](uint32_t c) { ++out.counted[(size_t)cls.cls[r] * C + c]; },
          [&](uint32_t c, uint32_t is_err) { out.render.insert(out.render.end(), {r, c | is_err << 31}); });
  }
}

inline void Backend::audit_resultants(void* res, void* amb, const EvalOut& rev, const EvalOut* ramb, const std::vector<uint32_t>& par,
                                      const std::vector<uint32_t>& off, const AuditRanks& ranks, const ResultantClasses& cls, ResultantSplit& out,
                                      float* device_ms) {
  (void)res, (void)amb;
  if (device_ms) *device_ms = 0.f;
  if (!off.empty() && (size_t)off.back() * rev.words > rev.viol.size()) throw BackendError{"audit resultants: more resultants than the planes hold"};
  GkResClassArgs a{};
  a.viol = rev.viol.data();
  a.err = rev.err.data();
  a.amb = ramb ? ramb->viol.data() : nullptr;
  a.single = cls.single;
  a.words = rev.words;
  a.nconstraints = cls.nconstraints;
  classify_resultants_host(a, par, off, cls, [&](uint32_t p, uint32_t c) { return ranks.rank[p] <= ranks.thr[c]; }, out);
}

inline void Backend::select_generators(void* batch, const GvkOf& gvk_of, const GvkWanted& wanted, std::vector<uint32_t>& sel, uint32_t* kinds,
                                       float* device_ms) {
  BatchIdentity id;
  identity(batch, id);
  std::unordered_map<std::string, bool> seen;
  sel.clear();
  for (uint32_t o = 0; o < (uint32_t)id.flags.size(); ++o) {
    std::string g, v, k;
    gvk_of(o, g, v, k);
    auto it = seen.find(g + '\0' + v + '\0' + k);
    if (it == seen.end()) it = seen.emplace(g + '\0' + v + '\0' + k, wanted(g, v, k)).first;
    if (it->second) sel.push_back(o);
  }
  if (kinds) *kinds = (uint32_t)seen.size();
  if (device_ms) *device_ms = 0.f;
}

inline void Backend::eval_expanded(void* batch, void* res, const std::vector<uint32_t>& par, const std::vector<uint32_t>& off,
                                   const std::vector<uint32_t>& active, EvalOut& out, bool copy_back, EvalOut* own, EvalOut* rout) {
  (void)copy_back;   // (the planes are on the host anyway)
  eval(batch, active, out, true);
  EvalOut tmp;
  EvalOut& r = rout ? *rout : tmp;
  eval(res, active, r, true);
  if (own) {
    own->viol = out.viol;
    own->err = out.err;
  }
  const uint32_t C = out.nconstraints;
  GkFoldArgs a = fold_args_host(par, off, r, out.words, C);
  a.sviol = a.dviol = out.viol.data();
  a.serr = a.derr = out.err.data();
  std::vector<unsigned long long> t(2 * (size_t)C + 1, 0);
  a.totals = t.data();
  a.err_totals = t.data() + C;
  fold_host(a);
  for (uint32_t c = 0; c < C; ++c) out.totals[c] += t[c], out.err_totals[c] += t[C + c];
  out.kernel_ms += r.kernel_ms;
}

inline void Backend::fold_into(void* res, const std::vector<uint32_t>& par, const std::vector<uint32_t>& off, const std::vector<uint32_t>& active,
                               const DevOutPtrs& dst) {
  if (dst.npeers > GK_MAX_PEERS || (dst.npeers && dst.rank >= dst.npeers)) throw BackendError{"fold: bad peer addressing"};
  EvalOut r;
  eval(res, active, r, true);
  GkFoldArgs a = fold_args_host(par, off, r, r.words, r.nconstraints);
  a.sviol = dst.npeers ? reinterpret_cast<const uint32_t*>(dst.peer_viol[dst.rank]) : static_cast<const uint32_t*>(dst.viol);
  a.serr = a.derr = static_cast<uint32_t*>(dst.err);
  a.dviol = dst.npeers ? nullptr : static_cast<uint32_t*>(dst.viol);
  a.npeers = dst.npeers;
  a.tot_stride = dst.tot_stride;
  for (uint32_t q = 0; q < dst.npeers; ++q) {
    a.peer_viol[q] = reinterpret_cast<uint32_t*>(dst.peer_viol[q]);
    a.peer_tot[q] = reinterpret_cast<unsigned long long*>(dst.peer_tot[q]);
  }
  a.totals = static_cast<unsigned long long*>(dst.totals);
  a.err_totals = static_cast<unsigned long long*>(dst.err_totals);
  fold_host(a);
}

// ---- arena packing shared by both backends: every array of a HostBatch laid out contiguously
struct PackedBatch {
  std::vector<uint8_t> arena;          // host image
  size_t cols_off = 0, scopes_off = 0; // where the GkColumn[] / GkScope[] tables live in the arena
  GkBatch hdr{};                       // pointers are OFFSETS into the arena until rebased
};

inline size_t gk_align(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// Packing is two steps so that the bytes are copied exactly once, by all host threads, straight into the buffer the
// device copy reads from (pinned memory for the CUDA backend):
//   pack_layout : assigns every array its 256-byte aligned offset in the arena image and records one copy job per array
//   pack_copy   : runs the copy jobs (memcpy, parallel over arrays and over slices of big arrays) into `dst`
struct PackJob {
  const void* src;
  size_t bytes, off;
};
struct PackPlan {
  std::vector<PackJob> jobs;
  std::vector<GkColumn> cols;      // tables that live in the arena themselves (offsets, rebased later)
  std::vector<GkScope> scopes;
  size_t total = 0;
};

template <class T>
inline size_t plan_put(PackPlan& pl, const std::vector<T>& v) {
  size_t off = gk_align(pl.total);
  pl.total = off + std::max<size_t>(v.size() * sizeof(T), 16);
  if (!v.empty()) pl.jobs.push_back({v.data(), v.size() * sizeof(T), off});
  return off;
}

inline void pack_layout(const HostBatch& hb, const Compiled& c, PackedBatch& pb, PackPlan& pl) {
  GkBatch& h = pb.hdr;
  memset(&h, 0, sizeof h);
  h.n = hb.n;
  h.has_old = hb.has_old ? 1 : 0;
#define PUT(field, vec) h.field = reinterpret_cast<decltype(h.field)>(plan_put(pl, vec))
  PUT(flags, hb.flags);
  PUT(kind_sid, hb.kind_sid);
  PUT(group_sid, hb.group_sid);
  PUT(nsn_off, hb.nsn_off);
  PUT(nsn_bytes, hb.nsn_bytes);
  PUT(name_off, hb.name_off);
  PUT(name_bytes, hb.name_bytes);
  PUT(gen_off, hb.gen_off);
  PUT(gen_bytes, hb.gen_bytes);
  PUT(lbl_off, hb.lbl_off);
  PUT(lbl_kv, hb.lbl_kv);
  PUT(nsrow, hb.nsrow);
  PUT(nsl_off, hb.nsl_off);
  PUT(nsl_kv, hb.nsl_kv);
#undef PUT
  pl.cols.resize(hb.cols.size());
  for (size_t i = 0; i < hb.cols.size(); ++i) {
    GkColumn& g = pl.cols[i];
    memset(&g, 0, sizeof g);
    g.scope = c.schema.cols[i].scope;
    g.enc = c.schema.cols[i].enc;
    g.vt = reinterpret_cast<const uint8_t*>(plan_put(pl, hb.cols[i].vt));
    g.sid = reinterpret_cast<const uint32_t*>(plan_put(pl, hb.cols[i].sid));
    g.num = reinterpret_cast<const int64_t*>(plan_put(pl, hb.cols[i].num));
    g.boff = reinterpret_cast<const uint32_t*>(plan_put(pl, hb.cols[i].boff));
    g.bytes = reinterpret_cast<const uint8_t*>(plan_put(pl, hb.cols[i].bytes));
    g.head = reinterpret_cast<const uint32_t*>(plan_put(pl, hb.cols[i].head));
  }
  pl.scopes.resize(hb.scope_off.size());
  for (size_t s = 0; s < pl.scopes.size(); ++s) {
    memset(&pl.scopes[s], 0, sizeof(GkScope));
    pl.scopes[s].parent = c.schema.scopes[s].parent;
    pl.scopes[s].rows = hb.scope_rows[s];
    pl.scopes[s].off = reinterpret_cast<const uint32_t*>(plan_put(pl, hb.scope_off[s]));
  }
  pb.cols_off = plan_put(pl, pl.cols);
  pb.scopes_off = plan_put(pl, pl.scopes);
  h.cols = reinterpret_cast<const GkColumn*>(pb.cols_off);
  h.scopes = reinterpret_cast<const GkScope*>(pb.scopes_off);
  h.ncols = (uint32_t)pl.cols.size();
  h.nscopes = (uint32_t)pl.scopes.size();
  pl.total = gk_align(pl.total);
}

inline void pack_copy(const PackPlan& pl, uint8_t* dst, int threads) {
  // slice big arrays so that the work spreads evenly
  struct Piece {
    const uint8_t* src;
    uint8_t* dst;
    size_t bytes;
  };
  std::vector<Piece> pieces;
  const size_t kSlice = 4u << 20;
  for (auto& j : pl.jobs)
    for (size_t o = 0; o < j.bytes; o += kSlice)
      pieces.push_back({static_cast<const uint8_t*>(j.src) + o, dst + j.off + o, std::min(kSlice, j.bytes - o)});
  const size_t T = std::max<size_t>(1, std::min<size_t>((size_t)std::max(1, threads), pieces.size() / 4 + 1));
  if (T == 1) {
    for (auto& p : pieces) memcpy(p.dst, p.src, p.bytes);
    return;
  }
  std::atomic<size_t> next{0};
  std::vector<std::thread> th;
  for (size_t t = 0; t < T; ++t)
    th.emplace_back([&]() {
      for (;;) {
        size_t i = next.fetch_add(1);
        if (i >= pieces.size()) break;
        memcpy(pieces[i].dst, pieces[i].src, pieces[i].bytes);
      }
    });
  for (auto& x : th) x.join();
}

// one-shot form (host image in pb.arena): used by the test backend
inline void pack_batch(const HostBatch& hb, const Compiled& c, PackedBatch& pb) {
  PackPlan pl;
  pack_layout(hb, c, pb, pl);
  pb.arena.assign(pl.total, 0);
  pack_copy(pl, pb.arena.data(), 1);
}

// turn the arena-relative offsets into pointers valid at `base` (device or host); patches the in-arena tables
inline GkBatch rebase_batch(PackedBatch& pb, uint8_t* host_image, const uint8_t* base) {
  GkBatch h = pb.hdr;
#define RB(f) h.f = reinterpret_cast<decltype(h.f)>(base + reinterpret_cast<size_t>(h.f))
  RB(flags); RB(kind_sid); RB(group_sid); RB(nsn_off); RB(nsn_bytes); RB(name_off); RB(name_bytes); RB(gen_off); RB(gen_bytes);
  RB(lbl_off); RB(lbl_kv); RB(nsrow); RB(nsl_off); RB(nsl_kv); RB(cols); RB(scopes);
#undef RB
  GkColumn* cols = reinterpret_cast<GkColumn*>(host_image + pb.cols_off);
  for (uint32_t i = 0; i < h.ncols; ++i) {
    GkColumn& g = cols[i];
    g.vt = base + reinterpret_cast<size_t>(g.vt);
    g.sid = reinterpret_cast<const uint32_t*>(base + reinterpret_cast<size_t>(g.sid));
    g.num = reinterpret_cast<const int64_t*>(base + reinterpret_cast<size_t>(g.num));
    g.boff = reinterpret_cast<const uint32_t*>(base + reinterpret_cast<size_t>(g.boff));
    g.bytes = base + reinterpret_cast<size_t>(g.bytes);
    g.head = reinterpret_cast<const uint32_t*>(base + reinterpret_cast<size_t>(g.head));
  }
  GkScope* scopes = reinterpret_cast<GkScope*>(host_image + pb.scopes_off);
  for (uint32_t s = 0; s < h.nscopes; ++s) scopes[s].off = reinterpret_cast<const uint32_t*>(base + reinterpret_cast<size_t>(scopes[s].off));
  return h;
}

}  // namespace gk
