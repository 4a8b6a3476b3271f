// C ABI (include/gk_engine.h) over Engine + Backend.  No exceptions cross this file's extern "C" surface.
#include <chrono>
#include <condition_variable>
#include <deque>
#include <exception>
#include <mutex>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <thread>
#include <unordered_map>

#include "../../include/gk_engine.h"
#include "backend.hpp"
#include <algorithm>
#include <new>
#include "audit.hpp"
#include "engine.hpp"

// ---- page-locked result blocks (backend.hpp HostBlockAlloc): power-of-two buckets, a few spare blocks per bucket
namespace gk {
HostBlockHooks& host_block_hooks() {
  static HostBlockHooks h;
  return h;
}
namespace {
struct HostBlockPool {
  std::mutex mu;
  std::vector<void*> spare[48];
  static int bucket(size_t bytes) {
    int b = 12;   // 4 KB and up
    while (((size_t)1 << b) < bytes) ++b;
    return b;
  }
} g_block_pool;
}  // namespace
void* host_block_take(size_t bytes) {
  if (bytes == 0) bytes = 1;
  HostBlockHooks& h = host_block_hooks();
  if (!h.alloc || bytes < (1u << 16)) {   // small planes: not worth page-locking
    void* p = malloc(bytes);
    if (!p) throw std::bad_alloc();
    return p;
  }
  const int b = HostBlockPool::bucket(bytes);
  {
    std::lock_guard<std::mutex> l(g_block_pool.mu);
    auto& v = g_block_pool.spare[b];
    if (!v.empty()) {
      void* p = v.back();
      v.pop_back();
      return p;
    }
  }
  void* p = h.alloc((size_t)1 << b);
  if (!p) throw std::bad_alloc();
  return p;
}
void host_block_give(void* p, size_t bytes) {
  if (!p) return;
  if (bytes == 0) bytes = 1;
  HostBlockHooks& h = host_block_hooks();
  if (!h.alloc || bytes < (1u << 16)) {
    free(p);
    return;
  }
  const int b = HostBlockPool::bucket(bytes);
  {
    std::lock_guard<std::mutex> l(g_block_pool.mu);
    auto& v = g_block_pool.spare[b];
    if (v.size() < 8) {
      v.push_back(p);
      return;
    }
  }
  h.release(p);
}
}  // namespace gk

using namespace gk;

struct gk_engine {
  std::unique_ptr<Engine> eng;
  std::unique_ptr<Backend> be;
  std::mutex keys_mu;
  // constraint keys of the last compiled programs: a pointer handed out by gk_constraint_key stays valid until 16 further
  // constraint-set changes have been observed through gk_constraint_count (results carry their own keys: gk_result_constraint_key)
  std::deque<std::shared_ptr<std::vector<std::string>>> key_sets;
  uint64_t keys_version = 0;
  // The backend holds ONE program (the tables of one compiled snapshot).  Reviews of the same snapshot run concurrently; a
  // review that needs another snapshot (constraints changed meanwhile) waits until the ones in flight have finished.
  std::mutex lease_mu;
  std::condition_variable lease_cv;
  uint64_t lease_version = 0;
  int lease_active = 0;
};

namespace {
struct ProgramLease {
  gk_engine* e;
  ProgramLease(gk_engine* eng, const Compiled& c) : e(eng) {
    std::unique_lock<std::mutex> l(e->lease_mu);
    e->lease_cv.wait(l, [&] { return e->lease_active == 0 || e->lease_version == c.version; });
    e->be->set_program(c);   // (a no-op when the backend already holds this version)
    e->lease_version = c.version;
    ++e->lease_active;
  }
  ~ProgramLease() {
    std::lock_guard<std::mutex> l(e->lease_mu);
    if (--e->lease_active == 0) e->lease_cv.notify_all();
  }
  ProgramLease(const ProgramLease&) = delete;
  ProgramLease& operator=(const ProgramLease&) = delete;
};

// Releases a backend handle -- a device batch or a kept page source -- when its owner dies.  No exception leaves it: it runs in
// destructors.
struct BackendRelease {
  Backend* be = nullptr;
  void (Backend::*call)(void*) = nullptr;
  void operator()(void* p) const noexcept {
    try {
      (be->*call)(p);
    } catch (...) {
    }
  }
};
using BackendHandle = std::unique_ptr<void, BackendRelease>;

struct Expanded;   // an expanded batch's resultants (GK_F_EXPAND), below

BackendHandle device_batch(gk_engine* e, void* dev) { return BackendHandle(dev, BackendRelease{e->be.get(), &Backend::release}); }
BackendHandle kept_source(gk_engine* e, void* source) { return BackendHandle(source, BackendRelease{e->be.get(), &Backend::release_source}); }
}  // namespace

// A resident batch.  It owns its device batch and its kept source: both are released with it, through the backend that made them.
struct gk_batch {
  BackendHandle dev;
  std::shared_ptr<const Compiled> compiled;
  std::shared_ptr<HostBatch> host;     // kept for object_errors / alg_bytes (column data is released after upload)
  std::vector<gk_obj> objs;            // shallow copy: the caller keeps the JSON alive while the batch lives
  // a blob batch (device ingest) keeps only the blob and its offsets
  const char* blob = nullptr;
  const uint64_t* blob_off = nullptr;
  uint8_t blob_source = 0;
  uint32_t n = 0;
  uint32_t flags = 0;                  // the upload's flags (the process whose excluder applied): the audit reviews resultants with the same
  uint64_t alg_bytes = 0;
  uint64_t data_version = 0;           // data.inventory as of the flatten (referential snapshots only)
  std::vector<std::string> excluded;   // the excluder patterns of the upload's process the batch was flattened with
  // GK_F_KEEP_SOURCE: the page's source (Backend::ingest_keep -- on the GPU its device JSON, offsets and token tape), and the
  // review-level errors of its objects (they depend on the page alone)
  BackendHandle source;
  std::vector<std::string> source_errors;
  std::shared_ptr<Expanded> ex;        // GK_F_EXPAND: the page's resultants (null: a batch uploaded without the flag)
  ObjIn obj_in(size_t i) const;
  // a page of plain objects of one source (gk_batch_upload_blob): `blob`, or -- once patched (gk_batch_patch) -- `objs`, one span each
  bool plain_page() const { return blob || source; }
};

namespace {

// ---- expansion (pkg/audit/manager.go:733-765, pkg/webhook/policy.go:610-646), the step gk_review_batch, the expanded batches and the
// audit share: the resultants of generator objects are reviewed as generated resources, and their results folded back onto their parents
struct Child {
  uint32_t parent;
  std::string json, tmpl, action;
};

struct Expansion {
  std::vector<Child> children;       // in object order
  std::vector<std::string> errors;   // per object: "" or why its expansion failed
};

// An expanded batch's resultants: a resident batch of their own, in parent order, and what folds them onto their parents
struct Expanded {
  uint64_t version = 0;              // Engine::expansion_version the page was expanded at
  Expansion x;                       // children[k].parent: an object of the parent batch; errors: [parents] or empty
  std::string blob;                  // blob parents: the resultants' JSON as one page ...
  std::vector<uint64_t> off;         // ... and its offsets
  std::vector<gk_obj> objs;          // object parents: the resultants as review objects (their JSON in x.children)
  std::unique_ptr<gk_batch> res;     // null: the page has no resultants
  std::vector<uint32_t> par, off_par;   // its parents, a CSR over the parents that have resultants (Backend::set_parents)
};

struct ResultPriv {
  std::shared_ptr<const Compiled> compiled;   // the snapshot the result was computed with (constraint indices refer to it)
  std::vector<std::string> keys;              // "Kind/name" per constraint index
  EvalOut ev;
  std::vector<Violation> vio;
  std::vector<gk_violation> cvio;
  std::vector<std::string> obj_errors;
  std::vector<const char*> obj_error_ptrs;
};

char* dup_str(const std::string& s) {
  char* p = (char*)malloc(s.size() + 1);
  if (p) memcpy(p, s.c_str(), s.size() + 1);
  return p;
}

template <class F>
int guard(char** err, F&& f) {
  try {
    f();
    return GK_OK;
  } catch (RegoError& e) {
    if (err) *err = dup_str(e.msg);
    return GK_ERR_REGO;
  } catch (BackendError& e) {
    if (err) *err = dup_str(e.msg);
    return GK_ERR_BACKEND;
  } catch (JsonError& e) {
    if (err) *err = dup_str(e.msg);
    return GK_ERR_INVALID;
  } catch (std::exception& e) {
    if (err) *err = dup_str(std::string("internal: ") + e.what());
    return GK_ERR_INTERNAL;
  } catch (...) {
    if (err) *err = dup_str("internal: unknown exception");
    return GK_ERR_INTERNAL;
  }
}

double now_ms() {
  using namespace std::chrono;
  return duration<double, std::milli>(steady_clock::now().time_since_epoch()).count();
}

ObjIn to_in(const gk_obj& o) {
  ObjIn in;
  in.json = o.json;
  in.len = o.len;
  in.old_json = o.old_json;
  in.old_len = o.old_len;
  in.ns_json = o.ns_json;
  in.ns_len = o.ns_len;
  in.ns_name = o.ns_name;
  in.operation = o.operation;
  in.userinfo_json = o.userinfo_json;
  in.userinfo_len = o.userinfo_len;
  in.source = o.source;
  return in;
}

}  // namespace

ObjIn gk_batch::obj_in(size_t i) const {
  if (!blob) return to_in(objs[i]);
  ObjIn in;
  in.json = blob + blob_off[i];
  in.len = (size_t)(blob_off[i + 1] - blob_off[i]);
  in.source = blob_source;
  return in;
}

namespace {

void fill_result(gk_result* out, ResultPriv* rp, bool have_bits) {
  out->n_objects = rp->ev.n;
  out->n_constraints = rp->ev.nconstraints;
  out->words = rp->ev.words;
  out->viol_bits = have_bits && !rp->ev.viol.empty() ? rp->ev.viol.data() : nullptr;
  out->err_bits = have_bits && !rp->ev.err.empty() ? rp->ev.err.data() : nullptr;
  out->totals = rp->ev.totals.data();
  out->err_totals = rp->ev.err_totals.data();
  rp->cvio.clear();
  for (auto& v : rp->vio) {
    gk_violation g;
    g.object = v.object;
    g.constraint = v.constraint;
    g.msg = v.msg.c_str();
    g.details_json = v.details_json.c_str();
    g.enforcement_action = v.action.c_str();
    g.scoped_actions_json = v.scoped_json.c_str();
    g.autoreject = v.autoreject ? 1 : 0;
    rp->cvio.push_back(g);
  }
  out->violations = rp->cvio.data();
  out->n_violations = rp->cvio.size();
  rp->obj_error_ptrs.clear();
  bool any_err = false;
  for (auto& s : rp->obj_errors) any_err = any_err || !s.empty();
  if (any_err)
    for (auto& s : rp->obj_errors) rp->obj_error_ptrs.push_back(s.empty() ? nullptr : s.c_str());
  out->object_errors = any_err ? rp->obj_error_ptrs.data() : nullptr;   // null: no object of the batch has a review-level error
  out->kernel_ms = rp->ev.kernel_ms;
  out->gpu_launches = rp->ev.launches;
  out->priv = rp;
}

// The results of every flagged pair of batch `b`'s rows in `viol` / `err` (its evaluation's matcher-error list `errlist`): matcher errors
// first (autoreject results), then rendered violations, both in (object, constraint) order
std::vector<Violation> render(gk_engine* e, const Compiled& c, const gk_batch& b, const BitPlane& viol, const BitPlane& err, const std::vector<uint32_t>& errlist,
                              uint32_t W, uint32_t C, const std::string& ep) {
  std::vector<Violation> vio;
  std::unordered_map<uint64_t, uint32_t> err_code;
  for (size_t i = 0; i + 2 < errlist.size(); i += 3) err_code[((uint64_t)errlist[i] << 32) | errlist[i + 1]] = errlist[i + 2];
  // one DOM parse per object, all of its flagged constraints rendered from it; objects are spread over the host threads
  const uint32_t n = b.n;
  const size_t T = std::min<size_t>((size_t)std::max(1, e->eng->threads()), std::max<size_t>(1, n / 16));
  std::vector<std::vector<Violation>> part(T);
  std::vector<std::string> errs(T);
  auto work = [&](size_t t) {
    std::vector<Engine::Flagged> flagged;
    Engine::MaterializeCtx mctx;
    try {
      for (uint32_t o = (uint32_t)(n * t / T); o < (uint32_t)(n * (t + 1) / T); ++o) {
        flagged.clear();
        for (uint32_t w = 0; w < W; ++w) {
          const uint32_t vb = viol[(size_t)o * W + w], eb = err[(size_t)o * W + w];
          uint32_t any = vb | eb;
          while (any) {
            const uint32_t k = (uint32_t)__builtin_ctz(any);
            any &= any - 1;
            const uint32_t cix = w * 32 + k;
            if (cix >= C) continue;
            const bool is_err = eb >> k & 1u;
            uint32_t code = 0;
            if (is_err) {
              auto it = err_code.find(((uint64_t)o << 32) | c.cons_match[cix]);   // error list is keyed by match block
              if (it != err_code.end()) code = it->second;
            }
            flagged.push_back({cix, is_err, code});
          }
        }
        if (!flagged.empty()) e->eng->materialize_object(c, b.obj_in(o), o, flagged, ep, part[t], nullptr, &mctx);
      }
    } catch (RegoError& x) {
      errs[t] = x.msg;
    } catch (std::exception& x) {
      errs[t] = x.what();
    }
  };
  if (T == 1) work(0);
  else {
    std::vector<std::thread> th;
    for (size_t t = 0; t < T; ++t) th.emplace_back(work, t);
    for (auto& x : th) x.join();
  }
  for (auto& x : errs)
    if (!x.empty()) throw RegoError{x};
  for (auto& v : part) vio.insert(vio.end(), std::make_move_iterator(v.begin()), std::make_move_iterator(v.end()));
  return vio;
}

// The resultants' results and review-level errors reported on their parents (aggregate.go:19-63): `vio` holds the results of the
// parents 0 .. n-1 and those of resultant k as object n + k, `obj_errors` the review-level errors of the same rows (empty: none).
// Results are re-indexed with "[Implied by <template>]" and the template's enforcement-action override, a resultant's review-level
// error is reported on its parent, and so is a failed expansion (`expand_errors`: per parent, or empty).
void fold_results(std::vector<Violation>& vio, std::vector<std::string>& obj_errors, size_t n, const std::vector<Child>& children,
                  const std::vector<std::string>& expand_errors) {
  for (auto& v : vio)
    if (v.object >= n) {
      const Child& ch = children[v.object - n];
      v.object = ch.parent;
      v.msg = ExpansionSystem::implied_by(ch.tmpl, v.msg);
      if (!ch.action.empty()) v.action = ch.action;   // OverrideEnforcementAction (aggregate.go:47-58) sets EnforcementAction only: the scoped list stays
    }
  std::stable_sort(vio.begin(), vio.end(), [](const Violation& a, const Violation& b2) { return a.object < b2.object; });
  const bool any_expand_err = std::any_of(expand_errors.begin(), expand_errors.end(), [](const std::string& m) { return !m.empty(); });
  if (obj_errors.empty() && any_expand_err) obj_errors.assign(n + children.size(), std::string());
  if (!obj_errors.empty()) {
    for (size_t k = 0; k < children.size(); ++k)
      if (!obj_errors[n + k].empty() && obj_errors[children[k].parent].empty())
        obj_errors[children[k].parent] = ExpansionSystem::implied_by(children[k].tmpl, obj_errors[n + k]);
    obj_errors.resize(n);
    for (size_t i = 0; i < n && i < expand_errors.size(); ++i)
      if (!expand_errors[i].empty() && obj_errors[i].empty()) obj_errors[i] = expand_errors[i];
  }
}

// evaluate a resident batch; optionally render messages for flagged pairs.  An expanded batch: the parents, then the resultants, then
// the fold of the resultants' rows into the parents' rows on the device; the results are rendered from the unfolded rows and folded
// as gk_review_batch folds them.
void eval_batch(gk_engine* e, gk_batch* b, const char* ep_c, uint32_t flags, gk_result* out) {
  std::string ep = ep_c ? ep_c : "";
  const Compiled& c = *b->compiled;
  auto rp = std::make_unique<ResultPriv>();
  rp->compiled = b->compiled;
  for (auto* k : c.order) rp->keys.push_back(k->kind + "/" + k->name);
  std::vector<uint32_t> active;
  e->eng->active_mask(c, ep, active);
  const bool materialize = (flags & GK_F_MATERIALIZE) != 0;
  bool copy_back = !(flags & GK_F_NO_COPY_BACK) || materialize;
  const gk_batch* res = b->ex ? b->ex->res.get() : nullptr;
  double t0 = now_ms();
  EvalOut own, rev;   // the parents' unfolded rows and the resultants' own rows (materialize)
  if (res) e->be->eval_expanded(b->dev.get(), res->dev.get(), b->ex->par, b->ex->off_par, active, rp->ev, copy_back, materialize ? &own : nullptr,
                                materialize ? &rev : nullptr);
  else e->be->eval(b->dev.get(), active, rp->ev, copy_back);
  double t1 = now_ms();
  rp->obj_errors = b->host->obj_errors;
  out->d2h_bytes = copy_back ? (uint64_t)rp->ev.viol.size() * 8 : 0;
  out->d2h_ms = (t1 - t0) - rp->ev.kernel_ms;
  if (out->d2h_ms < 0) out->d2h_ms = 0;
  out->alg_bytes = b->alg_bytes + (uint64_t)(b->n + (res ? res->n : 0)) * rp->ev.words * 8;
  out->materialize_ms = 0;
  if (materialize) {
    double m0 = now_ms();
    const uint32_t W = rp->ev.words, C = rp->ev.nconstraints;
    rp->vio = render(e, c, *b, res ? own.viol : rp->ev.viol, res ? own.err : rp->ev.err, rp->ev.errlist, W, C, ep);
    if (res) {
      std::vector<Violation> rv = render(e, c, *res, rev.viol, rev.err, rev.errlist, W, C, ep);
      for (auto& v : rv) v.object += b->n;
      rp->vio.insert(rp->vio.end(), std::make_move_iterator(rv.begin()), std::make_move_iterator(rv.end()));
    }
    out->materialize_ms = now_ms() - m0;
  }
  if (b->ex) {
    const Expanded& x = *b->ex;
    if (res && !res->host->obj_errors.empty()) {
      rp->obj_errors.resize(b->n);
      rp->obj_errors.insert(rp->obj_errors.end(), res->host->obj_errors.begin(), res->host->obj_errors.end());
      rp->obj_errors.resize((size_t)b->n + x.x.children.size());
    } else if (!rp->obj_errors.empty()) {
      rp->obj_errors.resize((size_t)b->n + x.x.children.size());
    }
    fold_results(rp->vio, rp->obj_errors, b->n, x.x.children, x.x.errors);
  }
  bool give_bits = !(flags & GK_F_NO_COPY_BACK);
  fill_result(out, rp.release(), give_bits);
}

const char* process_of(uint32_t flags) { return flags & GK_F_PROCESS_AUDIT ? "audit" : flags & GK_F_PROCESS_WEBHOOK ? "webhook" : ""; }

// the excluder patterns a batch uploaded with `flags` is flattened with (none without a process flag)
std::vector<std::string> excluded_of(gk_engine* e, uint32_t flags) {
  const std::string process = process_of(flags);
  return process.empty() ? std::vector<std::string>() : e->eng->excluded_namespaces(process);
}

// A resident batch of `n` objects flattened against `c` onto the device batch `dev`: the fields every upload fills, and its
// statistics.  `errors`: the objects' review-level errors (empty: none).
std::unique_ptr<gk_batch> make_batch(gk_engine* e, const std::shared_ptr<const Compiled>& c, BackendHandle dev, uint32_t n, uint32_t flags,
                                     std::vector<std::string> errors, std::vector<std::string> excluded, const IngestStats& ist, double flatten_ms,
                                     gk_result* stats) {
  auto b = std::make_unique<gk_batch>();
  b->dev = std::move(dev);
  b->compiled = c;
  if (c->uses_data) e->eng->data_doc(&b->data_version);
  b->n = n;
  b->flags = flags;
  b->alg_bytes = ist.alg_bytes;
  b->excluded = std::move(excluded);
  // the host column data is not kept; the small per-object error list is
  auto slim = std::make_shared<HostBatch>();
  slim->n = n;
  slim->obj_errors = std::move(errors);
  slim->alg_bytes = ist.alg_bytes;
  b->host = slim;
  if (stats) {
    stats->flatten_ms = flatten_ms;
    stats->h2d_ms = ist.h2d_ms;
    stats->h2d_bytes = ist.h2d_bytes;
    stats->alg_bytes = ist.alg_bytes;
    stats->n_objects = n;
    stats->n_constraints = (uint32_t)c->cons_match.size();
  }
  return b;
}

std::unique_ptr<gk_batch> upload_batch(gk_engine* e, const std::shared_ptr<const Compiled>& c, const gk_obj* objs, size_t n, uint32_t flags,
                                       gk_result* stats) {
  std::vector<std::string> excluded = excluded_of(e, flags);   // (read before the flatten: a later change makes the batch stale, never current)
  std::vector<ObjIn> ins(n);
  for (size_t i = 0; i < n; ++i) ins[i] = to_in(objs[i]);
  double t0 = now_ms();
  auto hb = e->eng->flatten(ins.data(), n, *c, process_of(flags));
  double t1 = now_ms();
  e->be->sync_strings(e->eng->strings());
  IngestStats ist;
  uint64_t h2d_bytes = 0;
  BackendHandle dev = device_batch(e, e->be->upload(*hb, *c, &ist.h2d_ms, &h2d_bytes));
  ist.h2d_bytes = h2d_bytes;
  ist.alg_bytes = hb->alg_bytes;
  auto b = make_batch(e, c, std::move(dev), hb->n, flags, std::move(hb->obj_errors), std::move(excluded), ist, t1 - t0, stats);
  b->objs.assign(objs, objs + n);
  return b;
}

static std::vector<gk_obj> blob_objs(const char* buf, const uint64_t* off, size_t n, uint8_t source) {
  std::vector<gk_obj> v(n);
  for (size_t i = 0; i < n; ++i) {
    memset(&v[i], 0, sizeof(gk_obj));
    v[i].json = buf + off[i];
    v[i].len = (size_t)(off[i + 1] - off[i]);
    v[i].source = source;
  }
  return v;
}

bool device_ingest(const Compiled& c, size_t n) {
  static const bool host_only = getenv("GK_NO_DEVICE_INGEST") != nullptr;
  return c.device_ingest && !host_only && n != 0 && !getenv("GK_NO_DEVICE_INGEST_RUNTIME");   // (the runtime switch is for A/B tests)
}

// the review-level error of an object the device ingest rejected (`status`: its GK_ING_* code), worded by the host parser (bad JSON,
// not an object, kind missing)
std::string ingest_error(gk_engine* e, uint32_t status, const ObjIn& in) {
  std::string err;
  VP doc = e->eng->review_doc(in, nullptr, nullptr, nullptr, &err);
  if (doc && status != GK_ING_NULL) err = "device ingest refused the object (status " + std::to_string(status) + "): JSON nesting deeper than " +
                                          std::to_string(GK_TAPE_MAX_DEPTH) + " levels or a token longer than 128 MiB";
  if (!doc && err.empty()) err = "invalid request object";
  return err;
}

// a blob of plain objects: flattened by the ingest kernels on the device when the compiled snapshot allows it
std::unique_ptr<gk_batch> upload_blob(gk_engine* e, const std::shared_ptr<const Compiled>& c, const char* buf, const uint64_t* off, size_t n, uint8_t source,
                                      uint32_t flags, gk_result* stats) {
  std::unique_ptr<gk_batch> b;
  if (!device_ingest(*c, n)) {
    auto v = blob_objs(buf, off, n, source);
    b = upload_batch(e, c, v.data(), n, flags, stats);   // (kept as a blob too: a later gk_batch_refresh may ingest it on the device)
  } else {
    double t0 = now_ms();
    IngestReq rq = e->eng->ingest_request(c, reinterpret_cast<const uint8_t*>(buf), reinterpret_cast<const unsigned long long*>(off), n, source, process_of(flags));
    IngestStats ist;
    std::vector<uint32_t> status;
    void* kept = nullptr;
    BackendHandle dev = device_batch(e, (flags & GK_F_KEEP_SOURCE) ? e->be->ingest_keep(rq, &ist, &status, &kept) : e->be->ingest(rq, &ist, &status));
    BackendHandle source_kept = kept_source(e, kept);
    std::vector<std::string> errors;
    for (size_t i = 0; i < n; ++i)
      if (status[i] != GK_ING_OK) {
        if (errors.empty()) errors.assign(n, std::string());   // (left empty when every object is fine)
        ObjIn in;
        in.json = buf + off[i];
        in.len = (size_t)(off[i + 1] - off[i]);
        in.source = source;
        errors[i] = ingest_error(e, status[i], in);
      }
    b = make_batch(e, c, std::move(dev), (uint32_t)n, flags, errors, std::move(rq.excluded), ist, (now_ms() - t0) - ist.h2d_ms, stats);
    if (source_kept) {
      b->source = std::move(source_kept);
      b->source_errors = std::move(errors);
    }
  }
  b->blob = buf;
  b->blob_off = off;
  b->blob_source = source;
  return b;
}

// gk_batch_refresh of a batch that kept its source, for a snapshot flattened on the device: the extraction passes again, from the
// page's token tape in HBM -- no copy, no tokeniser, and the caller's blob is not read
std::unique_ptr<gk_batch> refresh_from_source(gk_engine* e, const std::shared_ptr<const Compiled>& c, const gk_batch& old, gk_result* stats) {
  double t0 = now_ms();
  IngestReq rq = e->eng->ingest_request(c, nullptr, nullptr, old.n, old.blob_source, process_of(old.flags));
  IngestStats ist;
  BackendHandle dev = device_batch(e, e->be->reextract(old.source.get(), rq, &ist, nullptr));
  auto b = make_batch(e, c, std::move(dev), old.n, old.flags, old.source_errors, std::move(rq.excluded), ist, (now_ms() - t0) - ist.h2d_ms, stats);
  b->objs = old.objs;
  b->blob = old.blob;
  b->blob_off = old.blob_off;
  b->blob_source = old.blob_source;
  return b;
}

// the bitmap-only calls: they would leave out the resultants of generator objects, silently
void refuse_while_expanding(gk_engine* e) {
  if (e->eng->has_expansion())
    throw RegoError{"ExpansionTemplates are registered: this entry point does not expand generator objects -- review them through gk_review_batch, or "
                    "aggregate the batch with gk_audit_add_batch, which do"};
}

// why batch `b` is stale against snapshot `c` (null: it is current)
const char* stale_reason(gk_engine* e, const Compiled& c, const gk_batch& b) {
  if (c.version != b.compiled->version) return "batch was flattened against an older constraint set; upload it again";
  if (c.uses_data) {   // the columns of a referential snapshot hold values computed from data.inventory
    uint64_t dv = 0;
    e->eng->data_doc(&dv);
    if (dv != b.data_version) return "data.inventory changed since the batch was flattened (referential constraints); upload it again";
  }
  return nullptr;
}

void require_current(gk_engine* e, const Compiled& c, const gk_batch& b) {
  if (const char* why = stale_reason(e, c, b)) throw RegoError{why};
}



// Expands every object of `ins` but those with a non-empty skip[i] (`skip` may be empty); a large page is spread over the host threads.
Expansion expand_page(Engine& eng, const std::vector<ObjIn>& ins, const std::vector<std::string>& skip, int threads) {
  const size_t n = ins.size();
  const size_t T = std::min<size_t>((size_t)std::max(1, threads), std::max<size_t>(1, n / 256));
  Expansion x;
  x.errors.assign(n, std::string());
  std::vector<std::vector<Child>> part(T);
  std::vector<std::exception_ptr> failed(T);
  auto work = [&](size_t t) {
    try {
      std::vector<Resultant> res;
      for (size_t i = n * t / T; i < n * (t + 1) / T; ++i) {
        if (i < skip.size() && !skip[i].empty()) continue;
        res.clear();
        try {
          eng.expand_object(ins[i], res);
        } catch (std::runtime_error& e) {   // (System.Expand's errors)
          x.errors[i] = std::string("unable to expand object: ") + e.what();
          continue;
        }
        for (auto& r : res) part[t].push_back(Child{(uint32_t)i, json_str(r.obj), r.template_name, r.action});
      }
    } catch (...) {
      failed[t] = std::current_exception();
    }
  };
  if (T == 1) work(0);
  else {
    std::vector<std::thread> th;
    for (size_t t = 0; t < T; ++t) th.emplace_back(work, t);
    for (auto& h : th) h.join();
  }
  for (auto& f : failed)
    if (f) std::rethrow_exception(f);
  for (auto& p : part) x.children.insert(x.children.end(), std::make_move_iterator(p.begin()), std::make_move_iterator(p.end()));
  return x;
}

// the resultants as review objects: the parent's Namespace (createReviewForResultant), source Generated
std::vector<gk_obj> resultant_objs(const std::vector<Child>& children, const std::vector<ObjIn>& parents) {
  std::vector<gk_obj> v(children.size());
  for (size_t k = 0; k < children.size(); ++k) {
    gk_obj& o = v[k];
    memset(&o, 0, sizeof o);
    o.json = children[k].json.data();
    o.len = children[k].json.size();
    const ObjIn& par = parents[children[k].parent];
    o.ns_json = par.ns_json;
    o.ns_len = par.ns_len;
    o.ns_name = par.ns_name;
    o.source = GK_SOURCE_GENERATED;
  }
  return v;
}

// the (group, version, kind) of a review's generator -- the old object of a DELETE, as Engine::expand_object expands it; empty when
// it has none or it is not a JSON object
void generator_gvk(const ObjIn& in, std::string& g, std::string& v, std::string& k) {
  const bool del = in.operation && std::string(in.operation) == "DELETE";
  const char* gj = del ? in.old_json : in.json;
  if (!gj) return;
  try {
    VP o = json_parse(gj, del ? in.old_len : in.len);
    if (o && o->t == VT::Obj) split_gv(o, g, v, k);
  } catch (JsonError&) {
  }
}

// GK_F_EXPAND, after the upload of batch `b` against snapshot `c`: the generators are selected on the device, expanded on the host, and
// their resultants uploaded as the batch's resultant batch.  `version`: the expansion version read before the parents were flattened.
// `from_source`: the parents' JSON comes from the batch's kept source (a refresh does not read the caller's page).
void expand_batch(gk_engine* e, const std::shared_ptr<const Compiled>& c, gk_batch& b, uint64_t version, bool from_source) {
  auto ex = std::make_shared<Expanded>();
  ex->version = version;
  b.ex = ex;
  if (!b.n || !e->eng->has_expansion()) return;
  std::string kept;   // from_source: the gathered JSON of the objects being read
  std::vector<uint64_t> kept_off;
  auto fetch = [&](const std::vector<uint32_t>& idx) {
    std::vector<ObjIn> ins(idx.size());
    if (from_source) {
      e->be->source_bytes(b.source.get(), idx, kept, kept_off);
      for (size_t i = 0; i < idx.size(); ++i) {
        ins[i].json = kept.data() + kept_off[i];
        ins[i].len = (size_t)(kept_off[i + 1] - kept_off[i]);
        ins[i].source = b.blob_source;
      }
    } else {
      for (size_t i = 0; i < idx.size(); ++i) ins[i] = b.obj_in(idx[i]);
    }
    return ins;
  };
  const double t0 = now_ms();
  std::vector<uint32_t> sel;
  uint32_t kinds = 0;
  float sel_ms = 0.f;
  e->be->select_generators(
      b.dev.get(), [&](uint32_t o, std::string& g, std::string& v, std::string& k) { generator_gvk(fetch({o})[0], g, v, k); },
      [e](const std::string& g, const std::string& v, const std::string& k) { return e->eng->expansion_selects(g, v, k); }, sel, &kinds, &sel_ms);
  const double t1 = now_ms();
  const std::vector<ObjIn> ins = fetch(sel);
  Expansion x = expand_page(*e->eng, ins, {}, e->eng->threads());
  const double t2 = now_ms();
  std::vector<gk_obj> robjs = resultant_objs(x.children, ins);
  for (auto& ch : x.children) ch.parent = sel[ch.parent];
  if (std::any_of(x.errors.begin(), x.errors.end(), [](const std::string& m) { return !m.empty(); })) {
    ex->x.errors.assign(b.n, std::string());
    for (size_t i = 0; i < sel.size(); ++i) ex->x.errors[sel[i]] = std::move(x.errors[i]);
  }
  const size_t m = x.children.size();
  const uint32_t rflags = b.flags & ~(uint32_t)(GK_F_KEEP_SOURCE | GK_F_EXPAND);
  if (m) {
    if (b.plain_page()) {   // blob parents (no Namespace objects): the resultants as one page, for the device ingest
      ex->off.assign(1, 0);
      for (auto& ch : x.children) {
        ex->blob += ch.json;
        ex->off.push_back(ex->blob.size());
        std::string().swap(ch.json);
      }
      robjs.clear();
      ex->res = upload_blob(e, c, ex->blob.data(), ex->off.data(), m, GK_SOURCE_GENERATED, rflags, nullptr);
    } else {
      ex->objs = std::move(robjs);
      ex->res = upload_batch(e, c, ex->objs.data(), m, rflags, nullptr);
    }
    std::vector<uint32_t>& par = ex->par;
    std::vector<uint32_t>& off = ex->off_par;
    off.assign(1, 0);
    for (size_t k = 0; k < m; ++k) {
      if (par.empty() || par.back() != x.children[k].parent) {
        if (!par.empty()) off.push_back((uint32_t)k);
        par.push_back(x.children[k].parent);
      }
    }
    off.push_back((uint32_t)m);
    e->be->set_parents(ex->res->dev.get(), par, off);
    b.alg_bytes += ex->res->alg_bytes;
  }
  ex->x.children = std::move(x.children);
  if (getenv("GK_TRACE_LAUNCH"))
    fprintf(stderr, "[expand] %u objects, %u distinct kinds, %zu selected, %zu resultants; selection %.3f ms on the device (%.3f ms wall), expansion %.3f ms, resultant upload %.3f ms\n",
            b.n, kinds, sel.size(), m, sel_ms, t1 - t0, t2 - t1, now_ms() - t2);
}

// the eval calls' check of an expanded batch (and their refusal of any other batch while templates are registered)
bool expansion_stale(gk_engine* e, const gk_batch& b) { return b.ex && b.ex->version != e->eng->expansion_version(); }
void require_expanded_or_none(gk_engine* e, const gk_batch& b) {
  if (!b.ex) refuse_while_expanding(e);
  else if (expansion_stale(e, b)) throw RegoError{"ExpansionTemplates changed since the batch was expanded; refresh it with gk_batch_refresh or upload it again"};
}

}  // namespace

namespace {
// gk_batch_eval_device and gk_batch_eval_device_peers: the kernel's outputs go to the caller's device buffers `d` (an expanded batch:
// then its resultants' evaluation and the fold, on the same stream)
void eval_device(gk_engine* e, const gk_batch& b, const char* ep, const DevOutPtrs& d) {
  require_expanded_or_none(e, b);
  auto c = e->eng->compiled();
  require_current(e, *c, b);
  ProgramLease lease(e, *c);
  std::vector<uint32_t> active;
  e->eng->active_mask(*c, ep ? ep : "", active);
  e->be->eval_into(b.dev.get(), active, d);
  if (b.ex && b.ex->res) e->be->fold_into(b.ex->res->dev.get(), b.ex->par, b.ex->off_par, active, d);
}
}  // namespace

extern "C" {

gk_engine_t* gk_engine_create(const gk_cfg* cfg, char** err) {
  gk_engine* e = nullptr;
  int rc = guard(err, [&]() {
    auto x = std::make_unique<gk_engine>();
    x->eng.reset(new Engine(cfg ? cfg->threads : 0));
    x->be.reset(make_backend(cfg ? cfg->device : 0));
    e = x.release();
  });
  return rc == GK_OK ? e : nullptr;
}

void gk_engine_destroy(gk_engine_t* e) { delete e; }
const char* gk_backend_name(gk_engine_t* e) { return e && e->be ? e->be->name() : ""; }
const char* gk_last_kernel(gk_engine_t* e) { return e && e->be ? e->be->last_kernel() : ""; }

int gk_add_template(gk_engine_t* e, const char* kind, const char* rego_src, size_t len, char** err) {
  if (!e || !kind || !rego_src) return GK_ERR_INVALID;
  return guard(err, [&]() { e->eng->add_template(kind, std::string(rego_src, len)); });
}
int gk_add_template_libs(gk_engine_t* e, const char* kind, const char* rego_src, size_t len, const char* const* libs, const size_t* lib_lens,
                         size_t n_libs, char** err) {
  if (!e || !kind || !rego_src || (n_libs && (!libs || !lib_lens))) return GK_ERR_INVALID;
  return guard(err, [&]() {
    std::vector<std::string> ls;
    for (size_t i = 0; i < n_libs; ++i) ls.emplace_back(libs[i] ? libs[i] : "", libs[i] ? lib_lens[i] : 0);
    e->eng->add_template(kind, std::string(rego_src, len), ls);
  });
}
int gk_remove_template(gk_engine_t* e, const char* kind) {
  if (!e || !kind) return GK_ERR_INVALID;
  return guard(nullptr, [&]() { e->eng->remove_template(kind); });
}
int gk_add_constraint(gk_engine_t* e, const char* json, size_t len, char** err) {
  if (!e || !json) return GK_ERR_INVALID;
  return guard(err, [&]() { e->eng->add_constraint(std::string(json, len)); });
}
int gk_validate_constraint(gk_engine_t* e, const char* json, size_t len, char** err) {
  (void)e;
  if (!json) return GK_ERR_INVALID;
  return guard(err, [&]() {
    std::string msg = validate_constraint_json(std::string(json, len));
    if (!msg.empty()) throw RegoError{msg};
  });
}
int gk_remove_constraint(gk_engine_t* e, const char* kind, const char* name) {
  if (!e || !kind || !name) return GK_ERR_INVALID;
  return guard(nullptr, [&]() { e->eng->remove_constraint(kind, name); });
}
int gk_put_namespace(gk_engine_t* e, const char* name, const char* ns_json, size_t len, char** err) {
  if (!e || !name || !ns_json) return GK_ERR_INVALID;
  return guard(err, [&]() { e->eng->put_namespace(name, std::string(ns_json, len)); });
}
int gk_add_data(gk_engine_t* e, const char* const* path, size_t npath, const char* json, size_t len, char** err) {
  if (!e || !json || (!path && npath)) return GK_ERR_INVALID;
  return guard(err, [&]() {
    std::vector<std::string> p;
    for (size_t i = 0; i < npath; ++i) p.push_back(path[i] ? path[i] : "");
    e->eng->add_data(p, std::string(json, len));
  });
}
int gk_remove_data(gk_engine_t* e, const char* const* path, size_t npath) {
  if (!e || !path || !npath) return GK_ERR_INVALID;
  return guard(nullptr, [&]() {
    std::vector<std::string> p;
    for (size_t i = 0; i < npath; ++i) p.push_back(path[i] ? path[i] : "");
    e->eng->remove_data(p);
  });
}
int gk_remove_namespace(gk_engine_t* e, const char* name) {
  if (!e || !name) return GK_ERR_INVALID;
  return guard(nullptr, [&]() { e->eng->remove_namespace(name); });
}

uint32_t gk_constraint_count(gk_engine_t* e) {
  if (!e) return 0;
  uint32_t n = 0;
  guard(nullptr, [&]() {
    auto c = e->eng->compiled();
    std::lock_guard<std::mutex> l(e->keys_mu);
    if (e->keys_version != c->version || e->key_sets.empty()) {
      auto ks = std::make_shared<std::vector<std::string>>();
      for (auto* k : c->order) ks->push_back(k->kind + "/" + k->name);
      e->key_sets.push_back(ks);
      if (e->key_sets.size() > 16) e->key_sets.pop_front();
      e->keys_version = c->version;
    }
    n = (uint32_t)e->key_sets.back()->size();
  });
  return n;
}
const char* gk_constraint_key(gk_engine_t* e, uint32_t index) {
  uint32_t n = gk_constraint_count(e);
  if (!e) return nullptr;
  std::lock_guard<std::mutex> l(e->keys_mu);
  return !e->key_sets.empty() && index < n && index < e->key_sets.back()->size() ? (*e->key_sets.back())[index].c_str() : nullptr;
}
const char* gk_result_constraint_key(const gk_result* r, uint32_t index) {
  if (!r || !r->priv) return nullptr;
  auto* rp = static_cast<const ResultPriv*>(r->priv);
  return index < rp->keys.size() ? rp->keys[index].c_str() : nullptr;
}

int gk_add_expansion_template(gk_engine_t* e, const char* json, size_t len, char** err) {
  if (!e || !json) return GK_ERR_INVALID;
  return guard(err, [&]() { e->eng->add_expansion_template(std::string(json, len)); });
}
int gk_remove_expansion_template(gk_engine_t* e, const char* name) {
  if (!e || !name) return GK_ERR_INVALID;
  return guard(nullptr, [&]() { e->eng->remove_expansion_template(name); });
}

char* gk_expansion_conflicts(gk_engine_t* e) {
  if (!e) return nullptr;
  std::string o = "[";
  guard(nullptr, [&]() {
    bool first = true;
    for (auto& n : e->eng->expansion_conflicts()) {
      if (!first) o += ",";
      first = false;
      json_quote(n, o);
    }
  });
  o += "]";
  return dup_str(o);
}

int gk_review_batch(gk_engine_t* e, const gk_obj* objs, size_t n, const char* ep, uint32_t flags, gk_result* out, char** err) {
  if (!e || !out || (!objs && n)) return GK_ERR_INVALID;
  memset(out, 0, sizeof *out);
  return guard(err, [&]() {
    // ---- expansion: the resultants are appended to the batch, reviewed with it, and folded back below
    Expansion x;
    std::vector<gk_obj> all;   // (empty: the objects alone)
    if (e->eng->has_expansion()) {
      std::vector<ObjIn> ins(n);
      for (size_t i = 0; i < n; ++i) ins[i] = to_in(objs[i]);
      x = expand_page(*e->eng, ins, {}, e->eng->threads());
      if (!x.children.empty()) {
        all.assign(objs, objs + n);
        const std::vector<gk_obj> res = resultant_objs(x.children, ins);
        all.insert(all.end(), res.begin(), res.end());
      }
    }
    const gk_obj* use = all.empty() ? objs : all.data();
    const size_t total = all.empty() ? n : all.size();
    gk_result stats;
    memset(&stats, 0, sizeof stats);
    auto c = e->eng->compiled();
    ProgramLease lease(e, *c);   // flatten + upload + kernel + rendering all against this one snapshot
    auto b = upload_batch(e, c, use, total, flags, &stats);
    eval_batch(e, b.get(), ep, flags, out);
    out->flatten_ms = stats.flatten_ms;
    out->h2d_ms = stats.h2d_ms;
    out->h2d_bytes = stats.h2d_bytes;
    const std::vector<Child>& children = x.children;
    const bool any_expand_err = std::any_of(x.errors.begin(), x.errors.end(), [](const std::string& m) { return !m.empty(); });
    if (children.empty() && !any_expand_err) return;
    // ---- fold the resultants back: bits ORed into the parent's row, results re-indexed with "[Implied by <template>]" and the
    // template's enforcement-action override (aggregate.go:19-63), their review-level errors reported on the parent
    auto* rp = static_cast<ResultPriv*>(out->priv);
    const uint32_t W = rp->ev.words;
    for (size_t k = 0; k < children.size(); ++k) {
      const size_t row = n + k, par = children[k].parent;
      if (!rp->ev.viol.empty())
        for (uint32_t w = 0; w < W; ++w) rp->ev.viol[par * W + w] |= rp->ev.viol[row * W + w];
      if (!rp->ev.err.empty())
        for (uint32_t w = 0; w < W; ++w) rp->ev.err[par * W + w] |= rp->ev.err[row * W + w];
    }
    if (!rp->ev.viol.empty()) rp->ev.viol.resize(n * (size_t)W);
    if (!rp->ev.err.empty()) rp->ev.err.resize(n * (size_t)W);
    rp->ev.n = (uint32_t)n;
    fold_results(rp->vio, rp->obj_errors, n, children, x.errors);
    const bool give_bits = !(flags & GK_F_NO_COPY_BACK);
    fill_result(out, rp, give_bits);
  });
}

int gk_batch_upload(gk_engine_t* e, const gk_obj* objs, size_t n, uint32_t flags, gk_batch_t** outb, gk_result* stats, char** err) {
  if (!e || !outb || (!objs && n)) return GK_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  return guard(err, [&]() {
    const uint64_t xv = e->eng->expansion_version();   // (read before the flatten, as the excluder is)
    auto c = e->eng->compiled();
    ProgramLease lease(e, *c);
    auto b = upload_batch(e, c, objs, n, flags, stats);
    if (flags & GK_F_EXPAND) {
      expand_batch(e, c, *b, xv, false);
      if (stats) stats->alg_bytes = b->alg_bytes;
    }
    *outb = b.release();
  });
}

int gk_batch_eval(gk_engine_t* e, gk_batch_t* b, const char* ep, uint32_t flags, gk_result* out, char** err) {
  if (!e || !b || !out) return GK_ERR_INVALID;
  memset(out, 0, sizeof *out);
  return guard(err, [&]() {
    require_expanded_or_none(e, *b);
    auto c = e->eng->compiled();
    require_current(e, *c, *b);
    ProgramLease lease(e, *c);
    eval_batch(e, b, ep, flags, out);
  });
}

int gk_batch_eval_device(gk_engine_t* e, gk_batch_t* b, const char* ep, void* d_viol, void* d_err, void* d_totals, void* d_err_totals,
                         void* stream, char** err) {
  if (!e || !b || !d_viol || !d_err || !d_totals || !d_err_totals) return GK_ERR_INVALID;
  DevOutPtrs d;
  d.viol = d_viol;
  d.err = d_err;
  d.totals = d_totals;
  d.err_totals = d_err_totals;
  d.stream = stream;
  return guard(err, [&]() { eval_device(e, *b, ep, d); });
}

int gk_batch_eval_device_peers(gk_engine_t* e, gk_batch_t* b, const char* ep, const uint64_t* peer_bases, uint32_t npeers, uint32_t rank,
                               uint64_t slot_i32, uint64_t tot_off_i32, uint32_t tot_stride, void* d_err, void* d_totals, void* d_err_totals,
                               void* stream, char** err) {
  if (!e || !b || !peer_bases || !npeers || npeers > 8 || rank >= npeers || !d_err || !d_totals || !d_err_totals) return GK_ERR_INVALID;
  DevOutPtrs d;
  d.err = d_err;
  d.totals = d_totals;
  d.err_totals = d_err_totals;
  d.stream = stream;
  d.npeers = npeers;
  d.tot_stride = tot_stride;
  d.rank = rank;
  for (uint32_t q = 0; q < npeers; ++q) {
    d.peer_viol[q] = peer_bases[q] + (uint64_t)rank * slot_i32 * 4;
    d.peer_tot[q] = peer_bases[q] + ((uint64_t)rank * slot_i32 + tot_off_i32) * 4;
  }
  return guard(err, [&]() { eval_device(e, *b, ep, d); });
}

int gk_batch_upload_blob(gk_engine_t* e, const char* buf, const uint64_t* offsets, size_t n, uint8_t source, uint32_t flags, gk_batch_t** outb,
                         gk_result* stats, char** err) {
  if (!e || !outb || ((!buf || !offsets) && n)) return GK_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  return guard(err, [&]() {
    const uint64_t xv = e->eng->expansion_version();
    auto c = e->eng->compiled();
    ProgramLease lease(e, *c);
    auto b = upload_blob(e, c, buf, offsets, n, source, flags, stats);
    if (flags & GK_F_EXPAND) {
      expand_batch(e, c, *b, xv, false);
      if (stats) stats->alg_bytes = b->alg_bytes;
    }
    *outb = b.release();
  });
}

int gk_review_blob(gk_engine_t* e, const char* buf, const uint64_t* offsets, size_t n, uint8_t source, const char* ep, uint32_t flags,
                   gk_result* out, char** err) {
  if (!e || !out || ((!buf || !offsets) && n)) return GK_ERR_INVALID;
  memset(out, 0, sizeof *out);
  return guard(err, [&]() {
    if (!(flags & GK_F_EXPAND)) refuse_while_expanding(e);
    gk_result stats;
    memset(&stats, 0, sizeof stats);
    const uint64_t xv = e->eng->expansion_version();
    auto c = e->eng->compiled();
    ProgramLease lease(e, *c);
    auto b = upload_blob(e, c, buf, offsets, n, source, flags & ~(uint32_t)GK_F_KEEP_SOURCE, &stats);   // (the batch lives for this call only)
    if (flags & GK_F_EXPAND) expand_batch(e, c, *b, xv, false);
    eval_batch(e, b.get(), ep, flags, out);
    out->flatten_ms = stats.flatten_ms;
    out->h2d_ms = stats.h2d_ms;
    out->h2d_bytes = stats.h2d_bytes;
  });
}

uint32_t gk_batch_size(gk_batch_t* b) { return b ? b->n : 0; }
uint64_t gk_batch_alg_bytes(gk_batch_t* b) { return b ? b->alg_bytes : 0; }
void gk_batch_free(gk_engine_t* e, gk_batch_t* b) {
  if (e) delete b;
}

int gk_batch_refresh(gk_engine_t* e, gk_batch_t* b, gk_result* stats, char** err) {
  if (!e || !b) return GK_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  bool rebuilt = false;
  const int rc = guard(err, [&]() {
    const uint64_t xv = e->eng->expansion_version();
    auto c = e->eng->compiled();
    if (excluded_of(e, b->flags) == b->excluded && !stale_reason(e, *c, *b) && !expansion_stale(e, *b)) {
      if (stats) {
        stats->alg_bytes = b->alg_bytes;
        stats->n_objects = b->n;
        stats->n_constraints = (uint32_t)c->cons_match.size();
      }
      return;
    }
    ProgramLease lease(e, *c);
    std::unique_ptr<gk_batch> nb;
    const bool from_source = b->source && device_ingest(*c, b->n);
    if (from_source) nb = refresh_from_source(e, c, *b, stats);
    else if (!b->blob) nb = upload_batch(e, c, b->objs.data(), b->objs.size(), b->flags, stats);
    else nb = upload_blob(e, c, b->blob, b->blob_off, b->n, b->blob_source, b->flags, stats);
    // the new columns replace the old ones; a kept source stays with the batch (a batch that had none may have gained one)
    if (!nb->source) {
      nb->source = std::move(b->source);
      nb->source_errors = std::move(b->source_errors);
    }
    nb->blob_source = b->blob_source;   // (a patched page flattened on the host: its objects are review objects of that source)
    if (b->flags & GK_F_EXPAND) {   // (expanded again whatever changed: the resultants' columns follow the constraint set too)
      expand_batch(e, c, *nb, xv, from_source);
      if (stats) stats->alg_bytes = nb->alg_bytes;
    }
    std::swap(*b, *nb);   // (the old columns are released with nb)
    rebuilt = true;
  });
  return rc == GK_OK && rebuilt ? 1 : rc;
}

int gk_batch_patch(gk_engine_t* e, gk_batch_t* b, const uint32_t* drop, size_t n_drop, const char* buf, const uint64_t* offsets, size_t n_add,
                   gk_result* stats, char** err) {
  if (!e || !b || (!drop && n_drop) || ((!buf || !offsets) && n_add)) return GK_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  auto invalid = [err](const std::string& why) {
    if (err) *err = dup_str(why);
    return GK_ERR_INVALID;
  };
  if (!b->source)
    return invalid("the batch keeps no device source to patch: only a gk_batch_upload_blob batch uploaded with GK_F_KEEP_SOURCE while its constraint "
                   "set was flattened on the device keeps one; upload the page again");
  std::vector<uint8_t> dropped(b->n, 0);
  for (size_t k = 0; k < n_drop; ++k) {
    if (drop[k] >= b->n) return invalid("drop index " + std::to_string(drop[k]) + " is out of range: the batch holds " + std::to_string(b->n) + " objects");
    if (dropped[drop[k]]++) return invalid("drop index " + std::to_string(drop[k]) + " is given twice");
  }
  if ((uint64_t)b->n - n_drop + n_add > 0x7fffff00ull) return invalid("a patched batch would hold more than 2^31 objects");
  int refused = 0;
  const int rc = guard(err, [&]() {
    const uint64_t xv = e->eng->expansion_version();
    auto c = e->eng->compiled();
    if (!device_ingest(*c, 1)) {   // (a fresh upload would flatten the page on the host and keep no device source)
      refused = invalid("the constraint set is flattened on the host (" + (c->host_ingest_reason.empty() ? std::string("device ingest turned off") : c->host_ingest_reason) +
                        "): a patch splices the page on the device only; upload the page again");
      return;
    }
    ProgramLease lease(e, *c);
    const double t0 = now_ms();
    std::vector<uint32_t> keep;
    keep.reserve(b->n - n_drop);
    for (uint32_t i = 0; i < b->n; ++i)
      if (!dropped[i]) keep.push_back(i);
    const uint32_t nk = (uint32_t)keep.size(), n = nk + (uint32_t)n_add;
    IngestStats pst;
    BackendHandle src = kept_source(e, e->be->patch_source(b->source.get(), keep, reinterpret_cast<const uint8_t*>(buf),
                                                           reinterpret_cast<const unsigned long long*>(offsets), n_add, &pst));
    // the objects as the host reads them (messages, audit, expansion): the staying ones where they were given, the added ones in buf
    std::vector<gk_obj> objs(n);
    for (uint32_t j = 0; j < n; ++j) {
      gk_obj& o = objs[j];
      memset(&o, 0, sizeof o);
      if (j < nk) {
        const ObjIn in = b->obj_in(keep[j]);
        o.json = in.json;
        o.len = in.len;
      } else {
        o.json = buf + offsets[j - nk];
        o.len = (size_t)(offsets[j - nk + 1] - offsets[j - nk]);
      }
      o.source = b->blob_source;
    }
    std::unique_ptr<gk_batch> nb;
    std::vector<std::string> errors;
    if (n) {
      IngestReq rq = e->eng->ingest_request(c, nullptr, nullptr, n, b->blob_source, process_of(b->flags));
      IngestStats ist;
      std::vector<uint32_t> status;
      BackendHandle dev = device_batch(e, e->be->reextract(src.get(), rq, &ist, &status));
      for (uint32_t j = 0; j < n; ++j)
        if (status[j] != GK_ING_OK) {
          if (errors.empty()) errors.assign(n, std::string());
          errors[j] = j < nk && !b->source_errors.empty() ? b->source_errors[keep[j]] : ingest_error(e, status[j], to_in(objs[j]));
        }
      ist.h2d_ms += pst.h2d_ms;
      ist.h2d_bytes += pst.h2d_bytes;
      nb = make_batch(e, c, std::move(dev), n, b->flags, errors, std::move(rq.excluded), ist, (now_ms() - t0) - ist.h2d_ms, stats);
      if (stats) stats->kernel_ms = pst.h2d_ms + ist.extract_ms;
    } else {
      nb = upload_batch(e, c, nullptr, 0, b->flags, stats);   // (as gk_batch_upload_blob of an empty page)
    }
    nb->objs = std::move(objs);
    nb->blob_source = b->blob_source;
    nb->source = std::move(src);
    nb->source_errors = std::move(errors);
    if (b->flags & GK_F_EXPAND) {
      expand_batch(e, c, *nb, xv, true);
      if (stats) stats->alg_bytes = nb->alg_bytes;
    }
    std::swap(*b, *nb);   // (the old columns and source are released with nb)
  });
  if (rc != GK_OK) return rc;
  return refused ? refused : (int)b->n;
}

int gk_set_excluded_namespaces(gk_engine_t* e, const char* process, const char* const* patterns, size_t n, char** err) {
  if (!e || !process || (!patterns && n)) return GK_ERR_INVALID;
  return guard(err, [&]() {
    std::vector<std::string> v;
    for (size_t i = 0; i < n; ++i) v.push_back(patterns[i] ? patterns[i] : "");
    e->eng->set_excluded_namespaces(process, v);
  });
}

struct gk_audit {
  gk_engine* e;
  AuditRun run;
  float select_ms = 0.f;   // device time of the last gk_audit_add_batch_ordered's ranking, selection and resultant classification
};

gk_audit_t* gk_audit_begin(gk_engine_t* e, uint32_t violations_limit, uint32_t msg_size, char** err) {
  if (!e) return nullptr;
  gk_audit* a = nullptr;
  guard(err, [&]() {
    a = new gk_audit{e, {}};
    a->run.limit = violations_limit ? violations_limit : 20;
    a->run.msg_size = msg_size ? msg_size : 256;
  });
  return a;
}

namespace {
// The results `vio` of resultants (object k: children[k]) entered into `run` as results of their parents (parent i's JSON: ins[i]) --
// addAuditResponsesToUpdateLists names the parent object: "[Implied by <template>]", the template's enforcement-action override
void fold_resultant_results(AuditRun& run, const Compiled& c, const std::vector<Violation>& vio, const std::vector<Child>& children,
                            const std::vector<ObjIn>& ins) {
  struct Ident {
    std::string g, v, k, ns, name;
  };
  std::unordered_map<uint32_t, Ident> ident;   // parents that have results from resultants, parsed once each
  for (auto& v : vio) {
    const Child& ch = children[v.object];
    auto it = ident.find(ch.parent);
    if (it == ident.end()) {
      Ident id2;
      try {
        VP po = json_parse(ins[ch.parent].json, ins[ch.parent].len);
        split_gv(po, id2.g, id2.v, id2.k);
        id2.ns = meta_str(po, "namespace");
        id2.name = meta_str(po, "name");
      } catch (JsonError&) {
      }
      it = ident.emplace(ch.parent, std::move(id2)).first;
    }
    const Constraint& con = *c.order[v.constraint];
    StatusViolation sv;
    sv.group = it->second.g, sv.version = it->second.v, sv.kind = it->second.k, sv.ns = it->second.ns, sv.name = it->second.name;
    sv.message = ExpansionSystem::implied_by(ch.tmpl, v.msg);
    sv.action = ch.action.empty() ? v.action : ch.action;   // OverrideEnforcementAction: the action only
    sv.scoped_json = v.scoped_json;
    run.fold(con.kind + "/" + con.name, std::move(sv));
    run.results++;
  }
}

// a resultant the review refused (manager.go:757-760 logs it and goes on): reported on its parent, unless the parent has an error
void resultant_errors(std::vector<std::string>& obj_errs, const std::vector<std::string>& res_errors, const std::vector<Child>& children) {
  for (size_t k = 0; k < res_errors.size() && k < children.size(); ++k)
    if (!res_errors[k].empty() && obj_errs[children[k].parent].empty())
      obj_errs[children[k].parent] = ExpansionSystem::implied_by(children[k].tmpl, res_errors[k]);
}
}  // namespace

// gk_audit_add_batch and gk_audit_add_batch_ordered: `ordered` takes the lazy path's candidates from Backend::audit_candidates (any mix
// of kinds) instead of the host threshold scan over (namespace, name), which only a page of one kind allows
static int audit_add(gk_audit_t* a, gk_batch_t* b, const char* ep_c, bool ordered, char** err) {
  if (!a || !b) return GK_ERR_INVALID;
  return guard(err, [&]() {
    gk_engine* e = a->e;
    auto c = e->eng->compiled();
    require_current(e, *c, *b);
    std::string ep = ep_c ? ep_c : "";
    std::vector<uint32_t> active;
    e->eng->active_mask(*c, ep, active);
    // An expanded batch whose templates are current brings its resultants: they are not expanded again but evaluated where they are
    // resident, their pairs sorted against the parents' candidates.  Its resultants must also be current for the constraint set,
    // data.inventory and the excluder (the audit flattens re-expanded resultants with the current excluder).
    const gk_batch* res = b->ex ? b->ex->res.get() : nullptr;
    // action classes of the resultants: 0 = the constraint's own action, k > 0 = the k-th distinct template override
    std::vector<std::string> actions(1);
    std::vector<uint8_t> cls(res ? res->n : 0, 0);
    for (size_t k = 0; k < cls.size() && actions.size() <= 256; ++k) {
      const std::string& act = b->ex->x.children[k].action;
      if (act.empty()) continue;
      const size_t j = (size_t)(std::find(actions.begin(), actions.end(), act) - actions.begin());
      if (j == actions.size()) actions.push_back(act);
      cls[k] = (uint8_t)j;
    }
    const bool resident = b->ex && !expansion_stale(e, *b) && !getenv("GK_AUDIT_EAGER") && actions.size() <= 256 &&
                          (!res || (!stale_reason(e, *c, *res) && excluded_of(e, res->flags) == res->excluded));
    if (!resident) res = nullptr;
    // The lazy path (audit.hpp): the namespace / name arrays of the batch and the bitmap of the ambiguity netlist let the run count
    // the pairs that have exactly one result and evaluate only what can still enter a constraint's list.
    const bool lazy = !getenv("GK_AUDIT_EAGER") && (c->amb || std::any_of(c->single_result.begin(), c->single_result.end(), [](uint8_t x) { return x != 0; }));
    // (the ordered lazy path sorts the resultants' pairs on the device, from the planes their evaluation leaves there)
    const bool res_on_device = ordered && lazy;
    EvalOut ev, ev_amb, rev, rev_amb;
    {
      ProgramLease lease(e, *c);
      e->be->eval(b->dev.get(), active, ev, true);
      if (res) e->be->eval(res->dev.get(), active, rev, !res_on_device);   // (unfolded: each resultant's pairs are counted on their own)
    }
    std::vector<ObjIn> ins(b->n);
    for (size_t i = 0; i < ins.size(); ++i) ins[i] = b->obj_in(i);
    BatchIdentity id;
    if (lazy && !ordered) e->be->identity(b->dev.get(), id);
    const bool use_amb = lazy && (ordered || id.uniform_gvk) && c->amb && !getenv("GK_AUDIT_NO_AMB");
    BackendHandle res_fork;   // the resultants' ambiguity fork: its planes stay on the device for Backend::audit_resultants
    if (use_amb) {
      ProgramLease lease(e, *c->amb);   // (the backend holds one netlist at a time: waits until no review uses the other)
      BackendHandle fork = device_batch(e, e->be->fork_batch(b->dev.get(), *c->amb));
      e->be->eval(fork.get(), active, ev_amb, true);
      if (res) {
        res_fork = device_batch(e, e->be->fork_batch(res->dev.get(), *c->amb));
        e->be->eval(res_fork.get(), active, rev_amb, !res_on_device);
      }
    }
    // ---- expansion inside the audit loop (pkg/audit/manager.go:733-765): every reviewed object is expanded; its resultants are reviewed
    // as Generated resources with the parent's Namespace, their results -- "[Implied by <template>]", the template's action override --
    // are the PARENT's results (addAuditResponsesToUpdateLists names the parent object).  An object whose expansion fails contributes
    // nothing at all, not even its own violations (the reference logs the error and `continue`s past the bookkeeping of the response).
    std::vector<std::string> obj_errs = b->host->obj_errors.empty() ? std::vector<std::string>(b->n) : b->host->obj_errors;
    obj_errs.resize(b->n);
    // (an object whose own review failed is not expanded: the reference never gets to its expansion)
    Expansion x;
    if (resident) {
      for (size_t i = 0; i < b->ex->x.errors.size(); ++i)
        if (obj_errs[i].empty()) x.errors.push_back(b->ex->x.errors[i]);
        else x.errors.emplace_back();
    } else if (e->eng->has_expansion()) {
      const double t0 = now_ms();
      x = expand_page(*e->eng, ins, obj_errs, e->eng->threads());
      if (getenv("GK_TRACE_LAUNCH"))
        fprintf(stderr, "[audit] expanded %u objects on the host: %zu resultants, %.3f ms\n", b->n, x.children.size(), now_ms() - t0);
    }
    const std::vector<Child>& children = resident ? b->ex->x.children : x.children;
    const uint32_t W = ev.words;
    for (size_t i = 0; i < x.errors.size(); ++i)
      if (!x.errors[i].empty()) {
        obj_errs[i] = x.errors[i];
        for (uint32_t w = 0; w < W; ++w) {
          if (!ev.viol.empty()) ev.viol[i * W + w] = 0;
          if (!ev.err.empty()) ev.err[i * W + w] = 0;
        }
      }
    // (after the expansion above: the rows of objects whose expansion failed are cleared, and they are no candidates either)
    std::vector<uint32_t> cand;
    AuditRanks ranks;   // the parents' ranking, kept for the resultants
    if (lazy && ordered) {
      auto gvk_of = [&ins](uint32_t o, std::string& g, std::string& v, std::string& k) {
        try {
          split_gv(json_parse(ins[o].json, ins[o].len), g, v, k);
        } catch (JsonError&) {
        }
      };
      e->be->audit_candidates(b->dev.get(), ev.viol.data(), ev.words, (uint32_t)c->order.size(), (uint32_t)a->run.limit, gvk_of, cand, &a->select_ms,
                              res ? &ranks : nullptr);
    }
    HostCandidates hc;   // the host threshold scan's rule, kept for the resultants
    a->run.add_batch(*e->eng, *c, ins, ev.viol.data(), ev.err.empty() ? nullptr : ev.err.data(), ev.words, ev.errlist, ep,
                     lazy && !ordered ? &id : nullptr, use_amb ? ev_amb.viol.data() : nullptr, lazy && ordered ? cand.data() : nullptr, &hc);
    if (res) {
      // ---- the resident resultants.  Their pairs are sorted against the parents' candidates (a resultant's results carry its
      // parent's identity, and each flagged parent has a result of its own: a resultant above its constraint's threshold cannot enter
      // the list), so the parents' selection stands as it is.  Matcher errors, candidates and pairs that may have several results are
      // rendered; the others are counted.  Pairs that cannot be sorted -- no lazy path -- are all rendered.
      const uint32_t m = res->n, C = (uint32_t)c->order.size();
      const bool sorted = ordered ? lazy : hc.lazy;
      std::vector<uint8_t> dead(b->n, 0);
      bool any_dead = false;
      for (uint32_t p : b->ex->par)
        if (!obj_errs[p].empty()) dead[p] = 1, any_dead = true;   // (own review failed: no resultants; failed expansions have none anyway)
      ResultantClasses rc;
      rc.single = c->single_result.data();
      rc.cls = cls.data();
      rc.classes = (uint32_t)actions.size();
      rc.nconstraints = C;
      rc.parents = b->n;
      rc.dead = any_dead ? dead.data() : nullptr;
      ResultantSplit split;
      float classify_ms = 0.f;
      if (res_on_device) {
        e->be->audit_resultants(res->dev.get(), res_fork.get(), rev, use_amb ? &rev_amb : nullptr, b->ex->par, b->ex->off_par, ranks, rc, split,
                                &classify_ms);
        a->select_ms += classify_ms;
      } else {
        GkResClassArgs ca{};
        ca.viol = rev.viol.data();
        ca.err = rev.err.data();
        ca.amb = use_amb ? rev_amb.viol.data() : nullptr;
        ca.single = rc.single;
        ca.words = rev.words;
        ca.nconstraints = C;
        classify_resultants_host(ca, b->ex->par, b->ex->off_par, rc, [&](uint32_t p, uint32_t cc) { return !sorted || hc(p, cc); }, split);
      }
      uint64_t counted = 0, errors = 0;
      for (uint32_t k = 0; k < rc.classes; ++k)
        for (uint32_t cix = 0; cix < C; ++cix)
          if (const uint64_t nc = split.counted[(size_t)k * C + cix]) {
            const Constraint& con = *c->order[cix];
            a->run.add_counted(con.kind + "/" + con.name, k ? actions[k] : con.action, nc);
            counted += nc;
          }
      // the listed pairs as planes of their own, rendered as any batch's flagged pairs are (one parse per listed resultant)
      BitPlane lv, le;
      lv.assign((size_t)m * W, 0u);
      le.assign((size_t)m * W, 0u);
      for (size_t i = 0; i + 1 < split.render.size(); i += 2) {
        const uint32_t r = split.render[i], cix = split.render[i + 1] & 0x7fffffffu, is_err = split.render[i + 1] >> 31;
        (is_err ? le : lv)[(size_t)r * W + (cix >> 5)] |= 1u << (cix & 31u);
        errors += is_err;
      }
      fold_resultant_results(a->run, *c, render(e, *c, *res, lv, le, rev.errlist, W, C, ep), children, ins);
      const uint64_t rendered = split.render.size() / 2 - errors;
      a->run.resultant_rendered += rendered;
      a->run.resultant_counted += counted;
      resultant_errors(obj_errs, res->host->obj_errors, children);
      if (getenv("GK_TRACE_LAUNCH"))
        fprintf(stderr, "[audit] %u resultants taken from the expanded batch: %llu pairs rendered, %llu counted, %llu matcher errors; sorted %s (%.3f ms on the device)\n",
                m, (unsigned long long)rendered, (unsigned long long)counted, (unsigned long long)errors,
                !sorted ? "no pair (every pair rendered)" : res_on_device ? "on the device" : "on the host", classify_ms);
    } else if (!children.empty()) {
      const std::vector<gk_obj> cobjs = resultant_objs(children, ins);
      gk_result cres;
      memset(&cres, 0, sizeof cres);
      {
        ProgramLease lease(e, *c);
        auto cb = upload_batch(e, c, cobjs.data(), cobjs.size(), b->flags, nullptr);
        eval_batch(e, cb.get(), ep_c, GK_F_MATERIALIZE | GK_F_NO_COPY_BACK, &cres);
      }
      std::unique_ptr<ResultPriv> crp(static_cast<ResultPriv*>(cres.priv));
      cres.priv = nullptr;
      fold_resultant_results(a->run, *c, crp->vio, children, ins);
      resultant_errors(obj_errs, crp->obj_errors, children);
    }
    a->run.add_object_errors(obj_errs);
  });
}

int gk_audit_add_batch(gk_audit_t* a, gk_batch_t* b, const char* ep, char** err) { return audit_add(a, b, ep, false, err); }

int gk_audit_add_batch_ordered(gk_audit_t* a, gk_batch_t* b, const char* ep, char** err) { return audit_add(a, b, ep, true, err); }

float gk_audit_select_ms(gk_audit_t* a) { return a ? a->select_ms : 0.f; }

int gk_audit_resultant_pairs(gk_audit_t* a, uint64_t* evaluated, uint64_t* counted) {
  if (!a) return GK_ERR_INVALID;
  if (evaluated) *evaluated = a->run.resultant_rendered;
  if (counted) *counted = a->run.resultant_counted;
  return GK_OK;
}

int gk_audit_export(gk_audit_t* a, char** buf, size_t* len, char** err) {
  if (!a || !buf || !len) return GK_ERR_INVALID;
  *buf = nullptr;
  *len = 0;
  return guard(err, [&]() {
    const std::string s = a->run.serialize();
    char* p = static_cast<char*>(malloc(s.size()));
    if (!p) throw std::bad_alloc();
    memcpy(p, s.data(), s.size());
    *buf = p;
    *len = s.size();
  });
}

int gk_audit_merge(gk_audit_t* a, const char* buf, size_t len, char** err) {
  if (!a || (!buf && len)) return GK_ERR_INVALID;
  const int rc = guard(err, [&]() {
    AuditRun other = AuditRun::parse(reinterpret_cast<const uint8_t*>(buf), len);   // (the run is untouched until the buffer is whole)
    if (other.limit != a->run.limit || other.msg_size != a->run.msg_size) {
      throw RegoError{"audit merge: the exported run has violations_limit " + std::to_string(other.limit) + " and msg_size " +
                      std::to_string(other.msg_size) + ", this run " + std::to_string(a->run.limit) + " and " + std::to_string(a->run.msg_size)};
    }
    a->run.merge(other);
  });
  return rc == GK_ERR_REGO ? GK_ERR_INVALID : rc;   // (every RegoError here is about the buffer)
}

char* gk_audit_report(gk_audit_t* a, char** err) {
  if (!a) return nullptr;
  char* out = nullptr;
  guard(err, [&]() { out = dup_str(a->run.report()); });
  return out;
}

void gk_audit_end(gk_audit_t* a) { delete a; }

char* gk_validation_messages(gk_engine_t* e, const gk_result* r, uint32_t object, char** err) {
  if (!e || !r || !r->priv) return nullptr;
  char* out = nullptr;
  guard(err, [&]() {
    auto* rp = static_cast<ResultPriv*>(r->priv);
    auto c = rp->compiled ? rp->compiled : e->eng->compiled();
    std::vector<std::string> deny, warn;
    validation_messages(*c, rp->vio, object, deny, warn);
    std::string o = "{\"deny\":[";
    for (size_t i = 0; i < deny.size(); ++i) {
      if (i) o += ",";
      json_quote(deny[i], o);
    }
    o += "],\"warn\":[";
    for (size_t i = 0; i < warn.size(); ++i) {
      if (i) o += ",";
      json_quote(warn[i], o);
    }
    o += "]}";
    out = dup_str(o);
  });
  return out;
}

int gk_host_cpus(void) { return effective_cpus(); }

int gk_blob_prefetch(gk_engine_t* e, const char* buf, const uint64_t* offsets, size_t n, char** err) {
  if (!e || ((!buf || !offsets) && n)) return GK_ERR_INVALID;
  return guard(err, [&]() {
    auto c = e->eng->compiled();
    if (!c->device_ingest || n == 0) return;   // host-flattened snapshots have nothing to stream ahead
    e->be->prefetch(reinterpret_cast<const uint8_t*>(buf), reinterpret_cast<const unsigned long long*>(offsets), n);
  });
}

int gk_pin_host(gk_engine_t* e, const void* p, size_t bytes, int pin, char** err) {
  if (!e || !p) return GK_ERR_INVALID;
  return guard(err, [&]() { e->be->pin_host(p, bytes, pin != 0); });
}

void gk_free_result(gk_result* r) {
  if (!r || !r->priv) return;
  delete static_cast<ResultPriv*>(r->priv);
  memset(r, 0, sizeof *r);
}
void gk_free_str(char* s) { free(s); }

char* gk_dump(gk_engine_t* e) {
  if (!e) return nullptr;
  std::string s;
  guard(nullptr, [&]() { s = e->eng->dump(); });
  return dup_str(s);
}

const char* gk_stat_description(const char* n) {
  // the StatsEntry names this driver emits (cf. runTimeNS in pkg/drivers/k8scel/driver.go:256-263)
  if (!n) return nullptr;
  if (!strcmp(n, "kernelTimeNS")) return "the number of nanoseconds the GPU kernel took to evaluate every constraint against the batch";
  if (!strcmp(n, "flattenTimeNS")) return "the number of nanoseconds spent flattening the batch of objects into columns on the host";
  if (!strcmp(n, "batchSize")) return "the number of objects evaluated together";
  if (!strcmp(n, "bytesRead")) return "the algorithmic bytes of column data the kernel read for the batch";
  return nullptr;
}

}  // extern "C"
