// C ABI (include/gk_engine.h) over Engine + Backend.  No exceptions cross this file's extern "C" surface.
#include <chrono>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <cstdlib>
#include <cstring>
#include <functional>
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
}  // namespace

struct gk_batch {
  void* dev = nullptr;
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
  void* source = nullptr;
  std::vector<std::string> source_errors;
  ObjIn obj_in(size_t i) const;
};

namespace {

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

// evaluate a resident batch; optionally render messages for flagged pairs
void eval_batch(gk_engine* e, gk_batch* b, const char* ep_c, uint32_t flags, gk_result* out) {
  std::string ep = ep_c ? ep_c : "";
  const Compiled& c = *b->compiled;
  auto rp = std::make_unique<ResultPriv>();
  rp->compiled = b->compiled;
  for (auto* k : c.order) rp->keys.push_back(k->kind + "/" + k->name);
  std::vector<uint32_t> active;
  e->eng->active_mask(c, ep, active);
  bool copy_back = !(flags & GK_F_NO_COPY_BACK) || (flags & GK_F_MATERIALIZE);
  double t0 = now_ms();
  e->be->eval(b->dev, active, rp->ev, copy_back);
  double t1 = now_ms();
  rp->obj_errors = b->host->obj_errors;
  out->d2h_bytes = copy_back ? (uint64_t)rp->ev.viol.size() * 8 : 0;
  out->d2h_ms = (t1 - t0) - rp->ev.kernel_ms;
  if (out->d2h_ms < 0) out->d2h_ms = 0;
  out->alg_bytes = b->alg_bytes + (uint64_t)b->n * rp->ev.words * 8;
  out->materialize_ms = 0;
  if (flags & GK_F_MATERIALIZE) {
    double m0 = now_ms();
    const uint32_t W = rp->ev.words, C = rp->ev.nconstraints;
    // matcher errors first (autoreject results), then rendered violations, both in (object, constraint) order
    std::unordered_map<uint64_t, uint32_t> err_code;
    for (size_t i = 0; i + 2 < rp->ev.errlist.size(); i += 3)
      err_code[((uint64_t)rp->ev.errlist[i] << 32) | rp->ev.errlist[i + 1]] = rp->ev.errlist[i + 2];
    // one DOM parse per object, all of its flagged constraints rendered from it; objects are spread over the host threads
    const uint32_t n = b->n;
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
            const uint32_t vb = rp->ev.viol[(size_t)o * W + w], eb = rp->ev.err[(size_t)o * W + w];
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
          if (!flagged.empty()) e->eng->materialize_object(c, b->obj_in(o), o, flagged, ep, part[t], nullptr, &mctx);
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
    for (auto& v : part) rp->vio.insert(rp->vio.end(), std::make_move_iterator(v.begin()), std::make_move_iterator(v.end()));
    out->materialize_ms = now_ms() - m0;
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

void upload_batch(gk_engine* e, const std::shared_ptr<const Compiled>& c, const gk_obj* objs, size_t n, uint32_t flags, gk_batch** outb,
                  gk_result* stats) {
  std::vector<std::string> excluded = excluded_of(e, flags);   // (read before the flatten: a later change makes the batch stale, never current)
  std::vector<ObjIn> ins(n);
  for (size_t i = 0; i < n; ++i) ins[i] = to_in(objs[i]);
  double t0 = now_ms();
  auto hb = e->eng->flatten(ins.data(), n, *c, process_of(flags));
  double t1 = now_ms();
  e->be->sync_strings(e->eng->strings());
  auto b = std::make_unique<gk_batch>();
  double h2d_ms = 0;
  uint64_t h2d_bytes = 0;
  b->dev = e->be->upload(*hb, *c, &h2d_ms, &h2d_bytes);
  b->compiled = c;
  if (c->uses_data) e->eng->data_doc(&b->data_version);
  b->n = hb->n;
  b->flags = flags;
  b->alg_bytes = hb->alg_bytes;
  b->excluded = std::move(excluded);
  b->objs.assign(objs, objs + n);
  // drop the host column data; keep the small per-object error list
  auto slim = std::make_shared<HostBatch>();
  slim->n = hb->n;
  slim->obj_errors = std::move(hb->obj_errors);
  slim->alg_bytes = hb->alg_bytes;
  b->host = slim;
  if (stats) {
    stats->flatten_ms = t1 - t0;
    stats->h2d_ms = h2d_ms;
    stats->h2d_bytes = h2d_bytes;
    stats->alg_bytes = hb->alg_bytes;
    stats->n_objects = hb->n;
    stats->n_constraints = (uint32_t)c->cons_match.size();
  }
  *outb = b.release();
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

// A batch ingested on the device, or re-extracted from its kept source (`ist`, `t0`: the ingest's statistics and start); the
// review-level errors of its objects are `errors` (empty: none).
std::unique_ptr<gk_batch> blob_batch(gk_engine* e, const std::shared_ptr<const Compiled>& c, void* dev, const char* buf, const uint64_t* off, size_t n,
                                     uint8_t source, uint32_t flags, std::vector<std::string> errors, const IngestStats& ist, double t0, gk_result* stats) {
  auto b = std::make_unique<gk_batch>();
  b->dev = dev;
  b->compiled = c;
  if (c->uses_data) e->eng->data_doc(&b->data_version);
  b->n = (uint32_t)n;
  b->flags = flags;
  b->alg_bytes = ist.alg_bytes;
  b->blob = buf;
  b->blob_off = off;
  b->blob_source = source;
  auto slim = std::make_shared<HostBatch>();
  slim->n = (uint32_t)n;
  slim->alg_bytes = ist.alg_bytes;
  slim->obj_errors = std::move(errors);
  b->host = slim;
  if (stats) {
    stats->flatten_ms = (now_ms() - t0) - ist.h2d_ms;
    stats->h2d_ms = ist.h2d_ms;
    stats->h2d_bytes = ist.h2d_bytes;
    stats->alg_bytes = ist.alg_bytes;
    stats->n_objects = (uint32_t)n;
    stats->n_constraints = (uint32_t)c->cons_match.size();
  }
  return b;
}

// a blob of plain objects: flattened by the ingest kernels on the device when the compiled snapshot allows it
void upload_blob(gk_engine* e, const std::shared_ptr<const Compiled>& c, const char* buf, const uint64_t* off, size_t n, uint8_t source, uint32_t flags,
                 gk_batch** outb, gk_result* stats) {
  if (!device_ingest(*c, n)) {
    auto v = blob_objs(buf, off, n, source);
    upload_batch(e, c, v.data(), n, flags, outb, stats);
    (*outb)->blob = buf;   // (the objects of `objs`, as a blob: a later gk_batch_refresh may ingest them on the device)
    (*outb)->blob_off = off;
    (*outb)->blob_source = source;
    return;
  }
  double t0 = now_ms();
  IngestReq rq = e->eng->ingest_request(c, reinterpret_cast<const uint8_t*>(buf), reinterpret_cast<const unsigned long long*>(off), n, source, process_of(flags));
  IngestStats ist;
  std::vector<uint32_t> status;
  void* kept = nullptr;
  void* dev = (flags & GK_F_KEEP_SOURCE) ? e->be->ingest_keep(rq, &ist, &status, &kept) : e->be->ingest(rq, &ist, &status);
  std::vector<std::string> errors;
  for (size_t i = 0; i < n; ++i)
    if (status[i] != GK_ING_OK) {
      if (errors.empty()) errors.assign(n, std::string());   // (left empty when every object is fine)
      // the rare rejected object: the host parser words the review-level error (bad JSON, not an object, kind missing)
      ObjIn in;
      in.json = buf + off[i];
      in.len = (size_t)(off[i + 1] - off[i]);
      in.source = source;
      std::string err;
      VP doc = e->eng->review_doc(in, nullptr, nullptr, nullptr, &err);
      if (doc && status[i] != GK_ING_NULL) err = "device ingest refused the object (status " + std::to_string(status[i]) + "): JSON nesting deeper than " +
                                               std::to_string(GK_TAPE_MAX_DEPTH) + " levels or a token longer than 128 MiB";
      if (!doc && err.empty()) err = "invalid request object";
      errors[i] = err;
    }
  auto b = blob_batch(e, c, dev, buf, off, n, source, flags, errors, ist, t0, stats);
  b->excluded = rq.excluded;
  if (kept) {
    b->source = kept;
    b->source_errors = std::move(errors);
  }
  *outb = b.release();
}

// gk_batch_refresh of a batch that kept its source, for a snapshot flattened on the device: the extraction passes again, from the
// page's token tape in HBM -- no copy, no tokeniser, and the caller's blob is not read
void refresh_from_source(gk_engine* e, const std::shared_ptr<const Compiled>& c, const gk_batch* old, gk_batch** outb, gk_result* stats) {
  double t0 = now_ms();
  IngestReq rq = e->eng->ingest_request(c, nullptr, nullptr, old->n, old->blob_source, process_of(old->flags));
  IngestStats ist;
  void* dev = e->be->reextract(old->source, rq, &ist);
  auto b = blob_batch(e, c, dev, old->blob, old->blob_off, old->n, old->blob_source, old->flags, old->source_errors, ist, t0, stats);
  b->excluded = rq.excluded;
  *outb = b.release();
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
    // ---- expansion (pkg/audit/manager.go:733-765, pkg/webhook/policy.go:610-646): the resultants of generator objects are
    // appended to the batch as generated resources, reviewed with it, and their results folded back onto their parents
    struct Child {
      uint32_t parent;
      std::string json, tmpl, action;
    };
    std::vector<Child> children;
    std::vector<std::string> expand_errors;
    if (e->eng->has_expansion()) {
      expand_errors.assign(n, std::string());
      std::vector<Resultant> res;
      for (size_t i = 0; i < n; ++i) {
        res.clear();
        try {
          e->eng->expand_object(to_in(objs[i]), res);
        } catch (std::runtime_error& x) {
          expand_errors[i] = std::string("unable to expand object: ") + x.what();
          continue;
        }
        for (auto& r : res) children.push_back(Child{(uint32_t)i, json_str(r.obj), r.template_name, r.action});
      }
    }
    std::vector<gk_obj> all;
    const gk_obj* use = objs;
    size_t total = n;
    if (!children.empty()) {
      all.assign(objs, objs + n);
      for (auto& c : children) {
        gk_obj o;
        memset(&o, 0, sizeof o);
        o.json = c.json.data();
        o.len = c.json.size();
        o.ns_json = objs[c.parent].ns_json;       // createReviewForResultant: the parent's Namespace, source Generated
        o.ns_len = objs[c.parent].ns_len;
        o.ns_name = objs[c.parent].ns_name;
        o.source = GK_SOURCE_GENERATED;
        all.push_back(o);
      }
      use = all.data();
      total = all.size();
    }
    gk_batch* b = nullptr;
    gk_result stats;
    memset(&stats, 0, sizeof stats);
    auto c = e->eng->compiled();
    ProgramLease lease(e, *c);   // flatten + upload + kernel + rendering all against this one snapshot
    upload_batch(e, c, use, total, flags, &b, &stats);
    std::unique_ptr<gk_batch, std::function<void(gk_batch*)>> hold(b, [&](gk_batch* x) {
      e->be->release(x->dev);
      delete x;
    });
    eval_batch(e, b, ep, flags, out);
    out->flatten_ms = stats.flatten_ms;
    out->h2d_ms = stats.h2d_ms;
    out->h2d_bytes = stats.h2d_bytes;
    bool any_expand_err = false;
    for (auto& x : expand_errors) any_expand_err = any_expand_err || !x.empty();
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
    for (auto& v : rp->vio)
      if (v.object >= n) {
        const Child& ch = children[v.object - n];
        v.object = ch.parent;
        v.msg = ExpansionSystem::implied_by(ch.tmpl, v.msg);
        if (!ch.action.empty()) v.action = ch.action;   // OverrideEnforcementAction (aggregate.go:47-58) sets EnforcementAction only: the scoped list stays
      }
    std::stable_sort(rp->vio.begin(), rp->vio.end(), [](const Violation& a, const Violation& b2) { return a.object < b2.object; });
    if (rp->obj_errors.empty() && any_expand_err) rp->obj_errors.assign(total, std::string());
    if (!rp->obj_errors.empty()) {
      for (size_t k = 0; k < children.size(); ++k)
        if (!rp->obj_errors[n + k].empty() && rp->obj_errors[children[k].parent].empty())
          rp->obj_errors[children[k].parent] = ExpansionSystem::implied_by(children[k].tmpl, rp->obj_errors[n + k]);
      rp->obj_errors.resize(n);
      for (size_t i = 0; i < n && i < expand_errors.size(); ++i)
        if (!expand_errors[i].empty() && rp->obj_errors[i].empty()) rp->obj_errors[i] = expand_errors[i];
    }
    const bool give_bits = !(flags & GK_F_NO_COPY_BACK);
    fill_result(out, rp, give_bits);
  });
}

int gk_batch_upload(gk_engine_t* e, const gk_obj* objs, size_t n, uint32_t flags, gk_batch_t** outb, gk_result* stats, char** err) {
  if (!e || !outb || (!objs && n)) return GK_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  return guard(err, [&]() {
    auto c = e->eng->compiled();
    ProgramLease lease(e, *c);
    upload_batch(e, c, objs, n, flags, outb, stats);
  });
}

int gk_batch_eval(gk_engine_t* e, gk_batch_t* b, const char* ep, uint32_t flags, gk_result* out, char** err) {
  if (!e || !b || !out) return GK_ERR_INVALID;
  memset(out, 0, sizeof *out);
  return guard(err, [&]() {
    if (e->eng->has_expansion())   // (bitmaps of the listed objects only: the resultants of generators would be missing, silently)
      throw RegoError{"ExpansionTemplates are registered: this entry point does not expand generator objects -- review them through gk_review_batch, or "
                      "aggregate the batch with gk_audit_add_batch, which do"};
    auto c = e->eng->compiled();
    if (c->version != b->compiled->version) throw RegoError{"batch was flattened against an older constraint set; upload it again"};
    if (c->uses_data) {   // the columns of a referential snapshot hold values computed from data.inventory
      uint64_t dv = 0;
      e->eng->data_doc(&dv);
      if (dv != b->data_version) throw RegoError{"data.inventory changed since the batch was flattened (referential constraints); upload it again"};
    }
    ProgramLease lease(e, *c);
    eval_batch(e, b, ep, flags, out);
  });
}

int gk_batch_eval_device(gk_engine_t* e, gk_batch_t* b, const char* ep, void* d_viol, void* d_err, void* d_totals, void* d_err_totals,
                         void* stream, char** err) {
  if (!e || !b || !d_viol || !d_err || !d_totals || !d_err_totals) return GK_ERR_INVALID;
  return guard(err, [&]() {
    if (e->eng->has_expansion())   // (bitmaps of the listed objects only: the resultants of generators would be missing, silently)
      throw RegoError{"ExpansionTemplates are registered: this entry point does not expand generator objects -- review them through gk_review_batch, or "
                      "aggregate the batch with gk_audit_add_batch, which do"};
    auto c = e->eng->compiled();
    if (c->version != b->compiled->version) throw RegoError{"batch was flattened against an older constraint set; upload it again"};
    if (c->uses_data) {   // the columns of a referential snapshot hold values computed from data.inventory
      uint64_t dv = 0;
      e->eng->data_doc(&dv);
      if (dv != b->data_version) throw RegoError{"data.inventory changed since the batch was flattened (referential constraints); upload it again"};
    }
    ProgramLease lease(e, *c);
    std::vector<uint32_t> active;
    e->eng->active_mask(*c, ep ? ep : "", active);
    DevOutPtrs d;
    d.viol = d_viol;
    d.err = d_err;
    d.totals = d_totals;
    d.err_totals = d_err_totals;
    d.stream = stream;
    e->be->eval_into(b->dev, active, d);
  });
}

int gk_batch_eval_device_peers(gk_engine_t* e, gk_batch_t* b, const char* ep, const uint64_t* peer_bases, uint32_t npeers, uint32_t rank,
                               uint64_t slot_i32, uint64_t tot_off_i32, uint32_t tot_stride, void* d_err, void* d_totals, void* d_err_totals,
                               void* stream, char** err) {
  if (!e || !b || !peer_bases || !npeers || npeers > 8 || rank >= npeers || !d_err || !d_totals || !d_err_totals) return GK_ERR_INVALID;
  return guard(err, [&]() {
    if (e->eng->has_expansion())   // (bitmaps of the listed objects only: the resultants of generators would be missing, silently)
      throw RegoError{"ExpansionTemplates are registered: this entry point does not expand generator objects -- review them through gk_review_batch, or "
                      "aggregate the batch with gk_audit_add_batch, which do"};
    auto c = e->eng->compiled();
    if (c->version != b->compiled->version) throw RegoError{"batch was flattened against an older constraint set; upload it again"};
    if (c->uses_data) {   // the columns of a referential snapshot hold values computed from data.inventory
      uint64_t dv = 0;
      e->eng->data_doc(&dv);
      if (dv != b->data_version) throw RegoError{"data.inventory changed since the batch was flattened (referential constraints); upload it again"};
    }
    ProgramLease lease(e, *c);
    std::vector<uint32_t> active;
    e->eng->active_mask(*c, ep ? ep : "", active);
    DevOutPtrs d;
    d.viol = nullptr;
    d.err = d_err;
    d.totals = d_totals;
    d.err_totals = d_err_totals;
    d.stream = stream;
    d.npeers = npeers;
    d.tot_stride = tot_stride;
    for (uint32_t q = 0; q < npeers; ++q) {
      d.peer_viol[q] = peer_bases[q] + (uint64_t)rank * slot_i32 * 4;
      d.peer_tot[q] = peer_bases[q] + ((uint64_t)rank * slot_i32 + tot_off_i32) * 4;
    }
    e->be->eval_into(b->dev, active, d);
  });
}

int gk_batch_upload_blob(gk_engine_t* e, const char* buf, const uint64_t* offsets, size_t n, uint8_t source, uint32_t flags, gk_batch_t** outb,
                         gk_result* stats, char** err) {
  if (!e || !outb || ((!buf || !offsets) && n)) return GK_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  return guard(err, [&]() {
    auto c = e->eng->compiled();
    ProgramLease lease(e, *c);
    upload_blob(e, c, buf, offsets, n, source, flags, outb, stats);
  });
}

int gk_review_blob(gk_engine_t* e, const char* buf, const uint64_t* offsets, size_t n, uint8_t source, const char* ep, uint32_t flags,
                   gk_result* out, char** err) {
  if (!e || !out || ((!buf || !offsets) && n)) return GK_ERR_INVALID;
  memset(out, 0, sizeof *out);
  return guard(err, [&]() {
    gk_batch* b = nullptr;
    gk_result stats;
    memset(&stats, 0, sizeof stats);
    if (e->eng->has_expansion())   // (bitmaps of the listed objects only: the resultants of generators would be missing, silently)
      throw RegoError{"ExpansionTemplates are registered: this entry point does not expand generator objects -- review them through gk_review_batch, or "
                      "aggregate the batch with gk_audit_add_batch, which do"};
    auto c = e->eng->compiled();
    ProgramLease lease(e, *c);
    upload_blob(e, c, buf, offsets, n, source, flags & ~(uint32_t)GK_F_KEEP_SOURCE, &b, &stats);   // (the batch lives for this call only)
    std::unique_ptr<gk_batch, std::function<void(gk_batch*)>> hold(b, [&](gk_batch* x) {
      e->be->release(x->dev);
      delete x;
    });
    eval_batch(e, b, ep, flags, out);
    out->flatten_ms = stats.flatten_ms;
    out->h2d_ms = stats.h2d_ms;
    out->h2d_bytes = stats.h2d_bytes;
  });
}

uint32_t gk_batch_size(gk_batch_t* b) { return b ? b->n : 0; }
uint64_t gk_batch_alg_bytes(gk_batch_t* b) { return b ? b->alg_bytes : 0; }
void gk_batch_free(gk_engine_t* e, gk_batch_t* b) {
  if (!e || !b) return;
  guard(nullptr, [&]() { e->be->release(b->dev); });
  guard(nullptr, [&]() { e->be->release_source(b->source); });
  delete b;
}

int gk_batch_refresh(gk_engine_t* e, gk_batch_t* b, gk_result* stats, char** err) {
  if (!e || !b) return GK_ERR_INVALID;
  if (stats) memset(stats, 0, sizeof *stats);
  bool rebuilt = false;
  const int rc = guard(err, [&]() {
    auto c = e->eng->compiled();
    const std::vector<std::string> excluded = excluded_of(e, b->flags);
    uint64_t dv = 0;
    if (c->uses_data) e->eng->data_doc(&dv);
    if (c->version == b->compiled->version && excluded == b->excluded && (!c->uses_data || dv == b->data_version)) {
      if (stats) {
        stats->alg_bytes = b->alg_bytes;
        stats->n_objects = b->n;
        stats->n_constraints = (uint32_t)c->cons_match.size();
      }
      return;
    }
    ProgramLease lease(e, *c);
    gk_batch* nb = nullptr;
    if (!b->blob) upload_batch(e, c, b->objs.data(), b->objs.size(), b->flags, &nb, stats);
    else if (b->source && device_ingest(*c, b->n)) refresh_from_source(e, c, b, &nb, stats);
    else upload_blob(e, c, b->blob, b->blob_off, b->n, b->blob_source, b->flags, &nb, stats);
    // the new columns replace the old ones; a kept source stays with the batch (a batch that had none may have gained one)
    if (!nb->source) {
      std::swap(nb->source, b->source);
      std::swap(nb->source_errors, b->source_errors);
    }
    std::swap(*b, *nb);
    e->be->release(nb->dev);
    delete nb;
    rebuilt = true;
  });
  return rc == GK_OK && rebuilt ? 1 : rc;
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
  float select_ms = 0.f;   // device time of the last gk_audit_add_batch_ordered's ranking and selection
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

// gk_audit_add_batch and gk_audit_add_batch_ordered: `ordered` takes the lazy path's candidates from Backend::audit_candidates (any mix
// of kinds) instead of the host threshold scan over (namespace, name), which only a page of one kind allows
static int audit_add(gk_audit_t* a, gk_batch_t* b, const char* ep_c, bool ordered, char** err) {
  if (!a || !b) return GK_ERR_INVALID;
  return guard(err, [&]() {
    gk_engine* e = a->e;
    auto c = e->eng->compiled();
    if (c->version != b->compiled->version) throw RegoError{"batch was flattened against an older constraint set; upload it again"};
    if (c->uses_data) {   // the columns of a referential snapshot hold values computed from data.inventory
      uint64_t dv = 0;
      e->eng->data_doc(&dv);
      if (dv != b->data_version) throw RegoError{"data.inventory changed since the batch was flattened (referential constraints); upload it again"};
    }
    std::string ep = ep_c ? ep_c : "";
    std::vector<uint32_t> active;
    e->eng->active_mask(*c, ep, active);
    EvalOut ev, ev_amb;
    {
      ProgramLease lease(e, *c);
      e->be->eval(b->dev, active, ev, true);
    }
    std::vector<ObjIn> ins(b->n);
    for (size_t i = 0; i < ins.size(); ++i) ins[i] = b->obj_in(i);
    // The lazy path (audit.hpp): the namespace / name arrays of the batch and the bitmap of the ambiguity netlist let the run count
    // the pairs that have exactly one result and evaluate only what can still enter a constraint's list.
    BatchIdentity id;
    const bool lazy = !getenv("GK_AUDIT_EAGER") && (c->amb || std::any_of(c->single_result.begin(), c->single_result.end(), [](uint8_t x) { return x != 0; }));
    if (lazy && !ordered) e->be->identity(b->dev, id);
    const bool use_amb = lazy && (ordered || id.uniform_gvk) && c->amb && !getenv("GK_AUDIT_NO_AMB");
    if (use_amb) {
      ProgramLease lease(e, *c->amb);   // (the backend holds one netlist at a time: waits until no review uses the other)
      void* fork = e->be->fork_batch(b->dev, *c->amb);
      try {
        e->be->eval(fork, active, ev_amb, true);
      } catch (...) {
        e->be->release(fork);
        throw;
      }
      e->be->release(fork);
    }
    // ---- expansion inside the audit loop (pkg/audit/manager.go:733-765): every reviewed object is expanded; its resultants are reviewed
    // as Generated resources with the parent's Namespace, their results -- "[Implied by <template>]", the template's action override --
    // are the PARENT's results (addAuditResponsesToUpdateLists names the parent object).  An object whose expansion fails contributes
    // nothing at all, not even its own violations (the reference logs the error and `continue`s past the bookkeeping of the response).
    std::vector<std::string> obj_errs = b->host->obj_errors.empty() ? std::vector<std::string>(b->n) : b->host->obj_errors;
    obj_errs.resize(b->n);
    struct Child {
      uint32_t parent;
      std::string json, tmpl, action;
    };
    std::vector<Child> children;
    if (e->eng->has_expansion() && b->n) {
      const size_t T = std::min<size_t>((size_t)std::max(1, e->eng->threads()), std::max<size_t>(1, b->n / 256));
      std::vector<std::vector<Child>> part(T);
      std::vector<std::vector<std::pair<uint32_t, std::string>>> perr(T);
      auto work = [&](size_t t) {
        std::vector<Resultant> res;
        for (uint32_t i = (uint32_t)((size_t)b->n * t / T); i < (uint32_t)((size_t)b->n * (t + 1) / T); ++i) {
          if (!obj_errs[i].empty()) continue;   // (the review of the object itself failed: the reference never gets to its expansion)
          res.clear();
          try {
            e->eng->expand_object(ins[i], res);
          } catch (std::exception& x) {
            perr[t].emplace_back(i, std::string("unable to expand object: ") + x.what());
            continue;
          }
          for (auto& r : res) part[t].push_back(Child{i, json_str(r.obj), r.template_name, r.action});
        }
      };
      if (T == 1) work(0);
      else {
        std::vector<std::thread> th;
        for (size_t t = 0; t < T; ++t) th.emplace_back(work, t);
        for (auto& x : th) x.join();
      }
      const uint32_t W = ev.words;
      for (auto& pe : perr)
        for (auto& x : pe) {
          obj_errs[x.first] = x.second;
          for (uint32_t w = 0; w < W; ++w) {
            if (!ev.viol.empty()) ev.viol[(size_t)x.first * W + w] = 0;
            if (!ev.err.empty()) ev.err[(size_t)x.first * W + w] = 0;
          }
        }
      for (auto& p : part) children.insert(children.end(), std::make_move_iterator(p.begin()), std::make_move_iterator(p.end()));
    }
    // (after the expansion above: the rows of objects whose expansion failed are cleared, and they are no candidates either)
    std::vector<uint32_t> cand;
    if (lazy && ordered) {
      auto gvk_of = [&ins](uint32_t o, std::string& g, std::string& v, std::string& k) {
        try {
          split_gv(json_parse(ins[o].json, ins[o].len), g, v, k);
        } catch (JsonError&) {
        }
      };
      e->be->audit_candidates(b->dev, ev.viol.data(), ev.words, (uint32_t)c->order.size(), (uint32_t)a->run.limit, gvk_of, cand, &a->select_ms);
    }
    a->run.add_batch(*e->eng, *c, ins, ev.viol.data(), ev.err.empty() ? nullptr : ev.err.data(), ev.words, ev.errlist, ep,
                     lazy && !ordered ? &id : nullptr, use_amb ? ev_amb.viol.data() : nullptr, lazy && ordered ? cand.data() : nullptr);
    if (!children.empty()) {
      std::vector<gk_obj> cobjs(children.size());
      for (size_t k = 0; k < children.size(); ++k) {
        gk_obj& o = cobjs[k];
        memset(&o, 0, sizeof o);
        o.json = children[k].json.data();
        o.len = children[k].json.size();
        const ObjIn& par = ins[children[k].parent];
        o.ns_json = par.ns_json;                // the parent's Namespace object (manager.go:745-749), source Generated
        o.ns_len = par.ns_len;
        o.ns_name = par.ns_name;
        o.source = GK_SOURCE_GENERATED;
      }
      gk_batch* cb = nullptr;
      gk_result cstats, cres;
      memset(&cstats, 0, sizeof cstats);
      memset(&cres, 0, sizeof cres);
      {
        ProgramLease lease(e, *c);
        upload_batch(e, c, cobjs.data(), cobjs.size(), b->flags, &cb, &cstats);
        std::unique_ptr<gk_batch, std::function<void(gk_batch*)>> hold(cb, [&](gk_batch* x) {
          e->be->release(x->dev);
          delete x;
        });
        eval_batch(e, cb, ep_c, GK_F_MATERIALIZE | GK_F_NO_COPY_BACK, &cres);
      }
      std::unique_ptr<ResultPriv> crp(static_cast<ResultPriv*>(cres.priv));
      cres.priv = nullptr;
      struct Ident {
        std::string g, v, k, ns, name;
      };
      std::unordered_map<uint32_t, Ident> ident;   // parents that have results from resultants
      for (auto& v : crp->vio) {
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
        const Constraint& con = *c->order[v.constraint];
        StatusViolation sv;
        sv.group = it->second.g, sv.version = it->second.v, sv.kind = it->second.k, sv.ns = it->second.ns, sv.name = it->second.name;
        sv.message = ExpansionSystem::implied_by(ch.tmpl, v.msg);
        sv.action = ch.action.empty() ? v.action : ch.action;   // OverrideEnforcementAction: the action only
        sv.scoped_json = v.scoped_json;
        a->run.fold(con.kind + "/" + con.name, std::move(sv));
        a->run.results++;
      }
      // a resultant the review refused (manager.go:757-760 logs it and goes on): reported on its parent
      for (size_t k = 0; k < crp->obj_errors.size() && k < children.size(); ++k)
        if (!crp->obj_errors[k].empty() && obj_errs[children[k].parent].empty())
          obj_errs[children[k].parent] = ExpansionSystem::implied_by(children[k].tmpl, crp->obj_errors[k]);
    }
    a->run.add_object_errors(obj_errs);
  });
}

int gk_audit_add_batch(gk_audit_t* a, gk_batch_t* b, const char* ep, char** err) { return audit_add(a, b, ep, false, err); }

int gk_audit_add_batch_ordered(gk_audit_t* a, gk_batch_t* b, const char* ep, char** err) { return audit_add(a, b, ep, true, err); }

float gk_audit_select_ms(gk_audit_t* a) { return a ? a->select_ms : 0.f; }

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
