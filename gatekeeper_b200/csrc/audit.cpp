// Audit-sweep aggregation and admission message assembly: the host work the reference does around Client.Review.
//
//   AuditRun            addAuditResponsesToUpdateLists   pkg/audit/manager.go:886-945
//   LimitQueue / sv_less LimitQueue, SVQueue.Less        pkg/audit/manager.go:117-202
//   truncate_string     truncateString                   pkg/audit/manager.go:1043-1052
//   report()            updateConstraintStatus           pkg/audit/manager.go:984-1041 (pops the heap: descending order)
//   validation_messages getValidationMessages            pkg/webhook/policy.go:238-355
//
// The kernel has already decided which (constraint, object) pairs violate; this code renders the messages of the flagged
// pairs (all host cores), counts results and keeps the K smallest per constraint.
#include "audit.hpp"

#include <algorithm>
#include <thread>

#include "val.hpp"

namespace gk {

std::string truncate_string(const std::string& s, size_t size) {
  if (s.size() <= size) return s;
  if (size > 3) size -= 3;
  return s.substr(0, size) + "...";
}

// SVQueue.Less is "greater than" so that Go's min-heap pops the LARGEST; sv_less is the natural order underneath it.
bool sv_less(const StatusViolation& a, const StatusViolation& b) {
  if (a.group != b.group) return a.group < b.group;
  if (a.version != b.version) return a.version < b.version;
  if (a.kind != b.kind) return a.kind < b.kind;
  if (a.ns != b.ns) return a.ns < b.ns;
  if (a.name != b.name) return a.name < b.name;
  if (a.message != b.message) return a.message < b.message;
  return a.action < b.action;
}

void LimitQueue::push(StatusViolation v) {
  if (limit == 0) return;
  if (heap.size() >= limit && !sv_less(v, heap.front())) return;   // would be popped straight away
  heap.push_back(std::move(v));
  std::push_heap(heap.begin(), heap.end(), sv_less);
  while (heap.size() > limit) {
    std::pop_heap(heap.begin(), heap.end(), sv_less);
    heap.pop_back();
  }
}

std::vector<StatusViolation> LimitQueue::drain_descending() {
  std::vector<StatusViolation> out;
  while (!heap.empty()) {
    std::pop_heap(heap.begin(), heap.end(), sv_less);
    out.push_back(std::move(heap.back()));
    heap.pop_back();
  }
  return out;
}

void AuditRun::fold(const std::string& key, StatusViolation sv) {
  auto& pc = per_constraint[key];
  if (pc.queue.limit != limit) pc.queue.limit = limit;
  pc.total++;
  by_action[sv.action]++;
  sv.message = truncate_string(sv.message, msg_size);
  pc.queue.push(std::move(sv));
}

void AuditRun::merge(AuditRun& o) {
  for (auto& kv : o.per_constraint) {
    auto& pc = per_constraint[kv.first];
    pc.queue.limit = limit;
    pc.total += kv.second.total;
    for (auto& sv : kv.second.queue.heap) pc.queue.push(std::move(sv));
  }
  for (auto& kv : o.by_action) by_action[kv.first] += kv.second;
  objects += o.objects;
  results += o.results;
  rendered_pairs += o.rendered_pairs;
  counted_pairs += o.counted_pairs;
  for (auto& fe : o.first_object_errors)
    if (first_object_errors.size() < 20) first_object_errors.emplace_back(seen_objects + fe.first, fe.second);
  object_errors += o.object_errors;
  seen_objects += o.seen_objects;
}

namespace {
// (namespace, name) of object o as the reference orders results (SVQueue.Less after group / version / kind): a Namespace's own
// namespace is empty; the header's nsname is the object's metadata.namespace otherwise
struct IdView {
  const BatchIdentity& id;
  void get(uint32_t o, const uint8_t*& ns, uint32_t& nsl, const uint8_t*& nm, uint32_t& nml) const {
    const uint32_t fl = id.flags[o];
    if ((fl & GK_F_IS_NS) || !(fl & GK_F_NSNAME)) ns = nullptr, nsl = 0;
    else ns = id.ns_bytes.data() + id.ns_off[o], nsl = id.ns_off[o + 1] - id.ns_off[o];
    nm = id.name_bytes.data() + id.name_off[o];
    nml = id.name_off[o + 1] - id.name_off[o];
  }
  static int cmp_bytes(const uint8_t* a, uint32_t al, const uint8_t* b, uint32_t bl) {
    const int r = memcmp(a, b, std::min(al, bl));
    return r ? r : (al < bl ? -1 : al > bl ? 1 : 0);
  }
  int cmp(uint32_t a, uint32_t b) const {
    const uint8_t *ans, *anm, *bns, *bnm;
    uint32_t ansl, anml, bnsl, bnml;
    get(a, ans, ansl, anm, anml);
    get(b, bns, bnsl, bnm, bnml);
    const int r = cmp_bytes(ans, ansl, bns, bnsl);
    return r ? r : cmp_bytes(anm, anml, bnm, bnml);
  }
};
}  // namespace

bool HostCandidates::operator()(uint32_t o, uint32_t c) const { return thr_all[c] || IdView{*id}.cmp(o, thr_obj[c]) <= 0; }

void AuditRun::add_counted(const std::string& key, const std::string& action, uint64_t n) {
  auto& pc = per_constraint[key];
  pc.queue.limit = limit;
  pc.total += n;
  by_action[action] += n;
  results += n;
}

void AuditRun::add_batch(Engine& eng, const Compiled& c, const std::vector<ObjIn>& objs, const uint32_t* viol, const uint32_t* err,
                         uint32_t words, const std::vector<uint32_t>& errlist, const std::string& ep, const BatchIdentity* id, const uint32_t* amb,
                         const uint32_t* cand, HostCandidates* keep) {
  const size_t n = objs.size();
  const uint32_t C = (uint32_t)c.order.size();
  // ---- lazy path: which pairs need the host at all
  // the candidates of c = the objects whose results can still enter constraint c's list.  Constraints that may have several results
  // per pair are evaluated for every pair (their totals count results: pkg/audit/manager.go:886-945).
  const bool lazy = (cand || (id && id->uniform_gvk && id->flags.size() == n)) &&
                    (amb || std::any_of(c.single_result.begin(), c.single_result.end(), [](uint8_t x) { return x != 0; }));
  if (cand) id = nullptr;   // (the candidate bitmap replaces the threshold scan below)
  // exactly one result for a violating pair: proven for the constraint when it was lowered, or for this pair by the ambiguity bitmap
  auto one_result = [&](size_t o, uint32_t cix) { return c.single_result[cix] || (amb && !(amb[o * words + (cix >> 5)] >> (cix & 31u) & 1u)); };
  std::vector<uint32_t> thr_obj(C, 0);     // per single-result constraint: an object holding the limit-th smallest identity
  std::vector<uint8_t> thr_all(C, 1);      // fewer than `limit` flagged objects: all are candidates
  if (lazy && limit && !cand) {
    const IdView iv{*id};
    const size_t TT = std::min<size_t>((size_t)std::max(1, eng.threads()), std::max<size_t>(1, n / 4096));
    // per thread, per constraint: max-heap of the `limit` smallest objects seen
    std::vector<std::vector<std::vector<uint32_t>>> heaps(TT, std::vector<std::vector<uint32_t>>(C));
    auto less = [&](uint32_t a, uint32_t b) { return iv.cmp(a, b) < 0; };
    auto scan = [&](size_t t) {
      auto& hp = heaps[t];
      const size_t lo = n * t / TT, hi = n * (t + 1) / TT;
      for (size_t o = lo; o < hi; ++o)
        for (uint32_t w = 0; w < words; ++w) {
          uint32_t vb = viol[o * words + w];
          while (vb) {
            const uint32_t k = (uint32_t)__builtin_ctz(vb);
            vb &= vb - 1;
            const uint32_t cix = w * 32 + k;
            if (cix >= C) continue;
            auto& h = hp[cix];
            if (h.size() < limit) {
              h.push_back((uint32_t)o);
              std::push_heap(h.begin(), h.end(), less);
            } else if (less((uint32_t)o, h.front())) {
              std::pop_heap(h.begin(), h.end(), less);
              h.back() = (uint32_t)o;
              std::push_heap(h.begin(), h.end(), less);
            }
          }
        }
    };
    if (TT == 1) scan(0);
    else {
      std::vector<std::thread> th;
      for (size_t t = 0; t < TT; ++t) th.emplace_back(scan, t);
      for (auto& x : th) x.join();
    }
    for (uint32_t cix = 0; cix < C; ++cix) {
      std::vector<uint32_t> all;
      for (size_t t = 0; t < TT; ++t) all.insert(all.end(), heaps[t][cix].begin(), heaps[t][cix].end());
      if (all.size() < limit) continue;
      std::nth_element(all.begin(), all.begin() + (long)(limit - 1), all.end(), less);
      thr_obj[cix] = all[limit - 1];
      thr_all[cix] = 0;
    }
  }
  if (keep) {
    keep->lazy = lazy && limit && !cand;
    keep->id = id;
    keep->thr_obj = thr_obj;
    keep->thr_all = thr_all;
  }
  std::unordered_map<uint64_t, uint32_t> err_code;
  for (size_t i = 0; i + 2 < errlist.size(); i += 3) err_code[((uint64_t)errlist[i] << 32) | errlist[i + 1]] = errlist[i + 2];
  size_t T = std::min<size_t>((size_t)std::max(1, eng.threads()), std::max<size_t>(1, n / 64));
  std::vector<AuditRun> parts(T);
  std::vector<std::string> errs(T);
  std::atomic<size_t> next{0};
  auto work = [&](size_t t) {
    AuditRun& part = parts[t];
    part.limit = limit;
    part.msg_size = msg_size;
    std::vector<Engine::Flagged> flagged;
    std::vector<Violation> vio;
    Engine::MaterializeCtx mctx;
    std::vector<uint64_t> counted(C, 0);   // pairs of single-result constraints taken from the bitmap
    try {
      for (;;) {
        size_t lo = next.fetch_add(256), hi = std::min(n, lo + 256);
        if (lo >= n) break;
        for (size_t o = lo; o < hi; ++o) {
          flagged.clear();
          for (uint32_t w = 0; w < words; ++w) {
            uint32_t vb = viol[o * words + w], eb = err ? err[o * words + w] : 0u;
            uint32_t any = vb | eb;
            while (any) {
              uint32_t k = (uint32_t)__builtin_ctz(any);
              any &= any - 1;
              uint32_t cix = w * 32 + k;
              if (cix >= C) continue;
              bool is_err = eb >> k & 1u;
              if (lazy && !is_err && one_result(o, cix)) {
                // one result per pair: counted here; evaluated only if the object can still enter the constraint's list
                const bool candidate = limit && (cand ? (cand[o * words + w] >> k & 1u) != 0
                                                      : (thr_all[cix] || IdView{*id}.cmp((uint32_t)o, thr_obj[cix]) <= 0));
                if (!candidate) {
                  ++counted[cix];
                  continue;
                }
              }
              part.rendered_pairs++;
              uint32_t code = 0;
              if (is_err) {
                auto it = err_code.find(((uint64_t)o << 32) | c.cons_match[cix]);
                if (it != err_code.end()) code = it->second;
              }
              flagged.push_back({cix, is_err, code});
            }
          }
          if (flagged.empty()) continue;
          vio.clear();
          VP obj;
          eng.materialize_object(c, objs[o], (uint32_t)o, flagged, ep, vio, &obj, &mctx);
          std::string g, v, k, ns, name;
          if (obj) {
            split_gv(obj, g, v, k);
            ns = meta_str(obj, "namespace");
            name = meta_str(obj, "name");
          }
          for (auto& x : vio) {
            const Constraint& con = *c.order[x.constraint];
            StatusViolation sv;
            sv.group = g, sv.version = v, sv.kind = k, sv.ns = ns, sv.name = name;
            sv.message = std::move(x.msg);
            sv.action = x.action;
            sv.scoped_json = std::move(x.scoped_json);
            part.fold(con.kind + "/" + con.name, std::move(sv));
            part.results++;
          }
        }
      }
    } catch (RegoError& e) {
      errs[t] = e.msg;
    } catch (std::exception& e) {
      errs[t] = e.what();
    }
    for (uint32_t cix = 0; cix < C; ++cix)
      if (counted[cix]) {
        const Constraint& con = *c.order[cix];
        part.add_counted(con.kind + "/" + con.name, con.action, counted[cix]);
        part.counted_pairs += counted[cix];
      }
  };
  if (T == 1) work(0);
  else {
    std::vector<std::thread> th;
    for (size_t t = 0; t < T; ++t) th.emplace_back(work, t);
    for (auto& x : th) x.join();
  }
  for (auto& e : errs)
    if (!e.empty()) throw RegoError{"audit: " + e};
  for (auto& p : parts) merge(p);
  objects += n;
}

// Backend::audit_candidates on the host: the flagged objects sorted by (group, version, kind, namespace, name), then per constraint
// the rank of its limit-th flagged object bounds its candidates.  With `keep`, every object is ranked, flagged or not.
void Backend::audit_candidates(void* batch, const uint32_t* viol, uint32_t words, uint32_t nconstraints, uint32_t limit, const GvkOf& gvk_of,
                               std::vector<uint32_t>& cand, float* device_ms, AuditRanks* keep) {
  if (device_ms) *device_ms = 0.f;
  BatchIdentity id;
  identity(batch, id);
  const size_t n = id.flags.size();
  cand.assign(n * words, 0u);
  const IdView iv{id};
  auto bit = [&](uint32_t o, uint32_t cix) { return (viol[(size_t)o * words + (cix >> 5)] >> (cix & 31u) & 1u) != 0; };
  struct Flagged {
    uint32_t o;
    std::string g, v, k;
  };
  std::vector<Flagged> fl;
  auto flagged = [&](uint32_t o) {
    for (uint32_t cix = 0; cix < nconstraints; ++cix)
      if (bit(o, cix)) return true;
    return false;
  };
  for (uint32_t o = 0; o < n; ++o)
    if (keep || flagged(o)) {
      fl.push_back({o, {}, {}, {}});
      gvk_of(o, fl.back().g, fl.back().v, fl.back().k);
    }
  auto cmp = [&](const Flagged& a, const Flagged& b) {
    if (a.g != b.g) return a.g < b.g ? -1 : 1;
    if (a.v != b.v) return a.v < b.v ? -1 : 1;
    if (a.k != b.k) return a.k < b.k ? -1 : 1;
    return iv.cmp(a.o, b.o);
  };
  std::sort(fl.begin(), fl.end(), [&](const Flagged& a, const Flagged& b) { return cmp(a, b) < 0; });
  std::vector<uint32_t> rank(fl.size(), 0);
  for (size_t p = 1; p < fl.size(); ++p) rank[p] = rank[p - 1] + (cmp(fl[p - 1], fl[p]) != 0);
  if (keep) {
    keep->rank.assign(n, 0);
    keep->thr.assign(nconstraints, ~0u);
    keep->dev.reset();
    for (size_t p = 0; p < fl.size(); ++p) keep->rank[fl[p].o] = rank[p];
  }
  for (uint32_t cix = 0; cix < nconstraints; ++cix) {
    uint32_t seen = 0, thr = ~0u;
    for (size_t p = 0; p < fl.size() && thr == ~0u; ++p)
      if (bit(fl[p].o, cix) && ++seen == limit) thr = rank[p];
    for (size_t p = 0; p < fl.size() && rank[p] <= thr; ++p)
      if (bit(fl[p].o, cix)) cand[(size_t)fl[p].o * words + (cix >> 5)] |= 1u << (cix & 31u);
    if (keep) keep->thr[cix] = thr;
  }
}

// ---- export / import of a run's partial state (gk_audit_export / gk_audit_merge)
//   "GKAUDIT\0", u32 format version, the fields in declaration order (integers u64 little-endian, strings as u64 length + bytes),
//   then an FNV-1a 64 checksum of every byte before it
namespace {
constexpr char kRunMagic[8] = {'G', 'K', 'A', 'U', 'D', 'I', 'T', '\0'};
constexpr uint32_t kRunFormat = 1;
uint64_t fnv64(const uint8_t* p, size_t n) {
  uint64_t h = 1469598103934665603ull;
  for (size_t i = 0; i < n; ++i) h = (h ^ p[i]) * 1099511628211ull;
  return h;
}
struct Writer {
  std::string s;
  void u64(uint64_t x) {
    for (int i = 0; i < 8; ++i) s.push_back((char)(x >> (8 * i) & 0xffu));
  }
  void str(const std::string& x) {
    u64(x.size());
    s += x;
  }
};
struct Reader {
  const uint8_t* p;
  size_t n, at = 0;
  void need(uint64_t k) {
    if (k > n - at) throw RegoError{"audit merge: the buffer is truncated"};
  }
  uint64_t u64() {
    need(8);
    uint64_t x = 0;
    for (int i = 0; i < 8; ++i) x |= (uint64_t)p[at + i] << (8 * i);
    at += 8;
    return x;
  }
  std::string str() {
    const uint64_t k = u64();
    need(k);
    std::string x(reinterpret_cast<const char*>(p + at), (size_t)k);
    at += (size_t)k;
    return x;
  }
  uint64_t count(uint64_t min_bytes_each) {   // an element count that the remaining bytes can hold
    const uint64_t k = u64();
    if (min_bytes_each && k > (n - at) / min_bytes_each) throw RegoError{"audit merge: the buffer is truncated"};
    return k;
  }
};
}  // namespace

std::string AuditRun::serialize() const {
  Writer w;
  w.s.assign(kRunMagic, sizeof kRunMagic);
  for (int i = 0; i < 4; ++i) w.s.push_back((char)(kRunFormat >> (8 * i) & 0xffu));
  for (uint64_t x : {(uint64_t)limit, (uint64_t)msg_size, objects, results, rendered_pairs, counted_pairs, object_errors, seen_objects}) w.u64(x);
  w.u64(first_object_errors.size());
  for (auto& fe : first_object_errors) w.u64(fe.first), w.str(fe.second);
  w.u64(by_action.size());
  for (auto& kv : by_action) w.str(kv.first), w.u64(kv.second);
  w.u64(per_constraint.size());
  for (auto& kv : per_constraint) {
    w.str(kv.first);
    w.u64(kv.second.total);
    w.u64(kv.second.queue.heap.size());
    for (auto& sv : kv.second.queue.heap)
      for (const std::string* f : {&sv.group, &sv.version, &sv.kind, &sv.ns, &sv.name, &sv.message, &sv.action, &sv.scoped_json}) w.str(*f);
  }
  w.u64(fnv64(reinterpret_cast<const uint8_t*>(w.s.data()), w.s.size()));
  return w.s;
}

AuditRun AuditRun::parse(const uint8_t* buf, size_t len) {
  if (!buf || len < sizeof kRunMagic + 4 + 8) throw RegoError{"audit merge: the buffer is truncated"};
  if (memcmp(buf, kRunMagic, sizeof kRunMagic) != 0) throw RegoError{"audit merge: not an exported audit run"};
  uint32_t format = 0;
  for (int i = 0; i < 4; ++i) format |= (uint32_t)buf[sizeof kRunMagic + i] << (8 * i);
  if (format != kRunFormat)
    throw RegoError{"audit merge: export format " + std::to_string(format) + ", this library reads format " + std::to_string(kRunFormat)};
  uint64_t sum = 0;
  for (int i = 0; i < 8; ++i) sum |= (uint64_t)buf[len - 8 + i] << (8 * i);
  if (sum != fnv64(buf, len - 8)) throw RegoError{"audit merge: checksum mismatch (the buffer is truncated or corrupted)"};
  Reader r{buf, len - 8, sizeof kRunMagic + 4};
  AuditRun run;
  run.limit = (size_t)r.u64();
  run.msg_size = (size_t)r.u64();
  run.objects = r.u64(), run.results = r.u64(), run.rendered_pairs = r.u64(), run.counted_pairs = r.u64();
  run.object_errors = r.u64(), run.seen_objects = r.u64();
  for (uint64_t i = 0, k = r.count(16); i < k; ++i) {
    const uint64_t at = r.u64();
    run.first_object_errors.emplace_back(at, r.str());
  }
  for (uint64_t i = 0, k = r.count(16); i < k; ++i) {
    std::string a = r.str();
    run.by_action[a] = r.u64();
  }
  for (uint64_t i = 0, k = r.count(24); i < k; ++i) {
    auto& pc = run.per_constraint[r.str()];
    pc.queue.limit = run.limit;
    pc.total = r.u64();
    for (uint64_t j = 0, m = r.count(64); j < m; ++j) {
      StatusViolation sv;
      for (std::string* f : {&sv.group, &sv.version, &sv.kind, &sv.ns, &sv.name, &sv.message, &sv.action, &sv.scoped_json}) *f = r.str();
      pc.queue.heap.push_back(std::move(sv));
    }
    if (pc.queue.heap.size() > run.limit || !std::is_heap(pc.queue.heap.begin(), pc.queue.heap.end(), sv_less))
      throw RegoError{"audit merge: a status list of the buffer is not a limit queue"};
  }
  if (r.at != r.n) throw RegoError{"audit merge: trailing bytes after the run"};
  return run;
}

static void sv_json(const StatusViolation& sv, std::string& o) {
  // StatusViolation's JSON tags -- pkg/audit/manager.go:100-109 (namespace and enforcementActions are omitempty)
  o += "{\"group\":";
  json_quote(sv.group, o);
  o += ",\"version\":";
  json_quote(sv.version, o);
  o += ",\"kind\":";
  json_quote(sv.kind, o);
  o += ",\"name\":";
  json_quote(sv.name, o);
  if (!sv.ns.empty()) {
    o += ",\"namespace\":";
    json_quote(sv.ns, o);
  }
  o += ",\"message\":";
  json_quote(sv.message, o);
  o += ",\"enforcementAction\":";
  json_quote(sv.action, o);
  if (!sv.scoped_json.empty() && sv.scoped_json != "[]") o += ",\"enforcementActions\":" + sv.scoped_json;
  o += "}";
}

void AuditRun::add_object_errors(const std::vector<std::string>& errs) {
  for (size_t i = 0; i < errs.size(); ++i)
    if (!errs[i].empty()) {
      if (first_object_errors.size() < 20) first_object_errors.emplace_back(seen_objects + i, errs[i]);
      ++object_errors;
    }
  seen_objects += errs.size();
}

std::string AuditRun::report() {
  std::string o = "{\"objects\":" + std::to_string(objects) + ",\"results\":" + std::to_string(results) + ",\"pairsEvaluated\":" + std::to_string(rendered_pairs) +
                  ",\"pairsCounted\":" + std::to_string(counted_pairs) + ",\"objectErrors\":{\"count\":" +
                  std::to_string(object_errors) + ",\"first\":[";
  for (size_t i = 0; i < first_object_errors.size(); ++i) {
    if (i) o += ",";
    o += "{\"object\":" + std::to_string(first_object_errors[i].first) + ",\"error\":";
    json_quote(first_object_errors[i].second, o);
    o += "}";
  }
  o += "]},\"totalViolations\":{";
  bool first = true;
  for (auto& kv : per_constraint) {
    if (!first) o += ",";
    first = false;
    json_quote(kv.first, o);
    o += ":" + std::to_string(kv.second.total);
  }
  o += "},\"totalViolationsPerEnforcementAction\":{";
  first = true;
  for (auto& kv : by_action) {
    if (!first) o += ",";
    first = false;
    json_quote(kv.first, o);
    o += ":" + std::to_string(kv.second);
  }
  o += "},\"violations\":{";
  first = true;
  for (auto& kv : per_constraint) {
    if (!first) o += ",";
    first = false;
    json_quote(kv.first, o);
    o += ":[";
    LimitQueue q = kv.second.queue;   // reporting does not consume the run
    auto list = q.drain_descending();
    for (size_t i = 0; i < list.size(); ++i) {
      if (i) o += ",";
      sv_json(list[i], o);
    }
    o += "]";
  }
  o += "}}";
  return o;
}

// getValidationMessages -- pkg/webhook/policy.go:238-355: per result, the effective actions are the scoped actions for
// the webhook enforcement point (results with none are dropped) or the constraint's own action; unsupported actions are
// skipped (ValidateEnforcementAction, pkg/util/enforcement_action.go:60-70); "deny" -> denyMsgs, "warn" -> warnMsgs,
// each formatted "[<constraint name>] <msg>".
void validation_messages(const Compiled& c, const std::vector<Violation>& vio, uint32_t object, std::vector<std::string>& deny,
                         std::vector<std::string>& warn) {
  auto supported = [](const std::string& a) { return a == "deny" || a == "dryrun" || a == "warn"; };
  // results are in object order: binary-search the object's range
  auto lo = std::lower_bound(vio.begin(), vio.end(), object, [](const Violation& v, uint32_t o) { return v.object < o; });
  for (auto it = lo; it != vio.end() && it->object == object; ++it) {
    const Violation& x = *it;
    const Constraint& con = *c.order[x.constraint];
    std::vector<std::string> actions;
    if (x.action == "scoped") {
      // each action listed for this enforcement point is validated on its own; unsupported ones are skipped
      VP arr = json_parse(x.scoped_json.data(), x.scoped_json.size());
      for (auto& a : arr->items)
        if (supported(a->s)) actions.push_back(a->s);
      if (actions.empty()) continue;
    } else {
      if (!supported(x.action)) continue;
      actions.push_back(x.action);
    }
    for (auto& a : actions) {
      if (a == "deny") deny.push_back("[" + con.name + "] " + x.msg);
      if (a == "warn") warn.push_back("[" + con.name + "] " + x.msg);
    }
  }
}

}  // namespace gk
