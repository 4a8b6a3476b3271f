// Host-side aggregation around the batch review: audit status lists and admission messages (see audit.cpp).
#pragma once
#include <map>
#include <string>
#include <vector>

#include "backend.hpp"
#include "engine.hpp"

namespace gk {

// StatusViolation -- pkg/audit/manager.go:99-109
struct StatusViolation {
  std::string group, version, kind, ns, name, message, action;
  std::string scoped_json;   // EnforcementActions as a JSON array ("[]" / "" when none)
};

std::string truncate_string(const std::string& s, size_t size);
bool sv_less(const StatusViolation& a, const StatusViolation& b);

// LimitQueue -- pkg/audit/manager.go:161-202: keeps the `limit` smallest violations (max-heap, largest on top)
struct LimitQueue {
  size_t limit = 20;
  std::vector<StatusViolation> heap;
  void push(StatusViolation v);
  std::vector<StatusViolation> drain_descending();
};

// The host threshold scan's candidate rule, as one add_batch over a page of one kind computed it: object o (identity in `id`) can still
// enter constraint c's list.  `lazy`: the scan ran; otherwise add_batch rendered every pair and there is no rule.
struct HostCandidates {
  bool lazy = false;
  const BatchIdentity* id = nullptr;
  std::vector<uint32_t> thr_obj;
  std::vector<uint8_t> thr_all;
  bool operator()(uint32_t o, uint32_t c) const;
};

struct AuditRun {
  size_t limit = 20;      // --constraint-violations-limit (manager.go:64)
  size_t msg_size = 256;  // msgSize (manager.go:48)
  struct PerConstraint {
    uint64_t total = 0;
    LimitQueue queue;
  };
  std::map<std::string, PerConstraint> per_constraint;   // key: "Kind/name"
  std::map<std::string, uint64_t> by_action;
  uint64_t objects = 0, results = 0;
  // objects the review refused (undecodable JSON, kind missing ...): counted and the first few kept, so that a sweep never
  // under-reports silently (the reference logs them per object: pkg/audit/manager.go:722-729)
  uint64_t object_errors = 0, seen_objects = 0;
  std::vector<std::pair<uint64_t, std::string>> first_object_errors;   // (object index within the run, text)
  void add_object_errors(const std::vector<std::string>& errs);

  void fold(const std::string& key, StatusViolation sv);
  // `other`'s partial state folded in as if its objects came after this run's (its object-error indices are offset by
  // seen_objects): merging shard runs in shard order gives the report of one run over the shards in that order
  void merge(AuditRun& other);
  // fold every result of a reviewed batch: viol/err are the kernel's bitmaps [n * words]
  // Lazy path: the pairs of constraints that have one result per pair (Compiled::single_result) are COUNTED from the bitmap, and only
  // the candidates -- the objects that can still enter a constraint's list -- are evaluated for their messages.  The candidates come
  // either from `cand` (Backend::audit_candidates: the `limit` smallest by (group, version, kind, namespace, name), any mix of kinds)
  // or, on a page of one kind, from `id` (the batch's namespace / name arrays: the `limit` smallest by (namespace, name)), ties
  // included either way.
  void add_batch(Engine& eng, const Compiled& c, const std::vector<ObjIn>& objs, const uint32_t* viol, const uint32_t* err,
                 uint32_t words, const std::vector<uint32_t>& errlist, const std::string& ep, const BatchIdentity* id = nullptr,
                 const uint32_t* amb = nullptr,    // amb: the ambiguity netlist's bitmap (bit clear = at most one result for the pair)
                 const uint32_t* cand = nullptr,   // cand: the candidate bitmap [n * words]
                 HostCandidates* keep = nullptr);  // keep: receives the threshold scan's rule (with `id`)
  uint64_t rendered_pairs = 0, counted_pairs = 0;   // pairs evaluated on the host / taken from the bitmap (lazy path)
  // `n` results of constraint `key` (enforcement action `action`) counted from the bitmap: in the totals, no status list entry
  void add_counted(const std::string& key, const std::string& action, uint64_t n);
  // An expanded batch's resultant violation pairs rendered on the host / counted from the bitmap (gk_audit_resultant_pairs).  Kept
  // apart from the two above, which count the parents' pairs only; not exported: they cover the batches added to this run.
  uint64_t resultant_rendered = 0, resultant_counted = 0;
  std::string report();
  // The run's partial state as a versioned byte string (gk_audit_export), and its inverse: parse() fills an empty run or throws
  // RegoError on a truncated, corrupted or foreign buffer.
  std::string serialize() const;
  static AuditRun parse(const uint8_t* buf, size_t len);
};

void validation_messages(const Compiled& c, const std::vector<Violation>& vio, uint32_t object, std::vector<std::string>& deny,
                         std::vector<std::string>& warn);

}  // namespace gk
