// Engine: templates + constraints + namespace cache -> compiled (schema, program); object batches ->
// flattened columnar batches -> GPU evaluation -> violation bitmaps (+ lazily rendered messages).
#pragma once
#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <shared_mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "lower.hpp"
#include "program.h"
#include "rego.hpp"
#include "expansion.hpp"
#include "xprog.hpp"

namespace gk {

// ---- review inputs (one per object) -- mirrors target.AugmentedUnstructured / AugmentedReview
struct ObjIn {
  const char* json = nullptr;
  size_t len = 0;
  const char* old_json = nullptr;
  size_t old_len = 0;
  const char* ns_json = nullptr;   // explicit Namespace object (review.namespace), optional
  size_t ns_len = 0;
  const char* ns_name = nullptr;   // AdmissionRequest.Namespace; null => object's metadata.namespace
  const char* operation = nullptr; // "", CREATE, UPDATE, DELETE
  const char* userinfo_json = nullptr;
  size_t userinfo_len = 0;
  uint8_t source = 0;              // GK_SRC_*
};

struct HostColumn {
  std::vector<uint8_t> vt;
  std::vector<uint32_t> sid;
  std::vector<int64_t> num;
  std::vector<uint32_t> boff;   // rows + 1
  std::vector<uint8_t> bytes;
  std::vector<uint32_t> head;   // rows * GK_HEAD_WORDS (GK_ENC_HEAD)
};

struct HostBatch {
  uint32_t n = 0;
  bool has_old = false;
  // header rows: [0,n) objects, [n,2n) old objects when has_old
  std::vector<uint32_t> flags, kind_sid, group_sid, nsn_off, name_off, gen_off, lbl_off, lbl_kv;
  std::vector<uint8_t> name_bytes, gen_bytes, nsn_bytes;
  std::vector<uint32_t> nsrow;                 // [n]
  std::vector<uint32_t> nsl_off, nsl_kv;       // per-batch namespace label table
  std::vector<std::vector<uint32_t>> scope_off;   // [scope][parent_rows+1]; [0] unused
  std::vector<uint32_t> scope_rows;
  std::vector<HostColumn> cols;
  std::vector<std::string> obj_errors;         // per object: "" or a review-level error (bad JSON, missing kind, ...)
  uint64_t alg_bytes = 0;                      // bytes of every array the kernel may read (each counted once)
  uint64_t schema_version = 0;
  uint64_t gvk_lo = ~0ull, gvk_hi = 0;         // min / max hash of (apiVersion, kind) over the objects that were not skipped
  std::vector<uint64_t> gvk;                   // [n] that hash per object, 0 for a skipped one (the audit ranks objects by kind)
};

struct MatchSpec {
  bool has = false;
  VP raw;                                      // spec.match
  GkMatch dev{};                               // pool offsets filled by the compiler
  std::string lsel_err, nssel_err, src_err;    // error texts when the corresponding *_INVALID flag is set
};

struct ScopedAction {
  std::string action;
  std::vector<std::string> points;
};

struct Constraint {
  std::string kind, name;
  VP obj, params;
  std::string params_key;                      // canonical JSON of spec.parameters: constraints of a kind with equal parameters render equal messages
  MatchSpec match;
  std::string action;                          // deny / dryrun / warn / scoped / unrecognized
  std::vector<ScopedAction> scoped;
};

struct TemplateEntry {
  std::string kind;
  std::string src;
  std::shared_ptr<Module> mod;
};

struct Compiled {
  uint64_t version = 0;
  Schema schema;
  std::vector<GkOp> ops;                       // the joint netlist (program.h)
  std::vector<uint32_t> items, phase_off;      // work items per dependency phase
  std::vector<GkOutEnt> outs;                  // per constraint: result / match / error slots
  std::vector<uint8_t> slot_level;             // scope of each shared-memory slot
  std::vector<uint32_t> pool;
  std::vector<uint8_t> cbytes;
  std::vector<GkMatch> match;                  // DISTINCT match blocks
  std::vector<uint32_t> cons_match;            // per constraint: match block id
  std::vector<const Constraint*> order;        // constraint index -> constraint (grouped by match block)
  // per constraint, owned by the snapshot (compiling never writes into a Constraint that an older snapshot may be reading):
  std::vector<FP> formulas;                              // the lowered violation predicate
  std::vector<uint8_t> single_result;                    // 1: a violating pair has exactly one result (lower.hpp)
  std::shared_ptr<const Compiled> amb;                   // the ambiguity netlist of the same constraints over the same schema (audit):
                                                         // bit c clear = at most one result for that pair (null: not available)
  struct MatchErrs { std::string lsel, nssel, src; };
  std::vector<MatchErrs> match_errs;                     // error texts behind the *_INVALID match flags
  std::vector<std::shared_ptr<const Constraint>> pins;   // keeps `order` alive while a review still uses this snapshot
                                                         // (RemoveConstraint / a replacing AddConstraint may run meanwhile)
  std::vector<std::shared_ptr<Module>> mods;   // constraint index -> its template's module (pinned by this snapshot)
  size_t n_nodes = 0, n_atoms = 0, n_gates = 0, n_phases = 0;
  std::shared_ptr<const XProgHost> xprog;      // the extraction program of the device ingest path (null: host flattener only)
  bool uses_data = false;                      // some template reads `data` (data.inventory: referential constraints)
  bool device_ingest = false;                  // every scope / column of `schema` can be computed by the ingest kernels
  std::string host_ingest_reason;              // why not (the first construct that needs the host flattener)
};

// K8sValidationTarget.ValidateConstraint (pkg/target/target.go:178-214) on a constraint document: "" or the error text
std::string validate_constraint_json(const std::string& json);

class StringTable : public Interner {
 public:
  StringTable();
  uint32_t intern(const std::string& key) override;
  uint32_t lookup(const std::string& key) const;   // GK_SID_UNDEF if absent
  // Lock-free lookups for the flatten workers: an immutable copy of the table as of the last freeze() plus the table's
  // size then.  A miss in the frozen copy is final unless the table has grown since (size_relaxed() != frozen size).
  using Frozen = std::unordered_map<std::string, uint32_t>;
  std::shared_ptr<const Frozen> freeze();
  uint32_t size_relaxed() const { return n_.load(std::memory_order_relaxed); }
  // snapshot for upload: offsets [n+1] and bytes
  void snapshot(std::vector<uint32_t>& off, std::vector<uint8_t>& bytes) const;
  uint32_t size() const;
  std::string get(uint32_t sid) const;

 private:
  mutable std::shared_mutex mu_;
  std::unordered_map<std::string, uint32_t> map_;
  std::vector<uint32_t> off_;
  std::vector<uint8_t> bytes_;
  std::shared_ptr<const Frozen> frozen_;
  std::atomic<uint32_t> n_{0};
};

struct Violation {
  uint32_t object, constraint;
  std::string msg, details_json, action, scoped_json;
  bool autoreject = false;
};

class Engine {
 public:
  explicit Engine(int threads);
  // mutators (exclusive) -- mirror drivers.Driver AddTemplate/RemoveTemplate/AddConstraint/RemoveConstraint/AddData
  void add_template(const std::string& kind, const std::string& rego, const std::vector<std::string>& libs = {});
  bool remove_template(const std::string& kind);
  void add_constraint(const std::string& json);
  bool remove_constraint(const std::string& kind, const std::string& name);
  void put_namespace(const std::string& name, const std::string& json);
  bool remove_namespace(const std::string& name);

  std::shared_ptr<const Compiled> compiled();                 // compiles lazily after mutations
  // process: "" (no excluder stage), "audit", "webhook" -- objects in a namespace excluded for that process are
  // skipped as the callers do before Review (pkg/audit/manager.go:531-538,600; pkg/webhook/policy.go:170-178)
  std::shared_ptr<HostBatch> flatten(const ObjIn* objs, size_t n, const Compiled& c, const std::string& process = "");
  // Config.spec.match[].excludedNamespaces per process -- pkg/controller/config/process/excluder.go:53-77
  void set_excluded_namespaces(const std::string& process, const std::vector<std::string>& patterns);
  std::vector<std::string> excluded_namespaces(const std::string& process);
  // all results of one object for the flagged constraints (one DOM parse); `obj_out` receives the reviewed object
  struct Flagged {
    uint32_t cix;
    bool is_err;
    uint32_t err_code;
  };
  // Per-worker state of message rendering over ONE Compiled snapshot: evaluators are kept across objects, and every
  // constraint's parameters are a thread-private deep copy (walking a shared document copies node references, and
  // reference counts shared by all workers bounce between their caches).
  struct MaterializeCtx {
    std::unordered_map<const Module*, std::unique_ptr<Eval>> evals;
    std::unordered_map<const Module*, uint64_t> eval_epoch;
    std::unordered_map<const Constraint*, VP> params;
    uint64_t epoch = 0;   // one per object
    VP data;              // {"inventory": ...} for referential templates (fetched once per context)
  };
  void materialize_object(const Compiled& c, const ObjIn& obj, uint32_t obj_ix, const std::vector<Flagged>& flagged,
                          const std::string& ep, std::vector<Violation>& out, VP* obj_out = nullptr, MaterializeCtx* ctx = nullptr);
  // which constraints apply at an enforcement point + their effective actions
  void active_mask(const Compiled& c, const std::string& ep, std::vector<uint32_t>& active) const;
  // render messages for one flagged pair (never decides a violation; throws if the GPU bit is unjustified)
  void materialize(const Compiled& c, const ObjIn& obj, uint32_t obj_ix, uint32_t cix, const std::string& ep,
                   std::vector<Violation>& out);
  void autoreject(const Compiled& c, const ObjIn& obj, uint32_t obj_ix, uint32_t cix, uint32_t code, const std::string& ep,
                  std::vector<Violation>& out);
  std::string dump();
  // ExpansionTemplates (pkg/expansion): generator resources imply resultants that are reviewed with them
  void add_expansion_template(const std::string& json);
  bool remove_expansion_template(const std::string& name);
  bool has_expansion();
  uint64_t expansion_version();   // ExpansionSystem::version: an expanded batch is current while it is unchanged
  // whether objects of (g, v, k) can have resultants: a stored template applies to it, or it is empty (expansion then fails)
  bool expansion_selects(const std::string& g, const std::string& v, const std::string& k);
  std::vector<std::string> expansion_conflicts();   // System.GetConflicts: templates set aside as part of an expansion cycle, by name
  // the resultants of one review's object (empty when no template applies); throws std::runtime_error like System.Expand
  void expand_object(const ObjIn& in, std::vector<Resultant>& out);
  // Client.AddData / RemoveData for any synced object (pkg/target/target.go:40-66 processUnstructured: the path is
  // cluster/<groupVersion>/<kind>/<name> or namespace/<ns>/<groupVersion>/<kind>/<name>): what referential templates read
  // as data.inventory.  data_doc() is the immutable {"inventory": {...}} document of the current contents.
  void add_data(const std::vector<std::string>& path, const std::string& json);   // empty path: derived from the object
  bool remove_data(const std::vector<std::string>& path);
  static std::vector<std::string> data_path(const std::string& json);
  VP data_doc(uint64_t* version = nullptr);
  std::map<std::string, VP> namespaces_snapshot();   // (deep copies: safe to read from another thread without touching shared reference counts)
  // everything a backend needs to flatten a blob of plain objects on the device (xprog.hpp); `blob` must outlive the request
  IngestReq ingest_request(const std::shared_ptr<const Compiled>& c, const uint8_t* blob, const unsigned long long* ooff, size_t n, uint32_t source,
                           const std::string& process);
  // host evaluation of Lut closures for the argument tuples the device has not seen yet
  void lut_fill(const Compiled& c, const uint8_t* blob, const GkMiss* misses, size_t n, std::vector<GkLutVal>& out);
  StringTable& strings() { return strings_; }
  int threads() const { return threads_; }
  VP review_doc(const ObjIn& in, VP* obj_out, VP* old_out, VP* ns_out, std::string* err, const std::map<std::string, VP>* ns_snapshot = nullptr);

 private:
  friend struct Flattener;
  void compile_locked();
  std::shared_mutex mu_;
  std::map<std::string, TemplateEntry> templates_;
  std::vector<std::shared_ptr<Constraint>> constraints_;   // (shared: a compiled snapshot pins the constraints it was built from)
  std::map<std::string, VP> namespaces_;
  uint64_t ns_version_ = 0;                                // bumped by put_namespace / remove_namespace
  std::shared_ptr<const NsTableHost> ns_table_;            // device form of namespaces_ (rebuilt when stale)
  uint64_t ns_table_version_ = ~0ull;
  uint32_t ns_table_strings_ = 0;
  std::map<std::vector<std::string>, VP> inventory_;       // processUnstructured path -> object
  uint64_t inventory_version_ = 0;
  VP inventory_doc_;                                       // built lazily from inventory_
  uint64_t inventory_doc_version_ = ~0ull;
  std::map<std::string, std::vector<std::string>> excluded_;
  ExpansionSystem expansion_;
  std::shared_ptr<Compiled> compiled_;
  bool dirty_ = true;
  uint64_t version_ = 0;
  StringTable strings_;
  int threads_;
};

int effective_cpus();   // affinity mask and cgroup quota respected
void split_gv(const VP& obj, std::string& group, std::string& version, std::string& kind);   // apiVersion -> (group, version), kind
std::string meta_str(const VP& obj, const char* field);                                       // metadata.<field> or ""

// scoped/unscoped action resolution -- pkg/util/enforcement_action.go:132-174
std::vector<std::string> scoped_actions_for(const Constraint& c, const std::string& ep);

}  // namespace gk
