/* gk_engine.h -- C ABI of the H100 constraint-evaluation engine.
 *
 * This is the boundary a Go `drivers.Driver` shim binds with cgo (see INTEGRATION.md and go/gpudriver/).
 * Each entry point names the reference interface it stands behind (paths relative to the gatekeeper repo):
 *
 *   gk_engine_create/destroy  <- rego.New(args...) / driver lifetime          main.go:457-462, pkg/gator/opa.go:32-37
 *   gk_add_template           <- Driver.AddTemplate(ctx, *ConstraintTemplate)  pkg/drivers/k8scel/driver.go:74-136
 *   gk_remove_template        <- Driver.RemoveTemplate                          pkg/drivers/k8scel/driver.go:138-143
 *   gk_add_constraint         <- Driver.AddConstraint + TargetHandler.ToMatcher pkg/drivers/k8scel/driver.go:145-147, pkg/target/target.go:239-254
 *   gk_remove_constraint      <- Driver.RemoveConstraint                        pkg/drivers/k8scel/driver.go:149-151
 *   gk_put_namespace / remove <- Driver.AddData/RemoveData for Namespace paths + nsCache   pkg/target/ns_cache.go:15-85, pkg/target/target.go:60-66
 *   gk_review_batch           <- Client.Review -> Matcher.Match -> Driver.Query, for a BATCH of reviews
 *                                pkg/audit/manager.go:622,720 ; pkg/webhook/policy.go:661 ; pkg/target/matcher.go:21-71 ;
 *                                pkg/drivers/k8scel/driver.go:161-250
 *   gk_batch_upload/eval/free <- the same, split so an audit sweep can keep flattened batches resident in HBM
 *   gk_dump                   <- Driver.Dump                                    pkg/drivers/k8scel/driver.go:252-254
 *   gk_stat_description       <- Driver.GetDescriptionForStat                   pkg/drivers/k8scel/driver.go:256-263
 *
 * Conventions: plain pointers and sizes; 0 = success, negative = error with *err set to an engine-allocated
 * message (free with gk_free_str); the caller owns inputs for the duration of a call; the engine owns
 * gk_result buffers until gk_free_result.  Mutators take an exclusive lock, reviews a shared one
 * (mirrors k8scel.Driver's sync.RWMutex, pkg/drivers/k8scel/driver.go:61,130,167).  No exceptions or
 * panics cross this boundary.  There is no CPU fallback: without a CUDA device gk_engine_create fails.
 */
#ifndef GK_ENGINE_H
#define GK_ENGINE_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct gk_engine gk_engine_t;
typedef struct gk_batch gk_batch_t;

enum { GK_OK = 0, GK_ERR_INVALID = -1, GK_ERR_REGO = -2, GK_ERR_BACKEND = -3, GK_ERR_INTERNAL = -4 };

/* review source -- pkg/mutation/types/mutator.go:14-27 */
enum { GK_SOURCE_UNSET = 0, GK_SOURCE_ORIGINAL = 1, GK_SOURCE_GENERATED = 2, GK_SOURCE_ALL = 3, GK_SOURCE_INVALID = 4 };

/* gk_review_batch / gk_batch_eval flags */
enum {
  GK_F_BITMAP_ONLY = 0,      /* violation / error bitmaps + per-constraint totals */
  GK_F_MATERIALIZE = 1,      /* also render {msg, details} for every flagged pair (types.Result list) */
  GK_F_NO_COPY_BACK = 2,     /* leave bitmaps on the device (throughput measurement); totals still returned */
  /* gk_batch_upload_blob: the batch keeps the page's device JSON, offsets and token tape until gk_batch_free, so that
   * gk_batch_refresh re-extracts its columns without copying or tokenising the page again (HBM cost: DESIGN.md section 5b) */
  GK_F_KEEP_SOURCE = 4,
  /* gk_batch_upload, gk_batch_upload_blob, gk_review_blob: expand the page's generator objects (see gk_add_expansion_template) */
  GK_F_EXPAND = 8,
  /* which caller's excluder applies at flatten time (gk_set_excluded_namespaces); neither bit = no excluder stage (gator) */
  GK_F_PROCESS_AUDIT = 16,   /* process.Audit   -- pkg/audit/manager.go:531-538,600 */
  GK_F_PROCESS_WEBHOOK = 32  /* process.Webhook -- pkg/webhook/policy.go:170-178 */
};

typedef struct {
  int32_t device;            /* CUDA device ordinal */
  int32_t threads;           /* host flatten threads; 0 = hardware concurrency */
} gk_cfg;

/* One review: target.AugmentedUnstructured / AugmentedReview (pkg/target/data.go:24-28, review.go:9-14). */
typedef struct {
  const char* json;          /* Object.Raw (may be NULL when only old_json is set) */
  size_t len;
  const char* old_json;      /* OldObject.Raw or NULL */
  size_t old_len;
  const char* ns_json;       /* the review's Namespace object, or NULL (then the namespace cache is consulted) */
  size_t ns_len;
  const char* ns_name;       /* AdmissionRequest.Namespace; NULL = object's metadata.namespace */
  const char* operation;     /* "", "CREATE", "UPDATE", "DELETE"; NULL = "" */
  const char* userinfo_json; /* AdmissionRequest.UserInfo or NULL */
  size_t userinfo_len;
  uint8_t source;            /* GK_SOURCE_* */
} gk_obj;

/* One types.Result (pkg/drivers/k8scel/driver.go:223-227 for the field set). */
typedef struct {
  uint32_t object;                 /* index into the batch */
  uint32_t constraint;             /* index, see gk_constraint_key */
  const char* msg;
  const char* details_json;        /* Metadata["details"] as JSON, "" when absent */
  const char* enforcement_action;  /* deny | dryrun | warn | scoped | unrecognized */
  const char* scoped_actions_json; /* JSON array of actions for the enforcement point ("[]" unless scoped) */
  uint8_t autoreject;              /* 1: the matcher returned an error; msg carries its text */
} gk_violation;

typedef struct {
  uint32_t n_objects, n_constraints, words;   /* words = ceil(n_constraints / 32) */
  const uint32_t* viol_bits;       /* [n_objects * words] or NULL with GK_F_NO_COPY_BACK */
  const uint32_t* err_bits;        /* [n_objects * words] matcher-error plane */
  const uint64_t* totals;          /* [n_constraints] violating (constraint, object) pairs */
  const uint64_t* err_totals;      /* [n_constraints] */
  const gk_violation* violations;  /* with GK_F_MATERIALIZE */
  size_t n_violations;
  const char* const* object_errors;/* NULL when no object has one; else [n_objects]: NULL or the review-level error (bad JSON, DELETE without oldObject) */
  /* instrumentation (StatsEntry material, pkg/instrumentation/types.go:28-59) */
  double flatten_ms, h2d_ms, kernel_ms, d2h_ms, materialize_ms;
  uint64_t alg_bytes;              /* algorithmic bytes the kernel had to read + bitmap bytes written */
  uint64_t h2d_bytes, d2h_bytes;
  uint64_t gpu_launches;
  void* priv;
} gk_result;

gk_engine_t* gk_engine_create(const gk_cfg* cfg, char** err);
void gk_engine_destroy(gk_engine_t* e);
const char* gk_backend_name(gk_engine_t* e);
/* Which kernel decided the engine's last evaluation: "gk_spec_kernel" (CUDA C++ generated from the constraint set's netlist and
 * compiled by NVRTC for sm_90a the first time a batch of >= GK_SPEC_MIN_OBJECTS objects meets the set; GK_SPEC=0 turns it off)
 * or "gk_eval_kernel" (the netlist interpreter: small batches, and objects with more than 32 rows in a scope -- with their whole
 * tile when a tile holds many of them).
 * Replaces nothing in the reference: frameworks' rego driver compiles a template's Rego once per AddTemplate
 * (pkg/drivers/k8scel/driver.go:79-146 is the CEL analogue in this tree); this is the per-constraint-set analogue on the device. */
const char* gk_last_kernel(gk_engine_t* e);

int gk_add_template(gk_engine_t* e, const char* kind, const char* rego_src, size_t len, char** err);
/* The same with the template's `spec.targets[].libs` (or `code[].source.libs`): Rego modules under `package lib.<...>` that the
 * entry point imports as `data.lib.<...>` (constraint framework: templates.Target.Libs / schema.Source.Libs). */
int gk_add_template_libs(gk_engine_t* e, const char* kind, const char* rego_src, size_t len, const char* const* libs, const size_t* lib_lens,
                         size_t n_libs, char** err);
int gk_remove_template(gk_engine_t* e, const char* kind);
int gk_add_constraint(gk_engine_t* e, const char* constraint_json, size_t len, char** err);
/* TargetHandler.ValidateConstraint (pkg/target/target.go:178-214: spec.match.labelSelector / namespaceSelector must be maps that
 * convert to metav1.LabelSelector and pass ValidateLabelSelector).  The frameworks client calls the Go handler's method before
 * Driver.AddConstraint; this is the same check for hosts that do not go through that client.  0 = valid, else *err has the text. */
int gk_validate_constraint(gk_engine_t* e, const char* constraint_json, size_t len, char** err);
int gk_remove_constraint(gk_engine_t* e, const char* kind, const char* name);
/* ExpansionTemplates (pkg/expansion/system.go:60-112 UpsertTemplate / RemoveTemplate): `json` is the ExpansionTemplate object.
 * gk_review_batch then expands every generator object of a batch (System.Expand, system.go:137-247: the resource under
 * spec.templateSource becomes a resource of spec.generatedGVK named "<parent>-<kind>", owned by the parent, in the parent's
 * namespace), reviews the resultants with the batch as Generated resources, and reports their results on the parent with the
 * "[Implied by <template>]" prefix and the template's enforcementAction override (pkg/expansion/aggregate.go:19-63) -- what the
 * audit loop (pkg/audit/manager.go:733-765) and the webhook (pkg/webhook/policy.go:610-646) do around Client.Review.  Mutators are
 * not applied (the mutation system is outside this engine).  gk_audit_add_batch does the same for a resident batch: the resultants'
 * results enter the run under the parent's identity, an object whose expansion fails contributes nothing and is an objectErrors entry.
 * The bitmap entry points (gk_batch_eval, gk_batch_eval_device(_peers), gk_review_blob) expand a page uploaded (or reviewed) with
 * GK_F_EXPAND: an EXPANDED batch.  Its upload selects the page's generators on the device (the objects of an apiVersion / kind some
 * stored template applies to), expands them on the host and uploads their resultants as a second resident batch, reviewed as
 * Generated resources with the page's process flags.  Each evaluation evaluates the parents, then the resultants, then ORs every
 * resultant's rows into its parent's rows on the device.  The planes, object_errors and (GK_F_MATERIALIZE) the violation list equal
 * gk_review_batch's for the same objects; totals / err_totals are the column popcounts of the returned planes (parents with at least
 * one result, own or implied -- gk_review_batch counts every resultant row).  gk_batch_size stays the number of parents; alg_bytes,
 * kernel_ms and gpu_launches include the resultants and the fold.  The resultant planes belong to the batch: two device evaluations of
 * one expanded batch must not overlap (order them on one stream).  An expanded batch is refused by the eval calls once templates have
 * been added or removed since it was expanded ("ExpansionTemplates changed since the batch was expanded"); gk_batch_refresh expands
 * it again (a GK_F_KEEP_SOURCE blob batch from its kept device copy).  gk_audit_add_batch(_ordered) takes an expanded batch's
 * resultants from the batch while its templates are current: they are not expanded again on the host (see gk_audit_add_batch).
 * Without GK_F_EXPAND these calls do not expand: while templates are registered they fail with a text that says so, instead of
 * returning rows in which the resultants' violations are missing. */
int gk_add_expansion_template(gk_engine_t* e, const char* json, size_t len, char** err);
int gk_remove_expansion_template(gk_engine_t* e, const char* name);
/* System.GetConflicts (pkg/expansion/system.go:81-83; db.go:62-70): the names of the stored ExpansionTemplates that are set aside
 * because they lie on an expansion cycle (a template that closes a cycle is stored all the same, gk_add_expansion_template
 * reports "template forms expansion cycle" for it -- db.go:222-245 -- and every template on the cycle stops expanding until the
 * cycle is broken).  A JSON array of names, sorted; free with gk_free_str. */
char* gk_expansion_conflicts(gk_engine_t* e);
int gk_put_namespace(gk_engine_t* e, const char* name, const char* ns_json, size_t len, char** err);
int gk_remove_namespace(gk_engine_t* e, const char* name);
/* Driver.AddData / RemoveData for ANY synced object (pkg/drivers/k8scel/driver.go:252-258 are no-ops for CEL; the Rego driver
 * stores the object under /external/<target>/<path...>, read by referential templates as data.inventory...).  `path` is what
 * K8sValidationTarget.ProcessData returns (pkg/target/target.go:40-66): {"cluster", groupVersion, kind, name} or
 * {"namespace", ns, groupVersion, kind, name}; npath == 0 derives it from the object.  gk_remove_data removes one object or a
 * whole sub-tree.  Namespaces are ALSO given to gk_put_namespace by the caller (Client.AddData feeds both). */
int gk_add_data(gk_engine_t* e, const char* const* path, size_t npath, const char* obj_json, size_t len, char** err);
int gk_remove_data(gk_engine_t* e, const char* const* path, size_t npath);

/* constraint index <-> identity ("Kind/name"); the returned string is engine-owned until the next mutation */
uint32_t gk_constraint_count(gk_engine_t* e);
const char* gk_constraint_key(gk_engine_t* e, uint32_t index);
/* The same mapping as of the snapshot a result was computed with: stays valid (until gk_free_result) when constraints are
 * added or removed concurrently -- use this one to interpret `gk_violation.constraint` and the bitmap columns of `r`. */
const char* gk_result_constraint_key(const gk_result* r, uint32_t index);

int gk_review_batch(gk_engine_t* e, const gk_obj* objs, size_t n, const char* enforcement_point, uint32_t flags,
                    gk_result* out, char** err);

/* resident batches: flatten + upload once, evaluate many times (audit sweep / benchmarking) */
int gk_batch_upload(gk_engine_t* e, const gk_obj* objs, size_t n, uint32_t flags, gk_batch_t** out, gk_result* stats, char** err);
int gk_batch_eval(gk_engine_t* e, gk_batch_t* b, const char* enforcement_point, uint32_t flags, gk_result* out, char** err);
/* writes into caller-owned DEVICE buffers on a caller stream and returns without synchronising:
 * viol/err u32[n*words], totals/err_totals u64[n_constraints] (multi-GPU gather path) */
int gk_batch_eval_device(gk_engine_t* e, gk_batch_t* b, const char* enforcement_point, void* d_viol, void* d_err,
                         void* d_totals, void* d_err_totals, void* cuda_stream, char** err);
/* Multi-GPU sweep with the exchange FUSED into the kernel (replaces kernel + NCCL all-gather): every rank's kernel stores its
 * bitmap words, and its per-constraint totals, straight into the receive buffer of each peer GPU over NVLink.
 * peer_bases[q] is the device address of rank q's receive buffer (this rank included) in this process' address space
 * (CUDA IPC / symmetric memory); a rank's slot in it starts at `rank * slot_i32` int32 words: bitmap [n * words], then at
 * `tot_off_i32` the totals as u64 [2 * tot_stride] (violations, matcher errors).  d_viol may be NULL.  The call returns
 * without synchronising; the caller orders a device-side barrier across ranks after it on `cuda_stream`. */
int gk_batch_eval_device_peers(gk_engine_t* e, gk_batch_t* b, const char* enforcement_point, const uint64_t* peer_bases, uint32_t npeers,
                               uint32_t rank, uint64_t slot_i32, uint64_t tot_off_i32, uint32_t tot_stride, void* d_err, void* d_totals,
                               void* d_err_totals, void* cuda_stream, char** err);
/* the same two calls for a page of objects held in ONE contiguous buffer (a LIST page / spill directory as the
 * audit loop reads it, pkg/audit/manager.go:502-561,686-695): document i is buf[offsets[i], offsets[i+1]).
 * Every object is reviewed as an AugmentedUnstructured with the given source and no oldObject. */
int gk_batch_upload_blob(gk_engine_t* e, const char* buf, const uint64_t* offsets, size_t n, uint8_t source, uint32_t flags, gk_batch_t** out,
                         gk_result* stats, char** err);
int gk_review_blob(gk_engine_t* e, const char* buf, const uint64_t* offsets, size_t n, uint8_t source, const char* enforcement_point,
                   uint32_t flags, gk_result* out, char** err);
uint32_t gk_batch_size(gk_batch_t* b);
uint64_t gk_batch_alg_bytes(gk_batch_t* b);
void gk_batch_free(gk_engine_t* e, gk_batch_t* b);
/* Bring a resident batch to the engine's current constraint set, excluder patterns of the upload's process, and (referential
 * constraint sets) data.inventory: afterwards it is what a fresh upload of the same objects with the same flags would be, and the
 * eval and audit calls accept it again.  Every column is extracted again (string ids depend on the engine-wide string table, which
 * new constraints extend).  A blob batch uploaded with GK_F_KEEP_SOURCE is re-extracted on the device from its kept token tape when
 * the constraint set is flattened on the device; every other batch is flattened again from the caller's objects or blob, which must
 * still be alive, as for any resident batch.  Returns 1 when the batch was rebuilt, 0 when it was already current (nothing done),
 * negative on error -- then the batch is unchanged, still on its old constraint set.  `stats` (may be NULL): flatten_ms, h2d_ms,
 * h2d_bytes, alg_bytes as for an upload. */
int gk_batch_refresh(gk_engine_t* e, gk_batch_t* b, gk_result* stats, char** err);
/* Replace the object set of a resident batch uploaded with gk_batch_upload_blob(..., GK_F_KEEP_SOURCE): the objects at indices
 * `drop` (indices of the batch before the call, any order) leave it, and the n_add documents of `buf` / `offsets` (as for
 * gk_batch_upload_blob) are appended after the objects that stay, which keep their relative order.  Afterwards the batch is what
 * gk_batch_upload_blob of (the staying objects in order, then the new ones) with the upload's source and flags would be, under the
 * engine's current constraint set, excluder and ExpansionTemplates -- so it also does what gk_batch_refresh does.  The staying
 * objects are neither copied from the host nor tokenised again: their JSON and token tape move within the kept device page, only the
 * added documents are copied and tokenised, and then every column is extracted again over the new page.  To replace an object, drop
 * it and add its new version.  Returns the new gk_batch_size, or negative on error: an index out of range or given twice, a batch
 * without a kept source -> GK_ERR_INVALID; then the batch is unchanged.  `stats` as for gk_batch_refresh (may be NULL); kernel_ms is
 * the device time of the splice, the added documents' copy and tokeniser, and the extraction.
 * A batch keeps no device source when its constraint set was flattened on the host at upload (referential sets, Dump's "ingest: host
 * flattener (...)"); the call refuses it (GK_ERR_INVALID, with a text that says so), and it refuses every batch while the current
 * constraint set is flattened on the host: a patch never flattens on the host -- upload the page again instead.
 * The host still reads the objects' JSON for messages, the audit and expansion, where it was given: `buf` must stay alive while the
 * batch lives, as must the pages of the upload and of earlier patches that hold objects still in the batch. */
int gk_batch_patch(gk_engine_t* e, gk_batch_t* b, const uint32_t* drop, size_t n_drop, const char* buf, const uint64_t* offsets,
                   size_t n_add, gk_result* stats, char** err);

/* ---- stage-0 excluder: Config.spec.match[].excludedNamespaces of one process ("audit", "webhook", "sync",
 * "mutation-webhook", or "*" = all four), pkg/controller/config/process/excluder.go:53-127.  Replaces the process' set.
 * Objects whose namespace (own name for a Namespace) matches a pattern are skipped by batches flattened with the
 * matching GK_F_PROCESS_* flag: no results, no error. */
int gk_set_excluded_namespaces(gk_engine_t* e, const char* process, const char* const* patterns, size_t n, char** err);

/* ---- audit aggregation: what addAuditResponsesToUpdateLists / updateConstraintStatus do with the results of a sweep
 * (pkg/audit/manager.go:886-945,984-1041): totalViolations per constraint and per enforcement action, and per
 * constraint the `violations_limit` smallest StatusViolations under SVQueue.Less (manager.go:117-137), messages
 * truncated to `msg_size` bytes (manager.go:1043-1052).  0 selects the reference defaults (20, 256). */
typedef struct gk_audit gk_audit_t;
gk_audit_t* gk_audit_begin(gk_engine_t* e, uint32_t violations_limit, uint32_t msg_size, char** err);
/* evaluate a resident batch at the enforcement point and fold every result into the run (messages are rendered for the
 * flagged pairs on all host cores).  With ExpansionTemplates registered, every object is expanded and its resultants' results enter
 * the run as the object's (see gk_add_expansion_template).  An EXPANDED batch (GK_F_EXPAND) whose templates have not changed since
 * its upload or refresh brings its resultants: they are evaluated where they are resident, unfolded, and not expanded again.  Their
 * pairs are sorted against the parents' candidates: a matcher error, a pair whose parent can still enter the constraint's list and a
 * pair that may have several results are rendered; the other pairs, provably one result each, are counted.  The report is the one
 * the same objects uploaded without GK_F_EXPAND give, counters included ("pairsEvaluated" / "pairsCounted" count the parents' own
 * pairs).  A stale expanded batch, GK_AUDIT_EAGER, and a batch without the flag are expanded on the host as before. */
int gk_audit_add_batch(gk_audit_t* a, gk_batch_t* b, const char* enforcement_point, char** err);
/* gk_audit_add_batch with the candidates selected on the device, for a page of any mix of kinds (manager.go:886-945; the order is
 * SVQueue.Less, manager.go:117-137): the batch's objects are ranked by (group, version, kind, namespace, name) and, per constraint,
 * only the flagged objects at or below the `violations_limit`-th smallest identity (ties included) are rendered on the host; the
 * other pairs of constraints with one result per pair are counted from the bitmap.  The ambiguity netlist runs whatever the kinds.
 * The report equals gk_audit_add_batch's except for "pairsEvaluated" / "pairsCounted".  An expanded batch's resultant pairs are
 * sorted on the device as well, against the parents' ranking and thresholds. */
int gk_audit_add_batch_ordered(gk_audit_t* a, gk_batch_t* b, const char* enforcement_point, char** err);
/* device time (ms) of the ranking and selection of the last gk_audit_add_batch_ordered, and of the sorting of its resultant pairs */
float gk_audit_select_ms(gk_audit_t* a);
/* The resultant violation pairs of expanded batches (GK_F_EXPAND) that this run rendered on the host (*evaluated) and counted from
 * the bitmap (*counted), over the batches added to it; matcher-error pairs, always rendered, are in neither.  Batches expanded on the
 * host add nothing, and neither does gk_audit_merge: an export does not carry them.  Either pointer may be NULL. */
int gk_audit_resultant_pairs(gk_audit_t* a, uint64_t* evaluated, uint64_t* counted);
/* A sharded sweep (manager.go:886-945 over each shard, one updateConstraintStatus at the end: manager.go:984-1041).
 * gk_audit_export: the run's partial state -- per-constraint totals and status lists, per-action totals, object / result / pair
 * counters, object errors -- as an opaque versioned byte string in *buf (free with gk_free_str), *len bytes.
 * gk_audit_merge: folds an exported run into `a` as if its objects came after a's (object-error indices are offset by the objects
 * `a` has seen): merging the shards' exports in shard order reports what one run over all shards in that order would.  A truncated
 * or corrupted buffer, another format version, or another violations_limit / msg_size: GK_ERR_INVALID, and `a` is unchanged. */
int gk_audit_export(gk_audit_t* a, char** buf, size_t* len, char** err);
int gk_audit_merge(gk_audit_t* a, const char* buf, size_t len, char** err);
/* JSON: {"objects", "results", "totalViolations": {"Kind/name": n}, "totalViolationsPerEnforcementAction": {action: n},
 * "violations": {"Kind/name": [StatusViolation...]}} -- lists in the order updateConstraintStatus emits them (descending).
 * Caller frees with gk_free_str. */
char* gk_audit_report(gk_audit_t* a, char** err);
void gk_audit_end(gk_audit_t* a);

/* ---- admission: getValidationMessages (pkg/webhook/policy.go:238-355) for object `object` of a materialised result:
 * JSON {"deny": ["[<constraint name>] <msg>", ...], "warn": [...]}.  Caller frees with gk_free_str. */
char* gk_validation_messages(gk_engine_t* e, const gk_result* r, uint32_t object, char** err);

/* ---- admission coalescer (SURVEY.md 8(b): "Webhook: internal coalescer inside Query"): concurrent single-review callers
 * -- the webhook's request goroutines around Client.Review, pkg/webhook/policy.go:580-675 -- are gathered into micro-batches
 * (flushed at `max_batch` reviews or after `max_wait_us`) and evaluated with one gk_review_batch.  gk_coalescer_review
 * blocks until the caller's batch is done and returns its own request's outcome as JSON:
 *   {"batch_size": n, "error": null | "review-level error", "messages": {"deny": [...], "warn": [...]}, "results": [{"constraint",
 *    "msg", "details", "enforcementAction", "scopedEnforcementActions", "autoreject"}]}     (free with gk_free_str)
 * `flags`: GK_F_PROCESS_WEBHOOK applies the webhook's namespace excluder.  Thread-safe; no background thread. */
typedef struct gk_coalescer gk_coalescer_t;
gk_coalescer_t* gk_coalescer_create(gk_engine_t* e, uint32_t max_batch, uint32_t max_wait_us, const char* enforcement_point, uint32_t flags,
                                    char** err);
int gk_coalescer_review(gk_coalescer_t* c, const gk_obj* obj, char** out_json, char** err);
void gk_coalescer_stats(gk_coalescer_t* c, uint64_t* batches, uint64_t* reviews);
void gk_coalescer_destroy(gk_coalescer_t* c);

/* CPUs the flattener will use by default (gk_cfg.threads = 0): affinity mask and cgroup CPU quota respected */
int gk_host_cpus(void);

/* Page-lock (pin != 0) or release (pin == 0) a caller-owned host buffer that blobs are reviewed from (a LIST page buffer the
 * audit manager reuses, pkg/audit/manager.go:502-561): the blob's host->device copy is then a direct DMA at link speed, chunked
 * and overlapped with the tokeniser.  Optional: unpinned buffers work, through the driver's staging copies. */
int gk_pin_host(gk_engine_t* e, const void* p, size_t bytes, int pin, char** err);

/* Start streaming the NEXT page of the sweep to the GPU (host->device copy of the raw JSON, chunked, each chunk tokenised as it
 * lands) and return at once; the gk_review_blob / gk_batch_upload_blob call for the same (buf, n) then finds it there.  The audit
 * loop calls it for page k+1 before it reviews page k (pkg/audit/manager.go:579-646 lists and reviews page after page), so the
 * copy of one page hides behind the extraction and evaluation of the one before.  Optional; the buffer must stay unchanged until
 * it has been reviewed. */
int gk_blob_prefetch(gk_engine_t* e, const char* buf, const uint64_t* offsets, size_t n, char** err);

void gk_free_result(gk_result* r);
void gk_free_str(char* s);
char* gk_dump(gk_engine_t* e);
const char* gk_stat_description(const char* stat_name);

#ifdef __cplusplus
}
#endif
#endif
