// Package gpudriver -- bindings for the batch-side host work the engine does around Review: the namespace excluder,
// the audit sweep's aggregation, and the webhook's deny / warn message lists.  (Source only: this image has no Go
// toolchain; see INTEGRATION.md.)
package gpudriver

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../gatekeeper_b200 -lgk_engine
#include <stdlib.h>
#include "gk_engine.h"
*/
import "C"

import (
	"encoding/json"
	"errors"
	"unsafe"
)

// SetExcludedNamespaces mirrors process.Excluder.Add for one process ("audit", "webhook", "sync", "mutation-webhook" or "*"):
// pkg/controller/config/process/excluder.go:53-77.  The config controller calls it whenever Config.spec.match changes.
func (d *Driver) SetExcludedNamespaces(process string, patterns []string) error {
	d.mux.Lock()
	defer d.mux.Unlock()
	cp := C.CString(process)
	defer C.free(unsafe.Pointer(cp))
	arr := make([]*C.char, len(patterns)+1)
	for i, p := range patterns {
		arr[i] = C.CString(p)
		defer C.free(unsafe.Pointer(arr[i]))
	}
	var cerr *C.char
	if rc := C.gk_set_excluded_namespaces(d.e, cp, (**C.char)(unsafe.Pointer(&arr[0])), C.size_t(len(patterns)), &cerr); rc != 0 {
		return takeErr(cerr)
	}
	return nil
}

// StatusViolation is pkg/audit/manager.go:99-109.
type StatusViolation struct {
	Group              string   `json:"group"`
	Version            string   `json:"version"`
	Kind               string   `json:"kind"`
	Name               string   `json:"name"`
	Namespace          string   `json:"namespace,omitempty"`
	Message            string   `json:"message"`
	EnforcementAction  string   `json:"enforcementAction"`
	EnforcementActions []string `json:"enforcementActions,omitempty"`
}

// AuditReport is what addAuditResponsesToUpdateLists accumulates and updateConstraintStatus writes
// (pkg/audit/manager.go:886-945,984-1041): keys are "Kind/name".
type AuditReport struct {
	Objects                             uint64                       `json:"objects"`
	Results                             uint64                       `json:"results"`
	TotalViolations                     map[string]int64             `json:"totalViolations"`
	TotalViolationsPerEnforcementAction map[string]int64             `json:"totalViolationsPerEnforcementAction"`
	Violations                          map[string][]StatusViolation `json:"violations"`
}

// AuditRun folds reviewed pages (resident batches) into one sweep's status lists.
type AuditRun struct {
	d *Driver
	a *C.gk_audit_t
}

// NewAuditRun: limit = --constraint-violations-limit (manager.go:64), msgSize = 256 (manager.go:48); 0 selects the defaults.
func (d *Driver) NewAuditRun(limit, msgSize uint32) (*AuditRun, error) {
	var cerr *C.char
	a := C.gk_audit_begin(d.e, C.uint32_t(limit), C.uint32_t(msgSize), &cerr)
	if a == nil {
		return nil, takeErr(cerr)
	}
	return &AuditRun{d: d, a: a}, nil
}

// AddPage evaluates a resident batch at the audit enforcement point and folds every result into the run.
func (r *AuditRun) AddPage(b *C.gk_batch_t, enforcementPoint string) error {
	cep := C.CString(enforcementPoint)
	defer C.free(unsafe.Pointer(cep))
	var cerr *C.char
	if rc := C.gk_audit_add_batch(r.a, b, cep, &cerr); rc != 0 {
		return takeErr(cerr)
	}
	return nil
}

// AddPageOrdered is AddPage with the candidates ranked and selected on the GPU (gk_audit_add_batch_ordered): pages of any mix of
// kinds take the lazy path.  The report equals AddPage's except for pairsEvaluated / pairsCounted.
func (r *AuditRun) AddPageOrdered(b *C.gk_batch_t, enforcementPoint string) error {
	cep := C.CString(enforcementPoint)
	defer C.free(unsafe.Pointer(cep))
	var cerr *C.char
	if rc := C.gk_audit_add_batch_ordered(r.a, b, cep, &cerr); rc != 0 {
		return takeErr(cerr)
	}
	return nil
}

// ResultantPairs returns the resultant violation pairs of expanded batches (GK_F_EXPAND) that this run rendered on the host and
// counted from the bitmap (gk_audit_resultant_pairs): matcher-error pairs are in neither, and merged exports do not carry them.
func (r *AuditRun) ResultantPairs() (evaluated, counted uint64, err error) {
	var ev, ct C.uint64_t
	if rc := C.gk_audit_resultant_pairs(r.a, &ev, &ct); rc != 0 {
		return 0, 0, errors.New("gk_audit_resultant_pairs: invalid run")
	}
	return uint64(ev), uint64(ct), nil
}

// Export returns the run's partial state as an opaque versioned byte string (gk_audit_export), for Merge on another process.
func (r *AuditRun) Export() ([]byte, error) {
	var buf *C.char
	var n C.size_t
	var cerr *C.char
	if rc := C.gk_audit_export(r.a, &buf, &n, &cerr); rc != 0 {
		return nil, takeErr(cerr)
	}
	defer C.gk_free_str(buf)
	return C.GoBytes(unsafe.Pointer(buf), C.int(n)), nil
}

// Merge folds an exported run in as if its objects came after this run's (gk_audit_merge): merging the shards' exports in shard
// order reports what one run over all shards would.  A damaged export, another format version or another limit / msgSize is
// refused and leaves the run unchanged.
func (r *AuditRun) Merge(data []byte) error {
	var cerr *C.char
	var p *C.char
	if len(data) > 0 {
		p = (*C.char)(C.CBytes(data))
		defer C.free(unsafe.Pointer(p))
	}
	if rc := C.gk_audit_merge(r.a, p, C.size_t(len(data)), &cerr); rc != 0 {
		return takeErr(cerr)
	}
	return nil
}

// RefreshBatch brings a resident batch to the current constraint set, excluder patterns and data.inventory (gk_batch_refresh), so
// that an audit run can add it again after a template or constraint changed.  A page uploaded with GK_F_KEEP_SOURCE is re-extracted
// from its token tape in HBM; any other is flattened again from the objects or blob it was uploaded from, which must still be alive.
// A batch that was already current is left as it is.  On error the batch is unchanged.
func (d *Driver) RefreshBatch(b *C.gk_batch_t) error {
	d.mux.RLock()
	defer d.mux.RUnlock()
	var cerr *C.char
	if rc := C.gk_batch_refresh(d.e, b, nil, &cerr); rc < 0 {
		return takeErr(cerr)
	}
	return nil
}

// PatchBatch replaces objects of a resident page uploaded with GK_F_KEEP_SOURCE (gk_batch_patch): the objects at indices `drop`
// leave it and `docs` are appended after the objects that stay, which keep their order; the batch is then what an upload of that
// page would be under the current constraint set.  The staying objects are neither sent nor tokenised again.  An updated object is
// dropped and its new version added.  The documents are copied into one C page, returned: the engine reads the objects' JSON from it
// for messages and the audit, so the caller frees it (C.free) only when none of its objects is in the batch any more, or after the
// batch is freed.  On error the batch is unchanged and no page is returned.
func (d *Driver) PatchBatch(b *C.gk_batch_t, drop []uint32, docs [][]byte) (unsafe.Pointer, int, error) {
	d.mux.RLock()
	defer d.mux.RUnlock()
	total := 0
	for _, doc := range docs {
		total += len(doc)
	}
	page := C.malloc(C.size_t(total + 1))
	offs := (*[1 << 30]C.uint64_t)(C.malloc(C.size_t(len(docs)+1) * 8))[: len(docs)+1 : len(docs)+1]
	defer C.free(unsafe.Pointer(&offs[0]))
	dst := (*[1 << 40]byte)(page)[:total:total]
	pos := 0
	for i, doc := range docs {
		offs[i] = C.uint64_t(pos)
		pos += copy(dst[pos:], doc)
	}
	offs[len(docs)] = C.uint64_t(pos)
	var cdrop *C.uint32_t
	if len(drop) > 0 {
		cdrop = (*C.uint32_t)(C.malloc(C.size_t(len(drop)) * 4))
		defer C.free(unsafe.Pointer(cdrop))
		copy((*[1 << 30]uint32)(unsafe.Pointer(cdrop))[:len(drop):len(drop)], drop)
	}
	var cerr *C.char
	rc := C.gk_batch_patch(d.e, b, cdrop, C.size_t(len(drop)), (*C.char)(page), &offs[0], C.size_t(len(docs)), nil, &cerr)
	if rc < 0 {
		C.free(page)
		return nil, 0, takeErr(cerr)
	}
	return page, int(rc), nil
}

func (r *AuditRun) Report() (*AuditReport, error) {
	var cerr *C.char
	js := C.gk_audit_report(r.a, &cerr)
	if js == nil {
		return nil, takeErr(cerr)
	}
	defer C.gk_free_str(js)
	out := &AuditReport{}
	if err := json.Unmarshal([]byte(C.GoString(js)), out); err != nil {
		return nil, err
	}
	return out, nil
}

func (r *AuditRun) Close() {
	if r.a != nil {
		C.gk_audit_end(r.a)
		r.a = nil
	}
}

// validationMessages is validationHandler.getValidationMessages (pkg/webhook/policy.go:238-355) for request i of a
// materialised micro-batch result.
func (d *Driver) validationMessages(res *C.gk_result, i int) (deny, warn []string, err error) {
	var cerr *C.char
	js := C.gk_validation_messages(d.e, res, C.uint32_t(i), &cerr)
	if js == nil {
		return nil, nil, takeErr(cerr)
	}
	defer C.gk_free_str(js)
	var m struct {
		Deny []string `json:"deny"`
		Warn []string `json:"warn"`
	}
	if err := json.Unmarshal([]byte(C.GoString(js)), &m); err != nil {
		return nil, nil, err
	}
	return m.Deny, m.Warn, nil
}

// Coalescer gathers the webhook's concurrent Query calls (one goroutine per admission request, policy.go:580-675) into
// micro-batches: each Review call blocks until the batch it joined has been evaluated on the GPU.
type Coalescer struct {
	c  *C.gk_coalescer_t
	ep string
}

// AdmissionOutcome is one request's share of a micro-batch.
type AdmissionOutcome struct {
	BatchSize int     `json:"batch_size"`
	Error     *string `json:"error"`
	Messages  struct {
		Deny []string `json:"deny"`
		Warn []string `json:"warn"`
	} `json:"messages"`
	Results []struct {
		Constraint               string      `json:"constraint"`
		Msg                      string      `json:"msg"`
		Details                  interface{} `json:"details"`
		EnforcementAction        string      `json:"enforcementAction"`
		ScopedEnforcementActions []string    `json:"scopedEnforcementActions"`
		Autoreject               bool        `json:"autoreject"`
	} `json:"results"`
}

func (d *Driver) NewCoalescer(maxBatch, maxWaitMicros uint32, enforcementPoint string) (*Coalescer, error) {
	cep := C.CString(enforcementPoint)
	defer C.free(unsafe.Pointer(cep))
	var cerr *C.char
	c := C.gk_coalescer_create(d.e, C.uint32_t(maxBatch), C.uint32_t(maxWaitMicros), cep, C.GK_F_PROCESS_WEBHOOK, &cerr)
	if c == nil {
		return nil, takeErr(cerr)
	}
	return &Coalescer{c: c, ep: enforcementPoint}, nil
}

// EnableCoalescing routes Query calls at `enforcementPoint` (the webhook's) through a Coalescer.
func (d *Driver) EnableCoalescing(maxBatch, maxWaitMicros uint32, enforcementPoint string) error {
	co, err := d.NewCoalescer(maxBatch, maxWaitMicros, enforcementPoint)
	if err != nil {
		return err
	}
	d.mux.Lock()
	d.coalescer = co
	d.mux.Unlock()
	return nil
}

// Review blocks until the request's micro-batch is done.  The gk_obj and every payload it points to live in C memory for the
// duration of the call (cgo: no Go pointer inside memory passed to C).
func (c *Coalescer) Review(in reviewIn) ([]BatchResult, error) {
	o := (*C.gk_obj)(C.calloc(1, C.size_t(unsafe.Sizeof(C.gk_obj{}))))
	defer C.free(unsafe.Pointer(o))
	var owned []unsafe.Pointer
	defer func() {
		for _, p := range owned {
			C.free(p)
		}
	}()
	cbytes := func(b []byte) (*C.char, C.size_t) {
		if len(b) == 0 {
			return nil, 0
		}
		p := C.CBytes(b)
		owned = append(owned, p)
		return (*C.char)(p), C.size_t(len(b))
	}
	ar := in.ar
	o.json, o.len = cbytes(ar.Object.Raw)
	o.old_json, o.old_len = cbytes(ar.OldObject.Raw)
	if in.ns != nil {
		b, err := json.Marshal(in.ns)
		if err != nil {
			return nil, err
		}
		o.ns_json, o.ns_len = cbytes(b)
	}
	if ar.Namespace != "" {
		p := C.CString(ar.Namespace)
		owned = append(owned, unsafe.Pointer(p))
		o.ns_name = p
	}
	if ar.Operation != "" {
		p := C.CString(string(ar.Operation))
		owned = append(owned, unsafe.Pointer(p))
		o.operation = p
	}
	if ub, err := json.Marshal(ar.UserInfo); err == nil && string(ub) != "{}" {
		o.userinfo_json, o.userinfo_len = cbytes(ub)
	}
	o.source = sourceCode(in.source)
	var out, cerr *C.char
	if rc := C.gk_coalescer_review(c.c, o, &out, &cerr); rc != 0 {
		return nil, takeErr(cerr)
	}
	defer C.gk_free_str(out)
	res := &AdmissionOutcome{}
	if err := json.Unmarshal([]byte(C.GoString(out)), res); err != nil {
		return nil, err
	}
	if res.Error != nil {
		return nil, errors.New(*res.Error)
	}
	br := make([]BatchResult, 0, len(res.Results))
	for _, r := range res.Results {
		br = append(br, BatchResult{Constraint: r.Constraint, Msg: r.Msg, Details: r.Details, EnforcementAction: r.EnforcementAction,
			ScopedActions: r.ScopedEnforcementActions, Autoreject: r.Autoreject})
	}
	return br, nil
}

func (c *Coalescer) Close() {
	if c.c != nil {
		C.gk_coalescer_destroy(c.c)
		c.c = nil
	}
}
