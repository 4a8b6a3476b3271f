// Package gpudriver is the Go side of the drop-in: a constraint-framework drivers.Driver whose Query and the
// additive ReviewBatch go through cgo into libgk_engine.so (include/gk_engine.h).
//
// NOT COMPILED IN THIS REPOSITORY'S IMAGE: there is no Go toolchain here (go: command not found) and the
// frameworks/constraint + OPA modules are not vendored.  The file is the binding a Gatekeeper maintainer would add;
// it follows the only in-tree Driver implementation line by line for locking, review type assertions and stats
// (pkg/drivers/k8scel/driver.go:60-263).  tests/ exercise the same C ABI through the ctypes mirror
// gatekeeper_b200/driver.py, method for method, and tests/c_abi/mirror.c repeats reviewBatch below CALL FOR CALL in C
// (C-allocated gk_obj array, every field this file populates) against the admission-shape vectors.
//
// Registration (replaces rego.New(args...) -- main.go:457-462, pkg/gator/opa.go:32-37, pkg/gator/test/test.go:48-53,
// pkg/gator/bench/bench.go:313-319):
//
//	d, err := gpudriver.New(gpudriver.Device(0))
//	client, err := constraintclient.NewClient(constraintclient.Targets(&target.K8sValidationTarget{}),
//	        constraintclient.Driver(k8scelDriver), constraintclient.Driver(d), constraintclient.EnforcementPoints(...))
package gpudriver

/*
#cgo CFLAGS: -I${SRCDIR}/../../include
#cgo LDFLAGS: -L${SRCDIR}/../../gatekeeper_b200 -lgk_engine
#include <stdlib.h>
#include "gk_engine.h"
*/
import "C"

import (
	"context"
	"encoding/json"
	"errors"
	"fmt"
	"sync"
	"unsafe"

	"github.com/open-policy-agent/frameworks/constraint/pkg/client/drivers"
	"github.com/open-policy-agent/frameworks/constraint/pkg/client/reviews"
	"github.com/open-policy-agent/frameworks/constraint/pkg/core/templates"
	"github.com/open-policy-agent/frameworks/constraint/pkg/instrumentation"
	"github.com/open-policy-agent/frameworks/constraint/pkg/types"
	"github.com/open-policy-agent/opa/v1/storage"
	admissionv1 "k8s.io/api/admission/v1"
	"k8s.io/apimachinery/pkg/apis/meta/v1/unstructured"
	"k8s.io/apimachinery/pkg/runtime"
)

// Name is "Rego": templates carrying targets[].rego / code[engine: Rego] route to this driver.  It replaces -- and
// cannot co-exist with -- rego.Driver (SURVEY.md 8(b)).
const Name = "Rego"

var _ drivers.Driver = &Driver{}

type Driver struct {
	mux sync.RWMutex // mutators exclusive, Query shared: pkg/drivers/k8scel/driver.go:61,130,167
	e   *C.gk_engine_t
	gatherStats bool
	coalescer   *Coalescer // set by EnableCoalescing: Query joins micro-batches at its enforcement point
}

type Arg func(*Driver, *C.gk_cfg)

func Device(i int) Arg   { return func(_ *Driver, c *C.gk_cfg) { c.device = C.int32_t(i) } }
func Threads(n int) Arg  { return func(_ *Driver, c *C.gk_cfg) { c.threads = C.int32_t(n) } }
func GatherStats() Arg   { return func(d *Driver, _ *C.gk_cfg) { d.gatherStats = true } }

func New(args ...Arg) (*Driver, error) {
	d := &Driver{}
	var cfg C.gk_cfg
	for _, a := range args {
		a(d, &cfg)
	}
	var cerr *C.char
	d.e = C.gk_engine_create(&cfg, &cerr)
	if d.e == nil {
		return nil, takeErr(cerr) // no CUDA device => error: there is no CPU fallback
	}
	return d, nil
}

func takeErr(c *C.char) error {
	if c == nil {
		return errors.New("gpudriver: unknown error")
	}
	defer C.gk_free_str(c)
	return errors.New(C.GoString(c))
}

func (d *Driver) Name() string { return Name }

// AddTemplate lowers the template's Rego ahead of time; unsupported constructs are an error here, exactly where a
// Rego compile error surfaces in the reference (pkg/controller/constrainttemplate/constrainttemplate_controller.go:476-479).
func (d *Driver) AddTemplate(_ context.Context, ct *templates.ConstraintTemplate) error {
	src, libs, err := regoSource(ct)
	if err != nil {
		return err
	}
	d.mux.Lock()
	defer d.mux.Unlock()
	kind := C.CString(ct.Spec.CRD.Spec.Names.Kind)
	defer C.free(unsafe.Pointer(kind))
	csrc := C.CString(src)
	defer C.free(unsafe.Pointer(csrc))
	var cerr *C.char
	if len(libs) == 0 {
		if rc := C.gk_add_template(d.e, kind, csrc, C.size_t(len(src)), &cerr); rc != 0 {
			return takeErr(cerr)
		}
		return nil
	}
	// the pointer array lives in C memory (cgo forbids Go memory that holds C pointers... and vice versa)
	n := len(libs)
	arr := (*[1 << 20]*C.char)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(uintptr(0)))))
	lens := (*[1 << 20]C.size_t)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof(C.size_t(0)))))
	defer C.free(unsafe.Pointer(arr))
	defer C.free(unsafe.Pointer(lens))
	for i, l := range libs {
		arr[i] = C.CString(l)
		lens[i] = C.size_t(len(l))
		defer C.free(unsafe.Pointer(arr[i]))
	}
	if rc := C.gk_add_template_libs(d.e, kind, csrc, C.size_t(len(src)), (**C.char)(unsafe.Pointer(arr)), (*C.size_t)(unsafe.Pointer(lens)), C.size_t(n), &cerr); rc != 0 {
		return takeErr(cerr)
	}
	return nil
}

func (d *Driver) RemoveTemplate(_ context.Context, ct *templates.ConstraintTemplate) error {
	d.mux.Lock()
	defer d.mux.Unlock()
	kind := C.CString(ct.Spec.CRD.Spec.Names.Kind)
	defer C.free(unsafe.Pointer(kind))
	C.gk_remove_template(d.e, kind)
	return nil
}

// AddConstraint hands the whole constraint (spec.match, spec.parameters, enforcement actions) to the engine: the match
// block becomes the in-kernel pre-filter (pkg/target/target.go:239-254, pkg/mutation/match/match.go:32-65).
func (d *Driver) AddConstraint(_ context.Context, c *unstructured.Unstructured) error {
	raw, err := c.MarshalJSON()
	if err != nil {
		return err
	}
	d.mux.Lock()
	defer d.mux.Unlock()
	var cerr *C.char
	if rc := C.gk_add_constraint(d.e, (*C.char)(unsafe.Pointer(&raw[0])), C.size_t(len(raw)), &cerr); rc != 0 {
		return takeErr(cerr)
	}
	return nil
}

func (d *Driver) RemoveConstraint(_ context.Context, c *unstructured.Unstructured) error {
	d.mux.Lock()
	defer d.mux.Unlock()
	kind, name := C.CString(c.GetKind()), C.CString(c.GetName())
	defer C.free(unsafe.Pointer(kind))
	defer C.free(unsafe.Pointer(name))
	C.gk_remove_constraint(d.e, kind, name)
	return nil
}

// cPath copies a storage path into C memory (cgo: no Go pointers to Go pointers); the caller frees with freePath.
func cPath(path storage.Path) (**C.char, func()) {
	n := len(path)
	arr := (**C.char)(C.malloc(C.size_t(n) * C.size_t(unsafe.Sizeof((*C.char)(nil)))))
	sl := unsafe.Slice(arr, n)
	for i, p := range path {
		sl[i] = C.CString(p)
	}
	return arr, func() {
		for i := range sl {
			C.free(unsafe.Pointer(sl[i]))
		}
		C.free(unsafe.Pointer(arr))
	}
}

// AddData: every synced object is stored at its path for referential templates (data.inventory); Namespaces also feed the
// namespaceSelector table (nsCache.Add).  Paths per pkg/target/target.go:40-66.
func (d *Driver) AddData(_ context.Context, _ string, path storage.Path, data interface{}) error {
	raw, err := json.Marshal(data)
	if err != nil {
		return err
	}
	if len(raw) == 0 {
		return nil
	}
	d.mux.Lock()
	defer d.mux.Unlock()
	buf := C.CBytes(raw)
	defer C.free(buf)
	var cerr *C.char
	if len(path) >= 4 && path[0] == "cluster" && path[2] == "Namespace" {
		name := C.CString(path[3])
		defer C.free(unsafe.Pointer(name))
		if rc := C.gk_put_namespace(d.e, name, (*C.char)(buf), C.size_t(len(raw)), &cerr); rc != 0 {
			return takeErr(cerr)
		}
	}
	arr, free := cPath(path)
	defer free()
	if rc := C.gk_add_data(d.e, arr, C.size_t(len(path)), (*C.char)(buf), C.size_t(len(raw)), &cerr); rc != 0 {
		return takeErr(cerr)
	}
	return nil
}

func (d *Driver) RemoveData(_ context.Context, _ string, path storage.Path) error {
	d.mux.Lock()
	defer d.mux.Unlock()
	if len(path) >= 4 && path[0] == "cluster" && path[2] == "Namespace" {
		name := C.CString(path[3])
		defer C.free(unsafe.Pointer(name))
		C.gk_remove_namespace(d.e, name)
	}
	if len(path) > 0 {
		arr, free := cPath(path)
		defer free()
		C.gk_remove_data(d.e, arr, C.size_t(len(path)))
	}
	return nil
}

// UpsertExpansionTemplate / RemoveExpansionTemplate: the expansion system's templates (pkg/expansion/system.go:60-135).  With them
// in place ReviewBatch reviews the resultants of every object in the same batch and folds their results onto the parent
// ([Implied by <template>] prefix, enforcement-action override: pkg/expansion/aggregate.go:19-63).  The bitmap sweep entry points
// (gk_batch_eval*, gk_review_blob), which this shim does not call, expand only a page uploaded with GK_F_EXPAND (gk_engine.h).
func (d *Driver) UpsertExpansionTemplate(templateJSON []byte) error {
	d.mux.Lock()
	defer d.mux.Unlock()
	buf := C.CBytes(templateJSON)
	defer C.free(buf)
	var cerr *C.char
	if rc := C.gk_add_expansion_template(d.e, (*C.char)(buf), C.size_t(len(templateJSON)), &cerr); rc != 0 {
		return takeErr(cerr)
	}
	return nil
}

func (d *Driver) RemoveExpansionTemplate(name string) {
	d.mux.Lock()
	defer d.mux.Unlock()
	cn := C.CString(name)
	defer C.free(unsafe.Pointer(cn))
	C.gk_remove_expansion_template(d.e, cn)
}

// ExpansionConflicts mirrors expansion.System.GetConflicts (pkg/expansion/system.go:81-83): the names of the stored templates that are
// set aside because they lie on an expansion cycle, as a JSON array.
func (d *Driver) ExpansionConflicts() string {
	d.mux.RLock()
	defer d.mux.RUnlock()
	cs := C.gk_expansion_conflicts(d.e)
	if cs == nil {
		return "[]"
	}
	defer C.gk_free_str(cs)
	return C.GoString(cs)
}

// ARGetter / IsAdmissionGetter: how drivers reach the unexported *gkReview -- pkg/drivers/k8scel/driver.go:265-271.
type ARGetter interface {
	GetAdmissionRequest() *admissionv1.AdmissionRequest
}

// SourceGetter: the review's source (pkg/target/review.go:24, `source types.SourceType`).  gkReview needs the one-line accessor
// `func (g *gkReview) GetSource() types.SourceType { return g.source }` (INTEGRATION.md section 3): the engine runs the spec.match
// pre-filter itself, and match.source is one of its eight criteria (pkg/mutation/match/match.go:229-253).
type SourceGetter interface {
	GetSource() string
}

// reviewIn is everything of one gkReview the engine consumes (pkg/target/review.go:16-29, target.go:86-172).
type reviewIn struct {
	ar     *admissionv1.AdmissionRequest
	ns     map[string]interface{} // reviews.ReviewCfg.Namespace (the review's Namespace object), may be nil
	source string                 // "", "Original", "Generated"
}

func sourceCode(s string) C.uint8_t {
	switch s {
	case "":
		return C.GK_SOURCE_UNSET
	case "Original":
		return C.GK_SOURCE_ORIGINAL
	case "Generated":
		return C.GK_SOURCE_GENERATED
	case "All":
		return C.GK_SOURCE_ALL
	}
	return C.GK_SOURCE_INVALID
}

// Query: one review, the constraints Client.Review already matched (pkg/drivers/k8scel/driver.go:161-250).  With a Coalescer
// attached (EnableCoalescing) concurrent Query calls of the webhook's handler goroutines join one micro-batch and share one
// kernel launch; without one the review is a batch of one.
func (d *Driver) Query(ctx context.Context, target string, constraints []*unstructured.Unstructured, review interface{},
	opts ...reviews.ReviewOpt) (*drivers.QueryResponse, error) {
	cfg := &reviews.ReviewCfg{}
	for _, o := range opts {
		o(cfg)
	}
	arGetter, ok := review.(ARGetter)
	if !ok {
		return nil, errors.New("cannot convert review to ARGetter")
	}
	in := reviewIn{ar: arGetter.GetAdmissionRequest(), ns: cfg.Namespace}
	if sg, ok := review.(SourceGetter); ok {
		in.source = sg.GetSource()
	} else {
		in.source = "Original"
	}
	var results []BatchResult
	var stats []*instrumentation.StatsEntry
	var err error
	if co := d.coalescer; co != nil && cfg.EnforcementPoint == co.ep {
		results, err = co.Review(in)
	} else {
		results, stats, err = d.reviewBatch(ctx, []reviewIn{in}, cfg.EnforcementPoint, true)
	}
	if err != nil {
		return nil, err
	}
	want := map[string]*unstructured.Unstructured{}
	for _, c := range constraints {
		want[c.GetKind()+"/"+c.GetName()] = c
	}
	out := &drivers.QueryResponse{}
	for _, r := range results {
		if c, ok := want[r.Constraint]; ok {
			out.Results = append(out.Results, &types.Result{Target: target, Msg: r.Msg,
				Metadata: map[string]interface{}{"details": r.Details}, Constraint: c})
		}
	}
	if d.gatherStats || cfg.StatsEnabled {
		out.StatsEntries = stats
	}
	return out, nil
}

// BatchReviewer is the additive entry point pkg/audit type-asserts for at manager.go:622/:720 (SURVEY.md 8(b)).
type BatchReviewer interface {
	ReviewBatch(ctx context.Context, target string, objs []*unstructured.Unstructured, namespaces []map[string]interface{},
		enforcementPoint string) ([]BatchResult, error)
}

var _ BatchReviewer = (*Driver)(nil)

type BatchResult struct {
	Object            int
	Constraint        string // "Kind/name"
	Msg               string
	Details           interface{}
	EnforcementAction string
	ScopedActions     []string
	Autoreject        bool
}

// ReviewBatch reviews a page of listed objects (the audit loop's unit of work: pkg/audit/manager.go:579-646,668-777) in one call.
// A review-level error of one object (undecodable JSON, kind missing) is returned as an error naming that object, like the
// per-object Review error the audit loop logs at manager.go:722-729.
func (d *Driver) ReviewBatch(ctx context.Context, _ string, objs []*unstructured.Unstructured, namespaces []map[string]interface{},
	enforcementPoint string) ([]BatchResult, error) {
	ins := make([]reviewIn, len(objs))
	for i, o := range objs {
		raw, err := o.MarshalJSON()
		if err != nil {
			return nil, err
		}
		ins[i] = reviewIn{ar: &admissionv1.AdmissionRequest{Object: runtime.RawExtension{Raw: raw}, Name: o.GetName(), Namespace: o.GetNamespace()},
			source: "Original"}
		if namespaces != nil {
			ins[i].ns = namespaces[i]
		}
	}
	res, _, err := d.reviewBatch(ctx, ins, enforcementPoint, true)
	return res, err
}

// cgo rule: no Go pointer may be stored in memory handed to C.  Every payload is therefore copied into C memory (C.CBytes /
// C.CString) for the duration of the call, and the gk_obj array itself lives in C memory.
func (d *Driver) reviewBatch(_ context.Context, ins []reviewIn, ep string, materialize bool) ([]BatchResult, []*instrumentation.StatsEntry, error) {
	d.mux.RLock()
	defer d.mux.RUnlock()
	n := len(ins)
	if n == 0 {
		return nil, nil, nil
	}
	objs := (*C.gk_obj)(C.calloc(C.size_t(n), C.size_t(unsafe.Sizeof(C.gk_obj{}))))
	defer C.free(unsafe.Pointer(objs))
	arr := unsafe.Slice(objs, n)
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
	cstr := func(s string) *C.char {
		p := C.CString(s)
		owned = append(owned, unsafe.Pointer(p))
		return p
	}
	for i, in := range ins {
		o := &arr[i]
		ar := in.ar
		o.json, o.len = cbytes(ar.Object.Raw)
		o.old_json, o.old_len = cbytes(ar.OldObject.Raw)
		if in.ns != nil {
			b, err := json.Marshal(in.ns)
			if err != nil {
				return nil, nil, err
			}
			o.ns_json, o.ns_len = cbytes(b)
		}
		if ar.Namespace != "" { // AdmissionRequest.Namespace: review.namespace and the namespace-cache key (target.go:99-105)
			o.ns_name = cstr(ar.Namespace)
		}
		if ar.Operation != "" { // DELETE reviews the old object (target.go:262-280); templates read input.review.operation
			o.operation = cstr(string(ar.Operation))
		}
		if ub, err := json.Marshal(ar.UserInfo); err == nil && string(ub) != "{}" { // input.review.userInfo
			o.userinfo_json, o.userinfo_len = cbytes(ub)
		}
		o.source = sourceCode(in.source)
	}
	cep := C.CString(ep)
	defer C.free(unsafe.Pointer(cep))
	var res C.gk_result
	var cerr *C.char
	flags := C.uint32_t(0)
	if materialize {
		flags = C.GK_F_MATERIALIZE
	}
	if rc := C.gk_review_batch(d.e, objs, C.size_t(n), cep, flags, &res, &cerr); rc != 0 {
		return nil, nil, takeErr(cerr)
	}
	defer C.gk_free_result(&res)
	// a review-level error of an object is an error of the call: admission must not fail open, audit must not under-report
	if res.object_errors != nil {
		oe := unsafe.Slice(res.object_errors, n)
		for i, e := range oe {
			if e != nil {
				return nil, nil, fmt.Errorf("review of object %d: %s", i, C.GoString(e))
			}
		}
	}
	out := make([]BatchResult, 0, int(res.n_violations))
	vs := unsafe.Slice(res.violations, int(res.n_violations))
	for _, v := range vs {
		var details interface{}
		if dj := C.GoString(v.details_json); dj != "" {
			_ = json.Unmarshal([]byte(dj), &details)
		}
		var scoped []string
		_ = json.Unmarshal([]byte(C.GoString(v.scoped_actions_json)), &scoped)
		out = append(out, BatchResult{Object: int(v.object), Constraint: C.GoString(C.gk_result_constraint_key(&res, v.constraint)),
			Msg: C.GoString(v.msg), Details: details, EnforcementAction: C.GoString(v.enforcement_action), ScopedActions: scoped,
			Autoreject: v.autoreject != 0})
	}
	stats := []*instrumentation.StatsEntry{{Scope: "batch", StatsFor: fmt.Sprintf("%d reviews", n),
		Stats: []*instrumentation.Stat{
			{Name: "kernelTimeNS", Value: uint64(float64(res.kernel_ms) * 1e6), Source: instrumentation.Source{Type: instrumentation.EngineSourceType, Value: Name}},
			{Name: "flattenTimeNS", Value: uint64(float64(res.flatten_ms) * 1e6), Source: instrumentation.Source{Type: instrumentation.EngineSourceType, Value: Name}},
			{Name: "batchSize", Value: n, Source: instrumentation.Source{Type: instrumentation.EngineSourceType, Value: Name}},
			{Name: "bytesRead", Value: uint64(res.alg_bytes), Source: instrumentation.Source{Type: instrumentation.EngineSourceType, Value: Name}},
		}}}
	return out, stats, nil
}

func (d *Driver) Dump(_ context.Context) (string, error) {
	d.mux.RLock()
	defer d.mux.RUnlock()
	c := C.gk_dump(d.e)
	defer C.gk_free_str(c)
	return C.GoString(c), nil
}

func (d *Driver) GetDescriptionForStat(statName string) (string, error) {
	cs := C.CString(statName)
	defer C.free(unsafe.Pointer(cs))
	if desc := C.gk_stat_description(cs); desc != nil {
		return C.GoString(desc), nil
	}
	return "", fmt.Errorf("unknown stat name for Rego (GPU): %s", statName)
}

// regoSource returns the entry-point module and the template's libs (`package lib.<...>` modules the entry point imports as
// data.lib.<...>): `code[engine=Rego].source.{rego,libs}` first, the legacy `rego` / `libs` target fields otherwise.
func regoSource(ct *templates.ConstraintTemplate) (string, []string, error) {
	if len(ct.Spec.Targets) != 1 {
		return "", nil, errors.New("expected exactly one target")
	}
	t := ct.Spec.Targets[0]
	for _, code := range t.Code {
		if code.Engine == Name {
			if m, ok := code.Source.Value.(map[string]interface{}); ok {
				if s, ok := m["rego"].(string); ok {
					var libs []string
					if ls, ok := m["libs"].([]interface{}); ok {
						for _, l := range ls {
							if str, ok := l.(string); ok {
								libs = append(libs, str)
							}
						}
					}
					return s, libs, nil
				}
			}
		}
	}
	if t.Rego != "" {
		return t.Rego, t.Libs, nil
	}
	return "", nil, errors.New("no Rego source in template (ErrNoDriver)")
}
