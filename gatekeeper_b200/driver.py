"""Host-side mirror of the constraint-framework `drivers.Driver` interface over the C ABI.

The reference is Go and its host side would bind include/gk_engine.h with cgo (go/gpudriver/driver.go,
INTEGRATION.md).  There is no Go toolchain in this image, so this module is the same thin shim in Python
(ctypes): identical method names, argument meaning and error behaviour as the Driver implementation in
the reference tree (pkg/drivers/k8scel/driver.go:70-263), plus the additive batch entry point the audit
sweep uses.  Everything that decides a violation happens below the C ABI on the GPU; this file only
marshals arguments.  It fails loudly when the native library or a CUDA device is missing.
"""
from __future__ import annotations

import ctypes as C
import json
import os
from dataclasses import dataclass, field
from typing import Any, Iterable, Optional, Sequence

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("GK_ENGINE_LIB") or os.path.join(_HERE, "libgk_engine.so")   # override only for kernel-variant experiments

WEBHOOK_EP = "validation.gatekeeper.sh"   # pkg/util/enforcement_action.go:24-39
AUDIT_EP = "audit.gatekeeper.sh"
GATOR_EP = "gator.gatekeeper.sh"

SOURCE = {"": 0, None: 0, "Original": 1, "Generated": 2, "All": 3}

F_BITMAP_ONLY, F_MATERIALIZE, F_NO_COPY_BACK = 0, 1, 2
F_KEEP_SOURCE = 4
F_EXPAND = 8          # expand the page's generator objects (ExpansionTemplates): an expanded batch
F_PROCESS_AUDIT, F_PROCESS_WEBHOOK = 16, 32
PROCESS_FLAG = {"": 0, None: 0, "audit": F_PROCESS_AUDIT, "webhook": F_PROCESS_WEBHOOK}


class GkError(RuntimeError):
    """Error returned across the C ABI (AddTemplate compile errors, CUDA failures, ...)."""

    def __init__(self, code: int, msg: str):
        super().__init__(msg)
        self.code = code


class gk_cfg(C.Structure):
    _fields_ = [("device", C.c_int32), ("threads", C.c_int32)]


class gk_obj(C.Structure):
    _fields_ = [("json", C.c_char_p), ("len", C.c_size_t), ("old_json", C.c_char_p), ("old_len", C.c_size_t),
                ("ns_json", C.c_char_p), ("ns_len", C.c_size_t), ("ns_name", C.c_char_p), ("operation", C.c_char_p),
                ("userinfo_json", C.c_char_p), ("userinfo_len", C.c_size_t), ("source", C.c_uint8)]


class gk_violation(C.Structure):
    _fields_ = [("object", C.c_uint32), ("constraint", C.c_uint32), ("msg", C.c_char_p), ("details_json", C.c_char_p),
                ("enforcement_action", C.c_char_p), ("scoped_actions_json", C.c_char_p), ("autoreject", C.c_uint8)]


class gk_result(C.Structure):
    _fields_ = [("n_objects", C.c_uint32), ("n_constraints", C.c_uint32), ("words", C.c_uint32),
                ("viol_bits", C.POINTER(C.c_uint32)), ("err_bits", C.POINTER(C.c_uint32)),
                ("totals", C.POINTER(C.c_uint64)), ("err_totals", C.POINTER(C.c_uint64)),
                ("violations", C.POINTER(gk_violation)), ("n_violations", C.c_size_t),
                ("object_errors", C.POINTER(C.c_char_p)),
                ("flatten_ms", C.c_double), ("h2d_ms", C.c_double), ("kernel_ms", C.c_double), ("d2h_ms", C.c_double),
                ("materialize_ms", C.c_double), ("alg_bytes", C.c_uint64), ("h2d_bytes", C.c_uint64),
                ("d2h_bytes", C.c_uint64), ("gpu_launches", C.c_uint64), ("priv", C.c_void_p)]


EXPORTS = [
    "gk_engine_create", "gk_engine_destroy", "gk_backend_name", "gk_last_kernel", "gk_add_template", "gk_add_template_libs", "gk_remove_template",
    "gk_add_constraint", "gk_add_expansion_template", "gk_remove_expansion_template", "gk_expansion_conflicts", "gk_validate_constraint", "gk_remove_constraint", "gk_put_namespace", "gk_remove_namespace", "gk_add_data", "gk_remove_data", "gk_constraint_count",
    "gk_constraint_key", "gk_result_constraint_key", "gk_review_batch", "gk_batch_upload", "gk_batch_eval", "gk_batch_eval_device",
    "gk_batch_eval_device_peers", "gk_batch_upload_blob", "gk_review_blob", "gk_set_excluded_namespaces", "gk_audit_begin", "gk_audit_add_batch", "gk_audit_report",
    "gk_audit_end", "gk_validation_messages", "gk_host_cpus", "gk_pin_host", "gk_blob_prefetch", "gk_coalescer_create", "gk_coalescer_review", "gk_coalescer_stats",
    "gk_coalescer_destroy", "gk_batch_size", "gk_batch_alg_bytes", "gk_batch_free", "gk_batch_refresh", "gk_batch_patch", "gk_free_result", "gk_free_str", "gk_dump",
    "gk_stat_description", "gk_audit_add_batch_ordered", "gk_audit_select_ms", "gk_audit_export", "gk_audit_merge",
    "gk_audit_resultant_pairs",
]


def load_library(path: Optional[str] = None) -> C.CDLL:
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise GkError(-3, f"native library {path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
    lib = C.CDLL(path)
    P, S, U32, U64 = C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint64
    PP = C.POINTER(C.c_char_p)
    lib.gk_engine_create.restype = P
    lib.gk_engine_create.argtypes = [C.POINTER(gk_cfg), PP]
    lib.gk_engine_destroy.argtypes = [P]
    lib.gk_backend_name.restype = S
    lib.gk_backend_name.argtypes = [P]
    lib.gk_last_kernel.restype = S
    lib.gk_last_kernel.argtypes = [P]
    lib.gk_add_template.argtypes = [P, S, S, C.c_size_t, PP]
    lib.gk_add_template_libs.argtypes = [P, S, S, C.c_size_t, C.POINTER(C.c_char_p), C.POINTER(C.c_size_t), C.c_size_t, PP]
    lib.gk_remove_template.argtypes = [P, S]
    lib.gk_add_constraint.argtypes = [P, S, C.c_size_t, PP]
    lib.gk_add_expansion_template.argtypes = [P, S, C.c_size_t, PP]
    lib.gk_remove_expansion_template.argtypes = [P, S]
    lib.gk_expansion_conflicts.restype = C.c_void_p
    lib.gk_expansion_conflicts.argtypes = [P]
    lib.gk_validate_constraint.argtypes = [P, S, C.c_size_t, PP]
    lib.gk_remove_constraint.argtypes = [P, S, S]
    lib.gk_put_namespace.argtypes = [P, S, S, C.c_size_t, PP]
    lib.gk_add_data.argtypes = [P, C.POINTER(C.c_char_p), C.c_size_t, S, C.c_size_t, PP]
    lib.gk_remove_data.argtypes = [P, C.POINTER(C.c_char_p), C.c_size_t]
    lib.gk_remove_namespace.argtypes = [P, S]
    lib.gk_constraint_count.restype = U32
    lib.gk_constraint_count.argtypes = [P]
    lib.gk_constraint_key.restype = S
    lib.gk_constraint_key.argtypes = [P, U32]
    lib.gk_result_constraint_key.restype = S
    lib.gk_result_constraint_key.argtypes = [C.POINTER(gk_result), U32]
    lib.gk_review_batch.argtypes = [P, C.POINTER(gk_obj), C.c_size_t, S, U32, C.POINTER(gk_result), PP]
    lib.gk_batch_upload.argtypes = [P, C.POINTER(gk_obj), C.c_size_t, U32, C.POINTER(P), C.POINTER(gk_result), PP]
    lib.gk_batch_eval.argtypes = [P, P, S, U32, C.POINTER(gk_result), PP]
    lib.gk_batch_eval_device.argtypes = [P, P, S, P, P, P, P, P, PP]
    lib.gk_batch_eval_device_peers.argtypes = [P, P, S, C.POINTER(C.c_uint64), U32, U32, C.c_uint64, C.c_uint64, U32, P, P, P, P, PP]
    lib.gk_batch_upload_blob.argtypes = [P, P, C.POINTER(C.c_uint64), C.c_size_t, C.c_uint8, U32, C.POINTER(P), C.POINTER(gk_result), PP]
    lib.gk_review_blob.argtypes = [P, P, C.POINTER(C.c_uint64), C.c_size_t, C.c_uint8, S, U32, C.POINTER(gk_result), PP]
    lib.gk_batch_size.restype = U32
    lib.gk_set_excluded_namespaces.argtypes = [P, S, C.POINTER(C.c_char_p), C.c_size_t, PP]
    lib.gk_audit_begin.argtypes = [P, U32, U32, PP]
    lib.gk_audit_begin.restype = P
    lib.gk_audit_add_batch.argtypes = [P, P, S, PP]
    lib.gk_audit_add_batch_ordered.argtypes = [P, P, S, PP]
    lib.gk_audit_select_ms.argtypes = [P]
    lib.gk_audit_select_ms.restype = C.c_float
    lib.gk_audit_resultant_pairs.argtypes = [P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.gk_audit_export.argtypes = [P, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), PP]
    lib.gk_audit_merge.argtypes = [P, C.c_char_p, C.c_size_t, PP]
    lib.gk_audit_report.argtypes = [P, PP]
    lib.gk_audit_report.restype = C.c_void_p
    lib.gk_audit_end.argtypes = [P]
    lib.gk_audit_end.restype = None
    lib.gk_validation_messages.argtypes = [P, C.POINTER(gk_result), U32, PP]
    lib.gk_validation_messages.restype = C.c_void_p
    lib.gk_coalescer_create.argtypes = [P, U32, U32, S, U32, PP]
    lib.gk_coalescer_create.restype = P
    lib.gk_coalescer_review.argtypes = [P, C.POINTER(gk_obj), C.POINTER(C.c_void_p), PP]
    lib.gk_coalescer_stats.argtypes = [P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    lib.gk_coalescer_stats.restype = None
    lib.gk_coalescer_destroy.argtypes = [P]
    lib.gk_coalescer_destroy.restype = None
    lib.gk_host_cpus.argtypes = []
    lib.gk_host_cpus.restype = C.c_int
    lib.gk_pin_host.argtypes = [P, C.c_void_p, C.c_size_t, C.c_int, PP]
    lib.gk_blob_prefetch.argtypes = [P, C.c_void_p, C.POINTER(C.c_uint64), C.c_size_t, PP]
    lib.gk_batch_size.argtypes = [P]
    lib.gk_batch_alg_bytes.restype = U64
    lib.gk_batch_alg_bytes.argtypes = [P]
    lib.gk_batch_free.argtypes = [P, P]
    lib.gk_batch_refresh.argtypes = [P, P, C.POINTER(gk_result), PP]
    lib.gk_batch_patch.argtypes = [P, P, C.POINTER(C.c_uint32), C.c_size_t, P, C.POINTER(C.c_uint64), C.c_size_t, C.POINTER(gk_result), PP]
    lib.gk_free_result.argtypes = [C.POINTER(gk_result)]
    lib.gk_free_str.argtypes = [C.c_void_p]
    lib.gk_dump.restype = C.c_void_p
    lib.gk_dump.argtypes = [P]
    lib.gk_stat_description.restype = S
    lib.gk_stat_description.argtypes = [S]
    return lib


@dataclass
class Review:
    """What target.HandleReview accepts: an object (+ optional oldObject / Namespace / source / operation)
    -- pkg/target/target.go:86-138, pkg/target/data.go:24-28."""
    object: Any = None                 # dict, JSON str/bytes, or None
    old_object: Any = None
    namespace: Any = None              # explicit Namespace object
    namespace_name: Optional[str] = None
    source: str = ""
    operation: str = ""
    user_info: Any = None


@dataclass
class Result:
    """types.Result -- fields as used at pkg/audit/manager.go:895-923."""
    object: int
    constraint: str                    # "Kind/name"
    msg: str
    details: Any
    enforcement_action: str
    scoped_enforcement_actions: list
    autoreject: bool = False


@dataclass
class BatchResponse:
    n_objects: int
    constraints: list                  # index -> "Kind/name"
    viol_bits: Any                     # numpy uint32 [n, words] or None
    err_bits: Any
    totals: list
    err_totals: list
    results: list = field(default_factory=list)
    object_errors: list = field(default_factory=list)
    stats: dict = field(default_factory=dict)
    _owner: Any = None                 # zero-copy responses: the engine-side result the bitmaps live in

    def pairs(self):
        """Set of (object index, constraint key) with the violation bit set."""
        out = set()
        if self.viol_bits is None:
            return out
        n, w = self.viol_bits.shape
        for o in range(n):
            for k in range(w):
                bits = int(self.viol_bits[o, k])
                while bits:
                    b = bits & -bits
                    out.add((o, self.constraints[k * 32 + b.bit_length() - 1]))
                    bits ^= b
        return out


def _to_bytes(x) -> Optional[bytes]:
    if x is None:
        return None
    if isinstance(x, bytes):
        return x
    if isinstance(x, str):
        return x.encode()
    return json.dumps(x, separators=(",", ":")).encode()


class Driver:
    """Mirror of `drivers.Driver` (method set at pkg/drivers/k8scel/driver.go:70-263).  `Name()` is "Rego":
    templates carrying `targets[].rego` / `code[engine: Rego]` route to this driver (SURVEY.md 8(b))."""

    def __init__(self, device: int = 0, threads: int = 0, lib_path: Optional[str] = None):
        self._lib = load_library(lib_path)
        err = C.c_char_p()
        cfg = gk_cfg(device, threads)
        self._e = self._lib.gk_engine_create(C.byref(cfg), C.byref(err))
        if not self._e:
            raise GkError(-3, self._take(err) or "gk_engine_create failed")

    # ---- plumbing
    def _take(self, err) -> str:
        if not err or not err.value:
            return ""
        s = err.value.decode(errors="replace")
        self._lib.gk_free_str(C.cast(err, C.c_void_p))
        return s

    def _check(self, rc: int, err):
        if rc != 0:
            raise GkError(rc, self._take(err) or f"error {rc}")

    def close(self):
        if getattr(self, "_e", None):
            self._lib.gk_engine_destroy(self._e)
            self._e = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- drivers.Driver
    def Name(self) -> str:
        return "Rego"

    def backend(self) -> str:
        return self._lib.gk_backend_name(self._e).decode()

    def last_kernel(self) -> str:
        """"gk_spec_kernel" (generated for the constraint set, NVRTC) or "gk_eval_kernel" (the netlist interpreter)."""
        return self._lib.gk_last_kernel(self._e).decode()

    def AddTemplate(self, template: dict) -> None:
        kind = template["spec"]["crd"]["spec"]["names"]["kind"]
        tgt = template["spec"]["targets"][0]
        src, libs = None, None
        for c in tgt.get("code") or []:      # `code` wins over the legacy fields, as in the framework's rego driver
            if c.get("engine") == "Rego":
                src = (c.get("source") or {}).get("rego")
                libs = (c.get("source") or {}).get("libs")
        if not src:
            src, libs = tgt.get("rego"), tgt.get("libs")
        if not src:
            raise GkError(-2, "no Rego source for this driver in the template (ErrNoDriver)")
        self.add_template(kind, src, libs or ())

    def add_template(self, kind: str, rego: str, libs: Sequence[str] = ()) -> None:
        err = C.c_char_p()
        b = rego.encode()
        if libs:
            lb = [x.encode() for x in libs]
            arr = (C.c_char_p * len(lb))(*lb)
            lens = (C.c_size_t * len(lb))(*[len(x) for x in lb])
            self._check(self._lib.gk_add_template_libs(self._e, kind.encode(), b, len(b), arr, lens, len(lb), C.byref(err)), err)
            return
        self._check(self._lib.gk_add_template(self._e, kind.encode(), b, len(b), C.byref(err)), err)

    def RemoveTemplate(self, template_or_kind) -> None:
        kind = template_or_kind if isinstance(template_or_kind, str) else template_or_kind["spec"]["crd"]["spec"]["names"]["kind"]
        self._lib.gk_remove_template(self._e, kind.encode())

    def AddConstraint(self, constraint: dict) -> None:
        err = C.c_char_p()
        b = _to_bytes(constraint)
        self._check(self._lib.gk_add_constraint(self._e, b, len(b), C.byref(err)), err)

    def AddExpansionTemplate(self, template: dict) -> None:
        """expansion.System.UpsertTemplate (pkg/expansion/system.go:60-73)"""
        b = json.dumps(template).encode()
        err = C.c_char_p()
        self._check(self._lib.gk_add_expansion_template(self._e, b, len(b), C.byref(err)), err)

    def RemoveExpansionTemplate(self, name: str) -> None:
        self._lib.gk_remove_expansion_template(self._e, name.encode())

    def ExpansionConflicts(self) -> list:
        """expansion.System.GetConflicts (pkg/expansion/system.go:81-83): names of the templates set aside as part of an expansion cycle"""
        p = self._lib.gk_expansion_conflicts(self._e)
        s = C.string_at(p).decode() if p else "[]"
        if p:
            self._lib.gk_free_str(p)
        return json.loads(s)

    def ValidateConstraint(self, constraint: dict) -> None:
        """TargetHandler.ValidateConstraint (pkg/target/target.go:178-214); raises GkError for a constraint the reference's
        client would refuse before it reaches the driver."""
        err = C.c_char_p()
        b = json.dumps(constraint).encode()
        self._check(self._lib.gk_validate_constraint(self._e, b, len(b), C.byref(err)), err)

    def RemoveConstraint(self, constraint: dict) -> None:
        self._lib.gk_remove_constraint(self._e, constraint["kind"].encode(), constraint["metadata"]["name"].encode())

    def AddData(self, target: str, path: Sequence[str], data: Any) -> None:
        """Client.AddData (frameworks client): Namespaces feed the namespaceSelector table (nsCache.Add), and every object is
        stored at its path for referential templates (data.inventory); path shapes per pkg/target/target.go:60-66."""
        err = C.c_char_p()
        b = _to_bytes(data)
        if len(path) >= 4 and path[0] == "cluster" and path[2] == "Namespace":
            self._check(self._lib.gk_put_namespace(self._e, path[3].encode(), b, len(b), C.byref(err)), err)
        arr = (C.c_char_p * len(path))(*[p.encode() for p in path])
        self._check(self._lib.gk_add_data(self._e, arr, len(path), b, len(b), C.byref(err)), err)

    def RemoveData(self, target: str, path: Sequence[str]) -> None:
        if len(path) >= 4 and path[0] == "cluster" and path[2] == "Namespace":
            self._lib.gk_remove_namespace(self._e, path[3].encode())
        arr = (C.c_char_p * len(path))(*[p.encode() for p in path])
        self._lib.gk_remove_data(self._e, arr, len(path))

    def Dump(self) -> str:
        p = self._lib.gk_dump(self._e)
        s = C.string_at(p).decode() if p else ""
        if p:
            self._lib.gk_free_str(p)
        return s

    def GetDescriptionForStat(self, name: str) -> str:
        d = self._lib.gk_stat_description(name.encode())
        if d is None:
            raise GkError(-1, f"unknown stat name for Rego (GPU): {name}")
        return d.decode()

    def constraints(self) -> list:
        n = self._lib.gk_constraint_count(self._e)
        out = []
        for i in range(n):
            k = self._lib.gk_constraint_key(self._e, i)      # None: the constraint set shrank between the two calls
            if k is None:
                break
            out.append(k.decode())
        return out

    # ---- reviews
    def _marshal(self, reviews: Iterable):
        keep = []
        arr_t = []
        for r in reviews:
            if not isinstance(r, Review):
                r = Review(object=r)
            o = gk_obj()
            j, oj, nj, uj = _to_bytes(r.object), _to_bytes(r.old_object), _to_bytes(r.namespace), _to_bytes(r.user_info)
            nn = r.namespace_name.encode() if r.namespace_name is not None else None
            op = r.operation.encode() if r.operation else None
            keep.append((j, oj, nj, uj, nn, op))
            o.json, o.len = j, len(j) if j else 0
            o.old_json, o.old_len = oj, len(oj) if oj else 0
            o.ns_json, o.ns_len = nj, len(nj) if nj else 0
            o.ns_name = nn
            o.operation = op
            o.userinfo_json, o.userinfo_len = uj, len(uj) if uj else 0
            o.source = SOURCE.get(r.source, 4)
            arr_t.append(o)
        arr = (gk_obj * max(1, len(arr_t)))(*arr_t)
        return arr, len(arr_t), keep

    def _unpack(self, res: gk_result, keys: list, with_results: bool = True, zero_copy: bool = False) -> BatchResponse:
        """zero_copy: the bitmaps stay in the engine's (page-locked) result buffers; the response owns the result and frees it
        when it is collected -- what a C / Go caller does by reading gk_result in place."""
        import numpy as np
        n, w, c = res.n_objects, res.words, res.n_constraints
        take = (lambda a: a) if zero_copy else (lambda a: a.copy())
        if res.priv:
            # the result names its own columns (the engine's constraint set may have changed since the review started)
            own = [self._lib.gk_result_constraint_key(C.byref(res), i) for i in range(c)]
            if all(k is not None for k in own):
                keys = [k.decode() for k in own]
        if keys is None:
            keys = self.constraints()
        vb = eb = None
        if res.viol_bits:
            vb = take(np.ctypeslib.as_array(res.viol_bits, shape=(n * w,))).reshape(n, w) if n else np.zeros((0, w), np.uint32)
        if res.err_bits:
            eb = take(np.ctypeslib.as_array(res.err_bits, shape=(n * w,))).reshape(n, w) if n else np.zeros((0, w), np.uint32)
        out = BatchResponse(
            n_objects=n, constraints=keys, viol_bits=vb, err_bits=eb,
            totals=[int(res.totals[i]) for i in range(c)], err_totals=[int(res.err_totals[i]) for i in range(c)],
            stats={k: getattr(res, k) for k in ("flatten_ms", "h2d_ms", "kernel_ms", "d2h_ms", "materialize_ms", "alg_bytes",
                                                "h2d_bytes", "d2h_bytes", "gpu_launches")})
        out.stats["n_violations"] = int(res.n_violations)
        for i in range(res.n_violations if with_results else 0):
            v = res.violations[i]
            dj = v.details_json.decode() if v.details_json else ""
            out.results.append(Result(v.object, keys[v.constraint], v.msg.decode(errors="replace"), json.loads(dj) if dj else None,
                                      v.enforcement_action.decode(), json.loads(v.scoped_actions_json.decode()), bool(v.autoreject)))
        if res.object_errors:
            out.object_errors = [(res.object_errors[i].decode() if res.object_errors[i] else None) for i in range(n)]
        if zero_copy:
            out._owner = _ResultOwner(self._lib, res)
        return out

    def ReviewBatch(self, reviews: Iterable, enforcement_point: str = AUDIT_EP, materialize: bool = True, process: str = "") -> BatchResponse:
        """The additive batch entry point (SURVEY.md 8(b) `BatchReviewer`): Client.Review semantics -- match
        pre-filter, enforcement-point filter, evaluation, EnforcementAction stamping -- for many reviews at once."""
        arr, n, keep = self._marshal(reviews)
        res = gk_result()
        err = C.c_char_p()
        keys = None           # (the result names its own constraint columns)
        rc = self._lib.gk_review_batch(self._e, arr, n, enforcement_point.encode(),
                                       (F_MATERIALIZE if materialize else 0) | PROCESS_FLAG.get(process, 0), C.byref(res), C.byref(err))
        self._check(rc, err)
        try:
            return self._unpack(res, keys)
        finally:
            self._lib.gk_free_result(C.byref(res))

    def review_marshalled(self, arr, n: int, enforcement_point: str, flags: int = 0) -> BatchResponse:
        """gk_review_batch on requests already marshalled by _marshal(); results stay in the engine's buffers (stats only)."""
        res = gk_result()
        err = C.c_char_p()
        self._check(self._lib.gk_review_batch(self._e, arr, n, enforcement_point.encode(), flags, C.byref(res), C.byref(err)), err)
        try:
            return self._unpack(res, None, with_results=False)
        finally:
            self._lib.gk_free_result(C.byref(res))

    def Query(self, target: str, constraints: Sequence[dict], review, enforcement_point: str = AUDIT_EP) -> list:
        """drivers.Driver.Query shape (pkg/drivers/k8scel/driver.go:161-250): one review, the (already
        matched) constraints; returns the Results for those constraints."""
        want = {f"{c['kind']}/{c['metadata']['name']}" for c in constraints}
        resp = self.ReviewBatch([review], enforcement_point)
        if resp.object_errors and resp.object_errors[0]:
            raise GkError(-1, resp.object_errors[0])
        return [r for r in resp.results if r.constraint in want]

    def SetExcludedNamespaces(self, process: str, patterns: Sequence[str]):
        """process.Excluder.Add for one process (pkg/controller/config/process/excluder.go:53-77)."""
        arr = (C.c_char_p * max(1, len(patterns)))(*[p.encode() for p in patterns])
        err = C.c_char_p()
        self._check(self._lib.gk_set_excluded_namespaces(self._e, process.encode(), arr, len(patterns), C.byref(err)), err)

    def ValidationMessages(self, reviews: Iterable, process: str = "webhook"):
        """validationHandler.review + getValidationMessages (pkg/webhook/policy.go:238-355,661) for a micro-batch of
        admission reviews: per request (denyMsgs, warnMsgs)."""
        arr, n, keep = self._marshal(reviews)
        res = gk_result()
        err = C.c_char_p()
        self._check(self._lib.gk_review_batch(self._e, arr, n, WEBHOOK_EP.encode(), F_MATERIALIZE | PROCESS_FLAG.get(process, 0),
                                              C.byref(res), C.byref(err)), err)
        out = []
        try:
            for i in range(n):
                p = self._lib.gk_validation_messages(self._e, C.byref(res), i, C.byref(err))
                if not p:
                    self._check(-1, err)
                d = json.loads(C.string_at(p).decode(errors="surrogateescape"))
                self._lib.gk_free_str(p)
                out.append((d["deny"], d["warn"]))
        finally:
            self._lib.gk_free_result(C.byref(res))
        return out

    # ---- resident batches (audit sweep / bench)
    def upload(self, reviews: Iterable, process: str = "", expand: bool = False):
        """Flatten + upload review objects.  expand: an expanded batch (F_EXPAND) -- its generators' resultants are kept with it and
        folded into their parents' rows by every evaluation."""
        arr, n, keep = self._marshal(reviews)
        h = C.c_void_p()
        stats = gk_result()
        err = C.c_char_p()
        flags = PROCESS_FLAG.get(process, 0) | (F_EXPAND if expand else 0)
        self._check(self._lib.gk_batch_upload(self._e, arr, n, flags, C.byref(h), C.byref(stats), C.byref(err)), err)
        return ResidentBatch(self, h, (arr, keep), {"flatten_ms": stats.flatten_ms, "h2d_ms": stats.h2d_ms,
                                                    "h2d_bytes": stats.h2d_bytes, "alg_bytes": stats.alg_bytes})


    def pin_blob(self, blob, pin: bool = True):
        """Page-lock the blob's host buffer (gk_pin_host) so its host->device copy runs at link speed."""
        err = C.c_char_p()
        self._check(self._lib.gk_pin_host(self._e, blob.buf, blob.total_bytes(), 1 if pin else 0, C.byref(err)), err)

    def prefetch_blob(self, blob):
        """Start streaming `blob` to the GPU (gk_blob_prefetch); the following ReviewBlob / upload_blob of it picks the copy up."""
        err = C.c_char_p()
        self._check(self._lib.gk_blob_prefetch(self._e, blob.buf, blob.offsets, len(blob), C.byref(err)), err)

    def upload_blob(self, blob, source: str = "Original", process: str = "", keep_source: bool = False, expand: bool = False):
        """Flatten + upload a page of objects held in one contiguous buffer (workloads.ObjectBlob).  keep_source: the batch keeps the
        page's JSON and token tape on the device, so that ResidentBatch.refresh() re-extracts it without copying it again.  expand: an
        expanded batch (F_EXPAND), as for upload()."""
        h = C.c_void_p()
        stats = gk_result()
        err = C.c_char_p()
        flags = PROCESS_FLAG.get(process, 0) | (F_KEEP_SOURCE if keep_source else 0) | (F_EXPAND if expand else 0)
        self._check(self._lib.gk_batch_upload_blob(self._e, blob.buf, blob.offsets, len(blob), SOURCE.get(source, 4), flags, C.byref(h),
                                                   C.byref(stats), C.byref(err)), err)
        return ResidentBatch(self, h, blob, {"flatten_ms": stats.flatten_ms, "h2d_ms": stats.h2d_ms, "h2d_bytes": stats.h2d_bytes,
                                             "alg_bytes": stats.alg_bytes})

    def ReviewBlob(self, blob, enforcement_point: str = AUDIT_EP, flags: int = 0, source: str = "Original", with_results: bool = True,
                   zero_copy: bool = False) -> BatchResponse:
        """End-to-end audit page: host JSON -> flatten -> H2D -> kernel -> D2H (+ optional message rendering).  `flags` go to
        gk_review_blob as they are: F_MATERIALIZE, F_EXPAND (expand the page's generators), F_PROCESS_*."""
        res = gk_result()
        err = C.c_char_p()
        keys = None
        self._check(self._lib.gk_review_blob(self._e, blob.buf, blob.offsets, len(blob), SOURCE.get(source, 4), enforcement_point.encode(),
                                             flags, C.byref(res), C.byref(err)), err)
        if zero_copy:
            return self._unpack(res, keys, with_results, zero_copy=True)
        try:
            return self._unpack(res, keys, with_results)
        finally:
            self._lib.gk_free_result(C.byref(res))


class _ResultOwner:
    """Keeps a gk_result alive for a zero-copy BatchResponse."""

    def __init__(self, lib, res):
        self._lib, self._res = lib, res

    def __del__(self):
        try:
            self._lib.gk_free_result(C.byref(self._res))
        except Exception:
            pass


class Coalescer:
    """Admission micro-batching (gk_coalescer_*): `review()` may be called from many threads; each call blocks until the
    micro-batch it joined has been evaluated and returns that request's outcome."""

    def __init__(self, drv: "Driver", max_batch: int = 64, max_wait_us: int = 200, enforcement_point: str = WEBHOOK_EP, process: str = "webhook"):
        self.drv = drv
        err = C.c_char_p()
        self._c = drv._lib.gk_coalescer_create(drv._e, max_batch, max_wait_us, enforcement_point.encode(), PROCESS_FLAG.get(process, 0), C.byref(err))
        if not self._c:
            drv._check(-1, err)

    def review(self, review: "Review") -> dict:
        arr, n, keep = self.drv._marshal([review])
        out = C.c_void_p()
        err = C.c_char_p()
        self.drv._check(self.drv._lib.gk_coalescer_review(self._c, arr, C.byref(out), C.byref(err)), err)   # (ctypes releases the GIL)
        try:
            return json.loads(C.string_at(out).decode(errors="surrogateescape"))
        finally:
            self.drv._lib.gk_free_str(out)

    def stats(self):
        b, r = C.c_uint64(), C.c_uint64()
        self.drv._lib.gk_coalescer_stats(self._c, C.byref(b), C.byref(r))
        return {"batches": b.value, "reviews": r.value}

    def close(self):
        if self._c:
            self.drv._lib.gk_coalescer_destroy(self._c)
            self._c = None


class AuditRun:
    """One audit sweep's aggregation (pkg/audit/manager.go:886-945,984-1041): fold reviewed batches, then report
    totalViolations and the per-constraint status lists."""

    def __init__(self, drv: "Driver", violations_limit: int = 0, msg_size: int = 0):
        self.drv = drv
        err = C.c_char_p()
        self._a = drv._lib.gk_audit_begin(drv._e, violations_limit, msg_size, C.byref(err))
        if not self._a:
            drv._check(-1, err)

    def add_batch(self, rb: "ResidentBatch", enforcement_point: str = AUDIT_EP):
        err = C.c_char_p()
        self.drv._check(self.drv._lib.gk_audit_add_batch(self._a, rb.h, enforcement_point.encode(), C.byref(err)), err)

    def add_batch_ordered(self, rb: "ResidentBatch", enforcement_point: str = AUDIT_EP):
        """add_batch with the candidates ranked and selected on the device: the lazy path for a page of any mix of kinds."""
        err = C.c_char_p()
        self.drv._check(self.drv._lib.gk_audit_add_batch_ordered(self._a, rb.h, enforcement_point.encode(), C.byref(err)), err)

    def select_ms(self) -> float:
        """Device time of the last add_batch_ordered's ranking and selection kernels (ms)."""
        return float(self.drv._lib.gk_audit_select_ms(self._a))

    def resultant_pairs(self) -> tuple:
        """(rendered, counted): the resultant violation pairs of expanded batches this run rendered on the host and counted from the
        bitmap (matcher-error pairs are in neither; merged exports do not carry them)."""
        ev, ct = C.c_uint64(), C.c_uint64()
        self.drv._check(self.drv._lib.gk_audit_resultant_pairs(self._a, C.byref(ev), C.byref(ct)), C.c_char_p())
        return ev.value, ct.value

    def export(self) -> bytes:
        """The run's partial state as an opaque, versioned byte string (merge() it into another run)."""
        err, buf, n = C.c_char_p(), C.c_void_p(), C.c_size_t()
        self.drv._check(self.drv._lib.gk_audit_export(self._a, C.byref(buf), C.byref(n), C.byref(err)), err)
        try:
            return C.string_at(buf, n.value)
        finally:
            self.drv._lib.gk_free_str(buf)

    def merge(self, data: bytes):
        """Fold an exported run in, as if its objects came after this run's."""
        err = C.c_char_p()
        self.drv._check(self.drv._lib.gk_audit_merge(self._a, bytes(data), len(data), C.byref(err)), err)

    def report(self) -> dict:
        err = C.c_char_p()
        p = self.drv._lib.gk_audit_report(self._a, C.byref(err))
        if not p:
            self.drv._check(-1, err)
        try:
            return json.loads(C.string_at(p).decode(errors="surrogateescape"))
        finally:
            self.drv._lib.gk_free_str(p)

    def close(self):
        if self._a:
            self.drv._lib.gk_audit_end(self._a)
            self._a = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class ResidentBatch:
    def __init__(self, drv: Driver, handle, keep, stats):
        self.drv, self.h, self._keep, self.stats = drv, handle, keep, stats

    def __len__(self):
        return self.drv._lib.gk_batch_size(self.h)

    @property
    def alg_bytes(self) -> int:
        return self.drv._lib.gk_batch_alg_bytes(self.h)

    def eval(self, enforcement_point: str = AUDIT_EP, flags: int = 0) -> BatchResponse:
        res = gk_result()
        err = C.c_char_p()
        keys = None
        self.drv._check(self.drv._lib.gk_batch_eval(self.drv._e, self.h, enforcement_point.encode(), flags, C.byref(res), C.byref(err)), err)
        try:
            return self.drv._unpack(res, keys)
        finally:
            self.drv._lib.gk_free_result(C.byref(res))

    def eval_device(self, enforcement_point, d_viol: int, d_err: int, d_totals: int, d_err_totals: int, stream: int = 0):
        err = C.c_char_p()
        self.drv._check(self.drv._lib.gk_batch_eval_device(self.drv._e, self.h, enforcement_point.encode(), d_viol, d_err, d_totals,
                                                           d_err_totals, stream, C.byref(err)), err)

    def eval_device_peers(self, enforcement_point, peer_bases, rank: int, slot_i32: int, tot_off_i32: int, tot_stride: int,
                          d_err: int, d_totals: int, d_err_totals: int, stream: int = 0):
        """Kernel with the fused exchange: bitmap words and totals go straight into every peer's receive buffer."""
        err = C.c_char_p()
        arr = (C.c_uint64 * len(peer_bases))(*peer_bases)
        self.drv._check(self.drv._lib.gk_batch_eval_device_peers(self.drv._e, self.h, enforcement_point.encode(), arr, len(peer_bases), rank,
                                                                 slot_i32, tot_off_i32, tot_stride, d_err, d_totals, d_err_totals, stream,
                                                                 C.byref(err)), err)

    def refresh(self) -> dict:
        """gk_batch_refresh: bring the batch to the engine's current constraint set (and excluder patterns, and data.inventory) so that
        eval() accepts it again.  Returns the call's statistics; "rebuilt" is False when the batch was already current."""
        stats = gk_result()
        err = C.c_char_p()
        rc = self.drv._lib.gk_batch_refresh(self.drv._e, self.h, C.byref(stats), C.byref(err))
        if rc < 0:
            self.drv._check(rc, err)
        out = {"flatten_ms": stats.flatten_ms, "h2d_ms": stats.h2d_ms, "h2d_bytes": stats.h2d_bytes, "alg_bytes": stats.alg_bytes}
        if rc == 1:
            self.stats = out
        return dict(out, rebuilt=rc == 1)

    def patch(self, drop: Sequence[int], docs) -> dict:
        """gk_batch_patch: the objects at indices `drop` leave the batch and `docs` (a workloads.ObjectBlob, or a list of JSON
        documents as bytes) are appended after the objects that stay; the batch is then what an upload of that page would be under the
        current constraint set.  The batch must have been uploaded with keep_source=True.  It keeps a reference to every page it
        was given, since the engine reads the objects' JSON from where it was handed over.  Returns the call's statistics and the
        new size as "n"."""
        import numpy as np
        from . import workloads as W
        page = docs if hasattr(docs, "offsets") else W.PyBlob(list(docs))
        idx = np.ascontiguousarray(list(drop) if not isinstance(drop, np.ndarray) else drop, dtype=np.uint32)
        stats = gk_result()
        err = C.c_char_p()
        rc = self.drv._lib.gk_batch_patch(self.drv._e, self.h, idx.ctypes.data_as(C.POINTER(C.c_uint32)), len(idx), page.buf if len(page) else None,
                                          page.offsets if len(page) else None, len(page), C.byref(stats), C.byref(err))
        if rc < 0:
            self.drv._check(rc, err)
        self._keep = (self._keep, page)
        self.stats = {"flatten_ms": stats.flatten_ms, "h2d_ms": stats.h2d_ms, "h2d_bytes": stats.h2d_bytes, "alg_bytes": stats.alg_bytes}
        return dict(self.stats, kernel_ms=stats.kernel_ms, n=rc)

    def free(self):
        if self.h:
            self.drv._lib.gk_batch_free(self.drv._e, self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass
