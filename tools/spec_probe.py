"""GPU probe: the kernels generated for the constraint set (gk_spec_rows_kernel + gk_spec_kernel, NVRTC) against the netlist
interpreter (gk_eval_kernel) on a resident page of a BASELINE configuration -- identical bitmaps / totals / error lists, and the
launch time (both kernels) of several build variants (threads per CTA x minimum resident CTAs = register cap).

    python tools/spec_probe.py [--config 2] [--objects 1000000] [--variants 256x3,256x3@256x8,256x2,256x3:NOMATCH,256x3:STAGEONLY]
                               [--wide 1000] [--handover 0,4,8,16]

A variant is TILExMINB[@ROWSxMINB][:SWITCH+SWITCH]: the shape of gk_spec_kernel, optionally of gk_spec_rows_kernel, and measurement
switches of the text (GENERIC = spec.match through the shared gk_match(); otherwise -DGK_SPEC_X_<SWITCH>: NOMATCH, STAGEONLY).
With --handover, every variant runs once per value of GK_HANDOVER_MAX (program.h; 0 = every tile with a wide object handed over
whole).  Each line reports the units handed to the interpreter and the objects they hold (traced once, outside the timed loop).
"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--config", type=int, default=2)
ap.add_argument("--objects", type=int, default=1000000)
ap.add_argument("--variants", default="256x3,256x3@256x8,256x2,256x3:NOMATCH,256x3:STAGEONLY")
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--wide", type=int, default=0, help="every WIDE-th object gets 40 containers (exercises the hand-over)")
ap.add_argument("--handover", default="", help="comma-separated values of GK_HANDOVER_MAX to run each variant at")
a = ap.parse_args()

from gatekeeper_b200 import driver as D, workloads as Wl  # noqa: E402


def engine():
    drv = D.Driver()
    if a.config == 2:
        tmpls, cons = Wl.config2()
    elif a.config == 4:
        tmpls, cons = Wl.config4()
    else:
        tmpls, cons = Wl.config5()
    for kind, rego in tmpls:
        drv.add_template(kind, rego)
    for c in cons:
        drv.AddConstraint(c)
    for ns in Wl.synth_namespaces():
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    return drv


mode = 1 if a.config == 4 else 0
blob = Wl.synth_objects(0, a.objects, mode=mode)
if a.wide:
    docs = [blob.get(i) for i in range(a.objects)]
    for i in range(0, a.objects, a.wide):
        d = json.loads(docs[i])
        cs = d.get("spec", {}).get("containers") or [{"name": "c", "image": "nginx"}]
        d["spec"]["containers"] = [dict(cs[k % len(cs)], name="c%d" % k) for k in range(40)]
        docs[i] = json.dumps(d).encode()
    blob = Wl.PyBlob(docs)


def run(label, env):
    for k in ("GK_SPEC", "GK_SPEC_THREADS", "GK_SPEC_MINB", "GK_SPEC_ROWS_THREADS", "GK_SPEC_ROWS_MINB", "GK_SPEC_DEFS"):
        os.environ.pop(k, None)
    os.environ.update(env)
    drv = engine()
    drv.pin_blob(blob)
    rb = drv.upload_blob(blob)
    # the first evaluation builds the kernel and, traced, reports the hand-over: outside the timed launches below
    err = tempfile.TemporaryFile()
    saved = os.dup(2)
    os.dup2(err.fileno(), 2)
    os.environ["GK_TRACE_LAUNCH"] = "1"
    try:
        t0 = time.perf_counter()
        r = rb.eval(D.AUDIT_EP)
        first_s = time.perf_counter() - t0
    finally:
        os.environ.pop("GK_TRACE_LAUNCH", None)
        os.dup2(saved, 2)
        os.close(saved)
    err.seek(0)
    m = re.findall(rb"handed to the interpreter: (\d+) units .*?, (\d+) objects", err.read())
    handed = [int(x) for x in m[-1]] if m else None
    ms = []
    for _ in range(3 + a.steps):
        ms.append(rb.eval(D.AUDIT_EP, D.F_NO_COPY_BACK).stats["kernel_ms"])
    ms = ms[3:]
    out = {"label": label, "kernel": drv.last_kernel(), "kernel_ms": round(sum(ms) / len(ms), 4), "min_ms": round(min(ms), 4), "first_eval_s": round(first_s, 2),
           "alg_bytes": rb.alg_bytes + a.objects * r.viol_bits.shape[1] * 8, "handed_units_objects": handed}
    out["GBps"] = round(out["alg_bytes"] / out["kernel_ms"] / 1e6, 1)
    res = (np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True), list(r.totals), list(r.err_totals), sorted((x.object, x.constraint, x.msg) for x in r.results if x.autoreject))
    rb.free()
    drv.pin_blob(blob, False)
    drv.close()
    return out, res


base, want = run("interpreter", {"GK_SPEC": "0"})
print(json.dumps(base), flush=True)
for v, k in [(v, k) for v in a.variants.split(",") for k in (a.handover.split(",") if a.handover else [None])]:
    v, _, sw = v.partition(":")
    v, _, rv = v.partition("@")
    th, mb = v.split("x")
    rows = dict(zip(("GK_SPEC_ROWS_THREADS", "GK_SPEC_ROWS_MINB"), rv.split("x"))) if rv else {}
    toks = [x for x in sw.split("+") if x]
    defs = " ".join(["-DGK_SPEC_X_" + x for x in toks if x != "GENERIC"] + (["-DGK_HANDOVER_MAX=%su" % k] if k is not None else []))
    os.environ["GK_SPEC_MATCHGEN"] = "0" if "GENERIC" in toks else "1"
    o, got = run("spec " + v + ("@" + rv if rv else "") + (" " + sw if sw else "") + (" K=%s" % k if k is not None else ""),
                 dict(rows, GK_SPEC_THREADS=th, GK_SPEC_MINB=mb, GK_SPEC_MIN_OBJECTS="0", GK_SPEC_DEFS=defs))
    o["identical"] = bool(np.array_equal(want[0], got[0]) and np.array_equal(want[1], got[1]) and want[2:] == got[2:])
    print(json.dumps(o), flush=True)
    assert o["identical"] or "NOMATCH" in sw or "STAGEONLY" in sw, "generated kernel and interpreter disagree"
    assert o["kernel"] == "gk_spec_kernel" or "hostemu" in os.environ.get("GK_ENGINE_LIB", ""), "the generated kernel did not run"
