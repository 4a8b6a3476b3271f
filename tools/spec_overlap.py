"""GPU probe: the timeline of one evaluation of a resident page through the generated kernel -- the interpreter's units
(gk_eval_kernel, list mode) on the side stream, gk_spec_rows_kernel and gk_spec_kernel on the caller's --
from a torch.profiler trace.  Prints, per kernel, its mean duration and its start and end relative to the evaluation's first kernel,
and how much of the interpreter's time overlaps the rows kernel; writes the trace to OUT/spec_overlap.pt.trace.json.

    python tools/spec_overlap.py [--config 2] [--objects 1000000] [--wide 0] [--steps 5] [--out DIR] [--trace FILE]
"""
import argparse
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ap = argparse.ArgumentParser()
ap.add_argument("--config", type=int, default=2)
ap.add_argument("--objects", type=int, default=1000000)
ap.add_argument("--wide", type=int, default=0, help="every WIDE-th object gets 40 containers (as tools/spec_probe.py)")
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "spec_overlap"))
ap.add_argument("--trace", help="only summarise this trace, written before")
a = ap.parse_args()

def profile():
    import torch

    from gatekeeper_b200 import driver as D, workloads as Wl

    tmpls, cons = {2: Wl.config2, 4: Wl.config4, 5: Wl.config5}[a.config]()
    drv = D.Driver()
    for kind, rego in tmpls:
        drv.add_template(kind, rego)
    for c in cons:
        drv.AddConstraint(c)
    for ns in Wl.synth_namespaces():
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    blob = Wl.synth_objects(0, a.objects, mode=1 if a.config == 4 else 0)
    if a.wide:
        docs = [blob.get(i) for i in range(a.objects)]
        for i in range(0, a.objects, a.wide):
            d = json.loads(docs[i])
            cs = d.get("spec", {}).get("containers") or [{"name": "c", "image": "nginx"}]
            d["spec"]["containers"] = [dict(cs[k % len(cs)], name="c%d" % k) for k in range(40)]
            docs[i] = json.dumps(d).encode()
        blob = Wl.PyBlob(docs)
    rb = drv.upload_blob(blob)

    # one traced evaluation, outside the profiled ones
    err = tempfile.TemporaryFile()
    saved = os.dup(2)
    os.dup2(err.fileno(), 2)
    os.environ["GK_TRACE_LAUNCH"] = "1"
    try:
        rb.eval(D.AUDIT_EP, D.F_NO_COPY_BACK)
    finally:
        os.environ.pop("GK_TRACE_LAUNCH", None)
        os.dup2(saved, 2)
        os.close(saved)
    err.seek(0)
    handed = re.findall(rb"\[spec\] handed to the interpreter: [^\n]*", err.read())
    print("kernel:", drv.last_kernel(), "|", handed[-1].decode() if handed else "no hand-over line")
    for _ in range(3):
        rb.eval(D.AUDIT_EP, D.F_NO_COPY_BACK)
    torch.cuda.synchronize()

    os.makedirs(a.out, exist_ok=True)
    path = os.path.join(a.out, "spec_overlap.pt.trace.json")
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            rb.eval(D.AUDIT_EP, D.F_NO_COPY_BACK)
        torch.cuda.synchronize()
    prof.export_chrome_trace(path)
    rb.free()
    drv.close()
    return path


path = a.trace or profile()
NAMES = ("gk_spec_plan_kernel", "gk_eval_kernel", "gk_spec_rows_kernel", "gk_spec_kernel")
ev = []
for e in json.load(open(path))["traceEvents"]:
    name = next((k for k in NAMES if e.get("cat") == "kernel" and re.match(r"(gk::)?%s\b" % k, e.get("name", ""))), None)
    if name:
        ev.append(dict(e, name=name))
ev.sort(key=lambda e: e["ts"])
# an evaluation ends with its tile kernel: the next kernel starts the next one
steps, cur = [], None
for e in ev:
    if cur is None or "gk_spec_kernel" in cur:
        cur = {}
        steps.append(cur)
    cur.setdefault(e["name"], (e["ts"], e["ts"] + e["dur"]))
steps = [s for s in steps if all(k in s for k in NAMES[1:])]   # (the evaluations with units)
print("%d evaluations in the trace (%s)" % (len(steps), path))
for k in NAMES:
    got = [s[k] for s in steps if k in s]
    if not got:
        continue
    t0s = [min(v[0] for v in s.values()) for s in steps if k in s]
    print("  %-20s %8.1f us  starts %+8.1f us  ends %+8.1f us" % (k, sum(b - a for a, b in got) / len(got), sum(a - t for (a, _), t in zip(got, t0s)) / len(got),
                                                           sum(b - t for (_, b), t in zip(got, t0s)) / len(got)))
ov = [max(0.0, min(s["gk_eval_kernel"][1], s["gk_spec_rows_kernel"][1]) - max(s["gk_eval_kernel"][0], s["gk_spec_rows_kernel"][0])) for s in steps]
span = [max(v[1] for v in s.values()) - min(v[0] for v in s.values()) for s in steps]
if steps:
    print("  gk_eval_kernel overlaps gk_spec_rows_kernel by %.1f us on average; first kernel start to last kernel end %.1f us" % (sum(ov) / len(ov), sum(span) / len(span)))
