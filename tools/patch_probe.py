#!/usr/bin/env python
"""What replacing a few objects of a resident page costs: gk_batch_patch of a page uploaded with GK_F_KEEP_SOURCE against a fresh
gk_batch_upload_blob of the same resulting page.

    python tools/patch_probe.py [objects] [reps] [configs]

For config 2 (synthetic Pods) and config 4 (mixed kinds), `objects` objects (default 1 000 000), and 0.1 %, 1 % and 10 % of them
replaced by new versions (dropped, then added with a changed label).  Each rep uploads the page with its kept source (not timed),
then times the patch and a fresh upload of the resulting page, alternated.  Wall times end in a device synchronise (both calls return
with the batch ready); the patch's device time is its kernel_ms statistic (splice, the added objects' copy and tokeniser, the
extraction).  Each share checks that the patched batch and the fresh upload give identical planes and totals and a byte-identical
gk_audit_add_batch_ordered report.  The card's name, power limit and maximum SM clock are read in the same run.  One JSON line per
rep, then a summary line per configuration."""
import json
import os
import random
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from refresh_probe import gpu_info, planes

AUDIT = "audit.gatekeeper.sh"
SHARES = (0.001, 0.01, 0.1)


def new_version(doc, k):
    d = json.loads(doc)
    d.setdefault("metadata", {}).setdefault("labels", {})["patched"] = "v%d" % k
    return json.dumps(d, separators=(",", ":")).encode()


def report(drv, rb):
    run = D.AuditRun(drv, violations_limit=20)
    run.add_batch_ordered(rb, AUDIT)
    rep = run.report()
    run.close()
    for k in ("pairsEvaluated", "pairsCounted"):
        rep.pop(k, None)
    return json.dumps(rep, sort_keys=True)


def timed(f):
    t0 = time.perf_counter()
    out = f()
    return out, (time.perf_counter() - t0) * 1e3


def probe(config, n, reps):
    tm, cons = W.config2() if config == 2 else W.config4()
    drv = D.Driver()
    for k, r in tm:
        drv.add_template(k, r)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    page = W.synth_objects(0, n, mode=0 if config == 2 else 1)
    docs = [page.get(i) for i in range(n)]
    warm = drv.upload_blob(page, keep_source=True)     # (the generated kernel and the front buffers made outside the timings)
    warm.eval(AUDIT, flags=D.F_NO_COPY_BACK)
    warm.free()
    rnd = random.Random(config)
    summary = {}
    for share in SHARES:
        m = max(1, int(n * share))
        drop = sorted(rnd.sample(range(n), m))
        add = [new_version(docs[i], i) for i in drop]
        gone = set(drop)
        result = W.PyBlob([d for i, d in enumerate(docs) if i not in gone] + add)
        added = W.PyBlob(add)
        drv.pin_blob(result)
        drv.pin_blob(added)
        rows = []
        for rep in range(reps):
            kept = drv.upload_blob(page, keep_source=True)
            st, t_patch = timed(lambda: kept.patch(drop, added))
            fresh, t_upload = timed(lambda: drv.upload_blob(result))
            row = {"config": config, "objects": n, "share": share, "replaced": m, "rep": rep, "patch_ms": round(t_patch, 2),
                   "patch_device_ms": round(st["kernel_ms"], 2), "patch_h2d_bytes": st["h2d_bytes"], "upload_blob_ms": round(t_upload, 2),
                   "upload_h2d_bytes": fresh.stats["h2d_bytes"]}
            if rep == 0:
                a, b = kept.eval(AUDIT), fresh.eval(AUDIT)
                row["identical_planes"] = planes(a) == planes(b)
                row["identical_audit_report"] = report(drv, kept) == report(drv, fresh)
                row["violations"] = int(sum(a.totals))
                if not (row["identical_planes"] and row["identical_audit_report"]):
                    print(json.dumps(row))
                    sys.exit("the patched batch and the fresh upload differ")
            kept.free()
            fresh.free()
            rows.append(row)
            print(json.dumps(row), flush=True)
        drv.pin_blob(result, False)
        drv.pin_blob(added, False)
        med = lambda k: round(statistics.median(r[k] for r in rows), 2)
        summary[str(share)] = {"patch_ms": med("patch_ms"), "patch_device_ms": med("patch_device_ms"), "upload_blob_ms": med("upload_blob_ms")}
    print(json.dumps({"summary": {"config": config, "objects": n, "gpu": gpu_info(), "by_share": summary}}), flush=True)
    drv.close()


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    configs = [int(x) for x in sys.argv[3].split(",")] if len(sys.argv) > 3 else [2, 4]
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for config in configs:
        probe(config, n, reps)


if __name__ == "__main__":
    main()
