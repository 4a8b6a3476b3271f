#!/usr/bin/env python
"""What auditing an expanded page costs (gk_audit_add_batch_ordered), with the card's name and power limit read in the same run.

    python tools/audit_expand_probe.py [objects] [reps] [limit]

The config-4 page (synthetic objects of mixed kinds, default 1 000 000) with the "expand-deployments" ExpansionTemplate, uploaded
twice on one engine: with GK_F_EXPAND (the audit takes the resultants from the batch) and without it (the audit expands the page on
the host, uploads the resultants and renders all their pairs).  Alternated reps of one audit run each; every rep checks that the two
reports are byte-identical and reports the wall time of the call, the device time of the ranking, selection and resultant sorting
(gk_audit_select_ms), and the resultant pairs rendered / counted.  One JSON line per rep, then a summary line."""
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gatekeeper_b200 import driver as D   # noqa: E402
from gatekeeper_b200 import workloads as W   # noqa: E402

import audit_expand_cases as A   # noqa: E402
from expand_probe import EXPAND_DEPLOYMENTS, engine   # noqa: E402
from refresh_probe import gpu_info   # noqa: E402


def one(drv, rb, limit):
    run = D.AuditRun(drv, violations_limit=limit)
    t0 = time.perf_counter()
    run.add_batch_ordered(rb, A.EP)
    wall = (time.perf_counter() - t0) * 1e3
    out = A.raw_report(run), wall, run.select_ms(), run.resultant_pairs()
    run.close()
    return out


def main(n=1000000, reps=5, limit=20, lib=None):
    gpu = gpu_info()
    print(json.dumps({"gpu": gpu}))
    drv = engine(W.config4, lib)
    drv.AddExpansionTemplate(EXPAND_DEPLOYMENTS)
    blob = W.synth_objects(0, n, mode=1)
    xb = drv.upload_blob(blob, expand=True)
    pb = drv.upload_blob(blob)
    one(drv, xb, limit), one(drv, pb, limit)   # warm-up of both shapes (module loads, the generated kernel's compile)
    rows = {"expanded": [], "plain": []}
    for rep in range(reps):   # alternated
        rx, wx, sx, px = one(drv, xb, limit)
        rp, wp, sp, pp = one(drv, pb, limit)
        assert rx == rp, "the expanded batch's audit report differs from the plain batch's"
        rows["expanded"].append(wx)
        rows["plain"].append(wp)
        print(json.dumps({"rep": rep, "objects": n, "limit": limit, "identical": True, "expanded_wall_ms": round(wx, 1), "plain_wall_ms": round(wp, 1),
                          "expanded_select_classify_ms": round(sx, 3), "plain_select_ms": round(sp, 3), "resultant_pairs_rendered": px[0],
                          "resultant_pairs_counted": px[1]}))
    rep = json.loads(rx)
    summary = {"summary": True, "gpu": gpu, "objects": n, "limit": limit, "reps": reps, "results": rep["results"],
               "pairsEvaluated": rep["pairsEvaluated"], "pairsCounted": rep["pairsCounted"], "resultant_pairs_rendered": px[0],
               "resultant_pairs_counted": px[1]}
    for k, v in rows.items():
        summary[k + "_wall_ms_median"] = round(statistics.median(v), 1)
        summary[k + "_wall_ms_min"] = round(min(v), 1)
        summary[k + "_wall_ms_max"] = round(max(v), 1)
    print(json.dumps(summary))
    xb.free(), pb.free()
    drv.close()
    return summary


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:4]))
