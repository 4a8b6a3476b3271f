#!/usr/bin/env python
"""What expanding a sweep page costs (GK_F_EXPAND) on one GPU, with the card's name and power limit read in the same run.

    python tools/expand_probe.py [objects] [reps]

(1) The config-4 page (synthetic objects of mixed kinds, default 1 000 000) with the "expand-deployments" ExpansionTemplate: the
upload's generator selection (device time), host expansion and resultant upload (from the [expand] launch-trace line); the device time
of one evaluation of the expanded batch (parents, resultants, fold) against the same page as a plain batch on an engine without
templates, alternated rep by rep; the wall time of gk_review_batch over the page, which was the only way to expand it before.  The
expanded evaluation's planes must equal gk_review_batch's, its totals their popcounts.
(2) The config-2 page (synthetic Pods) with the template registered and the flag set, against the plain batch: no generators, so no
difference is expected beyond the spread.  The planes must be identical.
One JSON line per measurement, then a summary line."""
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

import expand_sweep_cases as X   # noqa: E402
from refresh_probe import gpu_info   # noqa: E402

AUDIT = "audit.gatekeeper.sh"
EXPAND_DEPLOYMENTS = X.T._expansion_template("expand-deployments", ["Deployment"], ("", "v1", "Pod"))


def engine(config, lib=None):
    tm, cons = config()
    drv = D.Driver(lib_path=lib)
    for k, rego in tm:
        drv.add_template(k, rego)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData(X.T.T, ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    return drv


def compare(name, config, mode, n, reps, lib=None, review=False):
    blob = W.synth_objects(0, n, mode=mode)
    plain_drv, x_drv = engine(config, lib), engine(config, lib)
    x_drv.AddExpansionTemplate(EXPAND_DEPLOYMENTS)
    plain = plain_drv.upload_blob(blob)
    t0 = time.perf_counter()
    with X.launch_trace() as lines:
        xb = x_drv.upload_blob(blob, expand=True)
    up_ms = (time.perf_counter() - t0) * 1e3
    trace = [l for l in lines if l.startswith("[expand]")]
    print(json.dumps({"page": name, "objects": n, "expanded_upload_ms": round(up_ms, 1), "plain_upload_h2d_ms": plain.stats["h2d_ms"], "trace": trace}))
    got = xb.eval(AUDIT)
    C = len(got.totals)
    assert list(got.totals) == X.popcounts(got.viol_bits, C) and list(got.err_totals) == X.popcounts(got.err_bits, C), "totals are not the popcounts"
    base = plain.eval(AUDIT)
    for _ in range(3):   # warm-up of both shapes (module loads, the generated kernel's compile)
        plain.eval(AUDIT, flags=D.F_NO_COPY_BACK), xb.eval(AUDIT, flags=D.F_NO_COPY_BACK)
    tp, tx = [], []
    for _ in range(reps):   # alternated
        tp.append(plain.eval(AUDIT, flags=D.F_NO_COPY_BACK).stats["kernel_ms"])
        tx.append(xb.eval(AUDIT, flags=D.F_NO_COPY_BACK).stats["kernel_ms"])
    out = {"page": name, "objects": n, "plain_kernel_ms_median": round(statistics.median(tp), 4), "plain_kernel_ms_min": round(min(tp), 4),
           "plain_kernel_ms_max": round(max(tp), 4), "expanded_kernel_ms_median": round(statistics.median(tx), 4),
           "expanded_kernel_ms_min": round(min(tx), 4), "expanded_kernel_ms_max": round(max(tx), 4), "reps": reps}
    if review:
        revs = [D.Review(object=json.loads(blob.get(i)), source="Original") for i in range(n)]
        t0 = time.perf_counter()
        want = x_drv.ReviewBatch(revs, AUDIT, materialize=False)
        out["review_batch_wall_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
        out["identical_to_review_batch"] = bool((got.viol_bits == want.viol_bits).all() and (got.err_bits == want.err_bits).all())
        assert out["identical_to_review_batch"], "the expanded batch's planes differ from gk_review_batch's"
    else:
        out["identical_to_plain"] = bool((got.viol_bits == base.viol_bits).all() and (got.err_bits == base.err_bits).all()
                                         and got.totals == base.totals)
        assert out["identical_to_plain"], "a page without generators must give the plain batch's outputs"
    print(json.dumps(out))
    xb.free(), plain.free()
    x_drv.close(), plain_drv.close()
    return out


def main(n=1000000, reps=20, lib=None):
    gpu = gpu_info()
    print(json.dumps({"gpu": gpu}))
    a = compare("config-4 + expand-deployments", W.config4, 1, n, reps, lib, review=True)
    b = compare("config-2, template registered, no generators", W.config2, 0, n, reps, lib)
    print(json.dumps({"summary": True, "gpu": gpu, "config4": a, "config2": b}))


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 1000000, int(sys.argv[2]) if len(sys.argv) > 2 else 20)
