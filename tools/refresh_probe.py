#!/usr/bin/env python
"""What a constraint change costs a resident page: gk_batch_refresh of a page uploaded with GK_F_KEEP_SOURCE (re-extraction from the
token tape kept in HBM) against a fresh gk_batch_upload_blob of the same page, and the first gk_batch_eval after each.

    python tools/refresh_probe.py [objects] [reps]

The config-2 constraint set over `objects` synthetic Pods (default 1 000 000), page-locked.  Each rep adds one constraint (a new
K8sRequiredLabels), then times refresh -> first eval -> second eval, and fresh upload -> first eval.  The first eval after a
constraint change includes the one-off NVRTC compile of the generated kernel for the new set: the second eval gives the evaluation
alone, and their difference is reported as the compile.  Every rep checks that the refreshed batch and the fresh upload give
identical violation / error bitmaps and totals.  Device time (kernels + copies, every stream) comes from one extra rep run under
torch.profiler.  One JSON line per rep, then a summary line."""
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W

AUDIT = "audit.gatekeeper.sh"


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # (the numbers are still printed; the line says why the card is unnamed)
        return "unknown (%s)" % e


def planes(r):
    return r.viol_bits.tobytes(), r.err_bits.tobytes(), list(r.totals), list(r.err_totals), list(r.constraints)


def timed(f):
    t0 = time.perf_counter()
    out = f()
    return out, (time.perf_counter() - t0) * 1e3


def device_ms(f):
    """Sum of the device activity (kernels, copies, memsets) recorded while f() runs."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = f()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.events() if e.device_time_total and e.device_type.name == "CUDA")
    return out, us / 1e3


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 1_000_000
    reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    tm, cons = W.config2()
    drv = D.Driver()
    for k, r in tm:
        drv.add_template(k, r)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    page = W.synth_objects(0, n)
    drv.pin_blob(page)
    kept = drv.upload_blob(page, keep_source=True)
    kept.eval(AUDIT, flags=D.F_NO_COPY_BACK)        # (the generated kernel of the starting set compiled outside the timings)
    fresh = drv.upload_blob(page)                    # (the front buffers allocated outside the timings)
    fresh.free()
    print(json.dumps({"gpu": gpu_info(), "objects": n, "blob_bytes": page.total_bytes(), "constraints": len(cons)}))
    rows = []

    def rep(i, measure):
        drv.AddConstraint(W._constraint("K8sRequiredLabels", "probe-%d" % i, match=dict(W.POD), params={"labels": ["probe-label-%d" % i]}))
        st, t_refresh = measure(kept.refresh)
        assert st["rebuilt"]
        r1, t_eval1 = timed(lambda: kept.eval(AUDIT))
        r2, t_eval2 = timed(lambda: kept.eval(AUDIT))
        nb, t_upload = measure(lambda: drv.upload_blob(page))
        r3, t_eval3 = timed(lambda: nb.eval(AUDIT))
        same = planes(r1) == planes(r3) == planes(r2)
        nb.free()
        return {"rep": i, "refresh_ms": round(t_refresh, 2), "refresh_stats": {k: (round(v, 3) if isinstance(v, float) else v) for k, v in st.items()},
                "first_eval_after_refresh_ms": round(t_eval1, 2), "eval_ms": round(t_eval2, 2), "nvrtc_compile_ms": round(t_eval1 - t_eval2, 1),
                "upload_blob_ms": round(t_upload, 2), "first_eval_after_upload_ms": round(t_eval3, 2), "identical_outputs": same,
                "violations": int(sum(r1.totals))}

    for i in range(reps):
        row = rep(i, timed)
        rows.append(row)
        print(json.dumps(row))
        if not row["identical_outputs"]:
            sys.exit("refreshed batch and fresh upload differ")
    prof = rep(reps, device_ms)
    med = lambda k: round(statistics.median(r[k] for r in rows), 2)
    print(json.dumps({"summary": {"refresh_ms": med("refresh_ms"), "upload_blob_ms": med("upload_blob_ms"), "eval_ms": med("eval_ms"),
                                  "first_eval_after_refresh_ms": med("first_eval_after_refresh_ms"), "nvrtc_compile_ms": med("nvrtc_compile_ms"),
                                  "refresh_device_ms": round(prof["refresh_ms"], 2), "upload_blob_device_ms": round(prof["upload_blob_ms"], 2)},
                      "identical_outputs": all(r["identical_outputs"] for r in rows) and prof["identical_outputs"]}))
    kept.free()
    drv.close()


if __name__ == "__main__":
    main()
