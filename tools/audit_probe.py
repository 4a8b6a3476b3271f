#!/usr/bin/env python
"""What the audit's device-side candidate selection buys: gk_audit_add_batch (host threshold scan over (namespace, name), uniform pages
only) against gk_audit_add_batch_ordered (identities ranked and candidates selected on the GPU, any mix of kinds), and the sharded
audit's export / exchange / merge.

    python tools/audit_probe.py [--objects 1000000] [--reps 3] [--limit 20]
    python -m torch.distributed.run --nproc_per_node 2 tools/audit_probe.py --dist [--objects 1000000] [--limit 20]

Single-process mode: a config-2 page (Pods only) and a config-4 page (synth mode 1: mixed kinds), `--objects` objects each, one resident raw-JSON
batch per page.  Each rep folds the batch into a fresh run with each call, alternating, and prints one JSON line: wall time of each
call, its pairsEvaluated / pairsCounted, and the device time of the ranking and selection kernels (CUDA events).  Every rep checks
that both reports are equal except for the pair counters.

--dist: every rank folds its shard (sweep.shard_range) of the config-4 page with sweep.ShardedAudit, exchanges the exports over the
default process group (gloo) and merges them; rank 0 also runs one process over the whole page and checks that every rank's report
equals it.  Prints the export / exchange / merge times."""
import argparse
import hashlib
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
PAIRS = ("pairsEvaluated", "pairsCounted")


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # (the numbers are still printed; the line says why the card is unnamed)
        return "unknown (%s)" % e


def strip(rep):
    return {k: v for k, v in rep.items() if k not in PAIRS}


def engine(config):
    tm, cons = W.config2() if config == 2 else W.config4()
    drv = D.Driver()
    for k, r in tm:
        drv.add_template(k, r)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    return drv


def fold(drv, rb, limit, ordered):
    run = D.AuditRun(drv, violations_limit=limit)
    t0 = time.perf_counter()
    (run.add_batch_ordered if ordered else run.add_batch)(rb, AUDIT)
    ms = (time.perf_counter() - t0) * 1e3
    rep = run.report()
    sel = run.select_ms()
    run.close()
    return rep, ms, sel


def single(args):
    for config, mode in ((2, 0), (4, 1)):
        drv = engine(config)
        blob = W.synth_objects(0, args.objects, mode=mode)
        drv.pin_blob(blob)
        rb = drv.upload_blob(blob)
        fold(drv, rb, args.limit, False)      # warm-up: the generated kernel's compile, first-touch allocations
        fold(drv, rb, args.limit, True)
        rows = []
        for rep_i in range(args.reps):
            order = (False, True) if rep_i % 2 == 0 else (True, False)
            got = {}
            for ordered in order:
                got[ordered] = fold(drv, rb, args.limit, ordered)
            (ra, ma, _), (ro, mo, so) = got[False], got[True]
            assert strip(ra) == strip(ro), "add_batch and add_batch_ordered reports differ"
            row = {"config": config, "objects": args.objects, "limit": args.limit, "rep": rep_i,
                   "add_batch_ms": round(ma, 2), "add_batch_pairs": [ra[k] for k in PAIRS],
                   "ordered_ms": round(mo, 2), "ordered_pairs": [ro[k] for k in PAIRS], "select_device_ms": round(so, 3),
                   "violations": sum(ra["totalViolations"].values())}
            rows.append(row)
            print(json.dumps(row), flush=True)
        print(json.dumps({"config": config, "summary": True, "gpu": gpu_info(),
                          "add_batch_ms_median": statistics.median(r["add_batch_ms"] for r in rows),
                          "ordered_ms_median": statistics.median(r["ordered_ms"] for r in rows),
                          "select_device_ms_median": statistics.median(r["select_device_ms"] for r in rows)}), flush=True)
        rb.free()
        drv.pin_blob(blob, False)
        drv.close()


def distributed(args):
    import torch
    import torch.distributed as dist
    from gatekeeper_b200.sweep import ShardedAudit, shard_range
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    drv = engine(4)
    lo, hi = shard_range(args.objects, rank, world)
    blob = W.synth_objects(lo, hi - lo, mode=1)
    rb = drv.upload_blob(blob)
    sa = ShardedAudit(drv, violations_limit=args.limit)
    t0 = time.perf_counter()
    sa.add_batch(rb, AUDIT)
    fold_ms = (time.perf_counter() - t0) * 1e3
    dist.barrier()
    rep = sa.exchange()
    digest = hashlib.sha256(json.dumps(strip(rep), sort_keys=True).encode()).digest()
    mine = torch.frombuffer(bytearray(digest), dtype=torch.uint8)
    all_d = [torch.zeros(32, dtype=torch.uint8) for _ in range(world)]
    dist.all_gather(all_d, mine)
    same_on_ranks = all(bytes(d.numpy()) == digest for d in all_d)
    row = {"rank": rank, "world": world, "objects": args.objects, "fold_ms": round(fold_ms, 2), **{k: round(v, 3) for k, v in sa.timing.items()},
           "same_on_every_rank": same_on_ranks}
    if rank == 0:
        whole = W.synth_objects(0, args.objects, mode=1)
        wb = drv.upload_blob(whole)
        ref, _, _ = fold(drv, wb, args.limit, True)
        row["equals_single_process"] = strip(ref) == strip(rep)
        row["gpu"] = gpu_info()
    print(json.dumps(row), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    ok = same_on_ranks and row.get("equals_single_process", True)
    sys.exit(0 if ok else 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--objects", type=int, default=1000000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--limit", type=int, default=20)
    ap.add_argument("--dist", action="store_true")
    args = ap.parse_args()
    distributed(args) if args.dist else single(args)


if __name__ == "__main__":
    main()
