"""The sharded audit on CPU: two `gloo` ranks fold their shard of a mixed-kind page into a run (add_batch_ordered, test-only CPU
backend), exchange the exports and merge them in rank order; both ranks must hold the single-process report."""
import json
import os
import socket
import sys

import pytest
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import HOSTEMU, ROOT

N_TOTAL = 500
LIMIT = 5


def _setup():
    import audit_order_cases as A
    orc, drv, nss = A.mixed_engine(HOSTEMU)
    objs = A.mixed_objects(nss, n_extra=N_TOTAL, seed=21)
    return drv, objs


def _worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    import audit_order_cases as A
    from gatekeeper_b200 import driver as D
    from gatekeeper_b200.sweep import ShardedAudit, shard_range
    drv, objs = _setup()
    lo, hi = shard_range(len(objs), rank, world)
    sa = ShardedAudit(drv, violations_limit=LIMIT)
    keep = A.upload(drv, objs[lo:hi], "blob", page=97)
    for _, rb in keep:
        sa.add_batch(rb, D.AUDIT_EP)
    rep = sa.exchange()
    with open(os.path.join(out_dir, "rank%d.json" % rank), "w") as f:
        json.dump(rep, f)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_gloo_audit_equals_single_process(tmp_path):
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mp.spawn(_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    import audit_order_cases as A
    from gatekeeper_b200 import driver as D
    drv, objs = _setup()
    run = D.AuditRun(drv, violations_limit=LIMIT)
    keep = A.upload(drv, objs, "blob")
    for _, rb in keep:
        run.add_batch_ordered(rb, D.AUDIT_EP)
    want = run.report()
    for r in range(2):
        with open(tmp_path / ("rank%d.json" % r)) as f:
            got = json.load(f)
        assert A.strip(got) == A.strip(want)
        assert got["pairsCounted"] > 0
