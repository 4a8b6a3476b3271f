"""GPU-only paths of the evaluation kernels: the generated kernel's launch wrapper at every bitmap width and on the mask registers'
row edge, the entry points that write into caller-owned device memory (one rank's buffers, and the fused exchange into its peers'),
the matcher-error list past its first capacity, and the fall-back to the interpreter when a tile's staging area does not fit.
Run on an H100:  python -m pytest tests/test_gpu_paths.py -m gpu -q"""
import json
import random

import numpy as np
import pytest

import gpu_path_cases as P
from conftest import assert_same, has_cuda, make_pair
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from gatekeeper_b200.sweep import shard_range
from oracle import k8s

pytestmark = pytest.mark.gpu
LIB = None   # the product library, gatekeeper_b200/libgk_engine.so
KERNELS = {"interpreter": ({"GK_SPEC": "0"}, "gk_eval_kernel"), "generated": ({"GK_SPEC_MIN_OBJECTS": "0"}, "gk_spec_kernel")}


@pytest.fixture(scope="module", autouse=True)
def _needs_gpu():
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    d = D.Driver()
    assert d.backend() == "cuda-sm90a"
    d.close()


def _driver(monkeypatch, env, tm, cons, nss=()):
    """A driver whose backend was built with `env` (the backend reads the GK_SPEC* switches when it is constructed)."""
    for k in ("GK_SPEC", "GK_SPEC_MIN_OBJECTS", "GK_SPEC_CHECK"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    drv = D.Driver(lib_path=LIB)
    for k, r in tm:
        drv.add_template(k, r)
    for c in cons:
        drv.AddConstraint(c)
    for ns in nss:
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    return drv


# ---- A: the generated kernel at every bitmap width (W = 1, 1, 1, 2, 2, 3, 7) and on the 32/33-row edge, against the interpreter and the oracle
@pytest.mark.parametrize("C", [1, 31, 32, 33, 64, 65, 200])
def test_generated_kernel_at_every_bitmap_width_and_row_edge(C, monkeypatch):
    assert P.case_spec_widths(LIB, monkeypatch, C) > 0


# ---- B: gk_batch_eval_device and gk_batch_eval_device_peers into torch tensors on a side stream
@pytest.mark.parametrize("kernel", ["interpreter", "generated"])
@pytest.mark.parametrize("C", [32, 64, 200])
def test_device_outputs_and_the_fused_exchange(C, kernel, monkeypatch):
    """eval_device into one rank's buffers, and eval_device_peers from three ranks' shards into three "peer" buffers of this GPU (the
    slot layout of ShardedSweep).  Buffers start as 0xff bytes, so a word a kernel fails to store shows.  Shards 0 and 1 hold 33-row
    objects: behind the generated kernel the interpreter then evaluates their tiles in list mode and, as the last CTA, publishes the
    totals of both kernels to every peer; shard 2 has none, so its interpreter launch evaluates no tile and publishes only."""
    import torch
    env, kname = KERNELS[kernel]
    tm, cons, _ = P.width_constraints(C)
    nss = W.synth_namespaces()
    world, n_local = 3, 700
    n = world * n_local
    docs, plan = P.row_edge_page(n, 512, (1,))
    assert {i // n_local for i, (_, k) in plan.items() if k == 33} == {0, 1}
    drv = _driver(monkeypatch, env, tm, cons, nss)
    words = (C + 31) // 32
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    keep = []

    def upload(lo, hi):
        blob = W.PyBlob(docs[lo:hi])
        rb = drv.upload_blob(blob)
        keep.append((blob, rb))
        return rb

    whole = upload(0, n)
    for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP):
        viol = torch.full((n, words), -1, dtype=torch.int32, device=dev)
        err = torch.full((n, words), -1, dtype=torch.int32, device=dev)
        tot = torch.full((2, C), -1, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        whole.eval_device(ep, viol.data_ptr(), err.data_ptr(), tot[0].data_ptr(), tot[1].data_ptr(), side.cuda_stream)
        assert drv.last_kernel() == kname
        side.synchronize()
        ref = whole.eval(ep)
        assert np.array_equal(viol.cpu().numpy().view(np.uint32), ref.viol_bits), ep
        assert np.array_equal(err.cpu().numpy().view(np.uint32), ref.err_bits), ep
        assert tot[0].tolist() == ref.totals and tot[1].tolist() == ref.err_totals, ep
    ref = whole.eval(k8s.AUDIT_EP)
    assert sum(ref.totals) > 0

    # the fused exchange: every rank writes its shard and totals into every peer's buffer at its own slot
    tot_off = n_local * words + (n_local * words) % 2
    slot = tot_off + 4 * C
    recv = [torch.full((world * slot,), -1, dtype=torch.int32, device=dev) for _ in range(world)]
    bases = [r.data_ptr() for r in recv]
    shard_out = []
    for rank in range(world):
        lo, hi = shard_range(n, rank, world)
        assert hi - lo == n_local
        rb = upload(lo, hi)
        err = torch.full((n_local, words), -1, dtype=torch.int32, device=dev)
        tot = torch.full((2, C), -1, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        rb.eval_device_peers(k8s.AUDIT_EP, bases, rank, slot, tot_off, C, err.data_ptr(), tot[0].data_ptr(), tot[1].data_ptr(), side.cuda_stream)
        assert drv.last_kernel() == kname
        shard_out.append((lo, hi, err, tot))
    side.synchronize()
    for r in recv:
        g = r.view(world, slot)
        bitmap = g[:, :n_local * words].reshape(n, words).cpu().numpy().view(np.uint32)
        assert np.array_equal(bitmap, ref.viol_bits)
        totals = g[:, tot_off:].contiguous().view(torch.int64).view(world, 2, C)
        assert totals.sum(0)[0].tolist() == ref.totals and totals.sum(0)[1].tolist() == ref.err_totals
    for rank, (lo, hi, err, tot) in enumerate(shard_out):
        assert np.array_equal(err.cpu().numpy().view(np.uint32), ref.err_bits[lo:hi]), rank
        got = recv[0].view(world, slot)[rank, tot_off:].contiguous().view(torch.int64).view(2, C)
        assert torch.equal(got.cpu(), tot.cpu()), rank   # what the last CTA published == what this rank's launch summed
        col = (ref.viol_bits[lo:hi, np.arange(C) // 32] >> (np.arange(C) % 32).astype(np.uint32)) & np.uint32(1)
        assert tot[0].tolist() == col.sum(0).tolist(), rank
    for _, rb in keep:
        rb.free()
    drv.close()


# ---- C: more matcher errors than the device list first holds
def test_matcher_errors_past_the_first_list_capacity_keep_their_reason(monkeypatch):
    assert P.case_matcher_error_list(LIB, monkeypatch) > 1 << 20


# ---- D: a page whose staging area exceeds the shared memory of a CTA runs on the interpreter
def test_staging_area_beyond_shared_memory_runs_the_interpreter(monkeypatch):
    """The generated kernel stages a tile's rows at 32 bits per row of a scope with atoms; the interpreter holds one bit per row per
    live slot.  One constraint with one atom over Pods of 128 containers: 512 x 128 rows make 256 KiB of staging, more than a CTA may
    have, while the interpreter's tile fits.  The same constraint set over narrow Pods runs the generated kernel."""
    t = W.templates()["psp_privileged"]
    tm, cons = [(t["kind"], t["rego"])], [W._constraint(t["kind"], "priv", match=dict(W.POD))]
    orc, _, _ = make_pair(tm, cons, lib_path=LIB)
    drv = _driver(monkeypatch, KERNELS["generated"][0], tm, cons)

    def page(n, rows):
        docs = []
        for i in range(n):
            cs = [P._row("containers", j) for j in range(rows)]
            if i % 3:   # privileged containers in every third Pod only
                for c in cs:
                    c.pop("securityContext", None)
            docs.append(json.dumps({"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "p-%d" % i, "namespace": "default"},
                                    "spec": {"containers": cs}}).encode())
        return docs

    narrow = W.PyBlob(page(600, 3))
    rb = drv.upload_blob(narrow)
    rb.eval(k8s.AUDIT_EP)
    assert drv.last_kernel() == "gk_spec_kernel"
    rb.free()
    docs = page(600, 128)
    wide = W.PyBlob(docs)
    rb = drv.upload_blob(wide)
    r = rb.eval(k8s.AUDIT_EP)
    assert drv.last_kernel() == "gk_eval_kernel"
    objs = sorted(set(random.Random(3).sample(range(600), 30)) | {0, 511, 512, 599})
    viol, err = P.oracle_pairs(orc, docs, objs, k8s.AUDIT_EP)
    assert viol and not err
    assert_same(viol, P.bit_pairs(r.viol_bits, r.constraints, objs))
    assert r.totals[0] == int(np.count_nonzero(r.viol_bits[:, 0] & 1)) > 0
    rb.free()
    drv.close()
