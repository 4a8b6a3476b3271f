"""The hand-over plan on the GPU: gk_spec_plan_kernel lists the objects too wide for the mask registers before any row is evaluated,
and the interpreter evaluates them on a side stream while gk_spec_rows_kernel and gk_spec_kernel do the rest of the page.  Forced
through the generated kernel, every page must give the interpreter's bitmaps and totals at both enforcement points, evaluation after
evaluation, hand over what the rule says, and in the fused exchange publish the totals of both kernels once.
Run on an H100:  python -m pytest tests/test_spec_plan_gpu.py -m gpu -q"""
import re

import numpy as np
import pytest

from conftest import has_cuda
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import k8s

from test_spec_plan_hostemu import CASES, constraint_set, expected_plan, page

pytestmark = pytest.mark.gpu
HANDED = re.compile(r"handed to the interpreter: (\d+) units \((\d+) of more than one object\), (\d+) objects")


@pytest.fixture(scope="module", autouse=True)
def _needs_gpu():
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")


def driver(monkeypatch, env):
    for k in ("GK_SPEC", "GK_SPEC_MIN_OBJECTS", "GK_SPEC_CHECK", "GK_TRACE_LAUNCH"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    drv = D.Driver()
    tm, cons = constraint_set()
    for k, r in tm:
        drv.add_template(k, r)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    return drv


def results(r):
    return np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True), list(r.totals), list(r.err_totals)


def same(a, b):
    return all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(a, b))


@pytest.mark.parametrize("case", sorted(CASES))
def test_plan_beside_the_generated_kernel(case, monkeypatch, capfd):
    n, wide = CASES[case]
    docs = page(n, wide, ns_missing={i + 1 for i in sorted(wide)[:2]})
    drv = driver(monkeypatch, {"GK_SPEC": "0"})
    rb = drv.upload_blob(W.PyBlob(docs))
    want = {ep: results(rb.eval(ep)) for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP)}
    assert drv.last_kernel() == "gk_eval_kernel"
    rb.free()
    drv.close()

    drv = driver(monkeypatch, {"GK_SPEC_MIN_OBJECTS": "0", "GK_TRACE_LAUNCH": "1"})
    rb = drv.upload_blob(W.PyBlob(docs))
    capfd.readouterr()
    for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP):
        for k in range(3):   # the two streams overlap differently every time; the results may not
            got = results(rb.eval(ep))
            assert drv.last_kernel() == "gk_spec_kernel"
            assert same(want[ep], got), "%s, evaluation %d: the generated kernel and the plan's units differ from the interpreter" % (ep, k)
    rb.free()
    drv.close()
    units, whole = expected_plan(n, wide)
    handed = HANDED.findall(capfd.readouterr().err)
    assert len(handed) == 6 and set(handed) == {(str(len(units)), str(len(whole)), str(sum(u[1] for u in units)))}, handed
    if case == "edges":
        assert want[k8s.AUDIT_EP][3][-1] >= 2, "the unknown Namespace's objects are not matcher errors"


def test_fused_exchange_publishes_the_totals_of_both_kernels(monkeypatch):
    """eval_device_peers of one rank whose only peer buffer is its own: the bitmap and both totals arrive, whichever of the two
    kernels finishes last.  The buffer starts as 0xff bytes, so a word nobody stores shows."""
    import torch
    n, wide = CASES["edges"]
    docs = page(n, wide)
    drv = driver(monkeypatch, {"GK_SPEC_MIN_OBJECTS": "0"})
    rb = drv.upload_blob(W.PyBlob(docs))
    ref = rb.eval(k8s.AUDIT_EP)
    C, words = len(ref.totals), ref.viol_bits.shape[1]
    assert sum(ref.totals) > 0
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    tot_off = n * words + (n * words) % 2
    slot = tot_off + 4 * C
    for _ in range(3):
        recv = torch.full((slot,), -1, dtype=torch.int32, device=dev)
        err = torch.full((n, words), -1, dtype=torch.int32, device=dev)
        tot = torch.full((2, C), -1, dtype=torch.int64, device=dev)
        torch.cuda.synchronize()
        rb.eval_device_peers(k8s.AUDIT_EP, [recv.data_ptr()], 0, slot, tot_off, C, err.data_ptr(), tot[0].data_ptr(), tot[1].data_ptr(), side.cuda_stream)
        assert drv.last_kernel() == "gk_spec_kernel"
        side.synchronize()
        assert np.array_equal(recv[:n * words].view(n, words).cpu().numpy().view(np.uint32), ref.viol_bits)
        assert np.array_equal(err.cpu().numpy().view(np.uint32), ref.err_bits)
        published = recv[tot_off:].contiguous().view(torch.int64).view(2, C)
        assert published[0].tolist() == ref.totals and published[1].tolist() == ref.err_totals
        assert tot[0].tolist() == ref.totals and tot[1].tolist() == ref.err_totals
    rb.free()
    drv.close()
