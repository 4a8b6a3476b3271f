"""gk_batch_refresh on the GPU: the shared cases (batch_refresh_cases.py) on the product library, the refusal of a refresh that
cannot be laid out in tiles, the device memory of upload -> refresh -> free cycles, the generated kernel on a refreshed page, and
the launch trace of a refresh from the kept source."""
import json

import numpy as np
import pytest

import batch_refresh_cases as R
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import k8s

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind,keep,process", [("blob", True, "audit"), ("blob", False, "audit"), ("objs", False, "audit"), ("blob", True, "")])
def test_refresh_after_every_kind_of_change(kind, keep, process):
    R.case_refresh_steps(None, kind=kind, keep=keep, process=process)


@pytest.mark.parametrize("keep", [True, False])
def test_refresh_referential(keep):
    R.case_refresh_referential(None, keep=keep)


def test_refresh_with_prefetch():
    R.case_refresh_with_prefetch(None)


def test_failed_refresh_leaves_the_batch_as_it_was():
    R.case_refresh_failure_leaves_batch(None)


def test_refresh_cycles_free_their_device_memory(monkeypatch):
    """20 upload (keeping the source) -> refresh -> free cycles of a 20 000-object page: the device's free memory comes back to
    where it was after the first cycles, which leave the backend's pooled scratch and front buffers allocated.  (One leaked kept
    source of this page is about 60 MB.)  The interpreter evaluates: every cycle is a new constraint set, and the generated kernel
    would be compiled for each."""
    import torch
    monkeypatch.setenv("GK_SPEC", "0")
    eng, _ = R.config2_start(None)
    page = W.synth_objects(90000, 20000)

    def cycle(i):
        rb = eng.drv.upload_blob(page, keep_source=True)
        eng.drv.AddConstraint(W._constraint("K8sRequiredLabels", "cycle-%d" % i, match=dict(W.POD), params={"labels": ["cycle-%d" % i]}))
        assert rb.refresh()["rebuilt"]
        rb.eval(k8s.AUDIT_EP)
        rb.free()
        eng.drv.RemoveConstraint({"kind": "K8sRequiredLabels", "metadata": {"name": "cycle-%d" % i}})

    for i in range(3):
        cycle(i)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for i in range(3, 23):
        cycle(i)
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    assert free1 >= free0 - (64 << 20), "device memory lost over 20 refresh cycles: %d MB" % ((free0 - free1) >> 20)
    eng.close()


def test_kept_source_refresh_of_a_large_page_runs_the_generated_kernel(capfd, monkeypatch):
    """A kept-source refresh of 8 500 config-2 Pods: no tokeniser launch and no copy of the page in the launch trace, the generated
    kernel evaluates the refreshed batch, and its results are a fresh upload's."""
    tm, cons = W.config2()
    drv = D.Driver()
    for k, r in tm[:6]:
        drv.add_template(k, r)
    for c in cons[:30]:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData(R.T, ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    page = W.synth_objects(100000, 8500)
    monkeypatch.setenv("GK_TRACE_LAUNCH", "1")
    rb = drv.upload_blob(page, keep_source=True)
    assert "gk_tape_kernel" in capfd.readouterr().err
    for k, r in tm[6:]:
        drv.add_template(k, r)
    for c in cons[30:]:
        drv.AddConstraint(c)
    st = rb.refresh()
    trace = capfd.readouterr().err
    assert st["rebuilt"] and "gk_tape_kernel" not in trace and "from the kept source: no copy, no tokeniser" in trace, trace
    assert st["h2d_bytes"] < page.total_bytes() // 8, st
    got = R.snapshot(rb.eval(k8s.AUDIT_EP))
    assert drv.last_kernel() == "gk_spec_kernel"
    fresh = drv.upload_blob(page)
    want = R.snapshot(fresh.eval(k8s.AUDIT_EP))
    assert drv.last_kernel() == "gk_spec_kernel"
    R.assert_same_as_fresh(got, want, "the constraint set completed to config 2")
    assert len(got[0]) == len(cons) and sum(got[3]) > 0
    fresh.free()
    rb.free()
    drv.close()
