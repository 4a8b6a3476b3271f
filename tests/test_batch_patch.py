"""gk_batch_patch on the GPU: the shared cases (batch_patch_cases.py) on the product library, a page large enough for the generated
kernel, and the launch trace of a patch: the tokeniser runs over the added documents only, and the staying objects' tape is moved by
gk_splice_kernel -- the results equal a fresh upload only if the moved tape is right where it lands."""
import pytest

import batch_patch_cases as P
import batch_refresh_cases as R
from gatekeeper_b200 import workloads as W
from oracle import k8s

pytestmark = pytest.mark.gpu


def test_patch_page_for_the_generated_kernel():
    P.case_replace_share(None, n=8500, share=0.01, oracle=False, kernel="gk_spec_kernel")


@pytest.mark.parametrize("process", ["audit", ""])
def test_patch_small_page_for_the_interpreter(process):
    P.case_replace_share(None, process=process, kernel="gk_eval_kernel")


def test_patch_mixed_kinds():
    P.case_mixed_kinds(None)


def test_patch_sequence():
    P.case_sequence(None)


def test_patch_edges():
    P.case_edges(None)


def test_patch_after_a_constraint_change():
    P.case_constraint_between(None)


def test_patch_expanded_batch():
    P.case_expanded(None)


def test_patch_invalid_calls():
    P.case_invalid(None)


def test_patch_refused_while_the_set_is_flattened_on_the_host():
    P.case_host_flattened(None)


def test_patch_tokenises_only_the_added_objects(monkeypatch, capfd):
    eng, _ = R.config2_start(None)
    docs = R.damaged_page(3000, start=99900)
    rb = eng.drv.upload_blob(W.PyBlob(docs), keep_source=True)
    capfd.readouterr()
    monkeypatch.setenv("GK_TRACE_LAUNCH", "1")
    drop = list(range(0, 3000, 97))
    add = [P.renamed(docs[i], i) for i in drop] + [docs[5]]
    docs = P.patch(rb, docs, drop, add)
    trace = capfd.readouterr().err
    monkeypatch.delenv("GK_TRACE_LAUNCH")
    tape = [l for l in trace.splitlines() if "gk_tape_kernel" in l]
    assert len(tape) == 1 and "gk_tape_kernel over %d objects," % len(add) in tape[0], trace
    assert "gk_splice_kernel over %d staying objects" % (3003 - len(drop)) in trace, trace
    P.check(eng, rb, docs, "", "the tape relocation", oracle=False)
    rb.eval(k8s.AUDIT_EP)
    rb.free()
    eng.close()
