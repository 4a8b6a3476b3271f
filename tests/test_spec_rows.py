"""The generated kernel's two launches (spec_codegen.cpp): gk_spec_rows_kernel evaluates every row of the batch -- atoms, row-local
gates, and on an object's own row the spec.match blocks, listing their errors -- into export arrays in global memory, and
gk_spec_kernel copies each tile's slice of them into shared memory and walks the objects.  On the test-only host emulation the same
text (rows of the object's tile into a poisoned export buffer, the copy, the object walk) is compared object by object, and its
matcher-error list as a multiset, with the interpreted netlist (GK_SPEC_CHECK=1); the pairs are the oracle's.  On the GPU the two
kernels, forced at any page size, against the interpreter: bitmaps, totals and the autoreject results."""
import json

import numpy as np
import pytest

import gpu_path_cases as G
from conftest import HOSTEMU, make_pair
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import k8s

from test_spec_fold import POD, allowed_repos, check, container, pod, tmpl, traced

NEVER = "fixtures_TemplateNeverValidate"


def _nssel(i):
    return W._constraint(W.templates()[NEVER]["kind"], "nssel-%02d" % i, match={"namespaceSelector": {"matchLabels": {"sel-%02d" % i: "on"}}})


def _match_error_set():
    """Matcher errors from three kinds of block next to config 2: a namespaceSelector over Pods without a cached Namespace (missing
    namespace), an invalid labelSelector and an invalid source, plus a block that matches by kind."""
    tm, cons = W.config2()
    tm = tm + tmpl(NEVER)
    kind = W.templates()[NEVER]["kind"]
    cons = cons + [_nssel(0), _nssel(1),
                   W._constraint(kind, "bad-lsel", match={"labelSelector": {"matchExpressions": [{"key": "a", "operator": "Bogus", "values": ["x"]}]}}),
                   W._constraint(kind, "bad-source", match=dict(POD, source="Nowhere"))]
    return tm, cons


def _mixed_pods(n, start=0):
    """Pods with 0 to 4 containers, some in namespaces with no cached Namespace, every 11th not valid JSON."""
    docs = []
    for i in range(start, start + n):
        if i % 11 == 5:
            docs.append(b'{"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "broken-%d"' % i)
            continue
        o = pod(i, [container(i + j) for j in range(i % 5)])
        o["metadata"]["namespace"] = "ns-%d" % (i % 7)
        o["metadata"]["labels"] = {"app": "a%d" % (i % 3)}
        docs.append(json.dumps(o).encode())
    return docs


def _host_check(tm, cons, docs, monkeypatch, capfd, tmp_path, old=None):
    """Review `docs` on the host emulation with the generated text checked against the interpreted netlist (which raises on any
    difference, matcher-error list included); returns the number of objects too big for the mask registers and the response."""
    traced(monkeypatch, tmp_path)
    orc, drv, _ = make_pair(tm, cons, lib_path=HOSTEMU)
    capfd.readouterr()
    if old is None:
        resp = drv.ReviewBlob(W.PyBlob(docs), k8s.AUDIT_EP, flags=D.F_MATERIALIZE)
    else:
        revs = [D.Review(object=json.loads(d), old_object=json.loads(o), operation="UPDATE", source="Original") for d, o in zip(docs, old)]
        resp = drv.ReviewBatch(revs, k8s.WEBHOOK_EP)
    drv.close()
    lines = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("[spec check]")]
    assert lines, "no [spec check] line: was the generated text checked?"
    return int(lines[-1].split("(")[1].split()[0]), resp


def test_tiles_where_a_scope_has_no_rows(monkeypatch, capfd, tmp_path):
    """Whole tiles (of the host emulation's 96 objects) without any container or init container, between tiles that have them: the
    export slices of those scopes are empty and the rows kernel has nothing to write there."""
    objs = [pod(i, [] if (i // 96) % 2 == 0 else [container(i)], init=[container(i)] if i // 96 == 3 else ()) for i in range(96 * 5 + 7)]
    _, big = check(tmpl("allowedrepos"), [allowed_repos(0, ["gcr.io/"]), allowed_repos(1, ["quay.io/"])], objs, monkeypatch, capfd, tmp_path)
    assert big == 0


def test_object_with_more_than_32_rows_is_handed_over(monkeypatch, capfd, tmp_path):
    """An object with 40 containers in the middle of a tile: the tile kernel hands its tile to the interpreter; every other object of
    the page is the generated text's, identical to the interpreter's and the oracle's."""
    objs = [pod(i, [container(i + j) for j in range(40 if i == 150 else 1 + i % 3)]) for i in range(300)]
    _, big = check(tmpl("allowedrepos"), [allowed_repos(0, ["gcr.io/"]), allowed_repos(1, ["quay.io/"])], objs, monkeypatch, capfd, tmp_path)
    assert big == 1


def test_skipped_objects_and_matcher_errors_of_several_blocks(monkeypatch, capfd, tmp_path):
    """Objects that are not valid JSON evaluate no block and list no error; the others list matcher errors of a missing Namespace, an
    invalid label selector and an invalid source, as the interpreter does (compared as a multiset) and as the oracle does."""
    tm, cons = _match_error_set()
    docs = _mixed_pods(400)
    big, resp = _host_check(tm, cons, docs, monkeypatch, capfd, tmp_path)
    assert big == 0
    auto = [r for r in resp.results if r.autoreject]
    assert {r.constraint.split("/")[1] for r in auto} >= {"nssel-00", "nssel-01", "bad-lsel", "bad-source"}, sorted({r.constraint for r in auto})
    assert not any(r.object % 11 == 5 for r in resp.results), "a skipped object has results"
    assert resp.object_errors and all(resp.object_errors[i] for i in range(5, 400, 11))


def test_old_objects_above_the_threshold(monkeypatch, capfd, tmp_path):
    """UPDATE reviews carry an OldObject row per object: a match block that fails on the new object and not on the old one, and the
    reverse, are decided on the scope-0 row the rows kernel evaluates (errors of the old object carry its own code)."""
    tm, cons = _match_error_set()
    docs = _mixed_pods(300, start=1)
    docs = [d if not d.startswith(b'{"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "broken') else json.dumps(pod(9, [])).encode() for d in docs]
    old = []
    for i, d in enumerate(docs):
        o = json.loads(d)
        o["metadata"]["namespace"] = "" if i % 4 == 0 else "ns-%d" % (i % 5)
        o["metadata"]["labels"] = {"app": "old"}
        old.append(json.dumps(o).encode())
    big, resp = _host_check(tm, cons, docs, monkeypatch, capfd, tmp_path, old=old)
    assert big == 0 and any(r.autoreject for r in resp.results)


@pytest.mark.parametrize("extra", [14, 22])
def test_row_loop_with_more_than_32_exports(extra, monkeypatch, capfd, tmp_path):
    """A container row loop with two export words, next to the match blocks of config 2 on the object's row: both words are copied
    from the export array."""
    tm, cons = _match_error_set()
    cons = cons + [allowed_repos(100 + i, template="allowedrepos_prefixmatch") for i in range(extra)]
    big, _ = _host_check(tm, cons, _mixed_pods(200), monkeypatch, capfd, tmp_path)
    assert big == 0
    head = (tmp_path / "spec.cu").read_text().split("\n", 1)[0]
    assert " in 2 words" in head, head


def test_both_entry_points_compile_with_nvrtc(monkeypatch, tmp_path):
    """The text with the match blocks on the object's row: NVRTC (the backend's options) builds gk_spec_rows_kernel and gk_spec_kernel,
    and the object walk no longer calls a match block."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("spec_nvrtc", os.path.join(os.path.dirname(os.path.dirname(__file__)), "tools", "spec_nvrtc.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    tm, cons = _match_error_set()
    dump = traced(monkeypatch, tmp_path)
    monkeypatch.delenv("GK_SPEC_CHECK")
    _, drv, _ = make_pair(tm, cons, lib_path=HOSTEMU)
    drv.ReviewBlob(W.PyBlob(_mixed_pods(50)), with_results=False)
    drv.close()
    text = dump.read_text()
    walk = text[text.index("GK_SPEC_FN bool gk_spec_object"):text.index("#define GK_SPEC_NS ")]
    assert "GK_SPEC_MATCH(" not in walk and "B.flags" not in walk
    try:
        cubin, _, _ = tool.nvrtc_compile(text.encode())
    except RuntimeError as e:
        if "libnvrtc not found" in str(e):
            pytest.skip("no NVRTC in this container")
        raise
    assert b"gk_spec_rows_kernel" in cubin and b"gk_spec_kernel" in cubin


def _gpu_pair(tm, cons, docs, monkeypatch, eps=(k8s.AUDIT_EP,)):
    out = []
    for env in ({"GK_SPEC": "0"}, {"GK_SPEC_MIN_OBJECTS": "0"}):
        for k in ("GK_SPEC", "GK_SPEC_MIN_OBJECTS", "GK_SPEC_CHECK"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        drv = D.Driver()
        for k, r in tm:
            drv.add_template(k, r)
        for c in cons:
            drv.AddConstraint(c)
        rb = drv.upload_blob(W.PyBlob(docs))
        got = {}
        for ep in eps:
            r = rb.eval(ep, flags=D.F_MATERIALIZE)
            got[ep] = (drv.last_kernel(), np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True), list(r.totals), list(r.err_totals),
                       sorted((x.object, x.constraint, x.msg) for x in r.results if x.autoreject))
        rb.free()
        drv.close()
        out.append(got)
    return out


@pytest.mark.gpu
def test_gpu_rows_and_tile_kernels_against_the_interpreter(monkeypatch):
    """On the GPU, both launches over a page of skipped objects, matcher errors of three kinds of block, empty scopes, and a 40-row
    object every 997: bitmaps, totals and the autoreject results identical to the interpreter's."""
    tm, cons = _match_error_set()
    docs = _mixed_pods(9000)
    for i in range(3, len(docs), 997):
        docs[i] = json.dumps(pod(i, [container(i + j) for j in range(40)])).encode()
    want, got = _gpu_pair(tm, cons, docs, monkeypatch, eps=(k8s.AUDIT_EP, k8s.WEBHOOK_EP))
    for ep in want:
        assert want[ep][0] == "gk_eval_kernel" and got[ep][0] == "gk_spec_kernel", (ep, want[ep][0], got[ep][0])
        for a, b, what in zip(want[ep][1:], got[ep][1:], ("violation bitmap", "error bitmap", "totals", "error totals", "autoreject results")):
            assert (a == b) if what == "autoreject results" else np.array_equal(a, b), (ep, what)
    assert sum(want[k8s.AUDIT_EP][4]) > 0 and sum(want[k8s.AUDIT_EP][3]) > 0
