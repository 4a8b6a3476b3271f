"""The offset image of the generated kernel (spec_codegen.cpp): gk_spec_plan_kernel writes, once per batch and constraint set, every
tile's run of tile-relative CSR offsets as 16-bit values, in the layout gk_spec_stage() copies verbatim (cp.async, with the export
planes).  Run t starts at t * stride values; stride bounds every run from the largest tile's rows per scope (SpecSource::image_stride).
A batch with a tile of more than 65535 rows in a nested scope is interpreted.  Checked here: the layout the host build traces against
a restatement; the generated text against the interpreted netlist object by object (GK_SPEC_CHECK=1, the image and the staging area
poisoned) and the oracle, over pages with empty scopes in a tile, wide objects alone and in whole tiles, a refresh that adds a
nested scope, an expanded batch and a fork; the 16-bit limit; on the GPU, the generated kernel against the interpreter and the
backend's image allocation against the traced layout."""
import json
import re

import numpy as np
import pytest

import expand_sweep_cases as X
import gpu_path_cases as G
from conftest import HOSTEMU, has_cuda, make_pair
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import k8s

from test_spec_fold import container, pod

TILE = 512   # the device's tile, and the host build's plan tile (GK_SPEC_HOST_PLAN_TILE)
OFFSETS = re.compile(r"\[spec offsets\] tiles of (\d+): scopes([^;]*); rows([^;]*); stride (\d+) bytes; runs (\d+) bytes; image (\d+) bytes$")

PORTS = ("K8sOffsetPorts", """package k8soffsetports

violation[{"msg": msg}] {
  c := input.review.object.spec.containers[_]
  p := c.ports[_]
  p.hostPort > 1000
  msg := sprintf("hostPort %v", [p.hostPort])
}
""")
IMAGES = ("K8sOffsetImages", """package k8soffsetimages

violation[{"msg": msg}] {
  c := input.review.object.spec.containers[_]
  endswith(c.image, ":latest")
  msg := sprintf("latest %v", [c.name])
}
""")


def restate(line):
    """The traced image restated: {parent scope per nested scope}, every tile's rows of those parents, and the stride, run and image
    bytes the layout gives for them (cap: the largest tile's rows of a scope, the tile itself in scope 0)."""
    m = OFFSETS.match(line)
    assert m, line
    tile = int(m.group(1))
    scopes = [tuple(int(x) for x in s.split("/")) for s in m.group(2).split()]
    tiles = [[int(x) for x in t.split()] for t in m.group(3).split("|")]
    assert all(len(t) == len(scopes) for t in tiles), line
    cap = {}
    for t in tiles:
        for (_, p), c in zip(scopes, t):
            cap[p] = max(cap.get(p, 0), c)
    cap[0] = tile
    stride = (sum(cap[p] + 1 for _, p in scopes) + 7) // 8 * 8
    runs = [sum(c + 1 for c in t) for t in tiles]
    return {"tile": tile, "scopes": scopes, "tiles": tiles, "stride": 2 * stride, "runs": sum((r + 7) // 8 * 16 for r in runs),
            "image": 2 * stride * len(tiles), "values": runs,
            "traced": (int(m.group(4)), int(m.group(5)), int(m.group(6)))}


def offsets_line(lines):
    got = [ln for ln in lines if ln.startswith("[spec offsets]")]
    assert got, "no [spec offsets] line"
    r = restate(got[-1])
    assert r["traced"] == (r["stride"], r["runs"], r["image"]), r
    return r


def host_eval(monkeypatch, capfd, tm, cons, docs, audit=False):
    """The page on the host emulation, the generated text checked against the interpreted netlist; every object's pairs against the
    oracle.  With `audit`, also an audit of the batch (which evaluates a fork of it).  Returns stderr's lines and the too-big count."""
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    orc, drv, _ = make_pair(tm, cons, W.synth_namespaces(), lib_path=HOSTEMU)
    rb = drv.upload_blob(W.PyBlob(docs))
    capfd.readouterr()
    r = rb.eval(k8s.AUDIT_EP)
    keys, viol, err = list(r.constraints), np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True)
    if audit:
        au = D.AuditRun(drv, violations_limit=5)
        au.add_batch(rb)
        au.report()
        au.close()
    rb.free()
    drv.close()
    lines = capfd.readouterr().err.splitlines()
    check = [ln for ln in lines if ln.startswith("[spec check]")]
    assert check, "no [spec check] line: was the generated text checked?"
    every = range(len(docs))
    want_v, want_e = G.oracle_pairs(orc, docs, every, k8s.AUDIT_EP)
    G.assert_same(want_v, G.bit_pairs(viol, keys, every))
    G.assert_same(want_e, G.bit_pairs(err, keys, every))
    assert want_v, "the page violates nothing: the case checks nothing"
    return lines, int(re.search(r"\((\d+) too big", check[-1]).group(1))


def ports_container(j, nports):
    return container(j, image="repo/img-%d:%s" % (j, "latest" if j % 3 == 0 else "v1"),
                     ports=[{"containerPort": 80 + k, "hostPort": 900 + 70 * ((j + k) % 4)} for k in range(nports)])


def counts_page(counts, nports=lambda i, j: (i + j) % 3):
    return [json.dumps(pod(i, [ports_container(j, nports(i, j)) for j in range(k)])).encode() for i, k in enumerate(counts)]


def edge_counts(n):
    """Containers per object: 0 to 4, every object of the second device tile without any (a tile with no rows in the nested scopes),
    a wide object (40) every 97th; n not a multiple of the tile (a partial last tile)."""
    return [0 if TILE <= i < 2 * TILE else 40 if i % 97 == 50 else (i * 5 + i // 7) % 5 for i in range(n)]


def test_edge_page_layout_and_check(monkeypatch, capfd):
    """Two nested scopes (containers, their ports) over a page with an empty tile, wide objects and a partial last tile: the traced
    image is the restated layout, its rows are the page's, and the text equals the interpreter and the oracle on every object."""
    n = 3 * TILE + 77
    ks = edge_counts(n)
    docs = counts_page(ks)
    lines, big = host_eval(monkeypatch, capfd, [PORTS, IMAGES], [W._constraint(PORTS[0], "ports", match=W.POD), W._constraint(IMAGES[0], "images", match=W.POD)], docs)
    assert big == sum(1 for k in ks if k > 32)
    r = offsets_line(lines)
    assert r["tile"] == TILE and len(r["tiles"]) == 4
    parents = [p for _, p in r["scopes"]]
    assert 0 in parents and len(r["scopes"]) == 2, r["scopes"]
    conts = [sum(ks[t * TILE:(t + 1) * TILE]) for t in range(4)]
    for t, rows in enumerate(r["tiles"]):
        assert rows[parents.index(0)] == min(TILE, n - t * TILE)
        assert rows[1 - parents.index(0)] == conts[t], (t, rows, conts)
    assert conts[1] == 0
    assert any(v % 8 for v in r["values"]), r["values"]


def test_config2_layout(monkeypatch, capfd):
    """The flagship constraint set over synthetic Pods: 14 nested scopes, and the traced image is the restated layout."""
    tm, cons = W.config2()
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    _, drv, _ = make_pair(tm, cons, W.synth_namespaces(), lib_path=HOSTEMU)
    capfd.readouterr()
    drv.ReviewBlob(W.synth_objects(0, 2 * TILE + 300), k8s.AUDIT_EP, with_results=False)
    drv.close()
    lines = capfd.readouterr().err.splitlines()
    assert [ln for ln in lines if ln.startswith("[spec check]")]
    r = offsets_line(lines)
    assert len(r["scopes"]) == 14 and len(r["tiles"]) == 3
    assert [rows[0] for rows in r["tiles"]] == [TILE, TILE, 300]


def test_whole_tiles_of_wide_objects(monkeypatch, capfd):
    """A device tile of wide objects only (handed over whole) between tiles with single wide ones: the image still covers every tile."""
    n = 2 * TILE + 130
    ks = [40 if TILE <= i < 2 * TILE else 40 if i % 150 == 3 else i % 4 for i in range(n)]
    lines, big = host_eval(monkeypatch, capfd, [PORTS], [W._constraint(PORTS[0], "ports", match=W.POD)], counts_page(ks, lambda i, j: j % 2))
    assert big == sum(1 for k in ks if k > 32)
    r = offsets_line(lines)
    assert r["tiles"][1][[p for _, p in r["scopes"]].index(0)] == TILE
    plan = [ln for ln in lines if ln.startswith("[spec plan]")]
    assert plan and plan[-1].endswith("disagreements: 0") and "whole tiles: 1;" in plan[-1], plan


def test_refresh_adds_a_nested_scope(monkeypatch, capfd):
    """A resident batch checked with a constraint on the containers alone, then refreshed after one that reads their ports: the image
    gains a scope, and the refreshed batch is checked again."""
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    _, drv, _ = make_pair([IMAGES, PORTS], [W._constraint(IMAGES[0], "images", match=W.POD)], lib_path=HOSTEMU)
    rb = drv.upload_blob(W.PyBlob(counts_page(edge_counts(TILE + 200))))
    capfd.readouterr()
    r0 = rb.eval(k8s.AUDIT_EP)
    before = capfd.readouterr().err.splitlines()
    assert [ln for ln in before if ln.startswith("[spec check]")]
    assert len(offsets_line(before)["scopes"]) == 1
    drv.AddConstraint(W._constraint(PORTS[0], "ports", match=W.POD))
    assert rb.refresh()["rebuilt"] is True
    capfd.readouterr()
    r1 = rb.eval(k8s.AUDIT_EP)
    after = capfd.readouterr().err.splitlines()
    assert [ln for ln in after if ln.startswith("[spec check]")]
    assert len(offsets_line(after)["scopes"]) == 2
    assert len(r1.constraints) == len(r0.constraints) + 1 and sum(r1.totals) > sum(r0.totals)
    rb.free()
    drv.close()


def test_expanded_batch(monkeypatch, capfd):
    """A GK_F_EXPAND batch (its resultants are a batch of their own, with an image of their own), every eval checked."""
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    X.case_every_call_equals_review(HOSTEMU, "blob")
    err = capfd.readouterr().err.splitlines()
    assert [ln for ln in err if ln.startswith("[spec check]")]
    offsets_line(err)


def test_fork_of_the_batch(monkeypatch, capfd):
    """An audit of the batch evaluates a fork of it under another netlist: checked too, with its own image."""
    lines, _ = host_eval(monkeypatch, capfd, [PORTS, IMAGES], [W._constraint(PORTS[0], "ports", match=W.POD), W._constraint(IMAGES[0], "images", match=W.POD)],
                         counts_page(edge_counts(TILE + 90)), audit=True)
    assert len([ln for ln in lines if ln.startswith("[spec check]")]) >= 2
    offsets_line(lines)


def big_page():
    """One object with 65536 containers (a tile of more rows in a nested scope than 16 bits hold) among ordinary ones."""
    ks = [i % 3 for i in range(200)]
    docs = counts_page(ks, lambda i, j: 0)
    docs[70] = json.dumps(pod(70, [{"name": "c%d" % j, "image": "x:latest" if j % 9 == 0 else "x:v1"} for j in range(65536)])).encode()
    return docs


def test_tile_beyond_16_bits_is_interpreted(monkeypatch, capfd):
    """The host build hands every object of such a batch to the interpreter, which agrees with the oracle."""
    docs = big_page()
    lines, big = host_eval(monkeypatch, capfd, [IMAGES], [W._constraint(IMAGES[0], "images", match=W.POD)], docs)
    assert big == len(docs)


# ---- on the GPU

def gpu_case(monkeypatch, env, tm, cons, docs, extra=None):
    """The page through one build of the evaluation (env) at both enforcement points, an audit (a fork), and, with `extra`, again after
    a refresh that adds it."""
    from test_spec_planes import gpu_driver
    drv = gpu_driver(monkeypatch, tm, cons, env)
    rb = drv.upload_blob(W.PyBlob(docs))
    out = []
    for step in range(2 if extra else 1):
        if step:
            drv.AddConstraint(extra)
            assert rb.refresh()["rebuilt"] is True
        for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP):
            r = rb.eval(ep, flags=D.F_MATERIALIZE)
            out.append((drv.last_kernel(), np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True), list(r.totals), list(r.err_totals),
                        sorted((x.object, x.constraint, x.msg) for x in r.results if x.autoreject)))
        au = D.AuditRun(drv, violations_limit=5)
        au.add_batch(rb)
        out.append(json.dumps(au.report(), sort_keys=True))
        au.close()
    rb.free()
    drv.close()
    return out


def gpu_pages():
    return {"edges": counts_page(edge_counts(3 * TILE + 77)),
            "whole_tile": counts_page([40 if TILE <= i < 2 * TILE else 40 if i % 150 == 3 else i % 4 for i in range(2 * TILE + 130)], lambda i, j: j % 2)}


@pytest.mark.gpu
@pytest.mark.parametrize("page", ["edges", "whole_tile"])
def test_gpu_against_the_interpreter(page, monkeypatch):
    """The pages forced through the generated kernel, before and after a refresh that adds the ports scope: bitmaps, error planes,
    totals, matcher errors and audit reports identical to the interpreter's at both enforcement points."""
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    tm, cons, extra = [IMAGES, PORTS], [W._constraint(IMAGES[0], "images", match=W.POD)], W._constraint(PORTS[0], "ports", match=W.POD)
    docs = gpu_pages()[page]
    want = gpu_case(monkeypatch, {"GK_SPEC": "0"}, tm, cons, docs, extra)
    got = gpu_case(monkeypatch, {"GK_SPEC_MIN_OBJECTS": "0"}, tm, cons, docs, extra)
    for a, b in zip(want, got):
        if isinstance(a, str):
            assert a == b, "audit reports differ"
            continue
        assert a[0] == "gk_eval_kernel" and b[0] == "gk_spec_kernel", (a[0], b[0])
        for x, y, what in zip(a[1:], b[1:], ("violation bitmap", "error bitmap", "totals", "error totals", "matcher errors")):
            assert (x == y) if what == "matcher errors" else np.array_equal(x, y), (page, what)
    assert sum(want[-2][3]) > sum(want[0][3]) > 0


@pytest.mark.gpu
def test_gpu_tile_beyond_16_bits_is_interpreted(monkeypatch):
    """The page with a tile of 65536 container rows runs the interpreter even when the generated kernel is forced, and agrees with it
    (and so with the oracle, as the host case shows)."""
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    tm, cons = [IMAGES], [W._constraint(IMAGES[0], "images", match=W.POD)]
    docs = big_page()
    want = gpu_case(monkeypatch, {"GK_SPEC": "0"}, tm, cons, docs)
    got = gpu_case(monkeypatch, {"GK_SPEC_MIN_OBJECTS": "0"}, tm, cons, docs)
    assert [x[0] for x in got if not isinstance(x, str)] == ["gk_eval_kernel"] * 2
    for a, b in zip(want, got):
        if isinstance(a, str):
            assert a == b
            continue
        for x, y in zip(a[1:], b[1:]):
            assert (x == y) if isinstance(x, list) else np.array_equal(x, y)
    assert sum(want[0][3]) > 0


@pytest.mark.gpu
def test_gpu_image_bytes_are_the_layout(monkeypatch, capfd):
    """The backend's image for the config-2 page: the stride and bytes the host build traces for the same page."""
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    from test_spec_planes import gpu_driver
    tm, cons = W.config2()
    n = 3 * TILE + 77
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    _, drv, _ = make_pair(tm, cons, W.synth_namespaces(), lib_path=HOSTEMU)
    capfd.readouterr()
    drv.ReviewBlob(W.synth_objects(0, n), k8s.AUDIT_EP, with_results=False)
    drv.close()
    r = offsets_line(capfd.readouterr().err.splitlines())
    drv = gpu_driver(monkeypatch, tm, cons, {"GK_SPEC_MIN_OBJECTS": "0", "GK_TRACE_LAUNCH": "1"})
    capfd.readouterr()
    drv.ReviewBlob(W.synth_objects(0, n), k8s.AUDIT_EP, with_results=False)
    assert drv.last_kernel() == "gk_spec_kernel"
    drv.close()
    got = re.findall(r"\[spec\] offset image: (\d+) bytes, (\d+) bytes per tile x (\d+) tiles", capfd.readouterr().err)
    assert got and got[-1] == (str(r["image"]), str(r["stride"]), str(len(r["tiles"]))), (got, r)
