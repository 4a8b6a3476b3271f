"""The generated kernel's hand-over plan (spec_codegen.cpp: gk_spec_wide, gk_spec_tile_whole, gk_spec_plan_kernel): which objects are too
wide for the mask registers is decided from the CSR offsets alone, before any row is evaluated, and a tile with more than
GK_HANDOVER_MAX of them goes to the interpreter whole.  On the test-only host emulation the plan's per-object test must agree with the
object walk's for every object (the host build of the generated text counts the objects where they differ), and the plan's units
and whole tiles must be the rule restated here, over the device's 512-object tiles."""
import json
import os
import random
import re

import pytest

import gpu_path_cases as G
from conftest import HOSTEMU, assert_same, make_pair
from gatekeeper_b200 import workloads as W
from oracle import k8s

from test_spec_fold import container, pod

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = int(re.search(r"#define GK_HANDOVER_MAX (\d+)u", open(os.path.join(ROOT, "gatekeeper_b200", "csrc", "program.h")).read()).group(1))
TILE = 512
MISSING_NS = "plan-no-such-namespace"
PLAN = re.compile(r"\[spec plan\] tiles of (\d+): (\d+) units:([^;]*); whole tiles:([^;]*); disagreements: (\d+)$")


def constraint_set():
    """The config-2 constraints, plus one whose namespaceSelector makes a Pod in an uncached Namespace a matcher error."""
    tm, cons = W.config2()
    c = json.loads(json.dumps(cons[0]))
    c["metadata"]["name"] = "plan-nssel"
    c["spec"]["match"] = {"kinds": [{"apiGroups": [""], "kinds": ["Pod"]}], "namespaceSelector": {"matchLabels": {"env": "prod"}}}
    return tm, cons + [c]


def page(n, wide, ns_missing=()):
    """One-container Pods (never wide); the objects `wide` get 33 rows in one scope, cycling through the scope kinds."""
    scope = {i: G.ROW_SCOPES[m % len(G.ROW_SCOPES)] for m, i in enumerate(sorted(wide))}
    docs = []
    for i in range(n):
        d = pod(i, [container(i)])
        if i in wide:
            G._set_rows(d, scope[i], 33)
        if i in ns_missing:
            d["metadata"]["namespace"] = MISSING_NS
        docs.append(json.dumps(d).encode())
    return docs


def expected_plan(n, wide):
    """The rule: per tile, more than K wide objects hand the tile over whole; otherwise each wide object is a unit of its own."""
    units, whole = [], []
    for t in range((n + TILE - 1) // TILE):
        lo, hi = t * TILE, min(n, (t + 1) * TILE)
        w = sorted(i for i in wide if lo <= i < hi)
        if len(w) > K:
            units.append((lo, hi - lo))
            whole.append(t)
        else:
            units += [(i, 1) for i in w]
    return units, whole


def plan_of(monkeypatch, capfd, n, wide, ns_missing=()):
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    tm, cons = constraint_set()
    docs = page(n, wide, ns_missing)
    orc, drv, _ = make_pair(tm, cons, W.synth_namespaces(), lib_path=HOSTEMU)
    rb = drv.upload_blob(W.PyBlob(docs))
    capfd.readouterr()
    r = rb.eval(k8s.AUDIT_EP)
    keys, viol, err = list(r.constraints), r.viol_bits.copy(), r.err_bits.copy()
    rb.free()
    drv.close()
    lines = capfd.readouterr().err.splitlines()
    check = [ln for ln in lines if ln.startswith("[spec check]")]
    assert check, "no [spec check] line: was the generated text checked?"
    assert int(re.search(r"\((\d+) too big", check[-1]).group(1)) == len(wide), check[-1]
    m = [PLAN.match(ln) for ln in lines if ln.startswith("[spec plan]")]
    assert m and m[-1], "no [spec plan] line"
    m = m[-1]
    assert int(m.group(1)) == TILE
    units = [tuple(int(x) for x in u.split("+")) for u in m.group(3).split()]
    assert int(m.group(2)) == len(units)
    assert int(m.group(5)) == 0, "the plan's test and the object walk disagree on %s objects" % m.group(5)
    # the wide objects and the unknown Namespace's are the interpreter's here: the oracle's pairs on them and on a sample
    objs = sorted(set(wide) | set(ns_missing) | set(random.Random(n).sample(range(n), min(n, 40))))
    v, e = G.oracle_pairs(orc, docs, objs, k8s.AUDIT_EP)
    assert_same(v, G.bit_pairs(viol, keys, objs))
    assert_same(e, G.bit_pairs(err, keys, objs))
    return units, [int(t) for t in m.group(4).split()], keys, err


CASES = {
    # object 0, lanes 31 / 32, the first and last object of a tile, a run across a warp boundary, a run across a tile boundary
    # (2 + 2), more than K in one tile between tiles with few, the last object of a partial last tile
    "edges": (7 * TILE + 100, {0, 31, 32, TILE, 2 * TILE - 1} | set(range(2 * TILE + 31, 2 * TILE + 34)) | set(range(4 * TILE - 2, 4 * TILE + 2))
              | {5 * TILE + 40 * i for i in range(K + 1)} | {6 * TILE + 200, 6 * TILE + 300, 7 * TILE + 99}),
    # exactly K in one tile (each alone), K + 1 in the next (whole), K + 1 in a partial last tile of 10 objects (whole)
    "at_the_threshold": (3 * TILE + 10, {TILE + 7 * i for i in range(K)} | {2 * TILE + 3 * i for i in range(K + 1)} | set(range(3 * TILE, 3 * TILE + K + 1))),
    "none": (TILE + 1, set()),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_plan_units_and_whole_tiles(case, monkeypatch, capfd):
    n, wide = CASES[case]
    assert K >= 3
    units, whole, _, _ = plan_of(monkeypatch, capfd, n, wide)
    assert (units, whole) == expected_plan(n, wide)


def test_wide_object_that_is_a_matcher_error(monkeypatch, capfd):
    """A wide object whose Namespace is unknown: a unit of its own, and its matcher error is in the error plane."""
    n, wide, missing = 2 * TILE, {TILE + 300, TILE + 400}, {TILE + 300, TILE + 301}
    units, whole, keys, err = plan_of(monkeypatch, capfd, n, wide, missing)
    assert (units, whole) == expected_plan(n, wide) and units == [(TILE + 300, 1), (TILE + 400, 1)]
    c = [i for i, k in enumerate(keys) if k.endswith("/plan-nssel")][0]
    assert (int(err[TILE + 300, c // 32]) >> (c % 32)) & 1
