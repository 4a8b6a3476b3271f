"""The generated kernel's hand-over of objects too wide for its mask registers (more than 32 rows in a scope): a tile with at most
GK_HANDOVER_MAX of them hands each over alone, a tile with more hands itself over whole, and the interpreter behind it evaluates
exactly those object ranges.  Forced through the generated kernel, every page must give the interpreter's bitmaps and totals at
the audit and the webhook enforcement points, and the oracle's pairs on a sample holding every wide object.
Run on an H100:  python -m pytest tests/test_spec_handover.py -m gpu -q"""
import json
import os
import random
import re

import numpy as np
import pytest

import gpu_path_cases as P
from conftest import assert_same, has_cuda, make_pair
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import k8s

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = int(re.search(r"#define GK_HANDOVER_MAX (\d+)u", open(os.path.join(ROOT, "gatekeeper_b200", "csrc", "program.h")).read()).group(1))
TILE = 512
MISSING_NS = "handover-no-such-namespace"


@pytest.fixture(scope="module", autouse=True)
def _needs_gpu():
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")


def constraint_set():
    """The config-2 constraints, plus one whose namespaceSelector makes a Pod in an uncached Namespace a matcher error."""
    tm, cons = W.config2()
    c = json.loads(json.dumps(cons[0]))
    c["metadata"]["name"] = "handover-nssel"
    c["spec"]["match"] = {"kinds": [{"apiGroups": [""], "kinds": ["Pod"]}], "namespaceSelector": {"matchLabels": {"env": "prod"}}}
    return tm, cons + [c]


def page(n, wide, ns_missing=()):
    """Synthetic Pods; the objects `wide` get 33 rows in one scope (cycling through the scope kinds), the objects `ns_missing` live in a
    Namespace the engine does not know."""
    blob = W.synth_objects(515151, n)
    docs = [blob.get(i) for i in range(n)]
    for m, i in enumerate(sorted(set(wide) | set(ns_missing))):
        d = json.loads(docs[i])
        if i in wide:
            P._set_rows(d, P.ROW_SCOPES[m % len(P.ROW_SCOPES)], 33)
        if i in ns_missing:
            d["metadata"]["namespace"] = MISSING_NS
        docs[i] = json.dumps(d).encode()
    return docs


def expected_handover(n, wide):
    """(units, objects) the generated kernel hands over for 512-object tiles."""
    per_tile = {}
    for i in wide:
        per_tile[i // TILE] = per_tile.get(i // TILE, 0) + 1
    units = objs = 0
    for t, c in per_tile.items():
        if c > K:
            units, objs = units + 1, objs + min(TILE, n - t * TILE)
        else:
            units, objs = units + c, objs + c
    return units, objs


def run(monkeypatch, capfd, tm, cons, docs, env):
    for k in ("GK_SPEC", "GK_SPEC_MIN_OBJECTS", "GK_SPEC_CHECK", "GK_TRACE_LAUNCH"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    drv = D.Driver()
    for k, r in tm:
        drv.add_template(k, r)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    rb = drv.upload_blob(W.PyBlob(docs))
    capfd.readouterr()
    out = {}
    for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP):
        r = rb.eval(ep)
        out[ep] = (drv.last_kernel(), np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True), list(r.totals), list(r.err_totals))
    keys = list(r.constraints)
    rb.free()
    drv.close()
    return keys, out, capfd.readouterr().err


def check(monkeypatch, capfd, n, wide, ns_missing=(), sample=100):
    tm, cons = constraint_set()
    docs = page(n, wide, ns_missing)
    keys, want, _ = run(monkeypatch, capfd, tm, cons, docs, {"GK_SPEC": "0"})
    keys_s, got, trace = run(monkeypatch, capfd, tm, cons, docs, {"GK_SPEC_MIN_OBJECTS": "0", "GK_TRACE_LAUNCH": "1"})
    assert keys_s == keys
    for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP):
        assert want[ep][0] == "gk_eval_kernel" and got[ep][0] == "gk_spec_kernel", (ep, want[ep][0], got[ep][0])
        for a, b, what in zip(want[ep][1:], got[ep][1:], ("violation bitmap", "error bitmap", "totals", "error totals")):
            assert np.array_equal(np.asarray(a), np.asarray(b)), "%s at %s: the generated kernel differs from the interpreter" % (what, ep)
    # the page was tiled as planned and handed over as planned, at both enforcement points
    assert set(re.findall(r"tiles of (\d+) objects", trace)) == {str(TILE)}, trace
    handed = re.findall(r"handed to the interpreter: (\d+) units \(\d+ of more than one object\), (\d+) objects, on (\d+) CTAs", trace)
    assert len(handed) == 2 and handed[0] == handed[1], handed
    # (a synthetic Pod can be wide by itself -- the join of its volumes and volume mounts -- and is then handed over alone, too)
    units, objs = expected_handover(n, wide)
    extra = int(handed[0][0]) - units
    assert 0 <= extra == int(handed[0][1]) - objs <= max(2, n // 5000), (handed, units, objs)
    # the oracle on every wide object, every object of a Namespace it does not know, and a sample of the rest
    orc, _, _ = make_pair(tm, cons, W.synth_namespaces())
    objs = sorted(set(wide) | set(ns_missing) | set(random.Random(n).sample(range(n), min(n, sample))))
    for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP):
        viol, err = P.oracle_pairs(orc, docs, objs, ep)
        assert_same(viol, P.bit_pairs(got[ep][1], keys, objs))
        assert_same(err, P.bit_pairs(got[ep][2], keys, objs))
    return keys, got, [int(h[2]) for h in handed]


def test_single_objects_runs_and_whole_tiles(monkeypatch, capfd):
    """Wide objects at object 0, at lanes 31 / 32, at the first and last object of a tile, as the last object of a partial last tile;
    a run across a warp boundary and one across a tile boundary; a tile with K + 1 between tiles with few; a wide object whose
    Namespace is unknown, which is a matcher error of the namespaceSelector constraint."""
    n = 7 * TILE + 100
    assert K >= 3
    wide = {0, 31, 32, TILE, 2 * TILE - 1}
    wide |= set(range(2 * TILE + 31, 2 * TILE + 34))                 # across the warp boundary at 2 * TILE + 32
    wide |= set(range(4 * TILE - 2, 4 * TILE + 2))                   # across the tile boundary: 2 + 2
    wide |= {5 * TILE + 40 * i for i in range(K + 1)}                # more than K: the whole tile, between tiles 4 and 6
    wide |= {6 * TILE + 200, 6 * TILE + 300, n - 1}
    keys, got, _ = check(monkeypatch, capfd, n, wide, ns_missing={6 * TILE + 300, 6 * TILE + 301})
    e = got[k8s.AUDIT_EP]
    c = [i for i, k in enumerate(keys) if k.endswith("/handover-nssel")][0]
    assert e[4][c] >= 2 and (int(e[2][6 * TILE + 300, c // 32]) >> (c % 32)) & 1


def test_more_units_than_interpreter_ctas(monkeypatch, capfd):
    """Two wide objects in every tile: more one-object units than the interpreter has resident CTAs, which stride over the list."""
    assert K >= 3
    n = 300 * TILE
    wide = {t * TILE + off for t in range(n // TILE) for off in (130, TILE - 1)}
    _, _, grids = check(monkeypatch, capfd, n, wide, sample=50)
    assert all(len(wide) > g for g in grids), grids
