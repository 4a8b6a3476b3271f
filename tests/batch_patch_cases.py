"""Cases shared by the tests of gk_batch_patch on the GPU (test_batch_patch.py) and on the test-only host emulation
(test_batch_patch_hostemu.py).  Each case takes the library path.  After every patch the batch must be what a fresh
gk_batch_upload_blob of the resulting object list is: the same planes, totals, object errors and materialised violations, the same
gk_audit_add_batch_ordered report, and the pairs and the audit of the oracle."""
import json
import random

import numpy as np

import batch_refresh_cases as R
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import audit as OA
from oracle import k8s

LIMIT = 5


def violations(r):
    return [(v.object, v.constraint, v.msg, json.dumps(v.details, sort_keys=True), v.enforcement_action, v.scoped_enforcement_actions, v.autoreject)
            for v in r.results]


def audit_report(eng, rb):
    run = D.AuditRun(eng.drv, violations_limit=LIMIT)
    run.add_batch_ordered(rb, k8s.AUDIT_EP)
    rep = run.report()
    run.close()
    for k in ("pairsEvaluated", "pairsCounted"):
        rep.pop(k, None)
    return json.dumps(rep, sort_keys=True)


def check(eng, rb, docs, process="", what="", expand=False, oracle=True):
    """The patched batch against a fresh upload of `docs` with the same flags, and against the oracle."""
    assert len(rb) == len(docs), (what, len(rb), len(docs))
    fresh = eng.drv.upload_blob(W.PyBlob(docs), process=process, keep_source=True, expand=expand)
    for flags in (0, D.F_MATERIALIZE):
        got, want = rb.eval(k8s.AUDIT_EP, flags), fresh.eval(k8s.AUDIT_EP, flags)
        R.assert_same_as_fresh(R.snapshot(got), R.snapshot(want), what)
        if flags:
            assert violations(got) == violations(want), what
    got_rep = audit_report(eng, rb)
    assert got_rep == audit_report(eng, fresh), what
    fresh.free()
    if oracle and not expand:
        snap = R.snapshot(rb.eval(k8s.AUDIT_EP))
        R.assert_oracle(eng, docs, snap, process, what)
        objs = [json.loads(d) for o, d in enumerate(docs) if not (snap[5] and snap[5][o])]
        want = OA.audit(eng.orc, objs, namespaces={x["metadata"]["name"]: x for x in eng.nss},
                        excluded_namespaces=eng.excluded.get(process, ()) if process else (), limit=LIMIT)
        rep = json.loads(got_rep)
        assert rep["totalViolations"] == {"%s/%s" % k: v for k, v in want["totals"].items()}, what
        for key, lst in want["violations"].items():
            w = [{k: v for k, v in sv.items() if not (k in ("namespace", "enforcementActions") and not v)} for sv in lst]
            assert rep["violations"]["%s/%s" % key] == w, (what, key)


def patch(rb, docs, drop, add):
    """Patches rb and the list `docs` the same way; returns the new list."""
    st = rb.patch(drop, add)
    gone = set(drop)
    out = [d for i, d in enumerate(docs) if i not in gone] + list(add)
    assert st["n"] == len(out)
    return out


def renamed(doc, k):
    """A new version of a document: another label value, so that its results may change."""
    try:
        d = json.loads(doc)
    except ValueError:
        return doc
    if isinstance(d, dict) and isinstance(d.get("metadata"), dict):
        d["metadata"].setdefault("labels", {})
        if isinstance(d["metadata"]["labels"], dict):
            d["metadata"]["labels"]["patched"] = "v%d" % k
            if k % 3 == 0:
                d["metadata"]["labels"].pop("app", None)
        return json.dumps(d, separators=(",", ":")).encode()
    return doc


def replace_some(rnd, docs, share, k=0):
    m = max(1, int(len(docs) * share))
    drop = rnd.sample(range(len(docs)), m)
    return drop, [renamed(docs[i], k + j) for j, i in enumerate(drop)]


def case_replace_share(lib, n=160, share=0.01, process="audit", seed=1, oracle=True, kernel=None):
    """A random share of a config-2 page replaced by new versions: the damaged and refused documents of damaged_page are on both
    sides, and their object errors move with them.  `kernel`: the kernel that must have evaluated the patched batch."""
    eng, _ = R.config2_start(lib)
    if process:
        eng.exclude(process, ["ns-00*", "*-system"])
    rnd = random.Random(seed)
    docs = R.damaged_page(n, start=91000)
    rb = eng.drv.upload_blob(W.PyBlob(docs), process=process, keep_source=True)
    bad = [i for i, d in enumerate(docs) if d in R.BAD_DOCS]
    drop, add = replace_some(rnd, docs, share)
    drop = sorted(set(drop) | {bad[0]})
    add = add + [R.BAD_DOCS[1], R.BAD_DOCS[0]]
    docs = patch(rb, docs, drop, add)
    check(eng, rb, docs, process, "a replaced share of %g" % share, oracle=oracle)
    if kernel:
        rb.eval(k8s.AUDIT_EP)
        assert eng.drv.last_kernel() == kernel
    rb.free()
    eng.close()


def case_mixed_kinds(lib, n=300, seed=2):
    """Config-4 objects (several kinds) with wide objects that the hand-over sends to the interpreter, dropped and staying."""
    tm, cons = W.config4()
    eng = R.Engine(lib, W.synth_namespaces())
    for kind, rego in tm:
        eng.template(kind, rego)
    for c in cons:
        eng.constraint(c)
    blob = W.synth_objects(93000, n, mode=1)
    docs = [blob.get(i) for i in range(n)]
    pods = [i for i, d in enumerate(docs) if json.loads(d).get("kind") == "Pod"]
    assert len(pods) > 2 and len({json.loads(d).get("kind") for d in docs}) > 1
    for i in pods[:2]:   # (more containers than the mask registers hold: the hand-over sends them to the interpreter)
        wide = json.loads(docs[i])
        wide["spec"]["containers"] = [dict(wide["spec"]["containers"][0], name="c%d" % k) for k in range(48)]
        docs[i] = json.dumps(wide, separators=(",", ":")).encode()
    rb = eng.drv.upload_blob(W.PyBlob(docs), keep_source=True)
    rnd = random.Random(seed)
    drop, add = replace_some(rnd, [d for d in docs], 0.05)
    drop = sorted(set(drop) | {pods[1]} - {pods[0]})
    add.append(docs[pods[0]])
    docs = patch(rb, docs, drop, add)
    check(eng, rb, docs, "", "mixed kinds")
    rb.free()
    eng.close()


def case_sequence(lib, n=200, steps=5, seed=3):
    """Five patches in a row, each checked against a fresh upload: offsets must not drift across splices."""
    eng, _ = R.config2_start(lib)
    rnd = random.Random(seed)
    docs = R.damaged_page(n, start=95000)
    rb = eng.drv.upload_blob(W.PyBlob(docs), keep_source=True)
    for s in range(steps):
        drop, add = replace_some(rnd, docs, 0.05 * (s + 1), k=100 * s)
        extra = [json.dumps(json.loads(W.synth_objects(96000 + 10 * s, 1).get(0))).encode()]
        docs = patch(rb, docs, drop, add + extra)
        check(eng, rb, docs, "", "patch %d of a sequence" % s, oracle=s in (0, steps - 1))
    rb.free()
    eng.close()


def case_edges(lib, n=40):
    """Drop nothing and add nothing; drop the first and the last; drop everything; add to an empty batch; a document of 0 bytes."""
    eng, _ = R.config2_start(lib)
    docs = R.damaged_page(n, start=97000)
    rb = eng.drv.upload_blob(W.PyBlob(docs), keep_source=True)
    docs = patch(rb, docs, [], [])
    check(eng, rb, docs, "", "an empty patch")
    docs = patch(rb, docs, [len(docs) - 1, 0], [docs[0]])
    check(eng, rb, docs, "", "the first and the last dropped")
    docs = patch(rb, docs, list(range(len(docs))), [])
    assert docs == [] and len(rb) == 0
    check(eng, rb, docs, "", "everything dropped", oracle=False)
    more = R.damaged_page(12, start=98000)
    docs = patch(rb, docs, [], more)
    check(eng, rb, docs, "", "added to an empty batch")
    docs = patch(rb, docs, [3], [b""])
    check(eng, rb, docs, "", "a document of 0 bytes")
    rb.free()
    eng.close()


def case_constraint_between(lib, n=120):
    """A template and a constraint added between the upload and the patch: the patched batch is a fresh upload under the new set."""
    t = W.templates()
    eng, by_kind = R.config2_start(lib)
    docs = R.damaged_page(n, start=99000)
    rb = eng.drv.upload_blob(W.PyBlob(docs), process="audit", keep_source=True)
    eng.template(t["containerlimits"]["kind"], t["containerlimits"]["rego"])
    eng.constraint(by_kind[t["containerlimits"]["kind"]][0])
    eng.exclude("audit", ["ns-01*"])
    docs = patch(rb, docs, [2, 9, 50], [docs[9]])
    check(eng, rb, docs, "audit", "a constraint added before the patch")
    rb.free()
    eng.close()


class _DriverOnly:
    def __init__(self, drv):
        self.drv = drv


def case_expanded(lib, n=400):
    """An expanded batch (expand-deployments over a config-4 page): Deployments dropped and added; every call equals a fresh upload
    and gk_review_batch of the resulting objects."""
    import expand_sweep_cases as X
    import test_capi_entry_points as T
    drv = X.engine(lib)
    drv.AddExpansionTemplate(T._expansion_template("expand-deployments", ["Deployment"], ("", "v1", "Pod")))
    blob = W.synth_objects(94000, n, mode=1)
    docs = [blob.get(i) for i in range(n)]
    rb = drv.upload_blob(W.PyBlob(docs), keep_source=True, expand=True)
    deps = [i for i, d in enumerate(docs) if json.loads(d).get("kind") == "Deployment"]
    assert len(deps) > 2
    docs = patch(rb, docs, deps[:2] + [1], [docs[deps[0]], renamed(docs[deps[1]], 7), renamed(docs[deps[2]], 8)])
    check(_DriverOnly(drv), rb, docs, "", "an expanded batch", expand=True)
    X.check_against_review(lib, drv, rb, [D.Review(object=json.loads(d), source="Original") for d in docs], "", "a patched expanded batch")
    rb.free()
    drv.close()


def case_invalid(lib, n=30):
    """Refused calls (GK_ERR_INVALID) leave the batch as it was."""
    eng, _ = R.config2_start(lib)
    docs = R.damaged_page(n, start=99500)
    rb = eng.drv.upload_blob(W.PyBlob(docs), keep_source=True)
    before = R.snapshot(rb.eval(k8s.AUDIT_EP))

    def refused(batch, drop, match):
        with np.testing.assert_raises_regex(D.GkError, match) as cm:
            batch.patch(drop, [docs[0]])
        assert cm.exception.code == -1   # GK_ERR_INVALID

    refused(rb, [len(docs)], "out of range")
    refused(rb, [3, 4, 3], "given twice")
    R.assert_same_as_fresh(R.snapshot(rb.eval(k8s.AUDIT_EP)), before, "refused patches")
    assert len(rb) == len(docs)
    plain = eng.drv.upload_blob(W.PyBlob(docs))
    refused(plain, [0], "keeps no device source")
    objs = eng.drv.upload([D.Review(object=d, source="Original") for d in docs])
    refused(objs, [0], "keeps no device source")
    R.assert_same_as_fresh(R.snapshot(plain.eval(k8s.AUDIT_EP)), before, "a refused patch of a batch without a kept source")
    for b in (rb, plain, objs):
        b.free()
    eng.close()


def case_host_flattened(lib, n=40):
    """A referential constraint set is flattened on the host: a batch uploaded under it keeps no device source and is refused, and a
    kept batch is refused while such a set is current (a patch never flattens on the host); both evaluate as before."""
    v = R.golden("referential_vectors.json")["uniquelabel"]
    eng, _ = R.config2_start(lib, per_template=1)
    docs = R.damaged_page(n, start=99700)
    kept = eng.drv.upload_blob(W.PyBlob(docs), keep_source=True)
    kind, rego, *_ = k8s.template_from_yaml_obj(v["template"])
    eng.template(kind, rego)
    eng.constraint(v["constraint"])
    assert "ingest: device" not in eng.drv.Dump()
    late = eng.drv.upload_blob(W.PyBlob(docs), keep_source=True)
    before = R.snapshot(late.eval(k8s.AUDIT_EP))
    for rb, match in ((late, "keeps no device source"), (kept, "flattened on the host")):
        with np.testing.assert_raises_regex(D.GkError, match) as cm:
            rb.patch([0], [docs[0]])
        assert cm.exception.code == -1 and len(rb) == len(docs)
    R.assert_same_as_fresh(R.snapshot(late.eval(k8s.AUDIT_EP)), before, "a refused patch")
    assert kept.refresh()["rebuilt"]
    R.assert_same_as_fresh(R.snapshot(kept.eval(k8s.AUDIT_EP)), before, "a refused patch, then a refresh")
    kept.free()
    late.free()
    eng.close()
