"""Cases shared by the tests of gk_batch_refresh on the GPU (test_batch_refresh.py) and on the test-only host emulation
(test_batch_refresh_hostemu.py).  Each case takes the library path.  After every change to the engine a resident batch is
refreshed and evaluated: its bitmaps, totals and review-level errors must be those of a fresh upload of the same page under the
same snapshot, and its pairs those of the oracle."""
import ctypes as C
import fnmatch
import json
import random

import numpy as np

import parity_cases as P
from conftest import golden, oracle_results
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import audit as OA
from oracle import k8s

T = "admission.k8s.gatekeeper.sh"
FIRST = ("requiredlabels_basic", "allowedrepos_prefixmatch", "bannedimagetags", "psp_privileged")
BAD_DOCS = [b'{"apiVersion":"v1","kind":"Pod","metadata":{"name":"cut"', b'[1,2,3]', b'{"apiVersion":"v1","metadata":{"name":"nokind"}}']


class Engine:
    """An engine Driver and the oracle Client with the same templates, constraints, namespaces and data."""

    def __init__(self, lib, namespaces=()):
        self.drv = D.Driver(lib_path=lib)
        self.orc = k8s.Client()
        self.nss = list(namespaces)
        for ns in self.nss:
            self.orc.add_namespace(ns)
            self.orc.add_data(ns)
            self.drv.AddData(T, ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
        self.excluded = {}

    def template(self, kind, rego):
        self.drv.add_template(kind, rego)
        self.orc.add_template(kind, rego)

    def constraint(self, c):
        self.drv.AddConstraint(c)
        self.orc.add_constraint(c)

    def remove_constraint(self, kind, name):
        self.drv.RemoveConstraint({"kind": kind, "metadata": {"name": name}})
        self.orc.remove_constraint(kind, name)

    def data(self, obj):
        self.drv.AddData(T, self.orc.data_path(obj), obj)
        self.orc.add_data(obj)

    def exclude(self, process, patterns):
        self.drv.SetExcludedNamespaces(process, patterns)
        self.excluded[process] = list(patterns)

    def close(self):
        self.drv.close()


def config2_start(lib, per_template=2):
    """Four config-2 templates, `per_template` of their constraints each, and the synthetic Namespaces."""
    t = W.templates()
    tm, cons = W.config2()
    eng = Engine(lib, W.synth_namespaces())
    for name in FIRST:
        eng.template(t[name]["kind"], t[name]["rego"])
    by_kind = {}
    for c in cons:
        by_kind.setdefault(c["kind"], []).append(c)
    for name in FIRST:
        for c in by_kind[t[name]["kind"]][:per_template]:
            eng.constraint(c)
    return eng, by_kind


def damaged_page(n, start=31000, seed=11):
    """Synthetic Pods, every fifth one structurally damaged, and three documents the review refuses."""
    rnd = random.Random(seed)
    blob = W.synth_objects(start, n)
    docs = []
    for i in range(n):
        d = json.loads(blob.get(i))
        docs.append(json.dumps(P._mutate(rnd, d, rnd.choice([1, 2, 3])) if i % 5 == 0 else d).encode())
    for k, b in enumerate(BAD_DOCS):
        docs.insert(7 + 31 * k, b)
    return docs


def upload(eng, page, docs, kind, process, keep):
    if kind == "blob":
        return eng.drv.upload_blob(page, process=process, keep_source=keep)
    return eng.drv.upload([D.Review(object=d, source="Original") for d in docs], process=process)


def snapshot(r):
    return (list(r.constraints), np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True), list(r.totals), list(r.err_totals),
            list(r.object_errors or []))


def assert_same_as_fresh(got, want, what):
    for a, b, name in zip(got, want, ("constraint keys", "violation bitmap", "error bitmap", "totals", "error totals", "object errors")):
        assert np.array_equal(np.asarray(a, dtype=object) if name in ("constraint keys", "object errors") else np.asarray(a),
                              np.asarray(b, dtype=object) if name in ("constraint keys", "object errors") else np.asarray(b)), \
            "%s after %s: the refreshed batch differs from a fresh upload" % (name, what)


def _namespace_of(doc):
    md = doc.get("metadata") if isinstance(doc, dict) else None
    ns = md.get("namespace") if isinstance(md, dict) else None
    return ns if isinstance(ns, str) else None


def assert_oracle(eng, docs, got, process, what, ep=k8s.AUDIT_EP):
    """The oracle's (object, constraint) pairs for every document the review accepts; the excluder's objects have none."""
    keys = got[0]
    pats = eng.excluded.get(process, []) if process else []
    want_v, want_e, got_v, got_e = set(), set(), set(), set()
    for o, d in enumerate(docs):
        if got[5] and got[5][o]:
            continue
        doc = json.loads(d)
        ns = _namespace_of(doc)
        if any(fnmatch.fnmatchcase(ns or "", p) for p in pats):
            assert not got[1][o].any() and not got[2][o].any(), (what, o, "an excluded object has results")
            continue
        if pats and ns is None:
            continue
        for x in oracle_results(eng.orc, [D.Review(object=doc, source="Original")], ep):
            (want_e if x[-1] else want_v).add((o, x[1]))
        for c, key in enumerate(keys):
            w, b = c // 32, 1 << (c % 32)
            if int(got[1][o, w]) & b:
                got_v.add((o, key))
            if int(got[2][o, w]) & b:
                got_e.add((o, key))
    assert want_v == got_v, (what, "violations", sorted(want_v - got_v)[:5], sorted(got_v - want_v)[:5])
    assert want_e == got_e, (what, "matcher errors", sorted(want_e - got_e)[:5], sorted(got_e - want_e)[:5])
    return len(want_v)


class Scrambled:
    """Overwrites a PyBlob's bytes for the duration of a block: what is computed inside may not read the caller's page."""

    def __init__(self, page):
        self.page = page

    def __enter__(self):
        C.memset(self.page.buf, ord(" "), len(self.page._data))

    def __exit__(self, *a):
        C.memmove(self.page.buf, self.page._data, len(self.page._data))


def refresh_and_check(eng, rb, page, docs, kind, process, keep, what, expect_rebuilt=True, oracle=True):
    # (a constraint set the host flattens reads the caller's page, kept source or not)
    with Scrambled(page) if keep and "ingest: device" in eng.drv.Dump() else _Null():
        st = rb.refresh()
    assert st["rebuilt"] == expect_rebuilt, (what, st)
    got = snapshot(rb.eval(k8s.AUDIT_EP))
    fresh = upload(eng, W.PyBlob(docs), docs, kind, process, keep)
    want = snapshot(fresh.eval(k8s.AUDIT_EP))
    fresh.free()
    assert_same_as_fresh(got, want, what)
    if st["rebuilt"]:
        assert st["alg_bytes"] == rb.alg_bytes > 0
    if oracle:
        assert_oracle(eng, docs, got, process, what)
    return got, st


class _Null:
    def __enter__(self):
        pass

    def __exit__(self, *a):
        pass


def case_refresh_steps(lib, kind="blob", keep=True, n=160, process="audit", limit=5):
    """Every kind of change a constraint set goes through, each followed by a refresh of one resident batch: a constraint of a
    loaded template with new parameters and string constants, a template that brings new scopes and columns, a removed constraint,
    a changed spec.match with a namespaceSelector, the excluder of the upload's process, a refresh of a current batch (nothing to
    do), and the audit of the refreshed batch against oracle/audit.py.  With `keep`, the caller's page is overwritten during every
    refresh: the device path must not read it."""
    t = W.templates()
    eng, by_kind = config2_start(lib)
    docs = damaged_page(n)
    page = W.PyBlob(docs)
    rb = upload(eng, page, docs, kind, process, keep)
    got, _ = refresh_and_check(eng, rb, page, docs, kind, process, keep, "nothing changed", expect_rebuilt=False)
    assert got[5] and sum(1 for e in got[5] if e) == len(BAD_DOCS)
    # a constraint of a loaded template with new parameters: string constants the string table has never seen
    eng.constraint(W._constraint("K8sAllowedRepos", "repos-new", match=dict(W.POD), params={"repos": ["never-seen.example/", "gcr.io/proj-0"]}))
    eng.constraint(W._constraint("K8sRequiredLabels", "labels-new", match=dict(W.POD), params={"labels": ["never-seen-label"]}))
    eng.constraint(W._constraint("K8sBannedImageTags", "tags-new", match=dict(W.POD), params={"tags": ["v0.0.1", "never-seen-tag"]}))
    with np.testing.assert_raises_regex(D.GkError, "older constraint set"):
        rb.eval(k8s.AUDIT_EP)
    refresh_and_check(eng, rb, page, docs, kind, process, keep, "new parameters")
    # templates that bring scopes (volumes, probes of every container), columns the batch never had, and lookups the device table
    # has never answered (canonify_cpu / canonify_mem of containerlimits: the host evaluates them from the bytes of the page)
    for name in ("psp_volumetypes", "requiredprobes", "containerlimits"):
        eng.template(t[name]["kind"], t[name]["rego"])
        for c in by_kind[t[name]["kind"]][:2]:
            eng.constraint(c)
    refresh_and_check(eng, rb, page, docs, kind, process, keep, "new templates")
    # a removed constraint
    eng.remove_constraint("K8sAllowedRepos", by_kind["K8sAllowedRepos"][0]["metadata"]["name"])
    refresh_and_check(eng, rb, page, docs, kind, process, keep, "a removed constraint")
    # a changed spec.match, now with a namespaceSelector
    c = json.loads(json.dumps(by_kind["K8sContainerLimits"][0]))
    c["spec"]["match"] = dict(W.POD, namespaceSelector={"matchExpressions": [{"key": "env", "operator": "In", "values": ["prod"]}]})
    eng.constraint(c)
    refresh_and_check(eng, rb, page, docs, kind, process, keep, "a changed spec.match")
    # the excluder of the upload's process (the constraint set's version does not change)
    eng.exclude("audit", ["ns-00*", "*-system"])
    refresh_and_check(eng, rb, page, docs, kind, process, keep, "the excluder", expect_rebuilt=process == "audit")
    # refreshed twice in a row: the second call has nothing to do
    refresh_and_check(eng, rb, page, docs, kind, process, keep, "a second refresh", expect_rebuilt=False, oracle=False)
    # the audit of the refreshed batch
    run = D.AuditRun(eng.drv, violations_limit=limit)
    run.add_batch(rb, k8s.AUDIT_EP)
    rep = run.report()
    run.close()
    objs = [json.loads(d) for d in docs if d not in BAD_DOCS]
    want = OA.audit(eng.orc, objs, namespaces={x["metadata"]["name"]: x for x in eng.nss}, excluded_namespaces=eng.excluded.get(process, ()) if process else (),
                    limit=limit)
    assert rep["totalViolations"] == {"%s/%s" % k: v for k, v in want["totals"].items()}
    assert rep["totalViolationsPerEnforcementAction"] == want["by_action"]
    for key, lst in want["violations"].items():
        w = [{k: v for k, v in sv.items() if not (k in ("namespace", "enforcementActions") and not v)} for sv in lst]
        assert rep["violations"]["%s/%s" % key] == w, key
    assert sum(rep["totalViolations"].values()) > 0
    rb.free()
    eng.close()
    return rep


def case_refresh_referential(lib, keep=True, n=120):
    """A referential constraint (data.inventory) moves the snapshot to the host flattener: the refresh flattens the page on the host;
    a change of data.inventory makes the batch stale again, and a refresh brings it back; without the referential template the
    snapshot is flattened on the device again, from the kept source when there is one."""
    v = golden("referential_vectors.json")["uniquelabel"]
    eng, _ = config2_start(lib, per_template=1)
    cms = [dict(d) for d in v["synced"]] + [v["denied"]]
    cms += [{"apiVersion": "v1", "kind": "ConfigMap", "metadata": {"name": "cm-%d" % i, "namespace": "gatekeeper-test-playground",
                                                                      "labels": {"gatekeeper": "v%d" % (i % 7)}}} for i in range(12)]
    docs = [json.dumps(d).encode() for d in cms] + damaged_page(n, start=52000)
    page = W.PyBlob(docs)
    rb = upload(eng, page, docs, "blob", "", keep)
    kind, rego, *_ = k8s.template_from_yaml_obj(v["template"])
    eng.template(kind, rego)
    eng.constraint(v["constraint"])
    for d in v["synced"]:
        eng.data(d)
    assert "ingest: device" not in eng.drv.Dump()
    got, _ = refresh_and_check(eng, rb, page, docs, "blob", "", False, "a referential constraint")
    assert any(k.startswith("K8sUniqueLabel/") for k in got[0])
    for i in range(3):
        eng.data(cms[3 + i])
    with np.testing.assert_raises_regex(D.GkError, "data.inventory changed"):
        rb.eval(k8s.AUDIT_EP)
    got, _ = refresh_and_check(eng, rb, page, docs, "blob", "", False, "new data.inventory")
    assert sum(got[3]) > 0
    eng.drv.RemoveTemplate(kind)
    eng.orc = _without_kind(eng, kind)
    assert "ingest: device" in eng.drv.Dump()
    refresh_and_check(eng, rb, page, docs, "blob", "", keep, "the referential template removed")
    rb.free()
    eng.close()


def _without_kind(eng, kind):
    """The oracle rebuilt without the constraints of `kind` (it has no template removal)."""
    orc = k8s.Client()
    for ns in eng.nss:
        orc.add_namespace(ns)
        orc.add_data(ns)
    t = W.templates()
    tm, cons = W.config2()
    for name in FIRST:
        orc.add_template(t[name]["kind"], t[name]["rego"])
    seen = set()
    for c in cons:
        if c["kind"] not in seen:
            seen.add(c["kind"])
            if c["kind"] in {t[x]["kind"] for x in FIRST}:
                orc.add_constraint(c)
    return orc


def case_refresh_failure_leaves_batch(lib, n=64, volumes=400000):
    """A refresh that fails leaves the batch as it was: one object whose own volumes overflow a 32-object tile of an evaluation that
    iterates them is refused when the batch is laid out in tiles, before any launch.  The batch stays on its old constraint set
    (eval() still refuses it as stale); with the constraint removed, a later refresh succeeds."""
    t = W.templates()
    eng, _ = config2_start(lib, per_template=1)
    docs = damaged_page(n, start=61000)
    big = json.loads(W.synth_objects(61000 + n, 1).get(0))
    big["spec"]["volumes"] = [{"name": "v%d" % i, "emptyDir": {}} for i in range(volumes)]
    docs.insert(n // 2, json.dumps(big, separators=(",", ":")).encode())
    page = W.PyBlob(docs)
    rb = upload(eng, page, docs, "blob", "", True)
    before = snapshot(rb.eval(k8s.AUDIT_EP))
    eng.template(t["psp_volumetypes"]["kind"], t["psp_volumetypes"]["rego"])
    c = W._constraint(t["psp_volumetypes"]["kind"], "volumes", match=dict(W.POD), params={"volumes": ["configMap", "secret"]})
    eng.constraint(c)
    with np.testing.assert_raises_regex(D.GkError, "slot area|shared memory|tile"):
        rb.refresh()
    with np.testing.assert_raises_regex(D.GkError, "older constraint set"):
        rb.eval(k8s.AUDIT_EP)
    eng.remove_constraint(c["kind"], "volumes")
    st = rb.refresh()
    assert st["rebuilt"]
    got = snapshot(rb.eval(k8s.AUDIT_EP))
    assert_same_as_fresh(got, before, "a failed refresh and the constraint removed")
    rb.free()
    eng.close()


def case_refresh_with_prefetch(lib, n=300):
    """The next page streamed in (gk_blob_prefetch) while a kept-source batch is refreshed: both pages' results are those of fresh
    uploads and of the oracle."""
    t = W.templates()
    eng, by_kind = config2_start(lib)
    docs_a, docs_b = damaged_page(n, start=70000, seed=3), damaged_page(n, start=80000, seed=4)
    page_a, page_b = W.PyBlob(docs_a), W.PyBlob(docs_b)
    rb_a = upload(eng, page_a, docs_a, "blob", "", True)
    eng.template(t["psp_volumetypes"]["kind"], t["psp_volumetypes"]["rego"])
    eng.constraint(by_kind[t["psp_volumetypes"]["kind"]][0])
    eng.drv.prefetch_blob(page_b)
    with Scrambled(page_a):
        assert rb_a.refresh()["rebuilt"]
    rb_b = upload(eng, page_b, docs_b, "blob", "", True)
    for rb, docs in ((rb_a, docs_a), (rb_b, docs_b)):
        got = snapshot(rb.eval(k8s.AUDIT_EP))
        fresh = upload(eng, W.PyBlob(docs), docs, "blob", "", False)
        assert_same_as_fresh(got, snapshot(fresh.eval(k8s.AUDIT_EP)), "a refresh between a prefetch and its upload")
        fresh.free()
        assert_oracle(eng, docs, got, "", "a refresh between a prefetch and its upload")
    # the other way round: a refresh of page b while page a streams in again
    eng.constraint(by_kind[t["psp_volumetypes"]["kind"]][1])
    eng.drv.prefetch_blob(page_a)
    with Scrambled(page_b):
        assert rb_b.refresh()["rebuilt"]
    rb_a2 = upload(eng, page_a, docs_a, "blob", "", False)   # (the prefetched copy)
    with Scrambled(page_a):
        assert rb_a.refresh()["rebuilt"]
    fresh_b = upload(eng, W.PyBlob(docs_b), docs_b, "blob", "", False)
    assert_same_as_fresh(snapshot(rb_b.eval(k8s.AUDIT_EP)), snapshot(fresh_b.eval(k8s.AUDIT_EP)), "a refresh during a prefetch")
    got_a = snapshot(rb_a.eval(k8s.AUDIT_EP))
    assert_same_as_fresh(got_a, snapshot(rb_a2.eval(k8s.AUDIT_EP)), "a refresh after a prefetched upload")
    assert_oracle(eng, docs_a, got_a, "", "a refresh after a prefetched upload")
    for rb in (rb_a, rb_b, rb_a2, fresh_b):
        rb.free()
    eng.close()
