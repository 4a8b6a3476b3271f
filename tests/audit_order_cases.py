"""Shared cases of gk_audit_add_batch_ordered and of exporting / merging audit runs, run on the GPU by test_audit_order.py and on the
test-only host emulation by test_audit_order_hostemu.py.

add_batch_ordered takes the lazy path's candidates from Backend::audit_candidates: the flagged objects at or below the limit-th
smallest (group, version, kind, namespace, name), ties included, for any mix of kinds.  Every case compares its report with
oracle/audit.py and with add_batch's report, field for field except the two pair counters."""
import json
import random

from conftest import golden, make_pair
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import audit as OA
from oracle import k8s

PAIR_COUNTERS = ("pairsEvaluated", "pairsCounted")


def strip(rep):
    return {k: v for k, v in rep.items() if k not in PAIR_COUNTERS}


def check_oracle(rep, want):
    assert rep["totalViolations"] == {"%s/%s" % k: v for k, v in want["totals"].items()}, (rep["totalViolations"], want["totals"])
    assert rep["totalViolationsPerEnforcementAction"] == want["by_action"]
    assert set(rep["violations"]) == {"%s/%s" % k for k in want["violations"]}
    for key, lst in want["violations"].items():
        g = rep["violations"]["%s/%s" % key]
        w = [{k: v for k, v in sv.items() if not (k in ("namespace", "enforcementActions") and not v)} for sv in lst]
        assert g == w, (key, g[:3], w[:3])


def dumps(o, escape=False):
    """JSON of one object; with `escape`, a name with a '/' spelt '\\/' (the same decoded string)."""
    s = json.dumps(o)          # (ensure_ascii: non-ASCII names and namespaces arrive as \\u escapes)
    if escape:
        s = s.replace('"name": "slash/ed"', '"name": "slash\\/ed"')
    return s.encode()


def upload(drv, objs, kind, page=None, raw=None):
    """Resident batches of `objs` (host-flattened "objs" or raw-JSON "blob"), `page` objects each; `raw` replaces the JSON of some
    objects in blob mode (undecodable ones).  Returns [(keepalive, batch)]."""
    out = []
    page = page or max(1, len(objs))
    for lo in range(0, len(objs), page):
        chunk = objs[lo:lo + page]
        if kind == "objs":
            out.append((None, drv.upload([D.Review(object=o, source="Original") for o in chunk], process="audit")))
        else:
            pb = W.PyBlob([(raw or {}).get(lo + i) or dumps(o, escape=(lo + i) % 7 == 3) for i, o in enumerate(chunk)])
            out.append((pb, drv.upload_blob(pb, process="audit")))
    return out


def run_both(drv, batches, limit):
    plain, ordered = D.AuditRun(drv, violations_limit=limit), D.AuditRun(drv, violations_limit=limit)
    for _, rb in batches:
        plain.add_batch(rb, k8s.AUDIT_EP)
        ordered.add_batch_ordered(rb, k8s.AUDIT_EP)
    return plain.report(), ordered.report()


# ------------------------------------------------------------------------------------------------ hand-made mixed pages
def mixed_engine(lib):
    t = golden("templates.json")
    tm = [(t[k]["kind"], t[k]["rego"]) for k in ("requiredlabels_basic", "allowedrepos")]
    rl, ar = t["requiredlabels_basic"]["kind"], t["allowedrepos"]["kind"]
    cons = [W._constraint(rl, "team-owner", params={"labels": ["team", "owner"]}),
            W._constraint(rl, "app", params={"labels": ["app"]}, action="warn"),
            W._constraint(rl, "tier-scoped", params={"labels": ["tier"]}, action="scoped",
                          scoped=[{"action": "warn", "enforcementPoints": [{"name": k8s.AUDIT_EP}]}]),
            # a namespaceSelector: objects of namespaces missing from the cache are matcher errors (autoreject), always evaluated
            W._constraint(rl, "selected", params={"labels": ["cost"]}, match={"namespaceSelector": {"matchLabels": {"env": "prod"}}}),
            W._constraint(ar, "repos", params={"repos": ["gcr.io/"]})]
    nss = W.synth_namespaces()
    orc, drv, _ = make_pair(tm, cons, nss, lib_path=lib)
    return orc, drv, nss


def mixed_objects(nss, n_extra=300, seed=3):
    rnd = random.Random(seed)
    nsn = [x["metadata"]["name"] for x in nss]
    kinds = [("v1", "Pod"), ("v1", "ConfigMap"), ("v1", "Service"), ("apps/v1", "Deployment"), ("apps/v1beta1", "Deployment"),
             ("batch/v1", "Job"), ("example.com/v1", "Pod"), ("v2", "Pod"), ("rbac.authorization.k8s.io/v1", "ClusterRole"), ("v1", "Node")]
    cluster_scoped = {"ClusterRole", "Node"}
    long = "x" * 200

    def labels():
        return {k: "v" for k in ("team", "owner", "app", "tier", "cost") if rnd.random() < 0.45}

    def obj(api, kind, name, ns, lab=None, image=None):
        o = {"apiVersion": api, "kind": kind, "metadata": {"name": name, "labels": lab if lab is not None else labels()}}
        if ns is not None:
            o["metadata"]["namespace"] = ns
        if kind == "Pod":
            o["spec"] = {"containers": [{"name": "c%d" % j, "image": image or rnd.choice(["gcr.io/a:1", "docker.io/b:2", "quay.io/c"])}
                                        for j in range(rnd.randint(1, 3))]}
        return o

    objs = []
    # the same namespace / name under every kind, group and version
    for api, kind in kinds:
        for name in ("a", "same", "zz"):
            objs.append(obj(api, kind, name, None if kind in cluster_scoped else nsn[0]))
    # Namespace objects (their own namespace is empty), cluster-scoped and namespaced objects of one name
    for nm in nsn[:4] + ["unknown-ns"]:
        objs.append(obj("v1", "Namespace", nm, None))
    # identities that differ only after a long common prefix; names with characters JSON escapes
    for j in range(6):
        objs.append(obj("v1", "Pod", long + "%d" % (5 - j), nsn[1]))
        objs.append(obj("v1", "ConfigMap", long + chr(0x61 + j), long[:150] + "-ns"))
    for nm in ("naïve-é", "tab\there", "quote\"d", "slash/ed", "ünï", "☃-snow"):
        objs.append(obj("v1", "Pod", nm, nsn[2]))
        objs.append(obj("apps/v1", "Deployment", nm, nsn[2]))
    # exact identity ties whose messages differ (other label sets, other images)
    for j in range(5):
        objs.append(obj("v1", "Pod", "tie", nsn[0], lab={"app": "x"} if j % 2 else {}, image=["docker.io/%d" % j, "gcr.io/ok"][j % 2]))
        objs.append(obj("apps/v1", "Deployment", "tie", nsn[0], lab={"team": str(j)} if j % 2 else {}))
    # namespaces outside the cache (matcher errors) and the excluded process namespace
    for j in range(8):
        objs.append(obj("v1", "Pod", "lost-%d" % j, "unknown-ns"))
        objs.append(obj("v1", "ConfigMap", "sys-%d" % j, "kube-system"))
    for i in range(n_extra):
        api, kind = rnd.choice(kinds)
        objs.append(obj(api, kind, "o-%04d" % rnd.randrange(n_extra // 2), None if kind in cluster_scoped else rnd.choice(nsn + [nsn[0]] * 3)))
    rnd.shuffle(objs)
    return objs


def case_mixed_page(lib, kind, limit, page=None):
    """Hand-made pages of many kinds: add_batch_ordered == add_batch == the oracle; the lazy path counts pairs on the mixed page."""
    orc, drv, nss = mixed_engine(lib)
    excluded = ("kube-*",)
    drv.SetExcludedNamespaces("audit", list(excluded))
    objs = mixed_objects(nss)
    raw = {}
    if kind == "blob":      # undecodable objects: object errors, never candidates
        raw = {5: b'{"apiVersion": "v1", "kind": "Pod", "metadata": {"name": ', 40: b'[1, 2]'}
    keep = upload(drv, objs, kind, page, raw)
    plain, ordered = run_both(drv, keep, limit)
    assert strip(plain) == strip(ordered)
    good = [o for i, o in enumerate(objs) if i not in raw]
    want = OA.audit(orc, good, namespaces={x["metadata"]["name"]: x for x in nss}, excluded_namespaces=excluded, limit=limit)
    check_oracle(ordered, want)
    assert ordered["objectErrors"]["count"] == len(raw)
    flagged = sum(want["totals"].values())
    assert plain["pairsCounted"] == 0              # (a page of several kinds: add_batch evaluates every flagged pair)
    if limit < 100:
        assert ordered["pairsCounted"] > 0
        assert ordered["pairsEvaluated"] < 0.6 * flagged, (ordered["pairsEvaluated"], flagged)
    else:                                          # (more room than violators: every flagged pair is a candidate)
        assert ordered["pairsCounted"] == 0
    return plain, ordered


def case_config4_page(lib, kind, n=3000, limit=20):
    """Config 4's constraint set over a page of its mixed objects (synth mode 1)."""
    tm, cons = W.config4()
    nss = W.synth_namespaces()
    orc, drv, _ = make_pair(tm, cons, nss, lib_path=lib)
    blob = W.synth_objects(0, n, mode=1)
    objs = [json.loads(blob.get(i)) for i in range(n)]
    assert len({(o["apiVersion"], o["kind"]) for o in objs}) > 1
    keep = upload(drv, objs, kind) if kind == "objs" else [(blob, drv.upload_blob(blob))]
    plain, ordered = run_both(drv, keep, limit)
    assert strip(plain) == strip(ordered)
    want = OA.audit(orc, objs, namespaces={x["metadata"]["name"]: x for x in nss}, limit=limit)
    check_oracle(ordered, want)
    flagged = sum(want["totals"].values())
    assert plain["pairsCounted"] == 0 and ordered["pairsCounted"] > 0
    assert ordered["pairsEvaluated"] < 0.5 * flagged, (ordered["pairsEvaluated"], flagged)
    return ordered


def case_expansion(lib, kind, limit=3):
    """A run with ExpansionTemplates registered: resultants fold into their parents as in add_batch; failed expansions are reported."""
    from oracle import expansion as X
    t = golden("templates.json")
    tm = [(t[k]["kind"], t[k]["rego"]) for k in ("psp_privileged", "requiredlabels_basic")]
    cons = [W._constraint(t["psp_privileged"]["kind"], "priv", match=dict(W.POD)),
            W._constraint(t["requiredlabels_basic"]["kind"], "team", params={"labels": ["team"]})]
    nss = W.synth_namespaces()
    orc, drv, _ = make_pair(tm, cons, nss, lib_path=lib)
    xs = X.System()
    d = {"apiVersion": "expansion.gatekeeper.sh/v1alpha1", "kind": "ExpansionTemplate", "metadata": {"name": "expand-deployments"},
         "spec": {"applyTo": [{"groups": ["apps"], "versions": ["v1"], "kinds": ["Deployment"]}], "templateSource": "spec.template",
                  "generatedGVK": {"group": "", "version": "v1", "kind": "Pod"}}}
    xs.upsert(d)
    drv.AddExpansionTemplate(d)
    nsn = [x["metadata"]["name"] for x in nss]
    rnd = random.Random(4)
    objs = []
    for i in range(120):
        priv = {"metadata": {"labels": {}}, "spec": {"containers": [{"name": "c", "image": "a", "securityContext": {"privileged": rnd.random() < 0.6}}]}}
        if i % 3 == 0:
            objs.append({"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "d-%d" % (i % 17), "namespace": rnd.choice(nsn),
                         **({"labels": {"team": "t"}} if i % 2 else {})}, "spec": {"template": priv}})
        else:
            objs.append({"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "p-%d" % (i % 23), "namespace": rnd.choice(nsn)}, "spec": priv["spec"]})
    objs.append({"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "bad", "namespace": nsn[0]}, "spec": {"template": "nope"}})
    rnd.shuffle(objs)
    keep = upload(drv, objs, kind)
    plain, ordered = run_both(drv, keep, limit)
    assert strip(plain) == strip(ordered)
    want = OA.audit(orc, objs, namespaces={x["metadata"]["name"]: x for x in nss}, limit=limit, expansion=xs)
    check_oracle(ordered, want)
    assert ordered["objectErrors"]["count"] == len(want["expand_errors"]) == 1
    return ordered


# ------------------------------------------------------------------------------------------------ candidate exactness
def case_candidates_exact(lib, kind, seed, limit):
    """Random identities and bitmaps over constraints that have one result per pair: the pairs evaluated on the host are exactly the
    candidates computed here -- per constraint, the flagged objects at or below the limit-th smallest identity, ties included."""
    t = golden("templates.json")
    rl = t["requiredlabels_basic"]["kind"]
    labs = ["l%d" % j for j in range(6)]
    cons = [W._constraint(rl, "need-%s" % l, params={"labels": [l]}) for l in labs]
    orc, drv, _ = make_pair([(rl, t["requiredlabels_basic"]["rego"])], cons, lib_path=lib)
    single = {l.split()[2] for l in drv.Dump().splitlines() if l.startswith("constraint ") and "[one result per pair]" in l}
    assert len(single) == len(cons), single
    rnd = random.Random(seed)
    gvks = [("", "v1", "Pod"), ("", "v1", "ConfigMap"), ("apps", "v1", "Deployment"), ("apps", "v1beta2", "Deployment"), ("x.io", "v1", "Pod"),
            ("", "v1", "Namespace")]
    alpha = "abé"
    objs = []
    for i in range(rnd.randint(40, 400)):
        g, v, k = rnd.choice(gvks)
        o = {"apiVersion": (g + "/" if g else "") + v, "kind": k,
             "metadata": {"name": "".join(rnd.choice(alpha) for _ in range(rnd.randint(0, 3))),
                          "labels": {l: "x" for l in labs if rnd.random() < 0.5}}}
        if k != "Namespace" and rnd.random() < 0.8:
            o["metadata"]["namespace"] = "".join(rnd.choice(alpha) for _ in range(rnd.randint(1, 2)))
        objs.append(o)
    keep = upload(drv, objs, kind)
    plain, ordered = run_both(drv, keep, limit)
    assert strip(plain) == strip(ordered)
    want = OA.audit(orc, objs, limit=limit)
    check_oracle(ordered, want)

    def ident(o):
        g, v, k = k8s._gvk(o)
        md = o["metadata"]
        return (g.encode(), v.encode(), k.encode(), ("" if k == "Namespace" and not g else md.get("namespace", "")).encode(), md["name"].encode())

    expect = 0
    for con in cons:
        key = (con["kind"], con["metadata"]["name"])
        flagged = sorted({r["object"] for r in want["results"] if r["constraint"] == key}, key=lambda i: ident(objs[i]))
        if len(flagged) > limit:
            thr = ident(objs[flagged[limit - 1]])
            flagged = [i for i in flagged if ident(objs[i]) <= thr]
        expect += len(flagged)
    assert ordered["pairsEvaluated"] == expect, (ordered["pairsEvaluated"], expect)
    assert ordered["pairsEvaluated"] + ordered["pairsCounted"] == sum(want["totals"].values())


# ------------------------------------------------------------------------------------------------ export / merge
def case_shards_merge(lib, kind, shards, limit=4):
    """Objects split into `shards` contiguous shards, one run each, exported and merged in shard order == one run over all objects,
    object-error indices included."""
    orc, drv, nss = mixed_engine(lib)
    objs = mixed_objects(nss, n_extra=200, seed=11)
    raw = {}
    if kind == "blob":
        raw = {3: b'{"kind": ', 70: b'"str"', len(objs) - 2: b'{]'}
    whole = D.AuditRun(drv, violations_limit=limit)
    keep = upload(drv, objs, kind, raw=raw)
    for _, rb in keep:
        whole.add_batch_ordered(rb, k8s.AUDIT_EP)
    want = whole.report()
    merged = D.AuditRun(drv, violations_limit=limit)
    n = len(objs)
    for s in range(shards):
        lo, hi = n * s // shards, n * (s + 1) // shards
        part = D.AuditRun(drv, violations_limit=limit)
        sub = upload(drv, objs[lo:hi], kind, raw={i - lo: b for i, b in raw.items() if lo <= i < hi})
        for _, rb in sub:
            part.add_batch_ordered(rb, k8s.AUDIT_EP)
        keep += sub
        merged.merge(part.export())
    got = merged.report()
    assert strip(got) == strip(want)
    assert got["objectErrors"]["count"] == len(raw)
    assert [e["object"] for e in got["objectErrors"]["first"]] == sorted(raw)
    return got


def case_export_roundtrip_and_refusals(lib, kind):
    orc, drv, nss = mixed_engine(lib)
    objs = mixed_objects(nss, n_extra=100, seed=5)
    run = D.AuditRun(drv, violations_limit=5, msg_size=64)
    keep = upload(drv, objs, kind)
    for _, rb in keep:
        run.add_batch_ordered(rb, k8s.AUDIT_EP)
    rep = run.report()
    buf = run.export()
    empty = D.AuditRun(drv, violations_limit=5, msg_size=64)
    empty.merge(buf)
    assert empty.report() == rep
    # refusals leave the run as it was
    target = D.AuditRun(drv, violations_limit=5, msg_size=64)
    target.merge(buf)
    bad = [buf[:len(buf) // 2], buf[:-1], b"", buf[:8], bytes(buf[:40]) + bytes([buf[40] ^ 0x10]) + buf[41:],
           buf[:-9] + bytes([buf[-9] ^ 1]) + buf[-8:], buf[:8] + bytes([2, 0, 0, 0]) + buf[12:],
           D.AuditRun(drv, violations_limit=6, msg_size=64).export(), D.AuditRun(drv, violations_limit=5, msg_size=65).export()]
    for b in bad:
        try:
            target.merge(b)
        except D.GkError as e:
            assert "audit merge" in str(e), str(e)
        else:
            raise AssertionError("a bad export was merged: %r" % b[:16])
        assert target.report() == rep
    return rep
