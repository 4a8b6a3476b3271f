"""The audit of expanded batches (GK_F_EXPAND): the cases test_audit_expand_hostemu.py runs on the test-only host emulation and
test_audit_expand.py on the GPU.  An expanded batch whose templates are current brings its resultants to gk_audit_add_batch(_ordered):
they are neither expanded nor uploaded again, and their pairs are sorted against the parents' candidates.  Every case builds each page
twice, uploaded with GK_F_EXPAND and without it, and requires the two audits' reports to be byte-identical, counters included, and
equal to oracle/audit.py with the expansion system.  `lib`: the host emulation's library, or None for the product library."""
import copy
import ctypes as C
import json
import random

import audit_order_cases as A
import test_capi_entry_points as T
from conftest import golden, make_pair
import expand_sweep_cases as S
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import audit as OA
from oracle import expansion as X
from oracle import k8s

EP = k8s.AUDIT_EP
EXCLUDED = ("kube-*",)
FROM_BATCH = "taken from the expanded batch"
ON_HOST = "on the host:"


def engine(lib):
    """Pods (several results per pair: one per container), Generated Pods, a scoped constraint, Deployments, every kind, and a namespaceSelector
    whose objects in namespaces outside the cache are matcher errors; the three templates of test_capi_entry_points (a chain
    CronJob -> Job -> Pod, and a dryrun override); the audit's excluder skips kube-*."""
    t = golden("templates.json")
    tm = [(t[k]["kind"], t[k]["rego"]) for k in ("allowedrepos", "psp_privileged", "requiredlabels_basic")]
    rl = t["requiredlabels_basic"]["kind"]
    cons = S.constraints(t)
    # (every kind: flags parents and resultants alike, so that a resultant's pair can lie above its parents' threshold and be counted)
    cons.append(W._constraint(rl, "owner", params={"labels": ["owner"]}))
    cons.append(W._constraint(rl, "selected", params={"labels": ["cost"]},
                              match={"kinds": [{"apiGroups": [""], "kinds": ["Pod"]}], "namespaceSelector": {"matchLabels": {"env": "prod"}}}))
    nss = W.synth_namespaces()
    orc, drv, skipped = make_pair(tm, cons, nss, lib_path=lib)
    assert not skipped
    xs = X.System()
    for d in T.EXPANSION:
        xs.upsert(d)
        drv.AddExpansionTemplate(d)
    drv.SetExcludedNamespaces("audit", list(EXCLUDED))
    return orc, drv, xs, {x["metadata"]["name"]: x for x in nss}


def page(n_pods=300, seed=21, extra=True):
    """test_capi_entry_points' review page without its DELETE, plus parents that tie on namespace and name, generators in an
    excluded namespace, and an object with neither apiVersion nor kind (its own review fails; it is not expanded)."""
    objs = [r.object for r in T._review_page(n_pods=n_pods, seed=seed) if r.object is not None and not r.operation]
    if not extra:
        return objs
    rnd = random.Random(seed)
    nsn = [x["metadata"]["name"] for x in W.synth_namespaces()]
    for j in range(6):
        spec = copy.deepcopy([T.PRIV_POD, T.GOOD_POD][j % 2])
        spec["spec"]["containers"].append({"name": "d", "image": "docker.io/x:%d" % j, "securityContext": {"privileged": j % 3 == 0}})
        for kind in ("Deployment", "ReplicaSet"):
            objs.append({"apiVersion": "apps/v1", "kind": kind, "metadata": {"name": "tie", "namespace": nsn[0]}, "spec": {"template": spec}})
    for j in range(4):
        objs.append({"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "sys-%d" % j, "namespace": "kube-system"},
                     "spec": {"template": T.PRIV_POD}})
    objs.append({"metadata": {"name": "no-gvk", "namespace": nsn[1]}, "spec": {"template": T.PRIV_POD}})
    rnd.shuffle(objs)
    return objs


def upload(drv, objs, kind, expand):
    """One page as review objects ("objs"), a raw-JSON blob ("blob") or a blob with its kept source ("kept")."""
    if kind == "objs":
        return drv.upload([D.Review(object=o, source="Original") for o in objs], process="audit", expand=expand)
    blob = W.PyBlob([json.dumps(o).encode() for o in objs])
    rb = drv.upload_blob(blob, process="audit", keep_source=kind == "kept", expand=expand)
    rb._blob = blob
    return rb


def raw_report(run):
    err = C.c_char_p()
    p = run.drv._lib.gk_audit_report(run._a, C.byref(err))
    assert p, err.value
    try:
        return C.string_at(p)
    finally:
        run.drv._lib.gk_free_str(p)


def audit(drv, batches, limit, ordered):
    """(raw report, resultant pairs, trace lines) of one run over `batches`."""
    run = D.AuditRun(drv, violations_limit=limit)
    with S.launch_trace() as lines:
        for rb in batches:
            (run.add_batch_ordered if ordered else run.add_batch)(rb, EP)
    out = raw_report(run), run.resultant_pairs(), [l for l in lines if l.startswith("[audit]")]
    run.close()
    return out


def resultant_pairs(orc, xs, objs, nsmap):
    """(violation pairs, matcher-error pairs) of the resultants the oracle reviews: one per (resultant, constraint) with a result."""
    viol = errs = 0
    for o in objs:
        if k8s.is_namespace_excluded(EXCLUDED, o) or not (o.get("apiVersion") or o.get("kind")):
            continue
        ns = nsmap.get(k8s._meta(o, "namespace"))
        try:
            res = xs.expand(o, ns["metadata"]["name"] if ns else None)
        except X.ExpansionError:
            continue
        for robj, _, _ in res:
            if k8s.is_namespace_excluded(EXCLUDED, robj):
                continue
            by = {}
            for r in orc.review(k8s.Review(obj=robj, ns=ns, source="Generated"), EP):
                by[r["constraint"]] = by.get(r["constraint"], False) or bool(r.get("autoreject"))
            errs += sum(by.values())
            viol += len(by) - sum(by.values())
    return viol, errs


def compare(drv, orc, xs, nsmap, objs, kinds=("blob", "kept", "objs"), limits=None, oracle=True):
    """Each kind, each limit, both calls: the expanded batch's report == the plain batch's, byte for byte, and == the oracle's; the
    expanded batch is not expanded again.  Returns {(kind, limit, ordered): resultant pairs} of the expanded runs."""
    out, wants = {}, {}
    good = [o for o in objs if o.get("apiVersion") or o.get("kind")]
    for kind in kinds:
        xb, pb = upload(drv, objs, kind, True), upload(drv, objs, kind, False)
        for limit in limits or (1, 7, 20, 100000):
            for ordered in (False, True):
                rx, pairs, lx = audit(drv, [xb], limit, ordered)
                rp, none, lp = audit(drv, [pb], limit, ordered)
                assert rx == rp, (kind, limit, ordered, _diff(rx, rp))
                assert none == (0, 0)
                assert any(FROM_BATCH in l for l in lx) and not any(ON_HOST in l for l in lx), lx
                assert any(ON_HOST in l for l in lp), lp
                if oracle:
                    if limit not in wants:
                        wants[limit] = OA.audit(orc, good, namespaces=nsmap, excluded_namespaces=EXCLUDED, limit=limit, expansion=xs)
                    A.check_oracle(json.loads(rx), wants[limit])
                out[(kind, limit, ordered)] = pairs
        xb.free()
        pb.free()
    return out


def _diff(a, b):
    a, b = json.loads(a), json.loads(b)
    return {k: (a.get(k), b.get(k)) for k in set(a) | set(b) if a.get(k) != b.get(k)}


# ------------------------------------------------------------------------------------------------ cases
def case_mixed(lib, kinds=("blob", "kept", "objs"), n_pods=300):
    """Mixed kinds, three templates with a chain and an override, identity ties, matcher errors on resultants, multi-result pairs,
    the excluder, a failed expansion and a refused object: every kind, limit and call."""
    orc, drv, xs, nsmap = engine(lib)
    objs = page(n_pods=n_pods)
    pairs = compare(drv, orc, xs, nsmap, objs, kinds)
    viol, errs = resultant_pairs(orc, xs, objs, nsmap)
    assert viol and errs, (viol, errs)
    for (kind, limit, ordered), (ev, ct) in pairs.items():
        assert ev + ct == viol, (kind, limit, ordered, ev, ct, viol)
        if limit == 100000:
            assert ct == 0, (kind, ordered, ct)
    drv.close()


def case_laziness(lib, n_gen=800):
    """A page of many generators at limit 7, of one kind (so that gk_audit_add_batch's host threshold scan runs too): the resultant
    pairs of a constraint that flags more than `limit` parents are counted but for the candidates; those of Pod-only constraints, which
    flag no parent, are all candidates.  Evaluated + counted + matcher-error pairs are the resultants' flagged pairs."""
    orc, drv, xs, nsmap = engine(lib)
    rnd = random.Random(7)
    nsn = list(nsmap)
    objs = []
    for i in range(n_gen):
        spec = copy.deepcopy(T.PRIV_POD if i % 8 == 0 else T.GOOD_POD)
        if i % 4 == 0:   # (two containers: a pair that may have two results, which the ambiguity plane decides)
            spec["spec"]["containers"].append({"name": "d", "image": "docker.io/x", "securityContext": {"privileged": i % 8 == 0}})
        objs.append({"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "g-%d" % rnd.randrange(n_gen // 2),
                     "namespace": rnd.choice(nsn + ["unknown-ns"])}, "spec": {"template": spec}})
    viol, errs = resultant_pairs(orc, xs, objs, nsmap)
    assert errs > 0
    pairs = compare(drv, orc, xs, nsmap, objs, kinds=("blob",), limits=(7,))
    for ordered in (False, True):
        ev, ct = pairs[("blob", 7, ordered)]
        assert ct > 0 and ev < 0.5 * viol, (ordered, ev, ct, viol)
        assert ev + ct == viol, (ordered, ev, ct, viol, errs)
    drv.close()
    return pairs


def case_stale_then_refresh(lib, kind):
    """A batch whose templates changed is expanded on the host as before (the trace shows it); after gk_batch_refresh its resultants
    come from the batch again.  Both audits equal the plain batch's."""
    orc, drv, xs, nsmap = engine(lib)
    objs = page(n_pods=120, seed=5)
    xb, pb = upload(drv, objs, kind, True), upload(drv, objs, kind, False)
    extra = T._expansion_template("expand-statefulsets", ["StatefulSet"], ("", "v1", "Pod"))
    drv.AddExpansionTemplate(extra)
    xs.upsert(extra)
    objs.append({"apiVersion": "apps/v1", "kind": "StatefulSet", "metadata": {"name": "ss", "namespace": list(nsmap)[0]}, "spec": {"template": T.PRIV_POD}})
    for limit in (1, 7):
        for ordered in (False, True):
            rx, pairs, lx = audit(drv, [xb], limit, ordered)
            rp, _, _ = audit(drv, [pb], limit, ordered)
            assert rx == rp and pairs == (0, 0)
            assert any(ON_HOST in l for l in lx) and not any(FROM_BATCH in l for l in lx), lx
    assert xb.refresh()["rebuilt"] is True
    for limit in (1, 7):
        for ordered in (False, True):
            rx, _, lx = audit(drv, [xb], limit, ordered)
            rp, _, _ = audit(drv, [pb], limit, ordered)
            assert rx == rp
            assert any(FROM_BATCH in l for l in lx) and not any(ON_HOST in l for l in lx), lx
    xb.free()
    pb.free()
    drv.close()


def case_patched(lib):
    """A kept-source expanded page patched (generators dropped and added): its audit equals the plain upload of the patched page."""
    orc, drv, xs, nsmap = engine(lib)
    objs = page(n_pods=150, seed=8)
    xb = upload(drv, objs, "kept", True)
    rnd = random.Random(3)
    drop = sorted(rnd.sample(range(len(objs)), 40))
    add = [{"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "new-%d" % i, "namespace": list(nsmap)[i % 3]},
            "spec": {"template": [T.PRIV_POD, T.GOOD_POD][i % 2]}} for i in range(25)]
    xb.patch(drop, [json.dumps(o).encode() for o in add])
    dropped = set(drop)
    now = [o for i, o in enumerate(objs) if i not in dropped] + add
    pb = upload(drv, now, "blob", False)
    good = [o for o in now if o.get("apiVersion") or o.get("kind")]
    for limit in (1, 7, 20):
        for ordered in (False, True):
            rx, _, lx = audit(drv, [xb], limit, ordered)
            rp, _, _ = audit(drv, [pb], limit, ordered)
            assert rx == rp, (limit, ordered, _diff(rx, rp))
            assert any(FROM_BATCH in l for l in lx), lx
            A.check_oracle(json.loads(rx), OA.audit(orc, good, namespaces=nsmap, excluded_namespaces=EXCLUDED, limit=limit, expansion=xs))
    xb.free()
    pb.free()
    drv.close()


def case_shards_merge(lib, kind, limit=4):
    """Two ranks' exports of expanded shards merged == the merge of the plain shards' exports == one run over the whole page."""
    orc, drv, xs, nsmap = engine(lib)
    objs = page(n_pods=200, seed=13)
    half = len(objs) // 2
    reps = []
    for expand in (True, False):
        merged = D.AuditRun(drv, violations_limit=limit)
        keep = []
        for part in (objs[:half], objs[half:]):
            rb = upload(drv, part, kind, expand)
            keep.append(rb)
            run = D.AuditRun(drv, violations_limit=limit)
            run.add_batch_ordered(rb, EP)
            merged.merge(run.export())
            run.close()
        reps.append(raw_report(merged))
        merged.close()
        for rb in keep:
            rb.free()
    assert reps[0] == reps[1], _diff(reps[0], reps[1])
    good = [o for o in objs if o.get("apiVersion") or o.get("kind")]
    A.check_oracle(json.loads(reps[0]), OA.audit(orc, good, namespaces=nsmap, excluded_namespaces=EXCLUDED, limit=limit, expansion=xs))
    drv.close()
