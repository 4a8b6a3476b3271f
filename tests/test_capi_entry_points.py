"""The rules the C entry points share, on the test-only host emulation: the bitmap-only calls refuse to run while ExpansionTemplates
are registered, every call on a resident batch refuses a stale one, a page reviewed in one gk_review_batch expands its generators as
the same page reviewed in admission-sized chunks does, and the audit does not expand an object whose own review failed.  On the host
emulation the "device" output pointers of gk_batch_eval_device* are host memory."""
import json
import random

import numpy as np
import pytest

from conftest import HOSTEMU, golden
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import k8s

T = "admission.k8s.gatekeeper.sh"
EP = k8s.AUDIT_EP
ERR_REGO = -2
PRIV_POD = {"metadata": {"labels": {"app": "x"}},
            "spec": {"containers": [{"name": "c", "image": "evil.example.com/a:latest", "securityContext": {"privileged": True}}]}}
GOOD_POD = {"metadata": {"labels": {"app": "y"}}, "spec": {"containers": [{"name": "c", "image": "gcr.io/a:1"}]}}


def _expansion_template(name, kinds, gen, src="spec.template", action=None, groups=("apps",)):
    spec = {"applyTo": [{"groups": list(groups), "versions": ["v1"], "kinds": kinds}], "templateSource": src,
            "generatedGVK": {"group": gen[0], "version": gen[1], "kind": gen[2]}}
    if action:
        spec["enforcementAction"] = action
    return {"apiVersion": "expansion.gatekeeper.sh/v1alpha1", "kind": "ExpansionTemplate", "metadata": {"name": name}, "spec": spec}


EXPANSION = [_expansion_template("expand-deployments", ["Deployment", "ReplicaSet"], ("", "v1", "Pod")),
             _expansion_template("expand-cronjobs", ["CronJob"], ("batch", "v1", "Job"), src="spec.jobTemplate", groups=("batch",)),
             _expansion_template("expand-jobs", ["Job"], ("", "v1", "Pod"), action="dryrun", groups=("batch",))]


def _engine(threads=0):
    """A driver on the host emulation with three templates, constraints on Pods (one of them on generated Pods only) and on
    Deployments, and the synthetic Namespaces."""
    t = golden("templates.json")
    drv = D.Driver(threads=threads, lib_path=HOSTEMU)
    for k in ("allowedrepos", "psp_privileged", "requiredlabels_basic"):
        drv.add_template(t[k]["kind"], t[k]["rego"])
    for c in (W._constraint(t["allowedrepos"]["kind"], "repos", match=dict(W.POD), params={"repos": ["gcr.io/"]}, action="warn"),
              W._constraint(t["psp_privileged"]["kind"], "priv", match={"kinds": [{"apiGroups": [""], "kinds": ["Pod"]}], "source": "Generated"}),
              W._constraint(t["psp_privileged"]["kind"], "priv-scoped", match=dict(W.POD), action="scoped",
                            scoped=[{"action": "warn", "enforcementPoints": [{"name": EP}]}]),
              W._constraint(t["requiredlabels_basic"]["kind"], "team", match={"kinds": [{"apiGroups": ["apps"], "kinds": ["Deployment"]}]},
                            params={"labels": ["team"]})):
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData(T, ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    return drv


def _bitmap_calls(drv, rb, page):
    """gk_batch_eval, gk_batch_eval_device, gk_batch_eval_device_peers (one rank) and gk_review_blob, each returning its violation
    bitmap.  The output buffers are sized for the constraint set of the moment."""
    def shape():
        n, C = len(rb), len(drv.constraints())
        return n, C, max(1, (C + 31) // 32)

    def device():
        n, C, words = shape()
        viol, err, tot = np.zeros((n, words), np.uint32), np.zeros((n, words), np.uint32), np.zeros((2, C), np.int64)
        rb.eval_device(EP, viol.ctypes.data, err.ctypes.data, tot[0].ctypes.data, tot[1].ctypes.data)
        return viol

    def peers():
        n, C, words = shape()
        tot_off = n * words + (n * words) % 2
        slot = tot_off + 4 * C
        recv, err, tot = np.zeros(slot, np.int32), np.zeros((n, words), np.uint32), np.zeros((2, C), np.int64)
        rb.eval_device_peers(EP, [recv.ctypes.data], 0, slot, tot_off, C, err.ctypes.data, tot[0].ctypes.data, tot[1].ctypes.data)
        return recv[:n * words].view(np.uint32).reshape(n, words)

    return {"gk_batch_eval": lambda: rb.eval(EP).viol_bits, "gk_batch_eval_device": device, "gk_batch_eval_device_peers": peers,
            "gk_review_blob": lambda: drv.ReviewBlob(page, EP, with_results=False).viol_bits}


def _resident_calls(drv, rb, page):
    """The bitmap calls and both audit entry points: every call that takes a resident batch."""
    calls = _bitmap_calls(drv, rb, page)
    del calls["gk_review_blob"]

    def audit(ordered):
        run = D.AuditRun(drv, violations_limit=5)
        try:
            (run.add_batch_ordered if ordered else run.add_batch)(rb, EP)
            return run.report()
        finally:
            run.close()

    calls["gk_audit_add_batch"] = lambda: audit(False)
    calls["gk_audit_add_batch_ordered"] = lambda: audit(True)
    return calls


def _refuses(call, code, text):
    with pytest.raises(D.GkError) as e:
        call()
    assert e.value.code == code and text in str(e.value), (e.value.code, str(e.value))


def test_bitmap_calls_refuse_while_expansion_templates_are_registered():
    drv = _engine()
    page = W.synth_objects(5000, 200)
    rb = drv.upload_blob(page, keep_source=True)
    calls = _bitmap_calls(drv, rb, page)
    want = rb.eval(EP).viol_bits
    assert want.any()
    drv.AddExpansionTemplate(EXPANSION[0])
    for name, call in calls.items():
        _refuses(call, ERR_REGO, "ExpansionTemplates are registered")
    drv.RemoveExpansionTemplate(EXPANSION[0]["metadata"]["name"])
    for name, call in calls.items():
        assert np.array_equal(call(), want), name
    rb.free()
    drv.close()


def test_resident_calls_refuse_a_stale_batch_until_it_is_refreshed():
    drv = _engine()
    page = W.synth_objects(6000, 160)
    rb = drv.upload_blob(page, process="audit", keep_source=True)
    calls = _resident_calls(drv, rb, page)
    for call in calls.values():
        call()
    assert rb.refresh()["rebuilt"] is False

    def stale(text, change):
        change()
        for name, call in calls.items():
            _refuses(call, ERR_REGO, text)
        assert rb.refresh()["rebuilt"] is True
        for call in calls.values():
            call()
        assert rb.refresh()["rebuilt"] is False

    t = golden("templates.json")
    stale("older constraint set", lambda: drv.AddConstraint(W._constraint(t["allowedrepos"]["kind"], "repos-2", match=dict(W.POD),
                                                                           params={"repos": ["docker.io/"]})))
    # a referential snapshot: its columns hold values computed from data.inventory
    v = golden("referential_vectors.json")["uniquelabel"]
    orc = k8s.Client()
    kind, rego, *_ = k8s.template_from_yaml_obj(v["template"])

    def referential():
        drv.add_template(kind, rego)
        drv.AddConstraint(v["constraint"])
        for d in v["synced"]:
            drv.AddData(T, orc.data_path(d), d)

    stale("older constraint set", referential)
    stale("data.inventory changed", lambda: drv.AddData(T, orc.data_path(v["denied"]), v["denied"]))
    rb.free()
    drv.close()


def _review_page(n_pods=520, seed=21):
    """Synthetic Pods, then Deployments, ReplicaSets and CronJobs in random namespaces, two generators whose expansion fails, and a
    DELETE of a Deployment (its generator is the old object), shuffled."""
    rnd = random.Random(seed)
    blob = W.synth_objects(9000, n_pods)
    revs = [D.Review(object=json.loads(blob.get(i)), source="Original") for i in range(n_pods)]
    nsn = [x["metadata"]["name"] for x in W.synth_namespaces()]
    for i in range(90):
        ns, spec = rnd.choice(nsn + ["unknown-ns"]), rnd.choice([PRIV_POD, PRIV_POD, GOOD_POD])
        kind = rnd.choice(["Deployment", "ReplicaSet", "CronJob"])
        if kind == "CronJob":
            o = {"apiVersion": "batch/v1", "kind": "CronJob", "metadata": {"name": "cj-%d" % i, "namespace": ns},
                 "spec": {"jobTemplate": {"spec": {"template": spec}}}}
        else:
            o = {"apiVersion": "apps/v1", "kind": kind, "metadata": {"name": "%s-%d" % (kind.lower(), i), "namespace": ns,
                                                                     **({"labels": {"team": "a"}} if i % 3 else {})},
                 "spec": {"replicas": 1, "template": spec}}
        revs.append(D.Review(object=o, source="Original"))
    revs.append(D.Review(object={"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "no-template", "namespace": nsn[0]},
                                 "spec": {"replicas": 1}}, source="Original"))
    revs.append(D.Review(object={"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "bad-template", "namespace": nsn[1]},
                                 "spec": {"template": "nope"}}, source="Original"))
    gone = {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "gone", "namespace": nsn[2]}, "spec": {"template": PRIV_POD}}
    revs.append(D.Review(object=None, old_object=gone, operation="DELETE", source="Original"))
    rnd.shuffle(revs)
    return revs


def _results(resp, offset=0):
    return [(r.object + offset, r.constraint, r.msg, json.dumps(r.details, sort_keys=True), r.enforcement_action,
             tuple(r.scoped_enforcement_actions), r.autoreject) for r in resp.results]


def test_review_expands_a_large_page_as_its_chunks():
    drv = _engine(threads=4)
    for d in EXPANSION:
        drv.AddExpansionTemplate(d)
    revs = _review_page()
    assert len(revs) >= 600
    whole = drv.ReviewBatch(revs, EP)
    res, viol, err, oerr, tot, etot = [], [], [], [], np.zeros(len(whole.totals), np.int64), np.zeros(len(whole.totals), np.int64)
    for lo in range(0, len(revs), 64):
        part = drv.ReviewBatch(revs[lo:lo + 64], EP)
        assert part.constraints == whole.constraints
        res += _results(part, lo)
        viol.append(part.viol_bits)
        err.append(part.err_bits)
        oerr += part.object_errors or [None] * part.n_objects
        tot += part.totals
        etot += part.err_totals
    got = _results(whole)
    assert got == res
    assert any(r[2].startswith("[Implied by expand-jobs] ") and r[4] == "dryrun" for r in got)
    assert any(r[2].startswith("[Implied by expand-deployments] ") for r in got)
    assert np.array_equal(whole.viol_bits, np.concatenate(viol)) and np.array_equal(whole.err_bits, np.concatenate(err))
    assert whole.totals == tot.tolist() and whole.err_totals == etot.tolist()
    assert whole.object_errors == oerr
    assert sum(1 for e in oerr if e and e.startswith("unable to expand object: ")) == 2
    drv.close()


@pytest.mark.parametrize("ordered", [False, True])
def test_audit_does_not_expand_an_object_whose_review_failed(ordered):
    """A generator whose own review fails (its old object is not JSON) is neither expanded nor reported with an expansion error: it
    reports its own error, and neither its bad template nor its privileged resultant shows."""
    drv = _engine()
    for d in EXPANSION:
        drv.AddExpansionTemplate(d)
    nsn = [x["metadata"]["name"] for x in W.synth_namespaces()]
    dep = lambda name, tmpl: {"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": name, "namespace": nsn[0]}, "spec": {"template": tmpl}}
    blob = W.synth_objects(7000, 40)
    revs = [D.Review(object=json.loads(blob.get(i)), source="Original") for i in range(40)]
    revs.insert(5, D.Review(object=dep("unreviewed-bad", "nope"), old_object=b'{"kind":', source="Original"))
    revs.insert(9, D.Review(object=dep("unreviewed-priv", PRIV_POD), old_object=b'{"kind":', source="Original"))
    revs.insert(13, D.Review(object=dep("reviewed-bad", "nope"), source="Original"))
    revs.insert(17, D.Review(object=dep("reviewed-priv", PRIV_POD), source="Original"))
    rb = drv.upload(revs, process="audit")
    run = D.AuditRun(drv, violations_limit=100)
    (run.add_batch_ordered if ordered else run.add_batch)(rb, EP)
    rep = run.report()
    run.close()
    errs = {x["object"]: x["error"] for x in rep["objectErrors"]["first"]}
    assert sorted(errs) == [5, 9, 13] and rep["objectErrors"]["count"] == 3, errs
    for i in (5, 9):
        assert errs[i].startswith("invalid request object: failed to unmarshal gkReview oldObject"), errs[i]
    assert errs[13].startswith("unable to expand object: "), errs[13]
    names = {sv["name"] for lst in rep["violations"].values() for sv in lst if sv["message"].startswith("[Implied by ")}
    assert "reviewed-priv" in names and not names & {"unreviewed-bad", "unreviewed-priv"}, names
    rb.free()
    drv.close()
