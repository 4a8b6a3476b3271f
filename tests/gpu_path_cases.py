"""Cases shared by the GPU tests of the evaluation kernels' GPU-only paths (test_gpu_paths.py) and their host-emulation counterparts
(test_gpu_paths_hostemu.py): constraint sets at every bitmap width, pages on the 32/33-row edge of the generated kernel's mask
registers, and a page with more matcher errors than the device list first holds."""
import json
import random

import numpy as np

from conftest import assert_same, golden, make_pair, oracle_results
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import k8s


SCOPED_TO_AUDIT = [{"action": "deny", "enforcementPoints": [{"name": k8s.AUDIT_EP}]}]
ROW_SCOPES = ("containers", "initContainers", "volumes", "ports")   # ports: of the first container (a nested scope)


def width_constraints(C):
    """C constraints, ceil(C / 32) bitmap words: config-2 constraints cloned under new names up to 65, the config-3 PSP clones above.
    Every 7th and the last are scoped to the audit enforcement point alone, so at the webhook their columns are inactive."""
    if C > 65:
        tm, cons, _ = W.config3(C)
    else:
        tm, base = W.config2()
        cons = []
        for i in range(C):
            c = json.loads(json.dumps(base[i % len(base)]))
            c["metadata"]["name"] = "%s-w%03d" % (c["metadata"]["name"], i)
            cons.append(c)
    inactive = [i for i in range(C) if C > 1 and (i % 7 == 3 or i == C - 1)]
    for i in inactive:
        cons[i]["spec"]["enforcementAction"] = "scoped"
        cons[i]["spec"]["scopedEnforcementActions"] = SCOPED_TO_AUDIT
    return tm, cons, inactive


def _row(scope, j):
    if scope == "volumes":
        # one member each: the scope of a volume's members then has as many rows as `volumes`, on the same edge
        return [{"emptyDir": {}}, {"hostPath": {"path": "/var/log/%d" % j}}, {"configMap": {"name": "cm"}}, {"nfs": {"server": "s", "path": "/"}}][j % 4]
    if scope == "ports":
        return {"containerPort": 1000 + j, "hostPort": (80, 8080, 30001, 0, 9000)[j % 5]}
    c = {"name": "%s-%d" % (scope[:4], j), "image": ("gcr.io/proj-0/a:v1.2.3", "docker.io/library/b:latest", "quay.io/c", "evil.io/d:v0.0.1")[j % 4]}
    if j % 3 == 0:
        c["resources"] = {"limits": {"cpu": ("250m", "1", "4")[j % 9 // 3], "memory": "256Mi"}}
    if j % 5 == 2:
        c["securityContext"] = {"privileged": True}
    if j % 7 == 1:
        c["readinessProbe"] = {"httpGet": {"path": "/", "port": 80}}
    return c


def _set_rows(doc, scope, k):
    """`k` rows in `scope`; besides them one container without ports or mounts and no other rows, so that no scope derived from two
    (the join of volumes and containers, the ports of every container) has more rows than `scope` itself."""
    spec = doc.setdefault("spec", {})
    first = dict((spec.get("containers") or [_row("containers", 0)])[0])
    first.pop("ports", None)
    first.pop("volumeMounts", None)
    spec.pop("initContainers", None)
    spec.pop("volumes", None)
    spec["containers"] = [first]
    if scope == "ports":
        first["ports"] = [_row("ports", j) for j in range(k)]
    else:
        spec[scope] = [_row(scope, j) for j in range(k)]


def row_edge_page(n, tile, big_tiles, start=424242, every=23):
    """Synthetic Pods, some with exactly 0, 1, 31, 32 or 33 rows in one scope.  Up to 32 rows fit the generated kernel's mask registers;
    33-row objects sit only in `big_tiles`, whose tiles the generated kernel hands to the interpreter, so the other tiles stay its own.
    The last partial tile ends with four 32-row objects.  Returns the JSON documents and {object: (scope, rows)}."""
    blob = W.synth_objects(start, n)
    fits = [(s, k) for k in (0, 1, 31, 32) for s in ROW_SCOPES]
    plan = {i: fits[m % len(fits)] for m, i in enumerate(range(0, n, every))}
    for m, i in enumerate(range(n - 4, n)):
        plan[i] = (ROW_SCOPES[m], 32)
    for m, i in enumerate(t * tile + off for t in big_tiles for off in (5, tile // 2, tile - 1)):
        plan[i] = (ROW_SCOPES[m % 4], 33)
    docs = []
    for i in range(n):
        if i in plan:
            d = json.loads(blob.get(i))
            _set_rows(d, *plan[i])
            docs.append(json.dumps(d).encode())
        else:
            docs.append(blob.get(i))
    return docs, plan


def bit_pairs(bits, keys, objs):
    """{(object, constraint key)} of the set bits of the rows `objs`."""
    out = set()
    for o in objs:
        for c, key in enumerate(keys):
            if (int(bits[o, c // 32]) >> (c % 32)) & 1:
                out.add((o, key))
    return out


def oracle_pairs(orc, docs, objs, ep):
    """The oracle's violating and erroring (object, constraint key) pairs for the objects `objs` of the page."""
    viol, err = set(), set()
    for o in objs:
        for x in oracle_results(orc, [D.Review(object=json.loads(docs[o]), source="Original")], ep):
            (err if x[-1] else viol).add((o, x[1]))
    return viol, err


def case_spec_widths(lib, monkeypatch, C, n=8192 + 37, tile=512, big_tiles=(2, 9, 15), sample=300, webhook_sample=100):
    """The kernel generated for a constraint set at bitmap width ceil(C / 32), on a page whose last tile and last warp are partial and
    whose objects sit on the 32/33-row edge of the mask registers in every kind of scope.  On the GPU, the generated kernel (forced at
    any page size) and the interpreter must store identical bitmaps and totals at the audit and the webhook enforcement point.  On the
    test-only host emulation the generated text is checked object by object against the interpreted netlist (GK_SPEC_CHECK=1).  Both:
    the oracle's pairs on a sample that holds every 32- and 33-row object and the last partial tile, and all-zero inactive columns."""
    tm, cons, inactive = width_constraints(C)
    nss = W.synth_namespaces()
    orc, _, _ = make_pair(tm, cons, nss, lib_path=lib)
    docs, plan = row_edge_page(n, tile, big_tiles)
    page = W.PyBlob(docs)
    is_emu = lib is not None and "hostemu" in lib

    def run(env):
        for k in ("GK_SPEC", "GK_SPEC_MIN_OBJECTS", "GK_SPEC_CHECK"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        drv = D.Driver(lib_path=lib)
        for k, r in tm:
            drv.add_template(k, r)
        for c in cons:
            drv.AddConstraint(c)
        for ns in nss:
            drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
        rb = drv.upload_blob(page)
        out = {}
        for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP):
            r = rb.eval(ep)
            out[ep] = (drv.last_kernel(), np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True), list(r.totals), list(r.err_totals))
        keys = list(r.constraints)
        rb.free()
        drv.close()
        return keys, out

    if is_emu:
        keys, got = run({"GK_SPEC_CHECK": "1"})
    else:
        keys, want = run({"GK_SPEC": "0"})
        keys_s, got = run({"GK_SPEC_MIN_OBJECTS": "0"})
        assert keys_s == keys
        for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP):
            assert want[ep][0] == "gk_eval_kernel" and got[ep][0] == "gk_spec_kernel", (ep, want[ep][0], got[ep][0])
            for a, b, what in zip(want[ep][1:], got[ep][1:], ("violation bitmap", "error bitmap", "totals", "error totals")):
                assert np.array_equal(np.asarray(a), np.asarray(b)), "%s at %s: the generated kernel differs from the interpreter" % (what, ep)
    assert len(keys) == C and got[k8s.AUDIT_EP][1].shape == (n, (C + 31) // 32)
    # the columns scoped to the audit: set at the audit, all zero at the webhook
    inactive = [keys.index("%s/%s" % (cons[i]["kind"], cons[i]["metadata"]["name"])) for i in inactive]
    for i in inactive:
        w, b = i // 32, np.uint32(1 << (i % 32))
        for ep_bits in got[k8s.WEBHOOK_EP][1:3]:
            assert not (ep_bits[:, w] & b).any(), (keys[i], "set at the webhook enforcement point")
        assert got[k8s.WEBHOOK_EP][3][i] == 0 and got[k8s.WEBHOOK_EP][4][i] == 0
    if inactive:
        assert sum(got[k8s.AUDIT_EP][3][i] for i in inactive) > 0
    # the oracle on a sample
    edge = sorted(i for i, (_, k) in plan.items() if k >= 32)
    last_tile = list(range(n - (n % tile or tile), n))
    rest = sorted(set(random.Random(C).sample(range(n), min(n, sample))) - set(edge) - set(last_tile))
    objs = sorted(set(edge) | set(last_tile) | set(rest[:max(0, sample - len(edge) - len(last_tile))]))
    assert any(plan.get(i, (None, 0))[1] == 33 for i in objs) and objs[-1] == n - 1
    for ep, objs_ep in ((k8s.AUDIT_EP, objs), (k8s.WEBHOOK_EP, sorted(set(edge[::2][:webhook_sample]) | set(last_tile)))):
        viol, err = oracle_pairs(orc, docs, objs_ep, ep)
        assert_same(viol, bit_pairs(got[ep][1], keys, objs_ep))
        assert_same(err, bit_pairs(got[ep][2], keys, objs_ep))
    return int(sum(got[k8s.AUDIT_EP][3]))


# ------------------------------------------------------------------------------------------ matcher errors past the list's first capacity
NS_MISSING = "failed to run Match criteria: namespace selector for namespace-scoped object but missing Namespace"


def case_matcher_error_list(lib, monkeypatch, n=33000, nsel=32, tail=200, limit=20):
    """`nsel` constraints, each with its own namespaceSelector (its own match block), over `n` namespaced Pods and no cached Namespace:
    n * nsel (object, match block) matcher errors, past 2^20 at the default size.  The kernels list every error's code for the host, which
    renders it into the autoreject message: every result -- reviewed with messages and listed by the audit -- must carry the reason.
    The last `tail` objects (the last tiles the persistent CTAs reach) are compared with the oracle.  On the GPU under both kernels."""
    t = golden("templates.json")["fixtures_TemplateNeverValidate"]
    cons = [{"kind": t["kind"], "metadata": {"name": "nssel-%02d" % i}, "spec": {"match": {"namespaceSelector": {"matchLabels": {"sel-%02d" % i: "on"}}}}}
            for i in range(nsel)]
    docs = [json.dumps({"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "p-%05d" % i, "namespace": "ns-%02d" % (i % 89)}}).encode() for i in range(n)]
    page = W.PyBlob(docs)
    orc, _, _ = make_pair([(t["kind"], t["rego"])], cons, lib_path=lib)
    lo = n - tail
    want = {(lo + x[0],) + x[1:] for x in oracle_results(orc, [D.Review(object=json.loads(d), source="Original") for d in docs[lo:]], k8s.AUDIT_EP)}
    assert len(want) == tail * nsel
    is_emu = lib is not None and "hostemu" in lib
    runs = [({}, None)] if is_emu else [({"GK_SPEC": "0"}, "gk_eval_kernel"), ({"GK_SPEC_MIN_OBJECTS": "0"}, "gk_spec_kernel")]
    for env, kernel in runs:
        for k in ("GK_SPEC", "GK_SPEC_MIN_OBJECTS", "GK_SPEC_CHECK"):
            monkeypatch.delenv(k, raising=False)
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        drv = D.Driver(lib_path=lib)
        drv.add_template(t["kind"], t["rego"])
        for c in cons:
            drv.AddConstraint(c)
        rb = drv.upload_blob(page)
        resp = rb.eval(k8s.AUDIT_EP, flags=D.F_MATERIALIZE)
        if kernel:
            assert drv.last_kernel() == kernel
        assert resp.err_totals == [n] * nsel and sum(resp.totals) == 0
        assert len(resp.results) == n * nsel and all(r.autoreject for r in resp.results)
        bad = [(r.object, r.constraint, r.msg) for r in resp.results if not r.msg.endswith(NS_MISSING)]
        assert not bad, "%d autoreject results without their reason, e.g. %r" % (len(bad), bad[:3])
        got = {(r.object, r.constraint, r.msg, json.dumps(r.details, sort_keys=True), r.enforcement_action, tuple(r.scoped_enforcement_actions), r.autoreject)
               for r in resp.results if r.object >= lo}
        assert_same(want, got)
        del resp, got
        run = D.AuditRun(drv, violations_limit=limit)
        run.add_batch(rb, k8s.AUDIT_EP)
        rep = run.report()
        run.close()
        assert rep["totalViolations"] == {"%s/%s" % (c["kind"], c["metadata"]["name"]): n for c in cons}
        listed = [v for lst in rep["violations"].values() for v in lst]
        assert len(listed) == nsel * min(limit, n) and all(v["message"].endswith(NS_MISSING) for v in listed), listed[:2]
        rb.free()
        drv.close()
    return n * nsel
