"""Expanded batches (GK_F_EXPAND): the cases test_expand_sweep_hostemu.py runs on the test-only host emulation and test_expand_sweep.py
on the GPU.  Every bitmap call on an expanded batch must give gk_review_batch's planes, object errors and results for the same objects,
with totals that are the column popcounts of the planes.  `lib`: the host emulation's library, or None for the product library (then
the "device" buffers of gk_batch_eval_device* are CUDA tensors, else host arrays)."""
import contextlib
import json
import os
import re
import tempfile

import numpy as np

import test_capi_entry_points as T
from conftest import golden
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import k8s

EP = k8s.AUDIT_EP


@contextlib.contextmanager
def launch_trace():
    """The engine's GK_TRACE_LAUNCH lines written while the block runs (the native library writes them to file descriptor 2)."""
    lines = []
    old_env = os.environ.get("GK_TRACE_LAUNCH")
    os.environ["GK_TRACE_LAUNCH"] = "1"
    with tempfile.TemporaryFile(mode="w+b") as f:
        saved = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            yield lines
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            if old_env is None:
                del os.environ["GK_TRACE_LAUNCH"]
            else:
                os.environ["GK_TRACE_LAUNCH"] = old_env
            f.seek(0)
            lines += f.read().decode(errors="replace").splitlines()


def expand_line(lines):
    """(objects, kinds, selected, resultants) of the [expand] trace lines."""
    return [tuple(int(x) for x in m.groups()) for m in (re.match(r"\[expand\] (\d+) objects, (\d+) distinct kinds, (\d+) selected, (\d+) resultants", l)
                                                       for l in lines) if m]


def engine(lib, threads=0):
    """test_capi_entry_points' constraint set (Pods, Generated Pods only, a scoped one, Deployments) and Namespaces on `lib`."""
    t = golden("templates.json")
    drv = D.Driver(threads=threads, lib_path=lib)
    for k in ("allowedrepos", "psp_privileged", "requiredlabels_basic"):
        drv.add_template(t[k]["kind"], t[k]["rego"])
    for c in constraints(t):
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData(T.T, ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    return drv


def popcounts(planes, C):
    return [int(((planes[:, c // 32] >> np.uint32(c % 32)) & 1).sum()) for c in range(C)] if planes.size else [0] * C


def results(resp):
    return T._results(resp)


class Calls:
    """The bitmap calls on resident batch `rb`, each returning (viol, err, totals, err_totals) as numpy arrays / lists."""

    def __init__(self, lib, drv, rb):
        self.lib, self.drv, self.rb = lib, drv, rb
        self.n, self.C = len(rb), len(drv.constraints())
        self.words = max(1, (self.C + 31) // 32)

    def _buffers(self, k):
        if self.lib is None:
            import torch
            return torch.zeros(k, dtype=torch.int32, device="cuda"), (lambda t: t.cpu().numpy()), (lambda t: t.data_ptr())
        return np.zeros(k, np.int32), (lambda a: a.copy()), (lambda a: int(a.ctypes.data))

    def eval(self):
        r = self.rb.eval(EP)
        return r.viol_bits, r.err_bits, list(r.totals), list(r.err_totals)

    def device(self):
        n, C, w = self.n, self.C, self.words
        mk = lambda k: self._buffers(k)
        (viol, get, ptr), (err, _, _), (tot, _, _) = mk(n * w), mk(n * w), mk(4 * C)
        self.rb.eval_device(EP, ptr(viol), ptr(err), ptr(tot), ptr(tot) + 8 * C)
        self._sync()
        t = get(tot).view(np.int64)
        return (get(viol).view(np.uint32).reshape(n, w), get(err).view(np.uint32).reshape(n, w), t[:C].tolist(), t[C:].tolist())

    def peers(self, world=1):
        """`world` ranks' receive buffers, this batch written as rank world - 1 into all of them; every buffer must hold the same."""
        n, C, w = self.n, self.C, self.words
        tot_off = n * w + (n * w) % 2
        slot = tot_off + 4 * C
        bufs = [self._buffers(world * slot) for _ in range(world)]
        (err, get, ptr), (tot, _, _) = self._buffers(n * w), self._buffers(4 * C)
        rank = world - 1
        self.rb.eval_device_peers(EP, [b[2](b[0]) for b in bufs], rank, slot, tot_off, C, ptr(err), ptr(tot), ptr(tot) + 8 * C)
        self._sync()
        outs = []
        for b in bufs:
            g = b[1](b[0]).reshape(world, slot)[rank]
            t = g[tot_off:tot_off + 4 * C].copy().view(np.int64)
            outs.append((g[:n * w].view(np.uint32).reshape(n, w), get(err).view(np.uint32).reshape(n, w), t[:C].tolist(), t[C:].tolist()))
        for o in outs[1:]:
            assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(o, outs[0])), "the peers' buffers differ"
        return outs[0]

    def _sync(self):
        if self.lib is None:
            import torch
            torch.cuda.synchronize()

    def all(self):
        calls = {"gk_batch_eval": self.eval, "gk_batch_eval_device": self.device, "gk_batch_eval_device_peers": self.peers}
        if self.lib is not None:   # (two ranks in one process: host arrays stand in for peer-mapped device memory)
            calls["gk_batch_eval_device_peers x2"] = lambda: self.peers(2)
        return calls


def assert_like_review(got, want, C, what):
    viol, err, tot, etot = got
    assert np.array_equal(viol, want.viol_bits), what + ": violation plane"
    assert np.array_equal(err, want.err_bits), what + ": error plane"
    assert list(tot) == popcounts(want.viol_bits, C), what + ": totals are not the plane's popcounts"
    assert list(etot) == popcounts(want.err_bits, C), what + ": error totals are not the plane's popcounts"


def upload(drv, revs, kind, process=""):
    """The page as review objects, as a blob, or as a blob with its kept source; the blob kinds leave out what a blob cannot hold."""
    if kind == "objs":
        return drv.upload(revs, process=process, expand=True), revs
    docs = [r.object for r in revs if r.object is not None and r.old_object is None and r.operation in (None, "")]
    blob = W.PyBlob(docs)
    rb = drv.upload_blob(blob, process=process, keep_source=kind == "kept", expand=True)
    rb._blob = blob
    return rb, [D.Review(object=d, source="Original") for d in docs]


def check_against_review(lib, drv, rb, revs, process, what):
    want = drv.ReviewBatch(revs, EP, process=process)
    C = len(want.totals)
    calls = Calls(lib, drv, rb)
    for name, call in calls.all().items():
        assert_like_review(call(), want, C, "%s %s" % (what, name))
    got = rb.eval(EP, flags=D.F_MATERIALIZE)
    assert results(got) == results(want), what + ": materialized results"
    assert got.object_errors == want.object_errors, what + ": object errors"
    assert rb.eval(EP).object_errors == want.object_errors, what + ": object errors without rendering"
    return want


def case_every_call_equals_review(lib, kind, process=""):
    """The mixed page (generators of three templates, a failing template source, a template-less Deployment, a DELETE) on every call."""
    drv = engine(lib, threads=4)
    for d in T.EXPANSION:
        drv.AddExpansionTemplate(d)
    revs = T._review_page()
    with launch_trace() as lines:
        rb, revs = upload(drv, revs, kind, process)
    n, k, g, m = expand_line(lines)[0]
    assert n == len(revs) and 0 < g < n and m > 0, (n, k, g, m)
    want = check_against_review(lib, drv, rb, revs, process, kind)
    assert any(r[2].startswith("[Implied by expand-jobs] ") and r[4] == "dryrun" for r in results(want))
    assert want.object_errors and sum(1 for e in want.object_errors if e and e.startswith("unable to expand object: ")) == 2
    if kind != "objs":   # gk_review_blob with the flag: the same
        got = drv.ReviewBlob(rb._blob, EP, flags=D.F_EXPAND | D.F_MATERIALIZE | D.PROCESS_FLAG[process])
        assert_like_review((got.viol_bits, got.err_bits, got.totals, got.err_totals), want, len(want.totals), "gk_review_blob")
        assert results(got) == results(want) and got.object_errors == want.object_errors
    rb.free()
    drv.close()


def case_oracle(lib):
    """Bit (o, c) is set exactly when the oracle's review with expansion gives object o at least one result of constraint c."""
    from conftest import make_pair
    from oracle import expansion as X
    t = golden("templates.json")
    tm = [(t[k]["kind"], t[k]["rego"]) for k in ("allowedrepos", "psp_privileged", "requiredlabels_basic")]
    orc, drv, skipped = make_pair(tm, constraints(t), W.synth_namespaces(), lib_path=lib)
    assert not skipped
    xs = X.System()
    for d in T.EXPANSION:
        xs.upsert(d)
        drv.AddExpansionTemplate(d)
    revs = [r for r in T._review_page(n_pods=120) if not r.operation]
    rb = drv.upload(revs, expand=True)
    got = rb.eval(EP)
    keys = got.constraints
    for o, r in enumerate(revs):
        rv = k8s.Review(obj=r.object, source="Original")
        try:
            res = X.review_with_expansion(orc, xs, rv, EP)
        except X.ExpansionError:   # (the engine reports it as the object's error, with the object's own results)
            res = orc.review(rv, EP)
        want = {keys.index("%s/%s" % x["constraint"]) for x in res}
        have = {c for c in range(len(keys)) if (got.viol_bits[o, c // 32] | got.err_bits[o, c // 32]) >> np.uint32(c % 32) & 1}
        assert have == want, (o, have, want)
    rb.free()
    drv.close()


def constraints(t):
    return [W._constraint(t["allowedrepos"]["kind"], "repos", match=dict(W.POD), params={"repos": ["gcr.io/"]}, action="warn"),
            W._constraint(t["psp_privileged"]["kind"], "priv", match={"kinds": [{"apiGroups": [""], "kinds": ["Pod"]}], "source": "Generated"}),
            W._constraint(t["psp_privileged"]["kind"], "priv-scoped", match=dict(W.POD), action="scoped",
                          scoped=[{"action": "warn", "enforcementPoints": [{"name": EP}]}]),
            W._constraint(t["requiredlabels_basic"]["kind"], "team", match={"kinds": [{"apiGroups": ["apps"], "kinds": ["Deployment"]}]},
                          params={"labels": ["team"]})]


def case_config4_selection(lib, n=3000, kind="blob"):
    """A config-4 page of mixed kinds with expand-deployments: only the Deployments and the objects without a hash are selected, and
    every call equals gk_review_batch."""
    tm, cons = W.config4()
    drv = D.Driver(lib_path=lib)
    for k, rego in tm:
        drv.add_template(k, rego)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData(T.T, ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    drv.AddExpansionTemplate(T._expansion_template("expand-deployments", ["Deployment"], ("", "v1", "Pod")))
    blob = W.synth_objects(0, n, mode=1)
    docs = [json.loads(blob.get(i)) for i in range(n)]
    deployments = sum(1 for d in docs if d.get("kind") == "Deployment" and d.get("apiVersion") == "apps/v1")
    assert deployments, "the config-4 page holds Deployments"
    revs = [D.Review(object=d, source="Original") for d in docs]
    with launch_trace() as lines:
        rb = drv.upload_blob(blob, expand=True, keep_source=kind == "kept") if kind != "objs" else drv.upload(revs, expand=True)
    (objs, kinds, g, m), = expand_line(lines)
    assert objs == n and g == deployments and m >= deployments and kinds > 1, (objs, kinds, g, m, deployments)
    check_against_review(lib, drv, rb, revs, "", "config-4 " + kind)
    rb.free()
    drv.close()


def case_no_generators(lib, n=2000):
    """A config-2 page with a template registered but no generators: the expanded batch has no resultants and returns what the plain
    batch returns (with no template registered)."""
    tm, cons = W.config2()
    drv = D.Driver(lib_path=lib)
    for k, rego in tm:
        drv.add_template(k, rego)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData(T.T, ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    blob = W.synth_objects(0, n)
    plain = drv.upload_blob(blob)
    want = [x for x in Calls(lib, drv, plain).eval()]
    want_results = results(plain.eval(EP, flags=D.F_MATERIALIZE))
    drv.AddExpansionTemplate(T.EXPANSION[0])
    with launch_trace() as lines:
        rb = drv.upload_blob(blob, expand=True)
        calls = Calls(lib, drv, rb)
        for name, call in calls.all().items():
            got = call()
            assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(got, want)), name
        assert results(rb.eval(EP, flags=D.F_MATERIALIZE)) == want_results
    (objs, kinds, g, m), = expand_line(lines)
    assert (objs, g, m) == (n, 0, 0), (objs, kinds, g, m)   # (no resultant batch: the evaluations run no fold)
    assert len(rb) == n and rb.alg_bytes == plain.alg_bytes
    rb.free()
    plain.free()
    drv.close()


def case_excluded_generators(lib, kind):
    """Generators in namespaces the audit's excluder skips: selected (no hash), expanded, and their resultants skipped as well."""
    drv = engine(lib)
    for d in T.EXPANSION:
        drv.AddExpansionTemplate(d)
    drv.SetExcludedNamespaces("audit", ["ns-000*"])
    revs = T._review_page(n_pods=200, seed=5)
    rb, revs = upload(drv, revs, kind, process="audit")
    check_against_review(lib, drv, rb, revs, "audit", "excluded " + kind)
    rb.free()
    drv.close()


def case_wide_resultant(lib, kind):
    """A Deployment whose Pod template has 40 containers: a resultant with more rows in a scope than the mask registers hold."""
    drv = engine(lib)
    drv.AddExpansionTemplate(T.EXPANSION[0])
    wide = {"metadata": {"labels": {"app": "w"}}, "spec": {"containers": [{"name": "c%d" % i, "image": "evil.example.com/%d" % i,
                                                                       "securityContext": {"privileged": i % 7 == 3}} for i in range(40)]}}
    revs = T._review_page(n_pods=300, seed=9)
    revs.insert(17, D.Review(object={"apiVersion": "apps/v1", "kind": "Deployment", "metadata": {"name": "wide", "namespace": "ns-0003",
                                                                                                  "labels": {"team": "x"}},
                                     "spec": {"template": wide}}, source="Original"))
    rb, revs = upload(drv, revs, kind)
    check_against_review(lib, drv, rb, revs, "", "wide " + kind)
    rb.free()
    drv.close()


def case_staleness_and_refresh(lib, kind):
    """Adding, removing, and a cycle-closing upsert each make the eval calls refuse the batch; a refresh rebuilds it (1, then 0) into
    what a fresh upload gives; the audit reports what it reports for the same batch uploaded without the flag."""
    drv = engine(lib)
    drv.AddExpansionTemplate(T.EXPANSION[0])
    revs = T._review_page(n_pods=150, seed=3)
    rb, revs = upload(drv, revs, kind)

    def evals():
        c = Calls(lib, drv, rb)
        return [c.eval, c.device, c.peers]

    def stale_then_refresh(change, what):
        change()
        for call in evals():
            T._refuses(call, T.ERR_REGO, "ExpansionTemplates changed since the batch was expanded")
        with launch_trace() as lines:
            assert rb.refresh()["rebuilt"] is True
        if kind == "kept" and lib is None:   # the page is neither copied nor tokenised again: only the resultants' own page is
            m = expand_line(lines)[0][3]
            assert [l for l in lines if "gk_tape_kernel" in l] == (["[launch] gk_tape_kernel over %d objects" % m] if m else []) or all(
                "over %d objects," % m in l for l in lines if "gk_tape_kernel" in l), lines
            assert any("from the kept source" in l for l in lines), lines
        assert rb.refresh()["rebuilt"] is False
        fresh, _ = upload(drv, [D.Review(object=r.object, source="Original") for r in revs] if kind != "objs" else revs, kind)
        want = Calls(lib, drv, fresh).eval()
        got = Calls(lib, drv, rb).eval()
        assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(got, want)), what
        assert results(rb.eval(EP, flags=D.F_MATERIALIZE)) == results(fresh.eval(EP, flags=D.F_MATERIALIZE)), what
        check_against_review(lib, drv, rb, revs, "", what)
        fresh.free()

    assert rb.refresh()["rebuilt"] is False
    stale_then_refresh(lambda: drv.AddExpansionTemplate(T.EXPANSION[1]), "upsert")
    stale_then_refresh(lambda: drv.RemoveExpansionTemplate("expand-deployments"), "remove")
    drv.AddExpansionTemplate(T.EXPANSION[0])
    assert rb.refresh()["rebuilt"] is True
    cyc = T._expansion_template("pods-to-deployments", ["Pod"], ("apps", "v1", "Deployment"), groups=("",))

    def closing():
        try:
            drv.AddExpansionTemplate(cyc)
        except D.GkError as e:
            assert "template forms expansion cycle" in str(e)
        else:
            raise AssertionError("the cycle was not reported")

    stale_then_refresh(closing, "cycle")
    # the audit: as for the same batch uploaded without the flag
    plain = drv.upload(revs) if kind == "objs" else drv.upload_blob(rb._blob, keep_source=kind == "kept")
    for ordered in (False, True):
        reps = []
        for b in (rb, plain):
            run = D.AuditRun(drv, violations_limit=7)
            (run.add_batch_ordered if ordered else run.add_batch)(b, EP)
            reps.append(run.report())
            run.close()
        assert reps[0] == reps[1], ordered
    plain.free()
    rb.free()
    drv.close()
