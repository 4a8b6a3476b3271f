"""The generated kernel's row-local folding (spec_codegen.cpp): phase 1 evaluates the gates that read one row alone and stages only
the bits something else reads (exports: "any" form for object-level EXISTS, "mask" form for everything else).  On the test-only host
emulation the generated text is compared object by object with the interpreted netlist (GK_SPEC_CHECK=1), its results with the
oracle, and the shape of the folding is read from the first line of the generated text (GK_SPEC_DUMP)."""
import json
import re

import numpy as np
import pytest

import audit_order_cases as A
import gpu_path_cases as G
from conftest import HOSTEMU, make_pair
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import audit as OA
from oracle import k8s

T = W.templates()
POD = W.POD
FOLD = re.compile(r"scope (\d+): (\d+) atoms \+ (\d+) gates -> (\d+) any \+ (\d+) mask in (\d+) words")
REPOS = ["gcr.io/", "docker.io/library/", "quay.io/", "registry.k8s.io/", "openpolicyagent/", "evil.io/", "ghcr.io/"]


def tmpl(*names):
    return [(T[n]["kind"], T[n]["rego"]) for n in names]


def allowed_repos(i, repos=None, template="allowedrepos"):
    return W._constraint(T[template]["kind"], "repos-%02d" % i, match=POD, params={"repos": repos or [REPOS[i % len(REPOS)], "r%d.example/" % i]})


def pod(i, containers, init=(), volumes=None, **spec):
    o = {"apiVersion": "v1", "kind": "Pod", "metadata": {"name": "p-%04d" % i, "namespace": "default"}, "spec": dict(spec, containers=list(containers))}
    if init:
        o["spec"]["initContainers"] = list(init)
    if volumes is not None:
        o["spec"]["volumes"] = volumes
    return o


def container(j, **kw):
    c = G._row("containers", j)
    c.update(kw)
    return c


def folding(capfd, dump):
    """The first line of the dumped text as {scope: (atoms, gates, any, mask, words)}, and the number of objects the last
    `[spec check]` line counts as too big for the masks."""
    lines = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("[spec check]")]
    assert lines, "no [spec check] line: was the generated text checked?"
    big = int(re.search(r"\((\d+) too big", lines[-1]).group(1))
    head = dump.read_text().split("\n", 1)[0]
    assert head.startswith("// folded:"), head
    return {int(m[0]): tuple(int(x) for x in m[1:]) for m in FOLD.findall(head)}, big


def traced(monkeypatch, tmp_path):
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    monkeypatch.setenv("GK_SPEC_DUMP", str(tmp_path / "spec.cu"))
    return tmp_path / "spec.cu"


def check(tm, cons, objs, monkeypatch, capfd, tmp_path):
    """Evaluate `objs` under the host emulation with the generated text checked against the interpreted netlist; every object's
    violating and erroring pairs must be the oracle's.  Returns the folding and the count of too-big objects."""
    dump = traced(monkeypatch, tmp_path)
    orc, drv, _ = make_pair(tm, cons, lib_path=HOSTEMU)
    docs = [json.dumps(o).encode() for o in objs]
    rb = drv.upload_blob(W.PyBlob(docs))
    capfd.readouterr()
    r = rb.eval(k8s.AUDIT_EP)
    keys = list(r.constraints)
    viol, err = np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True)
    rb.free()
    drv.close()
    every = range(len(objs))
    want_v, want_e = G.oracle_pairs(orc, docs, every, k8s.AUDIT_EP)
    G.assert_same(want_v, G.bit_pairs(viol, keys, every))
    G.assert_same(want_e, G.bit_pairs(err, keys, every))
    assert want_v, "the page violates nothing: the case checks nothing"
    return folding(capfd, dump)


def by_atoms(fold):
    """The scopes ordered by atom count, largest first."""
    return sorted(fold.values(), reverse=True)


def test_negating_row_local_gate_on_the_row_edges(monkeypatch, capfd, tmp_path):
    """`not startswith(image, repo)` is a negating gate of one container row: 0, 1, 32 and 33 containers and init containers.  The
    33-row objects do not fit a mask register: the generated code says so and the interpreter's words for them are the oracle's."""
    objs = []
    for k in (0, 1, 32, 33):
        objs.append(pod(len(objs), [container(j) for j in range(k)]))
        objs.append(pod(len(objs), [container(1)], init=[container(j) for j in range(k)]))
        # only the LAST row violates / no row violates
        objs.append(pod(len(objs), [container(0, image="gcr.io/ok")] * max(0, k - 1) + [container(0, image="evil.io/x")] * min(k, 1)))
        objs.append(pod(len(objs), [container(0, image="gcr.io/ok")] * k))
    fold, big = check(tmpl("allowedrepos"), [allowed_repos(0, ["gcr.io/"]), allowed_repos(1, ["quay.io/", "docker.io/"])], objs, monkeypatch, capfd, tmp_path)
    assert big == 4
    for atoms, gates, any_, mask, words in fold.values():
        assert gates > 0 and any_ > 0 and mask == 0 and words == 1 and any_ < atoms + gates


def test_atom_folded_and_exported_next_to_a_broadcast(monkeypatch, capfd, tmp_path):
    """Config 2's templates share the container row: some of its atoms are folded into gates that only an object-level EXISTS reads
    (allowed repositories, limits, banned tags) and are also exported as masks, because gates with an input broadcast from the
    object (hostNetwork) or from the row's own children (ports, probes) read them.  One constraint set: "any" and "mask" exports of
    one scope, and EXISTS under a nested parent beside the object-level ones -- on hand-made Pods that set those inputs."""
    tm, cons = W.config2()
    cons = [dict(c, spec=dict(c["spec"], match=POD)) for c in cons]
    objs = []
    for i in range(48):
        cs = [container(j, ports=[G._row("ports", i + j + m) for m in range((i + j) % 4)]) for j in range(1 + i % 4)]
        objs.append(pod(i, cs, init=cs[:i % 3], **({"hostNetwork": i % 4 == 0} if i % 2 else {})))
    fold, big = check(tm, cons, objs, monkeypatch, capfd, tmp_path)
    assert big == 0
    assert any(gates > 0 and any_ > 0 and mask > 0 for _, gates, any_, mask, _ in fold.values()), fold
    assert any(any_ == 0 and mask > 0 for _, _, any_, mask, _ in fold.values()), fold   # nested scopes: masks only


@pytest.mark.parametrize("extra", [14, 22])
def test_more_than_32_exports_in_one_scope(extra, monkeypatch, capfd, tmp_path):
    """Config 2 plus `extra` K8sAllowedRepos constraints with repositories of their own: the container row stages two words, with
    the mask-form bits (extra = 14) or the any-form bits (extra = 22) on both sides of the word boundary."""
    tm, cons = W.config2()
    cons = cons + [allowed_repos(100 + i, template="allowedrepos_prefixmatch") for i in range(extra)]
    blob = W.synth_objects(77, 150)
    objs = [json.loads(blob.get(i)) for i in range(150)]
    fold, _ = check(tm, cons, objs, monkeypatch, capfd, tmp_path)
    atoms, gates, any_, mask, words = by_atoms(fold)[0]
    assert words == 2 and 32 < any_ + mask <= 64
    assert (any_ < 32 < any_ + mask) if extra == 14 else (any_ > 32 and mask > 0), (any_, mask)


def test_results_that_are_row_local_or_constant(monkeypatch, capfd, tmp_path):
    """K8sPSPHostNamespace's result is a gate of the object's own row (scope 0: exported as a mask of one bit); a template that always
    violates and one that never does are constants, which phase 1 does not stage."""
    tm = tmpl("psp_hostnamespace", "fixtures_TemplateAlwaysValidate", "fixtures_TemplateNeverValidate")
    cons = [W._constraint(kind, "c-%d" % i, match=POD) for i, (kind, _) in enumerate(tm)]
    objs = [pod(i, [container(i)], **({"hostPID": True} if i % 3 == 0 else {"hostIPC": i % 3 == 1})) for i in range(12)]
    fold, _ = check(tm, cons, objs, monkeypatch, capfd, tmp_path)
    assert list(fold) == [0] and fold[0][1] > 0 and fold[0][2] == 0 and fold[0][3] >= 1, fold


def test_audit_of_a_page_whose_netlist_folds(monkeypatch):
    """gk_audit_add_batch over a page evaluated by the folded text: the report is oracle/audit.py's."""
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    tm, cons = W.config2()
    nss = W.synth_namespaces()
    orc, drv, _ = make_pair(tm, cons, nss, lib_path=HOSTEMU)
    blob = W.synth_objects(5, 500)
    objs = [json.loads(blob.get(i)) for i in range(500)]
    rb = drv.upload_blob(blob, process="audit")
    run = D.AuditRun(drv, violations_limit=20)
    run.add_batch(rb, k8s.AUDIT_EP)
    rep = run.report()
    run.close()
    A.check_oracle(rep, OA.audit(orc, objs, namespaces={x["metadata"]["name"]: x for x in nss}, limit=20))
    rb.free()
    drv.close()


def test_config2_folds_and_stages_one_word_per_container_row(monkeypatch, capfd, tmp_path):
    """The flagship constraint set: gates are folded into phase 1, `containers` and `initContainers` (the scopes with the most atoms)
    export fewer bits than they have atoms, and a container row is one staged word."""
    tm, cons = W.config2()
    blob = W.synth_objects(0, 300)
    dump = traced(monkeypatch, tmp_path)
    _, drv, _ = make_pair(tm, cons, W.synth_namespaces(), lib_path=HOSTEMU)
    capfd.readouterr()
    drv.ReviewBlob(blob, with_results=False)
    drv.close()
    fold, big = folding(capfd, dump)
    assert big == 0 and sum(f[1] for f in fold.values()) > 0
    for atoms, gates, any_, mask, words in by_atoms(fold)[:2]:
        assert atoms >= 29 and any_ + mask < atoms and words == 1, fold
