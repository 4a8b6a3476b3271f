import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")
HOSTEMU = os.path.join(ROOT, "tests", "_hostemu", "libgk_hostemu.so")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with `-m gpu`)")


@pytest.fixture(scope="session", autouse=True)
def _native_built():
    """Build the native libraries once per session if they are missing (nvcc cross-compiles without a GPU)."""
    from gatekeeper_b200 import build
    build.build()


def golden(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


def has_cuda():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


# ------------------------------------------------------------------------------------------------ helpers
def make_pair(tmpls, constraints, namespaces=(), lib_path=None, skip_unsupported=False):
    """An oracle Client and an engine Driver loaded with the same templates / constraints / namespaces."""
    from gatekeeper_b200 import driver as D
    from oracle import k8s
    orc = k8s.Client()
    drv = D.Driver(lib_path=lib_path)
    skipped = []
    dropped_kinds = set()
    for kind, rego, *rest in tmpls:      # (kind, rego) or (kind, rego, libs)
        libs = tuple(rest[0]) if rest and rest[0] else ()
        try:
            drv.add_template(kind, rego, libs)
        except D.GkError as e:
            if skip_unsupported and "rego_unsupported" in str(e):
                skipped.append((kind, None, str(e)))
                dropped_kinds.add(kind)
                continue
            raise
        orc.add_template(kind, rego, libs)
    for c in constraints:
        if c["kind"] in dropped_kinds:
            continue
        try:
            drv.AddConstraint(c)
        except D.GkError as e:
            if skip_unsupported and "rego_unsupported" in str(e):
                skipped.append((c["kind"], c["metadata"]["name"], str(e)))
                continue
            raise
        orc.add_constraint(c)
    for ns in namespaces:
        orc.add_namespace(ns)
        orc.add_data(ns)
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    return orc, drv, skipped


def oracle_results(orc, reviews, ep):
    """Set of (object index, 'Kind/name', msg, canonical details, action, scoped actions, autoreject)."""
    from oracle import k8s
    out = set()
    for i, r in enumerate(reviews):
        rv = k8s.Review(obj=r.object if not isinstance(r.object, (bytes, str)) else json.loads(r.object),
                        old=r.old_object, ns=r.namespace, source=r.source, operation=r.operation, user_info=r.user_info,
                        namespace=r.namespace_name)
        for x in orc.review(rv, ep):
            out.add((i, "%s/%s" % x["constraint"], x["msg"], json.dumps(x["details"], sort_keys=True), x["enforcementAction"],
                     tuple(x["scopedEnforcementActions"]), bool(x.get("autoreject"))))
    return out


def engine_results(resp):
    return {(r.object, r.constraint, r.msg, json.dumps(r.details, sort_keys=True), r.enforcement_action,
             tuple(r.scoped_enforcement_actions), r.autoreject) for r in resp.results}


def assert_same(want, got, limit=10):
    if want == got:
        return
    missing = sorted(want - got)[:limit]
    extra = sorted(got - want)[:limit]
    raise AssertionError(f"violation sets differ: {len(want - got)} missing, {len(got - want)} extra\n  missing: {missing}\n  extra: {extra}")
