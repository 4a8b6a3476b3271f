"""GPU parity tests: the product library (CUDA kernels, through the C ABI) against the oracle on the same
seeded inputs, the committed golden fixtures, and size-independent properties at larger sizes.
Run on an H100:  python -m pytest tests -m gpu -x -q"""
import json

import numpy as np
import pytest

import parity_cases as P
from conftest import golden, has_cuda
from gatekeeper_b200 import driver as D
from gatekeeper_b200 import workloads as W
from oracle import k8s

pytestmark = pytest.mark.gpu
LIB = None   # the product library, gatekeeper_b200/libgk_engine.so


@pytest.fixture(scope="module", autouse=True)
def _needs_gpu():
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    d = D.Driver()
    assert d.backend() == "cuda-sm90a"
    d.close()


@pytest.mark.parametrize("case", golden("gator_cases.json"), ids=lambda c: c["name"])
def test_gator_cases(case):
    resp = P.case_gator(LIB, case)
    assert resp.stats["gpu_launches"] >= 1 or resp.n_objects == 0


def test_psp_suite():
    P.case_psp(LIB)


def test_config2_parity_2000_objects():
    resp, want = P.case_config2(LIB, 2000)
    assert len(want) > 5000 and resp.stats["gpu_launches"] >= 1 and resp.stats["kernel_ms"] > 0


def test_config2_other_range_and_admission_ep():
    P.case_config2(LIB, 700, start=123456, ep=k8s.WEBHOOK_EP)


def test_config2_missing_namespace_cache():
    resp, want = P.case_config2(LIB, 300, start=9000, with_namespaces=False)
    assert sum(resp.err_totals) == sum(1 for w in want if w[-1]) > 0


def test_mixed_kinds():
    P.case_mixed_kinds(LIB, 1500)


def test_config5_wildcards():
    P.case_config5(LIB, 1500)


def test_allowedrepos_comprehension_variant():
    P.case_allowedrepos_comprehension_variant(LIB, 500)


def test_match_vectors():
    P.case_match_vectors(LIB)


def test_admission_shapes():
    P.case_admission_shapes(LIB)


def test_review_errors():
    P.case_review_errors(LIB)


def test_edge_batches():
    P.case_edge_batches(LIB)


def test_unsupported_is_an_error():
    P.case_unsupported_is_an_error_not_a_fallback(LIB)


def test_audit_aggregation_matches_oracle():
    P.case_audit(LIB, n=1500)


def test_validation_messages():
    P.case_validation_messages(LIB)


@pytest.mark.parametrize("seed", [101, 202])
def test_mutation_fuzz(seed):
    """Synthetic Pods with random structural damage (wrong types, nulls, missing members, boundary-length strings)."""
    nres, nbad = P.case_fuzz(LIB, n=1500, seed=seed, start=100000 + seed)
    assert nres > 1500


@pytest.mark.parametrize("seed", [11, 12])
def test_match_fuzz(seed):
    """Random spec.match blocks x random review shapes through the in-kernel pre-filter."""
    assert P.case_match_fuzz(LIB, n_constraints=96, n_objects=700, seed=seed) > 1000


def test_fuzz_other_templates():
    """The in-tree templates outside config 2 (regex labels, object.get(input, ...), namespaceObject, user info ...)."""
    assert P.case_fuzz_other_templates(LIB, n=600, seed=314) > 800


def test_template_libs():
    """A template with `libs` (the bats container-limits template: package lib.helpers imported as data.lib.helpers)."""
    assert P.case_template_libs(LIB, n=600) > 10


def test_more_builtins():
    """sort / object.* / numbers.range / rounding / set builtins as feature columns, folded parameters and device atoms."""
    assert P.case_more_builtins(LIB) > 30


@pytest.mark.parametrize("seed", [11, 12])
def test_rego_fuzz(seed):
    """Random policies assembled from ~80 statement shapes x random parameters x damaged Pods: whatever loads must agree."""
    accepted, n_results, _ = P.case_rego_fuzz(LIB, n_templates=30, seed=seed)
    assert accepted >= 20 and n_results > 500


def test_validate_constraint_vectors():
    """pkg/target/target_test.go TestValidateConstraint: 11 vectors + error-text agreement on hand-made selectors."""
    assert P.case_validate_constraint(LIB) == 8


def test_every():
    assert P.case_every(LIB) > 800


def test_cross_scope_join():
    assert P.case_cross_scope_join(LIB) > 20


def test_target_enforcement_vectors():
    """pkg/target/target_integration_test.go: 26 scenarios x 3 request shapes, allowed <=> no results."""
    P.case_target_enforcement(LIB)


def test_target_matcher_vectors():
    P.case_target_matcher(LIB)


def test_gator_test_table():
    """pkg/gator/test/test_test.go:85-268: exact (message, constraint, action, scoped actions) lists."""
    P.case_gator_test_table(LIB)


def test_verify_suite():
    """test/gator/verify/suite.yaml:1-37 (K8sFooIs) through the engine."""
    P.case_verify_suite(LIB)


def test_config3_admission_microbatches():
    """200 PSP constraints (7 bitmap words) x 64-request micro-batches, UPDATE with object + oldObject."""
    tm, cons, pods = W.config3(200)
    from conftest import assert_same, engine_results, make_pair, oracle_results
    orc, drv, _ = make_pair(tm, cons, lib_path=LIB)
    revs = [D.Review(object=pods[i % 5], old_object=pods[(i + 1) % 5], operation="UPDATE", user_info={"username": "u"}) for i in range(64)]
    resp = drv.ReviewBatch(revs, k8s.WEBHOOK_EP)
    assert resp.viol_bits.shape == (64, 7)
    assert_same(oracle_results(orc, revs, k8s.WEBHOOK_EP), engine_results(resp))


# ---- size-independent properties at larger sizes -----------------------------------------------------------
@pytest.fixture(scope="module")
def big():
    tm, cons = W.config2()
    drv = D.Driver()
    for k, r in tm:
        drv.add_template(k, r)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    n = 200_000
    blob = W.synth_objects(0, n)
    revs = [D.Review(object=blob.get(i), source="Original") for i in range(n)]
    return drv, blob, revs, n


def test_large_batch_properties(big):
    drv, blob, revs, n = big
    rb = drv.upload(revs)
    a = rb.eval()
    b = rb.eval()
    # determinism
    assert (a.viol_bits == b.viol_bits).all() and a.totals == b.totals
    # totals are the column popcounts of the bitmap (a checksum of checksums)
    bits = a.viol_bits
    for ci in range(len(a.constraints)):
        col = (bits[:, ci // 32] >> np.uint32(ci % 32)) & np.uint32(1)
        assert int(col.sum()) == a.totals[ci]
    # sharding invariance: evaluating halves separately and concatenating equals the whole
    h = n // 2
    r1 = drv.upload(revs[:h]).eval()
    r2 = drv.upload(revs[h:]).eval()
    assert (np.concatenate([r1.viol_bits, r2.viol_bits]) == bits).all()
    assert [x + y for x, y in zip(r1.totals, r2.totals)] == a.totals
    # spot-check 300 random objects of the big batch against the oracle
    rng = np.random.default_rng(1)
    idx = sorted(rng.choice(n, 300, replace=False).tolist())
    tm, cons = W.config2()
    orc = k8s.Client()
    for k, r in tm:
        orc.add_template(k, r)
    for c in cons:
        orc.add_constraint(c)
    for ns in W.synth_namespaces():
        orc.add_namespace(ns)
    keys = a.constraints
    for i in idx:
        want = {"%s/%s" % r["constraint"] for r in orc.review(k8s.Review(obj=json.loads(blob.get(i)), source="Original"), k8s.AUDIT_EP)
                if not r.get("autoreject")}
        got = {keys[c] for c in range(len(keys)) if (int(bits[i, c // 32]) >> (c % 32)) & 1}
        assert got == want, i
    rb.free()


def test_enforcement_point_mask_only_hides_scoped_constraints(big):
    drv, blob, revs, n = big
    rb = drv.upload(revs[:5000])
    audit = rb.eval(k8s.AUDIT_EP)
    vap = rb.eval("vap.k8s.io")   # scoped constraints list audit + "*": still active ("*")
    assert audit.totals == vap.totals
    rb.free()


# ---- device ingest: raw JSON flattened by the ingest kernels (csrc/ingest_kernels.cuh), then the same evaluation kernel
def test_blob_config2_device_ingest():
    resp, want = P.case_blob_config2(LIB, 3000)
    assert len(want) > 20000 and resp.stats["gpu_launches"] >= 4


def test_blob_fuzz_device_ingest():
    P.case_blob_fuzz(LIB)


def test_blob_json_oddities():
    P.case_blob_json_oddities(LIB)


def test_blob_other_templates():
    P.case_blob_other_templates(LIB)


def test_blob_rego_fuzz():
    accepted, n_results, rejected, n_device = P.case_rego_fuzz(LIB, n_templates=30, n_objects=100, seed=12, via_blob=True)
    assert n_device >= accepted // 2, (n_device, accepted)


def test_inexact_numbers_are_compared_not_skipped():
    P.case_inexact_numbers(LIB)


def test_blob_large_batch_properties():
    """200 k Pods through the device ingest path: same bitmap as the host-flattened batch, totals == popcounts."""
    tm, cons = W.config2()
    drv = D.Driver()
    for k, r in tm:
        drv.add_template(k, r)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData("t", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    n = 200_000
    blob = W.synth_objects(0, n)
    dev = drv.ReviewBlob(blob, k8s.AUDIT_EP, with_results=False)
    import os
    os.environ["GK_NO_DEVICE_INGEST_RUNTIME"] = "1"
    try:
        host = drv.ReviewBlob(blob, k8s.AUDIT_EP, with_results=False)
    finally:
        del os.environ["GK_NO_DEVICE_INGEST_RUNTIME"]
    assert (dev.viol_bits == host.viol_bits).all() and (dev.err_bits == host.err_bits).all() and dev.totals == host.totals
    assert sum(dev.totals) > n


def test_doc_pins():
    assert P.case_doc_pins(LIB) == 5


def test_wildcard_vectors_through_kernel():
    P.case_wildcard_vectors_through_kernel(LIB)


def test_expansion_templates_through_the_batch():
    assert P.case_expansion(LIB) >= 6


def test_referential_constraints_data_inventory():
    assert P.case_referential(LIB) > 40


def test_audit_counts_single_result_pairs_and_evaluates_only_list_candidates():
    got = P.case_audit_lazy(LIB)
    assert got["pairsEvaluated"] < got["results"]


def test_pages_of_wide_objects_shrink_the_tile():
    assert P.case_wide_objects(LIB) > 100


def test_audit_concurrent_with_reviews():
    P.case_audit_concurrent_with_reviews(LIB)


@pytest.mark.parametrize("config", [2, 4, 5])
def test_generated_kernel_is_identical_to_the_interpreter(config):
    assert P.case_spec_kernel(LIB, 20000 if config == 2 else 6000, config=config) > 500


def test_audit_expands_generators_like_the_audit_loop():
    got = P.case_audit_expansion(LIB)
    assert got["results"] > 50
