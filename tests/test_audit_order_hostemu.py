"""gk_audit_add_batch_ordered, gk_audit_export and gk_audit_merge on the test-only host emulation: the cases of test_audit_order.py
with Backend::audit_candidates' host default (test_audit_order.py runs them against the CUDA backend's ranking and selection)."""
import pytest

import audit_order_cases as A
from conftest import HOSTEMU


@pytest.mark.parametrize("kind", ["objs", "blob"])
@pytest.mark.parametrize("limit", [1, 20, 100000])
def test_mixed_page(kind, limit):
    A.case_mixed_page(HOSTEMU, kind, limit)


def test_mixed_page_in_small_pages():
    A.case_mixed_page(HOSTEMU, "blob", 3, page=37)


@pytest.mark.parametrize("kind", ["objs", "blob"])
def test_config4_page(kind):
    A.case_config4_page(HOSTEMU, kind, n=1500)


@pytest.mark.parametrize("kind", ["objs", "blob"])
def test_expansion(kind):
    A.case_expansion(HOSTEMU, kind)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("limit", [1, 3, 20])
def test_candidates_exact(seed, limit):
    A.case_candidates_exact(HOSTEMU, ["objs", "blob"][seed % 2], seed, limit)


@pytest.mark.parametrize("shards", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", ["objs", "blob"])
def test_shards_merge(kind, shards):
    A.case_shards_merge(HOSTEMU, kind, shards)


@pytest.mark.parametrize("kind", ["objs", "blob"])
def test_export_roundtrip_and_refusals(kind):
    A.case_export_roundtrip_and_refusals(HOSTEMU, kind)
