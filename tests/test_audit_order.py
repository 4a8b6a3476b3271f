"""gk_audit_add_batch_ordered on the GPU: the CUDA backend ranks the batch's identities and selects each constraint's candidates on the
device.  Every case compares the report with oracle/audit.py and with gk_audit_add_batch's (audit_order_cases.py); the same cases run
on the host emulation in test_audit_order_hostemu.py."""
import pytest

import audit_order_cases as A
from conftest import has_cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]


@pytest.mark.parametrize("kind", ["objs", "blob"])
@pytest.mark.parametrize("limit", [1, 20, 100000])
def test_mixed_page(kind, limit):
    A.case_mixed_page(None, kind, limit)


def test_mixed_page_in_small_pages():
    A.case_mixed_page(None, "blob", 3, page=37)


@pytest.mark.parametrize("kind", ["objs", "blob"])
def test_config4_page(kind):
    rep = A.case_config4_page(None, kind, n=20000)
    assert rep["objects"] == 20000


@pytest.mark.parametrize("kind", ["objs", "blob"])
def test_expansion(kind):
    A.case_expansion(None, kind)


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("limit", [1, 3, 20])
def test_candidates_exact(seed, limit):
    A.case_candidates_exact(None, ["objs", "blob"][seed % 2], seed, limit)


@pytest.mark.parametrize("shards", [1, 2, 3, 4])
@pytest.mark.parametrize("kind", ["objs", "blob"])
def test_shards_merge(kind, shards):
    A.case_shards_merge(None, kind, shards)


@pytest.mark.parametrize("kind", ["objs", "blob"])
def test_export_roundtrip_and_refusals(kind):
    A.case_export_roundtrip_and_refusals(None, kind)
