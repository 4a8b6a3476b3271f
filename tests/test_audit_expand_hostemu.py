"""The audit of expanded batches on the test-only host emulation: the cases of test_audit_expand.py, with Backend::audit_candidates'
and Backend::audit_resultants' host defaults (test_audit_expand.py runs them against the CUDA backend's ranking and sorting)."""
import pytest

import audit_expand_cases as X
from conftest import HOSTEMU


@pytest.mark.parametrize("kind", ["blob", "kept", "objs"])
def test_mixed(kind):
    X.case_mixed(HOSTEMU, kinds=(kind,))


def test_laziness():
    X.case_laziness(HOSTEMU)


@pytest.mark.parametrize("kind", ["blob", "kept", "objs"])
def test_stale_then_refresh(kind):
    X.case_stale_then_refresh(HOSTEMU, kind)


def test_patched():
    X.case_patched(HOSTEMU)


@pytest.mark.parametrize("kind", ["blob", "objs"])
def test_shards_merge(kind):
    X.case_shards_merge(HOSTEMU, kind)
