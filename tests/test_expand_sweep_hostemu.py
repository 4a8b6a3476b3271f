"""Expanded batches (GK_F_EXPAND) on the test-only host emulation: the selection and the fold run on host arrays there, through the same
C entry points, so the cases of expand_sweep_cases.py need no GPU.  test_expand_sweep.py runs them on the GPU."""
import pytest

import expand_sweep_cases as X
from conftest import HOSTEMU


@pytest.mark.parametrize("kind", ["objs", "blob", "kept"])
def test_every_call_equals_review(kind):
    X.case_every_call_equals_review(HOSTEMU, kind)


def test_every_call_equals_review_with_the_audit_process():
    X.case_every_call_equals_review(HOSTEMU, "blob", process="audit")


def test_bits_follow_the_oracle():
    X.case_oracle(HOSTEMU)


@pytest.mark.parametrize("kind", ["blob", "objs"])
def test_config4_selects_only_deployments(kind):
    X.case_config4_selection(HOSTEMU, n=1500, kind=kind)


def test_no_generators_is_a_plain_batch():
    X.case_no_generators(HOSTEMU, n=600)


@pytest.mark.parametrize("kind", ["objs", "kept"])
def test_excluded_generators(kind):
    X.case_excluded_generators(HOSTEMU, kind)


def test_wide_resultant():
    X.case_wide_resultant(HOSTEMU, "blob")


@pytest.mark.parametrize("kind", ["objs", "blob", "kept"])
def test_staleness_and_refresh(kind):
    X.case_staleness_and_refresh(HOSTEMU, kind)
