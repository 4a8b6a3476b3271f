"""Expanded batches (GK_F_EXPAND) on the GPU: the cases of expand_sweep_cases.py on the product library -- generator selection and the
fold as CUDA kernels, resultants evaluated by gk_spec_kernel and the interpreter -- with pages large enough (>= 8192 parents and
resultants) that the generated kernel runs on both."""
import pytest

import expand_sweep_cases as X

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("kind", ["objs", "blob", "kept"])
def test_every_call_equals_review(kind):
    X.case_every_call_equals_review(None, kind)


def test_every_call_equals_review_with_the_audit_process():
    X.case_every_call_equals_review(None, "blob", process="audit")


def test_bits_follow_the_oracle():
    X.case_oracle(None)


@pytest.mark.parametrize("kind,n", [("blob", 60000), ("kept", 20000), ("objs", 12000)])
def test_config4_selects_only_deployments(kind, n):
    X.case_config4_selection(None, n=n, kind=kind)


def test_no_generators_is_a_plain_batch():
    X.case_no_generators(None, n=20000)


@pytest.mark.parametrize("kind", ["objs", "kept"])
def test_excluded_generators(kind):
    X.case_excluded_generators(None, kind)


@pytest.mark.parametrize("kind", ["blob", "objs"])
def test_wide_resultant(kind):
    X.case_wide_resultant(None, kind)


@pytest.mark.parametrize("kind", ["objs", "blob", "kept"])
def test_staleness_and_refresh(kind):
    X.case_staleness_and_refresh(None, kind)
