"""The audit of expanded batches on the GPU: the CUDA backend evaluates the resident resultants and sorts their pairs on the device
(gk_res_classify_kernel) against the parents' ranking.  A page below GK_SPEC_MIN_OBJECTS runs the interpreter, a larger one the
kernel generated for the constraint set.  The same cases run on the host emulation in test_audit_expand_hostemu.py."""
import pytest

import audit_expand_cases as X
from conftest import has_cuda

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_cuda(), reason="needs a CUDA device")]


@pytest.mark.parametrize("kind", ["blob", "kept", "objs"])
def test_mixed(kind):
    X.case_mixed(None, kinds=(kind,))


def test_mixed_generated_kernel():
    X.case_mixed(None, kinds=("blob", "kept"), n_pods=9000)


def test_laziness():
    X.case_laziness(None)


@pytest.mark.parametrize("kind", ["blob", "kept", "objs"])
def test_stale_then_refresh(kind):
    X.case_stale_then_refresh(None, kind)


def test_patched():
    X.case_patched(None)


@pytest.mark.parametrize("kind", ["blob", "objs"])
def test_shards_merge(kind):
    X.case_shards_merge(None, kind)
