"""gk_batch_refresh on the test-only host emulation: the cases of test_batch_refresh.py that need no GPU.  The emulation keeps its
page source the way Backend's defaults do -- a host copy of the page, ingested again by a refresh -- so the C ABI's refresh logic is
covered here, and the CUDA backend's kept token tape and argument gathering on the GPU.  (The tile refusal of the failure case is
the CUDA backend's: it runs on the GPU only.)"""
import pytest

import batch_refresh_cases as R
from conftest import HOSTEMU


@pytest.mark.parametrize("kind,keep,process", [("blob", True, "audit"), ("blob", False, "audit"), ("objs", False, "audit"), ("blob", True, "")])
def test_refresh_after_every_kind_of_change(kind, keep, process):
    R.case_refresh_steps(HOSTEMU, kind=kind, keep=keep, process=process)


@pytest.mark.parametrize("keep", [True, False])
def test_refresh_referential(keep):
    R.case_refresh_referential(HOSTEMU, keep=keep)


def test_refresh_with_prefetch():
    R.case_refresh_with_prefetch(HOSTEMU, n=120)
