"""gk_batch_patch on the test-only host emulation: the shared cases (batch_patch_cases.py).  The emulation keeps its page source as
Backend's defaults do -- a host copy, concatenated by a patch and ingested again -- so the C ABI's patch logic (index checks, the
staying objects' errors and host spans, the refusals, expansion) is covered here, and the CUDA backend's splice on the GPU."""
import pytest

import batch_patch_cases as P
from conftest import HOSTEMU


@pytest.mark.parametrize("process", ["audit", ""])
def test_patch_replaces_a_share(process):
    P.case_replace_share(HOSTEMU, process=process)


def test_patch_mixed_kinds():
    P.case_mixed_kinds(HOSTEMU)


def test_patch_sequence():
    P.case_sequence(HOSTEMU)


def test_patch_edges():
    P.case_edges(HOSTEMU)


def test_patch_after_a_constraint_change():
    P.case_constraint_between(HOSTEMU)


def test_patch_expanded_batch():
    P.case_expanded(HOSTEMU)


def test_patch_invalid_calls():
    P.case_invalid(HOSTEMU)


def test_patch_refused_while_the_set_is_flattened_on_the_host():
    P.case_host_flattened(HOSTEMU)
