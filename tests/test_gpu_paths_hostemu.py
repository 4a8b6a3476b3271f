"""The cases of test_gpu_paths.py that the test-only host emulation can run: the generated kernel's text at every bitmap width and
row edge, checked object by object against the interpreted netlist (GK_SPEC_CHECK=1) and against the oracle, and every matcher
error's reason in the autoreject results and the audit report."""
import pytest

import gpu_path_cases as G
from conftest import HOSTEMU


@pytest.mark.parametrize("C", [1, 31, 32, 33, 64, 65, 200])
def test_generated_kernel_text_at_every_bitmap_width_and_row_edge(C, monkeypatch):
    """The widths and row edges of the GPU test of the generated kernel, on a page of the host build's 96-object tiles."""
    assert G.case_spec_widths(HOSTEMU, monkeypatch, C, n=4 * 96 + 17, tile=96, big_tiles=(1, 3), sample=120, webhook_sample=40) > 0


def test_every_matcher_error_keeps_its_reason(monkeypatch):
    """The case that, on the GPU, lists more than 2^20 matcher errors: here at a small size (the host list is unbounded)."""
    assert G.case_matcher_error_list(HOSTEMU, monkeypatch, n=400, tail=100) == 400 * 32
