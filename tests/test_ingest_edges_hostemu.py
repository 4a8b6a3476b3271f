"""The cases of test_ingest_edges.py on the test-only host emulation: the review envelope spelt with escapes, the native string
programs against the lookup table, and a page past the emulation's own miss list (2^16) and table growths (2^12 -> 2^14 -> 2^16)."""
import ingest_edge_cases as E
from conftest import HOSTEMU


def test_envelope_fields_in_every_spelling():
    """apiVersion / kind / name / namespace with \\/, \\u002f and \\u00XX escapes: device ingest == host flattener == oracle."""
    assert E.case_envelope(HOSTEMU) > 100


def test_string_programs_native_against_lookup_table(monkeypatch, capfd):
    assert E.case_string_programs(HOSTEMU, monkeypatch, capfd) > 0


def test_many_distinct_lookup_arguments(monkeypatch, capfd):
    """About 70 k distinct arguments in one upload, then the page refreshed and patched."""
    assert E.case_many_lookups(HOSTEMU, monkeypatch, capfd, n=4900, sample=120, n_patch=300, n_drop=200) > 1 << 16
