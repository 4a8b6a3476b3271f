"""The device ingest's edges on the GPU: the review envelope spelt with escapes, the native string programs against the lookup
table, and a page with more distinct lookup arguments than one round's miss list (2^17) holds, enough to grow the table past 2^19
entries inside one upload -- then refreshed and patched on the device."""
import pytest

import ingest_edge_cases as E


@pytest.mark.gpu
def test_envelope_fields_in_every_spelling():
    assert E.case_envelope(None) > 100


@pytest.mark.gpu
def test_string_programs_native_against_lookup_table(monkeypatch, capfd):
    assert E.case_string_programs(None, monkeypatch, capfd) > 0


@pytest.mark.gpu
def test_many_distinct_lookup_arguments(monkeypatch, capfd):
    assert E.case_many_lookups(None, monkeypatch, capfd, n=48000, n_patch=3000, n_drop=2000) > 1 << 19
