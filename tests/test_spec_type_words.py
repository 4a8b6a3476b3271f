"""Type words (program.h, eval_layout.h): a scope with GK_TW_MIN or more VT columns keeps them a second time as 4-bit nibbles, 8 per
32-bit word, W_s words per row (1, 2 or a multiple of 4), and the generated rows read a row's types with one aligned load instead of one
byte load per column.  Checked here: the pack function itself against a Python restatement (every value 0-9 in every nibble); the
layout the generated text's host build traces (GK_SPEC_TRACE) against the same restatement; the generated text against the interpreted
netlist object by object (GK_SPEC_CHECK=1) and the oracle, for scopes of 3, 4, 8, 9, 17 and 33 VT columns, after a refresh that
changes a scope's layout, and over an expanded batch; on the GPU, the generated kernel against the interpreter."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

import expand_sweep_cases as X
from conftest import HOSTEMU, has_cuda, make_pair
from gatekeeper_b200 import workloads as W
from oracle import k8s

from test_spec_fold import check, container, pod

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TYPES = re.compile(r"\[spec types\](.*) (\d+) type-word bytes$")
SCOPE = re.compile(r"scope (\d+): (\d+) vt columns in (\d+) words, (\d+) rows;")
# one JSON value per VT code a page can carry (GK_VT_SET has no JSON form): None = the field is absent
VALUES = [None, "null", False, True, 7, "s", [1], {"a": 1}, 1e300]


def tw_words(nvt):
    """gk_tw_words restated: none below 4 columns, else ceil(nvt / 8) words rounded up to 1, 2 or a multiple of 4."""
    w = (nvt + 7) // 8
    return 0 if nvt < 4 else w if w <= 2 else (w + 3) // 4 * 4


def pack_rows(vals, nvt):
    """The words of rows whose column k holds vals[row][k], restated."""
    W_ = tw_words(nvt)
    return [[sum((row[k] & 15) << 4 * (k % 8) for k in range(8 * w, min(nvt, 8 * w + 8))) for w in range(W_)] for row in vals]


HARNESS = r"""
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "program.h"
// argv: nvt rows; column k of row r holds (r + k) %% 10; prints W, then every row's words
int main(int argc, char** argv) {
  const uint32_t nvt = (uint32_t)atoi(argv[1]), rows = (uint32_t)atoi(argv[2]), W = gk_tw_words(nvt);
  std::vector<std::vector<uint8_t>> vt(nvt, std::vector<uint8_t>(rows));
  std::vector<GkColumn> cols(nvt + 1);
  std::vector<uint32_t> order(nvt);
  for (uint32_t k = 0; k < nvt; ++k) {
    for (uint32_t r = 0; r < rows; ++r) vt[k][r] = (uint8_t)((r + k) % 10u);
    cols[nvt - k].vt = vt[k].data();   // (column indices need not be the nibbles': the list maps them)
    order[k] = nvt - k;
  }
  std::vector<uint32_t> words((size_t)rows * W + 1, 0xdeadbeefu);
  for (uint32_t r = 0; r < rows; ++r) gk_tw_pack_row(cols.data(), order.data(), nvt, W, r, words.data());
  printf("%u\n", W);
  for (uint32_t r = 0; r < rows; ++r) {
    for (uint32_t w = 0; w < W; ++w) printf("%u ", words[(size_t)r * W + w]);
    printf("\n");
  }
  return words[(size_t)rows * W] == 0xdeadbeefu ? 0 : 1;
}
"""


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("tw")
    (d / "h.cpp").write_text(HARNESS.replace("%%", "%"))
    exe = d / "h"
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "gatekeeper_b200", "csrc"), str(d / "h.cpp"), "-o", str(exe)], check=True)
    return str(exe)


@pytest.mark.parametrize("nvt", [1, 3, 4, 5, 8, 9, 16, 17, 24, 32, 33, 40])
def test_pack_every_value_in_every_nibble(harness, nvt):
    """gk_tw_pack_row against the restatement: 10 rows, so that column k holds each of 0-9 once; no word past the last row written."""
    out = subprocess.run([harness, str(nvt), "10"], capture_output=True, text=True, check=True).stdout.split("\n")
    assert int(out[0]) == tw_words(nvt)
    got = [[int(x) for x in ln.split()] for ln in out[1:11]]
    want = pack_rows([[(r + k) % 10 for k in range(nvt)] for r in range(10)], nvt)
    assert got == want


def field_template(kind, n, first=0):
    """n rules, rule k violated by a container whose field f<first + k> is truthy: one VT column per field in the container scope."""
    rules = "\n\n".join('violation[{"msg": msg}] {\n  c := input.review.object.spec.containers[_]\n  c.f%d\n  msg := "f%d"\n}' % (k, k)
                        for k in range(first, first + n))
    return (kind, "package %s\n\n%s\n" % (kind.lower(), rules))


def field_value(i, j, k):
    return VALUES[(i + 3 * j + k) % len(VALUES)]


def field_page(n_objs, n_fields):
    """Pods of 0 to 4 containers (33 in every 40th: handed over as too wide), container j of pod i with field k set to
    VALUES[(i + 3 j + k) % 9]: every VT code in every nibble across the page."""
    objs = []
    for i in range(n_objs):
        k_cont = 33 if i % 40 == 39 else i % 5
        cs = []
        for j in range(k_cont):
            c = container(j)
            for k in range(n_fields):
                v = field_value(i, j, k)
                if v is not None:
                    c["f%d" % k] = None if v == "null" else v
            cs.append(c)
        objs.append(pod(i, cs))
    return objs


def types_line(capfd_err):
    m = [TYPES.match(ln) for ln in capfd_err if ln.startswith("[spec types]")]
    assert m and m[-1], "no [spec types] line"
    return {int(x[0]): tuple(int(y) for y in x[1:]) for x in SCOPE.findall(m[-1].group(1))}, int(m[-1].group(2))


def check_layout(scopes, nbytes):
    """The traced layout restated: W_s from the column count alone, 4 bytes per word per row."""
    for s, (nvt, w, rows) in scopes.items():
        assert nvt >= 4 and w == tw_words(nvt), (s, nvt, w)
    assert nbytes == sum(4 * w * rows for _, w, rows in scopes.values())


def nibbles_in_text(text, scope):
    """The row function of `scope`: {column: (word, shift)} of every type it takes from its type words, and its byte loads of types."""
    at = text.index("exports of one row of scope %d " % scope)
    body = text[at:text.index("\n}\n", at)]
    nib = {int(c): (int(w), int(s)) for c, w, s in re.findall(r"const uint32_t t(\d+) = \(tw(\d+) >> (\d+)u\) & 15u;", body)}
    return nib, re.findall(r"cols\[(\d+)\]\.vt \+ row", body)


@pytest.mark.parametrize("n", [3, 4, 8, 9, 17, 33])
def test_container_scope_of_n_vt_columns(n, monkeypatch, capfd, tmp_path):
    """A container scope of n VT columns: below GK_TW_MIN byte loads; from it one load of W_s words and nibbles in column order.
    The text equals the interpreted netlist on every object and the oracle on every pair."""
    tm = [field_template("K8sFields", n)]
    cons = [W._constraint("K8sFields", "fields", match=W.POD)]
    n_objs = 131   # (a partial last warp of objects and of containers)
    objs = field_page(n_objs, n)
    # check() reads the [spec check] line; the [spec types] line comes before it on stderr, so it is read from the dump's run here
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    orig = capfd.readouterr
    lines = []

    def keep():
        r = orig()
        lines.extend(r.err.splitlines())
        return r
    monkeypatch.setattr(capfd, "readouterr", keep)
    fold, big = check(tm, cons, objs, monkeypatch, capfd, tmp_path)
    assert big == sum(1 for i in range(n_objs) if i % 40 == 39)
    scopes, nbytes = types_line(lines)
    check_layout(scopes, nbytes)
    text = (tmp_path / "spec.cu").read_text()
    cont = [s for s in fold if s]   # (the container scope: the only nested one)
    assert len(cont) == 1, fold
    s = cont[0]
    nib, byte_loads = nibbles_in_text(text, s)
    if n < 4:
        assert s not in scopes and not nib and len(byte_loads) == n
        return
    assert scopes[s][0] == n and not byte_loads and len(nib) == n
    # column order: the k-th column of the scope is nibble k
    assert [8 * w + sh // 4 for _, (w, sh) in sorted(nib.items())] == list(range(n))
    w = tw_words(n)
    load = "uint32_t tw0 = GK_SPEC_LD(tws + row)" if w == 1 else "uint2 twv = " if w == 2 else "uint4 twv%d = " % (w // 4 - 1)
    assert load in text[text.index("exports of one row of scope %d " % s):]


def test_refresh_changes_a_scope_layout(monkeypatch, capfd, tmp_path):
    """A resident batch checked, then refreshed after a constraint that reads six more container fields was added: the container
    scope goes from 3 VT columns (byte loads) to 9 (two words per row), and the refreshed batch is checked again."""
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    tm = [field_template("K8sFieldsA", 3), field_template("K8sFieldsB", 6, first=3)]
    _, drv, _ = make_pair(tm, [W._constraint("K8sFieldsA", "a", match=W.POD)], lib_path=HOSTEMU)
    objs = field_page(97, 9)
    rb = drv.upload_blob(W.PyBlob([json.dumps(o).encode() for o in objs]))
    capfd.readouterr()
    r0 = rb.eval(k8s.AUDIT_EP)
    before = capfd.readouterr().err.splitlines()
    assert [ln for ln in before if ln.startswith("[spec check]")]
    s_before, _ = types_line(before)
    assert all(nvt != 3 for nvt, _, _ in s_before.values())
    cb = W._constraint("K8sFieldsB", "b", match=W.POD)
    drv.AddConstraint(cb)
    assert rb.refresh()["rebuilt"] is True
    capfd.readouterr()
    r1 = rb.eval(k8s.AUDIT_EP)
    after = capfd.readouterr().err.splitlines()
    assert [ln for ln in after if ln.startswith("[spec check]")]
    s_after, nbytes = types_line(after)
    check_layout(s_after, nbytes)
    assert any(nvt == 9 and w == 2 for nvt, w, _ in s_after.values()), s_after
    assert len(r1.constraints) == len(r0.constraints) + 1 and sum(r1.totals) > sum(r0.totals)
    rb.free()
    drv.close()


def test_expanded_batch(monkeypatch, capfd):
    """A GK_F_EXPAND batch (Deployments expanded into Pods: the resultants are a batch of their own) with every eval checked against
    the interpreted netlist: every call still equals a review of the page."""
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    X.case_every_call_equals_review(HOSTEMU, "blob")
    err = capfd.readouterr().err.splitlines()
    assert [ln for ln in err if ln.startswith("[spec check]")] and [ln for ln in err if ln.startswith("[spec types]")]


# ---- on the GPU

def gpu_case(monkeypatch, env, tm, cons, extra, docs):
    """The page through one build of the evaluation (env), at both enforcement points, before and after a refresh that adds `extra`."""
    from gatekeeper_b200 import driver as D
    from test_spec_planes import gpu_driver
    drv = gpu_driver(monkeypatch, tm, cons, env)
    rb = drv.upload_blob(W.PyBlob(docs))
    out = []
    for step in range(2):
        if step:
            drv.AddConstraint(extra)
            assert rb.refresh()["rebuilt"] is True
        for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP):
            r = rb.eval(ep, flags=D.F_MATERIALIZE)
            out.append((drv.last_kernel(), np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True), list(r.totals), list(r.err_totals),
                        sorted((x.object, x.constraint, x.msg) for x in r.results if x.autoreject)))
    rb.free()
    drv.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3, 9, 33])
def test_gpu_type_words_against_the_interpreter(n, monkeypatch):
    """Pages whose container scope has n VT columns (then n + 17 after a refresh adds a constraint), forced through the generated
    kernel: bitmaps, error planes, totals and matcher errors identical to the interpreter's at both enforcement points."""
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    tm = [field_template("K8sFieldsA", n), field_template("K8sFieldsB", 17, first=n)] + [t for t in W.config2()[0]]
    cons = [W._constraint("K8sFieldsA", "a", match=W.POD)] + W.config2()[1][:20]
    extra = W._constraint("K8sFieldsB", "b", match=W.POD)
    docs = [json.dumps(o).encode() for o in field_page(3 * 512 + 77, n + 17)]
    want = gpu_case(monkeypatch, {"GK_SPEC": "0"}, tm, cons, extra, docs)
    got = gpu_case(monkeypatch, {"GK_SPEC_MIN_OBJECTS": "0"}, tm, cons, extra, docs)
    for a, b in zip(want, got):
        assert a[0] == "gk_eval_kernel" and b[0] == "gk_spec_kernel", (a[0], b[0])
        for x, y, what in zip(a[1:], b[1:], ("violation bitmap", "error bitmap", "totals", "error totals", "matcher errors")):
            assert (x == y) if what == "matcher errors" else np.array_equal(x, y), (n, what)
    assert sum(want[0][3]) > 0 and sum(want[-1][3]) > sum(want[0][3])


@pytest.mark.gpu
def test_gpu_type_word_bytes_are_the_layout(monkeypatch, capfd):
    """The backend's type-word allocation for the config-2 page: the scopes and words the host build traces for the same page, each
    scope's words 16-byte aligned behind a pointer table of 8 bytes per scope."""
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    from test_spec_planes import gpu_driver
    tm, cons = W.config2()
    n = 2000
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    _, drv, _ = make_pair(tm, cons, W.synth_namespaces(), lib_path=HOSTEMU)
    capfd.readouterr()
    drv.ReviewBlob(W.synth_objects(0, n), k8s.AUDIT_EP, with_results=False)
    drv.close()
    scopes, _ = types_line(capfd.readouterr().err.splitlines())
    assert scopes
    drv = gpu_driver(monkeypatch, tm, cons, {"GK_SPEC_MIN_OBJECTS": "0", "GK_TRACE_LAUNCH": "1"})
    capfd.readouterr()
    drv.ReviewBlob(W.synth_objects(0, n), k8s.AUDIT_EP, with_results=False)
    assert drv.last_kernel() == "gk_spec_kernel"
    drv.close()
    got = re.findall(r"\[launch\] type words:(.*) (\d+) bytes for (\d+) objects", capfd.readouterr().err)
    assert got and got[-1][2] == str(n), got
    assert {int(s): (int(a), int(b)) for s, a, b in re.findall(r"scope (\d+): (\d+) vt columns in (\d+) words;", got[-1][0])} == \
        {s: (v[0], v[1]) for s, v in scopes.items()}
    table = int(got[-1][1]) - sum((4 * w * rows + 15) // 16 * 16 for _, w, rows in scopes.values())
    assert table % 16 == 0 and 8 * (1 + max(scopes)) <= table < 8 * 250 + 16, table
