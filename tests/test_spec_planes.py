"""The generated kernel's export planes (spec_codegen.cpp): gk_spec_rows_kernel stores a row loop's exports as bit planes, one 32 x 32
transpose per warp and export word (word (blk, k) of loop g = export k of rows 32 blk .. 32 blk + 31 of its scope), gk_spec_kernel copies the tile's
blocks of them with 16-byte copies, and the object walk reads each export of an object as one 32-bit window of its plane from the
object's first row.  On the test-only host emulation the same text (only the tile's own bits set in poisoned plane words, so a window
not masked to the object's rows shows) is compared object by object with the interpreted netlist (GK_SPEC_CHECK=1) and with the
oracle; the planes' size is checked against the layout restated here; on the GPU the kernels, forced at any page size, against the
interpreter."""
import json
import random
import re

import numpy as np
import pytest

import gpu_path_cases as G
from conftest import HOSTEMU, assert_same, has_cuda, make_pair
from gatekeeper_b200 import workloads as W
from oracle import k8s

from test_spec_fold import FOLD, allowed_repos, container, pod, tmpl
from test_spec_plan_hostemu import constraint_set
from test_spec_rows import _match_error_set

HOST_TILE, DEVICE_TILE = 96, 512
HOST_N, DEVICE_N = 3 * HOST_TILE + 41, 3 * DEVICE_TILE + 79   # (neither a multiple of 32 containers in all)
PLANES = re.compile(r"\[spec planes\](.*) (\d+) export words$")
LOOP = re.compile(r"loop (\d+): scope (\d+), (\d+) exports, (\d+) rows;")
MISSING_NS = "planes-no-such-namespace"


def container_counts(n):
    """Containers per object: the edges first, then a mix of 0 to 5 with a 32-row object every 61 and a 33-row (wide) one every 389."""
    head = [31, 2,        # rows 0-30; rows 31-32: starts at bit 31 of a block and runs into the next
            0,            # no rows
            32,           # rows 33-64: 32 rows, shift 1
            31,           # rows 65-95
            32,           # rows 96-127: 32 rows, shift 0
            33,           # wide: handed to the interpreter
            1]
    ks = head + [(i * 7 + i // 13) % 6 for i in range(len(head), n)]
    for i in range(len(head), n):
        if i % 61 == 17:
            ks[i] = 32
        if i % 389 == 101:
            ks[i] = 33
    return ks


def plane_page(n):
    """Pods with container_counts(n) containers, every fifth with init containers, every 37th in a Namespace that is not cached."""
    docs = []
    for i, k in enumerate(container_counts(n)):
        d = pod(i, [container(i + j) for j in range(k)], init=[container(1000 + i + j) for j in range(i % 3 + 1)] if i % 5 == 0 else ())
        if i % 37 == 3:
            d["metadata"]["namespace"] = MISSING_NS
        docs.append(json.dumps(d).encode())
    return docs


def test_the_page_covers_the_plane_edges():
    """What the cases below rely on: windows that start at bit 31 and cross a block, 32-row windows at shift 0 and not, objects with no
    rows and wide ones, tiles (of the host emulation and of the device) whose first container row is not on a block boundary, and a
    container count that is not a multiple of 32."""
    for n, tile in ((HOST_N, HOST_TILE), (DEVICE_N, DEVICE_TILE)):
        ks = container_counts(n)
        start = np.concatenate([[0], np.cumsum(ks)])
        assert any(k >= 2 and start[i] % 32 == 31 for i, k in enumerate(ks))
        assert {start[i] % 32 == 0 for i, k in enumerate(ks) if k == 32} == {True, False}
        assert 0 in ks and 33 in ks
        assert start[-1] % 32 != 0
        assert any(start[t] % 32 for t in range(tile, n, tile)), tile


def host_run(monkeypatch, capfd, tmp_path, tm, cons, docs, wide=True):
    """The page on the host emulation with the generated text checked against the interpreted netlist; every object with 32 or more
    containers, and a sample, against the oracle.  Returns the folding, the plane trace {loop: (scope, exports, rows)} and its words."""
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    monkeypatch.setenv("GK_SPEC_DUMP", str(tmp_path / "spec.cu"))
    orc, drv, _ = make_pair(tm, cons, W.synth_namespaces(), lib_path=HOSTEMU)
    rb = drv.upload_blob(W.PyBlob(docs))
    capfd.readouterr()
    r = rb.eval(k8s.AUDIT_EP)
    keys, viol, err = list(r.constraints), r.viol_bits.copy(), r.err_bits.copy()
    rb.free()
    drv.close()
    lines = capfd.readouterr().err.splitlines()
    check = [ln for ln in lines if ln.startswith("[spec check]")]
    assert check, "no [spec check] line: was the generated text checked?"
    n = len(docs)
    ks = container_counts(n)
    assert int(re.search(r"\((\d+) too big", check[-1]).group(1)) == (ks.count(33) if wide else 0), check[-1]
    plan = [ln for ln in lines if ln.startswith("[spec plan]")]
    assert plan and plan[-1].endswith("disagreements: 0"), plan
    objs = sorted({i for i, k in enumerate(ks) if k >= 31} | set(random.Random(n).sample(range(n), 60)))
    v, e = G.oracle_pairs(orc, docs, objs, k8s.AUDIT_EP)
    assert_same(v, G.bit_pairs(viol, keys, objs))
    assert_same(e, G.bit_pairs(err, keys, objs))
    m = [PLANES.match(ln) for ln in lines if ln.startswith("[spec planes]")]
    assert m and m[-1], "no [spec planes] line"
    loops = {int(x[0]): tuple(int(y) for y in x[1:]) for x in LOOP.findall(m[-1].group(1))}
    head = (tmp_path / "spec.cu").read_text().split("\n", 1)[0]
    fold = {int(x[0]): tuple(int(y) for y in x[1:]) for x in FOLD.findall(head)}
    return fold, loops, int(m[-1].group(2))


def plane_words(loops):
    """The layout restated: per row loop, roundup(exports, 4) planes, one word per plane per block of 32 rows, and one guard block."""
    return sum(((rows + 31) // 32 + 1) * ((e + 3) // 4 * 4) for _, e, rows in loops.values())


def check_layout(fold, loops, words, n):
    assert words == plane_words(loops)
    assert any(s == 0 and rows == n for s, _, rows in loops.values())
    for s, (_, _, any_, mask, w) in fold.items():   # the fold line's exports are the loop's
        assert [e for ls, e, _ in loops.values() if ls == s] == [any_ + mask], (s, loops)
        assert w == (any_ + mask + 31) // 32


def test_config2_edges(monkeypatch, capfd, tmp_path):
    """The config-2 constraints (and a namespaceSelector that makes the uncached Namespace's Pods matcher errors) over the edge page:
    row loops whose export count is not a multiple of 4, and a container count that is not a multiple of 32."""
    tm, cons = constraint_set()
    n = HOST_N
    fold, loops, words = host_run(monkeypatch, capfd, tmp_path, tm, cons, plane_page(n))
    check_layout(fold, loops, words, n)
    assert any(e % 4 for _, e, _ in loops.values()), loops
    assert sum(container_counts(n)) in {rows for _, _, rows in loops.values()}


def test_two_export_words_per_row(monkeypatch, capfd, tmp_path):
    """A container row loop with 33 to 64 exports: two words per row before the transpose, planes past the first 32."""
    tm, cons = _match_error_set()
    cons = cons + [allowed_repos(100 + i, template="allowedrepos_prefixmatch") for i in range(14)]
    n = 2 * HOST_TILE + 13
    fold, loops, words = host_run(monkeypatch, capfd, tmp_path, tm, cons, plane_page(n))
    check_layout(fold, loops, words, n)
    assert any(32 < e <= 64 for _, e, _ in loops.values()), loops


def test_exports_on_the_object_row_only(monkeypatch, capfd, tmp_path):
    """K8sPSPHostNamespace alone: every export is on the object's own row (scope 0), whose window is one bit."""
    tm = tmpl("psp_hostnamespace")
    cons = [W._constraint(tm[0][0], "hostns", match=W.POD)]
    n = HOST_TILE + 50
    docs = plane_page(n)
    for i in range(0, n, 3):
        d = json.loads(docs[i])
        d["spec"]["hostPID"] = i % 2 == 0
        docs[i] = json.dumps(d).encode()
    fold, loops, words = host_run(monkeypatch, capfd, tmp_path, tm, cons, docs, wide=False)   # (no nested scope: nothing is wide)
    assert list(fold) == [0] and {s for s, _, _ in loops.values()} == {0}, (fold, loops)
    check_layout(fold, loops, words, n)


def test_config2_page_plane_bytes(monkeypatch, capfd, tmp_path):
    """The flagship page (synthetic Pods under config 2): the planes are the restated layout, and smaller than one word per row."""
    tm, cons = W.config2()
    n = 2000
    blob = W.synth_objects(0, n)
    fold, loops, words = host_run_blob(monkeypatch, capfd, tmp_path, tm, cons, blob)
    check_layout(fold, loops, words, n)
    assert words < sum(rows * ((e + 31) // 32) for _, e, rows in loops.values())


def host_run_blob(monkeypatch, capfd, tmp_path, tm, cons, blob):
    monkeypatch.setenv("GK_SPEC_CHECK", "1")
    monkeypatch.setenv("GK_SPEC_TRACE", "1")
    monkeypatch.setenv("GK_SPEC_DUMP", str(tmp_path / "spec.cu"))
    _, drv, _ = make_pair(tm, cons, W.synth_namespaces(), lib_path=HOSTEMU)
    capfd.readouterr()
    drv.ReviewBlob(blob, k8s.AUDIT_EP, with_results=False)
    drv.close()
    lines = capfd.readouterr().err.splitlines()
    assert [ln for ln in lines if ln.startswith("[spec check]")], "no [spec check] line: was the generated text checked?"
    m = [PLANES.match(ln) for ln in lines if ln.startswith("[spec planes]")]
    assert m and m[-1], "no [spec planes] line"
    loops = {int(x[0]): tuple(int(y) for y in x[1:]) for x in LOOP.findall(m[-1].group(1))}
    head = (tmp_path / "spec.cu").read_text().split("\n", 1)[0]
    return {int(x[0]): tuple(int(y) for y in x[1:]) for x in FOLD.findall(head)}, loops, int(m[-1].group(2))


def test_text_compiles_with_nvrtc_and_walks_no_rows(monkeypatch, capfd, tmp_path):
    """The config-2 text builds both entry points with NVRTC (the backend's options); the rows kernel transposes, and the object walk
    has no per-row loop left: its only loops are the range loops over parent rows."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("spec_nvrtc", os.path.join(os.path.dirname(os.path.dirname(__file__)), "tools", "spec_nvrtc.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    tm, cons = W.config2()
    host_run_blob(monkeypatch, capfd, tmp_path, tm, cons, W.synth_objects(0, 300))
    text = (tmp_path / "spec.cu").read_text()
    walk = text[text.index("GK_SPEC_FN bool gk_spec_object"):text.index("#define GK_SPEC_NS ")]
    rows = text[text.index("gk_spec_rows_kernel("):text.index("GK_SPEC_FN void gk_spec_stage")]
    assert "gk_tr32(a0, lane)" in rows and "GK_SPEC_FUNNEL(" in walk
    assert re.findall(r"for \(uint32_t (\w+) = ", walk) and set(re.findall(r"for \(uint32_t (\w+) = ", walk)) == {"pj"}
    try:
        cubin, _, _ = tool.nvrtc_compile(text.encode())
    except RuntimeError as e:
        if "libnvrtc not found" in str(e):
            pytest.skip("no NVRTC in this container")
        raise
    assert b"gk_spec_rows_kernel" in cubin and b"gk_spec_kernel" in cubin


# ---- on the GPU

def gpu_driver(monkeypatch, tm, cons, env):
    from gatekeeper_b200 import driver as D
    for k in ("GK_SPEC", "GK_SPEC_MIN_OBJECTS", "GK_SPEC_CHECK", "GK_SPEC_TRACE", "GK_SPEC_DUMP", "GK_TRACE_LAUNCH"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    drv = D.Driver()
    for k, r in tm:
        drv.add_template(k, r)
    for c in cons:
        drv.AddConstraint(c)
    for ns in W.synth_namespaces():
        drv.AddData("admission.k8s.gatekeeper.sh", ["cluster", "v1", "Namespace", ns["metadata"]["name"]], ns)
    return drv


def gpu_results(monkeypatch, tm, cons, docs, env):
    from gatekeeper_b200 import driver as D
    drv = gpu_driver(monkeypatch, tm, cons, env)
    rb = drv.upload_blob(W.PyBlob(docs))
    out = {}
    for ep in (k8s.AUDIT_EP, k8s.WEBHOOK_EP):
        r = rb.eval(ep, flags=D.F_MATERIALIZE)
        out[ep] = (drv.last_kernel(), np.array(r.viol_bits, copy=True), np.array(r.err_bits, copy=True), list(r.totals), list(r.err_totals),
                   sorted((x.object, x.constraint, x.msg) for x in r.results if x.autoreject))
    rb.free()
    drv.close()
    return out


def _two_word_set():
    tm, cons = _match_error_set()
    return tm, cons + [allowed_repos(100 + i, template="allowedrepos_prefixmatch") for i in range(14)]


def _own_row_set():
    tm = tmpl("psp_hostnamespace")
    return tm, [W._constraint(tm[0][0], "hostns", match=W.POD)]


GPU_SETS = {"config2_edges": constraint_set, "two_export_words": _two_word_set, "own_row_only": _own_row_set}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(GPU_SETS))
def test_gpu_planes_against_the_interpreter(case, monkeypatch):
    """The edge page over three device tiles and a partial one, forced through the generated kernel: bitmaps, error planes, totals and
    matcher errors identical to the interpreter's at both enforcement points."""
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    tm, cons = GPU_SETS[case]()
    docs = plane_page(DEVICE_N)
    want = gpu_results(monkeypatch, tm, cons, docs, {"GK_SPEC": "0"})
    got = gpu_results(monkeypatch, tm, cons, docs, {"GK_SPEC_MIN_OBJECTS": "0"})
    for ep in want:
        assert want[ep][0] == "gk_eval_kernel" and got[ep][0] == "gk_spec_kernel", (ep, want[ep][0], got[ep][0])
        for a, b, what in zip(want[ep][1:], got[ep][1:], ("violation bitmap", "error bitmap", "totals", "error totals", "matcher errors")):
            assert (a == b) if what == "matcher errors" else np.array_equal(a, b), (case, ep, what)
    if case == "config2_edges":
        assert sum(want[k8s.AUDIT_EP][3]) > 0 and sum(want[k8s.AUDIT_EP][4]) > 0


@pytest.mark.gpu
def test_gpu_plane_bytes_are_the_layout(monkeypatch, capfd, tmp_path):
    """The backend's export-plane allocation for the config-2 page is the layout the host build traces for the same page."""
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    tm, cons = W.config2()
    n = 2000
    fold, loops, words = host_run_blob(monkeypatch, capfd, tmp_path, tm, cons, W.synth_objects(0, n))
    check_layout(fold, loops, words, n)
    drv = gpu_driver(monkeypatch, tm, cons, {"GK_SPEC_MIN_OBJECTS": "0", "GK_TRACE_LAUNCH": "1"})
    capfd.readouterr()
    drv.ReviewBlob(W.synth_objects(0, n), k8s.AUDIT_EP, with_results=False)
    assert drv.last_kernel() == "gk_spec_kernel"
    drv.close()
    got = re.findall(r"\[spec\] export arrays: (\d+) bytes for (\d+) objects", capfd.readouterr().err)
    assert got == [(str(4 * words), str(n))], got


@pytest.mark.gpu
def test_gpu_fused_exchange_of_the_edge_page(monkeypatch):
    """eval_device_peers of one rank whose only peer buffer is its own, over the edge page: the bitmap and both totals arrive.  The
    buffers start as 0xff bytes, so a word nobody stores shows."""
    import torch
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    tm, cons = constraint_set()
    n = DEVICE_N
    drv = gpu_driver(monkeypatch, tm, cons, {"GK_SPEC_MIN_OBJECTS": "0"})
    rb = drv.upload_blob(W.PyBlob(plane_page(n)))
    ref = rb.eval(k8s.AUDIT_EP)
    C, words = len(ref.totals), ref.viol_bits.shape[1]
    assert sum(ref.totals) > 0
    dev = torch.device("cuda", 0)
    side = torch.cuda.Stream(device=dev)
    tot_off = n * words + (n * words) % 2
    slot = tot_off + 4 * C
    recv = torch.full((slot,), -1, dtype=torch.int32, device=dev)
    err = torch.full((n, words), -1, dtype=torch.int32, device=dev)
    tot = torch.full((2, C), -1, dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    rb.eval_device_peers(k8s.AUDIT_EP, [recv.data_ptr()], 0, slot, tot_off, C, err.data_ptr(), tot[0].data_ptr(), tot[1].data_ptr(), side.cuda_stream)
    assert drv.last_kernel() == "gk_spec_kernel"
    side.synchronize()
    assert np.array_equal(recv[:n * words].view(n, words).cpu().numpy().view(np.uint32), ref.viol_bits)
    assert np.array_equal(err.cpu().numpy().view(np.uint32), ref.err_bits)
    published = recv[tot_off:].contiguous().view(torch.int64).view(2, C)
    assert published[0].tolist() == ref.totals and published[1].tolist() == ref.err_totals
    assert tot[0].tolist() == ref.totals and tot[1].tolist() == ref.err_totals
    rb.free()
    drv.close()
