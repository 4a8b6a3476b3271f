"""tests/c_abi/patch.c -- the Go shim's PatchBatch repeated call for call in C (this image has no Go toolchain): a config-2 page
uploaded with GK_F_KEEP_SOURCE, patched through gk_batch_patch from C memory, must give the violation plane of a fresh upload of the
resulting page, and the refused calls must return GK_ERR_INVALID and leave the batch's size as it was.  CPU: linked against the test
backend's library (same C ABI); `-m gpu`: the product."""
import json
import os
import subprocess

import pytest

import batch_refresh_cases as R
from conftest import HOSTEMU, ROOT, has_cuda
from gatekeeper_b200 import workloads as W

SRC = os.path.join(ROOT, "tests", "c_abi", "patch.c")
BIN = os.path.join(ROOT, "build", "c_abi_patch")


def _build():
    os.makedirs(os.path.dirname(BIN), exist_ok=True)
    if not os.path.exists(BIN) or os.path.getmtime(BIN) < os.path.getmtime(SRC):
        subprocess.run(["gcc", "-O1", "-Wall", "-o", BIN, SRC, "-ldl"], check=True)


def _run(lib, tmp_path, n=60):
    tm, cons = W.config2()
    docs = R.damaged_page(n, start=99800)
    drop = [0, 7, 20, len(docs) - 1]
    added = [docs[20], json.dumps(json.loads(W.synth_objects(99900, 1).get(0))).encode(), R.BAD_DOCS[0]]
    path = os.path.join(str(tmp_path), "patch_in.txt")
    with open(path, "wb") as f:
        for kind, rego in tm:
            b = rego.encode()
            f.write(b"T %s %d\n" % (kind.encode(), len(b)) + b + b"\n")
        for c in cons:
            b = json.dumps(c).encode()
            f.write(b"C %d\n" % len(b) + b + b"\n")
        for tag, lst in ((b"D", docs), (b"A", added)):
            for d in lst:
                f.write(tag + b" %d\n" % len(d) + d + b"\n")
        for x in drop:
            f.write(b"X %d\n" % x)
    out = subprocess.run([BIN, lib, path], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr
    lines = [ln.split("\t") for ln in out.stdout.splitlines()]
    size = len(docs) - len(drop) + len(added)
    assert ["N", str(size)] in lines, lines[:3]
    patched = [ln[1:] for ln in lines if ln[0] == "P"]
    fresh = [ln[1:] for ln in lines if ln[0] == "F"]
    assert len(patched) == size and patched == fresh
    assert any(int(w) for ln in patched for w in ln[1:]), "the page has violations"
    for what in ("DUP", "RANGE", "NOSOURCE"):
        assert [what, "-1"] in lines, (what, lines[-4:])
    assert ["SIZE", str(size)] in lines
    return size


def test_c_patch_of_the_go_shim_on_the_test_backend(tmp_path):
    _build()
    _run(HOSTEMU, tmp_path)


@pytest.mark.gpu
def test_c_patch_of_the_go_shim_on_the_cuda_library(tmp_path):
    if not has_cuda():
        pytest.fail("GPU tests selected but no CUDA device is visible")
    _build()
    _run(os.path.join(ROOT, "gatekeeper_b200", "libgk_engine.so"), tmp_path)
