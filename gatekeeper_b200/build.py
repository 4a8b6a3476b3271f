"""In-tree build of the native libraries (no JIT cache: the .so files travel with the repo snapshot).

  gatekeeper_b200/libgk_engine.so   -- the product: C++ host engine + CUDA kernels for sm_90a (nvcc)
  tests/_hostemu/libgk_hostemu.so   -- TEST-ONLY: same host engine linked against the CPU emulation backend
  gatekeeper_b200/libgk_synth.so    -- deterministic synthetic workload generator (bench / tests), not part of the engine
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "gatekeeper_b200", "csrc")
OBJ = os.path.join(ROOT, "build", "obj")
LIB = os.path.join(ROOT, "gatekeeper_b200", "libgk_engine.so")
EMU = os.path.join(ROOT, "tests", "_hostemu", "libgk_hostemu.so")

HOST_SRCS = ["val.cpp", "rego_parse.cpp", "rego_eval.cpp", "lower.cpp", "xprog.cpp", "expansion.cpp", "engine.cpp", "audit.cpp", "capi.cpp", "coalescer.cpp", "spec_codegen.cpp"]
SYNTH = os.path.join(ROOT, "gatekeeper_b200", "libgk_synth.so")
CXXFLAGS = ["-std=c++17", "-O2", "-g1", "-fPIC", "-Wall", "-Wextra", "-pthread", "-I", OBJ]
NVCCFLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O3", "-lineinfo", "-Xcompiler", "-fPIC"]


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _deps_mtime():
    m = 0.0
    for d in (CSRC, os.path.join(ROOT, "include")):
        for f in os.listdir(d):
            if f.endswith((".h", ".hpp", ".cuh")):
                m = max(m, os.path.getmtime(os.path.join(d, f)))
    return m


def _stale(out, srcs, hdr_m):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(s) > t for s in srcs) or hdr_m > t


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
    return r.stdout + r.stderr


def build_variant(suffix, defines):
    """Kernel experiment: libgk_engine<suffix>.so with extra -D flags on the CUDA translation unit
    (select it with GK_ENGINE_LIB=...).  The host objects of the regular build are reused."""
    build()
    ko = os.path.join(OBJ, "kernels%s.cu.o" % suffix)
    _run([_nvcc(), *NVCCFLAGS, *["-D" + d for d in defines], "-c", os.path.join(CSRC, "kernels.cu"), "-o", ko])
    objs = [os.path.join(OBJ, s + ".o") for s in HOST_SRCS]
    out = os.path.join(ROOT, "gatekeeper_b200", "libgk_engine%s.so" % suffix)
    _run([_nvcc(), "-shared", "-o", out, *objs, ko, "-Xcompiler", "-pthread", "-cudart", "static", "-ldl"])
    return out


def _spec_headers():
    """program.h and vm_core.h as string literals: the kernel generated for a constraint set (spec_codegen.cpp) is one
    self-contained translation unit that NVRTC compiles at run time, with no include path to find them on."""
    out = os.path.join(OBJ, "spec_headers.inc")
    txt = ""
    for name, f in (("kSpecHdrProgram", "program.h"), ("kSpecHdrVmCore", "vm_core.h")):
        body = open(os.path.join(CSRC, f)).read()
        assert ')GKHDR"' not in body
        txt += 'static const char %s[] = R"GKHDR(%s)GKHDR";\n' % (name, body)
    if not os.path.exists(out) or open(out).read() != txt:
        with open(out, "w") as fh:
            fh.write(txt)


def build(verbose=False, hostemu=True, force=False):
    os.makedirs(OBJ, exist_ok=True)
    _spec_headers()
    hdr_m = _deps_mtime()
    jobs = []
    objs = []
    for s in HOST_SRCS:
        src = os.path.join(CSRC, s)
        if not os.path.exists(src):
            continue
        o = os.path.join(OBJ, s + ".o")
        objs.append(o)
        if force or _stale(o, [src], hdr_m):
            jobs.append(["g++", *CXXFLAGS, "-c", src, "-o", o])
    ko = os.path.join(OBJ, "kernels.cu.o")
    ksrc = os.path.join(CSRC, "kernels.cu")
    if force or _stale(ko, [ksrc], hdr_m):
        jobs.append([_nvcc(), *NVCCFLAGS, "-c", ksrc, "-o", ko])
    eo = os.path.join(OBJ, "hostemu.cpp.o")
    esrc = os.path.join(ROOT, "tests", "_hostemu", "hostemu.cpp")
    if hostemu and (force or _stale(eo, [esrc], hdr_m)):
        jobs.append(["g++", *CXXFLAGS, "-c", esrc, "-o", eo])
    with ThreadPoolExecutor(max_workers=8) as ex:
        for out in ex.map(_run, jobs):
            if verbose and out.strip():
                print(out)
    if force or _stale(LIB, objs + [ko], 0):
        _run([_nvcc(), "-shared", "-o", LIB, *objs, ko, "-Xcompiler", "-pthread", "-cudart", "static", "-ldl"])
    if hostemu and (force or _stale(EMU, objs + [eo], 0)):
        _run(["g++", "-shared", "-o", EMU, *objs, eo, "-pthread", "-ldl"])
    # TEST / BENCH ONLY: the C++ CPU restatement of the reference's review loop (oracle/cpu_ref.cpp) over the engine's host objects
    csrc = os.path.join(ROOT, "oracle", "cpu_ref.cpp")
    cdir = os.path.join(ROOT, "oracle", "_build")
    os.makedirs(cdir, exist_ok=True)
    co = os.path.join(OBJ, "cpu_ref.cpp.o")
    if force or _stale(co, [csrc], hdr_m):
        _run(["g++", *CXXFLAGS, "-c", csrc, "-o", co])
    cobjs = [os.path.join(OBJ, s + ".o") for s in ("val.cpp", "rego_parse.cpp", "rego_eval.cpp", "lower.cpp", "xprog.cpp", "expansion.cpp", "engine.cpp")]
    CPUREF = os.path.join(cdir, "libgk_cpuref.so")
    if force or _stale(CPUREF, cobjs + [co], 0):
        _run(["g++", "-shared", "-o", CPUREF, *cobjs, co, "-pthread"])
    ssrc = os.path.join(CSRC, "synth.cpp")
    if force or _stale(SYNTH, [ssrc], 0):
        _run(["g++", *CXXFLAGS, "-shared", "-o", SYNTH, ssrc])
    return LIB


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--variant":      # python build.py --variant _timing GK_PHASE_TIMING=1 ...
        print("built", build_variant(sys.argv[2], sys.argv[3:]))
    else:
        build(verbose=True, force="--force" in sys.argv)
        print("built", LIB)
