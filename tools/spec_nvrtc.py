"""Compile a dumped generated kernel (tools/spec_dump.py) with NVRTC exactly as the CUDA backend does (kernels.cu: spec_compile) and
print the static picture: registers, spills, SASS instruction count, instructions per source region.  No GPU needed (NVRTC and
cuobjdump / nvdisasm run in the authoring container); these are static numbers, never a timing.

    python tools/spec_nvrtc.py /tmp/spec/config2.cu [--threads 256] [--minb 3] [--defs "-DGK_SPEC_X_NOMATCH"]
"""
import argparse
import collections
import ctypes
import os
import re
import subprocess
import sys
import time


def nvrtc_compile(src: bytes, threads=256, minb=3, defs=()):
    """-> (cubin bytes, log text, seconds).  Raises RuntimeError with the log when the text does not compile."""
    h = None
    for name in ("libnvrtc.so.12", "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so", "/usr/local/cuda/lib64/libnvrtc.so"):
        try:
            h = ctypes.CDLL(name)
            break
        except OSError:
            continue
    if h is None:
        raise RuntimeError("libnvrtc not found")
    prog = ctypes.c_void_p()
    if h.nvrtcCreateProgram(ctypes.byref(prog), src, b"gk_spec_kernel.cu", 0, None, None) != 0:
        raise RuntimeError("nvrtcCreateProgram failed")
    opts = [b"--gpu-architecture=sm_90a", b"-std=c++17", b"-lineinfo", b"-default-device", b"-DGK_SPEC_THREADS=%d" % threads, b"-DGK_SPEC_MINB=%d" % minb]
    opts += [d.encode() for d in defs]
    arr = (ctypes.c_char_p * len(opts))(*opts)
    t0 = time.time()
    rc = h.nvrtcCompileProgram(prog, len(opts), arr)
    dt = time.time() - t0
    n = ctypes.c_size_t()
    h.nvrtcGetProgramLogSize(prog, ctypes.byref(n))
    buf = ctypes.create_string_buffer(max(1, n.value))
    h.nvrtcGetProgramLog(prog, buf)
    log = buf.value.decode(errors="replace")
    if rc != 0:
        h.nvrtcDestroyProgram(ctypes.byref(prog))
        raise RuntimeError("NVRTC rc %d:\n%s" % (rc, log[:4000]))
    h.nvrtcGetCUBINSize(prog, ctypes.byref(n))
    cub = ctypes.create_string_buffer(n.value)
    h.nvrtcGetCUBIN(prog, cub)
    h.nvrtcDestroyProgram(ctypes.byref(prog))
    return cub.raw, log, dt


INSN = re.compile(r"^\s+/\*[0-9a-f]{4,}\*/\s+[A-Z@!]")


def static_report(cubin_path: str, cu_path: str):
    res = subprocess.run(["cuobjdump", "-res-usage", cubin_path], capture_output=True, text=True).stdout
    usage = [ln.strip() for ln in res.splitlines() if "REG:" in ln]
    sass = subprocess.run(["nvdisasm", "--print-line-info", cubin_path], capture_output=True, text=True).stdout
    src = open(cu_path).read().split("\n")
    start = next(i for i, s in enumerate(src) if "GK_SPEC_FN bool gk_spec_object" in s) + 1
    end = next(i for i, s in enumerate(src) if s.startswith("#ifndef GK_SPEC_HOST") and i > start)
    stage = next((i for i, s in enumerate(src) if "GK_SPEC_FN void gk_spec_stage" in s), start) + 1
    cur = None
    region = collections.Counter()
    total = 0
    for ln in sass.splitlines():
        m = re.search(r'//## File "[^"]*", line (\d+)', ln)
        if m:
            cur = int(m.group(1))
            continue
        if INSN.match(ln):
            total += 1
            if cur is None:
                region["?"] += 1
            elif stage <= cur < start:
                s = src[cur - 1].strip()
                if s.endswith("// row-local gate"):
                    region["stage: row-local gates"] += 1
                elif re.match(r"if \(v\d+\) a\d+ \|= ", s) or re.match(r"stg\[R\d+ ", s):
                    region["stage: export bits packed and stored"] += 1
                else:
                    region["stage: loads, atoms, offsets, control"] += 1
            elif cur < start:
                region["spec.match (written-out blocks / vm_core.h)"] += 1
            elif cur < end:
                s = src[cur - 1].strip()
                if "rm =" in s or s.startswith("for (uint32_t pj") or "pj" in s:
                    region["object: EXISTS / broadcast range loops"] += 1
                elif s.startswith("if (") and "|= bit" in s:
                    region["object: export bits, mask form"] += 1
                elif re.match(r"x\d+_\d+ \|= w\d+;", s) or re.match(r"const uint32_t v\d+ = \(x\d+_\d+ >> ", s):
                    region["object: export bits, any form"] += 1
                elif "GK_SPEC_LD(p" in s or "_Pragma" in s or "bit = " in s or re.search(r"\bw0 = a\d+\[", s):
                    region["object: row loops (loads, control)"] += 1
                elif "GK_SPEC_MATCH" in s or "GK_SPEC_ERR" in s:
                    region["object: match call sites"] += 1
                elif "vw[" in s or "ew[" in s or s.startswith("if (act["):
                    region["object: results"] += 1
                else:
                    region["object: gates, scope offsets, other"] += 1
            else:
                region["launch wrapper (staging, stores, totals)"] += 1
    return usage, total, region


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("cu")
    ap.add_argument("--threads", type=int, default=256)
    ap.add_argument("--minb", type=int, default=3)
    ap.add_argument("--defs", default="")
    a = ap.parse_args()
    cubin, log, dt = nvrtc_compile(open(a.cu, "rb").read(), a.threads, a.minb, a.defs.split())
    out = os.path.splitext(a.cu)[0] + ".cubin"
    open(out, "wb").write(cubin)
    usage, total, region = static_report(out, a.cu)
    print("NVRTC %.1f s, %d bytes of cubin" % (dt, len(cubin)))
    for u in usage:
        print(u)
    print("SASS instructions:", total)
    for k, v in region.most_common():
        print("  %5d  %s" % (v, k))
    sys.exit(0)
