"""Compile a dumped generated text (tools/spec_dump.py) with NVRTC exactly as the CUDA backend does (kernels.cu: spec_compile) and
print the static picture of each entry point (gk_spec_rows_kernel, gk_spec_kernel): registers, spills, SASS instruction count, and
instructions per source region.  No GPU needed (NVRTC and cuobjdump / nvdisasm run without a device); these are static numbers,
never a timing.

    python tools/spec_nvrtc.py /tmp/spec/config2.cu [--threads 256] [--minb 3] [--rows-threads 256] [--rows-minb 6] [--defs "-DGK_SPEC_X_NOMATCH"]
"""
import argparse
import collections
import ctypes
import os
import re
import subprocess
import sys
import time


def nvrtc_compile(src: bytes, threads=256, minb=3, defs=(), rows_threads=256, rows_minb=6):
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
    opts = [b"--gpu-architecture=sm_90a", b"-std=c++17", b"-lineinfo", b"-default-device", b"-DGK_SPEC_THREADS=%d" % threads, b"-DGK_SPEC_MINB=%d" % minb,
            b"-DGK_SPEC_ROWS_THREADS=%d" % rows_threads, b"-DGK_SPEC_ROWS_MINB=%d" % rows_minb]
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
    """-> (["<entry point>: REG:.. STACK:..", ...], SASS instructions, Counter of instructions per region).  A region names the entry
    point it was counted in ("rows: ..." / "tile: ..."); shared code (the match blocks) is counted where it is inlined."""
    res = subprocess.run(["cuobjdump", "-res-usage", cubin_path], capture_output=True, text=True).stdout
    usage, fn = [], "?"
    for ln in res.splitlines():
        m = re.match(r"\s*Function (\w+):", ln)
        if m:
            fn = m.group(1)
        elif "REG:" in ln:
            usage.append(fn + ": " + ln.strip())
    sass = subprocess.run(["nvdisasm", "--print-line-info", cubin_path], capture_output=True, text=True).stdout
    src = open(cu_path).read().split("\n")
    start = next(i for i, s in enumerate(src) if "GK_SPEC_FN bool gk_spec_object" in s) + 1
    end = next(i for i, s in enumerate(src) if s.startswith("#ifndef GK_SPEC_HOST") and i > start)
    stage = next((i for i, s in enumerate(src) if "GK_SPEC_FN void gk_spec_stage" in s), start) + 1
    rows = next((i for i, s in enumerate(src) if "GK_SPEC_FN void gk_spec_row_" in s), stage) + 1
    cur, kern = None, "?"
    region = collections.Counter()
    total = 0
    for ln in sass.splitlines():
        m = re.search(r"\.text\.(\w+)", ln)
        if m and ".section" in ln:
            kern = "rows" if m.group(1) == "gk_spec_rows_kernel" else "tile" if m.group(1) == "gk_spec_kernel" else m.group(1)
            continue
        m = re.search(r'//## File "[^"]*", line (\d+)', ln)
        if m:
            cur = int(m.group(1))
            continue
        if INSN.match(ln):
            total += 1
            if cur is None:
                region[kern + ": ?"] += 1
            elif rows <= cur < stage:
                s = src[cur - 1].strip()
                if s.endswith("// row-local gate"):
                    region["rows: row-local gates"] += 1
                elif re.match(r"if \(v\d+\) a\d+ \|= ", s) or re.match(r"xg\[", s):
                    region["rows: export bits packed and stored"] += 1
                elif "GK_SPEC_MATCH" in s or "GK_SPEC_ERR" in s or "skip" in s:
                    region["rows: match call sites"] += 1
                else:
                    region["rows: loads, atoms, control"] += 1
            elif stage <= cur < start:
                region["tile: copy of the exports and offsets" if kern == "tile" else kern + ": offset image and wide test"] += 1
            elif cur < start:
                region[kern + ": spec.match (written-out blocks / vm_core.h)"] += 1
            elif cur < end:
                s = src[cur - 1].strip()
                if "rm =" in s or s.startswith("for (uint32_t pj") or "pj" in s:
                    region["tile: object: EXISTS / broadcast range loops"] += 1
                elif s.startswith("if (") and "|= bit" in s:
                    region["tile: object: export bits, mask form"] += 1
                elif re.match(r"x\d+_\d+ \|= w\d+;", s) or re.match(r"const uint32_t v\d+ = \(x\d+_\d+ >> ", s):
                    region["tile: object: export bits, any form"] += 1
                elif "GK_SPEC_LD(p" in s or "_Pragma" in s or "bit = " in s or re.search(r"\bw0 = a\d+\[", s):
                    region["tile: object: row loops (loads, control)"] += 1
                elif "vw[" in s or "ew[" in s or s.startswith("if (act["):
                    region["tile: object: results"] += 1
                else:
                    region["tile: object: gates, scope offsets, other"] += 1
            else:
                region["tile: launch wrapper (stores, totals)"] += 1
    return usage, total, region


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("cu")
    ap.add_argument("--threads", type=int, default=256)
    ap.add_argument("--minb", type=int, default=3)
    ap.add_argument("--rows-threads", type=int, default=256)
    ap.add_argument("--rows-minb", type=int, default=6)
    ap.add_argument("--defs", default="")
    a = ap.parse_args()
    cubin, log, dt = nvrtc_compile(open(a.cu, "rb").read(), a.threads, a.minb, a.defs.split(), a.rows_threads, a.rows_minb)
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
