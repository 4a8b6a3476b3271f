"""eval_layout.h -- the interpreter's shared-memory layout, the slot area of a tile and the tile-size search -- through a small C++
harness (tests/eval_layout/check.cpp) compiled with g++: the same header gk_eval_kernel carves its shared memory with and the CUDA
backend sizes its launches and tiles with."""
import os
import subprocess

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "gatekeeper_b200", "csrc")
SRC = os.path.join(ROOT, "tests", "eval_layout", "check.cpp")
BIN = os.path.join(ROOT, "build", "eval_layout_check")
DEPS = [SRC, os.path.join(CSRC, "eval_layout.h"), os.path.join(CSRC, "program.h")]

REGIONS = ["s_tot", "s_err", "s_act", "s_lo", "s_cnt", "s_poff", "slots", "outs", "ops", "items", "match", "cols", "scopes", "pool", "cbytes"]


@pytest.fixture(scope="module")
def ask():
    os.makedirs(os.path.dirname(BIN), exist_ok=True)
    if not os.path.exists(BIN) or os.path.getmtime(BIN) < max(os.path.getmtime(d) for d in DEPS):
        subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", CSRC, "-o", BIN, SRC], check=True)

    def run(*requests):
        out = subprocess.run([BIN], input="".join(" ".join(str(x) for x in r) + "\n" for r in requests), capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
        lines = [ln.split() for ln in out.stdout.splitlines()]
        assert [ln[0] for ln in lines] == [str(r[0]) for r in requests]
        return [ln[1:] for ln in lines]
    return run


# (C, NS, NP, slot_words, nops, nitems, nmatch, ncols, npool, ncbytes) and the launch size added up by hand, term by term:
# 3*r16(4C) + 2*r16(4NS) + r16(4(NP+1)) + r16(4 slot_words) + 64 + r16(8C) + r16(16 nops) + r16(4 nitems) + r16(64 nmatch)
# + r16(64 ncols) + r16(16 NS) + r16(4 npool) + r16(ncbytes).  Resident CTAs per SM follow from this total: it must not drift.
LAYOUTS = [
    # shaped like config 2: 50 constraints, 14 iterated scopes + the root, 10 phases, 61 columns, 5 match blocks
    ((50, 15, 10, 6000, 450, 413, 5, 61, 900, 301),
     624 + 128 + 48 + 24000 + 64 + 400 + 7200 + 1664 + 320 + 3904 + 240 + 3600 + 304),   # = 42496
    # config 3: 200 constraints, 7 bitmap words per object
    ((200, 9, 7, 3000, 1200, 900, 1, 30, 500, 77),
     2400 + 96 + 32 + 12000 + 64 + 1600 + 19200 + 3600 + 64 + 1920 + 144 + 2000 + 80),    # = 43200
    # one of everything, no match blocks and no columns: empty regions take no room
    ((1, 1, 1, 4, 1, 1, 0, 0, 1, 1),
     48 + 32 + 16 + 16 + 64 + 16 + 16 + 16 + 0 + 0 + 16 + 16 + 16),                       # = 272
]


@pytest.mark.parametrize("counts,total", LAYOUTS)
def test_shared_memory_layout(ask, counts, total):
    got, sizes = ask(("layout", *counts), ("sizes", ))
    off = [int(x) for x in got]
    outent, op, match, column, scope = (int(x) for x in sizes)
    C, NS, NP, sw, nops, nitems, nmatch, ncols, npool, ncbytes = counts
    need = [4 * C, 4 * C, 4 * C, 4 * NS, 4 * NS, 4 * (NP + 1), 4 * sw, outent * C, op * nops, 4 * nitems, match * nmatch,
            column * ncols, scope * NS, 4 * npool, ncbytes]
    assert len(off) == len(REGIONS) + 2
    assert off[0] == 0
    for i, name in enumerate(REGIONS):
        assert off[i] % 16 == 0, name
        assert off[i] + need[i] <= off[i + 1], name        # large enough for its count, and in the kernel's order
        assert off[i + 1] - off[i] < need[i] + 16, name    # padded to 16 bytes, no more
    end, tot = off[-2], off[-1]
    assert end % 16 == 0 and tot == end + 64
    assert tot == total


def test_slot_layout(ask):
    cap = [512, 7, 100, 1000, 0]                  # cap[0] is the tile
    levels = [0, 1, 1, 2, 0, 2, 3, 4, 3]
    (got, ) = ask(("slots", len(cap), *cap, len(levels), *levels))
    words = [((cap[lv] + 31) // 32 + 1 + 3) & ~3 for lv in levels]
    assert words[:4] == [20, 4, 4, 8]
    offs = [sum(words[:i]) for i in range(len(words))]
    assert [int(x) for x in got] == [sum(words)] + offs


# tile-size search: one decision netlist over the objects (scope 0) and one collection of rows per object (scope 1)
NET = dict(C=50, NS=2, NP=4, nops=100, nitems=120, nmatch=2, ncols=10, npool=200, ncbytes=40, levels=[0] * 20 + [1] * 30)
AMB = dict(NET, levels=[0] * 20 + [1] * 60)     # the ambiguity netlist: more live columns over the rows
TILES = [512, 256, 128, 64, 32]


def _r16(x):
    return (x + 15) // 16 * 16


def _need(net, cap, tile):
    """(slot words, shared-memory bytes) of one launch, written out independently of the header"""
    cap = [tile] + list(cap[1:])
    sw = sum(((cap[lv] + 31) // 32 + 1 + 3) & ~3 for lv in net["levels"])
    C, NS = net["C"], net["NS"]
    smem = (3 * _r16(4 * C) + 2 * _r16(4 * NS) + _r16(4 * (net["NP"] + 1)) + _r16(4 * sw) + 64 + _r16(8 * C) + _r16(16 * net["nops"])
            + _r16(4 * net["nitems"]) + _r16(64 * net["nmatch"]) + _r16(64 * net["ncols"]) + _r16(16 * NS) + _r16(4 * net["npool"])
            + _r16(net["ncbytes"]))
    return sw, smem


def _page(n, rows):
    """rows of the largest tile per scope, for every tile size, of n objects with `rows` rows each"""
    return {t: [min(t, n), min(t, n) * rows] for t in TILES}


def _search(ask, nets, caps, max_smem):
    req = ["tile", max_smem, 512, len(nets)]
    for net in nets:
        req += [net[k] for k in ("C", "NS", "NP", "nops", "nitems", "nmatch", "ncols", "npool", "ncbytes")]
        req += [len(net["levels"]), *net["levels"]]
    req.append(len(caps))
    for t, cap in caps.items():
        req += [t, len(cap), *cap]
    (got, ) = ask(req)
    assert got[1] == "fits" and got[3] == "tried"
    return int(got[0]), got[2] == "1", [int(x) for x in got[4:]]


def test_tile_that_fits_stays(ask):
    caps = _page(4096, 4)
    assert _search(ask, [NET], caps, _need(NET, caps[512], 512)[1]) == (512, True, [512])


def test_tile_halves_until_it_fits(ask):
    caps = _page(4096, 40)
    lo, hi = _need(NET, caps[128], 128)[1], _need(NET, caps[256], 256)[1]
    assert lo < hi
    assert _search(ask, [NET], caps, (lo + hi) // 2) == (128, True, [512, 256, 128])


def test_tile_that_never_fits_ends_at_32(ask):
    caps = _page(4096, 40)
    assert _search(ask, [NET], caps, _need(NET, caps[32], 32)[1] - 1) == (32, False, TILES)


def test_ambiguity_netlist_shrinks_the_tile(ask):
    caps = _page(4096, 4)
    dec, amb = _need(NET, caps[512], 512)[1], _need(AMB, caps[512], 512)[1]
    max_smem = (dec + amb) // 2
    assert _need(AMB, caps[256], 256)[1] <= max_smem
    assert _search(ask, [NET], caps, max_smem) == (512, True, [512])
    assert _search(ask, [NET, AMB], caps, max_smem) == (256, True, [512, 256])


def test_slot_offsets_past_16_bits_shrink_the_tile(ask):
    caps = _page(4096, 200)
    assert _need(NET, caps[512], 512)[0] > 0xffff >= _need(NET, caps[256], 256)[0]
    assert _search(ask, [NET], caps, 1 << 30) == (256, True, [512, 256])


def test_object_slots_are_sized_by_the_tile(ask):
    # 100 objects: the largest 512-object tile holds 100 of them, but a launch still sizes every object-level slot for 512
    caps = _page(100, 4)
    assert _search(ask, [NET], caps, _need(NET, caps[512], 512)[1]) == (512, True, [512])
    assert _search(ask, [NET], caps, _need(NET, caps[512], 512)[1] - 1) == (256, True, [512, 256])
