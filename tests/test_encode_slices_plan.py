"""lzgpu_plan_encode_slices without a GPU: the planner of the one-pass multi-slice encode (slices_plan, csrc/fused_plan.h) against a
table of literal plans that covers its space, its argument refusals, and the layout of lzgpu_slices_plan against the header.

PLAN_TABLE holds one goal set per feature value the planner can produce: every largest-m instantiation (1..4), G = 1 and the largest G
(32, at L = 2), L from 2 to 63, a G capped by ceil(nb / L), a batch of one-combined-stripe chunks, every stage count, and every
refusal reason.  test_plan_table_covers_the_planner_space enumerates every pair of xor/ec goals on the CPU and fails when a feature
value it sees is missing from the table.  tests/test_gpu_encode_slices.py runs every fused entry of the table on the GPU."""
import ctypes as C
import itertools
import os
import subprocess

import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200.engine import Engine, LzGpuError

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("fused", "refusal", "L", "G", "threads", "stages", "crc_rows", "smem_bytes", "units")
SINGLE, CAUCHY, WIDE, NO_GEOMETRY = (_lib.SLICES_REFUSED_SINGLE, _lib.SLICES_REFUSED_CAUCHY, _lib.SLICES_REFUSED_WIDE,
                                     _lib.SLICES_REFUSED_NO_GEOMETRY)

PLAN_TABLE = [
    # goal set, chunks, blocks per chunk, plan: fused, refusal, L, G, threads, stages, CRC rows, shared memory, units
    (("xor2", "xor3"), 4, 1024, (1, 0, 6, 10, 512, 4, 240, 123528, 72)),             # m = 1: no parity streams at all
    (("xor2", "xor3"), 4, 1, (1, 0, 6, 1, 512, 4, 24, 12936, 4)),                    # one block: G capped to 1
    (("std", "xor2", "xor3"), 4, 1024, (1, 0, 6, 10, 512, 4, 240, 123528, 72)),      # goal.h's example
    (("ec(3,2)", "ec(8,2)"), 4, 1024, (1, 0, 24, 2, 512, 4, 280, 144008, 88)),       # m = 2
    (("ec(3,2)", "ec(8,2)"), 8, 24, (1, 0, 24, 1, 512, 4, 140, 74376, 8)),           # one combined stripe per chunk
    (("std", "ec(3,2)", "ec(8,2)"), 3, 12, (1, 0, 24, 1, 512, 4, 140, 74376, 3)),    # nb < L
    (("ec(8,2)", "ec(8,4)"), 4, 1024, (1, 0, 8, 8, 512, 4, 384, 197256, 64)),        # m = 4
    (("ec(5,3)", "ec(4,2)"), 4, 1024, (1, 0, 20, 3, 512, 3, 396, 174712, 72)),       # m = 3, three stages
    (("ec(8,3)", "ec(6,4)"), 4, 1024, (1, 0, 24, 2, 512, 4, 336, 172680, 88)),
    (("ec(7,2)", "ec(9,2)"), 4, 1024, (1, 0, 63, 1, 512, 4, 316, 164488, 68)),       # L = 63, the widest fused set
    (("xor2", "ec(2,2)"), 4, 1024, (1, 0, 2, 32, 512, 4, 384, 197256, 64)),          # L = 2, the largest G
    (("ec(2,1)", "ec(3,4)"), 1, 1024, (1, 0, 6, 10, 512, 2, 480, 184936, 18)),       # two stages
    (("ec(2,1)", "ec(3,4)"), 3, 12, (1, 0, 6, 2, 512, 4, 96, 49800, 3)),             # G capped by ceil(nb / L) = 2
    (("xor2", "xor3", "xor4", "xor5"), 2, 60, (1, 0, 60, 1, 512, 4, 240, 123528, 2)),  # four slices
    (("ec(8,2)",), 2, 1024, (0, SINGLE, 8, 0, 0, 0, 0, 0, 0)),
    (("std", "ec(8,2)"), 2, 1024, (0, SINGLE, 8, 0, 0, 0, 0, 0, 0)),
    (("ec(8,2)", "ec(10,5)"), 2, 1024, (0, CAUCHY, 40, 0, 0, 0, 0, 0, 0)),
    (("ec(8,2)", "ec(9,2)"), 2, 1024, (0, WIDE, 72, 0, 0, 0, 0, 0, 0)),
    (("ec(2,4)", "ec(25,1)"), 2, 1024, (0, NO_GEOMETRY, 50, 0, 0, 0, 0, 0, 0)),      # 200 data rows + 100 x 3 parity rows
]


def goals_of(names):
    return [L.SliceType(n) for n in names]


def plan_tuple(names, n_chunks, nb):
    p = Engine.plan_encode_slices(goals_of(names), n_chunks, nb)
    return tuple(p[f] for f in FIELDS)


def features(names, n_chunks, nb, plan):
    """the values of the plan the kernel and its launch depend on"""
    gs = goals_of(names)
    fused, refusal, Lc, G = plan[:4]
    f = {("refusal", refusal)}
    if fused:
        f |= {("m", max(g.m for g in gs)), ("stages", plan[5]),
              ("G", "1" if G == 1 else ("32" if G == 32 else "2-31")), ("G capped", G * Lc > nb),
              ("L", "2" if Lc == 2 else ("> 48" if Lc > 48 else "3-48"))}
    return f


@pytest.mark.parametrize("entry", PLAN_TABLE, ids=lambda e: "+".join(e[0]) + f"-n{e[1]}-nb{e[2]}")
def test_plan_table(entry):
    names, n_chunks, nb, want = entry
    assert plan_tuple(names, n_chunks, nb) == want


def test_plan_table_covers_the_planner_space():
    goals = [f"xor{k}" for k in range(2, 10)] + [f"ec({k},{m})" for k in range(2, 33) for m in range(1, 5)]
    seen = set()
    for a, b in itertools.combinations_with_replacement(goals, 2):
        for n_chunks, nb in ((4, 1024), (3, 12)):
            seen |= features((a, b), n_chunks, nb, plan_tuple((a, b), n_chunks, nb))
    table = set()
    for names, n_chunks, nb, plan in PLAN_TABLE:
        table |= features(names, n_chunks, nb, plan)
    assert seen - table == set()


def test_plan_geometry_rules():
    """the rules the table's literals come from, over every fused pair: R = G L blocks in one TMA box, the CRC rows fit the CTA,
    the stages fit the shared memory, the units tile the batch"""
    goals = [f"xor{k}" for k in range(2, 10)] + [f"ec({k},{m})" for k in range(2, 21) for m in range(1, 5)]
    for a, b in itertools.combinations(goals, 2):
        for n_chunks, nb in ((2, 1024), (3, 37)):
            fused, refusal, Lc, G, threads, stages, rows, smem, units = plan_tuple((a, b), n_chunks, nb)
            if not fused:
                continue
            R = G * Lc
            assert R <= 64 and 4 * R <= rows <= threads == 512 and 2 <= stages <= 4 and smem <= 200 * 1024
            assert G <= -(-nb // Lc) and units == n_chunks * -(-nb // R)


def test_plan_refuses_bad_arguments():
    lib = _lib.load()
    out = _lib.LzSlicesPlan()
    std = L.SliceType("std")
    ok = Engine.plan_encode_slices([std, L.SliceType("xor2"), L.SliceType("xor3")], 1, 16)
    assert ok["fused"] == 1
    five = goals_of(("xor2", "xor3", "xor4", "xor5", "xor6"))
    with pytest.raises(LzGpuError):
        Engine.plan_encode_slices(five, 1, 16)                      # more than four slices
    with pytest.raises(LzGpuError):
        Engine.plan_encode_slices([std, std], 1, 16)                # no xor/ec slice
    with pytest.raises(LzGpuError):
        Engine.plan_encode_slices(goals_of(("xor2", "xor3")), 1, 0)     # nb = 0
    with pytest.raises(LzGpuError):
        Engine.plan_encode_slices(goals_of(("xor2", "xor3")), 1, 1025)  # nb > 1024
    bad = (_lib.LzGoal * 2)()
    bad[0].kind, bad[0].k, bad[0].m = 1, 33, 2                      # not a goal
    bad[1].kind, bad[1].k, bad[1].m = 0, 3, 1
    assert lib.lzgpu_plan_encode_slices(bad, 2, 1, 16, C.byref(out)) == _lib.ERR_ARG
    assert lib.lzgpu_plan_encode_slices(bad, 0, 1, 16, C.byref(out)) == _lib.ERR_ARG


def test_slices_plan_layout_matches_the_header(tmp_path):
    fields = [f for f, _ in _lib.LzSlicesPlan._fields_]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(['#include <stdio.h>', '#include <stddef.h>', '#include "lzgpu.h"', 'int main(void) {',
                              'printf("%zu %zu", sizeof(lzgpu_slices_plan), _Alignof(lzgpu_slices_plan));'] +
                             [f'printf(" %zu", offsetof(lzgpu_slices_plan, {f}));' for f in fields] +
                             ['printf(" %d %d %d %d %d %d\\n", LZGPU_SLICES_FUSED, LZGPU_SLICES_REFUSED_SINGLE, LZGPU_SLICES_REFUSED_CAUCHY,',
                              '       LZGPU_SLICES_REFUSED_WIDE, LZGPU_SLICES_REFUSED_NO_GEOMETRY, LZGPU_KERNEL_ENCODE_SLICES);', 'return 0; }']))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    size, align, *rest = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    offsets, consts = rest[:len(fields)], rest[len(fields):]
    assert size == C.sizeof(_lib.LzSlicesPlan) == 36 and align == C.alignment(_lib.LzSlicesPlan) == 4
    assert offsets == [getattr(_lib.LzSlicesPlan, f).offset for f in fields]
    assert consts == [_lib.SLICES_FUSED, SINGLE, CAUCHY, WIDE, NO_GEOMETRY, _lib.KERNEL_ENCODE_SLICES] == [0, 1, 2, 3, 4, 11]
