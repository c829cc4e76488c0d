"""lzgpu_plan_salvage_slices without a GPU (csrc/host_math.cc, csrc/slices_solve.h).

The plan's four masks (known and determined for a full combined stripe and for the chunk's last, partial one) are checked against the
plain-Python rank model of tests/test_recover_slices_plan.py for every loss pattern of six goal sets, at a block count L divides and at
a ragged one.  The counts of patterns that are not wholly determined, that still determine some block, and that solve some block from
parity blocks are pinned per goal set, with the mean share of blocks salvaged.  The launch geometry is checked against a restatement
of rs_geometry's salvage sizing (every given part verified, the image with a CRC stream per block, nothing wanted), and the argument
refusals are covered."""
import ctypes as C

import numpy as np
import pytest

from lizardfs_b200 import _lib
from lizardfs_b200.engine import Engine, LzGpuError
from tests.test_recover_slices_geometry import ENTRY_CAP, SMEM_CAP, shape, slices
from tests.test_recover_slices_plan import goalset, layout, lcm_of, model

GOAL_SETS = [("xor2", "xor3"), ("std", "xor2", "xor3"), ("ec(3,2)", "ec(2,2)"), ("ec(3,2)", "ec(4,2)"), ("xor3",), ("ec(8,2)",)]


def plan(goals, nb, given):
    return Engine.plan_salvage_slices(goals, nb, given)


def block_counts(L):
    """a block count L divides and a ragged one (nb % L != 0), both within one chunk"""
    full = 1024 - 1024 % L
    ragged = full - 1 if L > 1 else None
    return full, ragged


@pytest.mark.parametrize("names", GOAL_SETS)
def test_every_loss_pattern_against_the_rank_model(names):
    goals = goalset(names)
    _, n = layout(goals)
    L = lcm_of(goals)
    full_nb, ragged_nb = block_counts(L)
    tail = ragged_nb % L
    for bits in range(1 << n):
        given = [(bits >> g) & 1 for g in range(n)]
        known, det = model(goals, given, L)
        p = plan(goals, full_nb, given)
        assert (p["L"], p["tail_blocks"]) == (L, 0)
        assert (p["known"], p["determined"], p["tail_known"], p["tail_determined"]) == (known, det, known, det), (names, given)
        # determined is lzgpu_plan_recover_slices' mask, for both shapes
        r = Engine.plan_recover_slices(goals, ragged_nb, given)
        t_known, t_det = model(goals, given, tail)
        p = plan(goals, ragged_nb, given)
        assert p["tail_blocks"] == tail
        assert (p["known"], p["determined"], p["tail_known"], p["tail_determined"]) == (known, det, t_known, t_det), (names, given)
        assert (r["determined"], r["tail_determined"], r["known"]) == (p["determined"], p["tail_determined"], p["known"])


# goal set: patterns not wholly determined, with some block determined, with some block solved from parity blocks, mean share of
# blocks salvaged, mean share solved (both over those patterns, not weighted by how likely a pattern is)
COUNTS = [
    (("xor2", "xor3"), 36, 33, 8, 0.565, 0.065),
    (("ec(3,2)", "ec(2,2)"), 54, 46, 16, 0.512, 0.086),
    (("ec(3,2)", "ec(4,2)"), 405, 396, 210, 0.641, 0.107),
    (("ec(8,2)",), 968, 964, 0, 0.481, 0.0),
]


@pytest.mark.parametrize("names,partial,some,solved,share,share_solved", COUNTS)
def test_what_there_is_to_salvage(names, partial, some, solved, share, share_solved):
    goals = goalset(names)
    _, n = layout(goals)
    L = lcm_of(goals)
    full = (1 << L) - 1
    counts = [0, 0, 0]
    shares, solved_shares = [], []
    for bits in range(1 << n):
        given = [(bits >> g) & 1 for g in range(n)]
        p = plan(goals, block_counts(L)[0], given)
        if p["determined"] == full:
            continue
        got = p["determined"] & ~p["known"]
        counts[0] += 1
        counts[1] += p["determined"] != 0
        counts[2] += got != 0
        shares.append(bin(p["determined"]).count("1") / L)
        solved_shares.append(bin(got).count("1") / L)
    assert counts == [partial, some, solved]
    assert round(float(np.mean(shares)), 3) == share
    assert round(float(np.mean(solved_shares)), 3) == share_solved


def salvage_geometry(names, nb, given):
    """restatement of rs_geometry(..., salvage = true): reads as for recovery, no wanted part, the image's `valid` writes each with a
    CRC stream, slots for the positions and the chosen equations only.  Returns the plan's fields and the CRC streams."""
    lay, _ = slices(names)
    L = lcm_of(goalset(names))
    tail = nb % L
    used = [(shape(lay, given, v), v) for v in {L if nb >= L else tail, tail if tail else L}]
    slots = max(L + s["E"] for s, _ in used)
    states = max(s["reads"] + v for s, v in used)
    smem = 4096 + 1024 * slots + 128 * states
    fits = all(s["reads"] <= ENTRY_CAP for s, _ in used) and states <= ENTRY_CAP
    return dict(ok=int(fits and smem <= SMEM_CAP), G=1 if L >= 8 else 8 // L, threads=256, stages=1, smem_bytes=smem), states


@pytest.mark.parametrize("names,given,nb,ok,states", [
    (("xor2", "xor3"), [0, 1, 1, 0, 0, 1, 1], 1024, 1, 16),       # 6 + 4 reads + 6 image streams
    (("xor2", "xor3"), [0, 1, 1, 0, 0, 1, 1], 5, 1, 15),          # nb < L, the tail only: the same reads + 5 image streams
    (("ec(3,2)", "ec(4,2)"), [1] * 11, 1023, 1, 50),              # 20 + 18 reads + 12 (the tail of 3: 11 + 3)
    (("ec(8,2)",), [1, 0, 1, 0, 1, 0, 1, 0, 1, 1], 1021, 1, 14),  # 6 reads + 8 (the tail of 5: 6 + 5)
    (("ec(3,3)", "ec(16,16)"), [0] * 6 + [1] * 32, 1024, 1, 144),  # every ec(16,16) part: 96 reads + 48 image streams
    (("ec(3,3)", "ec(16,16)"), [1] * 38, 1024, 0, 240),            # every part: 192 reads + 48 image streams > 192
    (("ec(3,3)", "ec(16,16)"), [1] * 38, 47, 0, 239),
])
def test_plan_geometry_against_a_restatement(names, given, nb, ok, states):
    p = plan(goalset(names), nb, given)
    want, got_states = salvage_geometry(names, nb, given)
    assert {f: p[f] for f in want} == want
    assert (p["ok"], got_states) == (ok, states)


def test_plan_geometry_on_every_pattern():
    for names in GOAL_SETS[:4]:
        _, n = layout(goalset(names))
        L = lcm_of(goalset(names))
        for bits in range(0, 1 << n, 7):
            given = [(bits >> g) & 1 for g in range(n)]
            for nb in (1, L + 1, 1024):
                p = plan(goalset(names), nb, given)
                assert {f: p[f] for f in ("ok", "G", "threads", "stages", "smem_bytes")} == salvage_geometry(names, nb, given)[0]


def test_argument_refusals():
    lib = _lib.load()
    ok = goalset(("xor2", "xor3"))
    for goals, nb in [
        (goalset(("xor2", "xor2")), 1024),                  # a repeated slice type
        (goalset(("ec(32,2)", "ec(31,2)")), 1024),          # L = 992 > 64
        (goalset(("std",)), 1024),                          # no xor/ec slice
        (goalset(("xor2", "xor3", "xor4", "xor5", "ec(2,2)")), 1024),  # five slices
        (ok, 0),
        (ok, 1025),
    ]:
        with pytest.raises(LzGpuError) as e:
            plan(goals, nb, [1] * 64)
        assert e.value.status == _lib.ERR_ARG
    out = _lib.LzSlicesSalvagePlan()
    arr = (_lib.LzGoal * 2)(*[g.c for g in ok])
    g = np.asarray([1] * 7, dtype=np.uint8)
    assert lib.lzgpu_plan_salvage_slices(arr, 2, 1024, None, C.byref(out)) == _lib.ERR_ARG
    assert lib.lzgpu_plan_salvage_slices(arr, 2, 1024, g.ctypes.data_as(C.c_void_p), None) == _lib.ERR_ARG
    assert lib.lzgpu_plan_salvage_slices(arr, 0, 1024, g.ctypes.data_as(C.c_void_p), C.byref(out)) == _lib.ERR_ARG
    # no part given is no plan refusal: nothing is determined (the call refuses it with LZGPU_ERR_TOO_FEW_PARTS)
    p = plan(ok, 1024, [0] * 7)
    assert (p["known"], p["determined"], p["ok"]) == (0, 0, 1)
