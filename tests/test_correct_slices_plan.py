"""lzgpu_plan_correct_slices and lzgpu_debug_correct_slices_rows without a GPU (csrc/slices_check.h).

A named part g is corrected when its columns H_g of the check matrix have full rank: then H_g e = S has one solution, e = P_g S.  Over
every given pattern of the six goal sets of tests/test_check_slices_plan.py, at a block count L divides and at a ragged one:
- `check` equals lzgpu_plan_check_slices;
- `correctable` equals a rank model over the debug check rows (g's columns have full rank), and contains `locatable`;
- on a seeded sample of patterns, every correctable part's debug rows satisfy P_g H_g = I.
Pinned: std + xor2 + xor3 with only the std part and both parities given (flat parts 0, 3, 7): a stale std block 0 is named std, the
only part whose columns span it, yet std is not correctable (its blocks 0 and 1 have equal columns); std + xor2 with every part given
corrects a divergent standard copy.  lzgpu_slices_fix is 32 bytes."""
import ctypes as C

import numpy as np
import pytest

from lizardfs_b200 import _lib
from lizardfs_b200.engine import SLICES_FIX_DTYPE, Engine, LzGpuError
from tests.test_check_slices_plan import GOAL_SETS, MUL, given_blocks, patterns, shapes
from tests.test_recover_slices_plan import goalset, lcm_of, rank


def columns(goals, given, valid):
    """{part: [column of each of its given blocks over the checks]} and the number of checks, from the debug check rows"""
    part, _, coef = Engine.debug_check_slices_rows(goals, given, valid)
    nc = len(part)
    cols = {}
    for g, s, _ in given_blocks(goals, given, valid):
        cols.setdefault(g, []).append([int(coef[h, g, s]) for h in range(nc)])
    return cols, nc


def correctable_model(goals, given, valid):
    cols, nc = columns(goals, given, valid)
    return sum(1 << g for g, c in cols.items() if rank(c, nc) == len(c))


@pytest.mark.parametrize("names", GOAL_SETS, ids="+".join)
def test_plan_against_the_rank_model(names):
    goals = goalset(names)
    for given in patterns(goals):
        for nb, vf, vt in shapes(goals):
            p = Engine.plan_correct_slices(goals, nb, given)
            c = Engine.plan_check_slices(goals, nb, given)
            assert {k: p[k] for k in c} == c
            assert p["correctable"] == correctable_model(goals, given, vf), (names, given)
            assert p["tail_correctable"] == correctable_model(goals, given, vt), (names, given)
            assert p["locatable"] & ~p["correctable"] == 0 and p["tail_locatable"] & ~p["tail_correctable"] == 0


@pytest.mark.parametrize("names", GOAL_SETS, ids="+".join)
def test_debug_rows_are_left_inverses(names):
    goals = goalset(names)
    for given in patterns(goals, limit=24, seed=3):
        for nb, vf, vt in shapes(goals):
            for valid in {vf, vt}:
                cols, nc = columns(goals, given, valid)
                mask = correctable_model(goals, given, valid)
                blocks = [(g, s) for g, s, _ in given_blocks(goals, given, valid)]
                for g in cols:
                    if not (mask >> g) & 1:
                        with pytest.raises(LzGpuError) as ex:
                            Engine.debug_correct_slices_rows(goals, given, valid, g)
                        assert ex.value.status == _lib.ERR_ARG
                        continue
                    blk_s, rows = Engine.debug_correct_slices_rows(goals, given, valid, g)
                    assert list(blk_s) == [s for h, s in blocks if h == g]
                    assert not rows[:, nc:].any()
                    Hg = np.array(cols[g], dtype=np.uint8)   # [block][check]
                    prod = np.zeros((len(blk_s), len(blk_s)), dtype=np.uint8)
                    for h in range(nc):
                        prod ^= MUL[rows[:, h][:, None], Hg[:, h][None, :]]
                    assert np.array_equal(prod, np.eye(len(blk_s), dtype=np.uint8)), (names, given, valid, g)


def test_undetermined_standard_part():
    goals = goalset(("std", "xor2", "xor3"))
    given = [1, 0, 0, 1, 0, 0, 0, 1]
    cols, nc = columns(goals, given, 6)
    p = Engine.plan_correct_slices(goals, 6, given)
    assert not (p["correctable"] >> 0) & 1
    assert cols[0][0] == cols[0][1] and any(cols[0][0])
    # the column of std block 0 lies in std's span and in no other given part's
    for g in (3, 7):
        assert rank(cols[g] + [cols[0][0]], nc) > rank(cols[g], nc)


def test_divergent_standard_copy_is_correctable():
    goals = goalset(("std", "xor2"))
    p = Engine.plan_correct_slices(goals, 8, [1] * 4)
    assert (p["correctable"] & 1) and (p["locatable"] & 1)
    blk_s, rows = Engine.debug_correct_slices_rows(goals, [1] * 4, 2, 0)
    assert list(blk_s) == [0, 1]


def test_fix_entry_layout():
    assert SLICES_FIX_DTYPE.itemsize == 32 and Engine.SLICES_FIX_DTYPE is SLICES_FIX_DTYPE
    assert C.sizeof(_lib.LzSlicesCorrectPlan) == C.sizeof(_lib.LzSlicesCheckPlan) + 16
    assert _lib.KERNEL_CORRECT_SLICES == 15 and _lib.FIX_UNDETERMINED == 7
