"""lzgpu_plan_check_slices and lzgpu_debug_check_slices_rows without a GPU (csrc/slices_check.h).

The checks of a stripe shape are the left null space of the given blocks' functionals over the combined stripe's positions (a given
parity block is its generator row over its slice stripe, a given data block at a position < valid is that position).  So, against
the plain-Python GF(2^8) rank model of tests/test_recover_slices_plan.py:
- n_checks is given blocks - rank, for every given pattern of the goal sets below, at a block count L divides and at a ragged
  one; 17 and 26 for std + xor2 + xor3 and ec(3,2) + ec(4,2) with every part given;
- every debug check has coefficient 1 on its defining block, the checks are ordered by that block, they are independent, and each
  annihilates a randomly encoded combined stripe;
- `checked` and `locatable` (on a seeded sample of patterns per set, every part given among them) follow from the codewords
  supported on a set of blocks B, of dimension rank(A) - rank(A without B);
- more than 64 checks makes the plan say ok = 0 and the debug rows refuse."""
import ctypes as C
import random

import numpy as np
import pytest

from lizardfs_b200 import _lib
from lizardfs_b200.engine import Engine, LzGpuError
from tests.test_recover_slices_plan import EXP, LOG, goalset, layout, lcm_of, rank

GOAL_SETS = [("std", "xor2"), ("std", "xor2", "xor3"), ("xor2", "xor3"), ("ec(3,2)", "ec(2,2)"), ("ec(3,2)", "ec(4,2)"),
             ("ec(5,5)", "xor2")]

MUL = np.zeros((256, 256), dtype=np.uint8)
for _a in range(1, 256):
    for _b in range(1, 256):
        MUL[_a, _b] = EXP[LOG[_a] + LOG[_b]]


def given_blocks(goals, given, valid):
    """the given blocks of a shape in flat order (part, then stripe): (flat part, stripe, functional over the L positions)"""
    lay, _ = layout(goals)
    L = lcm_of(goals)
    out = []
    for k, m, base, gen in lay:
        for p in range(k + m):
            if not given[base + p]:
                continue
            for s in range(L // k):
                if s * k >= valid:
                    continue
                row = [0] * L
                if p < k:
                    if s * k + p >= valid:
                        continue
                    row[s * k + p] = 1
                else:
                    for j in range(k):
                        if s * k + j < valid:
                            row[s * k + j] = gen[p - k][j]
                out.append((base + p, s, row))
    return out


def patterns(goals, limit=None, seed=0):
    _, n = layout(goals)
    all_ = [[(bits >> g) & 1 for g in range(n)] for bits in range(1, 1 << n)]
    if limit is None or len(all_) <= limit:
        return all_
    rng = random.Random(seed)
    return [[1] * n] + rng.sample(all_, limit)


def shapes(goals):
    """(nb, valid of the full shape or None, valid of the tail): a block count L divides and a ragged one"""
    L = lcm_of(goals)
    full = 1024 - 1024 % L
    return [(full, L, L), (full - 1, L, (full - 1) % L)] if L > 1 else [(full, L, L)]


def masks_model(goals, given, valid, rank=rank):
    """(checked, locatable) from the codewords supported on sets of blocks (rank: the GF(2^8) rank used, the plain one by default)"""
    blocks = given_blocks(goals, given, valid)
    L = lcm_of(goals)
    A = [r for _, _, r in blocks]
    rA = rank(A, L)

    def r_cols(idx):   # rank of the check-matrix columns of the blocks idx: |B| - (rank(A) - rank(A without B))
        rest = [A[b] for b in range(len(A)) if b not in idx]
        return len(idx) - (rA - rank(rest, L))

    parts = sorted({g for g, _, _ in blocks})
    of = {g: {b for b, (h, _, _) in enumerate(blocks) if h == g} for g in parts}
    checked = locatable = 0
    for g in parts:
        if all(r_cols({b}) == 1 for b in of[g]):
            checked |= 1 << g
        rg = r_cols(of[g])
        if rg == len(of[g]) and all(r_cols(of[g] | of[h]) == rg + r_cols(of[h]) for h in parts if h != g):
            locatable |= 1 << g
    return checked, locatable


@pytest.mark.parametrize("names", GOAL_SETS, ids="+".join)
def test_check_count_is_given_blocks_minus_rank(names):
    goals = goalset(names)
    L = lcm_of(goals)
    for given in patterns(goals):
        for nb, vf, vt in shapes(goals):
            p = Engine.plan_check_slices(goals, nb, given)
            assert (p["L"], p["tail_blocks"]) == (L, nb % L)
            for v, key in ((vf, "n_checks"), (vt, "tail_n_checks")):
                blocks = given_blocks(goals, given, v)
                assert p[key] == len(blocks) - rank([r for _, _, r in blocks], L), (names, given, v)
            assert p["ok"] == 1


def test_pinned_counts_with_every_part_given():
    assert Engine.plan_check_slices(goalset(("std", "xor2", "xor3")), 1020, [1] * 8)["n_checks"] == 17
    assert Engine.plan_check_slices(goalset(("ec(3,2)", "ec(4,2)")), 1020, [1] * 11)["n_checks"] == 26


@pytest.mark.parametrize("names", GOAL_SETS, ids="+".join)
def test_debug_rows_annihilate_a_random_stripe(names):
    goals = goalset(names)
    L = lcm_of(goals)
    rng = np.random.default_rng(7)
    for given in patterns(goals, limit=12, seed=1):
        for valid in sorted({L, max(1, L - 1), (L + 1) // 2}):
            blocks = given_blocks(goals, given, valid)
            n_checks = len(blocks) - rank([r for _, _, r in blocks], L)
            part, stripe, coef = Engine.debug_check_slices_rows(goals, given, valid)
            assert len(part) == n_checks
            where = [(g, s) for g, s, _ in blocks]
            # ordered by the defining block, coefficient 1 there, nothing outside the given blocks
            defs = [where.index((int(g), int(s))) for g, s in zip(part, stripe)]
            assert defs == sorted(set(defs))
            mask = np.zeros((64, 64), dtype=bool)
            for g, s in where:
                mask[g, s] = True
            for h in range(n_checks):
                assert coef[h, part[h], stripe[h]] == 1
                assert not coef[h][~mask].any()
            rows = [[int(coef[h, g, s]) for g, s in where] for h in range(n_checks)]
            assert rank(rows, len(where)) == n_checks
            # a random combined stripe: every check's syndrome is zero
            x = rng.integers(0, 256, size=(L, 16), dtype=np.uint8)
            x[valid:] = 0
            val = {}
            for g, s, r in blocks:
                v = np.zeros(16, dtype=np.uint8)
                for q in range(L):
                    v ^= MUL[r[q], x[q]]
                val[(g, s)] = v
            for h in range(n_checks):
                syn = np.zeros(16, dtype=np.uint8)
                for g, s in where:
                    syn ^= MUL[coef[h, g, s], val[(g, s)]]
                assert not syn.any(), (names, given, valid, h)


@pytest.mark.parametrize("names", GOAL_SETS, ids="+".join)
def test_checked_and_locatable_against_the_rank_model(names):
    goals = goalset(names)
    for given in patterns(goals, limit=25, seed=2):
        for nb, vf, vt in shapes(goals):
            p = Engine.plan_check_slices(goals, nb, given)
            assert (p["checked"], p["locatable"]) == masks_model(goals, given, vf), (names, given)
            assert (p["tail_checked"], p["tail_locatable"]) == masks_model(goals, given, vt), (names, given, nb)


def test_every_part_locatable_when_all_are_given():
    for names, n in ((("std", "xor2", "xor3"), 8), (("ec(3,2)", "ec(4,2)"), 11)):
        p = Engine.plan_check_slices(goalset(names), 1024 - 1024 % lcm_of(goalset(names)), [1] * n)
        assert p["checked"] == p["locatable"] == (1 << n) - 1


def test_more_than_64_checks():
    goals = goalset(("std", "ec(8,4)", "ec(3,4)"))   # L = 24: 24 + 36 + 56 given blocks over 24 positions
    n = 1 + 12 + 7
    p = Engine.plan_check_slices(goals, 1008, [1] * n)
    assert (p["n_checks"], p["ok"]) == (92, 0)
    with pytest.raises(LzGpuError) as ex:
        Engine.debug_check_slices_rows(goals, [1] * n, 24)
    assert ex.value.status == _lib.ERR_ARG
    # without the ec(3,4) parity parts: 24 + 36 + 24 - 24 = 60 checks fit
    p = Engine.plan_check_slices(goals, 1008, [1] * 16 + [0] * 4)
    assert (p["n_checks"], p["ok"]) == (60, 1)


def test_refusals():
    lib = _lib.load()
    goals = goalset(("xor2", "xor3"))
    arr = (_lib.LzGoal * 2)(*[g.c for g in goals])
    g = np.ones(7, dtype=np.uint8)
    gp = g.ctypes.data_as(C.c_void_p)
    out = _lib.LzSlicesCheckPlan()
    assert lib.lzgpu_plan_check_slices(arr, 2, 1024, None, C.byref(out)) == _lib.ERR_ARG
    assert lib.lzgpu_plan_check_slices(arr, 2, 1024, gp, None) == _lib.ERR_ARG
    assert lib.lzgpu_plan_check_slices(arr, 0, 1024, gp, C.byref(out)) == _lib.ERR_ARG
    assert lib.lzgpu_plan_check_slices(arr, 2, 0, gp, C.byref(out)) == _lib.ERR_ARG
    assert lib.lzgpu_plan_check_slices(arr, 2, 1025, gp, C.byref(out)) == _lib.ERR_ARG
    with pytest.raises(LzGpuError):
        Engine.debug_check_slices_rows(goals, [1] * 7, 7)   # valid > L
    with pytest.raises(LzGpuError):
        Engine.debug_check_slices_rows(goals, [1] * 7, 0)
