"""lzgpu_plan_recover_slices and the host solve of lzgpu_recover_slices without a GPU (csrc/slices_solve.h).

The plan's masks are checked against a plain-Python GF(2^8) rank computation written here: a position is determined when it is held
by a given data part of some slice, or when its unit vector lies in the row space of the given parity equations restricted to the
unknown positions (rank([A; e_x]) == rank(A)).  Every loss pattern of xor2+xor3, std+xor2+xor3, ec(3,2)+ec(2,2) and ec(3,2)+ec(4,2)
is covered, with the counts of chunks the per-slice rule loses and this call rescues; a sample of ec(3,2)+ec(8,2) (L = 24) and of a
set with a Cauchy slice; and the tail stripe at nb < L, nb % L != 0 and nb = 1024.  The debug rows, applied to random blocks with
Python arithmetic, reproduce the unknowns."""
import ctypes as C
import itertools
import random

import numpy as np
import pytest

from lizardfs_b200 import _lib
from lizardfs_b200.engine import Engine, LzGpuError, SliceType

# GF(2^8) with x^8 + x^4 + x^3 + x^2 + 1
EXP = [0] * 512
LOG = [0] * 256
_x = 1
for _i in range(255):
    EXP[_i] = EXP[_i + 255] = _x
    LOG[_x] = _i
    _x = (_x << 1) ^ (0x11D if _x & 0x80 else 0)


def gmul(a, b):
    return EXP[LOG[a] + LOG[b]] if a and b else 0


def ginv(a):
    return EXP[255 - LOG[a]]


def rank(rows, n):
    m = [list(r) for r in rows]
    r = 0
    for c in range(n):
        p = next((i for i in range(r, len(m)) if m[i][c]), None)
        if p is None:
            continue
        m[r], m[p] = m[p], m[r]
        inv = ginv(m[r][c])
        m[r] = [gmul(v, inv) for v in m[r]]
        for i in range(len(m)):
            if i != r and m[i][c]:
                f = m[i][c]
                m[i] = [v ^ gmul(f, w) for v, w in zip(m[i], m[r])]
        r += 1
    return r


def generator(goal):
    """parity rows [m][k] of an xor/ec slice, from lzgpu_rs_generator (Vandermonde (2^r)^j or Cauchy)"""
    k, m = goal.k, goal.m
    full = (C.c_uint8 * ((k + m) * k))()
    assert _lib.load().lzgpu_rs_generator(k, m, full) >= 0
    return [[full[(k + r) * k + j] for j in range(k)] for r in range(m)]


def layout(goals):
    """per slice (k, m, base, parity rows); the standard slice is k = 1, m = 0"""
    out, base = [], 0
    for g in goals:
        k, m = (1, 0) if g.is_std else (g.k, g.m)
        out.append((k, m, base, [] if g.is_std else generator(g)))
        base += k + m
    return out, base


def lcm_of(goals):
    L = 1
    for g in goals:
        if not g.is_std:
            a, b = L, g.k
            while b:
                a, b = b, a % b
            L = L // a * g.k
    return L


def model(goals, given, valid):
    """(known, determined) masks of one stripe shape by rank computations"""
    lay, _ = layout(goals)
    L = lcm_of(goals)
    known = 0
    for k, m, base, _ in lay:
        for j in range(k):
            if given[base + j]:
                for q in range(j, valid, k):
                    known |= 1 << q
    unk = [q for q in range(valid) if not (known >> q) & 1]
    col = {q: i for i, q in enumerate(unk)}
    eqs = []
    for k, m, base, gen in lay:
        for r in range(m):
            if not given[base + k + r]:
                continue
            for s in range(L // k):
                if s * k >= valid:
                    continue
                row = [0] * len(unk)
                for j in range(k):
                    q = s * k + j
                    if q in col:
                        row[col[q]] = gen[r][j]
                if any(row):
                    eqs.append(row)
    det = known | sum(1 << q for q in range(valid, L))
    r0 = rank(eqs, len(unk))
    for i, q in enumerate(unk):
        e = [0] * len(unk)
        e[i] = 1
        if rank(eqs + [e], len(unk)) == r0:
            det |= 1 << q
    return known, det


def plan(goals, nb, given):
    return Engine.plan_recover_slices(goals, nb, given)


def goalset(names):
    return [SliceType(2, 1, 0) if n == "std" else SliceType(n) for n in names]


def ref_lost(goals, given):
    """the per-slice rule (ChunkCopiesCalculator::evalRedundancyLevel): lost when every slice has fewer than k parts"""
    lay, _ = layout(goals)
    return all(sum(given[base:base + k + m]) < k for k, m, base, _ in lay)


@pytest.mark.parametrize("names,lost,rescued", [
    (("xor2", "xor3"), 44, 8),
    (("ec(3,2)", "ec(2,2)"), 80, 26),
    (("ec(3,2)", "ec(4,2)"), 672, 267),
    (("std", "xor2", "xor3"), None, None),
])
def test_every_loss_pattern_against_the_rank_model(names, lost, rescued):
    goals = goalset(names)
    _, n = layout(goals)
    L = lcm_of(goals)
    full = (1 << L) - 1
    n_lost = n_rescued = 0
    for bits in range(1 << n):
        given = [(bits >> g) & 1 for g in range(n)]
        p = plan(goals, 1024 if 1024 % L == 0 else 1023, given)
        known, det = model(goals, given, L)
        assert (p["L"], p["known"], p["determined"]) == (L, known, det), (names, given)
        if ref_lost(goals, given):
            n_lost += 1
            n_rescued += det == full
    if lost is not None:
        assert (n_lost, n_rescued) == (lost, rescued)


@pytest.mark.parametrize("names,nbs", [
    (("xor2", "xor3"), (1, 5, 7, 1000, 1024)),
    (("ec(3,2)", "ec(4,2)"), (3, 11, 13, 1024)),
    (("std", "xor2", "xor3"), (2, 1022, 1024)),
    (("ec(3,2)", "ec(2,2)"), (1, 4, 1024)),
])
def test_tail_masks(names, nbs):
    goals = goalset(names)
    _, n = layout(goals)
    L = lcm_of(goals)
    rng = random.Random(7)
    patterns = [[rng.randrange(2) for _ in range(n)] for _ in range(120)]
    for nb in nbs:
        for given in patterns:
            p = plan(goals, nb, given)
            tail = nb % L
            assert p["tail_blocks"] == tail
            want = model(goals, given, tail)[1] if tail else model(goals, given, L)[1]
            assert p["tail_determined"] == want, (names, nb, given)


@pytest.mark.parametrize("names,samples", [
    (("ec(3,2)", "ec(8,2)"), 250),       # L = 24
    (("ec(5,5)", "xor2"), 150),          # a Cauchy slice (m >= 5)
    (("std", "ec(3,2)", "ec(8,2)"), 100),
])
def test_sampled_patterns(names, samples):
    goals = goalset(names)
    _, n = layout(goals)
    L = lcm_of(goals)
    rng = random.Random(11)
    for _ in range(samples):
        # bias towards heavy loss, where the joint solve matters
        keep = rng.uniform(0.3, 0.8)
        given = [1 if rng.random() < keep else 0 for _ in range(n)]
        for nb in (1024, L - 1, 2 * L + 5):
            p = plan(goals, nb, given)
            known, det = model(goals, given, L)
            assert (p["known"], p["determined"]) == (known, det), (names, given)
            tail = nb % L
            if tail:
                assert p["tail_determined"] == model(goals, given, tail)[1]


def _debug_rows(goals, given, valid):
    lib = _lib.load()
    arr = (_lib.LzGoal * len(goals))(*[g.c for g in goals])
    g = np.asarray(given, dtype=np.uint8)
    nu, ne = C.c_uint32(), C.c_uint32()
    unk, es, er, est = (np.zeros(64, np.uint8) for _ in range(4))
    rows = np.zeros((64, 64), np.uint8)
    det = C.c_uint64()
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    rc = lib.lzgpu_debug_recover_slices_rows(arr, len(goals), ptr(g), valid, C.byref(nu), C.byref(ne), ptr(unk), ptr(es), ptr(er), ptr(est),
                                             ptr(rows), C.byref(det))
    assert rc == _lib.OK
    return nu.value, ne.value, unk, es, er, est, rows, det.value


@pytest.mark.parametrize("names", [("xor2", "xor3"), ("ec(3,2)", "ec(4,2)"), ("ec(3,2)", "ec(8,2)"), ("ec(5,5)", "xor2"),
                                   ("std", "xor2", "xor3")])
def test_debug_rows_reproduce_the_unknowns(names):
    goals = goalset(names)
    lay, n = layout(goals)
    L = lcm_of(goals)
    rng = random.Random(3)
    checked = 0
    for _ in range(60):
        given = [rng.randrange(2) for _ in range(n)]
        for valid in (L, max(1, L - 3)):
            nu, ne, unk, es, er, est, rows, det = _debug_rows(goals, given, valid)
            assert ne <= nu <= 64
            assert det == model(goals, given, valid)[1]
            d = [[rng.randrange(256) for _ in range(8)] if q < valid else [0] * 8 for q in range(L)]
            known = [q for q in range(L) if q >= valid or q not in set(unk[:nu].tolist())]
            syn = []
            for e in range(ne):
                k, m, base, gen = lay[es[e]]
                s = est[e]
                par = [0] * 8
                share = [0] * 8
                for j in range(k):
                    q = s * k + j
                    for b in range(8):
                        par[b] ^= gmul(gen[er[e]][j], d[q][b])
                        if q in known:
                            share[b] ^= gmul(gen[er[e]][j], d[q][b])
                syn.append([a ^ b for a, b in zip(par, share)])
            for x in range(nu):
                q = int(unk[x])
                if not (det >> q) & 1:
                    assert not rows[x].any()
                    continue
                got = [0] * 8
                for e in range(ne):
                    for b in range(8):
                        got[b] ^= gmul(int(rows[x][e]), syn[e][b])
                assert got == d[q], (names, given, valid, q)
                checked += 1
    assert checked > 0


def test_argument_refusals():
    lib = _lib.load()
    ok = goalset(("xor2", "xor3"))
    given = [1] * 7
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
    out = _lib.LzSlicesRecoverPlan()
    arr = (_lib.LzGoal * 2)(*[g.c for g in ok])
    g = np.asarray(given, dtype=np.uint8)
    assert lib.lzgpu_plan_recover_slices(arr, 2, 1024, None, C.byref(out)) == _lib.ERR_ARG
    assert lib.lzgpu_plan_recover_slices(arr, 2, 1024, g.ctypes.data_as(C.c_void_p), None) == _lib.ERR_ARG
    assert lib.lzgpu_plan_recover_slices(arr, 0, 1024, g.ctypes.data_as(C.c_void_p), C.byref(out)) == _lib.ERR_ARG


def test_plan_geometry():
    goals = goalset(("ec(3,2)", "ec(4,2)"))
    p = plan(goals, 1024, [1] * 11)
    assert p["ok"] == 1 and p["threads"] == 256 and p["stages"] == 1 and p["G"] == 1
    assert p["unknowns"] == 0 and p["equations"] == 0
    # every part lost: nothing determined, geometry still reported
    p = plan(goals, 1024, [0] * 11)
    assert p["known"] == 0 and p["determined"] == 0 and p["unknowns"] == 12
    p = plan(goalset(("xor2",)), 1024, [1, 0, 1])
    assert p["G"] == 4 and p["L"] == 2
