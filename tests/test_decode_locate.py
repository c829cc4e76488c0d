"""lzgpu_decode_stripes without a GPU: the code is MDS for every goal the engine accepts (which makes the located set unique within
the radius), the host build of the error locator the decode kernel runs (csrc/decode_locate.h) against a brute force over every set
of at most two given parts outside F, and the layout of lzgpu_stripe_decode against the header."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

from lizardfs_b200 import _lib
from lizardfs_b200.engine import Engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

EXP = np.zeros(512, dtype=np.int64)
LOG = np.zeros(256, dtype=np.int64)
_x = 1
for _i in range(255):
    EXP[_i] = EXP[_i + 255] = _x
    LOG[_x] = _i
    _x = (_x << 1) ^ (0x11D if _x & 0x80 else 0)
MUL = np.where((np.arange(256)[:, None] > 0) & (np.arange(256)[None, :] > 0), EXP[LOG[:, None] + LOG[None, :]], 0).astype(np.uint8)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def generator(lib, k, m):
    g = np.zeros((k + m, k), dtype=np.uint8)
    assert lib.lzgpu_rs_generator(k, m, _p(g)) == 0
    return g


def permanents(a):
    """the determinants of a batch of r x r matrices over GF(2^8) (characteristic 2: the determinant is the permanent)"""
    n, r, _ = a.shape
    out = np.zeros(n, dtype=np.uint8)
    for perm in itertools.permutations(range(r)):
        term = a[:, 0, perm[0]]
        for i in range(1, r):
            term = MUL[term, a[:, i, perm[i]]]
        out ^= term
    return out


def singular_submatrices(parity, size, rng=None, samples=None):
    m, k = parity.shape
    row_sets = list(itertools.combinations(range(m), size))
    col_sets = list(itertools.combinations(range(k), size))
    pairs = [(r, c) for r in row_sets for c in col_sets]
    if samples is not None and len(pairs) > samples:
        pairs = [pairs[i] for i in rng.choice(len(pairs), samples, replace=False)]
    rows = np.array([r for r, _ in pairs])
    cols = np.array([c for _, c in pairs])
    sub = parity[rows[:, :, None], cols[:, None, :]]
    return int((permanents(sub) == 0).sum())


def test_every_vandermonde_goal_is_mds():
    """every square submatrix of the parity rows of m <= 3 with k <= 32 and m = 4 with k <= 20 is non-singular"""
    lib = _lib.load()
    goals = [(k, m) for m in (1, 2, 3) for k in range(1, 33)] + [(k, 4) for k in range(1, 21)]
    for k, m in goals:
        parity = generator(lib, k, m)[k:]
        for size in range(1, min(k, m) + 1):
            assert singular_submatrices(parity, size) == 0, (k, m, size)


@pytest.mark.parametrize("k,m", [(4, 5), (10, 5), (10, 6), (21, 4), (32, 4), (8, 8)])
def test_cauchy_goals_are_mds_spot_check(k, m):
    lib = _lib.load()
    rng = np.random.default_rng(k * 64 + m)
    parity = generator(lib, k, m)[k:]
    for size in range(1, min(k, m, 6) + 1):
        assert singular_submatrices(parity, size, rng, samples=400) == 0, (k, m, size)


# ---- the locator against a brute force ------------------------------------------------------------------------------------------

LEN = 300


def encode(gen, data):
    """[k+m, LEN] parts of the codeword with these data parts"""
    out = np.zeros((gen.shape[0], data.shape[1]), dtype=np.uint8)
    for r in range(gen.shape[0]):
        for j in range(gen.shape[1]):
            out[r] ^= MUL[gen[r, j], data[j]]
    return out


def consistent(lib, k, m, parts, avail):
    """the parts in avail (ascending, >= k) agree with one codeword: the others re-encoded from the first k of them"""
    inputs, rest = avail[:k], avail[k:]
    if not rest:
        return True
    erased = np.ones(k + m, dtype=np.uint8)
    erased[list(inputs)] = 0
    want = np.zeros(k + m, dtype=np.uint8)
    want[list(rest)] = 1
    rows = np.zeros((m, k), dtype=np.uint8)
    assert lib.lzgpu_rs_recovery_matrix(k, m, _p(erased), _p(want), _p(rows)) == len(rest)
    for w, p in enumerate(rest):
        v = np.zeros(parts.shape[1], dtype=np.uint8)
        for j, q in enumerate(inputs):
            v ^= MUL[rows[w, j], parts[q]]
        if (v != parts[p]).any():
            return False
    return True


def brute_force(lib, k, m, parts, given, failed):
    """(|E|, E as a bit mask) for the smallest e <= 2 with 2e + |F| <= s that one set E explains, or None"""
    kept = [p for p in sorted(given) if p not in failed]
    s = len(given) - k
    if consistent(lib, k, m, parts, kept):
        return 0, 0
    for e in (1, 2):
        if 2 * e + len(failed) > s:
            break
        sets = [E for E in itertools.combinations(kept, e) if consistent(lib, k, m, parts, [p for p in kept if p not in E])]
        assert len(sets) <= 1, ("two sets within the radius explain the stripe", sets)  # MDS: never
        if sets:
            return e, sum(1 << p for p in sets[0])
    return None


def locate(lib, k, m, parts, given, failed, length=LEN):
    g = np.array([int(i in given) for i in range(k + m)], dtype=np.uint8)
    f = np.array([int(i in failed) for i in range(k + m)], dtype=np.uint8)
    blocks = [np.ascontiguousarray(parts[i]) for i in range(k + m)]
    ptrs = (C.c_void_p * (k + m))(*[b.ctypes.data for b in blocks])
    located = C.c_uint64(0)
    rc = lib.lzgpu_debug_locate_errors(k, m, _p(g), _p(f), ptrs, length, C.byref(located))
    return rc, located.value


def damage(parts, p, shape, rng):
    """a stale block: bytes of part p changed over a range, one byte, the first half or the second half"""
    if shape == "range":
        a = int(rng.integers(0, LEN // 2))
        parts[p, a:a + 100] ^= rng.integers(1, 256, min(100, LEN - a), dtype=np.uint8)
    elif shape == "byte":
        parts[p, int(rng.integers(0, LEN))] ^= int(rng.integers(1, 256))
    elif shape == "low":
        parts[p, :LEN // 2] ^= rng.integers(1, 256, LEN // 2, dtype=np.uint8)
    else:  # "high": disjoint from "low"
        parts[p, LEN // 2:] ^= rng.integers(1, 256, LEN - LEN // 2, dtype=np.uint8)


# (k, m): Vandermonde ec(5,3), ec(8,4), ec(20,4); Cauchy ec(4,5), ec(10,6)
GOALS = [(5, 3), (8, 4), (20, 4), (4, 5), (10, 6)]
SHAPES = [("range", "range"), ("low", "high"), ("byte", "byte"), ("byte", "range")]


def cases(k, m, rng):
    """(given, F, E, shapes): every F size the radius allows, with and without a lost part, pairs of every kind, and beyond it"""
    n = k + m
    for lost in ((), (int(rng.integers(0, k)),), (k + m - 1,)):
        given = [p for p in range(n) if p not in lost]
        s = len(given) - k
        for nf in range(0, max(0, s - 1)):
            for kind in ("dd", "dp", "pp", "one", "three"):
                data = [p for p in given if p < k]
                par = [p for p in given if p >= k]
                pool = list(rng.permutation(given))
                f = tuple(sorted(pool[:nf]))
                rest = [p for p in pool[nf:]]
                d_rest = [p for p in rest if p in data]
                p_rest = [p for p in rest if p in par]
                if kind == "dd" and len(d_rest) >= 2:
                    e = d_rest[:2]
                elif kind == "dp" and d_rest and p_rest:
                    e = [d_rest[0], p_rest[0]]
                elif kind == "pp" and len(p_rest) >= 2:
                    e = p_rest[:2]
                elif kind == "one":
                    e = rest[:1]
                elif kind == "three" and len(rest) >= 3:
                    e = rest[:3]
                else:
                    continue
                for shape in SHAPES:
                    yield tuple(given), f, tuple(int(x) for x in e), shape


@pytest.mark.parametrize("k,m", GOALS)
def test_locator_equals_the_brute_force(k, m):
    lib = _lib.load()
    gen = generator(lib, k, m)
    rng = np.random.default_rng(k * 100 + m)
    counts = {"located2": 0, "located1": 0, "refused": 0}
    for given, f, e, shape in cases(k, m, rng):
        data = rng.integers(0, 256, (k, LEN), dtype=np.uint8)
        parts = encode(gen, data)
        for p in f:
            parts[p] ^= rng.integers(0, 256, LEN, dtype=np.uint8)   # the punctured blocks: any bytes
        for i, p in enumerate(e):
            damage(parts, p, shape[i % 2], rng)
        want = brute_force(lib, k, m, parts, given, f)
        rc, located = locate(lib, k, m, parts, given, f)
        if want is None:
            assert rc == _lib.ERR_INCONSISTENT, (given, f, e, shape, rc, hex(located))
            counts["refused"] += 1
        else:
            assert (rc, located) == want, (given, f, e, shape, rc, hex(located), want)
            if want[0]:
                counts[f"located{want[0]}"] += 1
            if len(e) <= 2 and 2 * len(e) + len(f) <= len(given) - k:
                assert located == sum(1 << p for p in e), (given, f, e, shape)
    assert counts["located1"] and counts["refused"]
    if m >= 4:
        assert counts["located2"]


def test_locator_edge_cases():
    """ec(8,4): a pair whose differing bytes are disjoint (no byte shows both), one part differing in one byte only, zero-syndrome
    bytes around them, a codeword, and three parts beyond the radius"""
    lib = _lib.load()
    k, m = 8, 4
    gen = generator(lib, k, m)
    rng = np.random.default_rng(5)
    parts = encode(gen, rng.integers(0, 256, (k, LEN), dtype=np.uint8))
    given = tuple(range(12))
    assert locate(lib, k, m, parts, given, ()) == (0, 0)
    stale = parts.copy()
    stale[2, 10] ^= 0x11
    stale[9, 200] ^= 0x22
    assert locate(lib, k, m, stale, given, ()) == (2, 1 << 2 | 1 << 9)
    stale[2, 10] ^= 0x11
    assert locate(lib, k, m, stale, given, ()) == (1, 1 << 9)
    stale = parts.copy()
    stale[3, 50] ^= 0x5A                                  # one byte shows one error, another both
    stale[3, 60] ^= 0x01
    stale[6, 60] ^= 0x02
    assert locate(lib, k, m, stale, given, ()) == (2, 1 << 3 | 1 << 6)
    stale[11, 70] ^= 0x03                                 # a third part: beyond the radius
    assert locate(lib, k, m, stale, given, ())[0] == _lib.ERR_INCONSISTENT
    stale = parts.copy()
    stale[1, 5] ^= 0x40
    stale[0] ^= 0xFF                                      # F = {0}: punctured, so only part 1 is located
    assert locate(lib, k, m, stale, given, (0,)) == (1, 1 << 1)
    stale[5, 6] ^= 0x40                                   # two errors beside one erasure with s = 4: beyond the radius
    assert locate(lib, k, m, stale, given, (0,))[0] == _lib.ERR_INCONSISTENT


def test_locator_refuses_bad_arguments():
    lib = _lib.load()
    parts = np.zeros((12, LEN), dtype=np.uint8)
    assert locate(lib, 8, 4, parts, (0, 1, 2, 3, 4, 5, 6, 7, 8), (9,))[0] == _lib.ERR_ARG      # a failed part that is not given
    assert locate(lib, 8, 4, parts, tuple(range(9)), (0, 1))[0] == _lib.ERR_ARG               # fewer than k parts outside F
    assert locate(lib, 8, 4, parts, tuple(range(12)), (), length=0)[0] == _lib.ERR_ARG
    assert locate(lib, 33, 4, np.zeros((37, LEN), dtype=np.uint8), tuple(range(37)), ())[0] == _lib.ERR_ARG


def test_stripe_decode_layout_matches_the_header(tmp_path):
    fields = [f for f, _ in _lib.LzStripeDecode._fields_]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(['#include <stdio.h>', '#include <stddef.h>', '#include "lzgpu.h"', 'int main(void) {',
                              'printf("%zu %zu", sizeof(lzgpu_stripe_decode), _Alignof(lzgpu_stripe_decode));'] +
                             [f'printf(" %zu", offsetof(lzgpu_stripe_decode, {f}));' for f in fields] +
                             ['printf(" %zu %d\\n", sizeof(((lzgpu_stripe_decode *)0)->located_crc), LZGPU_FIX_DECODED);', 'return 0; }']))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    size, align, *rest = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    offsets, (crc_bytes, decoded) = rest[:len(fields)], rest[len(fields):]
    assert size == 40 == C.sizeof(_lib.LzStripeDecode) == Engine.STRIPE_DECODE_DTYPE.itemsize
    assert align == 8 and crc_bytes == 8
    assert offsets == [getattr(_lib.LzStripeDecode, f).offset for f in fields]
    assert offsets == [Engine.STRIPE_DECODE_DTYPE.fields[f][1] for f in fields]
    assert offsets[:5] == [_lib.LzStripeRepair.__dict__[f].offset for f, _ in _lib.LzStripeRepair._fields_]
    assert decoded == _lib.FIX_DECODED == 6
