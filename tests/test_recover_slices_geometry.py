"""The launch geometry of lzgpu_recover_slices without a GPU: lzgpu_plan_recover_slices against a plain-Python restatement of the rules
of rs_geometry (csrc/slices_solve.h).

recover_slices_kernel is driven by host tables with hard caps: 192 read, write and CRC-stream entries and 64 wanted parity blocks per
combined stripe, and shared memory of 4096 + 1024 slots + 128 streams bytes up to 220 KiB.  The restatement counts, per stripe shape
(a full combined stripe of L = lcm(k_i) blocks, and the chunk's last one when L does not divide nb), the blocks of every given part
(reads), the image's positions plus every block of every part not given (writes), the CRC streams (reads + writes - image), the
parity blocks not given (outs) and E, the GF(2^8) rank of the given parity equations restricted to the unknown positions; the
generators are the oracle's gf_gen_rs_matrix / gf_gen_cauchy1_matrix with the reference's switch to Cauchy rows.  Checked: every row
of EDGES (the GPU cases of test_gpu_recover_slices_edges.py, whose literal counts must equal the restatement), the requests that
must refuse, both sides of every cap, and a seeded sample of goal pairs and triples; the accepted request with the largest shared
memory the sample finds is SMEM_EDGE, which the GPU file runs."""
import math
import random

import numpy as np
import pytest

from lizardfs_b200.engine import Engine, SliceType
from tests import _oracle as O
from tests.test_recover_slices_plan import ginv, gmul, rank

ENTRY_CAP, OUT_CAP, SMEM_CAP = 192, 64, 220 * 1024

MUL = np.array([[gmul(a, b) for b in range(256)] for a in range(256)], dtype=np.uint8)
INV = np.array([0] + [ginv(a) for a in range(1, 256)], dtype=np.uint8)


def gf_rref(rows, n):
    """reduced row echelon form over GF(2^8) of a list of rows of length n (numpy row operations): its nonzero rows"""
    m = np.array(rows, dtype=np.uint8).reshape(len(rows), n)
    r = 0
    for c in range(n):
        if r == m.shape[0]:
            break
        nz = np.nonzero(m[r:, c])[0]
        if nz.size == 0:
            continue
        p = r + int(nz[0])
        m[[r, p]] = m[[p, r]]
        m[r] = MUL[INV[m[r, c]], m[r]]
        f = m[:, c].copy()
        f[r] = 0
        m ^= MUL[f[:, None], m[r][None, :]]
        r += 1
    return m[:r]


def gf_rank(rows, n):
    return len(gf_rref(rows, n)) if rows and n else 0


_oracle = None


def oracle():
    global _oracle
    if _oracle is None:
        _oracle = O.load_oracle()
    return _oracle


_gens = {}


def gen_rows(kind, k, m):
    """the m parity rows of an xor/ec slice: XOR is one row of ones; ec(k,m) takes the Cauchy matrix when m >= 5 or (m = 4 and
    k > 20) (reed_solomon.h), else the Vandermonde one"""
    if (kind, k, m) not in _gens:
        if kind == 0:
            rows = [[1] * k]
        else:
            cauchy = m >= 5 or (m == 4 and k > 20)
            full = (oracle().gen_cauchy1_matrix if cauchy else oracle().gen_rs_matrix)(k + m, k)
            rows = [[int(v) for v in full[k + r]] for r in range(m)]
        _gens[(kind, k, m)] = rows
    return _gens[(kind, k, m)]


def slices(names):
    """per slice (k, m, base, parity rows); the standard slice is k = 1, m = 0"""
    out, base = [], 0
    for n in names:
        if n == "std":
            out.append((1, 0, base, []))
            base += 1
            continue
        g = SliceType(n)
        out.append((g.k, g.m, base, gen_rows(g.kind, g.k, g.m)))
        base += g.k + g.m
    return out, base


def goals_of(names):
    return [SliceType(2, 1, 0) if n == "std" else SliceType(n) for n in names]


def lcm_of(lay):
    L = 1
    for k, m, _, _ in lay:
        if m:
            L = L * k // math.gcd(L, k)
    return L


def shape(lay, given, valid):
    """one stripe shape of `valid` chunk blocks: reads, writes (the image's `valid` entries included), states, outs, unknowns and E"""
    L = lcm_of(lay)
    reads, writes, outs = 0, valid, 0
    known = set()
    for k, m, base, _ in lay:
        for s in range(L // k):
            if s * k >= valid:       # the slice stripe has no chunk block in this shape
                continue
            for p in range(k + m):
                if given[base + p]:
                    reads += 1
                    if p < k and s * k + p < valid:
                        known.add(s * k + p)
                else:
                    writes += 1
                    outs += p >= k
    unk = [q for q in range(valid) if q not in known]
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
                    if s * k + j in col:
                        row[col[s * k + j]] = gen[r][j]
                if any(row):
                    eqs.append(row)
    # unknown x is determined when e_x lies in the row space of the equations, i.e. is a row of their reduced echelon form
    R = gf_rref(eqs, len(unk)) if eqs and unk else np.zeros((0, len(unk)), np.uint8)
    det = sum(1 << q for q in known) + sum(1 << q for q in range(valid, L))
    for row in R:
        nz = np.nonzero(row)[0]
        if nz.size == 1:
            det |= 1 << unk[int(nz[0])]
    return dict(reads=reads, writes=writes, states=reads + writes - valid, outs=outs, U=len(unk), E=len(R), det=det)


def geometry(names, nb, given):
    """the plan's ok, G, threads, stages and smem_bytes, and the shapes it is the maximum over: the full stripe when nb >= L, the
    tail when L does not divide nb (both the tail when nb < L; both the full one when L divides nb)"""
    lay, _ = slices(names)
    L = lcm_of(lay)
    tail = nb % L
    used = [shape(lay, given, v) for v in {L if nb >= L else tail, tail if tail else L}]
    slots = max(L + s["E"] + s["outs"] for s in used)
    states = max(s["states"] for s in used)
    smem = 4096 + 1024 * slots + 128 * states
    fits = all(s["reads"] <= ENTRY_CAP and s["writes"] <= ENTRY_CAP and s["states"] <= ENTRY_CAP and s["outs"] <= OUT_CAP for s in used)
    return dict(ok=int(fits and smem <= SMEM_CAP), G=1 if L >= 8 else 8 // L, threads=256, stages=1, smem_bytes=smem)


def pattern(names, spec):
    """given flags over the flat parts: "all", "data", "parity", ("slice", i) = every part of slice i alone, ("parity_of", i) = the
    parity parts of slice i alone, or an explicit list of flat parts"""
    lay, n = slices(names)
    given = [0] * n
    for i, (k, m, base, _) in enumerate(lay):
        for p in range(k + m):
            if spec == "all" or (spec == "data" and p < k) or (spec == "parity" and p >= k) or spec == ("slice", i) or \
                    (spec == ("parity_of", i) and p >= k):
                given[base + p] = 1
    if isinstance(spec, list):
        for g in spec:
            given[g] = 1
    return given


def check_plan(names, nb, given):
    p = Engine.plan_recover_slices(goals_of(names), nb, given)
    want = geometry(names, nb, given)
    assert {f: p[f] for f in want} == want, (names, nb, given)
    return want


# The GPU cases: goal set, given parts, the literal counts of the full combined stripe (L = 5: the row's own), block counts
EDGES = [
    # L = 48: writes = 192, states = 192; 48 unknowns from 48 Cauchy equations of ec(16,16); 48 wanted parity blocks
    (("ec(3,3)", "ec(16,16)"), ("parity_of", 1), dict(L=48, reads=48, writes=192, states=192, outs=48, U=48, E=48, G=1), (47, 113, 1024)),
    # reads = 192: every block of every part, the second copies and parity blocks only verified
    (("ec(3,3)", "ec(16,16)"), "all", dict(L=48, reads=192, writes=48, states=192, outs=0, U=0, E=0, G=1), (47, 113)),
    # 64 flat parts, outs = 64, Cauchy rows up to 15 of ec(16,16) and ec(8,16)
    (("ec(16,16)", "ec(8,16)", "ec(4,4)"), "data", dict(L=16, reads=48, writes=80, states=112, outs=64, U=0, E=0, G=1), (15, 41)),
    (("ec(16,16)", "ec(8,16)", "ec(4,4)"), "parity", dict(L=16, reads=64, writes=64, states=112, outs=0, U=16, E=16, G=1), (15, 41)),
    # known positions inside the stripes of Cauchy equations: ec(8,16) data parts 0-3 pin 8 positions, ec(16,16) parity rows 8-15
    # solve the other 8 (their syndromes carry the known positions' share), ec(4,4)'s parity is only verified
    (("ec(16,16)", "ec(8,16)", "ec(4,4)"), [32, 33, 34, 35] + list(range(24, 32)) + [60, 61, 62, 63],
     dict(L=16, reads=32, writes=96, states=112, outs=40, U=8, E=8, G=1), (15, 41)),
    # L = 63: outs = 64, states = 190
    (("ec(7,4)", "ec(9,4)"), "data", dict(L=63, reads=126, writes=127, states=190, outs=64, U=0, E=0, G=1), (62, 143, 1024)),
    # L = 63: 63 unknowns, 62 equations (27 Vandermonde, 35 Cauchy), only position 44 determined; at nb = 62 the last stripe's 62
    # unknowns are all determined by its 62 equations
    (("ec(7,3)", "ec(9,5)"), "parity", dict(L=63, reads=62, writes=189, states=188, outs=0, U=63, E=62, G=1), (62, 125)),
    # four striped slices, L = 4, G = 2: Vandermonde rows 0-2
    (("xor2", "ec(2,2)", "ec(4,2)", "ec(4,3)"), "parity", dict(L=4, reads=11, writes=20, states=27, outs=0, U=4, E=4, G=2), (3, 10, 1024)),
    # L = 3, G = 2: xor3 data 0 and parity, ec(3,2) data 1 and parity row 0
    (("xor3", "ec(3,2)"), [0, 3, 5, 7], dict(L=3, reads=4, writes=8, states=9, outs=1, U=1, E=1, G=2), (2, 8)),
    # L = 5, G = 1 (8 // L): xor5 data 0, 1 and parity, ec(5,3) data 1, 2 and parity rows 1, 2
    (("xor5", "ec(5,3)"), [0, 1, 5, 7, 8, 12, 13], dict(L=5, reads=7, writes=12, states=14, outs=1, U=2, E=2, G=1), (4, 12)),
]

# Requests that must refuse with LZGPU_ERR_ARG: the cap each one passes
REFUSED = [
    (("ec(3,3)", "ec(16,16)"), "data", dict(outs=96)),
    (("ec(3,2)", "ec(4,2)", "ec(5,2)"), "data", dict(states=274)),
    (("ec(3,2)", "ec(4,2)", "ec(5,2)"), "parity", dict(states=274)),
    (("ec(3,2)", "ec(4,2)", "ec(5,2)"), "all", dict(states=274)),
    (("xor2", "xor3", "xor4", "xor5"), "data", dict(states=317)),
]

# The accepted request with the largest shared memory the sample of test_sampled_goal_sets finds (goal set, given, nb)
# (ec(3,3)'s parity alone: 48 unknowns from 48 Vandermonde equations, the 48 parity blocks of ec(16,16) wanted, 192 streams)
SMEM_EDGE = (("ec(3,3)", "ec(16,16)"), [3, 4, 5], 121)
SMEM_EDGE_BYTES = 176128


def full_shape(names, spec):
    lay, _ = slices(names)
    L = lcm_of(lay)
    s = shape(lay, pattern(names, spec), L)
    del s["det"]
    return dict(L=L, G=1 if L >= 8 else 8 // L, **s)


def test_numpy_rank_matches_the_plain_rank():
    rng = random.Random(5)
    for _ in range(60):
        n = rng.randrange(1, 9)
        rows = [[rng.choice([0, 0, 1, rng.randrange(256)]) for _ in range(n)] for _ in range(rng.randrange(1, 10))]
        assert gf_rank(rows, n) == rank(rows, n)


def test_generators_are_the_reference_switch():
    """Cauchy row r of ec(k,m) is 1 / ((k + r) ^ j) from m >= 5, and for m = 4 above k = 20; Vandermonde row r is (2^r)^j"""
    for k, m in [(21, 4), (9, 5), (16, 16), (8, 16), (2, 32)]:
        for r in range(m):
            assert gen_rows(1, k, m)[r] == [ginv((k + r) ^ j) for j in range(k)], (k, m, r)
    for k, m in [(20, 4), (9, 4), (7, 3), (4, 2), (32, 1)]:
        for r in range(m):
            x, row = 1, []
            for _ in range(k):
                row.append(x)
                for _ in range(r):
                    x = gmul(x, 2)
            assert gen_rows(1, k, m)[r] == row, (k, m, r)


def edge_id(row):
    names, spec = row[0], row[1]
    return "+".join(names) + "-" + (spec if isinstance(spec, str) else "_".join(map(str, spec)))


@pytest.mark.parametrize("names,spec,lit,nbs", EDGES, ids=[edge_id(r) for r in EDGES])
def test_edge_rows_match_the_restatement(names, spec, lit, nbs):
    assert full_shape(names, spec) == lit
    given = pattern(names, spec)
    for nb in nbs:
        assert check_plan(names, nb, given)["ok"] == 1, (names, nb)


def test_the_caps_are_reached_and_refused_on_both_sides():
    by = {(n, str(s)): full_shape(n, s) for n, s, _, _ in EDGES}
    assert by[(("ec(3,3)", "ec(16,16)"), "('parity_of', 1)")]["writes"] == ENTRY_CAP
    assert by[(("ec(3,3)", "ec(16,16)"), "('parity_of', 1)")]["states"] == ENTRY_CAP
    assert by[(("ec(3,3)", "ec(16,16)"), "all")]["reads"] == ENTRY_CAP
    assert by[(("ec(16,16)", "ec(8,16)", "ec(4,4)"), "data")]["outs"] == OUT_CAP
    assert by[(("ec(7,4)", "ec(9,4)"), "data")]["outs"] == OUT_CAP
    assert slices(("ec(16,16)", "ec(8,16)", "ec(4,4)"))[1] == 64
    for names, spec, over in REFUSED:
        got = full_shape(names, spec)
        assert {f: got[f] for f in over} == over
        given = pattern(names, spec)
        for nb in (1024, 1023, lcm_of(slices(names)[0]) - 1):
            assert check_plan(names, nb, given)["ok"] == 0, (names, spec, nb)


def sample_sets(rng, count):
    """goal pairs and triples with L <= 64 and at most 64 parts"""
    types = ["std"] + [f"xor{k}" for k in range(2, 10)] + [f"ec({k},{m})" for k in range(2, 33) for m in range(1, 33)]
    out = []
    while len(out) < count:
        names = tuple(rng.sample(types, rng.choice((2, 3))))
        if all(n == "std" for n in names) or sum(n == "std" for n in names) > 1:
            continue
        lay, n = slices(names)
        if n <= 64 and lcm_of(lay) <= 64:
            out.append(names)
    return out


def test_sampled_goal_sets():
    """every request of a seeded sample against the restatement, at nb = 1024, L - 1 and a ragged count; the largest accepted shared
    memory is SMEM_EDGE, and the sample steps one past the write, stream and wanted-parity caps, where the plan refuses"""
    rng = random.Random(2026)
    best = (0, None)
    over = {}
    checked = 0
    for names in sample_sets(rng, 400) + [n for n, _, _, _ in EDGES]:
        lay, n = slices(names)
        L = lcm_of(lay)
        specs = ["all", "data", "parity"] + [(f, i) for f in ("slice", "parity_of") for i in range(len(lay))]
        for _ in range(3):
            keep = rng.uniform(0.05, 0.95)
            specs.append([g for g in range(n) if rng.random() < keep])
        for spec in specs:
            given = pattern(names, spec)
            parts = [g for g in range(n) if given[g]]
            full = shape(lay, given, L)
            for f, cap in (("reads", ENTRY_CAP), ("writes", ENTRY_CAP), ("states", ENTRY_CAP), ("outs", OUT_CAP)):
                if full[f] == cap + 1 and f not in over:
                    over[f] = (names, parts)
            for nb in sorted({1024, max(1, L - 1), min(1024, 2 * L + L // 2 + 1)}):
                g = check_plan(names, nb, given)
                checked += 1
                if g["ok"] and g["smem_bytes"] > best[0]:
                    best = (g["smem_bytes"], (names, parts, nb))
    assert checked > 5000
    assert best == (SMEM_EDGE_BYTES, SMEM_EDGE), best
    assert set(over) >= {"writes", "states", "outs"}, over
    for f, (names, parts) in over.items():
        assert check_plan(names, 1024, pattern(names, parts))["ok"] == 0, (f, names, parts)


def test_determined_masks_of_the_edge_rows():
    """the plan's masks for every edge row (the GPU test takes the wanted parts of the L = 63, E = 62 row from them): a position is
    determined when it is known or its unit vector lies in the row space of the equations (restated here with the oracle's rows)"""
    for names, spec, _, nbs in EDGES + [(SMEM_EDGE[0], SMEM_EDGE[1], None, (SMEM_EDGE[2],))]:
        lay, _ = slices(names)
        L = lcm_of(lay)
        given = pattern(names, spec)
        for nb in nbs:
            p = Engine.plan_recover_slices(goals_of(names), nb, given)
            assert p["determined"] == shape(lay, given, L)["det"], (names, spec)
            assert p["tail_determined"] == shape(lay, given, nb % L or L)["det"], (names, spec, nb)
    lay, _ = slices(("ec(7,3)", "ec(9,5)"))
    given = pattern(("ec(7,3)", "ec(9,5)"), "parity")
    assert shape(lay, given, 63)["det"] == 1 << 44
    assert shape(lay, given, 62)["det"] == (1 << 63) - 1 and shape(lay, given, 62)["E"] == 62
