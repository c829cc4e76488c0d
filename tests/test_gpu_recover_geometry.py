"""The fused degraded read (fused_recover_kernel, csrc/fused_kernel.cuh; bs_recover3_kernel, csrc/bs_recover_kernel.cuh) at every
kernel instantiation and geometry its router (recover_plan, csrc/fused_plan.h) selects.

recover_plan() picks, per call, one of about thirty instantiations: the geometry (one or two 9-warp CTAs, one 16-warp CTA, the
DIRECT form for Cauchy generators, bit planes for three lost data parts), the number of lost data parts e, a compile-time k, the
parity rows known at compile time, the item width, the form of the solve (RAID-6 elimination, three-unknown elimination, the
inverse with or without the last-unknown shortcut; x0 doublings or a multiply), the stripe group G and the stage ring.  A request
routed to the wrong instantiation still returns the right bytes, so every case below asserts its launch geometry as well.
CASES holds one request per feature value the router's space has, alone and paired with e
(test_recover_geometry_table_covers_the_router_space enumerates that space on the CPU through lzgpu_plan_recover and fails when a
table entry is missing, redundant, or its literal plan no longer matches), plus one request per rule that sends a call to the
generic route.

Every case runs at a ragged block count (nb % k != 0, three units per chunk, the last one partial), at nb < k G (one partial
unit) and, for k <= 8, at nb < k (pb = 1: lost data parts at positions >= nb are pure zero padding); three also at nb = 1024.
Each call runs on three contexts: the case's switches, the same plus LZGPU_GRID_CAP=2 (every CTA walks several units) and
LZGPU_DISABLE_FUSED=1 (the generic route), with and without stored CRCs and with and without the chunk-order image.  Outputs start
as 0xA5 bytes; every rebuilt byte must equal the original data part (which the oracle's recover_chunk returns too) and the generic
route's answer, the image must equal the chunk and keep the sentinel in the block of padding of its stride, outputs of lost parts
that are not wanted must keep the sentinel when no image is written, and lzgpu_debug_last_geometry must show the planned launch."""
import os
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import _oracle as O

BLOCK = 65536
N, N_CAP = 3, 5                 # chunks per call; under the cap of 2 CTAs, 5 chunks give more than 2 x 2 units at nb < k G as well
ZERO_CRC = 0xD7978EEB           # CRC of a 64 KiB zero block (the blocks a short data part does not have)
SENTINEL = 0xA5
K_NAMES = {_lib.KERNEL_RECOVER_GEO0: "GEO0", _lib.KERNEL_RECOVER_GEO1: "GEO1", _lib.KERNEL_RECOVER_GEO2: "GEO2",
           _lib.KERNEL_RECOVER_DIRECT: "DIRECT", _lib.KERNEL_RECOVER_BS3: "BS3"}
SOLVE_NAMES = {_lib.RECOVER_SOLVE_DIRECT: "direct", _lib.RECOVER_SOLVE_RAID6: "raid6", _lib.RECOVER_SOLVE_ELIM3: "elim3",
               _lib.RECOVER_SOLVE_INVERSE: "inverse", _lib.RECOVER_SOLVE_INVERSE_ROW0: "inverse, row 0"}
ROWS_NAMES = {_lib.RECOVER_ROWS_GENERAL: "general", _lib.RECOVER_ROWS_FIRST_E: "0..e-1", _lib.RECOVER_ROWS_DIRECT: "direct"}
REFUSALS = {_lib.RECOVER_REFUSED_DIRECT_OFF: "LZGPU_DIRECT_WIDE=-2", _lib.RECOVER_REFUSED_OVER_FOUR_LOST: "more than four lost",
            _lib.RECOVER_REFUSED_NO_LOST_DATA: "e = 0", _lib.RECOVER_REFUSED_DIRECT_SLOWER: "Cauchy, e >= 2, not verify + image",
            _lib.RECOVER_REFUSED_PARITY_WANTED: "a wanted parity part"}
# the context switches of a case (lzgpu_recover_switches fields) and the environment variables a context reads them from
SWITCHES = {"default": {}, "geo0": {"recover_geo": 0}, "geo1": {"recover_geo": 1}, "geo2": {"recover_geo": 2}, "two0": {"recover_two": 0},
            "two1": {"recover_two": 1}, "k3off": {"recover_k3": 0}, "bsoff": {"bs_recover": 0}, "wide0": {"direct_wide": 0},
            "wide1": {"direct_wide": 1}, "direct_off": {"direct_wide": -2}}
ENV = {"recover_geo": "LZGPU_RECOVER_GEO", "recover_two": "LZGPU_RECOVER_TWO", "recover_k3": "LZGPU_RECOVER_K3",
       "bs_recover": "LZGPU_BS_RECOVER", "direct_wide": "LZGPU_DIRECT_WIDE"}
PLAN_KEYS = ("kernel", "kt", "rows", "item_bytes", "solve", "doublings", "G", "stages", "threads", "gf_warps", "smem_bytes")

CASES = [
    # goal, lost parts (data parts first, then parity parts), switch set, verify, image, wanted ("data": the lost data parts,
    # "all": every lost part), literal plan: PLAN_KEYS values, or ("refused", rule).  kernel 3 / 4 / 5: fused_recover_kernel on
    # GEO 0 / 1 / 2, 6: its DIRECT form, 7: bs_recover3_kernel; rows 0 general, 1 rows 0 .. e-1, 2 DIRECT; solve 0 DIRECT, 1 RAID-6,
    # 2 three-unknown elimination, 3 inverse, 4 inverse with the last-unknown shortcut
    ('ec(8,2)', (1, 4), 'default', 1, 1, "data", (3, 8, 1, 16, 4, -1, 8, 6, 288, 0, 196768)),
    ('ec(17,1)', (16,), 'default', 0, 0, "data", (4, 0, 1, 16, 4, -1, 2, 3, 288, 0, 52336)),
    ('ec(5,2)', (0, 4), 'default', 0, 0, "data", (5, 5, 1, 16, 1, 0, 16, 5, 512, 0, 204944)),
    ('ec(22,4)', (21,), 'default', 0, 0, "data", (6, 0, 2, 16, 0, -1, 4, 4, 512, 0, 180352)),
    ('ec(17,2)', (16, 17), 'default', 0, 1, "data", (3, 0, 0, 16, 3, -1, 2, 6, 288, 0, 104608)),
    ('ec(11,3)', (0, 10, 12), 'geo1', 0, 0, "data", (4, 0, 0, 16, 3, -1, 4, 3, 288, 0, 67696)),
    ('ec(13,4)', (0, 3, 5, 12), 'default', 0, 0, "data", (5, 0, 1, 8, 4, -1, 8, 3, 512, 0, 159856)),
    ('ec(8,6)', (0, 7), 'default', 1, 1, "data", (6, 0, 2, 8, 0, -1, 16, 3, 512, 0, 196720)),
    ('ec(4,4)', (0, 2, 3, 5), 'geo0', 0, 0, "data", (3, 0, 0, 16, 3, -1, 16, 6, 288, 0, 196768)),
    ('ec(5,3)', (2, 3, 4), 'default', 1, 0, "data", (7, 5, 1, 32, 2, 2, 14, 5, 512, 7, 179344)),
    ('ec(5,3)', (4, 5, 6), 'geo2', 0, 0, "data", (5, 0, 0, 16, 3, -1, 16, 5, 512, 0, 204944)),
    ('ec(22,4)', (0, 11, 21), 'wide0', 0, 0, "data", (6, 0, 2, 4, 0, -1, 4, 4, 512, 0, 180352)),
    ('ec(8,4)', (0, 3, 5, 7), 'default', 0, 0, "data", (3, 0, 1, 16, 4, -1, 8, 6, 288, 0, 196768)),
    ('ec(5,3)', (0, 1, 2), 'bsoff', 0, 0, "data", (5, 5, 1, 8, 2, 0, 16, 5, 512, 0, 204944)),
    ('ec(22,4)', (0, 3, 5, 21), 'wide0', 0, 0, "data", (6, 0, 2, 4, 0, -1, 4, 4, 512, 0, 180352)),
    ('ec(22,3)', (0, 1, 22), 'default', 0, 0, "data", (5, 0, 0, 16, 3, -1, 4, 4, 512, 0, 180352)),
    ('ec(17,2)', (0, 16), 'geo0', 0, 0, "data", (3, 0, 1, 16, 1, 0, 2, 6, 288, 0, 104608)),
    ('ec(2,2)', (0, 1), 'geo1', 0, 0, "data", (4, 0, 1, 16, 1, 0, 32, 3, 288, 0, 98416)),
    ('ec(29,3)', (4, 5, 28), 'default', 1, 0, "data", (7, 0, 1, 32, 2, -1, 2, 6, 512, 1, 178336)),
    ('ec(8,3)', (0, 1, 2), 'bsoff', 0, 0, "data", (3, 0, 1, 16, 2, 0, 8, 6, 288, 0, 196768)),
    ('ec(11,4)', (0, 11, 12, 13), 'default', 0, 0, "data", (4, 0, 0, 16, 3, -1, 4, 3, 288, 0, 67696)),
    ('ec(4,2)', (1, 2), 'default', 0, 0, "data", (5, 4, 1, 16, 1, 1, 32, 3, 512, 0, 196720)),
    ('ec(2,4)', (0, 1, 3, 4), 'geo0', 0, 0, "data", (3, 0, 0, 16, 3, -1, 32, 6, 288, 0, 196768)),
    ('xor3', (0,), 'geo2', 0, 0, "data", (5, 3, 1, 16, 4, -1, 32, 4, 512, 0, 196736)),
    ('xor8', (0,), 'default', 0, 0, "data", (3, 8, 1, 16, 4, -1, 8, 6, 288, 0, 196768)),
    ('ec(12,3)', (0, 1, 2), 'default', 0, 0, "data", (7, 0, 1, 32, 2, 0, 8, 4, 512, 4, 196736)),
    ('ec(8,3)', (0, 1, 2), 'default', 0, 0, "data", (7, 8, 1, 32, 2, 0, 16, 3, 512, 8, 196720)),
    ('ec(6,3)', (3, 4, 5), 'bsoff', 0, 0, "data", (5, 6, 1, 8, 2, 3, 16, 4, 512, 0, 196736)),
    ('ec(13,4)', (0, 1, 2, 13), 'default', 0, 0, "data", (5, 0, 0, 8, 3, -1, 8, 3, 512, 0, 159856)),
    ('ec(17,2)', (3, 16), 'geo1', 0, 0, "data", (4, 0, 1, 16, 1, 3, 2, 3, 288, 0, 52336)),
    ('ec(8,2)', (0, 1), 'geo1', 0, 0, "data", (4, 8, 1, 16, 4, -1, 8, 3, 288, 0, 98416)),
    ('ec(22,4)', (0, 1), 'wide0', 0, 0, "data", (6, 0, 2, 4, 0, -1, 4, 4, 512, 0, 180352)),
    ('xor8', (0,), 'geo2', 0, 0, "data", (5, 8, 1, 16, 4, -1, 16, 3, 512, 0, 196720)),
    ('ec(8,6)', (0,), 'wide0', 0, 0, "data", (6, 0, 2, 4, 0, -1, 16, 3, 512, 0, 196720)),
    ('ec(8,6)', (0, 1, 2), 'wide1', 0, 0, "data", (6, 0, 2, 8, 0, -1, 16, 3, 512, 0, 196720)),
    ('ec(8,6)', (0, 1, 2, 3), 'wide1', 0, 0, "data", (6, 0, 2, 8, 0, -1, 16, 3, 512, 0, 196720)),
    ('ec(8,4)', (0, 1, 8, 10), 'default', 0, 0, "data", (3, 0, 0, 16, 3, -1, 8, 6, 288, 0, 196768)),
    ('ec(8,4)', (0, 1, 8, 9), 'default', 0, 0, "data", (3, 0, 0, 16, 3, -1, 8, 6, 288, 0, 196768)),
    ('ec(5,4)', (0, 1, 2, 3), 'default', 0, 0, "data", (5, 0, 1, 8, 4, -1, 16, 5, 512, 0, 204944)),
    ('ec(22,2)', (5, 6), 'default', 0, 0, "data", (5, 0, 1, 16, 1, -1, 4, 4, 512, 0, 180352)),
    ('ec(17,2)', (3, 16), 'geo0', 0, 0, "data", (3, 0, 1, 16, 1, 3, 2, 6, 288, 0, 104608)),
    ('ec(17,2)', (5, 6), 'geo0', 0, 0, "data", (3, 0, 1, 16, 1, -1, 2, 6, 288, 0, 104608)),
    ('ec(17,2)', (5, 6), 'geo1', 0, 0, "data", (4, 0, 1, 16, 1, -1, 2, 3, 288, 0, 52336)),
    ('ec(8,3)', (1, 4, 6), 'bsoff', 0, 0, "data", (3, 0, 1, 16, 2, 1, 8, 6, 288, 0, 196768)),
    ('ec(8,3)', (4, 5, 7), 'bsoff', 0, 0, "data", (3, 0, 1, 16, 2, -1, 8, 6, 288, 0, 196768)),
    ('ec(22,3)', (4, 5, 21), 'bsoff', 0, 0, "data", (5, 0, 1, 8, 2, -1, 4, 4, 512, 0, 180352)),
    ('ec(8,2)', (0, 1), 'geo2', 0, 0, "data", (5, 8, 1, 16, 4, -1, 16, 3, 512, 0, 196720)),
    ('xor2', (0,), 'default', 0, 0, "data", (4, 0, 1, 16, 4, -1, 32, 3, 288, 0, 98416)),
    ('xor2', (0,), 'default', 0, 1, "data", (3, 0, 1, 16, 4, -1, 32, 6, 288, 0, 196768)),
    ('ec(3,2)', (0, 1), 'default', 0, 0, "data", (5, 3, 1, 16, 1, 0, 32, 4, 512, 0, 196736)),
    ('ec(6,2)', (0, 1), 'default', 0, 0, "data", (5, 6, 1, 16, 1, 0, 16, 4, 512, 0, 196736)),
    ('ec(6,4)', (0, 1, 2, 3), 'default', 0, 0, "data", (5, 0, 1, 8, 4, -1, 16, 4, 512, 0, 196736)),
    ('ec(17,4)', (0, 1, 2, 19), 'geo0', 0, 0, "data", (3, 0, 0, 16, 3, -1, 2, 6, 288, 0, 104608)),
    ('ec(17,4)', (0, 1, 2, 3), 'geo0', 0, 0, "data", (3, 0, 1, 16, 4, -1, 2, 6, 288, 0, 104608)),
    ('ec(4,4)', (0, 1, 2, 3), 'geo0', 0, 0, "data", (3, 0, 1, 16, 4, -1, 16, 6, 288, 0, 196768)),
    ('xor8', (0,), 'geo1', 0, 0, "data", (4, 8, 1, 16, 4, -1, 8, 3, 288, 0, 98416)),
    ('ec(22,1)', (0,), 'geo2', 0, 0, "data", (5, 0, 1, 16, 4, -1, 4, 4, 512, 0, 180352)),
    # the generic route
    ("ec(8,2)", (8,), "default", 1, 1, "all", ("refused", _lib.RECOVER_REFUSED_NO_LOST_DATA)),
    ("ec(8,3)", (1, 8), "default", 1, 1, "all", ("refused", _lib.RECOVER_REFUSED_PARITY_WANTED)),
    ("ec(10,5)", (2, 7), "default", 0, 1, "data", ("refused", _lib.RECOVER_REFUSED_DIRECT_SLOWER)),
    ("ec(8,6)", (0, 1, 2, 3, 4), "default", 1, 1, "data", ("refused", _lib.RECOVER_REFUSED_OVER_FOUR_LOST)),
    ("ec(21,4)", (3,), "direct_off", 1, 1, "data", ("refused", _lib.RECOVER_REFUSED_DIRECT_OFF)),
]
FULL_SIZE = [("ec(8,2)", (1, 4), "default"), ("ec(5,3)", (2, 3, 4), "default"), ("ec(22,4)", (21,), "default")]   # also at nb = 1024


def goal_of(name):
    return L.SliceType(name)


def want_of(g, lost, wanted):
    return [1 if i in lost and (i < g.k or wanted == "all") else 0 for i in range(g.k + g.m)]


def plan_of(name, lost, switches, verify, image, wanted="data"):
    g = goal_of(name)
    avail = [0 if i in lost else 1 for i in range(g.k + g.m)]
    return L.Engine.plan_recover(g, avail, want_of(g, lost, wanted), verify, image, SWITCHES[switches] or None)


def literal(plan):
    return tuple(plan[k] for k in PLAN_KEYS) if plan["fused"] else ("refused", plan["refusal"])


def used_parts(g, lost):
    return [i for i in range(g.k + g.m) if i not in lost][: g.k]


def block_counts(name, lost, plan):
    """ragged (nb % k != 0, three units per chunk, the last one partial), one partial unit, and nb < k for k <= 8"""
    k = goal_of(name).k
    G = plan["G"] if plan["fused"] else 4
    out = [2 * k * G + k * (G // 2) + 1, k * (G // 2) + 1]
    if k <= 8 and k >= 3:
        out.append(k - 1)
    return out


# ---- the router's space, on the CPU ---------------------------------------------------------------------------------------------

def _goals():
    return ([f"xor{k}" for k in range(2, 10)] + [f"ec({k},{m})" for k in range(2, 33) for m in range(1, 5)] +
            ["ec(8,6)", "ec(21,4)", "ec(32,5)"])


def _data_losses(k, m):
    """each single data loss; pairs and triples: first / last, adjacent at both ends and in the middle, x0 at 3, 4, 5; four parts"""
    out = [(j,) for j in range(k)]
    pairs = {(0, k - 1), (0, 1), (k - 2, k - 1), (k // 2 - 1, k // 2), (3, k - 1), (4, k - 1), (5, k - 1), (5, 6)}
    triples = {(0, 1, 2), (0, k // 2, k - 1), (k - 3, k - 2, k - 1), (3, 5, k - 1), (4, 5, k - 1), (5, 6, k - 1), (1, 4, 6)}
    quads = {(0, 1, 2, 3), (k - 4, k - 3, k - 2, k - 1), (0, 3, 5, k - 1), (4, 5, 6, k - 1), (5, 7, 9, k - 1)}
    for sets, e in ((pairs, 2), (triples, 3), (quads, 4)):
        if m >= e:
            out += sorted(s for s in sets if len(set(s)) == e and all(0 <= a < b < k for a, b in zip(s, s[1:])))
    return out


def _losses(k, m):
    """each data loss with the first e parity rows in use; for the first, last and sixth single loss and for every pair, triple and
    quadruple also every other set of e parity rows in use (the parity parts below the highest row in use that are not in it lost)"""
    from itertools import combinations
    out = []
    for d in _data_losses(k, m):
        e = len(d)
        rows = list(combinations(range(m), e)) if e > 1 or d[0] in (0, k - 1, min(5, k - 1)) else [tuple(range(e))]
        for r in rows:
            out.append(d + tuple(k + x for x in range(max(r)) if x not in r))
    return out


def features(name, lost, verify, plan):
    """the values of the instantiation and geometry features the router chooses, alone and paired with e"""
    g = goal_of(name)
    kn, e = K_NAMES[plan["kernel"]], plan["lost_data_parts"]
    G = plan["G"]
    f = {("kernel", kn), ("kt", kn, plan["kt"]), ("rows", kn, ROWS_NAMES[plan["rows"]]), ("item bytes", kn, plan["item_bytes"]),
         ("solve", kn, SOLVE_NAMES[plan["solve"]]), ("stages", kn, plan["stages"]),
         ("G", kn, "2" if G == 2 else ("multiple of 16" if G % 16 == 0 else "other"))}
    if plan["solve"] in (_lib.RECOVER_SOLVE_RAID6, _lib.RECOVER_SOLVE_ELIM3):
        d = plan["doublings"]
        f.add(("x0", kn, SOLVE_NAMES[plan["solve"]], "0" if d == 0 else ("doublings" if d > 0 else "multiply")))
    if plan["kernel"] != _lib.KERNEL_RECOVER_DIRECT:
        f.add(("parity rows in use", tuple(i - g.k for i in used_parts(g, lost) if i >= g.k)))
    if plan["kernel"] == _lib.KERNEL_RECOVER_BS3:
        f.add(("BS3 G rule", "stream warps" if verify else "no stream warps", "<= 4 GF warps" if plan["gf_warps"] <= 4 else "> 4 GF warps"))
    if g.k - 1 in lost:
        f.add(("last data part lost", kn))
    return f | {(e,) + x for x in f}


def check_invariants(name, lost, sw, verify, image, p):
    """what the router's comments state of every plan it makes"""
    g = goal_of(name)
    kn, e, G = p["kernel"], p["lost_data_parts"], p["G"]
    what = (name, lost, sw, verify, image, p)
    assert p["refusal"] == 0 and 1 <= e <= 4 and G >= 2 and G % 2 == 0, what
    rows = g.k * G * 4
    assert p["smem_bytes"] == p["stages"] * rows * 128 + 16 * p["stages"] + 64, what
    if kn in (_lib.KERNEL_RECOVER_GEO0, _lib.KERNEL_RECOVER_GEO1):
        assert rows <= 256 and p["threads"] == 288 and p["gf_warps"] == 0, what
        assert p["stages"] == (3 if kn == _lib.KERNEL_RECOVER_GEO1 else 6), what
        assert p["smem_bytes"] <= (100 if kn == _lib.KERNEL_RECOVER_GEO1 else 200) * 1024, what
        assert kn == _lib.KERNEL_RECOVER_GEO0 or e <= 2, what          # GEO 1 only for e <= 2
    else:
        assert G * 4 <= 256 and p["threads"] == 512 and p["smem_bytes"] <= 208 * 1024 and 3 <= p["stages"] <= 6, what
        assert rows <= 512 or kn == _lib.KERNEL_RECOVER_BS3, what     # (bs_recover3 without stream warps: no thread per input row)
    if kn == _lib.KERNEL_RECOVER_BS3:
        stream = -(-rows // 32) if verify else 0
        assert e == 3 and p["gf_warps"] == -(-16 * G // 32) and p["gf_warps"] <= 8 and p["gf_warps"] + stream <= 16, what
        assert p["kt"] in ((g.k,) if g.k in (5, 8) else (0,)), what
    else:
        assert p["gf_warps"] == 0, what
    if kn == _lib.KERNEL_RECOVER_DIRECT:
        assert p["kt"] == 0 and p["item_bytes"] in ((4, 16) if e == 1 else (4, 8)), what
    # a compile-time k only at its own k, e, rows and verify / image conditions
    first_e = p["rows"] == _lib.RECOVER_ROWS_FIRST_E
    if kn in (_lib.KERNEL_RECOVER_GEO0, _lib.KERNEL_RECOVER_GEO1, _lib.KERNEL_RECOVER_GEO2) and p["kt"]:
        assert p["kt"] == g.k and first_e, what
        if g.k == 8:
            assert e <= 2, what
        else:
            assert kn == _lib.KERNEL_RECOVER_GEO2 and sw != "k3off", what
            assert (g.k, e) in ((3, 1), (3, 2), (4, 2), (5, 2), (5, 3), (6, 2), (6, 3)), what
            assert not (e == 2 and g.k != 3 and verify and image), what
    if kn == _lib.KERNEL_RECOVER_GEO2 or kn == _lib.KERNEL_RECOVER_DIRECT:
        assert p["item_bytes"] in ((8,) if e >= 3 and kn == _lib.KERNEL_RECOVER_GEO2 else (4, 8, 16)), what
    # the solve forms and their doubling counts
    x0 = min(x for x in lost if x < g.k)
    if p["solve"] == _lib.RECOVER_SOLVE_RAID6:
        assert e == 2 and first_e and p["kt"] != 8 and p["doublings"] == (x0 if x0 <= 4 else -1), what
    elif p["solve"] == _lib.RECOVER_SOLVE_ELIM3:
        assert e == 3 and first_e and p["doublings"] == (x0 if x0 <= 3 else -1), what
    else:
        assert p["doublings"] == -1, what


def router_space():
    """{(goal, lost, switches, verify, image): plan} of every request of the space the router takes (no refusal)"""
    out = {}
    refused = set()
    for name in _goals():
        g = goal_of(name)
        for lost in _losses(g.k, g.m):
            avail = [0 if i in lost else 1 for i in range(g.k + g.m)]
            want = want_of(g, lost, "data")
            for sw, switches in SWITCHES.items():
                for verify in (0, 1):
                    for image in (0, 1):
                        p = L.Engine.plan_recover(g, avail, want, verify, image, switches or None)
                        if p["fused"]:
                            out[(name, lost, sw, verify, image)] = p
                        else:
                            refused.add(p["refusal"])
    return out, refused


def test_recover_geometry_table_covers_the_router_space():
    """every feature value, and every (e, feature value), that some request of the router's space has also occurs in CASES, and each
    case brings one that no other case has; every literal plan of CASES is the router's; every plan of the space keeps the
    invariants the router's comments state; each rule that sends a call to the generic route has its case"""
    space, refused = router_space()
    assert _lib.RECOVER_REFUSED_NO_GEOMETRY not in refused
    feats = set()
    for (name, lost, sw, verify, image), p in space.items():
        check_invariants(name, lost, sw, verify, image, p)
        feats |= features(name, lost, verify, p)
    per_case = []
    rules = set()
    for name, lost, sw, verify, image, wanted, want in CASES:
        p = plan_of(name, lost, sw, verify, image, wanted)
        assert literal(p) == want, (name, lost, sw, verify, image, literal(p))
        if p["fused"]:
            per_case.append(features(name, lost, verify, p))
        else:
            rules.add(p["refusal"])
            per_case.append(set())
    table = set().union(*per_case)
    assert not feats - table, sorted(feats - table, key=str)
    for i, f in enumerate(per_case):
        if f:
            assert f - set().union(*(per_case[:i] + per_case[i + 1:])), ("a case that brings no feature of its own", CASES[i][:5])
    assert rules == set(REFUSALS), sorted(REFUSALS[r] for r in set(REFUSALS) - rules)
    assert ("ec(8,2)", (1, 4), "default", 1, 1) in {c[:5] for c in CASES}    # the geometry smoke() runs
    for name, lost, sw in FULL_SIZE:
        assert any(c[:3] == (name, lost, sw) and c[6][0] != "refused" for c in CASES), (name, lost, sw)


def test_plan_recover_defaults_and_errors():
    """NULL switches are the build's defaults; fewer than k available parts is an error, not a plan"""
    g = goal_of("ec(8,2)")
    avail, want = [1, 0, 1, 1, 0, 1, 1, 1, 1, 1], [0, 1, 0, 0, 1, 0, 0, 0, 0, 0]
    assert L.Engine.plan_recover(g, avail, want, 1, 1) == L.Engine.plan_recover(g, avail, want, 1, 1, dict(_lib.RECOVER_SWITCHES_DEFAULT))
    p = L.Engine.plan_recover(g, [0, 0, 0, 1, 1, 1, 1, 1, 1, 1], [1, 1, 1, 0, 0, 0, 0, 0, 0, 0], 1, 1)
    assert (p["fused"], p["refusal"]) == (0, _lib.RECOVER_REFUSED_TOO_FEW_PARTS)


# ---- GPU: contexts, inputs, one call -------------------------------------------------------------------------------------------

CONTEXTS = ("switches", "cap", "generic")
_engines = {}
_scratch = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in _engines.values():
        e.close()
    _engines.clear()
    _scratch.clear()


def engine(sw, ctx):
    """one context per (switch set, kind); the switches are read when a context is created, so they are set around its creation only"""
    env = {ENV[k]: str(v) for k, v in SWITCHES[sw].items()} if ctx != "generic" else {}
    env.update({"switches": {}, "cap": {"LZGPU_GRID_CAP": "2"}, "generic": {"LZGPU_DISABLE_FUSED": "1"}}[ctx])
    key = (sw, ctx) if ctx != "generic" else ("", ctx)      # (the generic route reads none of the switches)
    if key not in _engines:
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            _engines[key] = L.Engine(0)
        finally:
            for k, v in old.items():
                if v is None:
                    del os.environ[k]
                else:
                    os.environ[k] = v
    return _engines[key]


def _case_id(case, nb):
    name, lost, sw, verify, image = case[:5]
    return f"{name}-lost{''.join(f'.{x}' for x in lost)}-{sw}-v{verify}i{image}-nb{nb}"


def _params(full_size=False, ragged_only=False):
    """(case, nb) for the `inp` fixture; the 64 MiB runs last, so that every test's list starts with the same entries and pytest
    runs the tests of one input set one after the other (the input fixture is built once per set)"""
    out = []
    for case in CASES:
        nbs = block_counts(case[0], case[1], plan_of(*case[:6]))
        out += [pytest.param((case, nb), id=_case_id(case, nb)) for nb in (nbs[:1] if ragged_only else nbs)]
    if full_size:
        out += [pytest.param((case, 1024), id=_case_id(case, 1024)) for case in CASES if case[:3] in FULL_SIZE]
    return out


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def inputs(oracle, case, nb):
    """N_CAP chunks (N at 64 MiB) of random data, the k + m parts (data parts zero-padded) with their stored CRCs on the device, the
    chunks themselves on the device, and the oracle's answer for the lost parts, which must be the original parts"""
    name, lost, _, _, _, wanted, _ = case
    g = goal_of(name)
    k, m = g.k, g.m
    n = N if nb == 1024 else N_CAP
    pb = -(-nb // k)
    rng = np.random.default_rng(zlib.crc32(repr((name, lost, nb)).encode()))
    data = rng.integers(0, 256, size=(n, nb * BLOCK), dtype=np.uint8)
    enc = [oracle.encode_chunk(g.kind, k, m, data[c]) for c in range(n)]
    per = [O.split_parts(data[c], k)[0] for c in range(n)]
    parts = [np.stack([per[c][j] for c in range(n)]) for j in range(k)] + [np.stack([enc[c][0][r] for c in range(n)]) for r in range(m)]
    crc = np.stack([enc[c][1] for c in range(n)])
    crcs = []
    for j in range(k):
        cj = np.full((n, pb), ZERO_CRC, dtype=np.uint32)
        mine = crc[:, j:nb:k]
        cj[:, : mine.shape[1]] = mine
        crcs.append(cj)
    crcs += [np.ascontiguousarray(crc[:, nb + r * pb: nb + (r + 1) * pb]) for r in range(m)]
    want = want_of(g, lost, wanted)
    for c in range(n):
        rc, out, _ = oracle.recover_chunk(g.kind, k, m, [None if i in lost else parts[i][c] for i in range(k + m)],
                                          [None if i in lost else crcs[i][c] for i in range(k + m)], want, pb)
        assert rc == 0, (name, lost, c, rc)
        for i in range(k + m):
            if want[i]:
                assert (out[i] == parts[i][c]).all(), ("oracle", name, lost, c, i)
    return dict(case=case, g=g, lost=lost, nb=nb, pb=pb, n_cap=n, crcs=crcs, d_data=dev(data),
                d_orig={i: dev(parts[i]) for i in lost},
                d_parts=[None if i in lost else dev(parts[i]) for i in range(k + m)],
                d_crcs=[None if i in lost else dev(crcs[i].view(np.int32)) for i in range(k + m)])


@pytest.fixture(scope="module")
def inp(request, oracle):
    """the inputs of one (case, nb), built once for every test that takes them (pytest groups those tests)"""
    case, nb = request.param
    return inputs(oracle, case, nb)


def mark_launch(e):
    """a one-unit CRC launch first, so that last_geometry() afterwards shows the launch of the call under test and nothing older"""
    if "blk" not in _scratch:
        _scratch["blk"] = torch.zeros(BLOCK, dtype=torch.uint8, device="cuda")
        _scratch["crc"] = torch.zeros(1, dtype=torch.int32, device="cuda")
    e.crc_blocks_dev(_scratch["blk"].data_ptr(), 1, _scratch["crc"].data_ptr())
    assert e.last_launch() == (1, 1)


def run(ctx, inp, want, verify, image, d_crcs=None):
    """recover_chunks_dev on context `ctx` over N chunks (all of them under the cap).  Every lost data part, and every wanted lost
    parity part, gets a sentinel-filled output; the image has one block of sentinel padding in its stride.  Returns the outputs
    (device tensors by part) and the image (or None)."""
    case, g, nb, pb = inp["case"], inp["g"], inp["nb"], inp["pb"]
    e = engine(case[2], ctx)
    n = inp["n_cap"] if ctx == "cap" else N
    outs = {i: torch.full((n, pb * BLOCK), SENTINEL, dtype=torch.uint8, device="cuda") for i in inp["lost"] if i < g.k or want[i]}
    img = torch.full((n, (nb + 1) * BLOCK), SENTINEL, dtype=torch.uint8, device="cuda") if image else None
    crcs = d_crcs if d_crcs is not None else inp["d_crcs"]
    torch.cuda.synchronize()
    if ctx != "generic":      # (a context without the fused kernels launches no persistent kernel at all: its record stays empty)
        mark_launch(e)
    try:
        e.recover_chunks_dev(g, n, nb, [0 if t is None else t.data_ptr() for t in inp["d_parts"]], pb * BLOCK,
                             [0 if t is None else t.data_ptr() for t in crcs] if verify else None, want,
                             [outs[i].data_ptr() if i in outs else 0 for i in range(g.k + g.m)],
                             img.data_ptr() if image else None, (nb + 1) * BLOCK)
    finally:
        check_route(ctx, inp, n, want, verify, image)
    e.sync()
    return outs, img


def check_route(ctx, inp, n, want, verify, image):
    """the call that just ran launched the planned instantiation's kernel with the planned geometry, or (generic route) none"""
    case, g = inp["case"], inp["g"]
    avail = [0 if i in inp["lost"] else 1 for i in range(g.k + g.m)]
    plan = L.Engine.plan_recover(g, avail, want, verify, image, SWITCHES[case[2]] or None)
    if (verify, image, list(want)) == (case[3], case[4], want_of(g, case[1], case[5])):
        assert literal(plan) == case[6], (case, plan)
    e = engine(case[2], ctx)
    geo = e.last_geometry()
    assert (geo["grid"], geo["units"]) == e.last_launch()
    if ctx == "generic":
        assert geo["kernel"] == _lib.KERNEL_NONE, geo
        return
    if not plan["fused"]:
        assert geo["kernel"] not in K_NAMES, geo
        return
    units = n * -(-inp["pb"] // plan["G"])
    expect = {k: plan[k] for k in ("kernel", "threads", "G", "stages", "gf_warps", "smem_bytes")}
    assert {k: geo[k] for k in expect} == expect and geo["units"] == units, (geo, expect, units)
    if ctx == "cap":
        assert geo["grid"] == 2 and geo["units"] > 2 * geo["grid"], geo
    else:
        sm = torch.cuda.get_device_properties(0).multi_processor_count
        per_sm = 2 if plan["kernel"] == _lib.KERNEL_RECOVER_GEO1 else 1
        assert geo["grid"] == min(units, per_sm * sm), (geo, sm)


def assert_outputs(inp, outs, img, want, image, what):
    """wanted lost parts (every lost data part when the image is written) equal the originals, the others keep the sentinel; the
    image equals the chunks and keeps the sentinel past nb blocks"""
    g, nb = inp["g"], inp["nb"]
    for i, t in outs.items():
        n = t.shape[0]
        if want[i] or (image and i < g.k):
            bad = (t != inp["d_orig"][i][:n]).reshape(n, -1, BLOCK).any(dim=2).nonzero().tolist()
            assert not bad, (what, "part", i, "(chunk, block) differing", bad[:4])
        else:
            assert bool((t == SENTINEL).all()), (what, "unwanted part written", i)
    if img is not None:
        n = img.shape[0]
        bad = (img[:, : nb * BLOCK] != inp["d_data"][:n]).reshape(n, nb, BLOCK).any(dim=2).nonzero().tolist()
        assert not bad, (what, "image (chunk, block) differing", bad[:4])
        assert bool((img[:, nb * BLOCK:] == SENTINEL).all()), (what, "image written past nb blocks")


# ---- GPU: every byte, three contexts ---------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("inp", _params(full_size=True), indirect=True)
def test_recover_geometry_vs_oracle_and_generic(inp):
    case, g = inp["case"], inp["g"]
    want = want_of(g, inp["lost"], case[5])
    for verify in (1, 0):
        for image in (1, 0):
            got = {}
            for ctx in CONTEXTS:
                got[ctx] = run(ctx, inp, want, verify, image)
                assert_outputs(inp, *got[ctx], want, image, (ctx, verify, image))
            for ctx in ("switches", "cap"):
                outs, img = got[ctx]
                for i, t in outs.items():
                    assert torch.equal(t[:N], got["generic"][0][i]), (ctx, verify, image, i)
                if image:
                    assert torch.equal(img[:N], got["generic"][1]), (ctx, verify, image)


@pytest.mark.gpu
@pytest.mark.parametrize("inp", _params(), indirect=True)
def test_recover_geometry_wanted_subset(inp):
    """only the last lost data part wanted: without the image the other lost data parts' outputs keep the sentinel, with it they are
    written as well (lzgpu.h: with an image every data part is wanted)"""
    g, lost = inp["g"], inp["lost"]
    data_lost = [i for i in lost if i < g.k]
    if len(data_lost) < 2:
        pytest.skip("one lost data part: no subset")
    want = [1 if i == data_lost[-1] else 0 for i in range(g.k + g.m)]
    for image in (0, 1):
        for ctx in CONTEXTS:
            outs, img = run(ctx, inp, want, 1, image)
            assert_outputs(inp, outs, img, want, image, (ctx, image))


@pytest.mark.gpu
@pytest.mark.parametrize("inp", _params(ragged_only=True), indirect=True)
def test_recover_geometry_reports_stored_crc_errors(inp):
    """one wrong stored CRC word of a part read in a slot other than 0, at the last block that part has (the ragged last unit of
    chunk 1); then a second wrong word at a smaller position (lower part, chunk 1): each call reports the smaller position, on
    every route"""
    case, g, nb, pb = inp["case"], inp["g"], inp["nb"], inp["pb"]
    used = used_parts(g, inp["lost"])
    part = used[-1] if used[-1] >= g.k else used[1]
    last = pb - 1 if part >= g.k else (nb - 1 - part) // g.k
    plan = plan_of(*case[:6])
    if plan["fused"]:
        assert last >= (-(-pb // plan["G"]) - 1) * plan["G"], (part, last, plan["G"])   # in the last unit
    other = used[0]
    other_last = pb - 1 if other >= g.k else (nb - 1 - other) // g.k
    want = want_of(g, inp["lost"], case[5])
    for words, where in (([(1, part, last)], (1, part, last)), ([(1, part, 0), (1, other, other_last)], (1, other, other_last))):
        d_crcs = list(inp["d_crcs"])
        bad = {}
        for c, p, blk in words:
            bad.setdefault(p, inp["crcs"][p].copy())[c, blk] ^= 0x00010000
        for p, words_of_part in bad.items():
            d_crcs[p] = dev(words_of_part.view(np.int32))
        for image in (1, 0):
            for ctx in CONTEXTS:
                with pytest.raises(L.ChunkCrcError) as ei:
                    run(ctx, inp, want, 1, image, d_crcs)
                assert ei.value.where == where, (ctx, image, words)
