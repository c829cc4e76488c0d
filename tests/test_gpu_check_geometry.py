"""The stripe check, map and correction (lzgpu_check_stripes, lzgpu_check_stripe_map, lzgpu_correct_stripes and their _dev forms)
at every geometry the fused check kernel (fused_check_kernel / fused_check_map_kernel, csrc/check_kernel.cuh) selects, with more map
entries than CTAs for the two grid-stride kernels after it (locate_map_kernel, correct_map_kernel), with more suspect stripes than
one correction tile of the host call, and on Cauchy goals with more than four parity parts (the generic route's passes of four rows).

check_plan() (csrc/fused_plan.h) picks the stripes per unit G from the slot count NSLOT = k + checked parity rows, the depth of the
stage ring, the instantiation (R checked rows, rows 0 .. R-1 known at compile time or not) and with G the number of passes the CTA
makes over the 32 G GF items of a step; a unit's stripe bits of pass i live in nibble i of each item thread.  A stripe check at the
wrong geometry still sees most faults, so every case asserts its launch geometry as well.  CASES holds one goal and set of given
parity parts per value of that space (test_check_geometry_table_covers_the_planner_space enumerates it on the CPU through
lzgpu_plan_check and fails when a value is missing, a case brings none of its own, or a literal plan no longer matches).

Every GPU case has three chunks of pb = 2 G + G / 2 stripes (three units per chunk, the last one partial) and nb = k pb - (k - 1)
blocks (the last stripe holds data part 0 alone).  Faults go into chunks 0 and 2 at stripes 0, G - 1, G, G + 16 and G + 32 (passes 1
and 2 of unit 1, where G allows), 2 G (the partial unit) and pb - 1 (the short stripe), into data parts (corrected through the XOR
row when parity row 0 is given, through a general row when it is not) and given parity parts; one stripe has two faulty parts, a
seeded random set of single-part faults comes on top, and chunk 1 stays clean (a fault in a parity part that is not given is not
seen).  Faults flip bytes and recompute the block's stored CRC, so only the stripe check sees them.  Each case runs the host and the
_dev entry points (the _dev buffers at a padded stride) on three contexts: the default one, LZGPU_GRID_CAP=2 (9 units on 2 CTAs) and
LZGPU_DISABLE_FUSED=1 (the generic route).  Verdicts, map and fix entries must equal the oracle's (tests/test_gpu_stripe_map.py,
tests/test_gpu_stripe_correct.py) on every context, each chunk's verdict the lowest bad entry of its map, every corrected block the
pristine one and the oracle's rs_recover, every other byte unchanged, and a re-check with the new CRCs clean except for the stripes
left UNEXPLAINED / CRC_CONFLICT."""
import os
import zlib

import numpy as np
import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import test_gpu_stripe_correct as SC
from tests.test_gpu_stripe_check import BLOCK, Batch, Dev, as_tuples
from tests.test_gpu_stripe_correct import FIX, dev_parts, expected_status, fix_list, rebuilt, verify
from tests.test_gpu_stripe_map import STATE, as_list, expected_map, invariant

PLAN_KEYS = ("rows", "consecutive", "G", "stages", "threads", "item_passes", "smem_bytes")

CASES = [
    # goal, given parity rows, literal plan: PLAN_KEYS values (R, rows 0 .. R-1, G, stages, threads, item passes, shared memory)
    ("xor2", (0,), (1, 1, 42, 3, 512, 3, 193648)),
    ("ec(2,4)", (3,), (1, 0, 42, 3, 512, 3, 193648)),
    ("ec(2,2)", (0, 1), (2, 1, 32, 3, 512, 2, 196720)),
    ("ec(2,3)", (0, 2), (2, 0, 32, 3, 512, 2, 196720)),
    ("ec(2,4)", (1, 2, 3), (3, 0, 24, 3, 512, 2, 184432)),
    ("ec(3,3)", (0, 1, 2), (3, 1, 20, 3, 512, 2, 184432)),
    ("ec(3,4)", (0, 1, 2, 3), (4, 1, 18, 3, 512, 2, 193648)),
    ("ec(5,3)", (0, 1, 2), (3, 1, 16, 3, 512, 1, 196720)),
    ("xor8", (0,), (1, 1, 14, 3, 512, 1, 193648)),
    ("ec(8,2)", (0, 1), (2, 1, 12, 3, 512, 1, 184432)),
    ("ec(9,4)", (1, 2), (2, 0, 10, 3, 512, 1, 169072)),
    ("ec(14,3)", (0, 2), (2, 0, 8, 3, 512, 1, 196720)),
    ("ec(13,4)", (0, 1, 2, 3), (4, 1, 6, 4, 512, 1, 209024)),
    ("ec(20,4)", (1, 2, 3), (3, 0, 4, 4, 512, 1, 188544)),
    ("ec(21,3)", (1,), (1, 0, 4, 4, 512, 1, 180352)),
    ("ec(32,3)", (0, 1, 2), (3, 1, 2, 5, 512, 1, 179344)),
    ("ec(31,2)", (0, 1), (2, 1, 2, 6, 512, 1, 202912)),
]
# two stored-CRC mismatches: three item passes, two, and the 4-, 5- and 6-stage rings
STORED_CRC = [("xor2", (0,)), ("ec(3,4)", (0, 1, 2, 3)), ("ec(13,4)", (0, 1, 2, 3)), ("ec(32,3)", (0, 1, 2)), ("ec(31,2)", (0, 1))]
# Cauchy generators (m >= 5, or m = 4 with k > 20) take the generic route, which checks the parity rows in passes of four
CAUCHY = [("ec(2,6)", None), ("ec(2,6)", (1, 3, 5)), ("ec(3,7)", None), ("ec(3,7)", (0, 2, 3, 4, 6)), ("ec(4,9)", None),
          ("ec(4,9)", (0, 1, 2, 3, 5, 6, 7, 8)), ("ec(32,32)", None), ("ec(32,32)", tuple(range(1, 32, 2)))]
CONTEXTS = {"default": {}, "cap": {"LZGPU_GRID_CAP": 2}, "generic": {"LZGPU_DISABLE_FUSED": 1}}
_engines = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in list(_engines.values()) + list(SC._engines.values()):
        e.close()
    _engines.clear()
    SC._engines.clear()


def engine(name):
    """one context per entry of CONTEXTS (the switches are read when a context is created)"""
    if name not in _engines:
        env = {k: str(v) for k, v in CONTEXTS[name].items()}
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            _engines[name] = L.Engine(0)
        finally:
            for k, v in old.items():
                if v is None:
                    del os.environ[k]
                else:
                    os.environ[k] = v
    return _engines[name]


def given_flags(g, rows):
    return [1] * g.k + [1 if r in rows else 0 for r in range(g.m)]


def literal(plan):
    return tuple(plan[k] for k in PLAN_KEYS)


# ---- the planner's space, on the CPU ---------------------------------------------------------------------------------------------

def planner_space():
    """{(goal, given parity rows): plan} for every Vandermonde goal (xor2..9, ec(k,m) with k = 2..32, m = 1..4) and every non-empty set
    of given parity parts"""
    out = {}
    goals = [f"xor{k}" for k in range(2, 10)] + [f"ec({k},{m})" for k in range(2, 33) for m in range(1, 5)]
    for name in goals:
        g = L.SliceType(name)
        if g.m >= 5 or (g.m == 4 and g.k > 20):
            continue
        for mask in range(1, 1 << g.m):
            rows = tuple(r for r in range(g.m) if mask >> r & 1)
            out[(name, rows)] = L.Engine.plan_check(g, given_flags(g, rows))
    return out


def features(p):
    """the values of the space a plan has: G, stages, item passes, the instantiation (R, rows 0 .. R-1), and the instantiation at one
    pass and at two or more"""
    inst = (p["rows"], p["consecutive"])
    return {("G", p["G"]), ("stages", p["stages"]), ("item passes", p["item_passes"]), ("instantiation",) + inst,
            ("instantiation",) + inst + ("1 pass" if p["item_passes"] == 1 else ">= 2 passes",)}


def test_check_geometry_table_covers_the_planner_space():
    """every value of the planner's space occurs in CASES, each case brings one that no other case has, and every literal plan of
    CASES is the planner's; every plan of the space keeps what the planner's comments state"""
    space = planner_space()
    feats = set()
    for (name, rows), p in space.items():
        g = L.SliceType(name)
        nslot = g.k + len(rows)
        what = (name, rows, p)
        assert p["fused"] == 1 and p["rows"] == len(rows) and p["consecutive"] == (rows == tuple(range(len(rows)))), what
        assert p["G"] % 2 == 0 and nslot * p["G"] * 4 <= 512 and p["G"] * 4 <= 256 and p["threads"] == 512, what
        assert nslot * (p["G"] + 2) * 4 > 512 or 3 * nslot * (p["G"] + 2) * 4 * 128 + 256 > 208 * 1024, what   # the largest G
        assert 3 <= p["stages"] <= 6 and p["item_passes"] == -(-32 * p["G"] // 512), what
        assert p["smem_bytes"] == p["stages"] * nslot * p["G"] * 4 * 128 + 16 * p["stages"] + 64 <= 208 * 1024, what
        assert p["stages"] == 6 or (p["stages"] + 1) * nslot * p["G"] * 4 * 128 > 208 * 1024 - 256, what
        feats |= features(p)
    assert {f[1] for f in feats if f[0] == "G"} == {2, 4, 6, 8, 10, 12, 14, 16, 18, 20, 24, 32, 42}
    assert {f[1] for f in feats if f[0] == "stages"} == {3, 4, 5, 6}
    assert {f[1] for f in feats if f[0] == "item passes"} == {1, 2, 3}
    per_case = []
    for name, rows, want in CASES:
        assert (name, rows) in space, (name, rows)
        p = L.Engine.plan_check(L.SliceType(name), given_flags(L.SliceType(name), rows))
        assert literal(p) == want, (name, rows, literal(p))
        assert p == space[(name, rows)]
        per_case.append(features(p))
    table = set().union(*per_case)
    assert not feats - table, sorted(feats - table, key=str)
    for i, f in enumerate(per_case):
        assert f - set().union(*(per_case[:i] + per_case[i + 1:])), ("a case that brings no value of its own", CASES[i][:2])


def test_plan_check_cauchy_and_errors():
    """a Cauchy generator takes the generic route (the checked rows still reported); a missing data part, or no parity part, is the
    calls' error"""
    for name, rows in (("ec(2,6)", (0, 1, 2, 3, 4, 5)), ("ec(22,4)", (1, 3)), ("ec(32,32)", tuple(range(32)))):
        g = L.SliceType(name)
        p = L.Engine.plan_check(g, given_flags(g, rows))
        assert (p["fused"], p["rows"], p["G"], p["stages"], p["smem_bytes"]) == (0, len(rows), 0, 0, 0), (name, p)
    g = L.SliceType("ec(5,3)")
    for flags in ([0, 1, 1, 1, 1, 1, 1, 1], [1, 1, 1, 1, 1, 0, 0, 0]):
        with pytest.raises(L.LzGpuError) as ei:
            L.Engine.plan_check(g, flags)
        assert ei.value.status == _lib.ERR_TOO_FEW_PARTS


# ---- GPU: inputs, faults, one case on every entry point and context ---------------------------------------------------------------

_batches = {}


def batch(oracle, text, n, nb, seed=1, cache=True):
    """a fresh copy of a cached batch (parts and stored CRCs); cache=False: the batch itself, nothing kept"""
    key = (text, n, nb, seed)
    if key not in _batches:
        _batches.clear()                                 # one batch at a time: keeps the host memory of a case small
        if not cache:
            return Batch(oracle, text, n, nb, seed)
        _batches[key] = Batch(oracle, text, n, nb, seed)
    b = _batches[key]
    fresh = Batch.__new__(Batch)
    fresh.__dict__.update(b.__dict__)
    fresh.parts = [p.copy() for p in b.parts]
    fresh.crc = [c.copy() for c in b.crc]
    fresh.faulty = set()
    return fresh


def shape_of(g, G):
    pb = 2 * G + G // 2
    return pb, g.k * pb - (g.k - 1)


def inject(b, rows, G, seed):
    """the targeted faults, one two-part stripe and seeded random single-part faults in chunks 0 and 2; returns the faults"""
    k, pb = b.k, b.pb
    par = [k + r for r in rows]
    suspects = [0, par[0], k - 1, par[-1], k // 2]
    targets = [0, G - 1, G] + [G + 16] * (G > 16) + [G + 32] * (G > 32) + [2 * G, pb - 1]
    faults = []
    for c in (0, 2):
        for i, s in enumerate(sorted(set(targets))):
            p = suspects[(i + c) % len(suspects)]
            if s == pb - 1 and p in range(1, k):
                p = 0                                    # the short stripe: data part 0 alone has a block there
            faults.append((c, p, s))
    rng = np.random.default_rng(seed)
    used = {(c, s) for c, _, s in faults} | {(0, G + 1)}
    free = [(c, s) for c in (0, 2) for s in range(pb) if (c, s) not in used]
    for i in rng.permutation(len(free))[:4]:
        c, s = free[i]
        faults.append((c, int(rng.choice([0] + par if s == pb - 1 else list(range(k)) + par)), s))
    for c, p, s in faults:
        b.corrupt(c, p, s, offset=(977 * s + 131 * p + 7 * c) % 65000)
    b.corrupt(0, 0, G + 1, offset=100)                   # two faulty parts at different bytes: no single part explains the stripe
    b.corrupt(0, k + rows[-1] if len(rows) > 1 else 1 % k, G + 1, offset=30000)
    if len(rows) < b.m:                                  # a fault in a parity part that is not given is not seen
        b.corrupt(1, k + next(r for r in range(b.m) if r not in rows), 1)
    return faults


def host_call(fn, attr, where):
    """a host entry point; on a stored-CRC error its result (attribute attr of the error), the error's place appended to where"""
    try:
        return fn()
    except L.ChunkCrcError as e:
        where.append(e.where)
        return getattr(e, attr)


def dev_call(eng, call, b, dev, given, dtype, shape):
    """a _dev entry point into a guarded result buffer; returns (result, where of a stored-CRC error or None) and asserts that nothing
    outside the result changed"""
    import torch
    guard, size = 4096, dtype.itemsize * int(np.prod(shape))
    init = np.random.default_rng(3).integers(0, 256, 2 * guard + size, dtype=np.uint8)
    t = torch.from_numpy(init.copy()).cuda()
    ptrs = [p if i in given else None for i, p in enumerate(dev.ptrs)]
    crcs = [c if i in given else None for i, c in enumerate(dev.crcs)]
    where = None
    try:
        getattr(eng, call)(b.goal, b.n, b.nb, ptrs, dev.stride, crcs, t.data_ptr() + guard)
    except L.ChunkCrcError as e:
        where = e.where
    torch.cuda.synchronize()
    out = t.cpu().numpy()
    assert (out[:guard] == init[:guard]).all() and (out[guard + size:] == init[guard + size:]).all(), f"{call}: write outside the result"
    return out[guard:guard + size].copy().view(dtype).reshape(shape), where


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def expected_geometry(ctx, plan, b):
    """lzgpu_debug_last_geometry after a call of the case on context ctx: its plan's launch, or (generic route) None: no launch of
    the check kernel (the generic route's stored-CRC pass may launch the fused CRC kernel)"""
    if ctx == "generic" or not plan["fused"]:
        return None
    units = b.n * -(-b.pb // plan["G"])
    grid = min(units, sm_count(), 2 if ctx == "cap" else units)
    return {"kernel": _lib.KERNEL_CHECK, "grid": grid, "units": units, "threads": plan["threads"], "G": plan["G"],
            "stages": plan["stages"], "gf_warps": 0, "smem_bytes": plan["smem_bytes"]}


def geometry_after(eng, ctx, plan, b, call):
    before = eng.last_geometry()
    out = call()
    want, got = expected_geometry(ctx, plan, b), eng.last_geometry()
    if want is None:
        assert got["kernel"] != _lib.KERNEL_CHECK or got == before, (ctx, got)
    else:
        assert got == want, (ctx, got, want)
    return out


def run_everywhere(oracle, b, pristine, rows, plan, crcs, dev_pad=65536 + 48):
    """check, map and correction of batch b (given: data parts and parity rows `rows`), host and _dev, on every context; every
    assertion of the module docstring.  Returns {context: (verdicts, map, host fix, dev fix, where)} after asserting they agree."""
    given = set(range(b.k)) | {b.k + r for r in rows}
    parts = [b.parts[i] if i in given else None for i in range(b.k + b.m)]
    want_map = as_list(expected_map(oracle, b, list(rows)))
    results = {}
    ref = []                                             # (fix, parts after) of the first correction, checked by verify()

    def corrected(fix, after):
        """the first correction against the oracle (verify), every later one byte for byte against the first"""
        if not ref:
            verify(oracle, b, crcs, given, fix, after, list(rows), pristine=pristine.parts)
            ref.extend([fix_list(fix), after])
        else:
            assert fix_list(fix) == ref[0] and all((x == y).all() for x, y in zip(after, ref[1])), "a correction differs from the first"
    for ctx in CONTEXTS:
        eng = engine(ctx)
        where = []
        v = geometry_after(eng, ctx, plan, b, lambda: host_call(lambda: eng.check_stripes(b.goal, b.nb, parts, crcs), "verdict", where))
        m = geometry_after(eng, ctx, plan, b, lambda: host_call(lambda: eng.check_stripe_map(b.goal, b.nb, parts, crcs), "map", where))
        assert as_list(m) == want_map, ctx
        invariant(m, v)
        after = [p.copy() for p in b.parts]
        fix = geometry_after(eng, ctx, plan, b, lambda: host_call(lambda: eng.correct_stripes(
            b.goal, b.nb, [after[i] if i in given else None for i in range(b.k + b.m)], crcs), "fix", where))
        corrected(fix, after)
        del after
        # the _dev forms on the batch resident at a padded stride (a fresh upload: the correction writes into it)
        dev = Dev(b, dev_pad, 16)
        if crcs is not b.crc:
            for i, c in enumerate(crcs):
                dev.bufs[2 * i + 1].copy_(dev.torch.from_numpy(c.view(np.int32).copy()))
        dv, w1 = geometry_after(eng, ctx, plan, b, lambda: dev_call(eng, "check_stripes_dev", b, dev, given, L.Engine.VERDICT_DTYPE, (b.n,)))
        dm, w2 = geometry_after(eng, ctx, plan, b, lambda: dev_call(eng, "check_stripe_map_dev", b, dev, given, STATE, (b.n, b.pb)))
        assert as_tuples(dv) == as_tuples(v) and as_list(dm) == want_map, ctx
        dfix, w3 = geometry_after(eng, ctx, plan, b, lambda: dev_call(eng, "correct_stripes_dev", b, dev, given, FIX, (b.n, b.pb)))
        dafter, bufs = dev_parts(b, dev, 16)
        corrected(dfix, dafter)
        for i in range(b.k + b.m):                       # the stride gaps and the bytes past the last chunk
            outside = np.ones(len(bufs[i]), dtype=bool)
            for c in range(b.n):
                outside[16 + c * dev.stride: 16 + c * dev.stride + b.pb * BLOCK] = False
            host_init = np.random.default_rng(7).integers(0, 256, len(bufs[i]), dtype=np.uint8)
            assert (bufs[i][outside] == host_init[outside]).all(), (ctx, i)
        del dev, dafter, bufs
        assert w1 == w2 == w3 and [w1] * 3 == (where or [None] * 3), (ctx, where, w1, w2, w3)
        assert eng.status_slots()[1] == 0
        results[ctx] = (as_tuples(v), as_list(m), fix_list(fix), fix_list(dfix), w1)
    first = results["default"]
    for ctx, r in results.items():
        assert r[:3] == first[:3] and r[3] == first[2] and r[4] == first[4], f"{ctx} and the default context disagree"
    return results


gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("case", range(len(CASES)), ids=[f"{c[0]}-rows{''.join(map(str, c[1]))}" for c in CASES])
def test_geometry_case(oracle, case):
    name, rows, want = CASES[case]
    g = L.SliceType(name)
    plan = L.Engine.plan_check(g, given_flags(g, rows))
    assert literal(plan) == want
    pb, nb = shape_of(g, plan["G"])
    pristine = batch(oracle, name, 3, nb)
    b = batch(oracle, name, 3, nb)
    faults = inject(b, rows, plan["G"], seed=case)
    res = run_everywhere(oracle, b, pristine, rows, plan, b.crc)["default"]
    verdicts, smap, fix = res[0], res[1], res[2]
    assert verdicts[1] == (-1, 0, -1) and not any(e[0] for e in smap[1])                 # the clean chunk
    status = {(c, s): e[2] for c, row in enumerate(fix) for s, e in enumerate(row)}
    multi = len(rows) >= 2
    for c, p, s in faults:
        assert smap[c][s][0] != 0 and status[(c, s)] == (_lib.FIX_CORRECTED if multi else _lib.FIX_UNEXPLAINED), (c, p, s)
        if multi:
            assert smap[c][s][1] == p, (c, p, s)
    assert status[(0, plan["G"] + 1)] == _lib.FIX_UNEXPLAINED


@gpu
@pytest.mark.parametrize("name,rows", STORED_CRC, ids=[f"{n}-rows{''.join(map(str, r))}" for n, r in STORED_CRC])
def test_stored_crc_mismatches_report_the_smaller_part(oracle, name, rows):
    """two stored-CRC mismatches in chunk 0: a parity part in unit 0 and data part 0 in unit 1.  (chunk, part, block) of the smaller
    part is reported on every context and entry point, and the verdicts, the map and the fix entries are written in full"""
    case = [c[:2] for c in CASES].index((name, rows))
    g = L.SliceType(name)
    plan = L.Engine.plan_check(g, given_flags(g, rows))
    G = plan["G"]
    pb, nb = shape_of(g, G)
    pristine = batch(oracle, name, 3, nb)
    b = batch(oracle, name, 3, nb)
    inject(b, rows, G, seed=100 + case)
    crcs = [c.copy() for c in b.crc]
    crcs[b.k + rows[-1]][0, 1] ^= 0x40                   # unit 0, the largest given part
    crcs[0][0, G + 1] ^= 0x40                            # unit 1, part 0
    res = run_everywhere(oracle, b, pristine, rows, plan, crcs)
    assert all(r[4] == (0, 0, G + 1) for r in res.values())


@gpu
@pytest.mark.parametrize("name,rows", CAUCHY, ids=[f"{n}-{'all' if r is None else 'rows' + '.'.join(map(str, r))}" for n, r in CAUCHY])
def test_cauchy_goals_on_the_generic_route(oracle, name, rows):
    """passes of four parity rows (ec(2,6): 4 + 2, ec(3,7): 4 + 3, ec(4,9): 4 + 4 + 1, ec(32,32): eight), bad_rows up to bit 31,
    suspects up to part 63 and the 64-part given mask of the correction; and a subset of the parity parts"""
    g = L.SliceType(name)
    k, m = g.k, g.m
    rows = tuple(range(m)) if rows is None else rows
    plan = L.Engine.plan_check(g, given_flags(g, rows))
    assert plan["fused"] == 0 and plan["rows"] == len(rows)
    nb = 2 * k + 1                                       # three stripes, the last one data part 0 alone
    pristine = batch(oracle, name, 3, nb)
    b = batch(oracle, name, 3, nb)
    last, fifth = k + rows[-1], k + rows[min(4, len(rows) - 1)]
    faults = [(0, k - 1, 1), (0, last, 0), (0, 0, 2), (2, fifth, 1), (2, k + rows[0], 2)]
    for c, p, s in faults:
        b.corrupt(c, p, s, offset=1000 * s + 17 * p)
    b.corrupt(2, 0, 0, offset=100)                       # two faulty parts: no single suspect
    b.corrupt(2, last, 0, offset=40000)
    res = run_everywhere(oracle, b, pristine, rows, plan, b.crc)["default"]
    smap, fix = res[1], res[2]
    all_rows = sum(1 << r for r in rows)
    assert smap[0][1] == (all_rows, k - 1) and smap[0][0] == (1 << rows[-1], last) and smap[0][2] == (all_rows, 0)
    assert smap[2][1] == (1 << (fifth - k), fifth) and smap[2][0][1] == -1
    assert [fix[c][s][2] for c, _, s in faults] == [_lib.FIX_CORRECTED] * len(faults) and fix[2][0][2] == _lib.FIX_UNEXPLAINED
    if m == 32 and len(rows) == 32:
        assert smap[0][1][0] == 0xFFFFFFFF and smap[0][0] == (1 << 31, 63)


# ---- more entries than CTAs ------------------------------------------------------------------------------------------------------

@gpu
def test_more_map_and_fix_entries_than_ctas(oracle):
    """ec(2,2), full 64 MiB chunks.  correct_map_kernel runs at most 2 x SMs CTAs, locate_map_kernel at most 8 x SMs, each stepping
    over the entries by its grid.  The entries e, e + grid, e + 2 grid, e + 3 grid, e + 4 grid of every correction CTA hold, in this
    order, a data part 0 fault (corrected through the XOR row: parity row 0 is given), a clean stripe, two faulty parts (UNEXPLAINED),
    a parity row 1 fault (corrected through a general row) and a data part 1 fault next to a failing stored CRC of parity part 0
    (CRC_CONFLICT).  8 x SMs = 4 x (2 x SMs), so every locate CTA names the suspects of two bad stripes, e and e + 4 grid, which blame
    different parts.  Map and fix entries and every byte against the oracle, on the fused and the generic route."""
    import torch
    sms = sm_count()
    grid = 2 * sms
    k, nb, pb = 2, 1024, 512
    n = -(-max(5 * grid, 8 * sms + 1) // pb)
    b = batch(oracle, "ec(2,2)", n, nb, seed=9, cache=False)
    original = {}
    faults = {0: [(0, 0)], 2: [(0, 100), (1, 30000)], 3: [(3, 0)], 4: [(1, 0)]}   # kind -> (part, offset) of its faults
    kinds = []
    for e in range(n * pb):
        c, s = divmod(e, pb)
        kind = e // grid if e < 5 * grid else 1
        kinds.append(kind)
        for p, offset in faults.get(kind, []):
            original[(c, p, s)] = b.parts[p][c, s * BLOCK:(s + 1) * BLOCK].copy()
            b.corrupt(c, p, s, offset=offset + e % 30000)
    crcs = [x.copy() for x in b.crc]
    for e in range(4 * grid, 5 * grid):
        crcs[2][e // pb, e % pb] ^= 0x40
    assert n * pb > 8 * sms and n * pb >= 5 * grid
    want_map = expected_map(oracle, b, [0, 1])
    given = set(range(4))
    want_status = expected_status(want_map, b.parts, crcs, given)
    status_of = {0: _lib.FIX_CORRECTED, 1: _lib.FIX_CLEAN, 2: _lib.FIX_UNEXPLAINED, 3: _lib.FIX_CORRECTED, 4: _lib.FIX_CRC_CONFLICT}
    suspect_of = {0: 0, 1: -1, 2: -1, 3: 3, 4: 1}
    assert [int(x) for x in want_status.reshape(-1)] == [status_of[x] for x in kinds]
    assert [int(x) for x in want_map["suspect_part"].reshape(-1)] == [suspect_of[x] for x in kinds]
    corrected = {}
    for e, kind in enumerate(kinds):
        if kind in (0, 3):
            c, s = divmod(e, pb)
            p = suspect_of[kind]
            blk = rebuilt(oracle, b, b.parts, c, s, p, given)
            assert (blk == original[(c, p, s)]).all(), (c, s, p)
            corrected[(c, p, s)] = blk
    first_mismatch = (4 * grid // pb, 2, 4 * grid % pb)
    fixes = []
    for ctx in ("default", "generic"):
        eng = engine(ctx)
        dev = Dev(b, 16, 0)
        for i, x in enumerate(crcs):
            dev.bufs[2 * i + 1].copy_(torch.from_numpy(x.view(np.int32).copy()))
        m, where = dev_call(eng, "check_stripe_map_dev", b, dev, given, STATE, (n, pb))
        assert where == first_mismatch and as_list(m) == as_list(want_map), ctx
        if ctx == "default":
            assert eng.last_geometry()["kernel"] == _lib.KERNEL_CHECK
        fix, where = dev_call(eng, "correct_stripes_dev", b, dev, given, FIX, (n, pb))
        assert where == first_mismatch, ctx
        assert as_list(fix[["bad_rows", "suspect_part"]]) == as_list(want_map) and (fix["status"] == want_status).all(), ctx
        for (c, p, s), blk in corrected.items():
            assert int(fix[c, s]["crc"]) == zlib.crc32(blk.tobytes()), (ctx, c, s)
        assert (fix["crc"][fix["status"] != _lib.FIX_CORRECTED] == 0).all()
        for i in range(4):                               # part by part: every byte, the corrected blocks restored
            got = dev.bufs[2 * i].cpu().numpy()
            for c in range(n):
                want = b.parts[i][c].copy()
                for (cc, p, s), blk in corrected.items():
                    if cc == c and p == i:
                        want[s * BLOCK:(s + 1) * BLOCK] = blk
                assert (got[c * dev.stride: c * dev.stride + pb * BLOCK] == want).all(), (ctx, i, c)
            del got
        del dev
        torch.cuda.empty_cache()
        assert eng.status_slots()[1] == 0
        fixes.append(fix_list(fix))
    assert fixes[0] == fixes[1]


@gpu
def test_host_correction_takes_several_tiles(oracle):
    """ec(8,2), four chunks of 103 stripes, one faulty part in every stripe: 412 suspect stripes are more than one correction tile of
    2 x 128 MiB / (64 KiB x 10 given parts) = 409 stripes.  The batches_timed delta counts the check tiles and the correction tiles;
    every block is restored, on the fused and the generic route"""
    k, m, n, pb = 8, 2, 4, 103
    nb = k * pb
    tile_bytes = 2 * 128 << 20
    check_tiles = -(-n // max(1, tile_bytes // (pb * BLOCK * (k + m))))
    fix_tile = tile_bytes // (BLOCK * (k + m))
    assert n * pb > fix_tile
    b = batch(oracle, "ec(8,2)", n, nb, seed=4, cache=False)
    rng = np.random.default_rng(4)
    original = {}
    for c in range(n):
        for s in range(pb):
            p = int(rng.integers(0, k + m))
            original[(c, p, s)] = (b.parts[p][c, s * BLOCK:(s + 1) * BLOCK].copy(), int(b.crc[p][c, s]))
            b.corrupt(c, p, s, offset=int(rng.integers(0, 65000)))
    want_map = expected_map(oracle, b, [0, 1])
    assert [int(x) for x in want_map["suspect_part"].reshape(-1)] == [p for (c, p, s) in original]
    fixes = []
    for ctx in ("default", "generic"):
        eng = engine(ctx)
        after = [p.copy() for p in b.parts]
        before = eng.stats()["batches_timed"]
        fix = eng.correct_stripes(b.goal, nb, after, b.crc)
        assert eng.stats()["batches_timed"] - before == check_tiles + -(-n * pb // fix_tile), ctx
        assert as_list(fix[["bad_rows", "suspect_part"]]) == as_list(want_map), ctx
        assert (fix["status"] == _lib.FIX_CORRECTED).all(), ctx
        for (c, p, s), (blk, crc) in original.items():
            assert int(fix[c, s]["crc"]) == crc and (after[p][c, s * BLOCK:(s + 1) * BLOCK] == blk).all(), (ctx, c, p, s)
            after[p][c, s * BLOCK:(s + 1) * BLOCK] = b.parts[p][c, s * BLOCK:(s + 1) * BLOCK]
        assert all((x == y).all() for x, y in zip(after, b.parts)), ctx
        del after
        assert eng.status_slots()[1] == 0
        fixes.append(fix_list(fix))
    assert fixes[0] == fixes[1]
