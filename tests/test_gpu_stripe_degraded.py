"""The stripe map and correction of chunks that have lost parts (lzgpu_check_stripe_map_degraded, lzgpu_correct_stripes_degraded and
their _dev forms), and their planner (lzgpu_plan_check_degraded).

The inputs are the first k given parts, the spares the given parts after them (always parity parts).  The expected map comes from the
oracle: rs_recover rebuilds the spares from the inputs, bad_rows bit r is set where spare part k + r differs from its rebuild, and the
suspect is a numpy column test over [M | I], M the spares' recovery rows over the inputs (read off rs_recover of unit inputs).  With
every data part given, both calls must return what lzgpu_check_stripe_map / lzgpu_correct_stripes return.  Every GPU case runs on a
fused context and on LZGPU_DISABLE_FUSED=1 (the generic route), which must agree exactly.  Faults flip bytes and recompute the
block's stored CRC, so only the stripe check sees them."""
import ctypes
import os
import zlib

import numpy as np
import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200 import engine as E
from tests import test_gpu_stripe_map as SM
from tests.test_gpu_stripe_check import BLOCK, Batch, Dev
from tests.test_gpu_stripe_correct import FIX, block, dev_parts, expected_status, fix_list, rebuilt
from tests.test_gpu_stripe_map import STATE, as_list, gf_mul_table

PLAN_KEYS = ("fused", "rows", "consecutive", "G", "stages", "threads", "item_passes", "smem_bytes")
_engines = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in list(_engines.values()) + list(SM._engines.values()):
        e.close()
    _engines.clear()
    SM._engines.clear()


def engine(**env):
    """one context per set of switches (read when a context is created)"""
    env = {k: str(v) for k, v in env.items()}
    key = tuple(sorted(env.items()))
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


ROUTES = {"fused": {}, "generic": {"LZGPU_DISABLE_FUSED": 1}}


def is_cauchy(g):
    return g.m >= 5 or (g.m == 4 and g.k > 20)


def flags(g, lost):
    return [0 if i in lost else 1 for i in range(g.k + g.m)]


def literal(p):
    return tuple(p[k] for k in PLAN_KEYS)


# ---- the planner, on the CPU -----------------------------------------------------------------------------------------------------

VANDERMONDE = [f"xor{k}" for k in range(2, 10)] + [f"ec({k},{m})" for k in range(2, 33) for m in range(1, 5)
                                                    if not (m == 4 and k > 20)]


def degraded_space():
    """{(goal, lost data count, given parity rows): plan} for every Vandermonde goal, 1 .. 3 lost data parts and every set of given
    parity parts with a spare.  The plan depends on how many data parts are lost, not on which: the first and the last E are asked."""
    out = {}
    for name in VANDERMONDE:
        g = L.SliceType(name)
        for e in range(1, min(3, g.m - 1, g.k) + 1):
            for mask in range(1, 1 << g.m):
                rows = tuple(r for r in range(g.m) if mask >> r & 1)
                if len(rows) <= e:
                    continue
                lost_rows = {g.k + r for r in range(g.m) if r not in rows}
                first = L.Engine.plan_check_degraded(g, flags(g, set(range(e)) | lost_rows))
                last = L.Engine.plan_check_degraded(g, flags(g, set(range(g.k - e, g.k)) | lost_rows))
                assert first == last, (name, e, rows)
                out[(name, e, rows)] = first
    return out


# (goal, lost data parts, given parity rows, literal plan): every instantiation (E, R, rows 0 .. R-1) and every G and stage count
# the planner reaches with a lost data part
CASES = [
    ("ec(2,2)", (0,), (0, 1), (1, 2, 1, 42, 3, 512, 3, 193648)),
    ("ec(14,4)", (1,), (0, 1, 2, 3), (1, 4, 1, 6, 4, 512, 1, 209024)),
    ("ec(31,3)", (1,), (0, 1, 2), (1, 3, 1, 2, 6, 512, 1, 202912)),
    ("ec(2,4)", (0,), (0, 1, 3), (1, 3, 0, 32, 3, 512, 2, 196720)),
    ("ec(3,4)", (0, 1), (0, 1, 2, 3), (1, 4, 1, 24, 3, 512, 2, 184432)),
    ("ec(5,3)", (1,), (0, 2), (1, 2, 0, 20, 3, 512, 2, 184432)),
    ("ec(6,3)", (1, 2), (0, 1, 2), (1, 3, 1, 18, 3, 512, 2, 193648)),
    ("ec(7,4)", (1, 2), (0, 1, 3), (1, 3, 0, 16, 3, 512, 1, 196720)),
    ("ec(8,4)", (1, 2, 3), (0, 1, 2, 3), (1, 4, 1, 14, 3, 512, 1, 193648)),
    ("ec(7,4)", (1,), (0, 1, 2, 3), (1, 4, 1, 12, 3, 512, 1, 184432)),
    ("ec(8,4)", (1,), (0, 1, 2, 3), (1, 4, 1, 10, 3, 512, 1, 169072)),
    ("ec(10,4)", (1,), (0, 1, 2, 3), (1, 4, 1, 8, 3, 512, 1, 159856)),
    ("ec(19,4)", (1,), (0, 1, 2, 3), (1, 4, 1, 4, 4, 512, 1, 180352)),
]


def case_features(e, p):
    return {("instantiation", e, p["rows"], p["consecutive"]), ("G", p["G"]), ("stages", p["stages"])}


def test_degraded_plan_table_covers_the_planner_space():
    space = degraded_space()
    feats = set()
    for (name, e, rows), p in space.items():
        g = L.SliceType(name)
        nslot = g.k - e + len(rows)
        what = (name, e, rows, p)
        assert p["fused"] == 1 and p["rows"] == len(rows) and p["consecutive"] == (rows == tuple(range(len(rows)))), what
        assert p["G"] % 2 == 0 and nslot * p["G"] * 4 <= 512 and p["G"] * 4 <= 256 and p["threads"] == 512, what
        assert nslot * (p["G"] + 2) * 4 > 512 or 3 * nslot * (p["G"] + 2) * 4 * 128 + 256 > 208 * 1024, what
        assert p["smem_bytes"] == p["stages"] * nslot * p["G"] * 4 * 128 + 16 * p["stages"] + 64 <= 208 * 1024, what
        feats |= case_features(e, p)
    insts = {f[1:] for f in feats if f[0] == "instantiation"}
    assert insts == {(1, 2, 1), (1, 3, 1), (1, 4, 1), (2, 3, 1), (2, 4, 1), (3, 4, 1), (1, 2, 0), (1, 3, 0), (2, 3, 0)}, insts
    table = set()
    for name, lost, rows, want in CASES:
        g = L.SliceType(name)
        e = len(lost)
        p = L.Engine.plan_check_degraded(g, flags(g, set(lost) | {g.k + r for r in range(g.m) if r not in rows}))
        assert literal(p) == want, (name, lost, rows, literal(p))
        assert p == space[(name, e, rows)]
        table |= case_features(e, p)
    assert not feats - table, sorted(feats - table, key=str)


def test_degraded_plan_equals_plan_check_with_every_data_part():
    for name in VANDERMONDE + ["ec(22,4)", "ec(10,5)", "ec(2,6)"]:
        g = L.SliceType(name)
        for mask in range(1, min(1 << g.m, 64)):
            f = [1] * g.k + [mask >> r & 1 for r in range(g.m)]
            assert L.Engine.plan_check_degraded(g, f) == L.Engine.plan_check(g, f), (name, mask)


def test_degraded_plan_refusals_and_generic_route():
    for name, lost in (("ec(5,3)", (1, 2, 3)), ("ec(5,3)", (5, 6, 7)), ("ec(8,2)", (0, 8)), ("ec(3,2)", (0, 1))):
        g = L.SliceType(name)
        with pytest.raises(L.LzGpuError) as ei:
            L.Engine.plan_check_degraded(g, flags(g, set(lost)))
        assert ei.value.status == _lib.ERR_TOO_FEW_PARTS, (name, lost)
    for name, lost in (("ec(22,4)", (1,)), ("ec(22,4)", (0, 5, 23)), ("ec(10,5)", (3,)), ("ec(10,5)", (0, 1, 2, 3))):
        g = L.SliceType(name)
        p = L.Engine.plan_check_degraded(g, flags(g, set(lost)))
        assert p["fused"] == 0 and p["G"] == 0 and p["rows"] == sum(1 for r in range(g.m) if g.k + r not in lost), (name, p)


# ---- the expected map, on the CPU ------------------------------------------------------------------------------------------------

def roles(b, given):
    """(inputs, spares): the first k given parts and the given parts after them"""
    g = sorted(given)
    return g[:b.k], g[b.k:]


def recovery_rows(oracle, b, given):
    """M[i][j]: the coefficient of input j in spare i's rebuild from the inputs"""
    inputs, spares = roles(b, given)
    n = b.k + b.m
    ins = [None] * n
    for j, p in enumerate(inputs):
        ins[p] = np.zeros(b.k, dtype=np.uint8)
        ins[p][j] = 1
    erased = [0 if i in inputs else 1 for i in range(n)]
    out = oracle.rs_recover(b.k, b.m, ins, erased, [int(i in spares) for i in range(n)], b.k)
    return np.stack([out[s] for s in spares])


def suspect_of(oracle, b, given, M, syn):
    """syn [spares, 65536]: the one given part whose column of [M | I] explains every syndrome byte, else -1"""
    inputs, spares = roles(b, given)
    if len(spares) < 2:
        return -1
    mul = gf_mul_table(oracle)
    fits = []
    for j, p in enumerate(inputs):
        col = M[:, j]
        if col.any() and all((mul[syn[i], col[l]] == mul[syn[l], col[i]]).all()
                             for i in range(len(spares)) for l in range(i + 1, len(spares))) \
                and all(not syn[i].any() for i in range(len(spares)) if col[i] == 0):
            fits.append(p)
    for i, p in enumerate(spares):
        if not np.delete(syn, i, axis=0).any():
            fits.append(p)
    return fits[0] if len(fits) == 1 else -1


def expected_map(oracle, b, given, parts=None):
    parts = b.parts if parts is None else parts
    inputs, spares = roles(b, given)
    n = b.k + b.m
    M = recovery_rows(oracle, b, given)
    out = np.zeros((b.n, b.pb), dtype=STATE)
    out["suspect_part"] = -1
    erased = [0 if i in inputs else 1 for i in range(n)]
    for c in range(b.n):
        ins = [np.ascontiguousarray(parts[i][c]) if i in inputs else None for i in range(n)]
        rec = oracle.rs_recover(b.k, b.m, ins, erased, [int(i in spares) for i in range(n)], b.pb * BLOCK)
        syn = np.stack([(rec[s] ^ parts[s][c]).reshape(b.pb, BLOCK) for s in spares], axis=1)   # [pb, spares, B]
        for s in range(b.pb):
            bits = sum(1 << (p - b.k) for i, p in enumerate(spares) if syn[s, i].any())
            if bits:
                out[c, s] = (bits, suspect_of(oracle, b, given, M, syn[s]))
    return out


# ---- GPU runs --------------------------------------------------------------------------------------------------------------------

def host_result(fn, attr):
    try:
        return fn(), None
    except L.ChunkCrcError as e:
        return getattr(e, attr), e.where


def expect_kernel(eng_env, b, given):
    lost_data = any(j not in given for j in range(b.k))
    plan = L.Engine.plan_check_degraded(b.goal, [int(i in given) for i in range(b.k + b.m)])
    if eng_env.get("LZGPU_DISABLE_FUSED") or not plan["fused"]:
        return None, plan
    return (_lib.KERNEL_CHECK_DEGRADED if lost_data else _lib.KERNEL_CHECK), plan


def run_routes(oracle, b, given, crcs=None, want_map=None, contexts=ROUTES, pristine=None):
    """map and correction (host forms) of batch b with the parts `given`, on every context; each against the oracle, the routes
    against each other.  Returns (map, fix, parts after, where) of the first context."""
    crcs = b.crc if crcs is None else crcs
    n = b.k + b.m
    gcrcs = [crcs[i] if i in given else None for i in range(n)]
    want_map = expected_map(oracle, b, given) if want_map is None else want_map
    first = None
    for name, env in contexts.items():
        eng = engine(**env)
        kernel, plan = expect_kernel(env, b, given)
        before = eng.last_geometry()
        m, where = host_result(lambda: eng.check_stripe_map_degraded(b.goal, b.nb, [b.parts[i] if i in given else None for i in range(n)],
                                                                    gcrcs), "map")
        geo = eng.last_geometry()
        if kernel is None:
            assert geo["kernel"] not in (_lib.KERNEL_CHECK, _lib.KERNEL_CHECK_DEGRADED) or geo == before, (name, geo)
        else:
            assert geo["kernel"] == kernel and (geo["G"], geo["stages"], geo["smem_bytes"]) == (plan["G"], plan["stages"], plan["smem_bytes"])
            assert geo["units"] == b.n * -(-b.pb // plan["G"]), (name, geo)
        assert as_list(m) == as_list(want_map), name
        after = [p.copy() if i in given else None for i, p in enumerate(b.parts)]
        fix, where2 = host_result(lambda: eng.correct_stripes_degraded(b.goal, b.nb, after, gcrcs), "fix")
        assert where2 == where, name
        assert eng.status_slots()[1] == 0
        if first is None:
            check_correction(oracle, b, given, gcrcs, want_map, fix, after, pristine)
            first = (m, fix, after, where)
        else:
            assert fix_list(fix) == fix_list(first[1]) and all(x is None or (x == y).all() for x, y in zip(after, first[2])), name
    return first


def check_correction(oracle, b, given, crcs, want_map, fix, after, pristine=None):
    """fix entries against the map and the rule; every corrected block the oracle's rebuild with its zlib CRC; nothing else written"""
    assert as_list(fix[["bad_rows", "suspect_part"]]) == as_list(want_map)
    assert (fix["status"] == expected_status(want_map, b.parts, crcs, given)).all()
    want = [p.copy() if i in given else None for i, p in enumerate(b.parts)]
    for c, s in zip(*np.nonzero(fix["status"] == _lib.FIX_CORRECTED)):
        p = int(fix[c, s]["suspect_part"])
        assert p in given
        blk = rebuilt(oracle, b, b.parts, c, s, p, given)
        block(want, p, c, s)[:] = blk
        if pristine is not None:
            assert (blk == block(pristine, p, c, s)).all(), (c, s, p)
        assert int(fix[c, s]["crc"]) == zlib.crc32(blk.tobytes())
    assert (fix["crc"][fix["status"] != _lib.FIX_CORRECTED] == 0).all()
    for i in given:
        assert (after[i] == want[i]).all(), f"part {i}"


gpu = pytest.mark.gpu


# ---- with every data part: the full-parts calls, byte for byte --------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("fault", SM.FAULTS)
@pytest.mark.parametrize("text", SM.GOALS)
def test_full_parts_equal_the_map_and_the_correction(oracle, text, fault):
    b = SM.batch(oracle, text)
    SM.inject(b, fault)
    n = b.k + b.m
    for env in ROUTES.values():
        eng = engine(**env)
        m0, w0 = host_result(lambda: eng.check_stripe_map(b.goal, b.nb, b.parts, b.crc), "map")
        m1, w1 = host_result(lambda: eng.check_stripe_map_degraded(b.goal, b.nb, b.parts, b.crc), "map")
        assert as_list(m0) == as_list(m1) and w0 == w1
        if not env:
            assert eng.last_geometry()["kernel"] == (_lib.KERNEL_CHECK if not is_cauchy(b.goal) else eng.last_geometry()["kernel"])
        a0, a1 = [p.copy() for p in b.parts], [p.copy() for p in b.parts]
        f0, _ = host_result(lambda: eng.correct_stripes(b.goal, b.nb, a0, b.crc), "fix")
        f1, _ = host_result(lambda: eng.correct_stripes_degraded(b.goal, b.nb, a1, b.crc), "fix")
        assert fix_list(f0) == fix_list(f1) and all((x == y).all() for x, y in zip(a0, a1))
        dev0, dev1 = Dev(b, 48, 16), Dev(b, 48, 16)
        d0 = dev_fix(eng, "correct_stripes_dev", b, dev0, range(n))
        d1 = dev_fix(eng, "correct_stripes_degraded_dev", b, dev1, range(n))
        assert fix_list(d0) == fix_list(d1) == fix_list(f0)
        p0, _ = dev_parts(b, dev0, 16)
        p1, _ = dev_parts(b, dev1, 16)
        assert all((x == y).all() for x, y in zip(p0, p1))
        del dev0, dev1


def dev_fix(eng, call, b, dev, given, dtype=FIX, guard=4096):
    """a _dev call into a guarded result buffer ([n, pb] of dtype); asserts nothing outside it changed"""
    import torch
    size = dtype.itemsize * b.n * b.pb
    init = np.random.default_rng(3).integers(0, 256, 2 * guard + size, dtype=np.uint8)
    t = torch.from_numpy(init.copy()).cuda()
    ptrs = [p if i in given else None for i, p in enumerate(dev.ptrs)]
    crcs = [c if i in given else None for i, c in enumerate(dev.crcs)]
    try:
        getattr(eng, call)(b.goal, b.n, b.nb, ptrs, dev.stride, crcs, t.data_ptr() + guard)
    except L.ChunkCrcError:
        pass
    torch.cuda.synchronize()
    out = t.cpu().numpy()
    assert (out[:guard] == init[:guard]).all() and (out[guard + size:] == init[guard + size:]).all(), f"{call}: write outside the result"
    return out[guard:guard + size].copy().view(dtype).reshape(b.n, b.pb)


# ---- lost parts against the oracle -----------------------------------------------------------------------------------------------

def lost_sets(g):
    """one, two and three data parts (as the spares allow), a data part and a parity part, parity only"""
    k, m = g.k, g.m
    out = [(1,)]
    if m >= 3:
        out.append((0, k - 1))
    if m >= 4:
        out.append((1, k // 2, k - 1))
    if m >= 3:
        out.append((k // 2, k))
    if m >= 2:
        out.append((k + m - 1,))
    return out


LOST = [(name, lost) for name in ("ec(3,2)", "ec(5,3)", "ec(8,2)", "ec(8,3)", "ec(8,4)", "ec(20,4)", "ec(32,3)", "ec(22,4)", "ec(10,5)")
        for lost in lost_sets(L.SliceType(name))]


def inject_degraded(b, given):
    """faults in chunks 0 and 2: an input data part, a spare, an input parity part, two parts in one stripe, the short last stripe"""
    inputs, spares = roles(b, given)
    k, last = b.k, b.pb - 1
    b.corrupt(0, inputs[0], 0, offset=300)
    b.corrupt(0, spares[-1], 1, offset=4000)
    b.corrupt(2, inputs[-1], 0, offset=9000)
    b.corrupt(2, inputs[0], 1, offset=100)                 # two parts in one stripe
    b.corrupt(2, spares[0], 1, offset=50000)
    if 0 in given:
        b.corrupt(2, 0, last, offset=65530, length=6)      # the short last stripe: data part 0 alone has a block there
    else:
        b.corrupt(2, spares[0], last, offset=20)


@gpu
@pytest.mark.parametrize("name,lost", LOST, ids=[f"{n}-lost{'.'.join(map(str, l))}" for n, l in LOST])
def test_lost_parts_against_the_oracle(oracle, name, lost):
    g = L.SliceType(name)
    nb = 2 * g.k + 1
    pristine = Batch(oracle, name, 3, nb, seed=5)
    b = Batch(oracle, name, 3, nb, seed=5)
    given = [i for i in range(g.k + g.m) if i not in lost]
    inject_degraded(b, given)
    m, fix, after, where = run_routes(oracle, b, given, pristine=None)
    assert where is None and not any(e[0] for e in as_list(m)[1])           # chunk 1 clean
    inputs, spares = roles(b, given)
    if len(spares) >= 2:                                 # a single fault is named (the punctured code corrects one error)
        assert as_list(m)[0][0][1] == inputs[0] and as_list(m)[0][1][1] == spares[-1]
        assert fix[0, 0]["status"] == fix[0, 1]["status"] == _lib.FIX_CORRECTED
        for s, p in ((0, inputs[0]), (1, spares[-1])):
            assert (block(after, p, 0, s) == block(pristine.parts, p, 0, s)).all()


# ---- every fused instantiation at capped grids --------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("case", range(len(CASES)), ids=[f"{c[0]}-lost{'.'.join(map(str, c[1]))}-rows{''.join(map(str, c[2]))}" for c in CASES])
def test_geometry_case(oracle, case):
    name, lost, rows, want = CASES[case]
    g = L.SliceType(name)
    given = [i for i in range(g.k) if i not in lost] + [g.k + r for r in rows]
    G = want[3]
    pb = 2 * G + G // 2
    nb = g.k * pb - (g.k - 1)
    b = Batch(oracle, name, 2, nb, seed=case)
    inputs, spares = roles(b, given)
    for s in (0, G - 1, G, 2 * G, pb - 2):
        b.corrupt(s % 2, inputs[s % len(inputs)], s, offset=(977 * s) % 65000)
    b.corrupt(1, spares[-1], G + 1, offset=123)
    contexts = {"cap1": {"LZGPU_GRID_CAP": 1}, "cap3": {"LZGPU_GRID_CAP": 3}, "generic": {"LZGPU_DISABLE_FUSED": 1}}
    run_routes(oracle, b, given, contexts=contexts)
    for ctx, cap in (("cap1", 1), ("cap3", 3)):
        geo = engine(**contexts[ctx]).last_geometry()     # the correction's map launch
        assert geo["kernel"] == _lib.KERNEL_CHECK_DEGRADED and geo["grid"] == min(cap, geo["units"]) and geo["G"] == G


# ---- the motivating case, end to end -----------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("name", ["ec(5,3)", "ec(8,4)"])
def test_stale_input_is_corrected_before_the_rebuild(oracle, name):
    """data part 1 lost, data part 3 stale (valid CRCs) in stripes 10-12: a plain rebuild of part 1 is wrong in exactly those
    stripes; the degraded correction names part 3 there and restores it; the rebuild then returns the original bytes"""
    g = L.SliceType(name)
    k = g.k
    pb = 16
    nb = k * pb
    pristine = Batch(oracle, name, 1, nb, seed=11, tail=0)
    b = Batch(oracle, name, 1, nb, seed=11, tail=0)
    for s in (10, 11, 12):
        b.corrupt(0, 3, s, offset=1000 * s)
    given = [i for i in range(k + g.m) if i != 1]
    eng = engine()
    avail = [b.parts[i] if i in given else None for i in range(k + g.m)]
    out, _ = eng.recover_chunks(b.goal, nb, avail, part_crc=[b.crc[i] if i in given else None for i in range(k + g.m)])
    bad = [s for s in range(pb) if (block(out, 1, 0, s) != block(pristine.parts, 1, 0, s)).any()]
    assert bad == [10, 11, 12]
    after = [p.copy() if i in given else None for i, p in enumerate(b.parts)]
    fix = eng.correct_stripes_degraded(b.goal, nb, after, [b.crc[i] if i in given else None for i in range(k + g.m)])
    assert eng.last_geometry()["kernel"] == _lib.KERNEL_CHECK_DEGRADED
    for s in range(pb):
        if s in (10, 11, 12):
            assert fix[0, s]["status"] == _lib.FIX_CORRECTED and fix[0, s]["suspect_part"] == 3
            assert int(fix[0, s]["crc"]) == zlib.crc32(block(pristine.parts, 3, 0, s).tobytes())
        else:
            assert fix[0, s]["status"] == _lib.FIX_CLEAN
    for i in given:
        assert (after[i] == pristine.parts[i]).all(), i
    crcs = [None if i not in given else b.crc[i].copy() for i in range(k + g.m)]
    for s in (10, 11, 12):
        crcs[3][0, s] = fix[0, s]["crc"]
    out, _ = eng.recover_chunks(b.goal, nb, after, part_crc=crcs)
    assert (out[1] == pristine.parts[1]).all()


@gpu
def test_one_spare_detects_but_never_blames(oracle):
    """ec(8,2) with data part 1 lost: one spare, so a bad stripe is UNEXPLAINED and ERR_INCONSISTENT, and nothing is written"""
    b = Batch(oracle, "ec(8,2)", 2, 8 * 4, seed=3)
    b.corrupt(1, 4, 2)
    given = [i for i in range(10) if i != 1]
    for env in ROUTES.values():
        eng = engine(**env)
        after = [p.copy() if i in given else None for i, p in enumerate(b.parts)]
        fix = np.zeros((b.n, b.pb), dtype=FIX)
        rc = eng.lib.lzgpu_correct_stripes_degraded(eng.h, ctypes.byref(b.goal.c), b.n, b.nb, E._ptr_array(after), b.pb * BLOCK, None,
                                                     E._p(fix), None)
        assert rc == _lib.ERR_INCONSISTENT
        assert fix[1, 2]["status"] == _lib.FIX_UNEXPLAINED and fix[1, 2]["bad_rows"] == 2 and fix[1, 2]["suspect_part"] == -1
        assert all((after[i] == b.parts[i]).all() for i in given)


# ---- the rest: CRC gate, stored CRCs, deferred mode, refusals, layouts, tiles, one full chunk ------------------------------------------

@gpu
def test_crc_gate_and_stored_crc_failures(oracle):
    """ec(8,4) without data part 2: a stale input (valid CRC) is corrected; a stripe whose other block fails its stored CRC is a
    CRC_CONFLICT; the map is written whole and bad names the smallest failing position"""
    b = Batch(oracle, "ec(8,4)", 2, 8 * 6, seed=8)
    given = [i for i in range(12) if i != 2]
    b.corrupt(0, 5, 1)
    b.corrupt(1, 9, 3)
    crcs = [c.copy() for c in b.crc]
    crcs[10][1, 3] ^= 0x40           # fails: blocks the correction of stripe 3 of chunk 1
    crcs[11][0, 4] ^= 0x40           # fails in a clean stripe
    want = expected_map(oracle, b, given)
    m, fix, after, where = run_routes(oracle, b, given, crcs=crcs, want_map=want)
    assert where == (0, 11, 4)
    assert fix[0, 1]["status"] == _lib.FIX_CORRECTED and fix[1, 3]["status"] == _lib.FIX_CRC_CONFLICT


@gpu
def test_refusals_launch_nothing(oracle):
    import torch
    b = Batch(oracle, "ec(5,3)", 1, 10, seed=2)
    dev = Dev(b, 0, 0)
    eng = engine()
    before = eng.stats()["kernel_launches"]
    out = torch.zeros(64, dtype=torch.uint8, device="cuda")
    for call in ("check_stripe_map_degraded_dev", "correct_stripes_degraded_dev"):
        with pytest.raises(L.LzGpuError) as ei:          # k given parts
            getattr(eng, call)(b.goal, 1, b.nb, [p if i not in (0, 6, 7) else None for i, p in enumerate(dev.ptrs)], dev.stride, None,
                               out.data_ptr())
        assert ei.value.status == _lib.ERR_TOO_FEW_PARTS
        with pytest.raises(L.LzGpuError) as ei:          # misaligned part
            getattr(eng, call)(b.goal, 1, b.nb, [None] + [p + 8 if i == 3 else p for i, p in enumerate(dev.ptrs[1:], 1)], dev.stride,
                               None, out.data_ptr())
        assert ei.value.status == _lib.ERR_ARG
    for fn in (eng.check_stripe_map_degraded, eng.correct_stripes_degraded):
        with pytest.raises(L.LzGpuError) as ei:
            fn(b.goal, b.nb, [None, None, None] + [p.copy() for p in b.parts[3:]])
        assert ei.value.status == _lib.ERR_TOO_FEW_PARTS
    torch.cuda.synchronize()
    assert eng.stats()["kernel_launches"] == before


@gpu
def test_deferred_mode_collects_the_crc_mismatch(oracle):
    b = Batch(oracle, "ec(5,3)", 2, 5 * 4, seed=6)
    given = [i for i in range(8) if i != 1]
    dev = Dev(b, 0, 0)
    dev.bufs[2 * 6 + 1][1, 2] ^= 1                       # part 6, chunk 1, block 2
    eng = engine()
    import torch
    out = torch.zeros(b.n * b.pb * 8, dtype=torch.uint8, device="cuda")
    eng.set_deferred_verify(True)
    try:
        eng.check_stripe_map_degraded_dev(b.goal, b.n, b.nb, [p if i in given else None for i, p in enumerate(dev.ptrs)], dev.stride,
                                          [c if i in given else None for i, c in enumerate(dev.crcs)], out.data_ptr())
        with pytest.raises(L.ChunkCrcError) as ei:
            eng.sync()
        assert ei.value.where == (1, 6, 2)
    finally:
        eng.set_deferred_verify(False)


@gpu
@pytest.mark.parametrize("pad,lead", [(16, 16), (65536 + 48, 48)])
def test_dev_layouts_write_only_the_blocks_and_the_entries(oracle, pad, lead):
    b = Batch(oracle, "ec(8,3)", 3, 8 * 5 + 1, seed=4)
    given = [i for i in range(11) if i not in (1, 4)]
    b.corrupt(0, 0, 1)
    b.corrupt(2, 9, 3)
    want = expected_map(oracle, b, given)
    for env in ROUTES.values():
        eng = engine(**env)
        dev = Dev(b, pad, lead)
        m = dev_fix(eng, "check_stripe_map_degraded_dev", b, dev, given, dtype=STATE)
        assert as_list(m) == as_list(want)
        fix = dev_fix(eng, "correct_stripes_degraded_dev", b, dev, given)
        parts, bufs = dev_parts(b, dev, lead)
        check_correction(oracle, b, given, [b.crc[i] if i in given else None for i in range(11)], want, fix,
                         [parts[i] if i in given else None for i in range(11)])
        for i in range(11):
            if i not in given:
                assert (parts[i] == b.parts[i]).all()            # a lost part's buffer is never written
            outside = np.ones(len(bufs[i]), dtype=bool)
            for c in range(b.n):
                outside[lead + c * dev.stride: lead + c * dev.stride + b.pb * BLOCK] = False
            host_init = np.random.default_rng(7).integers(0, 256, len(bufs[i]), dtype=np.uint8)
            assert (bufs[i][outside] == host_init[outside]).all(), i
        del dev


@gpu
def test_host_tiles_and_one_full_size_chunk(oracle):
    """ec(8,4) without data parts 1 and 4: 51 chunks of 16 stripes take three host tiles of 25 chunks; one full 64 MiB chunk"""
    b = Batch(oracle, "ec(8,4)", 51, 8 * 16, seed=12)
    given = [i for i in range(12) if i not in (1, 4)]
    for c in range(0, 51, 5):
        b.corrupt(c, [0, 2, 8, 10][c % 4], c % 16)
    eng = engine()
    before = eng.stats()["batches_timed"]
    m, where = host_result(lambda: eng.check_stripe_map_degraded(b.goal, b.nb, [b.parts[i] if i in given else None for i in range(12)],
                                                                  [b.crc[i] if i in given else None for i in range(12)]), "map")
    tile = max(1, (2 * 128 << 20) // (16 * BLOCK * 10))
    assert tile == 25 and eng.stats()["batches_timed"] - before == 3
    assert as_list(m) == as_list(expected_map(oracle, b, given))
    del b
    big = Batch(oracle, "ec(8,4)", 1, 1024, seed=13, tail=0)
    big.corrupt(0, 3, 77)
    big.corrupt(0, 9, 127)
    given = [i for i in range(12) if i != 0]
    for env in ROUTES.values():
        eng = engine(**env)
        after = [p.copy() if i in given else None for i, p in enumerate(big.parts)]
        fix = eng.correct_stripes_degraded(big.goal, 1024, after, [big.crc[i] if i in given else None for i in range(12)])
        st = fix[0]["status"]
        assert st[77] == st[127] == _lib.FIX_CORRECTED and (st == _lib.FIX_CLEAN).sum() == 126
        assert fix[0, 77]["suspect_part"] == 3 and fix[0, 127]["suspect_part"] == 9
