"""The correction of several slices (lzgpu_correct_slices*: the CORRECT instantiation of recover_slices_kernel, the locate pass and
correct_slices_kernel in csrc/recover_slices_kernel.cuh) on the GPU.

Inputs are encoded by lzgpu_encode_slices and made stale as in tests/test_gpu_check_slices.py.  Every fix entry is compared with the
map lzgpu_check_slices returns before the call and with the rule computed here from the plan's correctable masks; a corrected part
with the encoded original, its new CRCs with zlib, and the result with lzgpu_check_slices and with one-combined-stripe windows of
lzgpu_recover_slices.  Covered: clean batches of six goal sets (nb < L, a ragged nb, one 64 MiB chunk) with sentinel buffers; a stale
part at every flat position of two goal sets, with every part given and with one lost; several combined stripes per chunk blaming
different parts; the tail stripe's padding; an undetermined suspect and two stale parts; stored-CRC conflicts, a stale and rotten
suspect block and new_crc aliasing part_crc; the one-goal case against lzgpu_correct_stripes; the _dev form with guard bytes in both
verification modes, the CRC-disabled mode, the refusals, the launch report and the host form's bytes_d2h; pools of two and three
slots on one device.  Each case runs on the default context and with LZGPU_GRID_CAP=2."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200.engine import ChunkCrcError, LzGpuError, _goal_array, _p, _ptr_array
from tests.test_gpu_check_slices import SETS, engine, make_stale, n_parts, nbs, raw, slice_of
from tests.test_gpu_salvage_slices import original, to_dev
from tests.test_recover_slices_plan import goalset, lcm_of

pytestmark = pytest.mark.gpu
BLOCK = 65536
SENTINEL = 0xA5A5A5A5
FIX = L.Engine.SLICES_FIX_DTYPE


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    from tests import test_gpu_check_slices as T
    for e in T._engines.values():
        e.close()
    T._engines.clear()


def ks(goals):
    return [1 if g.is_std else g.k for g in goals]


def pbs(goals, nb):
    return [-(-nb // k) for k in ks(goals)]


def correct(e, goals, nb, parts, crcs, new_crc=True, fn=None):
    """lzgpu_correct_slices (or fn, same arguments) on copies of the parts: (code, fix, bad, parts after, new CRC arrays filled with
    SENTINEL before the call, or None)"""
    n = next(p.shape[0] for p in parts if p is not None)
    sl = slice_of(goals)
    pb = pbs(goals, nb)
    out = [None if p is None else p.copy() for p in parts]
    nc = [None if p is None else np.full((n, pb[sl[g]]), SENTINEL, dtype=np.uint32) for g, p in enumerate(parts)] if new_crc else None
    fix = np.zeros((n, -(-nb // lcm_of(goals))), dtype=FIX)
    bad = (C.c_int64 * 4)(-1, -1, -1, -1)
    cr = None if crcs is None else _ptr_array([None if c is None else np.ascontiguousarray(c) for c in crcs])
    f = fn or e.lib.lzgpu_correct_slices
    rc = f(e.h, _goal_array(goals), len(goals), n, nb, _ptr_array(out), (C.c_size_t * len(goals))(*[p * BLOCK for p in pb]), cr,
           _ptr_array(nc) if nc is not None else None, _p(fix), bad)
    return rc, fix, tuple(bad), out, nc


def written_blocks(goals, nb, g, cs):
    """the part blocks of flat part g that a correction of combined stripe cs writes (real data blocks, parity of existing stripes)"""
    Lc, sl = lcm_of(goals), slice_of(goals)
    k = ks(goals)[sl[g]]
    j = g - sl.index(sl[g])
    valid = min(Lc, nb - cs * Lc)
    out = []
    for s in range(Lc // k):
        if s * k >= valid:
            continue
        if j < k and s * k + j >= valid:
            continue
        out.append(cs * (Lc // k) + s)
    return out


def expected_status(goals, nb, given, fix_before, crc_failed):
    """the rule, per entry, from the check map before the call"""
    plan = L.Engine.plan_correct_slices(goals, nb, given)
    n, n_cs = fix_before.shape
    st = np.zeros((n, n_cs), dtype=np.int32)
    for c in range(n):
        for cs in range(n_cs):
            tail = plan["tail_blocks"] and cs == n_cs - 1
            corr = plan["tail_correctable"] if tail else plan["correctable"]
            b, g = int(fix_before[c, cs]["bad_checks"]), int(fix_before[c, cs]["suspect_part"])
            f = int(crc_failed[c, cs])
            st[c, cs] = (_lib.FIX_CLEAN if not b else _lib.FIX_UNEXPLAINED if g < 0 else _lib.FIX_CRC_CONFLICT if f & ~(1 << g)
                         else _lib.FIX_UNDETERMINED if not (corr >> g) & 1 else _lib.FIX_CORRECTED)
    return st


def check_result(e, goals, nb, given, before, after, crcs, fix, nc, orig=None):
    """the map, the rule, the bytes written, changed and the new CRCs of one call; orig: the parts as encoded"""
    rc0, m0, _ = raw(e, goals, nb, [p if given[g] else None for g, p in enumerate(before)], None)
    assert np.array_equal(fix["bad_checks"], m0["bad_checks"]) and np.array_equal(fix["suspect_part"], m0["suspect_part"])
    assert np.array_equal(fix["status"], expected_status(goals, nb, given, m0, fix["crc_failed"]))
    Lc, sl = lcm_of(goals), slice_of(goals)
    n, n_cs = fix.shape
    rewritten = {g: set() for g in range(len(before))}
    for c in range(n):
        for cs in range(n_cs):
            f = fix[c, cs]
            if f["status"] != _lib.FIX_CORRECTED:
                assert f["changed"] == 0
                continue
            g = int(f["suspect_part"])
            spc = Lc // ks(goals)[sl[g]]
            ch = 0
            for b in written_blocks(goals, nb, g, cs):
                rewritten[g].add((c, b))
                if not np.array_equal(before[g][c, b * BLOCK:(b + 1) * BLOCK], after[g][c, b * BLOCK:(b + 1) * BLOCK]):
                    ch |= 1 << (b - cs * spc)
                if nc is not None:
                    assert nc[g][c, b] == zlib.crc32(after[g][c, b * BLOCK:(b + 1) * BLOCK].tobytes()), (g, c, b)
                if orig is not None:
                    assert np.array_equal(after[g][c, b * BLOCK:(b + 1) * BLOCK], orig[g][c, b * BLOCK:(b + 1) * BLOCK]), (g, c, b)
            assert int(f["changed"]) == ch
    for g in range(len(before)):
        if not given[g]:
            continue
        for c in range(n):
            for b in range(after[g].shape[1] // BLOCK):
                if (c, b) in rewritten[g]:
                    continue
                assert np.array_equal(before[g][c, b * BLOCK:(b + 1) * BLOCK], after[g][c, b * BLOCK:(b + 1) * BLOCK]), (g, c, b)
                if nc is not None:
                    assert nc[g][c, b] == SENTINEL
    return rewritten


def window_equals(e, goals, nb, given, after, c, cs, g):
    """where lzgpu_recover_slices accepts a one-combined-stripe window with g lost and wanted, it rebuilds g's blocks as corrected"""
    Lc, sl, k = lcm_of(goals), slice_of(goals), ks(goals)
    valid = min(Lc, nb - cs * Lc)
    win = []
    for h, p in enumerate(after):
        if not given[h] or h == g:
            win.append(None)
            continue
        spc, pbw = Lc // k[sl[h]], -(-valid // k[sl[h]])
        win.append(np.ascontiguousarray(p[c:c + 1, cs * spc * BLOCK:(cs * spc + pbw) * BLOCK]))
    want = [1 if h == g else 0 for h in range(len(after))]
    try:
        out, _, _ = e.recover_slices(goals, valid, win, want=want, with_crc=False)
    except LzGpuError as ex:
        assert ex.status == _lib.ERR_TOO_FEW_PARTS
        return False
    spc = Lc // k[sl[g]]
    for b in written_blocks(goals, nb, g, cs):
        s = b - cs * spc
        assert np.array_equal(out[g][0, s * BLOCK:(s + 1) * BLOCK], after[g][c, b * BLOCK:(b + 1) * BLOCK]), (g, c, cs, s)
    return True


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names", SETS, ids="+".join)
def test_clean_batches(names, ctx):
    e = engine(ctx)
    goals = goalset(names)
    n = n_parts(goals)
    for nb in nbs(lcm_of(goals)):
        _, parts, crcs = original(goals, 2, nb, nb)
        for given in ([1] * n, [1 if g % 3 else 0 for g in range(n)]):
            inp = [p if given[g] else None for g, p in enumerate(parts)]
            inc = [c if given[g] else None for g, c in enumerate(crcs)]
            p = L.Engine.plan_check_slices(goals, nb, given)
            if not (p["n_checks"] if nb >= p["L"] else 0) and not (p["tail_n_checks"] if p["tail_blocks"] else 0):
                continue
            rc, fix, bad, out, nc = correct(e, goals, nb, inp, inc)
            assert rc == _lib.OK and bad == (-1, -1, -1, -1), (names, nb, given)
            assert (fix["status"] == _lib.FIX_CLEAN).all() and (fix["bad_checks"] == 0).all() and (fix["suspect_part"] == -1).all()
            assert (fix["crc_failed"] == 0).all() and (fix["changed"] == 0).all()
            for g in range(n):
                if given[g]:
                    assert np.array_equal(out[g], parts[g]) and (nc[g] == SENTINEL).all()
            geo = e.last_geometry()
            assert geo["kernel"] == _lib.KERNEL_CORRECT_SLICES and (geo["threads"], geo["smem_bytes"]) == (p["threads"], p["smem_bytes"])
            if ctx == "cap2":
                assert geo["grid"] <= 2


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_clean_64mib_chunk(ctx):
    goals = goalset(("std", "xor2", "xor3"))
    _, parts, crcs = original(goals, 1, 1024, 5)
    rc, fix, _, out, nc = correct(engine(ctx), goals, 1024, parts, crcs)
    assert rc == _lib.OK and fix.shape == (1, 171) and (fix["status"] == _lib.FIX_CLEAN).all()
    assert all(np.array_equal(a, b) for a, b in zip(out, parts)) and all((x == SENTINEL).all() for x in nc)


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names", [("std", "xor2", "xor3"), ("ec(3,2)", "ec(4,2)")], ids="+".join)
def test_stale_part_at_every_position(names, ctx):
    e = engine(ctx)
    goals = goalset(names)
    n = n_parts(goals)
    Lc = lcm_of(goals)
    nb = 2 * Lc + Lc // 2
    sl = slice_of(goals)
    _, parts, crcs = original(goals, 2, nb, 11)
    for given in ([1] * n, [0 if g == n - 1 else 1 for g in range(n)]):
        plan = L.Engine.plan_correct_slices(goals, nb, given)
        for g in range(n):
            if not given[g]:
                continue
            k = ks(goals)[sl[g]]
            spc = Lc // k
            j = g - sl.index(sl[g])
            blocks = [(0, spc + s) for s in range(spc)] + [(1, 0), (1, 2 * spc)]
            blocks = [(c, b) for c, b in blocks if (b * k + j if j < k else b * k) < nb]
            sp, sc = make_stale(goals, nb, parts, crcs, g, blocks, g)
            inp = [p if given[h] else None for h, p in enumerate(sp)]
            inc = [c if given[h] else None for h, c in enumerate(sc)]
            rc, fix, bad, out, nc = correct(e, goals, nb, inp, inc)
            assert bad == (-1, -1, -1, -1)
            left = np.isin(fix["status"], [_lib.FIX_UNEXPLAINED, _lib.FIX_UNDETERMINED]).any()
            assert rc == (_lib.ERR_INCONSISTENT if left else _lib.OK), (names, given, g)
            check_result(e, goals, nb, given, inp, out, inc, fix, nc, orig=parts)
            if (plan["locatable"] >> g) & 1:   # combined stripe 1 of chunk 0 is a full one
                f = fix[0, 1]
                assert f["status"] == _lib.FIX_CORRECTED and f["suspect_part"] == g
                assert int(f["changed"]) == sum(1 << (b - spc) for c, b in blocks if c == 0)
            if (fix["status"] == _lib.FIX_CORRECTED).sum() == (fix["bad_checks"] != 0).sum():
                assert np.array_equal(out[g], parts[g]), (names, given, g)
                assert raw(e, goals, nb, out, None)[0] == _lib.OK
            for c, cs in zip(*np.nonzero(fix["status"] == _lib.FIX_CORRECTED)):
                window_equals(e, goals, nb, given, out, int(c), int(cs), g)


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_several_stripes_blame_different_parts(ctx):
    e = engine(ctx)
    goals = goalset(("ec(3,2)", "ec(4,2)"))
    Lc, nb = 12, 36
    _, parts, crcs = original(goals, 2, nb, 17)
    sp, sc = parts, crcs
    plan = [(1, 0, 0), (6, 1, 1), (9, 2, 1), (4, 1, 0)]   # (flat part, combined stripe, chunk)
    for g, cs, c in plan:
        spc = Lc // (3 if g < 5 else 4)
        sp, sc = make_stale(goals, nb, sp, sc, g, [(c, cs * spc)], g + cs)
    rc, fix, bad, out, nc = correct(e, goals, nb, sp, sc)
    assert rc == _lib.OK and bad == (-1, -1, -1, -1)
    for g, cs, c in plan:
        assert fix[c, cs]["status"] == _lib.FIX_CORRECTED and fix[c, cs]["suspect_part"] == g and fix[c, cs]["changed"] == 1
    assert (fix["status"] == _lib.FIX_CORRECTED).sum() == len(plan)
    check_result(e, goals, nb, [1] * 11, sp, out, sc, fix, nc, orig=parts)
    assert all(np.array_equal(a, b) for a, b in zip(out, parts))


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_tail_stripe_padding_is_never_written(ctx):
    e = engine(ctx)
    goals = goalset(("ec(3,2)", "ec(4,2)"))
    nb = 29                                   # the tail combined stripe holds positions 24 .. 28
    _, parts, crcs = original(goals, 1, nb, 23)
    g = 7                                     # ec(4,2) data part 2: blocks 6 (position 26) and 7 (position 30, padding)
    p, cr = [x.copy() for x in parts], [x.copy() for x in crcs]
    p[g][0, 7 * BLOCK:8 * BLOCK] = 0x3C       # padding is not a check: any bytes, with a matching CRC
    cr[g][0, 7] = zlib.crc32(p[g][0, 7 * BLOCK:8 * BLOCK].tobytes())
    sp, sc = make_stale(goals, nb, p, cr, g, [(0, 6)], 4)
    rc, fix, bad, out, nc = correct(e, goals, nb, sp, sc)
    assert rc == _lib.OK and fix[0, 2]["status"] == _lib.FIX_CORRECTED and fix[0, 2]["suspect_part"] == g and fix[0, 2]["changed"] == 1
    assert np.array_equal(out[g][0, 6 * BLOCK:7 * BLOCK], parts[g][0, 6 * BLOCK:7 * BLOCK])
    assert (out[g][0, 7 * BLOCK:] == 0x3C).all() and nc[g][0, 7] == SENTINEL
    check_result(e, goals, nb, [1] * 11, sp, out, sc, fix, nc)


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_undetermined_and_unexplained_write_nothing(ctx):
    e = engine(ctx)
    goals = goalset(("std", "xor2", "xor3"))
    nb = 12
    _, parts, crcs = original(goals, 1, nb, 31)
    given = [1, 0, 0, 1, 0, 0, 0, 1]
    sp, sc = make_stale(goals, nb, parts, crcs, 0, [(0, 0)], 2)   # std block 0: named std, which is not correctable
    inp = [p if given[g] else None for g, p in enumerate(sp)]
    inc = [c if given[g] else None for g, c in enumerate(sc)]
    rc, fix, _, out, nc = correct(e, goals, nb, inp, inc)
    assert rc == _lib.ERR_INCONSISTENT
    assert fix[0, 0]["suspect_part"] == 0 and fix[0, 0]["status"] == _lib.FIX_UNDETERMINED and fix[0, 0]["changed"] == 0
    assert np.array_equal(out[0], sp[0]) and (nc[0] == SENTINEL).all()
    check_result(e, goals, nb, given, inp, out, inc, fix, nc)
    goals = goalset(("ec(3,2)", "ec(4,2)"))
    nb = 24
    _, parts, crcs = original(goals, 1, nb, 37)
    sp, sc = make_stale(goals, nb, parts, crcs, 1, [(0, 4)], 1)    # combined stripe 1: ec(3,2) data part 1 ...
    sp, sc = make_stale(goals, nb, sp, sc, 6, [(0, 3)], 2)         # ... and ec(4,2) data part 1
    rc, fix, _, out, nc = correct(e, goals, nb, sp, sc)
    assert rc == _lib.ERR_INCONSISTENT
    assert fix[0, 1]["status"] == _lib.FIX_UNEXPLAINED and fix[0, 1]["suspect_part"] == -1
    assert all(np.array_equal(a, b) for a, b in zip(out, sp)) and all((x == SENTINEL).all() for x in nc)
    f2, _ = e.correct_slices(goals, nb, [p.copy() for p in sp], sc)   # LZGPU_ERR_INCONSISTENT is no failure: the entries say where
    assert np.array_equal(f2, fix)


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_stored_crc_cases(ctx):
    e = engine(ctx)
    goals = goalset(("ec(3,2)", "ec(4,2)"))
    nb = 30
    _, parts, crcs = original(goals, 3, nb, 8)
    # stale part 2 in combined stripe 0 of chunk 0; a rotten block of part 9 in the same stripe; another rotten block elsewhere
    sp, sc = make_stale(goals, nb, parts, crcs, 2, [(0, 1)], 3)
    sc[9] = sc[9].copy()
    sc[9][0, 2] ^= 1
    sc[5] = sc[5].copy()
    sc[5][1, 4] ^= 1
    rc, fix, bad, out, nc = correct(e, goals, nb, sp, sc)
    assert rc == _lib.ERR_CRC and bad == (0, 1, 4, 2)
    assert fix[0, 0]["status"] == _lib.FIX_CRC_CONFLICT and fix[0, 0]["crc_failed"] == 1 << 9
    assert fix[1, 1]["crc_failed"] == 1 << 5 and fix[1, 1]["status"] == _lib.FIX_CLEAN
    assert np.array_equal(out[2], sp[2]) and (nc[2] == SENTINEL).all()
    check_result(e, goals, nb, [1] * 11, sp, out, sc, fix, nc)
    with pytest.raises(ChunkCrcError) as ex:
        e.correct_slices(goals, nb, [p.copy() for p in sp], sc)
    assert tuple(ex.value.where) == (0, 1, 4, 2) and np.array_equal(ex.value.fix, fix)
    # a suspect block that is stale and rotten (its stored CRC is the original's) is corrected
    sp, _ = make_stale(goals, nb, parts, crcs, 8, [(2, 5)], 6)
    rc, fix, bad, out, nc = correct(e, goals, nb, sp, crcs)
    assert rc == _lib.ERR_CRC and bad == (2, 1, 3, 5)
    assert fix[2, 1]["status"] == _lib.FIX_CORRECTED and fix[2, 1]["crc_failed"] == 1 << 8 and fix[2, 1]["changed"] == 1 << 2
    assert np.array_equal(out[8], parts[8]) and nc[8][2, 5] == crcs[8][2, 5]
    # new_crc aliasing part_crc: the stored CRCs are read before any is written
    sp, sc = make_stale(goals, nb, parts, crcs, 10, [(1, 3), (2, 0)], 9)
    out = [p.copy() for p in sp]
    alias = [c.copy() for c in sc]
    fix = np.zeros((3, 3), dtype=FIX)
    bad = (C.c_int64 * 4)(-1, -1, -1, -1)
    arr = _ptr_array(alias)
    rc = e.lib.lzgpu_correct_slices(e.h, _goal_array(goals), 2, 3, nb, _ptr_array(out), (C.c_size_t * 2)(10 * BLOCK, 8 * BLOCK), arr, arr,
                                    _p(fix), bad)
    assert rc == _lib.OK and tuple(bad) == (-1, -1, -1, -1)
    assert fix[1, 1]["status"] == _lib.FIX_CORRECTED and fix[2, 0]["status"] == _lib.FIX_CORRECTED
    assert all(np.array_equal(a, b) for a, b in zip(out, parts)) and all(np.array_equal(a, b) for a, b in zip(alias, crcs))


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("name", ["ec(8,2)", "ec(6,3)", "ec(8,4)"])
def test_one_goal_equals_correct_stripes(name, ctx):
    e = engine(ctx)
    goal = L.SliceType(name)
    k, m_ = goal.k, goal.m
    rng = np.random.default_rng(k * 10 + m_)
    nb = 5 * k + 2
    pb = -(-nb // k)
    _, parts, crcs = original([goal], 2, nb, k)
    for trial in range(4):
        g = int(rng.integers(0, k + m_))
        real = [b for b in range(pb) if g >= k or b * k + g < nb]
        blocks = [(int(rng.integers(0, 2)), int(b)) for b in rng.choice(real, size=min(3, len(real)), replace=False)]
        sp, sc = make_stale([goal], nb, parts, crcs, g, blocks, trial)
        rc, fix, _, out, nc = correct(e, [goal], nb, sp, sc)
        ref_parts = [p.copy() for p in sp]
        ref = e.correct_stripes(goal, nb, ref_parts, sc)
        assert np.array_equal(fix["suspect_part"], ref["suspect_part"]) and np.array_equal(fix["status"], ref["status"]), (name, g)
        assert all(np.array_equal(a, b) for a, b in zip(out, ref_parts)) and np.array_equal(out[g], parts[g])
        for c, s in zip(*np.nonzero(fix["status"] == _lib.FIX_CORRECTED)):
            assert nc[g][c, s] == ref[c, s]["crc"]
        assert rc == _lib.OK


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("deferred", [False, True])
def test_dev_form_guard_bytes(ctx, deferred):
    e = engine(ctx)
    goals = goalset(("std", "xor2", "xor3"))
    n, nb = 2, 17
    given = [1, 1, 0, 1, 1, 1, 1, 1]
    _, parts, crcs = original(goals, n, nb, 21)
    sp, sc = make_stale(goals, nb, parts, crcs, 4, [(1, 2)], 5)
    sl = slice_of(goals)
    pb = pbs(goals, nb)
    GUARD, OFF = 4096, 4096 + 48
    pstride = [p * BLOCK + 4096 for p in pb]
    inp = [p if given[g] else None for g, p in enumerate(sp)]
    inc = [c if given[g] else None for g, c in enumerate(sc)]
    _, want, _, want_parts, want_nc = correct(engine("default"), goals, nb, inp, inc)
    assert want[1, 1]["status"] == _lib.FIX_CORRECTED
    n_cs = -(-nb // 6)
    for crc_mode in ("verify", "none", "disabled"):
        bufs = {g: to_dev(sp[g], 0x77, GUARD, OFF, pstride[sl[g]]) for g in range(8) if given[g]}
        cbufs = {g: torch.from_numpy(sc[g].view(np.int32).copy()).cuda() for g in bufs}
        nbufs = {g: torch.full((GUARD // 4 + n * pb[sl[g]] + GUARD // 4,), SENTINEL - 2 ** 32, dtype=torch.int32, device="cuda") for g in bufs}
        dfix = torch.full((GUARD + n * n_cs * 32 + GUARD,), 0xEE, dtype=torch.uint8, device="cuda")
        ptrs = [bufs[g].data_ptr() + OFF if g in bufs else 0 for g in range(8)]
        nptrs = [nbufs[g].data_ptr() + GUARD if g in nbufs else 0 for g in range(8)]
        lib = _lib.load()
        cptrs = [cbufs[g].data_ptr() if g in cbufs else 0 for g in range(8)] if crc_mode != "none" else None
        if crc_mode == "disabled":
            lib.lzgpu_set_crc_enabled(0)
        try:
            call = lambda: e.correct_slices_dev(goals, n, nb, ptrs, pstride, cptrs, nptrs, dfix.data_ptr() + GUARD)
            if crc_mode == "verify" and deferred:
                e.set_deferred_verify(True)
                try:
                    call()
                    e.sync()
                finally:
                    e.set_deferred_verify(False)
            elif crc_mode == "disabled":
                with pytest.raises(ChunkCrcError):   # the stored CRCs are not the constant: every other part conflicts
                    call()
            else:
                call()
        finally:
            lib.lzgpu_set_crc_enabled(1)
        torch.cuda.synchronize()
        geo = e.last_geometry()
        assert geo["kernel"] == _lib.KERNEL_CORRECT_SLICES
        hf = dfix.cpu().numpy()
        assert (hf[:GUARD] == 0xEE).all() and (hf[GUARD + n * n_cs * 32:] == 0xEE).all()
        got = hf[GUARD:GUARD + n * n_cs * 32].view(FIX).reshape(n, n_cs)
        if crc_mode == "disabled":
            assert got[1, 1]["status"] == _lib.FIX_CRC_CONFLICT and (got["changed"] == 0).all()
            assert np.array_equal(got["bad_checks"], want["bad_checks"]) and np.array_equal(got["suspect_part"], want["suspect_part"])
        else:
            assert np.array_equal(got, want), crc_mode
        for g in bufs:
            hb = bufs[g].cpu().numpy()
            assert (hb[:OFF] == 0x77).all() and (hb[OFF + (n - 1) * pstride[sl[g]] + pb[sl[g]] * BLOCK:] == 0x77).all()
            hn = nbufs[g].cpu().numpy().view(np.uint32)
            assert (hn[:GUARD // 4] == SENTINEL).all() and (hn[GUARD // 4 + n * pb[sl[g]]:] == SENTINEL).all()
            for c in range(n):
                blk = hb[OFF + c * pstride[sl[g]]: OFF + c * pstride[sl[g]] + pb[sl[g]] * BLOCK]
                assert np.array_equal(blk, (sp if crc_mode == "disabled" else want_parts)[g][c]), (crc_mode, g, c)
                assert (hb[OFF + c * pstride[sl[g]] + pb[sl[g]] * BLOCK: OFF + (c + 1) * pstride[sl[g]]] == 0x77).all() or c == n - 1
            want_words = np.full((n, pb[sl[g]]), SENTINEL, dtype=np.uint32) if crc_mode == "disabled" else want_nc[g]
            assert np.array_equal(hn[GUARD // 4:GUARD // 4 + n * pb[sl[g]]].reshape(n, -1), want_words), (crc_mode, g)
    # refusals write nothing
    dfix = torch.full((64 * 32,), 0xEE, dtype=torch.uint8, device="cuda")
    bufs = {g: torch.from_numpy(sp[g]).cuda() for g in range(8)}
    ptrs = [bufs[g].data_ptr() for g in range(8)]
    nptrs = [0] * 8
    strides = [p * BLOCK for p in pb]
    before = e.stats()["kernel_launches"]
    for args, status in (((ptrs, strides, None, nptrs, None), _lib.ERR_ARG),                            # no fix
                         ((ptrs, strides, None, [2] + nptrs[1:], dfix.data_ptr()), _lib.ERR_ARG),        # new_crc not 4-byte aligned
                         ((ptrs, strides, None, nptrs, dfix.data_ptr() + 4), _lib.ERR_ARG),              # fix not 8-byte aligned
                         (([0] * 8, strides, None, nptrs, dfix.data_ptr()), _lib.ERR_TOO_FEW_PARTS)):    # no part
        with pytest.raises(LzGpuError) as ex:
            e.correct_slices_dev(goals, 2, nb, *args)
        assert ex.value.status == status
    torch.cuda.synchronize()
    assert e.stats()["kernel_launches"] == before and bool((dfix == 0xEE).all())
    assert all(np.array_equal(bufs[g].cpu().numpy(), sp[g]) for g in range(8))
    assert _lib.load().lzgpu_pool_correct_slices(None, None, 0, 0, 0, None, None, None, None, None, None) == _lib.ERR_ARG


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_host_form_copies_back_only_the_rewritten_blocks(ctx):
    e = engine(ctx)
    goals = goalset(("ec(3,2)", "ec(4,2)"))
    nb = 48
    _, parts, crcs = original(goals, 4, nb, 61)
    sp, sc = make_stale(goals, nb, parts, crcs, 3, [(1, 2), (3, 13)], 7)   # ec(3,2) parity 0: combined stripes 0 and 3
    before = e.stats()["bytes_d2h"]
    rc, fix, _, out, _ = correct(e, goals, nb, sp, sc)
    d2h = e.stats()["bytes_d2h"] - before
    assert rc == _lib.OK and (fix["status"] == _lib.FIX_CORRECTED).sum() == 2
    assert all(np.array_equal(a, b) for a, b in zip(out, parts))
    assert d2h <= 2 * 4 * BLOCK + fix.nbytes + 64 * 1024


@pytest.mark.parametrize("slots", [2, 3])
@pytest.mark.parametrize("n", [0, 1, 2, 7])
def test_pool_equals_one_context(slots, n):
    goals = goalset(("ec(3,2)", "ec(4,2)"))
    nb = 25
    _, parts, crcs = original(goals, max(n, 1), nb, 41)
    sp, sc = make_stale(goals, nb, parts, crcs, 8, [(max(n, 1) - 1, 1)], 2)   # stale in the last chunk
    bad_crcs = [x.copy() for x in sc]
    bad_crcs[1][0, 2] ^= 1                                                  # failing in the first
    pool = L.Pool([0] * slots)
    e = engine("default")
    try:
        for cr in (sc, bad_crcs):
            inp, inc = [p[:n] for p in sp], [c[:n] for c in cr]
            rc0, f0, b0, o0, n0 = correct(e, goals, nb, inp, inc)
            rc1, f1, b1, o1, n1 = correct(e, goals, nb, inp, inc, fn=lambda h, *a: pool.lib.lzgpu_pool_correct_slices(pool.h, *a))
            assert (rc0, b0) == (rc1, b1) and np.array_equal(f0, f1)
            assert all(np.array_equal(a, b) for a, b in zip(o0, o1)) and all(np.array_equal(a, b) for a, b in zip(n0, n1))
            if n and cr is sc:
                assert (f0["status"] == _lib.FIX_CORRECTED).any() and rc0 == _lib.OK
            elif n:   # with one chunk the failing block shares the stale combined stripe: a conflict there
                assert rc0 == _lib.ERR_CRC and ((f0["status"] == _lib.FIX_CORRECTED) | (f0["status"] == _lib.FIX_CRC_CONFLICT)).any()
    finally:
        pool.close()
