"""The consistency map of several slices (lzgpu_check_slices*, the CHECK instantiation of recover_slices_kernel and the locate pass in
csrc/recover_slices_kernel.cuh) on the GPU.

Inputs are encoded by lzgpu_encode_slices.  A stale part has chosen blocks rewritten with their stored CRCs recomputed.  Each map is
compared with numpy: bad_checks with the syndromes of lzgpu_debug_check_slices_rows evaluated over the blocks, suspect_part with a
span test written here (an annihilator of each part's columns, applied to the syndrome vector at every byte).  Covered: clean batches
of six goal sets at nb < L, a ragged nb and one 64 MiB chunk; a stale part at every part position of two goal sets, named where the
plan says locatable; a divergent standard copy; the one-goal case against lzgpu_check_stripe_map_degraded (equal, except that a last
stripe in which a lost data part's block is padding has one more check here); stored-CRC failures; the
_dev form with guard bytes, deferred verification, the CRC-disabled mode and the refusals; the launch report; pools of two and three
slots on one device.  Each case runs on the default context and with LZGPU_GRID_CAP=2."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200.engine import ChunkCrcError, LzGpuError, _goal_array, _p, _ptr_array
from tests.test_check_slices_plan import MUL, given_blocks
from tests.test_gpu_salvage_slices import original, to_dev
from tests.test_recover_slices_plan import EXP, LOG, goalset, layout, lcm_of

pytestmark = pytest.mark.gpu
BLOCK = 65536
SETS = [("std", "xor2"), ("std", "xor2", "xor3"), ("xor2", "xor3"), ("ec(3,2)", "ec(2,2)"), ("ec(3,2)", "ec(4,2)"), ("ec(5,5)", "xor2")]
_engines = {}


def engine(kind):
    env = {"default": {}, "cap2": {"LZGPU_GRID_CAP": "2"}}[kind]
    if kind not in _engines:
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            _engines[kind] = L.Engine(0)
        finally:
            for k, v in old.items():
                if v is None:
                    del os.environ[k]
                else:
                    os.environ[k] = v
    return _engines[kind]


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in _engines.values():
        e.close()
    _engines.clear()


def n_parts(goals):
    return layout(goals)[1]


def slice_of(goals):
    return [i for i, g in enumerate(goals) for _ in range(1 if g.is_std else g.k + g.m)]


def raw(e, goals, nb, parts, crcs):
    """lzgpu_check_slices: (code, map, bad[0..3])"""
    pbs = [-(-nb // (1 if g.is_std else g.k)) for g in goals]
    n = next(p.shape[0] for p in parts if p is not None)
    out = np.zeros((n, -(-nb // lcm_of(goals))), dtype=L.Engine.SLICES_CHECK_DTYPE)
    bad = (C.c_int64 * 4)(-1, -1, -1, -1)
    cr = None if crcs is None else _ptr_array([None if c is None else np.ascontiguousarray(c) for c in crcs])
    rc = e.lib.lzgpu_check_slices(e.h, _goal_array(goals), len(goals), n, nb, _ptr_array(parts),
                                  (C.c_size_t * len(goals))(*[pb * BLOCK for pb in pbs]), cr, _p(out), bad)
    return rc, out, tuple(bad)


def ginv(a):
    return EXP[255 - LOG[a]]


def annihilator(cols, nc):
    """rows w with w . c = 0 for every column c (lists of length nc): the null space of the matrix whose rows are the columns"""
    m = [list(c) for c in cols]
    piv, r = [], 0
    for c in range(nc):
        p = next((i for i in range(r, len(m)) if m[i][c]), None)
        if p is None:
            continue
        m[r], m[p] = m[p], m[r]
        inv = ginv(m[r][c])
        m[r] = [MUL[v, inv] for v in m[r]]
        for i in range(len(m)):
            if i != r and m[i][c]:
                f = m[i][c]
                m[i] = [v ^ MUL[f, w] for v, w in zip(m[i], m[r])]
        piv.append(c)
        r += 1
    out = []
    for f in range(nc):
        if f in piv:
            continue
        w = [0] * nc
        w[f] = 1
        for i, c in enumerate(piv):
            w[c] = int(m[i][f])
        out.append(w)
    return out


def expected_map(goals, nb, given, parts):
    """bad_checks and suspect_part of every combined stripe, from the debug rows and the span test, in numpy"""
    Lc = lcm_of(goals)
    sl = slice_of(goals)
    ks = [1 if g.is_std else g.k for g in goals]
    n = next(p.shape[0] for p in parts if p is not None)
    n_cs = -(-nb // Lc)
    out = np.zeros((n, n_cs), dtype=L.Engine.SLICES_CHECK_DTYPE)
    rows = {}
    for cs in range(n_cs):
        valid = min(Lc, nb - cs * Lc)
        if valid not in rows:
            part, stripe, coef = L.Engine.debug_check_slices_rows(goals, given, valid)
            blocks = [(g, s) for g, s, _ in given_blocks(goals, given, valid)]
            nc = len(part)
            ann = {g: annihilator([[int(coef[h, b[0], b[1]]) for h in range(nc)] for b in blocks if b[0] == g], nc)
                   for g in sorted({b[0] for b in blocks})}
            rows[valid] = (coef, blocks, nc, ann)
        coef, blocks, nc, ann = rows[valid]
        for c in range(n):
            S = np.zeros((nc, BLOCK), dtype=np.uint8)
            for g, s in blocks:
                blk = cs * (Lc // ks[sl[g]]) + s
                y = parts[g][c, blk * BLOCK:(blk + 1) * BLOCK]
                for h in range(nc):
                    if coef[h, g, s]:
                        S[h] ^= MUL[coef[h, g, s], y]
            bad = sum(1 << h for h in range(nc) if S[h].any())
            suspect = -1
            if bad:
                nz = S.any(axis=0)
                Sn = S[:, nz]
                fits = []
                for g, A in ann.items():
                    ok = True
                    for w in A:
                        acc = np.zeros(Sn.shape[1], dtype=np.uint8)
                        for h in range(nc):
                            if w[h]:
                                acc ^= MUL[w[h], Sn[h]]
                        if acc.any():
                            ok = False
                            break
                    if ok:
                        fits.append(g)
                suspect = fits[0] if len(fits) == 1 else -1
            out[c, cs] = (bad, suspect, 0)
    return out


def make_stale(goals, nb, parts, crcs, g, blocks, seed):
    """part g with `blocks` (chunk, part block) rewritten, its stored CRCs recomputed"""
    rng = np.random.default_rng(seed)
    p = parts[g].copy()
    for c, b in blocks:
        off = int(rng.integers(0, BLOCK - 64))
        p[c, b * BLOCK + off: b * BLOCK + off + 64] ^= rng.integers(1, 256, size=64, dtype=np.uint8)
    cr = crcs[g].copy()
    for c, b in blocks:
        cr[c, b] = zlib.crc32(p[c, b * BLOCK:(b + 1) * BLOCK].tobytes())
    parts, crcs = list(parts), list(crcs)
    parts[g], crcs[g] = p, cr
    return parts, crcs


def check_geometry(e, goals, nb, n, given):
    p = L.Engine.plan_check_slices(goals, nb, given)
    geo = e.last_geometry()
    assert geo["kernel"] == _lib.KERNEL_CHECK_SLICES
    assert (geo["G"], geo["threads"], geo["stages"], geo["smem_bytes"]) == (p["G"], p["threads"], p["stages"], p["smem_bytes"])
    upc = -(-(-(-nb // p["L"])) // p["G"])
    assert geo["units"] == upc * n
    if e is engine("cap2"):
        assert geo["grid"] <= 2


def nbs(Lc):
    return sorted({max(1, Lc - 1), 2 * Lc + max(1, Lc // 2), 3 * Lc})


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names", SETS, ids="+".join)
def test_clean_batches(names, ctx):
    e = engine(ctx)
    goals = goalset(names)
    n = n_parts(goals)
    for nb in nbs(lcm_of(goals)):
        data, parts, crcs = original(goals, 2, nb, nb)
        for given in ([1] * n, [1 if g % 3 else 0 for g in range(n)]):
            inp = [p if given[g] else None for g, p in enumerate(parts)]
            inc = [c if given[g] else None for g, c in enumerate(crcs)]
            p = L.Engine.plan_check_slices(goals, nb, given)
            if not (p["n_checks"] if nb >= p["L"] else 0) and not (p["tail_n_checks"] if p["tail_blocks"] else 0):
                continue
            rc, m, bad = raw(e, goals, nb, inp, inc)
            assert rc == _lib.OK and bad == (-1, -1, -1, -1), (names, nb, given)
            assert (m["bad_checks"] == 0).all() and (m["suspect_part"] == -1).all() and (m["zero"] == 0).all()
            check_geometry(e, goals, nb, 2, given)


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_clean_64mib_chunk(ctx):
    goals = goalset(("std", "xor2", "xor3"))
    data, parts, crcs = original(goals, 1, 1024, 5)
    rc, m, _ = raw(engine(ctx), goals, 1024, parts, crcs)
    assert rc == _lib.OK and m.shape == (1, 171) and (m["bad_checks"] == 0).all() and (m["suspect_part"] == -1).all()


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names", [("std", "xor2", "xor3"), ("ec(3,2)", "ec(4,2)")], ids="+".join)
def test_stale_part_at_every_position(names, ctx):
    e = engine(ctx)
    goals = goalset(names)
    n = n_parts(goals)
    Lc = lcm_of(goals)
    nb = 2 * Lc + Lc // 2
    sl = slice_of(goals)
    data, parts, crcs = original(goals, 2, nb, 11)
    for given in ([1] * n, [0 if g == n - 1 else 1 for g in range(n)]):
        plan = L.Engine.plan_check_slices(goals, nb, given)
        for g in range(n):
            if not given[g]:
                continue
            k = 1 if goals[sl[g]].is_std else goals[sl[g]].k
            spc = Lc // k
            # chunk 0: every block of g in combined stripe 1; chunk 1: one block in combined stripe 0 and the tail's first block
            j = g - sl.index(sl[g])   # the part's index in its slice
            blocks = [(0, spc + s) for s in range(spc)] + [(1, 0), (1, 2 * spc)]
            blocks = [(c, b) for c, b in blocks if (b * k + j if j < k else b * k) < nb]   # real blocks, not padding
            sp, sc = make_stale(goals, nb, parts, crcs, g, blocks, g)
            inp = [p if given[h] else None for h, p in enumerate(sp)]
            inc = [c if given[h] else None for h, c in enumerate(sc)]
            rc, m, bad = raw(e, goals, nb, inp, inc)
            want = expected_map(goals, nb, given, inp)
            assert np.array_equal(m, want), (names, given, g)
            assert rc == (_lib.ERR_INCONSISTENT if want["bad_checks"].any() else _lib.OK)
            assert bad == (-1, -1, -1, -1)
            if (plan["locatable"] >> g) & 1:
                assert (m[0, 1]["bad_checks"] != 0) and m[0, 1]["suspect_part"] == g
            if (plan["checked"] >> g) & 1:
                assert m[0, 1]["bad_checks"] != 0


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_divergent_standard_copy(ctx):
    goals = goalset(("std", "xor2"))
    nb = 9
    data, parts, crcs = original(goals, 1, nb, 4)
    sp, sc = make_stale(goals, nb, parts, crcs, 0, [(0, 3)], 1)   # block 3 of the standard copy: combined stripe 1, position 1
    rc, m, _ = raw(engine(ctx), goals, nb, sp, sc)
    assert rc == _lib.ERR_INCONSISTENT
    assert np.array_equal(m, expected_map(goals, nb, [1] * 4, sp))
    assert m[0, 1]["bad_checks"] != 0 and (np.delete(m["bad_checks"][0], 1) == 0).all()
    assert m[0, 1]["suspect_part"] == 0   # the copy disagrees with both the xor2 data part and the xor2 parity


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("name", ["ec(8,2)", "ec(5,3)", "ec(8,4)", "xor3"])
def test_one_goal_equals_the_degraded_stripe_map(name, ctx):
    e = engine(ctx)
    goal = L.SliceType(name)
    k, m_ = goal.k, goal.m
    rng = np.random.default_rng(k * 10 + m_)
    nb = 5 * k + 2
    pb = -(-nb // k)
    data, parts, crcs = original([goal], 2, nb, k)
    for trial in range(6):
        n_given = int(rng.integers(k + 1, k + m_ + 1))
        given_set = sorted(rng.choice(k + m_, size=n_given, replace=False).tolist())
        given = [1 if g in given_set else 0 for g in range(k + m_)]
        g = int(rng.choice(given_set))
        real = [b for b in range(pb) if g >= k or b * k + g < nb]
        blocks = [(int(rng.integers(0, 2)), int(b)) for b in rng.choice(real, size=min(3, len(real)), replace=False)]
        sp, sc = make_stale([goal], nb, parts, crcs, g, blocks, trial)
        inp = [p if given[h] else None for h, p in enumerate(sp)]
        inc = [c if given[h] else None for h, c in enumerate(sc)]
        _, mm, _ = raw(e, [goal], nb, inp, inc)
        ref = e.check_stripe_map_degraded(goal, nb, inp, inc)
        assert np.array_equal(mm["bad_checks"] != 0, ref["bad_rows"] != 0), (name, given, g)
        # the last stripe holds nb % k blocks; where a lost data part's block there is past the chunk's end, this call knows it is
        # zero (one more check) while the degraded map solves for it, so only there may it name the stale part where that map cannot
        padded_loss = any(not given[j] and j >= nb % k for j in range(k))
        assert np.array_equal(mm["suspect_part"][:, :-1], ref["suspect_part"][:, :-1]), (name, given, g)
        if padded_loss:
            same = mm["suspect_part"][:, -1] == ref["suspect_part"][:, -1]
            assert (same | ((ref["suspect_part"][:, -1] == -1) & (mm["suspect_part"][:, -1] == g))).all(), (name, given, g)
        else:
            assert np.array_equal(mm["suspect_part"][:, -1], ref["suspect_part"][:, -1]), (name, given, g)


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_stored_crc_failures(ctx):
    e = engine(ctx)
    goals = goalset(("ec(3,2)", "ec(4,2)"))
    nb = 30
    data, parts, crcs = original(goals, 3, nb, 8)
    bad_crcs = [c.copy() for c in crcs]
    bad_crcs[7][2, 1] ^= 1       # chunk 2, ec(4,2) data part 2, block 1
    bad_crcs[9][1, 4] ^= 1       # chunk 1, ec(4,2) parity part 0, block 4: the smallest
    rc, m, bad = raw(e, goals, nb, parts, bad_crcs)
    assert rc == _lib.ERR_CRC and bad == (1, 1, 4, 4)
    _, m0, _ = raw(e, goals, nb, parts, None)
    assert np.array_equal(m, m0) and (m["bad_checks"] == 0).all()
    sp, sc = make_stale(goals, nb, parts, bad_crcs, 2, [(0, 2)], 3)
    rc, m, bad = raw(e, goals, nb, sp, sc)
    _, m0, _ = raw(e, goals, nb, sp, None)
    assert rc == _lib.ERR_CRC and bad == (1, 1, 4, 4) and np.array_equal(m, m0)
    assert np.array_equal(m, expected_map(goals, nb, [1] * 11, sp))
    with pytest.raises(ChunkCrcError) as ex:
        e.check_slices(goals, nb, sp, sc)
    assert tuple(ex.value.where) == (1, 1, 4, 4) and np.array_equal(ex.value.map, m)


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("deferred", [False, True])
def test_dev_form_guard_bytes(ctx, deferred):
    e = engine(ctx)
    goals = goalset(("std", "xor2", "xor3"))
    n, nb = 2, 17
    given = [1, 1, 0, 1, 1, 1, 1, 1]
    data, parts, crcs = original(goals, n, nb, 21)
    sp, sc = make_stale(goals, nb, parts, crcs, 4, [(1, 2)], 5)
    sc[6] = sc[6].copy()
    sc[6][0, 3] ^= 1               # chunk 0, xor3 data part 1, block 3
    GUARD, OFF = 4096, 4096 + 48
    sl = slice_of(goals)
    pbs = [-(-nb // (1 if g.is_std else g.k)) for g in goals]
    pstride = [pb * BLOCK + 4096 for pb in pbs]
    bufs = {g: to_dev(sp[g], 0x77, GUARD, OFF, pstride[sl[g]]) for g in range(8) if given[g]}
    cbufs = {g: torch.from_numpy(sc[g].view(np.int32).copy()).cuda() for g in bufs}
    n_cs = -(-nb // 6)
    dmap = torch.full((GUARD + n * n_cs * 16 + GUARD,), 0xEE, dtype=torch.uint8, device="cuda")
    ptrs = [bufs[g].data_ptr() + OFF if g in bufs else 0 for g in range(8)]
    want = expected_map(goals, nb, given, [p if given[g] else None for g, p in enumerate(sp)])
    for crc_mode in ("verify", "none", "disabled"):
        dmap.fill_(0xEE)
        lib = _lib.load()
        cptrs = [cbufs[g].data_ptr() if g in cbufs else 0 for g in range(8)] if crc_mode != "none" else None
        if crc_mode == "disabled":
            lib.lzgpu_set_crc_enabled(0)
        try:
            if crc_mode == "verify" and deferred:
                e.set_deferred_verify(True)
                try:
                    e.check_slices_dev(goals, n, nb, ptrs, pstride, cptrs, dmap.data_ptr() + GUARD)
                    with pytest.raises(ChunkCrcError) as ex:
                        e.sync()
                    assert tuple(ex.value.where) == (0, 6, 3)
                finally:
                    e.set_deferred_verify(False)
            elif crc_mode == "verify":
                with pytest.raises(ChunkCrcError) as ex:
                    e.check_slices_dev(goals, n, nb, ptrs, pstride, cptrs, dmap.data_ptr() + GUARD)
                assert tuple(ex.value.where) == (0, 2, 2, 3)
            elif crc_mode == "disabled":
                with pytest.raises(ChunkCrcError):   # the stored CRCs are not the constant
                    e.check_slices_dev(goals, n, nb, ptrs, pstride, cptrs, dmap.data_ptr() + GUARD)
            else:
                e.check_slices_dev(goals, n, nb, ptrs, pstride, cptrs, dmap.data_ptr() + GUARD)
        finally:
            lib.lzgpu_set_crc_enabled(1)
        torch.cuda.synchronize()
        check_geometry(e, goals, nb, n, given)
        hm = dmap.cpu().numpy()
        assert (hm[:GUARD] == 0xEE).all() and (hm[GUARD + n * n_cs * 16:] == 0xEE).all()
        got = hm[GUARD:GUARD + n * n_cs * 16].view(L.Engine.SLICES_CHECK_DTYPE).reshape(n, n_cs)
        assert np.array_equal(got, want), crc_mode
        assert got[1, 1]["bad_checks"] != 0
    for g in bufs:   # inputs untouched
        assert np.array_equal(bufs[g][OFF:OFF + pbs[sl[g]] * BLOCK].cpu().numpy(), sp[g][0])
    # misaligned pointers
    for bad_args in (dict(map_off=4), dict(part_off=8), dict(crc_off=2)):
        p2 = list(ptrs)
        if "part_off" in bad_args:
            p2[0] += bad_args["part_off"]
        c2 = [cbufs[g].data_ptr() + bad_args.get("crc_off", 0) if g in cbufs else 0 for g in range(8)]
        with pytest.raises(LzGpuError) as ex:
            e.check_slices_dev(goals, n, nb, p2, pstride, c2, dmap.data_ptr() + GUARD + bad_args.get("map_off", 0))
        assert ex.value.status == _lib.ERR_ARG


def test_refusals_write_nothing():
    e = engine("default")
    lib = _lib.load()
    goals = goalset(("xor2", "xor3"))
    nb = 7
    data, parts, crcs = original(goals, 1, nb, 1)
    dmap = torch.full((64,), 0xEE, dtype=torch.uint8, device="cuda")
    before = e.stats()["kernel_launches"]
    with pytest.raises(LzGpuError) as ex:   # no part given
        e.check_slices_dev(goals, 1, nb, [0] * 7, [4 * BLOCK, 3 * BLOCK], None, dmap.data_ptr())
    assert ex.value.status == _lib.ERR_TOO_FEW_PARTS
    with pytest.raises(LzGpuError) as ex:   # no stripe shape has a check: the xor2 data parts alone
        e.check_slices(goals, nb, [parts[0], parts[1], None, None, None, None, None])
    assert ex.value.status == _lib.ERR_TOO_FEW_PARTS
    d_parts = [torch.from_numpy(p).cuda() for p in parts]
    ptrs = [t.data_ptr() for t in d_parts]
    with pytest.raises(LzGpuError) as ex:   # no map
        e.check_slices_dev(goals, 1, nb, ptrs, [4 * BLOCK, 3 * BLOCK], None, None)
    assert ex.value.status == _lib.ERR_ARG
    with pytest.raises(LzGpuError) as ex:   # a repeated slice type
        e.check_slices(goalset(("xor2", "xor2")), nb, parts[:3] + parts[:3])
    assert ex.value.status == _lib.ERR_ARG
    big = goalset(("std", "ec(8,4)", "ec(3,4)"))   # 92 checks
    assert L.Engine.plan_check_slices(big, 48, [1] * 20)["ok"] == 0
    buf = torch.zeros(48 * BLOCK, dtype=torch.uint8, device="cuda")
    with pytest.raises(LzGpuError) as ex:
        e.check_slices_dev(big, 1, 48, [buf.data_ptr()] * 20, [48 * BLOCK, 6 * BLOCK, 16 * BLOCK], None, dmap.data_ptr())
    assert ex.value.status == _lib.ERR_ARG
    torch.cuda.synchronize()
    assert e.stats()["kernel_launches"] == before
    assert bool((dmap == 0xEE).all())
    assert lib.lzgpu_pool_check_slices(None, None, 0, 0, 0, None, None, None, None, None) == _lib.ERR_ARG


@pytest.mark.parametrize("slots", [2, 3])
@pytest.mark.parametrize("n", [0, 1, 2, 7])
def test_pool_equals_one_context(slots, n):
    goals = goalset(("ec(3,2)", "ec(4,2)"))
    nb = 25
    data, parts, crcs = original(goals, max(n, 1), nb, 41)
    sp, sc = make_stale(goals, nb, parts, crcs, 8, [(max(n, 1) - 1, 1)], 2)   # stale in the last chunk
    bad_crcs = [x.copy() for x in sc]
    bad_crcs[1][0, 2] ^= 1                                                  # failing in the first
    inp = [p[:n] for p in sp]
    pool = L.Pool([0] * slots)
    try:
        for cr in (sc, bad_crcs):
            incrc = [x[:n] for x in cr]
            res = []
            for fn in (engine("default").check_slices, pool.check_slices):
                try:
                    res.append((None, fn(goals, nb, inp, incrc)))
                except ChunkCrcError as ex:
                    res.append((tuple(ex.where), ex.map))
                except LzGpuError as ex:
                    res.append((ex.status, None))
            (w0, a), (w1, b) = res
            assert w0 == w1
            assert (a is None and b is None) or np.array_equal(a, b)
            if n and a is not None:
                assert np.array_equal(a, expected_map(goals, nb, [1] * 11, inp))
    finally:
        pool.close()
