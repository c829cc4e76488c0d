"""lzgpu_check_slices, lzgpu_correct_slices and lzgpu_salvage_slices at the limits of their tables, on the GPU.

The rows are those of tests/test_slices_check_edges.py, whose plan values are checked there against the rank models: 64 checks with
bit 63 of bad_checks, 64 candidate parts with a suspect at flat part 63, L = 62 and 63, a 62-block correction near the correct
kernel's shared-memory attribute, 192 salvage streams, failing read entries in words 4 and 5 of the salvage mask.  Every case runs on
the default context and with LZGPU_GRID_CAP=2.  Every expected byte is the random original data or the oracle's encode_chunk
(Original of tests/test_gpu_recover_slices_edges.py), every expected CRC zlib.crc32; bad_checks is the debug check rows applied in
numpy to the bytes a case changed (the original is a codeword); the launch report is checked against the plan.  Row E's tail holds
no block of flat parts 24..35: a rewritten block of part 24 there is padding, which no check reads, so the entry is CLEAN and the
block is left as it is."""
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200.engine import ChunkCrcError, LzGpuError
from tests import _oracle as O
from tests.test_check_slices_plan import MUL
from tests.test_gpu_check_slices import engine, make_stale, raw
from tests.test_gpu_correct_slices import SENTINEL, check_result, correct, written_blocks
from tests.test_gpu_recover_slices_edges import Original
from tests.test_gpu_salvage_slices import ZERO_CRC, check, corrupt_and_check, dependents, to_dev
from tests.test_slices_check_edges import EDGE, SALVAGE, given_of

pytestmark = pytest.mark.gpu
BLOCK = 65536
CTX = ["default", "cap2"]
KNOWN, SOLVED = _lib.SALVAGE_KNOWN, _lib.SALVAGE_SOLVED
GUARD, OFF = 4096, 4096 + 48


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    from tests import test_gpu_check_slices as T, test_gpu_salvage_slices as S
    for mod in (T, S):
        for e in mod._engines.values():
            e.close()
        mod._engines.clear()


_orig = {}


def original(names, n, nb, seed):
    key = (names, n, nb, seed)
    if key not in _orig:
        _orig.clear()
        _orig[key] = Original(O.load_oracle(), names, n, nb, seed)
    return _orig[key]


def inputs(o, given, parts=None, crcs=None):
    parts, crcs = parts or o.parts, crcs or o.crcs
    return [p if given[g] else None for g, p in enumerate(parts)], [c if given[g] else None for g, c in enumerate(crcs)]


_rows = {}


def debug_rows(o, given, valid):
    key = (o.names, tuple(given), valid)
    if key not in _rows:
        _rows[key] = L.Engine.debug_check_slices_rows(o.goals, given, valid)
    return _rows[key]


def expected_bad(o, given, before, after, c, cs):
    """bad_checks of combined stripe cs of chunk c: the debug rows applied to the bytes that differ between before (a codeword) and
    after"""
    Lc, nb = o.L, o.nb
    valid = min(Lc, nb - cs * Lc)
    part, stripe, coef = debug_rows(o, given, valid)
    deltas = {}
    for g in range(o.n_parts):
        if not given[g] or before[g] is after[g]:
            continue
        k = o.lay[o.slice_of[g]][0]
        for s in range(Lc // k):
            b = cs * (Lc // k) + s
            d = before[g][c, b * BLOCK:(b + 1) * BLOCK] ^ after[g][c, b * BLOCK:(b + 1) * BLOCK]
            if d.any():
                deltas[(g, s)] = d
    if not deltas:
        return 0
    nz = np.nonzero(np.any(np.stack(list(deltas.values())), axis=0))[0]
    bad = 0
    for h in range(len(part)):
        syn = np.zeros(nz.size, dtype=np.uint8)
        for (g, s), d in deltas.items():
            if coef[h, g, s]:
                syn ^= MUL[coef[h, g, s], d[nz]]
        if syn.any():
            bad |= 1 << h
    return bad


def check_geometry(e, ctx, o, given, kernel):
    p = (L.Engine.plan_salvage_slices if kernel == _lib.KERNEL_SALVAGE_SLICES else L.Engine.plan_check_slices)(o.goals, o.nb, given)
    geo = e.last_geometry()
    assert geo["kernel"] == kernel
    assert (geo["threads"], geo["smem_bytes"]) == (p["threads"], p["smem_bytes"])
    if kernel != _lib.KERNEL_CORRECT_SLICES:
        assert (geo["G"], geo["stages"]) == (p["G"], p["stages"])
        assert geo["units"] % -(-(-(-o.nb // p["L"])) // p["G"]) == 0
    if ctx == "cap2":
        assert geo["grid"] <= 2


def run_correct(e, ctx, o, given, parts, crcs, want_corrected=None):
    """lzgpu_check_slices then lzgpu_correct_slices on parts: the map equals the numpy syndromes, every entry follows the rule, and
    the corrected parts equal the originals.  Returns (rc, fix, bad, out, new CRCs)"""
    inp, inc = inputs(o, given, parts, crcs)
    rc0, m, _ = raw(e, o.goals, o.nb, inp, inc)
    check_geometry(e, ctx, o, given, _lib.KERNEL_CHECK_SLICES)
    for c in range(o.n):
        for cs in range(m.shape[1]):
            assert int(m[c, cs]["bad_checks"]) == expected_bad(o, given, o.parts, parts, c, cs), (o.names, c, cs)
    rc, fix, bad, out, nc = correct(e, o.goals, o.nb, inp, inc)
    check_geometry(e, ctx, o, given, _lib.KERNEL_CORRECT_SLICES)
    assert np.array_equal(fix["bad_checks"], m["bad_checks"]) and np.array_equal(fix["suspect_part"], m["suspect_part"])
    check_result(e, o.goals, o.nb, given, inp, out, inc, fix, nc, orig=o.parts)
    if want_corrected is not None:
        assert sorted(zip(*np.nonzero(fix["status"] == _lib.FIX_CORRECTED))) == sorted(want_corrected)
    return rc, fix, bad, out, nc


def assert_changed(fix, before, after, o, g, c, cs):
    """changed is exactly the blocks of g that differed before the correction"""
    k = o.lay[o.slice_of[g]][0]
    spc = o.L // k
    ch = 0
    for b in written_blocks(o.goals, o.nb, g, cs):
        if not np.array_equal(before[g][c, b * BLOCK:(b + 1) * BLOCK], after[g][c, b * BLOCK:(b + 1) * BLOCK]):
            ch |= 1 << (b - cs * spc)
    assert int(fix[c, cs]["changed"]) == ch
    return ch


# ------------------------------------------------------------------------------------------------------------------------------
# A: ec(8,8) + ec(16,32), all 64 parts, one 64 MiB chunk of 64 combined stripes
# ------------------------------------------------------------------------------------------------------------------------------
def stale_blocks(o, g, c, cs):
    """every real block of flat part g in combined stripe cs of chunk c"""
    return [(c, b) for b in written_blocks(o.goals, o.nb, g, cs)]


@pytest.mark.parametrize("ctx", CTX)
def test_a_64_checks_and_64_candidates(ctx):
    e = engine(ctx)
    names = EDGE["A"][1]
    o = original(names, 1, 1024, 64)
    given = [1] * 64
    # clean
    inp, inc = inputs(o, given)
    rc, m, bad = raw(e, o.goals, 1024, inp, inc)
    assert rc == _lib.OK and bad == (-1, -1, -1, -1) and m.shape == (1, 64)
    assert (m["bad_checks"] == 0).all() and (m["suspect_part"] == -1).all() and (m["zero"] == 0).all()
    rc, fix, bad, out, nc = correct(e, o.goals, 1024, inp, inc)
    assert rc == _lib.OK and (fix["status"] == _lib.FIX_CLEAN).all() and (fix["changed"] == 0).all() and (fix["crc_failed"] == 0).all()
    assert all(np.array_equal(a, b) for a, b in zip(out, o.parts)) and all((x == SENTINEL).all() for x in nc)
    # stale part g in combined stripe g, g = 0 .. 63, in one call
    sp, sc = o.parts, o.crcs
    for g in range(64):
        sp, sc = make_stale(o.goals, 1024, sp, sc, g, stale_blocks(o, g, 0, g), g)
    rc, fix, bad, out, nc = run_correct(e, ctx, o, given, sp, sc, want_corrected=[(0, g) for g in range(64)])
    assert rc == _lib.OK and bad == (-1, -1, -1, -1)
    assert list(fix[0]["suspect_part"]) == list(range(64))
    assert all(np.array_equal(a, b) for a, b in zip(out, o.parts))
    for g in range(64):
        assert assert_changed(fix, sp, o.parts, o, g, 0, g) != 0
        for _, b in stale_blocks(o, g, 0, g):
            assert nc[g][0, b] == o.crcs[g][0, b]
    # the defining block of check h stale in combined stripe h: bad_checks = 1 << h
    part, stripe, coef = debug_rows(o, given, 16)
    assert len(part) == 64
    sp, sc = o.parts, o.crcs
    for h in range(64):
        g, s = int(part[h]), int(stripe[h])
        spc = o.L // o.lay[o.slice_of[g]][0]
        sp, sc = make_stale(o.goals, 1024, sp, sc, g, [(0, h * spc + s)], 100 + h)
    rc, m, _ = raw(e, o.goals, 1024, *inputs(o, given, sp, sc))
    assert rc == _lib.ERR_INCONSISTENT
    assert [int(x) for x in m[0]["bad_checks"]] == [1 << h for h in range(64)]
    for h in range(64):
        assert int(m[0, h]["bad_checks"]) == expected_bad(o, given, o.parts, sp, 0, h)
    assert m[0, 63]["suspect_part"] == part[63]
    # beside a stale part 5 in combined stripe 3, block 3 of part 63 fails its stored CRC: with its bytes intact part 5 is named and
    # the entry is a conflict; with its bytes rotten (stored CRC kept) two parts differ and no part explains the stripe.  Either way
    # crc_failed has bit 63, nothing is written, and the call reports part 63's block
    stale, stale_crc = make_stale(o.goals, 1024, o.parts, o.crcs, 5, stale_blocks(o, 5, 0, 3), 7)
    for kind, status in (("crc", _lib.FIX_CRC_CONFLICT), ("bytes", _lib.FIX_UNEXPLAINED)):
        sp, sc = list(stale), list(stale_crc)
        if kind == "crc":
            sc[63] = o.crcs[63].copy()
            sc[63][0, 3] ^= 1
        else:
            sp[63] = o.parts[63].copy()
            sp[63][0, 3 * BLOCK + 999] ^= 0x24
        rc, fix, bad, out, nc = correct(e, o.goals, 1024, *inputs(o, given, sp, sc))
        assert rc == _lib.ERR_CRC and bad == (0, 1, 47, 3)
        f = fix[0, 3]
        assert f["status"] == status and int(f["crc_failed"]) == 1 << 63 and f["changed"] == 0, kind
        assert f["suspect_part"] == (5 if kind == "crc" else -1)
        assert (np.delete(fix[0]["status"], 3) == _lib.FIX_CLEAN).all()
        assert all(np.array_equal(a, b) for a, b in zip(out, sp)) and all((x == SENTINEL).all() for x in nc)


def dev_correct(e, o, given, sp, sc):
    """lzgpu_correct_slices_dev at padded strides with guard bytes: (fix, parts, new CRCs), the guards checked"""
    n, nb = o.n, o.nb
    pstride = [pb * BLOCK + 4096 + 16 * i for i, pb in enumerate(o.pbs)]
    bufs = {g: to_dev(sp[g], 0x77, GUARD, OFF, pstride[o.slice_of[g]]) for g in range(o.n_parts) if given[g]}
    cbufs = {g: torch.from_numpy(sc[g].view(np.int32).copy()).cuda() for g in bufs}
    nbufs = {g: torch.full((2 * GUARD // 4 + n * o.pbs[o.slice_of[g]],), SENTINEL - 2 ** 32, dtype=torch.int32, device="cuda")
             for g in bufs}
    n_cs = -(-nb // o.L)
    dfix = torch.full((2 * GUARD + n * n_cs * 32,), 0xEE, dtype=torch.uint8, device="cuda")
    e.correct_slices_dev(o.goals, n, nb, [bufs[g].data_ptr() + OFF if g in bufs else 0 for g in range(o.n_parts)], pstride,
                         [cbufs[g].data_ptr() if g in cbufs else 0 for g in range(o.n_parts)],
                         [nbufs[g].data_ptr() + GUARD if g in nbufs else 0 for g in range(o.n_parts)], dfix.data_ptr() + GUARD)
    torch.cuda.synchronize()
    hf = dfix.cpu().numpy()
    assert (hf[:GUARD] == 0xEE).all() and (hf[GUARD + n * n_cs * 32:] == 0xEE).all()
    fix = hf[GUARD:GUARD + n * n_cs * 32].view(L.Engine.SLICES_FIX_DTYPE).reshape(n, n_cs)
    parts, ncs = [None] * o.n_parts, [None] * o.n_parts
    for g in bufs:
        i = o.slice_of[g]
        size = o.pbs[i] * BLOCK
        hb = bufs[g].cpu().numpy()
        assert (hb[:OFF] == 0x77).all() and (hb[OFF + (n - 1) * pstride[i] + size:] == 0x77).all(), g
        for c in range(n - 1):
            assert (hb[OFF + c * pstride[i] + size: OFF + (c + 1) * pstride[i]] == 0x77).all(), g
        parts[g] = np.stack([hb[OFF + c * pstride[i]: OFF + c * pstride[i] + size] for c in range(n)])
        hn = nbufs[g].cpu().numpy().view(np.uint32)
        g0 = GUARD // 4
        assert (hn[:g0] == SENTINEL).all() and (hn[g0 + n * o.pbs[i]:] == SENTINEL).all(), g
        ncs[g] = hn[g0:g0 + n * o.pbs[i]].reshape(n, -1)
    return fix, parts, ncs


@pytest.mark.parametrize("ctx", CTX)
def test_a_dev_form(ctx):
    e = engine(ctx)
    o = original(EDGE["A"][1], 1, 1024, 64)
    given = [1] * 64
    sp, sc = o.parts, o.crcs
    for g in (0, 31, 47, 63):
        sp, sc = make_stale(o.goals, 1024, sp, sc, g, stale_blocks(o, g, 0, g), g)
    _, want, _, want_parts, want_nc = correct(engine("default"), o.goals, 1024, *inputs(o, given, sp, sc))
    fix, parts, ncs = dev_correct(e, o, given, sp, sc)
    assert np.array_equal(fix, want)
    assert [int(fix[0, g]["suspect_part"]) for g in (0, 31, 47, 63)] == [0, 31, 47, 63]
    assert all(np.array_equal(a, b) for a, b in zip(parts, o.parts))
    assert all(np.array_equal(a, b) for a, b in zip(ncs, want_nc))


# ------------------------------------------------------------------------------------------------------------------------------
# B: ec(7,3) + ec(9,4) with parts 0, 1, 2, 3, 5 and 9 lost: L = 63, 64 checks
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctx", CTX)
@pytest.mark.parametrize("nb", [126, 125, 40])
def test_b_every_locatable_part_at_l63(nb, ctx):
    e = engine(ctx)
    _, names, spec = EDGE["B"][:3]
    given = given_of(names, spec)
    o = original(names, 3, nb, 63)
    p = L.Engine.plan_correct_slices(o.goals, nb, given)
    n_cs = -(-nb // o.L)
    slots = [(c, cs) for c in range(3) for cs in range(n_cs)]
    rng = np.random.default_rng(nb)
    todo = [g for g in range(o.n_parts) if given[g]]
    for g in todo:
        tail = nb % o.L
        assert (p["tail_locatable"] if tail else p["locatable"]) >> g & 1 and (p["locatable"] >> g) & 1
    while todo:
        batch, todo = todo[:len(slots)], todo[len(slots):]
        sp, sc = o.parts, o.crcs
        for g, (c, cs) in zip(batch, slots):
            blks = written_blocks(o.goals, nb, g, cs)
            sp, sc = make_stale(o.goals, nb, sp, sc, g, [(c, int(rng.choice(blks)))], g)
        rc, fix, bad, out, nc = run_correct(e, ctx, o, given, sp, sc, want_corrected=slots[:len(batch)])
        assert rc == _lib.OK and bad == (-1, -1, -1, -1)
        for g, (c, cs) in zip(batch, slots):
            assert fix[c, cs]["suspect_part"] == g and bin(assert_changed(fix, sp, o.parts, o, g, c, cs)).count("1") == 1
        assert all(np.array_equal(a, b) for a, b in zip(out, o.parts) if a is not None)
    # two stale parts in one stripe: no part explains it, nothing written
    sp, sc = make_stale(o.goals, nb, o.parts, o.crcs, 4, [(1, written_blocks(o.goals, nb, 4, 0)[0])], 1)
    sp, sc = make_stale(o.goals, nb, sp, sc, 22, [(1, written_blocks(o.goals, nb, 22, 0)[0])], 2)
    rc, fix, _, out, nc = run_correct(e, ctx, o, given, sp, sc, want_corrected=[])
    assert rc == _lib.ERR_INCONSISTENT and fix[1, 0]["status"] == _lib.FIX_UNEXPLAINED and fix[1, 0]["suspect_part"] == -1
    assert all(a is None or np.array_equal(a, b) for a, b in zip(out, sp)) and all(x is None or (x == SENTINEL).all() for x in nc)


# ------------------------------------------------------------------------------------------------------------------------------
# C: std + ec(31,1) + ec(2,1), ec(2,1) lost: L = 62, a 62-block std correction
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctx", CTX)
def test_c_whole_std_copy(ctx):
    e = engine(ctx)
    _, names, spec = EDGE["C"][:3]
    given = given_of(names, spec)
    for nb, cs, full in ((992, 3, (1 << 62) - 1), (1007, 16, (1 << 15) - 1)):
        o = original(names, 1, nb, 62)
        n_blk = bin(full).count("1")
        sp, sc = make_stale(o.goals, nb, o.parts, o.crcs, 0, [(0, cs * 62 + s) for s in range(n_blk)], 3)
        rc, fix, bad, out, nc = run_correct(e, ctx, o, given, sp, sc, want_corrected=[(0, cs)])
        f = fix[0, cs]
        assert rc == _lib.OK and f["suspect_part"] == 0 and int(f["changed"]) == full
        assert np.array_equal(out[0], o.parts[0])
        assert np.array_equal(nc[0][0, cs * 62: cs * 62 + n_blk], o.crcs[0][0, cs * 62: cs * 62 + n_blk])
        assert (np.delete(nc[0][0], np.arange(cs * 62, cs * 62 + n_blk)) == SENTINEL).all()
        fixd, parts, ncs = dev_correct(e, o, given, sp, sc)
        assert np.array_equal(fixd, fix)
        assert all(a is None or np.array_equal(a, b) for a, b in zip(parts, o.parts))
        assert all(a is None or np.array_equal(a, b) for a, b in zip(ncs, nc))


# ------------------------------------------------------------------------------------------------------------------------------
# D: std + ec(32,31), all 64 parts, 63 checks
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctx", CTX)
def test_d_std_copy_and_part_63(ctx):
    e = engine(ctx)
    names = EDGE["D"][1]
    o = original(names, 1, 72, 32)          # two full combined stripes and the 8-block tail of nb = 1000
    given = [1] * 64
    sp, sc = make_stale(o.goals, 72, o.parts, o.crcs, 0, [(0, s) for s in range(32)], 4)
    sp, sc = make_stale(o.goals, 72, sp, sc, 63, [(0, 1)], 5)
    sp, sc = make_stale(o.goals, 72, sp, sc, 63, [(0, 2)], 6)
    rc, fix, bad, out, nc = run_correct(e, ctx, o, given, sp, sc, want_corrected=[(0, 0), (0, 1), (0, 2)])
    assert rc == _lib.OK and list(fix[0]["suspect_part"]) == [0, 63, 63]
    assert [int(x) for x in fix[0]["changed"]] == [(1 << 32) - 1, 1, 1]
    assert all(np.array_equal(a, b) for a, b in zip(out, o.parts))


# ------------------------------------------------------------------------------------------------------------------------------
# E: xor5 + ec(30,28), all 64 parts, the 18-block tail
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctx", CTX)
def test_e_part_24_in_the_tail_and_in_a_full_stripe(ctx):
    e = engine(ctx)
    names = EDGE["E"][1]
    o = original(names, 1, 78, 30)           # two full combined stripes and the 18-block tail of nb = 1008
    given = [1] * 64
    assert written_blocks(o.goals, 78, 24, 2) == []
    # block 2 of part 24 is position 2 * 30 + 18 = 78: padding
    sp, sc = make_stale(o.goals, 78, o.parts, o.crcs, 24, [(0, 2)], 8)
    rc, fix, bad, out, nc = run_correct(e, ctx, o, given, sp, sc, want_corrected=[])
    assert rc == _lib.OK and (fix["status"] == _lib.FIX_CLEAN).all()
    assert np.array_equal(out[24], sp[24]) and (nc[24] == SENTINEL).all()
    sp, sc = make_stale(o.goals, 78, sp, sc, 24, [(0, 1)], 9)
    rc, fix, bad, out, nc = run_correct(e, ctx, o, given, sp, sc, want_corrected=[(0, 1)])
    assert rc == _lib.OK and fix[0, 1]["suspect_part"] == 24 and fix[0, 1]["changed"] == 1
    assert np.array_equal(out[24][0, :2 * BLOCK], o.parts[24][0, :2 * BLOCK]) and np.array_equal(out[24][0, 2 * BLOCK:], sp[24][0, 2 * BLOCK:])


# ------------------------------------------------------------------------------------------------------------------------------
# salvage: F (192 streams), G (mask words 4 and 5), H (L = 63 from parity)
# ------------------------------------------------------------------------------------------------------------------------------
def salvage(e, ctx, o, given, parts=None, crcs=None):
    inp, inc = inputs(o, given, parts, crcs)
    img, icrc, smap = e.salvage_slices(o.goals, o.nb, inp, inc)
    check_geometry(e, ctx, o, given, _lib.KERNEL_SALVAGE_SLICES)
    return img, icrc, smap


@pytest.mark.parametrize("ctx", CTX)
def test_f_192_streams_and_one_past(ctx):
    e = engine(ctx)
    _, names, spec = SALVAGE["F"][:3]
    given = given_of(names, spec)
    o = original(names, 1, 1008, 48)
    img, icrc, smap = salvage(e, ctx, o, given)
    check(o.goals, 1008, given, o.data, img, icrc, smap)
    assert (smap == KNOWN).all()
    # parts 0 .. 22: 195 streams, refused with nothing launched or written
    over = given_of(names, SALVAGE["F_over"][2])
    assert L.Engine.plan_salvage_slices(o.goals, 1008, over)["ok"] == 0
    before = e.stats()["kernel_launches"]
    d_parts = {g: torch.from_numpy(o.parts[g]).cuda() for g in range(o.n_parts) if over[g]}
    dimg = torch.full((1008 * BLOCK,), 0x3C, dtype=torch.uint8, device="cuda")
    dmap = torch.full((1008,), 0xEE, dtype=torch.uint8, device="cuda")
    with pytest.raises(LzGpuError) as ex:
        e.salvage_slices_dev(o.goals, 1, 1008, [d_parts[g].data_ptr() if g in d_parts else 0 for g in range(o.n_parts)],
                             [pb * BLOCK for pb in o.pbs], None, dimg.data_ptr(), 1008 * BLOCK, None, dmap.data_ptr())
    assert ex.value.status == _lib.ERR_ARG
    with pytest.raises(LzGpuError) as ex:
        e.salvage_slices(o.goals, 1008, *inputs(o, over))
    assert ex.value.status == _lib.ERR_ARG
    torch.cuda.synchronize()
    assert e.stats()["kernel_launches"] == before
    assert bool((dimg == 0x3C).all()) and bool((dmap == 0xEE).all())


def rotten(o, g, c, blk, at=4321):
    parts = list(o.parts)
    parts[g] = o.parts[g].copy()
    parts[g][c, blk * BLOCK + at] ^= 0x5A
    return parts


@pytest.mark.parametrize("ctx", CTX)
def test_g_std_blocks_in_mask_words_4_and_5(ctx):
    e = engine(ctx)
    _, names, spec = SALVAGE["G"][:3]
    nb = 17                                   # two full combined stripes of L = 6 and a 5-block tail
    o = original(names, 2, nb, 6)
    # the data parts lost: the std blocks (read entries 146 .. 151) are the only staged copies
    given = given_of(names, spec)
    img, icrc, smap = salvage(e, ctx, o, given)
    check(o.goals, nb, given, o.data, img, icrc, smap)
    assert (smap == KNOWN).all()
    for blk in (8, 16):                       # position 2 of combined stripe 1; the tail's last block
        parts = rotten(o, 63, 1, blk)
        with pytest.raises(ChunkCrcError) as ex:
            e.salvage_slices(o.goals, nb, *inputs(o, given, parts))
        assert tuple(ex.value.where) == (1, 2, 0, blk)
        check(o.goals, nb, given, o.data, ex.value.image, ex.value.image_crc, ex.value.map, withheld=[(1, blk)])
        assert ex.value.image_crc[1, blk] == ZERO_CRC and not ex.value.image[1, blk * BLOCK:(blk + 1) * BLOCK].any()
    # two rotten blocks: reported at the smaller (chunk, slice, part, block); a parity block only verified withholds nothing
    parts = rotten(o, 63, 1, 8)
    parts[10] = o.parts[10].copy()
    parts[10][0, 2 * BLOCK + 5] ^= 1           # ec(2,30) parity part 8, block 2 of chunk 0
    with pytest.raises(ChunkCrcError) as ex:
        e.salvage_slices(o.goals, nb, *inputs(o, given, parts))
    assert tuple(ex.value.where) == (0, 0, 10, 2)
    check(o.goals, nb, given, o.data, ex.value.image, ex.value.image_crc, ex.value.map, withheld=[(1, 8)])
    # every part given: the std blocks are read entries 158 .. 163, only verified; blocks 2 .. 5 sit in word 5
    given = given_of(names, "all")
    for blk in (2, 5, 14):
        parts = rotten(o, 63, 1, blk)
        parts[63][0, (blk + 1) * BLOCK + 7] ^= 1  # and in chunk 0, one block later: reported first
        with pytest.raises(ChunkCrcError) as ex:
            e.salvage_slices(o.goals, nb, *inputs(o, given, parts))
        assert tuple(ex.value.where) == (0, 2, 0, blk + 1)
        check(o.goals, nb, given, o.data, ex.value.image, ex.value.image_crc, ex.value.map)
        check_geometry(e, ctx, o, given, _lib.KERNEL_SALVAGE_SLICES)


@pytest.mark.parametrize("ctx", CTX)
def test_h_position_44_from_parity(ctx):
    e = engine(ctx)
    _, names, spec = SALVAGE["H"][:3]
    given = given_of(names, spec)
    o = original(names, 1, 126, 44)
    img, icrc, smap = salvage(e, ctx, o, given)
    check(o.goals, 126, given, o.data, img, icrc, smap)
    assert [b for b in range(126) if smap[0, b] == SOLVED] == [44, 107] and not (smap == KNOWN).any()
    deps, unk, ne, es, er, est, rows = dependents(o.goals, given, 63)
    read = max(r for r, d in deps.items() if 44 in d)      # a parity block 44's row uses: only 44 is determined, so only it is withheld
    corrupt_and_check(e, o.goals, 126, 1, given, o.data, o.parts, o.crcs, 0, 1, read, {44})
    # the 62-block tail is wholly determined
    o = original(names, 2, 62, 62)
    img, icrc, smap = salvage(e, ctx, o, given)
    check(o.goals, 62, given, o.data, img, icrc, smap)
    assert np.array_equal(img, o.data) and (smap == SOLVED).all()
    for c in range(2):
        assert [int(x) for x in icrc[c]] == [zlib.crc32(o.data[c, b * BLOCK:(b + 1) * BLOCK]) for b in range(62)]


def test_65_checks_refused_with_nothing_launched():
    e = engine("default")
    goals = [L.SliceType("ec(8,9)"), L.SliceType("ec(16,31)")]
    assert L.Engine.plan_check_slices(goals, 48, [1] * 64)["ok"] == 0
    buf = torch.zeros(6 * BLOCK, dtype=torch.uint8, device="cuda")
    dfix = torch.full((3 * 32,), 0xEE, dtype=torch.uint8, device="cuda")
    before = e.stats()["kernel_launches"]
    for call in (lambda: e.check_slices_dev(goals, 1, 48, [buf.data_ptr()] * 64, [6 * BLOCK, 3 * BLOCK], None, dfix.data_ptr()),
                 lambda: e.correct_slices_dev(goals, 1, 48, [buf.data_ptr()] * 64, [6 * BLOCK, 3 * BLOCK], None, None, dfix.data_ptr())):
        with pytest.raises(LzGpuError) as ex:
            call()
        assert ex.value.status == _lib.ERR_ARG
    torch.cuda.synchronize()
    assert e.stats()["kernel_launches"] == before and bool((dfix == 0xEE).all()) and not buf.any()
