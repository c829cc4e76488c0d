"""Salvage of the determined blocks of lost chunks of a multi-slice goal (lzgpu_salvage_slices*, the SALVAGE instantiation of
recover_slices_kernel in csrc/recover_slices_kernel.cuh) on the GPU.

For each case the image, its block CRCs and the map are compared with what the plan (checked against the rank model on the CPU) and
the original data say: KNOWN and SOLVED blocks equal the original chunk, HOLE blocks are zero, the map is the plan expanded per block,
and the CRCs are zlib.crc32 of the blocks written.  Covered: partial patterns with solved blocks, hole-only patterns, nb < L, a ragged
nb, one full 64 MiB chunk; wholly determined patterns against lzgpu_recover_slices' image; a corrupt byte in a staged data block and
in a chosen equation's parity block, with the withheld positions derived here from lzgpu_debug_recover_slices_rows; a corrupt block
nothing depends on; the _dev form with guard bytes around padded buffers and in deferred mode; the CRC-disabled mode; the pool form
on a device listed twice; the refusals.  Each case runs on the default context and with LZGPU_GRID_CAP=2, and the launch is checked
through lzgpu_debug_last_geometry against the plan."""
import os
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200.engine import ChunkCrcError, LzGpuError
from tests.test_recover_slices_plan import _debug_rows, layout, lcm_of, model

pytestmark = pytest.mark.gpu
BLOCK = 65536
ZERO_CRC = zlib.crc32(bytes(BLOCK))
HOLE, KNOWN, SOLVED, WITHHELD = _lib.SALVAGE_HOLE, _lib.SALVAGE_KNOWN, _lib.SALVAGE_SOLVED, _lib.SALVAGE_WITHHELD

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


def goals_of(names):
    return [L.SliceType(n) for n in names]


def original(goals, n, nb, seed):
    """data [n, nb * 64K] and every flat part [n, pb_i * 64K] with its block CRCs [n, pb_i], encoded by lzgpu_encode_slices"""
    rng = np.random.default_rng(seed)
    data = rng.integers(0, 256, size=(n, nb * BLOCK), dtype=np.uint8)
    enc = engine("default").encode_slices(goals, data)
    parts, crcs = [], []
    for g, (par, crc) in zip(goals, enc):
        if g.is_std:
            parts.append(data)
            crcs.append(crc)
            continue
        k, pb = g.k, -(-nb // g.k)
        padded = np.zeros((n, pb * k * BLOCK), dtype=np.uint8)
        padded[:, :nb * BLOCK] = data
        blocks = padded.reshape(n, pb, k, BLOCK)
        for j in range(k):
            parts.append(np.ascontiguousarray(blocks[:, :, j, :]).reshape(n, pb * BLOCK))
            c = np.full((n, pb), ZERO_CRC, dtype=np.uint32)
            idx = np.arange(pb) * k + j
            c[:, idx < nb] = crc[:, idx[idx < nb]]
            crcs.append(c)
        for r in range(g.m):
            parts.append(np.ascontiguousarray(par[:, r]))
            crcs.append(np.ascontiguousarray(crc[:, nb + r * pb: nb + (r + 1) * pb]))
    return data, parts, crcs


def expected_map(goals, nb, given):
    """the plan expanded per block: [nb] of KNOWN / SOLVED / HOLE"""
    p = L.Engine.plan_salvage_slices(goals, nb, given)
    Lc, n_cs = p["L"], -(-nb // p["L"])
    out = np.zeros(nb, dtype=np.uint8)
    for b in range(nb):
        cs, q = divmod(b, Lc)
        tail = p["tail_blocks"] and cs == n_cs - 1
        known, det = (p["tail_known"], p["tail_determined"]) if tail else (p["known"], p["determined"])
        out[b] = KNOWN if (known >> q) & 1 else SOLVED if (det >> q) & 1 else HOLE
    return out


def check(goals, nb, given, data, img, icrc, smap, withheld=()):
    """withheld: (chunk, block) pairs that must be WITHHELD"""
    n = data.shape[0]
    want_map = np.tile(expected_map(goals, nb, given), (n, 1))
    for c, b in withheld:
        assert want_map[c, b] in (KNOWN, SOLVED)
        want_map[c, b] = WITHHELD
    assert np.array_equal(smap, want_map)
    good = np.isin(want_map, (KNOWN, SOLVED))
    blocks_in = data.reshape(n, nb, BLOCK)
    blocks_out = img.reshape(n, nb, BLOCK)
    assert np.array_equal(blocks_out[good], blocks_in[good])
    assert not blocks_out[~good].any()
    if icrc is not None:
        for c in range(n):
            for b in range(nb):
                assert icrc[c, b] == zlib.crc32(blocks_out[c, b].tobytes()), (c, b)
        assert (icrc[~good] == ZERO_CRC).all()


def check_geometry(e, goals, nb, n, given):
    p = L.Engine.plan_salvage_slices(goals, nb, given)
    geo = e.last_geometry()
    n_cs = -(-nb // p["L"])
    assert geo["kernel"] == _lib.KERNEL_SALVAGE_SLICES
    assert (geo["G"], geo["threads"], geo["stages"], geo["smem_bytes"]) == (p["G"], p["threads"], p["stages"], p["smem_bytes"])
    upc = -(-n_cs // p["G"])
    assert geo["units"] % upc == 0 and 0 < geo["units"] <= upc * n
    if e is engine("cap2"):
        assert geo["grid"] <= 2


def find_pattern(goals, kind):
    """the first loss pattern (ascending bits) of a kind: "solved" = not wholly determined, some block solved from parity;
    "holes" = not wholly determined, some block known, none solved; "whole" = every block determined, some solved"""
    _, n = layout(goals)
    Lc = lcm_of(goals)
    for bits in range(1, 1 << n):
        given = [(bits >> g) & 1 for g in range(n)]
        known, det = model(goals, given, Lc)
        solved = det & ~known
        if kind == "solved" and det != (1 << Lc) - 1 and solved:
            return given
        if kind == "holes" and det != (1 << Lc) - 1 and known and not solved:
            return given
        if kind == "whole" and det == (1 << Lc) - 1 and solved:
            return given
    raise AssertionError((kind, goals))


def run(e, goals, nb, n, given, seed, with_crc=True):
    data, parts, crcs = original(goals, n, nb, seed)
    inp = [p if given[g] else None for g, p in enumerate(parts)]
    incrc = [c if given[g] else None for g, c in enumerate(crcs)]
    img, icrc, smap = e.salvage_slices(goals, nb, inp, incrc, with_crc=with_crc)
    check_geometry(e, goals, nb, n, given)
    check(goals, nb, given, data, img, icrc, smap)
    return data, parts, crcs, img, icrc, smap


SETS = [("xor2", "xor3"), ("ec(3,2)", "ec(2,2)"), ("ec(3,2)", "ec(4,2)"), ("std", "xor2", "xor3"), ("ec(5,5)", "xor2")]


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names", SETS, ids="+".join)
@pytest.mark.parametrize("kind", ["solved", "holes"])
def test_partial_patterns(names, kind, ctx):
    goals = goals_of(names)
    Lc = lcm_of(goals)
    given = find_pattern(goals, kind)
    for nb in (4 * Lc, 3 * Lc + Lc // 2 + 1 if Lc > 2 else 7):
        run(engine(ctx), goals, nb, 2, given, seed=nb)


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names,nb,n,kind", [
    (("xor2", "xor3"), 1, 3, "solved"),             # nb < L
    (("xor2", "xor3"), 1023, 2, "solved"),          # ragged
    (("ec(3,2)", "ec(4,2)"), 7, 2, "solved"),       # nb < L = 12
    (("ec(3,2)", "ec(4,2)"), 1021, 1, "solved"),    # a tail of 1
    (("xor2", "ec(2,2)"), 11, 3, "holes"),          # L = 2, G = 4: a partial last unit (at L = 2 nothing is solved but the whole)
    (("ec(3,2)", "ec(4,2)"), 1020, 1, "solved"),    # one chunk of 1020 blocks (L divides nb)
    (("std", "xor2", "xor3"), 1024, 1, "solved"),   # one full 64 MiB chunk
])
def test_batch_shapes(names, nb, n, kind, ctx):
    goals = goals_of(names)
    run(engine(ctx), goals, nb, n, find_pattern(goals, kind), seed=nb)


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names", SETS, ids="+".join)
def test_wholly_determined_equals_recover_slices(names, ctx):
    e = engine(ctx)
    goals = goals_of(names)
    Lc = lcm_of(goals)
    given = find_pattern(goals, "whole")
    nb = 3 * Lc + 1
    data, parts, crcs, img, icrc, smap = run(e, goals, nb, 2, given, seed=5)
    inp = [p if given[g] else None for g, p in enumerate(parts)]
    _, _, rimg = e.recover_slices(goals, nb, inp, [c if given[g] else None for g, c in enumerate(crcs)], want=[0] * len(parts),
                                  chunk_image=True)
    assert np.array_equal(img, rimg)
    assert np.isin(smap, (KNOWN, SOLVED)).all()


def dependents(goals, given, valid):
    """per read block (flat part g, stripe s of its slice in the combined stripe): the positions whose value depends on it, from the
    debug rows: a known position on its staged copy (the first given data part in flat order that holds it), a solved one on the
    parity block of every equation its row uses and on the staged copies of the known positions of that equation's slice stripe"""
    lay, _ = layout(goals)
    nu, ne, unk, es, er, est, rows, det = _debug_rows(goals, given, valid)
    unknown = set(int(q) for q in unk[:nu])
    stager = {}
    for k, m, base, _ in lay:
        for j in range(k):
            if given[base + j]:
                for q in range(j, valid, k):
                    stager.setdefault(q, (base + j, q // k))
    assert set(stager) == set(range(valid)) - unknown
    deps = {}
    for q, r in stager.items():
        deps.setdefault(r, set()).add(q)
    for x in range(nu):
        for e in range(ne):
            if not rows[x][e]:
                continue
            k, m, base, _ = lay[es[e]]
            s = int(est[e])
            deps.setdefault((base + k + int(er[e]), s), set()).add(int(unk[x]))
            for j in range(k):
                if s * k + j in stager:
                    deps.setdefault(stager[s * k + j], set()).add(int(unk[x]))
    return deps, unk, ne, es, er, est, rows


def where_of(goals, g, blk, c):
    lay, _ = layout(goals)
    i = next(i for i, (k, m, base, _) in enumerate(lay) if base <= g < base + k + m)
    return (c, i, g - lay[i][2], blk)


def corrupt_and_check(e, goals, nb, n, given, data, parts, crcs, c, cs, read, positions):
    """one byte of read block `read` = (flat part, stripe s) of combined stripe cs of chunk c flipped, stored CRCs unchanged: exactly
    `positions` of that stripe are withheld, and the call reports the block"""
    lay, _ = layout(goals)
    Lc = lcm_of(goals)
    g, s = read
    k = next(k for k, m, base, _ in lay if base <= g < base + k + m)
    blk = cs * (Lc // k) + s
    bad_parts = [p.copy() if p is not None else None for p in parts]
    bad_parts[g][c, blk * BLOCK + 4321] ^= 0x5A
    inp = [p if given[h] else None for h, p in enumerate(bad_parts)]
    incrc = [x if given[h] else None for h, x in enumerate(crcs)]
    with pytest.raises(ChunkCrcError) as ex:
        e.salvage_slices(goals, nb, inp, incrc)
    assert tuple(ex.value.where) == where_of(goals, g, blk, c)
    check(goals, nb, given, data, ex.value.image, ex.value.image_crc, ex.value.map, withheld=[(c, cs * Lc + q) for q in positions])
    return bad_parts


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names", [("xor2", "xor3"), ("ec(3,2)", "ec(4,2)"), ("ec(5,5)", "xor2")], ids="+".join)
def test_corrupt_blocks_withhold_what_depends_on_them(names, ctx):
    e = engine(ctx)
    goals = goals_of(names)
    Lc = lcm_of(goals)
    given = find_pattern(goals, "solved")
    nb, n, c, cs = 3 * Lc + 2, 3, 1, 1
    data, parts, crcs = original(goals, n, nb, 77)
    deps, unk, ne, es, er, est, rows = dependents(goals, given, Lc)
    lay, _ = layout(goals)
    is_data = {base + j for k, m, base, _ in lay for j in range(k)}
    # the staged data block with the most dependents: its own position and solved ones
    read = max((r for r in deps if r[0] in is_data), key=lambda r: (len(deps[r]), r))
    assert len(deps[read]) > 1
    corrupt_and_check(e, goals, nb, n, given, data, parts, crcs, c, cs, read, deps[read])
    # a chosen equation's parity block that a solved position uses: exactly the unknowns whose rows use that equation
    e_used = next(x for x in range(ne) if rows[:, x].any())
    k, m, base, _ = lay[es[e_used]]
    read = (base + k + int(er[e_used]), int(est[e_used]))
    assert deps[read] == {int(unk[x]) for x in np.nonzero(rows[:, e_used])[0]}
    corrupt_and_check(e, goals, nb, n, given, data, parts, crcs, c, cs, read, deps[read])


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_corrupt_block_nothing_depends_on(ctx):
    e = engine(ctx)
    goals = goals_of(("xor2", "xor3"))
    given = [1, 1, 0, 1, 0, 0, 0]          # xor3 part 0 holds positions 0 and 3, staged from xor2 parts 0 and 1
    nb, n = 14, 2
    data, parts, crcs = original(goals, n, nb, 9)
    deps = dependents(goals, given, 6)[0]
    assert (3, 0) not in deps and (3, 1) not in deps
    corrupt_and_check(e, goals, nb, n, given, data, parts, crcs, 1, 1, (3, 1), set())


def to_dev(a, fill, guard, off, stride, dtype=torch.uint8):
    """a [n, size] copied into a device buffer of `fill` with chunk c at off + c * stride, `guard` bytes after the last"""
    n, size = a.shape
    t = torch.full((off + (n - 1) * stride + size + guard,), fill, dtype=dtype, device="cuda")
    for c in range(n):
        t[off + c * stride: off + c * stride + size] = torch.from_numpy(a[c]).cuda()
    return t


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("deferred", [False, True])
def test_dev_form_guard_bytes(ctx, deferred):
    e = engine(ctx)
    goals = goals_of(("ec(3,2)", "ec(4,2)"))
    given = find_pattern(goals, "solved")
    nb, n = 29, 2
    data, parts, crcs = original(goals, n, nb, 21)
    GUARD, OFF = 4096, 4096 + 48
    pbs = [-(-nb // g.k) for g in goals]
    slice_of = [i for i, g in enumerate(goals) for _ in range(g.k + g.m)]
    pstride = [pb * BLOCK + 4096 for pb in pbs]
    bufs = {g: to_dev(parts[g], 0x77, GUARD, OFF, pstride[slice_of[g]]) for g in range(len(parts)) if given[g]}
    bad_crcs = [x.copy() for x in crcs]
    g_bad = max(bufs)
    bad_crcs[g_bad][1, 3] ^= 1            # chunk 1, block 3 of the last given part: its dependents are withheld
    cbufs = {g: torch.from_numpy(bad_crcs[g].view(np.int32).copy()).cuda() for g in bufs}
    istride = (nb + 1) * BLOCK
    img = torch.full((OFF + n * istride + GUARD,), 0x3C, dtype=torch.uint8, device="cuda")
    icrc = torch.full((GUARD // 4 + n * nb + GUARD // 4,), 0x11223344, dtype=torch.int32, device="cuda")
    smap = torch.full((GUARD + n * nb + GUARD,), 0xEE, dtype=torch.uint8, device="cuda")
    args = (goals, n, nb, [bufs[g].data_ptr() + OFF if g in bufs else 0 for g in range(len(parts))], pstride,
            [cbufs[g].data_ptr() if g in cbufs else 0 for g in range(len(parts))], img.data_ptr() + OFF, istride,
            icrc.data_ptr() + GUARD, smap.data_ptr() + GUARD)
    i, j = slice_of[g_bad], g_bad - sum(goals[x].k + goals[x].m for x in range(slice_of[g_bad]))
    if deferred:
        e.set_deferred_verify(True)
        try:
            e.salvage_slices_dev(*args)
            with pytest.raises(ChunkCrcError) as ex:
                e.sync()
            assert tuple(ex.value.where) == (1, g_bad, 3)
        finally:
            e.set_deferred_verify(False)
    else:
        with pytest.raises(ChunkCrcError) as ex:
            e.salvage_slices_dev(*args)
        assert tuple(ex.value.where) == (1, i, j, 3)
    torch.cuda.synchronize()
    check_geometry(e, goals, nb, n, given)
    hi, hc, hm = img.cpu().numpy(), icrc.cpu().numpy().view(np.uint32), smap.cpu().numpy()
    assert (hi[:OFF] == 0x3C).all() and (hi[OFF + (n - 1) * istride + nb * BLOCK:] == 0x3C).all()
    for c in range(n):
        assert (hi[OFF + c * istride + nb * BLOCK: OFF + (c + 1) * istride] == 0x3C).all()
    g0 = GUARD // 4
    assert (hc[:g0] == 0x11223344).all() and (hc[g0 + n * nb:] == 0x11223344).all()
    assert (hm[:GUARD] == 0xEE).all() and (hm[GUARD + n * nb:] == 0xEE).all()
    Lc = lcm_of(goals)
    k = goals[i].k
    cs, s = divmod(3, Lc // k)                 # part block 3: combined stripe cs, stripe s of the slice
    deps = dependents(goals, given, Lc if cs < nb // Lc else nb % Lc)[0]
    withheld = [(1, cs * Lc + q) for q in deps.get((g_bad, s), set())]
    image = np.stack([hi[OFF + c * istride: OFF + c * istride + nb * BLOCK] for c in range(n)])
    check(goals, nb, given, data, image, hc[g0: g0 + n * nb].reshape(n, nb), hm[GUARD: GUARD + n * nb].reshape(n, nb), withheld)


def test_crc_disabled_mode():
    e = engine("default")
    goals = goals_of(("xor2", "xor3"))
    given = find_pattern(goals, "solved")
    nb, n = 15, 2
    data, parts, _ = original(goals, n, nb, 3)
    lib = _lib.load()
    lib.lzgpu_set_crc_enabled(0)
    try:
        fake = [np.full((n, -(-nb // (1 if g.is_std else g.k))), 0xFEDCBA98, dtype=np.uint32) for g in goals for _ in range(g.k + g.m)]
        img, icrc, smap = e.salvage_slices(goals, nb, [p if given[g] else None for g, p in enumerate(parts)],
                                           [f if given[g] else None for g, f in enumerate(fake)])
    finally:
        lib.lzgpu_set_crc_enabled(1)
    check(goals, nb, given, data, img, None, smap)
    assert (icrc == 0xFEDCBA98).all()


@pytest.mark.parametrize("n", [0, 1, 5])
def test_pool_on_a_device_listed_twice_equals_one_context(n):
    goals = goals_of(("ec(3,2)", "ec(4,2)"))
    given = find_pattern(goals, "solved")
    nb = 25
    data, parts, crcs = original(goals, max(n, 1), nb, 41)
    bad_crcs = [x.copy() for x in crcs]
    g_bad = max(g for g in range(len(parts)) if given[g])
    bad_crcs[g_bad][max(n, 1) - 1, 2] ^= 1
    inp = [p[:n] if given[g] else None for g, p in enumerate(parts)]
    pool = L.Pool([0, 0])
    try:
        for cr in (crcs, bad_crcs):
            incrc = [x[:n] if given[g] else None for g, x in enumerate(cr)]
            res = []
            for fn in (engine("default").salvage_slices, pool.salvage_slices):
                try:
                    res.append((None,) + fn(goals, nb, inp, incrc))
                except ChunkCrcError as ex:
                    res.append((tuple(ex.where), ex.image, ex.image_crc, ex.map))
            (w0, *a), (w1, *b) = res
            assert w0 == w1
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
            if n:
                check(goals, nb, given, data[:n], *a, withheld=[] if w0 is None else
                      [(w0[0], b) for b in range(nb) if a[2][w0[0], b] == WITHHELD])
    finally:
        pool.close()


def test_refusals_write_nothing():
    e = engine("default")
    lib = _lib.load()
    goals = goals_of(("xor2", "xor3"))
    nb = 7
    data, parts, crcs = original(goals, 1, nb, 1)
    img = torch.full((nb * BLOCK,), 0x3C, dtype=torch.uint8, device="cuda")
    smap = torch.full((nb,), 0xEE, dtype=torch.uint8, device="cuda")
    before = e.stats()["kernel_launches"]
    with pytest.raises(LzGpuError) as ex:   # no part given
        e.salvage_slices_dev(goals, 1, nb, [0] * 7, [4 * BLOCK, 3 * BLOCK], None, img.data_ptr(), nb * BLOCK, None, smap.data_ptr())
    assert ex.value.status == _lib.ERR_TOO_FEW_PARTS
    with pytest.raises(LzGpuError) as ex:
        e.salvage_slices(goals, nb, [None] * 7)
    assert ex.value.status == _lib.ERR_TOO_FEW_PARTS
    d_parts = [torch.from_numpy(p).cuda() for p in parts]
    ptrs = [t.data_ptr() for t in d_parts]
    with pytest.raises(LzGpuError) as ex:   # no map
        e.salvage_slices_dev(goals, 1, nb, ptrs, [4 * BLOCK, 3 * BLOCK], None, img.data_ptr(), nb * BLOCK, None, None)
    assert ex.value.status == _lib.ERR_ARG
    with pytest.raises(LzGpuError) as ex:   # a misaligned image
        e.salvage_slices_dev(goals, 1, nb, ptrs, [4 * BLOCK, 3 * BLOCK], None, img.data_ptr() + 8, nb * BLOCK, None, smap.data_ptr())
    assert ex.value.status == _lib.ERR_ARG
    with pytest.raises(LzGpuError) as ex:   # a repeated slice type
        e.salvage_slices(goals_of(("xor2", "xor2")), nb, parts[:3] + parts[:3])
    assert ex.value.status == _lib.ERR_ARG
    # a goal set whose salvage does not fit the kernel's tables (the plan says ok = 0)
    big = goals_of(("ec(3,3)", "ec(16,16)"))
    assert L.Engine.plan_salvage_slices(big, 48, [1] * 38)["ok"] == 0
    pbs = [16 * BLOCK, 3 * BLOCK]
    buf = torch.zeros(16 * BLOCK, dtype=torch.uint8, device="cuda")
    with pytest.raises(LzGpuError) as ex:
        e.salvage_slices_dev(big, 1, 48, [buf.data_ptr()] * 38, pbs, None, img.data_ptr(), 48 * BLOCK, None, smap.data_ptr())
    assert ex.value.status == _lib.ERR_ARG
    torch.cuda.synchronize()
    assert e.stats()["kernel_launches"] == before
    assert bool((img == 0x3C).all()) and bool((smap == 0xEE).all())
    assert lib.lzgpu_pool_salvage_slices(None, None, 0, 0, 0, None, None, None, None, 0, None, None, None) == _lib.ERR_ARG
