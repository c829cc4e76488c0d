"""lzgpu_repair_stripes / _dev: the degraded correction, plus the blocks that fail their stored CRCs rebuilt in place as erasures.

Batches, devices layouts and the map and correction helpers come from test_gpu_stripe_check, test_gpu_stripe_map,
test_gpu_stripe_correct and test_gpu_stripe_degraded.  `rot` flips bytes of a block and leaves its stored CRC alone (bit rot: the CRC
names the block); Batch.corrupt recomputes the CRC (a stale block: only the code sees it).  Expected bytes are the oracle's: the
encoded batch before any fault, and rs_recover of the failing blocks from the first k given parts outside them; CRCs are zlib's.
Every GPU case runs on a fused context and on LZGPU_DISABLE_FUSED=1 (the generic route), each on its own copy of the parts, and both
must give identical entries and bytes."""
import zlib

import numpy as np
import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import test_gpu_stripe_map as SM
from tests.test_gpu_stripe_check import BLOCK, Batch, Dev
from tests.test_gpu_stripe_correct import block, dev_parts, fix_list
from tests.test_gpu_stripe_degraded import ROUTES, dev_fix, engine, host_result
from tests.test_gpu_stripe_map import full_chunk

REPAIR = L.Engine.STRIPE_REPAIR_DTYPE
gpu = pytest.mark.gpu


def rot(b, c, part, s, offset=321, length=3):
    """flip bytes of a block and keep its stored CRC: the block fails it"""
    block(b.parts, part, c, s)[offset:offset + length] ^= np.arange(1, length + 1, dtype=np.uint8) * 91


def twin(oracle, name, n, nb, seed, **kw):
    """(pristine, b): one batch and a copy of its parts and stored CRCs to damage"""
    pristine = Batch(oracle, name, n, nb, seed=seed, **kw)
    b = Batch.__new__(Batch)
    b.__dict__.update(pristine.__dict__)
    b.parts = [p.copy() for p in pristine.parts]
    b.crc = [c.copy() for c in pristine.crc]
    b.faulty = set()
    return pristine, b


def given_list(b, given, parts=None):
    parts = b.parts if parts is None else parts
    return [parts[i] if i in given else None for i in range(b.k + b.m)]


def crc_list(b, given, crcs=None):
    crcs = b.crc if crcs is None else crcs
    return [crcs[i] if i in given else None for i in range(b.k + b.m)]


def repair_routes(b, given, crcs=None, contexts=ROUTES):
    """the host call on every context, each on its own copy; returns (entries, parts after, ChunkCrcError.where or None) of the
    first, after checking that every context gave the same"""
    results = []
    for name, env in contexts.items():
        eng = engine(**env)
        after = [p.copy() for p in b.parts]
        fix, where = host_result(lambda: eng.repair_stripes(b.goal, b.nb, given_list(b, given, after), crc_list(b, given, crcs)), "fix")
        assert fix.shape == (b.n, b.pb) and eng.status_slots()[1] == 0, name
        results.append((fix, after, where))
    f0, p0, w0 = results[0]
    for f, p, w in results[1:]:
        assert fix_list(f) == fix_list(f0), "the routes disagree on the entries"
        assert all((x == y).all() for x, y in zip(p, p0)), "the routes wrote different bytes"
        assert w == w0
    return f0, p0, w0


def oracle_rebuild(oracle, b, parts, c, s, failed, given):
    """the oracle's rebuild of the blocks of `failed` from the first k given parts outside them (a one-stripe recover window)"""
    n = b.k + b.m
    inputs = [i for i in sorted(given) if i not in failed][:b.k]
    ins = [np.ascontiguousarray(block(parts, i, c, s)) if i in inputs else None for i in range(n)]
    out = oracle.rs_recover(b.k, b.m, ins, [0 if i in inputs else 1 for i in range(n)], [int(i in failed) for i in range(n)], BLOCK)
    return {p: out[p] for p in failed}


def assert_repaired(oracle, b, given, fix, after, pristine, rotten):
    """rotten {(c, s): parts}: those stripes REBUILT with crc_failed = their bits, every other stripe clean; every given part back to the
    pristine bytes (the oracle's rebuild too), every stored CRC valid, and the map of the result clean"""
    for c in range(b.n):
        for s in range(b.pb):
            e = fix[c, s]
            f = rotten.get((c, s), ())
            if f:
                assert int(e["status"]) == _lib.FIX_REBUILT and int(e["crc_failed"]) == sum(1 << p for p in f) and int(e["crc"]) == 0, (c, s, e)
                assert int(e["bad_rows"]) != 0
                for p, blk in oracle_rebuild(oracle, b, b.parts, c, s, f, given).items():
                    assert (blk == block(pristine.parts, p, c, s)).all(), (c, s, p)
            else:
                assert tuple(int(x) for x in e) == (0, -1, _lib.FIX_CLEAN, 0, 0), (c, s, e)
    for i in given:
        assert (after[i] == pristine.parts[i]).all(), f"part {i}"
        for c in range(b.n):
            for s in range(b.pb):
                assert zlib.crc32(block(after, i, c, s).tobytes()) == int(b.crc[i][c, s])
    m = engine().check_stripe_map_degraded(b.goal, b.nb, given_list(b, given, after), crc_list(b, given))
    assert not (m["bad_rows"] != 0).any()


# ---- rule 1: no failing CRC, the degraded correction byte for byte ---------------------------------------------------------------

@gpu
@pytest.mark.parametrize("fault", SM.FAULTS)
@pytest.mark.parametrize("text", SM.GOALS)
def test_without_crc_failures_equals_the_correction(oracle, text, fault):
    b = SM.batch(oracle, text)
    SM.inject(b, fault)
    given = set(range(b.k + b.m))
    fix, after, where = repair_routes(b, given)
    assert where is None
    for env in ROUTES.values():
        eng = engine(**env)
        want_parts = [p.copy() for p in b.parts]
        want, _ = host_result(lambda: eng.correct_stripes_degraded(b.goal, b.nb, want_parts, b.crc), "fix")
        assert fix_list(fix[["bad_rows", "suspect_part", "status", "crc"]]) == fix_list(want)
        assert all((x == y).all() for x, y in zip(after, want_parts))
    assert (fix["crc_failed"] == 0).all()


# ---- rebuilt: the failing blocks as erasures ----------------------------------------------------------------------------------------

# (goal, lost parts, {(chunk, stripe): rotten parts}); batches of 3 chunks, nb = 2k + 1 (3 stripes, the last one short)
REBUILT = [
    ("xor2", (), {(0, 0): (0,), (1, 1): (2,), (2, 2): (0,)}),
    ("xor3", (), {(0, 1): (1,), (2, 0): (3,)}),
    ("ec(8,2)", (1,), {(0, 1): (4,), (1, 0): (9,)}),                 # one spare: the correction never blames
    ("ec(8,2)", (), {(0, 1): (2, 6), (2, 0): (0, 8)}),               # two in one stripe: CRC_CONFLICT for the correction
    ("ec(5,3)", (), {(1, 1): (0, 3, 6)}),
    ("ec(8,4)", (), {(0, 0): (1, 2, 8, 11), (2, 1): (7,)}),
    ("ec(6,5)", (), {(1, 0): (0, 2, 4, 6, 10)}),                      # Cauchy, generic route
    ("ec(5,3)", (2,), {(2, 2): (0,), (0, 2): (5, 7)}),               # the short last stripe: data part 0 alone has data
]


@gpu
@pytest.mark.parametrize("case", range(len(REBUILT)), ids=[f"{c[0]}-lost{''.join(map(str, c[1]))}-{i}" for i, c in enumerate(REBUILT)])
def test_rotten_blocks_are_rebuilt(oracle, case):
    name, lost, rotten = REBUILT[case]
    g = L.SliceType(name)
    nb = 2 * g.k + 1
    pristine, b = twin(oracle, name, 3, nb, seed=20 + case)
    given = {i for i in range(g.k + g.m) if i not in lost}
    for (c, s), ps in rotten.items():
        for p in ps:
            rot(b, c, p, s, offset=65530 if s == b.pb - 1 and p < g.k else 300 + 1000 * p)
    fix, after, where = repair_routes(b, given)
    assert where is None
    assert_repaired(oracle, b, given, fix, after, pristine, rotten)


@gpu
def test_rot_in_every_stripe_of_a_chunk(oracle):
    name, nb = "ec(8,4)", 8 * 12 + 3
    pristine, b = twin(oracle, name, 2, nb, seed=31)
    rotten = {}
    for s in range(b.pb):
        ps = (0,) if s == b.pb - 1 else tuple(sorted({s % 12, (5 * s + 3) % 12}))[:1 + s % 2]
        rotten[(1, s)] = ps
        for p in ps:
            rot(b, 1, p, s, offset=65000 if s == b.pb - 1 else 64 * s)
    fix, after, where = repair_routes(b, set(range(12)), contexts={**ROUTES, "cap1": {"LZGPU_GRID_CAP": 1}, "cap3": {"LZGPU_GRID_CAP": 3}})
    assert where is None
    assert_repaired(oracle, b, set(range(12)), fix, after, pristine, rotten)


# ---- refused: nothing written ------------------------------------------------------------------------------------------------------

@gpu
def test_refused_stripes_change_no_byte(oracle):
    """ec(8,4): more failing blocks than spares; rot beside a stale input (valid CRC), which makes the rebuild fail its CRC; a wrong
    stored CRC on a clean stripe.  ec(8,2) with a part lost: two failing blocks, one spare."""
    _, b = twin(oracle, "ec(8,4)", 3, 8 * 3, seed=41)
    for p in (0, 3, 5, 9, 10):
        rot(b, 0, p, 1)                                   # |F| = 5 > 4
    b.corrupt(1, 0, 2, offset=4000)                      # stale input, valid CRC
    rot(b, 1, 6, 2)
    crcs = [c.copy() for c in b.crc]
    crcs[3][2, 0] ^= 0x10                                # a clean stripe, a wrong stored CRC
    before = [p.copy() for p in b.parts]
    fix, after, where = repair_routes(b, set(range(12)), crcs=crcs)
    assert where is not None
    st = fix["status"]
    assert st[0, 1] == st[1, 2] == _lib.FIX_CRC_CONFLICT and st[2, 0] == _lib.FIX_CRC_ONLY
    assert int(fix[0, 1]["crc_failed"]) == sum(1 << p for p in (0, 3, 5, 9, 10)) and int(fix[1, 2]["crc_failed"]) == 1 << 6
    assert int(fix[2, 0]["crc_failed"]) == 1 << 3 and int(fix[2, 0]["bad_rows"]) == 0
    assert ((st == _lib.FIX_CLEAN).sum() == b.n * b.pb - 3)
    assert all((x == y).all() for x, y in zip(after, before))
    _, b2 = twin(oracle, "ec(8,2)", 2, 8 * 2, seed=42)
    rot(b2, 1, 0, 1)
    rot(b2, 1, 8, 1)
    before = [p.copy() for p in b2.parts]
    given = set(range(10)) - {4}
    fix, after, where = repair_routes(b2, given)
    assert fix[1, 1]["status"] == _lib.FIX_CRC_CONFLICT and where is not None
    assert all((after[i] == before[i]).all() for i in given)


# ---- the follow-up call ----------------------------------------------------------------------------------------------------------

@gpu
def test_stale_spare_beside_rot_takes_a_second_call(oracle):
    """ec(8,4): rot in data part 2 and a stale spare (parity part 11, valid CRC) in the same stripe.  The rebuild of part 2 does not
    read part 11, so the first call reports REBUILT and leaves 11; the second finds no failing CRC and CORRECTS it."""
    pristine, b = twin(oracle, "ec(8,4)", 1, 8 * 3, seed=51)
    rot(b, 0, 2, 1)
    b.corrupt(0, 11, 1, offset=2000)
    stale_crc = int(b.crc[11][0, 1])
    for env in ROUTES.values():
        eng = engine(**env)
        parts = [p.copy() for p in b.parts]
        crcs = [c.copy() for c in b.crc]
        first = eng.repair_stripes(b.goal, b.nb, parts, crcs)
        assert first[0, 1]["status"] == _lib.FIX_REBUILT and int(first[0, 1]["crc_failed"]) == 1 << 2
        assert (parts[2] == pristine.parts[2]).all() and not (parts[11] == pristine.parts[11]).all()
        assert int(crcs[11][0, 1]) == stale_crc
        second = eng.repair_stripes(b.goal, b.nb, parts, crcs)
        e = second[0, 1]
        assert (int(e["status"]), int(e["suspect_part"]), int(e["crc_failed"])) == (_lib.FIX_CORRECTED, 11, 0)
        assert int(e["crc"]) == zlib.crc32(block(pristine.parts, 11, 0, 1).tobytes())
        assert all((x == y).all() for x, y in zip(parts, pristine.parts))


# ---- call mechanics ---------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("pad,lead", [(16, 16), (65536 + 48, 48)])
def test_dev_layouts_write_only_the_blocks_and_the_entries(oracle, pad, lead):
    """ec(8,3) without parts 1 and 9 at a padded stride from an offset base: the _dev call equals the host call, and nothing outside
    the rewritten blocks and the entries changes"""
    pristine, b = twin(oracle, "ec(8,3)", 3, 8 * 5 + 1, seed=61)
    given = {i for i in range(11) if i not in (1, 9)}
    rot(b, 0, 0, 1)
    rot(b, 2, 10, 3)
    b.corrupt(1, 2, 4)                                   # no spare left to name it: UNEXPLAINED
    want, want_parts, _ = repair_routes(b, given)
    for env in ROUTES.values():
        eng = engine(**env)
        dev = Dev(b, pad, lead)
        fix = dev_fix(eng, "repair_stripes_dev", b, dev, given, dtype=REPAIR)
        assert fix_list(fix) == fix_list(want)
        parts, bufs = dev_parts(b, dev, lead)
        for i in range(11):
            assert (parts[i] == (want_parts[i] if i in given else b.parts[i])).all(), i
            outside = np.ones(len(bufs[i]), dtype=bool)
            for c in range(b.n):
                outside[lead + c * dev.stride: lead + c * dev.stride + b.pb * BLOCK] = False
            host_init = np.random.default_rng(7).integers(0, 256, len(bufs[i]), dtype=np.uint8)
            assert (bufs[i][outside] == host_init[outside]).all(), i
        del dev
    assert want[0, 1]["status"] == want[2, 3]["status"] == _lib.FIX_REBUILT and want[1, 4]["status"] == _lib.FIX_UNEXPLAINED
    assert (block(want_parts, 0, 0, 1) == block(pristine.parts, 0, 0, 1)).all()


@gpu
def test_refusals_launch_nothing(oracle):
    import torch
    lib = _lib.load()
    _, b = twin(oracle, "ec(5,3)", 1, 10, seed=71)
    rot(b, 0, 1, 0)
    dev = Dev(b, 0, 0)
    out = torch.zeros(64 + REPAIR.itemsize * b.pb, dtype=torch.uint8, device="cuda")
    for env in ROUTES.values():
        eng = engine(**env)
        before = eng.stats()["kernel_launches"]
        cases = [(dev.ptrs, dev.crcs, out.data_ptr() + 4),                                    # d_fix 4- but not 8-byte aligned
                 (dev.ptrs, [c if i != 6 else None for i, c in enumerate(dev.crcs)], out.data_ptr()),  # a given part without CRCs
                 (dev.ptrs, None, out.data_ptr())]
        for ptrs, crcs, fix in cases:
            with pytest.raises(L.LzGpuError) as ei:
                eng.repair_stripes_dev(b.goal, 1, b.nb, ptrs, dev.stride, crcs, fix)
            assert ei.value.status == _lib.ERR_ARG
        with pytest.raises(L.LzGpuError) as ei:
            eng.repair_stripes(b.goal, b.nb, [p.copy() for p in b.parts], [c if i != 0 else None for i, c in enumerate(b.crc)])
        assert ei.value.status == _lib.ERR_ARG
        lib.lzgpu_set_crc_enabled(0)
        try:
            with pytest.raises(L.LzGpuError) as ei:
                eng.repair_stripes_dev(b.goal, 1, b.nb, dev.ptrs, dev.stride, dev.crcs, out.data_ptr())
            assert ei.value.status == _lib.ERR_ARG
            with pytest.raises(L.LzGpuError) as ei:
                eng.repair_stripes(b.goal, b.nb, [p.copy() for p in b.parts], b.crc)
            assert ei.value.status == _lib.ERR_ARG
        finally:
            lib.lzgpu_set_crc_enabled(1)
        torch.cuda.synchronize()
        assert eng.stats()["kernel_launches"] == before
    assert (dev_parts(b, dev, 0)[0][1] == b.parts[1]).all()


@gpu
def test_deferred_mode_has_no_effect(oracle):
    """the _dev call neither waits nor leaves a verdict for sync: a failing CRC is in the entries, and sync reports nothing"""
    pristine, b = twin(oracle, "ec(5,3)", 2, 5 * 4, seed=81)
    rot(b, 1, 6, 2)
    b.crc[3][0, 1] ^= 1                                  # CRC_ONLY
    given = set(range(8)) - {1}
    for env in ROUTES.values():
        eng = engine(**env)
        dev = Dev(b, 0, 0)
        eng.set_deferred_verify(True)
        try:
            fix = dev_fix(eng, "repair_stripes_dev", b, dev, given, dtype=REPAIR)
            eng.sync()
        finally:
            eng.set_deferred_verify(False)
        assert eng.status_slots()[1] == 0
        assert fix[1, 2]["status"] == _lib.FIX_REBUILT and fix[0, 1]["status"] == _lib.FIX_CRC_ONLY
        parts, _ = dev_parts(b, dev, 0)
        assert all((parts[i] == pristine.parts[i]).all() for i in given)
        del dev


@gpu
def test_host_tiles_and_one_full_size_chunk(oracle):
    """ec(8,4) without parts 1 and 4: 51 chunks of 16 stripes take three host tiles of 25 chunks; then one 64 MiB chunk"""
    pristine, b = twin(oracle, "ec(8,4)", 51, 8 * 16, seed=91)
    given = {i for i in range(12) if i not in (1, 4)}
    rotten = {}
    for c in range(0, 51, 5):
        ps = (0, 8) if c % 2 else (10,)
        rotten[(c, c % 16)] = ps
        for p in ps:
            rot(b, c, p, c % 16)
    eng = engine()
    before = eng.stats()["batches_timed"]
    parts = [p.copy() for p in b.parts]
    fix = eng.repair_stripes(b.goal, b.nb, given_list(b, given, parts), crc_list(b, given))
    assert eng.stats()["batches_timed"] - before >= 3
    assert_repaired(oracle, b, given, fix, parts, pristine, rotten)
    del b, pristine, parts
    goal = L.SliceType("ec(8,4)")
    for env in ROUTES.values():
        eng = engine(**env)
        parts, crcs = full_chunk(engine(), goal, 92)
        original = [p.copy() for p in parts]
        for s, ps in ((3, (2,)), (77, (0, 9)), (127, (5, 6, 10, 11))):
            for p in ps:
                parts[p][0, s * BLOCK + 100 * p] ^= 0x5A
        fix = eng.repair_stripes(goal, 1024, parts, crcs)
        done = {int(s): int(fix[0, s]["crc_failed"]) for s in np.nonzero(fix[0]["status"])[0]}
        assert done == {3: 1 << 2, 77: 1 | 1 << 9, 127: sum(1 << p for p in (5, 6, 10, 11))}
        assert all(fix[0, s]["status"] == _lib.FIX_REBUILT for s in done)
        assert all((p == o).all() for p, o in zip(parts, original))
