"""lzgpu_decode_stripes / _dev: the repair of lzgpu_repair_stripes, then errors-and-erasures decoding up to the code's radius.

Batches, device layouts and helpers come from the stripe check, map, correction, degraded and repair tests.  Batch.corrupt makes a
block stale (wrong bytes, its stored CRC recomputed: only the code sees it); `rot` flips bytes and keeps the stored CRC (the CRC names
the block).  Every GPU case runs on a fused context and on LZGPU_DISABLE_FUSED=1, each on its own copy of the parts, and both must
give identical entries and bytes."""
import zlib

import numpy as np
import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import test_gpu_stripe_map as SM
from tests.test_gpu_stripe_check import BLOCK, Dev
from tests.test_gpu_stripe_correct import block, dev_parts
from tests.test_gpu_stripe_degraded import ROUTES, dev_fix, engine, host_result
from tests.test_gpu_stripe_map import full_chunk
from tests.test_gpu_stripe_repair import REBUILT, crc_list, given_list, rot, twin

DECODE = L.Engine.STRIPE_DECODE_DTYPE
REPAIR_FIELDS = ["bad_rows", "suspect_part", "status", "crc", "crc_failed"]
gpu = pytest.mark.gpu


def entries(f):
    return [[(int(e["bad_rows"]), int(e["suspect_part"]), int(e["status"]), int(e["crc"]), int(e["crc_failed"]), int(e["located"]),
              int(e["located_crc"][0]), int(e["located_crc"][1])) for e in row] for row in f]


def decode_routes(b, given, crcs=None, contexts=ROUTES, call="decode_stripes"):
    """the host call on every context, each on its own copy; returns (entries, parts after, ChunkCrcError.where or None) of the
    first, after checking that every context gave the same"""
    results = []
    for name, env in contexts.items():
        eng = engine(**env)
        after = [p.copy() for p in b.parts]
        fix, where = host_result(lambda: getattr(eng, call)(b.goal, b.nb, given_list(b, given, after), crc_list(b, given, crcs)), "fix")
        assert fix.shape == (b.n, b.pb) and eng.status_slots()[1] == 0, name
        results.append((fix, after, where))
    f0, p0, w0 = results[0]
    for f, p, w in results[1:]:
        assert (entries(f) if call == "decode_stripes" else f.tolist()) == (entries(f0) if call == "decode_stripes" else f0.tolist())
        assert all((x == y).all() for x, y in zip(p, p0)), "the routes wrote different bytes"
        assert w == w0
    return f0, p0, w0


def assert_decoded(b, given, fix, after, pristine, stale, rotten=None):
    """stale {(c, s): parts located}, rotten {(c, s): parts failing their CRCs}: those stripes DECODED with located and located_crc
    as the pristine blocks have them, every other stripe clean; every given part back to the pristine bytes; with the located
    blocks' new CRCs stored, the degraded map of the result is clean"""
    rotten = rotten or {}
    crcs = [c.copy() for c in b.crc]
    for c in range(b.n):
        for s in range(b.pb):
            e = fix[c, s]
            if (c, s) in stale:
                ps = sorted(stale[(c, s)])
                want_crc = [zlib.crc32(block(pristine.parts, p, c, s).tobytes()) for p in ps] + [0] * (2 - len(ps))
                assert int(e["status"]) == _lib.FIX_DECODED and int(e["located"]) == sum(1 << p for p in ps), (c, s, e)
                assert [int(x) for x in e["located_crc"]] == want_crc and int(e["crc"]) == 0, (c, s, e)
                assert int(e["crc_failed"]) == sum(1 << p for p in rotten.get((c, s), ())), (c, s, e)
                for p, v in zip(ps, want_crc):
                    crcs[p][c, s] = v
            else:
                assert int(e["status"]) == _lib.FIX_CLEAN and int(e["located"]) == 0, (c, s, e)
    for i in given:
        assert (after[i] == pristine.parts[i]).all(), f"part {i}"
    m = engine().check_stripe_map_degraded(b.goal, b.nb, given_list(b, given, after), crc_list(b, given, crcs))
    assert not (m["bad_rows"] != 0).any()


# ---- rule 1: the repair's entry and bytes ------------------------------------------------------------------------------------------

def equal_to_the_repair(b, given):
    fix, after, where = decode_routes(b, given)
    rep, rep_after, rep_where = decode_routes(b, given, call="repair_stripes", contexts={"fused": {}})
    served = np.isin(rep["status"], [_lib.FIX_UNEXPLAINED, _lib.FIX_CRC_CONFLICT])
    for c in range(b.n):
        for s in range(b.pb):
            e, r = fix[c, s], rep[c, s]
            if int(e["status"]) == _lib.FIX_DECODED:
                assert served[c, s]
                continue
            assert tuple(int(e[f]) for f in REPAIR_FIELDS) == tuple(int(r[f]) for f in REPAIR_FIELDS), (c, s, e, r)
            assert int(e["located"]) == 0 and not e["located_crc"].any()
            for i in given:
                assert (block(after, i, c, s) == block(rep_after, i, c, s)).all(), (c, s, i)
    if not (fix["status"] == _lib.FIX_DECODED).any():
        assert where == rep_where
    return fix


@gpu
@pytest.mark.parametrize("fault", SM.FAULTS)
@pytest.mark.parametrize("text", SM.GOALS)
def test_rule_one_equals_the_repair(oracle, text, fault):
    b = SM.batch(oracle, text)
    SM.inject(b, fault)
    equal_to_the_repair(b, set(range(b.k + b.m)))


@gpu
@pytest.mark.parametrize("case", range(len(REBUILT)), ids=[f"{c[0]}-lost{''.join(map(str, c[1]))}-{i}" for i, c in enumerate(REBUILT)])
def test_rot_equals_the_repair(oracle, case):
    name, lost, rotten = REBUILT[case]
    g = L.SliceType(name)
    _, b = twin(oracle, name, 3, 2 * g.k + 1, seed=20 + case)
    given = {i for i in range(g.k + g.m) if i not in lost}
    for (c, s), ps in rotten.items():
        for p in ps:
            rot(b, c, p, s, offset=65530 if s == b.pb - 1 and p < g.k else 300 + 1000 * p)
    fix = equal_to_the_repair(b, given)
    assert (fix["status"] == _lib.FIX_REBUILT).sum() == len(rotten)


# ---- two stale parts in one stripe ---------------------------------------------------------------------------------------------------

# (goal, lost parts, {(chunk, stripe): ((part, offset), (part, offset))}); batches of 3 chunks, nb = 2k + 1 (the last stripe short:
# data part 0 alone has data there).  Same offsets: overlapping bytes; far apart: disjoint.
TWO_STALE = [
    ("ec(8,4)", (), {(0, 0): ((1, 100), (5, 100)), (0, 1): ((2, 100), (9, 40000)), (1, 1): ((8, 7), (11, 7)), (2, 2): ((0, 500), (10, 502))}),
    ("ec(4,4)", (), {(0, 1): ((0, 10), (3, 60000)), (2, 0): ((4, 1), (7, 2))}),
    ("ec(20,4)", (), {(1, 0): ((19, 65000), (0, 3)), (1, 1): ((4, 1000), (21, 1000)), (2, 2): ((0, 65531), (23, 5))}),
    ("ec(10,5)", (), {(0, 0): ((9, 200), (14, 200)), (2, 1): ((3, 9), (6, 30000))}),            # Cauchy
    ("ec(8,6)", (3,), {(0, 1): ((1, 4), (12, 4)), (1, 2): ((0, 100), (8, 60000)), (2, 0): ((11, 9), (13, 9))}),  # Cauchy, a lost part
]


@gpu
@pytest.mark.parametrize("case", range(len(TWO_STALE)), ids=[f"{c[0]}-{i}" for i, c in enumerate(TWO_STALE)])
def test_two_stale_parts_are_decoded(oracle, case):
    name, lost, stale = TWO_STALE[case]
    g = L.SliceType(name)
    pristine, b = twin(oracle, name, 3, 2 * g.k + 1, seed=100 + case)
    given = {i for i in range(g.k + g.m) if i not in lost}
    for (c, s), faults in stale.items():
        for p, off in faults:
            b.corrupt(c, p, s, offset=off)
    fix, after, where = decode_routes(b, given)
    assert where is None
    assert_decoded(b, given, fix, after, pristine, {cs: [p for p, _ in f] for cs, f in stale.items()})


@gpu
def test_two_stale_parts_in_every_stripe_of_a_chunk(oracle):
    name, nb = "ec(8,4)", 8 * 12 + 3
    pristine, b = twin(oracle, name, 2, nb, seed=131)
    stale = {}
    for s in range(b.pb):
        ps = (0, 8 + s % 4) if s == b.pb - 1 else tuple(sorted({s % 12, (5 * s + 3) % 12} | {(s + 6) % 12}))[:2]
        stale[(1, s)] = ps
        for i, p in enumerate(ps):
            b.corrupt(1, p, s, offset=64 * s + 3000 * i * (s % 2))
    fix, after, where = decode_routes(b, set(range(12)), contexts={**ROUTES, "cap1": {"LZGPU_GRID_CAP": 1}, "cap3": {"LZGPU_GRID_CAP": 3}})
    assert where is None
    assert_decoded(b, set(range(12)), fix, after, pristine, stale)


# ---- one stale part beside rotten blocks -----------------------------------------------------------------------------------------

# (goal, lost parts, rotten parts, a stale input, a stale spare); one stripe of a 2-chunk batch
STALE_AND_ROT = [
    ("ec(8,3)", (), (1,), 5, 10),
    ("ec(8,4)", (), (0, 9), 3, 11),
    ("ec(8,4)", (6,), (2,), 8, 11),
    ("ec(6,5)", (), (0, 7, 9), 4, 10),                    # Cauchy: |F| = 3, s = 5
]


@gpu
@pytest.mark.parametrize("case", range(len(STALE_AND_ROT)), ids=[f"{c[0]}-{i}" for i, c in enumerate(STALE_AND_ROT)])
def test_stale_input_beside_rot_is_decoded(oracle, case):
    name, lost, rotten, stale_in, _ = STALE_AND_ROT[case]
    g = L.SliceType(name)
    pristine, b = twin(oracle, name, 2, 3 * g.k, seed=140 + case)
    given = {i for i in range(g.k + g.m) if i not in lost}
    assert stale_in in [p for p in sorted(given) if p not in rotten][:g.k]
    for p in rotten:
        rot(b, 1, p, 1, offset=200 + 777 * p)
    b.corrupt(1, stale_in, 1, offset=5000)
    rep, _, _ = decode_routes(b, given, call="repair_stripes", contexts={"fused": {}})
    assert rep[1, 1]["status"] == _lib.FIX_CRC_CONFLICT
    fix, after, where = decode_routes(b, given)
    assert where is None
    assert_decoded(b, given, fix, after, pristine, {(1, 1): [stale_in]}, {(1, 1): rotten})
    for p in rotten:                                      # F matches its old stored CRCs
        assert zlib.crc32(block(after, p, 1, 1).tobytes()) == int(b.crc[p][1, 1])


@gpu
@pytest.mark.parametrize("case", range(len(STALE_AND_ROT)), ids=[f"{c[0]}-{i}" for i, c in enumerate(STALE_AND_ROT)])
def test_stale_spare_beside_rot_stays_rebuilt_until_a_second_call(oracle, case):
    """the rebuild of F does not read a stale spare, so the first call ends REBUILT as the repair does; the second finds F empty"""
    name, lost, rotten, _, stale_sp = STALE_AND_ROT[case]
    g = L.SliceType(name)
    pristine, b = twin(oracle, name, 2, 3 * g.k, seed=150 + case)
    given = {i for i in range(g.k + g.m) if i not in lost}
    assert stale_sp not in [p for p in sorted(given) if p not in rotten][:g.k]
    for p in rotten:
        rot(b, 0, p, 2, offset=100 + 333 * p)
    b.corrupt(0, stale_sp, 2, offset=9000)
    for env in ROUTES.values():
        eng = engine(**env)
        parts = [p.copy() for p in b.parts]
        first = eng.decode_stripes(b.goal, b.nb, given_list(b, given, parts), crc_list(b, given))
        e = first[0, 2]
        assert int(e["status"]) == _lib.FIX_REBUILT and int(e["located"]) == 0 and int(e["crc_failed"]) == sum(1 << p for p in rotten)
        assert not (block(parts, stale_sp, 0, 2) == block(pristine.parts, stale_sp, 0, 2)).all()
        second = eng.decode_stripes(b.goal, b.nb, given_list(b, given, parts), crc_list(b, given))
        e = second[0, 2]
        assert (int(e["status"]), int(e["suspect_part"]), int(e["crc_failed"])) == (_lib.FIX_CORRECTED, stale_sp, 0)
        assert int(e["crc"]) == zlib.crc32(block(pristine.parts, stale_sp, 0, 2).tobytes())
        assert all((parts[i] == pristine.parts[i]).all() for i in given)


# ---- beyond the radius: nothing written -------------------------------------------------------------------------------------------

@gpu
def test_beyond_the_radius_nothing_is_written(oracle):
    """ec(8,3): two stale parts (s = 3 < 4) stay UNEXPLAINED; ec(8,2): a stale input beside rot (|F| + 2 > s) stays CRC_CONFLICT"""
    _, b = twin(oracle, "ec(8,3)", 2, 8 * 2, seed=161)
    b.corrupt(1, 2, 0, offset=100)
    b.corrupt(1, 6, 0, offset=100)
    before = [p.copy() for p in b.parts]
    fix, after, where = decode_routes(b, set(range(11)))
    assert where is None and int(fix[1, 0]["status"]) == _lib.FIX_UNEXPLAINED and int(fix[1, 0]["located"]) == 0
    assert all((x == y).all() for x, y in zip(after, before))
    _, b = twin(oracle, "ec(8,2)", 2, 8 * 2, seed=162)
    rot(b, 0, 7, 1)
    b.corrupt(0, 1, 1, offset=3000)
    before = [p.copy() for p in b.parts]
    fix, after, where = decode_routes(b, set(range(10)))
    assert where is not None and int(fix[0, 1]["status"]) == _lib.FIX_CRC_CONFLICT and int(fix[0, 1]["located"]) == 0
    assert all((x == y).all() for x, y in zip(after, before))


# ---- call mechanics ---------------------------------------------------------------------------------------------------------------

@gpu
@pytest.mark.parametrize("pad,lead", [(16, 16), (65536 + 48, 48)])
def test_dev_layouts_write_only_the_blocks_and_the_entries(oracle, pad, lead):
    """ec(8,4) without part 9 at a padded stride from an offset base: the _dev call equals the host call, and nothing outside the
    rewritten blocks and the entries changes"""
    pristine, b = twin(oracle, "ec(8,4)", 3, 8 * 5 + 1, seed=171)
    given = {i for i in range(12) if i != 9}
    rot(b, 0, 0, 1)
    b.corrupt(0, 4, 1, offset=60000)                      # stale input beside rot: DECODED
    b.corrupt(2, 1, 3)
    b.corrupt(2, 10, 3, offset=2)                         # two stale parts with s = 3: UNEXPLAINED
    b.corrupt(1, 2, 4)
    want, want_parts, _ = decode_routes(b, given)
    assert want[0, 1]["status"] == _lib.FIX_DECODED and want[2, 3]["status"] == _lib.FIX_UNEXPLAINED
    assert want[1, 4]["status"] == _lib.FIX_CORRECTED
    for env in ROUTES.values():
        eng = engine(**env)
        dev = Dev(b, pad, lead)
        fix = dev_fix(eng, "decode_stripes_dev", b, dev, given, dtype=DECODE)
        assert entries(fix) == entries(want)
        parts, bufs = dev_parts(b, dev, lead)
        for i in range(12):
            assert (parts[i] == (want_parts[i] if i in given else b.parts[i])).all(), i
            outside = np.ones(len(bufs[i]), dtype=bool)
            for c in range(b.n):
                outside[lead + c * dev.stride: lead + c * dev.stride + b.pb * BLOCK] = False
            host_init = np.random.default_rng(7).integers(0, 256, len(bufs[i]), dtype=np.uint8)
            assert (bufs[i][outside] == host_init[outside]).all(), i
        del dev
    assert (block(want_parts, 4, 0, 1) == block(pristine.parts, 4, 0, 1)).all()


@gpu
def test_refusals_launch_nothing(oracle):
    import torch
    lib = _lib.load()
    _, b = twin(oracle, "ec(5,3)", 1, 10, seed=181)
    rot(b, 0, 1, 0)
    dev = Dev(b, 0, 0)
    out = torch.zeros(64 + DECODE.itemsize * b.pb, dtype=torch.uint8, device="cuda")
    for env in ROUTES.values():
        eng = engine(**env)
        before = eng.stats()["kernel_launches"]
        cases = [(dev.ptrs, dev.crcs, out.data_ptr() + 4),                                    # d_fix 4- but not 8-byte aligned
                 (dev.ptrs, [c if i != 6 else None for i, c in enumerate(dev.crcs)], out.data_ptr()),  # a given part without CRCs
                 (dev.ptrs, None, out.data_ptr())]
        for ptrs, crcs, fix in cases:
            with pytest.raises(L.LzGpuError) as ei:
                eng.decode_stripes_dev(b.goal, 1, b.nb, ptrs, dev.stride, crcs, fix)
            assert ei.value.status == _lib.ERR_ARG
        with pytest.raises(L.LzGpuError) as ei:
            eng.decode_stripes(b.goal, b.nb, [p.copy() for p in b.parts], [c if i != 0 else None for i, c in enumerate(b.crc)])
        assert ei.value.status == _lib.ERR_ARG
        lib.lzgpu_set_crc_enabled(0)
        try:
            with pytest.raises(L.LzGpuError) as ei:
                eng.decode_stripes_dev(b.goal, 1, b.nb, dev.ptrs, dev.stride, dev.crcs, out.data_ptr())
            assert ei.value.status == _lib.ERR_ARG
            with pytest.raises(L.LzGpuError) as ei:
                eng.decode_stripes(b.goal, b.nb, [p.copy() for p in b.parts], b.crc)
            assert ei.value.status == _lib.ERR_ARG
        finally:
            lib.lzgpu_set_crc_enabled(1)
        torch.cuda.synchronize()
        assert eng.stats()["kernel_launches"] == before
    assert (dev_parts(b, dev, 0)[0][1] == b.parts[1]).all()


@gpu
def test_deferred_mode_has_no_effect(oracle):
    """the _dev call neither waits nor leaves a verdict for sync: failing CRCs are in the entries, and sync reports nothing"""
    pristine, b = twin(oracle, "ec(8,4)", 2, 8 * 4, seed=191)
    rot(b, 1, 6, 2)
    b.corrupt(1, 0, 2, offset=1234)                        # stale input beside rot
    b.corrupt(0, 3, 1)
    b.corrupt(0, 10, 1)                                    # two stale parts
    for env in ROUTES.values():
        eng = engine(**env)
        dev = Dev(b, 0, 0)
        eng.set_deferred_verify(True)
        try:
            fix = dev_fix(eng, "decode_stripes_dev", b, dev, set(range(12)), dtype=DECODE)
            eng.sync()
        finally:
            eng.set_deferred_verify(False)
        assert eng.status_slots()[1] == 0
        assert fix[1, 2]["status"] == fix[0, 1]["status"] == _lib.FIX_DECODED
        assert int(fix[1, 2]["located"]) == 1 and int(fix[0, 1]["located"]) == 1 << 3 | 1 << 10
        parts, _ = dev_parts(b, dev, 0)
        assert all((parts[i] == pristine.parts[i]).all() for i in range(12))
        del dev


@gpu
def test_host_tiles_and_one_full_size_chunk(oracle):
    """ec(8,4) without part 4: 51 chunks of 16 stripes take three host tiles of 25 chunks (every stripe with work travels); then one
    64 MiB chunk with two stale parts in three stripes"""
    pristine, b = twin(oracle, "ec(8,4)", 51, 8 * 16, seed=201)
    given = {i for i in range(12) if i != 4}
    stale, rotten = {}, {}
    for c in range(0, 51, 2):
        s, (r, p) = c % 16, ((9, 0), (10, 1))[c % 4 // 2]  # one rotten block and one stale input
        rot(b, c, r, s)
        b.corrupt(c, p, s, offset=700)
        stale[(c, s)], rotten[(c, s)] = (p,), (r,)
    eng = engine()
    before = eng.stats()["batches_timed"]
    parts = [p.copy() for p in b.parts]
    fix = eng.decode_stripes(b.goal, b.nb, given_list(b, given, parts), crc_list(b, given))
    assert eng.stats()["batches_timed"] - before >= 3
    assert_decoded(b, given, fix, parts, pristine, stale, rotten)
    del b, pristine, parts
    goal = L.SliceType("ec(8,4)")
    for env in ROUTES.values():
        eng = engine(**env)
        parts, crcs = full_chunk(engine(), goal, 202)
        original = [p.copy() for p in parts]
        for s, ps in ((3, (2, 6)), (77, (0, 9)), (127, (10, 11))):
            for p in ps:
                parts[p][0, s * BLOCK + 100 * p: s * BLOCK + 100 * p + 50] ^= 0x5A
                crcs[p][0, s] = zlib.crc32(parts[p][0, s * BLOCK:(s + 1) * BLOCK].tobytes())
        fix = eng.decode_stripes(goal, 1024, parts, crcs)
        done = {int(s): int(fix[0, s]["located"]) for s in np.nonzero(fix[0]["status"])[0]}
        assert done == {3: 1 << 2 | 1 << 6, 77: 1 | 1 << 9, 127: 1 << 10 | 1 << 11}
        assert all(fix[0, s]["status"] == _lib.FIX_DECODED for s in done)
        assert all((p == o).all() for p, o in zip(parts, original))
        for s in done:
            for i, p in enumerate(sorted(p for p in range(12) if done[s] >> p & 1)):
                assert int(fix[0, s]["located_crc"][i]) == zlib.crc32(original[p][0, s * BLOCK:(s + 1) * BLOCK].tobytes())
        del parts, original
