"""lzgpu_correct_stripes / _dev: the stripe map, and every stripe that names a suspect part corrected in place.

Batches, fault injection (part bytes flipped, the block's stored CRC recomputed), the device layouts and the expected map come from
test_gpu_stripe_check and test_gpu_stripe_map.  The expected status of a stripe follows from the expected map and the rule: clean;
bad without a suspect (UNEXPLAINED); bad with a suspect and a given block other than the suspect's failing its stored CRC
(CRC_CONFLICT); otherwise CORRECTED, and the corrected block must equal what the oracle's rs_recover rebuilds for the suspect from
the first k given other parts of that stripe (the original block, when one part was faulty).  Every case runs on the fused route
and, with LZGPU_DISABLE_FUSED=1, on the generic route, each on its own copy of the input; both must give identical fix arrays and
identical bytes.  After the call every byte outside the corrected blocks is unchanged, and the map of the corrected parts, with the
new CRCs stored, is clean except for the stripes left UNEXPLAINED / CRC_CONFLICT, which are still bad."""
import ctypes
import os
import subprocess
import zlib

import numpy as np
import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests.test_gpu_stripe_check import BLOCK, GOALS, ZERO_CRC, Dev
from tests.test_gpu_stripe_map import FAULTS, as_list, batch, corrupt_block, expected_map, full_chunk, inject

FIX = L.Engine.STRIPE_FIX_DTYPE
FAKE_CRC = 0xFEDCBA98
_engines = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in _engines.values():
        e.close()
    _engines.clear()


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


def both_engines():
    return [engine(), engine(LZGPU_DISABLE_FUSED=1)]


# ---- the expected result, on the CPU --------------------------------------------------------------
def block(parts, p, c, s):
    return parts[p][c, s * BLOCK:(s + 1) * BLOCK]


def rebuilt(oracle, b, parts, c, s, suspect, given):
    """the oracle's rebuild of the suspect's block from the first k given other parts of stripe s"""
    n = b.k + b.m
    inputs = [i for i in range(n) if i in given and i != suspect][:b.k]
    ins = [np.ascontiguousarray(block(parts, i, c, s)) if i in inputs else None for i in range(n)]
    erased = [0 if i in inputs else 1 for i in range(n)]
    return oracle.rs_recover(b.k, b.m, ins, erased, [int(i == suspect) for i in range(n)], BLOCK)[suspect]


def stored_ok(parts, crcs, p, c, s):
    return crcs is None or crcs[p] is None or int(crcs[p][c, s]) == zlib.crc32(block(parts, p, c, s).tobytes())


def expected_status(smap, parts, crcs, given):
    """[n, pb] of LZGPU_FIX_* from the map and the rule"""
    out = np.zeros(smap.shape, dtype=np.int32)
    for c in range(smap.shape[0]):
        for s in range(smap.shape[1]):
            rows, suspect = int(smap[c, s]["bad_rows"]), int(smap[c, s]["suspect_part"])
            if not rows:
                out[c, s] = _lib.FIX_CLEAN
            elif suspect < 0:
                out[c, s] = _lib.FIX_UNEXPLAINED
            elif all(stored_ok(parts, crcs, p, c, s) for p in given if p != suspect):
                out[c, s] = _lib.FIX_CORRECTED
            else:
                out[c, s] = _lib.FIX_CRC_CONFLICT
    return out


def map_of(eng, goal, nb, parts, crcs):
    """check_stripe_map whether or not a stored CRC fails"""
    try:
        return eng.check_stripe_map(goal, nb, parts, crcs)
    except L.ChunkCrcError as e:
        return e.map


def fix_list(f):
    return [[tuple(int(x) for x in e) for e in row] for row in f]


def verify(oracle, b, crcs, given, fix, after, rows, pristine=None, crc_value=None):
    """every assertion of a case, for one route's result: fix = the entries, after = the parts after the call (b.parts: before)"""
    before = b.parts
    ref = map_of(engine(), b.goal, b.nb, [before[i] if i in given else None for i in range(b.k + b.m)], crcs)
    assert as_list(fix[["bad_rows", "suspect_part"]]) == as_list(ref) == as_list(expected_map(oracle, b, rows))
    assert (fix["status"] == expected_status(ref, before, crcs, given)).all(), (fix["status"], expected_status(ref, before, crcs, given))
    want = [p.copy() for p in before]
    new_crcs = None if crcs is None else [None if x is None else x.copy() for x in crcs]
    for c, s in zip(*np.nonzero(fix["status"] == _lib.FIX_CORRECTED)):
        p = int(fix[c, s]["suspect_part"])
        blk = rebuilt(oracle, b, before, c, s, p, given)
        block(want, p, c, s)[:] = blk
        if pristine is not None:
            assert (blk == block(pristine, p, c, s)).all(), (c, s, p)
        assert int(fix[c, s]["crc"]) == (zlib.crc32(blk.tobytes()) if crc_value is None else crc_value)
        if new_crcs is not None and new_crcs[p] is not None:
            new_crcs[p][c, s] = fix[c, s]["crc"]
    assert (fix["crc"][fix["status"] != _lib.FIX_CORRECTED] == 0).all()
    for i in range(b.k + b.m):
        assert (after[i] == want[i]).all(), f"part {i}: bytes outside the corrected blocks changed, or a wrong corrected block"
    if crc_value is not None:
        return
    left = map_of(engine(), b.goal, b.nb, [after[i] if i in given else None for i in range(b.k + b.m)], new_crcs)
    still = (fix["status"] == _lib.FIX_UNEXPLAINED) | (fix["status"] == _lib.FIX_CRC_CONFLICT)
    assert ((left["bad_rows"] != 0) == still).all()


def run_host(b, given, crcs):
    """the host call on both routes, each on its own copy; returns (fix, parts after, rc) of the fused route"""
    results = []
    for eng in both_engines():
        parts = [p.copy() for p in b.parts]
        rc = _lib.OK
        try:
            fix = eng.correct_stripes(b.goal, b.nb, [parts[i] if i in given else None for i in range(b.k + b.m)], crcs)
            if (fix["status"] == _lib.FIX_UNEXPLAINED).any():
                rc = _lib.ERR_INCONSISTENT
        except L.ChunkCrcError as e:
            fix, rc = e.fix, (_lib.ERR_CRC, e.where)
        assert fix.shape == (b.n, b.pb)
        assert eng.status_slots()[1] == 0
        results.append((fix, parts, rc))
    (f0, p0, r0), (f1, p1, r1) = results
    assert fix_list(f0) == fix_list(f1), "fused and generic routes disagree"
    assert all((x == y).all() for x, y in zip(p0, p1)), "fused and generic routes wrote different bytes"
    assert r0 == r1
    return f0, p0, r0


gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("fault", FAULTS)
@pytest.mark.parametrize("text", GOALS)
def test_correction_matches_the_oracle(oracle, text, fault):
    pristine = batch(oracle, text)
    b = batch(oracle, text)
    inject(b, fault)
    given = set(range(b.k + b.m))
    fix, after, rc = run_host(b, given, b.crc)
    verify(oracle, b, b.crc, given, fix, after, list(range(b.m)),
           pristine=None if fault == "two_parts_one_stripe" else pristine.parts)
    status = fix["status"]
    if b.m == 1 or fault == "none":
        assert not (status == _lib.FIX_CORRECTED).any()     # xorN never names a suspect
    if fault == "two_parts_one_stripe" and b.m >= 3:
        assert status[1, 1] == status[2, 2] == _lib.FIX_UNEXPLAINED
    if fault in ("one_stripe", "stripes_blame_different_parts", "short_last_stripe", "parity_parts", "every_stripe") and b.m >= 2:
        assert (status[fix["bad_rows"] != 0] == _lib.FIX_CORRECTED).all()
        assert rc == _lib.OK
    if fault == "every_stripe" and b.m >= 2:
        assert (status[1] == _lib.FIX_CORRECTED).all()


@gpu
@pytest.mark.parametrize("text", ["ec(8,2)", "ec(5,3)", "ec(22,4)"])
@pytest.mark.parametrize("case", ["bit_rot_in_the_suspect", "another_block_fails", "clean_stripe_fails"])
def test_crc_gate(oracle, text, case):
    pristine = batch(oracle, text)
    b = batch(oracle, text)
    k = b.k
    b.corrupt(2, 1, 1)                                  # corrected in every case
    crcs = [c.copy() for c in b.crc]
    if case == "bit_rot_in_the_suspect":                # the syndromes and the failing CRC name the same block
        old = int(crcs[2][0, 1])
        b.corrupt(0, 2, 1)
        crcs[2][0, 1] = old
        where, stripe = (0, 2, 1), (0, 1)
    elif case == "another_block_fails":                 # two faults can mimic a third part: a failing CRC blocks the write
        b.corrupt(1, 3, 0)
        crcs[3][1, 0] = b.crc[3][1, 0]
        crcs[0][1, 0] ^= 0x40
        where, stripe = (1, 0, 0), (1, 0)
    else:
        crcs[k][0, 2] ^= 1
        where, stripe = (0, k, 2), (0, 2)
    given = set(range(b.k + b.m))
    fix, after, rc = run_host(b, given, crcs)
    assert rc == (_lib.ERR_CRC, where)
    verify(oracle, b, crcs, given, fix, after, list(range(b.m)), pristine=pristine.parts)
    assert fix[2, 1]["status"] == _lib.FIX_CORRECTED
    want = {"bit_rot_in_the_suspect": _lib.FIX_CORRECTED, "another_block_fails": _lib.FIX_CRC_CONFLICT,
            "clean_stripe_fails": _lib.FIX_CLEAN}[case]
    assert fix[stripe]["status"] == want
    if case == "another_block_fails":
        for i in range(b.k + b.m):
            assert (block(after, i, 1, 0) == block(b.parts, i, 1, 0)).all()


@gpu
@pytest.mark.parametrize("text,skip", [("ec(8,4)", (8,)), ("ec(5,3)", (6,)), ("ec(5,3)", (6, 7)), ("ec(8,4)", (9, 11))])
def test_missing_parity_rows(oracle, text, skip):
    pristine = batch(oracle, text)
    b = batch(oracle, text)
    rows = [r for r in range(b.m) if b.k + r not in skip]
    b.corrupt(0, 2, 1)
    b.corrupt(2, b.k + rows[-1], 2)
    given = set(range(b.k + b.m)) - set(skip)
    fix, after, rc = run_host(b, given, b.crc)
    verify(oracle, b, b.crc, given, fix, after, rows, pristine=pristine.parts)
    corrected = fix["status"] == _lib.FIX_CORRECTED
    if len(rows) == 1:
        assert not corrected.any() and rc == _lib.ERR_INCONSISTENT
    else:
        assert corrected[0, 1] and corrected[2, 2] and corrected.sum() == 2 and rc == _lib.OK


# ---- device pointers ------------------------------------------------------------------------------
def run_dev(eng, b, dev, guard=4096, lead=0):
    """the correction of a resident batch into a guarded fix buffer; asserts nothing outside the entries changed"""
    torch = dev.torch
    size = 16 * b.n * b.pb
    init = np.random.default_rng(3).integers(0, 256, 2 * guard + lead + size, dtype=np.uint8)
    t = torch.from_numpy(init.copy()).cuda()
    eng.correct_stripes_dev(b.goal, b.n, b.nb, dev.ptrs, dev.stride, dev.crcs, t.data_ptr() + guard + lead)
    torch.cuda.synchronize()
    out = t.cpu().numpy()
    o = guard + lead
    assert (out[:o] == init[:o]).all() and (out[o + size:] == init[o + size:]).all(), "write outside d_fix"
    return out[o:o + size].copy().view(FIX).reshape(b.n, b.pb)


def dev_parts(b, dev, lead):
    """the parts back from the device, and the whole buffers (guard bytes included)"""
    bufs = [dev.bufs[2 * i].cpu().numpy() for i in range(b.k + b.m)]
    parts = [np.stack([buf[lead + c * dev.stride: lead + c * dev.stride + b.pb * BLOCK] for c in range(b.n)]) for buf in bufs]
    return parts, bufs


@gpu
@pytest.mark.parametrize("text", ["ec(8,2)", "ec(5,3)", "xor2", "ec(22,4)"])
@pytest.mark.parametrize("pad,lead", [(0, 0), (16, 20), (65536 + 48, 52)])
def test_dev_layouts_write_only_the_blocks_and_the_entries(oracle, text, pad, lead):
    pristine = batch(oracle, text)
    b = batch(oracle, text)
    b.corrupt(1, 2, 1)
    b.corrupt(0, b.k, 2)
    b.corrupt(2, b.k - 1, 0)
    given = set(range(b.k + b.m))
    results = []
    for eng in both_engines():
        dev = Dev(b, pad, lead & ~15)
        base = lead & ~15
        _, before_bufs = dev_parts(b, dev, base)
        fix = run_dev(eng, b, dev, lead=lead % 64)        # the entries at 4-byte alignment only
        after, bufs = dev_parts(b, dev, base)
        verify(oracle, b, b.crc, given, fix, after, list(range(b.m)), pristine=pristine.parts)
        for i in range(b.k + b.m):                          # the guard bytes around every part
            outside = np.ones(len(bufs[i]), dtype=bool)
            for c in range(b.n):
                outside[base + c * dev.stride: base + c * dev.stride + b.pb * BLOCK] = False
            assert (bufs[i][outside] == before_bufs[i][outside]).all(), i
        results.append((fix_list(fix), after))
    assert results[0][0] == results[1][0]
    assert all((x == y).all() for x, y in zip(results[0][1], results[1][1]))


@gpu
def test_misaligned_pointers_are_refused_without_a_launch(oracle):
    import torch
    b = batch(oracle, "ec(8,2)")
    b.corrupt(0, 1, 0)
    dev = Dev(b)
    out = torch.zeros(64 + 16 * b.n * b.pb, dtype=torch.uint8, device="cuda")
    for eng in both_engines():
        launches = eng.stats()["kernel_launches"]
        for parts, fix in ((dev.ptrs, out.data_ptr() + 2), ([p + (8 if i == 3 else 0) for i, p in enumerate(dev.ptrs)], out.data_ptr())):
            with pytest.raises(L.LzGpuError) as ei:
                eng.correct_stripes_dev(b.goal, b.n, b.nb, parts, dev.stride, dev.crcs, fix)
            assert ei.value.status == _lib.ERR_ARG
        assert eng.stats()["kernel_launches"] == launches
    for i in range(b.k + b.m):
        assert (dev_parts(b, dev, 0)[0][i] == b.parts[i]).all()


@gpu
def test_deferred_mode_collects_the_crc_mismatch(oracle):
    pristine = batch(oracle, "ec(8,2)")
    b = batch(oracle, "ec(8,2)")
    b.corrupt(0, 4, 1)
    b.corrupt(0, 6, 0)
    b.crc[9][2, 1] ^= 1                                  # a clean stripe: reported at sync, corrections still made
    given = set(range(b.k + b.m))
    for eng in both_engines():
        dev = Dev(b)
        eng.set_deferred_verify(True)
        try:
            fix = run_dev(eng, b, dev)
            with pytest.raises(L.ChunkCrcError) as ei:
                eng.sync()
            assert ei.value.where == (2, 9, 1)
        finally:
            eng.set_deferred_verify(False)
        assert eng.status_slots()[1] == 0
        after, _ = dev_parts(b, dev, 0)
        verify(oracle, b, b.crc, given, fix, after, [0, 1], pristine=pristine.parts)
        assert (fix["status"] == _lib.FIX_CORRECTED).sum() == 2


# ---- host tiles, a full chunk, the CRC-disabled mode -----------------------------------------------
@gpu
def test_host_tiles_correct_at_batch_wide_chunks():
    """ec(8,2), one-stripe chunks: 823 chunks take three tiles of the check.  Faults in tiles 1 and 2."""
    goal, k, m, nb, n = L.SliceType("ec(8,2)"), 8, 2, 8, 823
    fixes = []
    for eng in both_engines():
        parts = [np.zeros((n, BLOCK), dtype=np.uint8) for _ in range(k + m)]
        crcs = [np.full((n, 1), ZERO_CRC, dtype=np.uint32) for _ in range(k + m)]
        for c, p in ((500, 3), (820, 9), (300, 0)):
            parts[p][c, 10:14] = 0xA5
            crcs[p][c, 0] = zlib.crc32(parts[p][c].tobytes())
        fix = eng.correct_stripes(goal, nb, parts, crcs)
        got = {c: tuple(int(x) for x in fix[c, 0]) for c in range(n) if fix[c, 0]["status"] != _lib.FIX_CLEAN}
        assert got == {300: (3, 0, _lib.FIX_CORRECTED, ZERO_CRC), 500: (3, 3, _lib.FIX_CORRECTED, ZERO_CRC),
                       820: (2, 9, _lib.FIX_CORRECTED, ZERO_CRC)}
        assert not any(p.any() for p in parts)
        assert eng.status_slots()[1] == 0
        fixes.append(fix_list(fix))
    assert fixes[0] == fixes[1]


def window_repair(eng, goal, nb, parts, bad):
    """the existing route: one lzgpu_recover_chunks_dev call per bad stripe over a one-stripe window"""
    import torch
    k, m = goal.k, goal.m
    parts = [p.copy() for p in parts]
    dev = [torch.from_numpy(p[0]).cuda() for p in parts]
    out = torch.zeros(BLOCK, dtype=torch.uint8, device="cuda")
    for s, p in bad:
        window = [0 if i == p else dev[i].data_ptr() + s * BLOCK for i in range(k + m)]
        d_out = [out.data_ptr() if i == p else 0 for i in range(k + m)]
        eng.recover_chunks_dev(goal, 1, min(k, nb - s * k), window, parts[0].shape[1], None, [int(i == p) for i in range(k + m)], d_out)
        torch.cuda.synchronize()
        parts[p][0, s * BLOCK:(s + 1) * BLOCK] = out.cpu().numpy()
    return parts


@gpu
def test_one_call_restores_a_full_size_chunk():
    """ec(8,2), one 64 MiB chunk, three bad stripes blaming three different parts (the map test's repair scenario)"""
    goal, nb = L.SliceType("ec(8,2)"), 1024
    results = []
    for eng in both_engines():
        parts, crcs = full_chunk(engine(), goal, 12)
        original = [p.copy() for p in parts]
        for s, p in ((7, 2), (40, 6), (127, 8)):
            corrupt_block(parts, crcs, p, s, 4321, 0x3C)
        windows = window_repair(eng, goal, nb, parts, [(7, 2), (40, 6), (127, 8)])
        fix = eng.correct_stripes(goal, nb, parts, crcs)
        done = {int(s): tuple(int(x) for x in fix[0, s]) for s in np.nonzero(fix[0]["status"])[0]}
        assert done == {s: (3 if p < 8 else 1 << (p - 8), p, _lib.FIX_CORRECTED, zlib.crc32(original[p][0, s * BLOCK:(s + 1) * BLOCK].tobytes()))
                        for s, p in ((7, 2), (40, 6), (127, 8))}
        for p, o, w in zip(parts, original, windows):
            assert (p == o).all() and (w == o).all()
        for s, p in ((7, 2), (40, 6), (127, 8)):
            crcs[p][0, s] = fix[0, s]["crc"]
        again = eng.correct_stripes(goal, nb, parts, crcs)
        assert (again["status"] == _lib.FIX_CLEAN).all()
        results.append(fix_list(fix))
    assert results[0] == results[1]


@gpu
def test_crc_disabled_mode_reports_the_constant(oracle):
    lib = _lib.load()
    pristine = batch(oracle, "ec(5,3)")
    b = batch(oracle, "ec(5,3)")
    b.corrupt(1, 3, 1)
    b.corrupt(2, 6, 0)
    fake = [np.full(c.shape, FAKE_CRC, dtype=np.uint32) for c in b.crc]
    given = set(range(b.k + b.m))
    lib.lzgpu_set_crc_enabled(0)
    try:
        fix, after, rc = run_host(b, given, fake)
        assert rc == _lib.OK
        assert (fix["status"] == _lib.FIX_CORRECTED).sum() == 2
        verify(oracle, b, None, given, fix, after, [0, 1, 2], pristine=pristine.parts, crc_value=FAKE_CRC)
        bad = [c.copy() for c in fake]
        bad[0][2, 0] = ZERO_CRC                          # the real CRC is a mismatch in this mode: it blocks stripe (2, 0)
        fix, after, rc = run_host(b, given, bad)
        assert rc == (_lib.ERR_CRC, (2, 0, 0))
        assert fix[1, 1]["status"] == _lib.FIX_CORRECTED and fix[2, 0]["status"] == _lib.FIX_CRC_CONFLICT
    finally:
        lib.lzgpu_set_crc_enabled(1)


def test_stripe_fix_layout_matches_the_header(tmp_path):
    """(no GPU needed) the ctypes and numpy mirrors of lzgpu_stripe_fix and the LZGPU_FIX_* values against include/lzgpu.h"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lzgpu.h"\nint main(void) { printf("%zu %zu %zu %zu %zu %zu '
                   '%d %d %d %d\\n", sizeof(lzgpu_stripe_fix), _Alignof(lzgpu_stripe_fix), offsetof(lzgpu_stripe_fix, bad_rows), '
                   'offsetof(lzgpu_stripe_fix, suspect_part), offsetof(lzgpu_stripe_fix, status), offsetof(lzgpu_stripe_fix, crc), '
                   'LZGPU_FIX_CLEAN, LZGPU_FIX_CORRECTED, LZGPU_FIX_UNEXPLAINED, LZGPU_FIX_CRC_CONFLICT); return 0; }\n')
    subprocess.run(["gcc", "-std=c11", "-I", os.path.join(root, "include"), str(src), "-o", str(tmp_path / "s")], check=True)
    out = [int(x) for x in subprocess.run([str(tmp_path / "s")], capture_output=True, text=True, check=True).stdout.split()]
    cls = _lib.LzStripeFix
    assert out[0] == ctypes.sizeof(cls) == FIX.itemsize == 16
    assert out[1] == ctypes.alignment(cls) == 4
    assert out[2:6] == [getattr(cls, f).offset for f, _ in cls._fields_] == [FIX.fields[f][1] for f in FIX.names]
    assert [f for f, _ in cls._fields_] == list(FIX.names)
    assert out[6:] == [_lib.FIX_CLEAN, _lib.FIX_CORRECTED, _lib.FIX_UNEXPLAINED, _lib.FIX_CRC_CONFLICT]
