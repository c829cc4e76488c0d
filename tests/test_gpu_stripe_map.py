"""lzgpu_check_stripe_map / _dev: the state of every stripe of every chunk, and the part to blame in each bad one.

Batches, fault injection (part bytes flipped, the block's stored CRC recomputed) and the device layouts come from
test_gpu_stripe_check.  The expected map is computed here on the CPU: the oracle re-encodes a chunk's data parts, the syndrome of
checked row r is the re-encoded parity XOR the stored parity, and a stripe's bad_rows are the rows with a non-zero syndrome in it.
The expected suspect comes from a numpy restatement of the column test written as 2x2 minors: data part j explains a stripe when
S_i * g_0j == S_0 * g_ij at every byte and row (g = the generator rows the oracle encodes with, read off a unit encode), parity part
k+r when every other checked row is zero; one such part, with two or more rows checked, is the suspect.  Every case runs on the fused
route and, with LZGPU_DISABLE_FUSED=1, on the generic route; both maps must be identical, the route is asserted through
last_geometry(), and each chunk's lowest bad stripe must equal lzgpu_check_stripes' verdict on both routes."""
import ctypes
import os
import subprocess
import zlib

import numpy as np
import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests.test_gpu_stripe_check import BLOCK, GOALS, ZERO_CRC, Batch, Dev, fused_goal, given_parts, nb_for

STATE = L.Engine.STRIPE_STATE_DTYPE
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


def fused_engine():
    return engine()


def generic_engine():
    return engine(LZGPU_DISABLE_FUSED=1)


# ---- the expected map, on the CPU ---------------------------------------------------------------
_mul = {}
_gen = {}


def gf_mul_table(oracle):
    if "t" not in _mul:
        _mul["t"] = np.array([[oracle.gf_mul(a, b) for b in range(256)] for a in range(256)], dtype=np.uint8)
    return _mul["t"]


def generator(oracle, b):
    """g[r][j]: the coefficient of data part j in parity row r, from one oracle encode (block j holds 1 at byte j, zeros elsewhere)"""
    key = (b.kind, b.k, b.m)
    if key not in _gen:
        chunk = np.zeros(b.k * BLOCK, dtype=np.uint8)
        for j in range(b.k):
            chunk[j * BLOCK + j] = 1
        parity, _ = oracle.encode_chunk(b.kind, b.k, b.m, chunk)
        _gen[key] = np.stack([parity[r][:b.k] for r in range(b.m)])
    return _gen[key]


def suspect_of(oracle, b, rows, syn):
    """syn [len(rows), 65536]: the syndromes of one bad stripe; the one part whose column explains them, else -1"""
    if len(rows) < 2:
        return -1
    mul, g = gf_mul_table(oracle), generator(oracle, b)
    fits = []
    for j in range(b.k):
        col = g[rows, j]
        if all((mul[syn[i], col[0]] == mul[syn[0], col[i]]).all() for i in range(1, len(rows))):
            fits.append(j)
    for i, r in enumerate(rows):
        if not np.delete(syn, i, axis=0).any():
            fits.append(b.k + r)
    return fits[0] if len(fits) == 1 else -1


def expected_map(oracle, b, rows):
    """[n, pb] of STATE: bad_rows and suspect per stripe, from the oracle's re-encode of every chunk"""
    out = np.zeros((b.n, b.pb), dtype=STATE)
    out["suspect_part"] = -1
    for c in range(b.n):
        blocks = np.stack([b.parts[j][c].reshape(b.pb, BLOCK) for j in range(b.k)], axis=1).reshape(-1, BLOCK)
        parity, _ = oracle.encode_chunk(b.kind, b.k, b.m, np.ascontiguousarray(blocks[:b.nb]).reshape(-1))
        syn = np.stack([(parity[r] ^ b.parts[b.k + r][c]).reshape(b.pb, BLOCK) for r in rows], axis=1)   # [pb, rows, B]
        for s in range(b.pb):
            bits = sum(1 << r for i, r in enumerate(rows) if syn[s, i].any())
            if bits:
                out[c, s] = (bits, suspect_of(oracle, b, rows, syn[s]))
    return out


# ---- runs -----------------------------------------------------------------------------------------
def as_list(m):
    return [[(int(x["bad_rows"]), int(x["suspect_part"])) for x in row] for row in m]


def invariant(smap, verdicts):
    """the lowest bad stripe of each chunk and its entry against lzgpu_check_stripes' verdict"""
    for c, v in enumerate(verdicts):
        bad = np.nonzero(smap[c]["bad_rows"])[0]
        first = (int(bad[0]), int(smap[c, bad[0]]["bad_rows"]), int(smap[c, bad[0]]["suspect_part"])) if len(bad) else (-1, 0, -1)
        assert first == (int(v["first_bad_stripe"]), int(v["bad_rows"]), int(v["suspect_part"])), (c, first, v)


def run_both(b, parts, crcs, expect_fused):
    """the host call on both routes, the invariant on each; returns the (identical) maps"""
    maps = []
    for eng, fused in ((fused_engine(), expect_fused), (generic_engine(), False)):
        before = eng.last_geometry()
        m = eng.check_stripe_map(b.goal, b.nb, parts, crcs)
        geo = eng.last_geometry()
        if fused:
            assert geo["kernel"] == _lib.KERNEL_CHECK
            assert geo["units"] == b.n * -(-b.pb // geo["G"])
        else:
            assert geo["kernel"] != _lib.KERNEL_CHECK or geo == before
        assert eng.status_slots()[1] == 0
        assert m.shape == (b.n, b.pb)
        invariant(m, eng.check_stripes(b.goal, b.nb, parts, crcs))
        maps.append(m)
    assert as_list(maps[0]) == as_list(maps[1]), "fused and generic routes disagree"
    return maps[0]


_batches = {}


def batch(oracle, text, n=3, seed=1):
    key = (text, n, seed)
    if key not in _batches:
        _batches[key] = Batch(oracle, text, n, nb_for(L.SliceType(text).k), seed)
    b = _batches[key]
    fresh = Batch.__new__(Batch)
    fresh.__dict__.update(b.__dict__)
    fresh.parts = [p.copy() for p in b.parts]
    fresh.crc = [c.copy() for c in b.crc]
    fresh.faulty = set()
    return fresh


def inject(b, fault):
    """faults by name; every one recomputes the block's stored CRC"""
    k, m, last = b.k, b.m, b.pb - 1
    if fault == "one_stripe":
        b.corrupt(1, 1, 1)
    elif fault == "stripes_blame_different_parts":   # the case a whole-part rebuild would spread
        b.corrupt(0, 0, 0)
        b.corrupt(0, k - 1, 1)
        b.corrupt(0, k + m - 1, 2)
    elif fault == "two_parts_one_stripe":
        b.corrupt(1, 0, 1, offset=100)
        b.corrupt(1, 1, 1, offset=100)
        b.corrupt(2, 0, 2, offset=100)
        b.corrupt(2, k, 2, offset=5000)
    elif fault == "short_last_stripe":               # nb = 2k + 1: only data part 0 has a block in the last stripe
        b.corrupt(2, 0, last, offset=65530, length=6)
    elif fault == "parity_parts":
        b.corrupt(1, k + m - 1, 0)
        b.corrupt(2, k, last)
    elif fault == "every_stripe":
        for s in range(b.pb):                        # data part 0 in the last stripe: the others are zero padding there
            b.corrupt(1, s % k if s < last else 0, s, offset=1000 * s)


FAULTS = ["none", "one_stripe", "stripes_blame_different_parts", "two_parts_one_stripe", "short_last_stripe", "parity_parts",
          "every_stripe"]
gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("fault", FAULTS)
@pytest.mark.parametrize("text", GOALS)
def test_map_matches_the_oracle(oracle, text, fault):
    b = batch(oracle, text)
    inject(b, fault)
    got = run_both(b, given_parts(b), b.crc, fused_goal(text))
    want = expected_map(oracle, b, list(range(b.m)))
    assert as_list(got) == as_list(want)
    if fault == "none":
        assert not got["bad_rows"].any()
    if fault == "every_stripe":
        assert (got[1]["bad_rows"] == (1 << b.m) - 1).all()
    if fault == "stripes_blame_different_parts" and b.m >= 2:
        assert list(got[0]["suspect_part"]) == [0, b.k - 1, b.k + b.m - 1]


@gpu
@pytest.mark.parametrize("text,skip", [("ec(5,3)", (6,)), ("ec(8,4)", (8,)), ("ec(8,4)", (9, 11)), ("ec(8,2)", (8,)),
                                       ("ec(4,4)", (4, 5, 6)), ("ec(6,5)", (7, 9))])
def test_missing_parity_rows_are_not_checked(oracle, text, skip):
    b = batch(oracle, text)
    rows = [r for r in range(b.m) if b.k + r not in skip]
    b.corrupt(0, 2, 1)
    b.corrupt(0, 3, 0)
    b.corrupt(2, b.k + rows[-1], 2)
    for p in skip:                                   # a fault in a part that is not given is not seen
        b.corrupt(1, p, 0)
    got = run_both(b, given_parts(b, skip), b.crc, fused_goal(text))
    want = expected_map(oracle, b, rows)
    assert as_list(got) == as_list(want)
    assert not got[1]["bad_rows"].any()
    assert got[0, 1]["bad_rows"] == got[0, 0]["bad_rows"] == sum(1 << r for r in rows)


@gpu
def test_missing_parts_are_refused(oracle):
    b = batch(oracle, "ec(5,3)")
    for eng in (fused_engine(), generic_engine()):
        launches = eng.stats()["kernel_launches"]
        for skip in ((0,), (5, 6, 7)):
            with pytest.raises(L.LzGpuError) as ei:
                eng.check_stripe_map(b.goal, b.nb, given_parts(b, skip), b.crc)
            assert ei.value.status == _lib.ERR_TOO_FEW_PARTS
        assert eng.stats()["kernel_launches"] == launches


@gpu
@pytest.mark.parametrize("text", ["ec(8,2)", "ec(5,3)", "xor3", "ec(6,5)"])
def test_stored_crc_failure_keeps_the_whole_map(oracle, text):
    b = batch(oracle, text)
    b.corrupt(2, 1, 1)
    b.corrupt(0, 0, 2)
    want = expected_map(oracle, b, list(range(b.m)))
    crcs = [c.copy() for c in b.crc]
    crcs[b.k][1, 2] ^= 0x40                          # (chunk 1, parity part 0, block 2)
    crcs[0][1, 0] ^= 0x40                            # the same chunk, a smaller part: this one is reported
    crcs[0][2, 0] ^= 0x40                            # a later chunk
    maps = []
    for eng in (fused_engine(), generic_engine()):
        with pytest.raises(L.ChunkCrcError) as ei:
            eng.check_stripe_map(b.goal, b.nb, given_parts(b), crcs)
        assert ei.value.where == (1, 0, 0)
        assert as_list(ei.value.map) == as_list(want)
        maps.append(as_list(ei.value.map))
        assert eng.status_slots()[1] == 0
    assert maps[0] == maps[1]


def run_dev(eng, b, dev, skip=(), crcs=True, guard=4096, lead=0):
    """the map of a resident batch into a guarded buffer; asserts nothing outside the n * pb entries changed"""
    torch = dev.torch
    size = 8 * b.n * b.pb
    init = np.random.default_rng(3).integers(0, 256, 2 * guard + lead + size, dtype=np.uint8)
    t = torch.from_numpy(init.copy()).cuda()
    parts = [None if i in skip else p for i, p in enumerate(dev.ptrs)]
    eng.check_stripe_map_dev(b.goal, b.n, b.nb, parts, dev.stride, dev.crcs if crcs else None, t.data_ptr() + guard + lead)
    torch.cuda.synchronize()
    after = t.cpu().numpy()
    o = guard + lead
    assert (after[:o] == init[:o]).all() and (after[o + size:] == init[o + size:]).all(), "write outside d_map"
    return after[o:o + size].copy().view(STATE).reshape(b.n, b.pb)


@gpu
@pytest.mark.parametrize("text", ["ec(8,2)", "ec(5,3)", "xor2", "ec(22,4)"])
@pytest.mark.parametrize("pad,lead", [(0, 0), (16, 20), (65536 + 48, 52)])
def test_dev_layouts_write_only_the_map(oracle, text, pad, lead):
    b = batch(oracle, text)
    b.corrupt(1, 2, 1)
    b.corrupt(1, b.k, 2)
    want = as_list(expected_map(oracle, b, list(range(b.m))))
    dev = Dev(b, pad, lead & ~15)
    got = []
    for eng, fused in ((fused_engine(), fused_goal(text)), (generic_engine(), False)):
        m = run_dev(eng, b, dev, lead=lead % 64)    # the map at 4-byte alignment only
        if fused:
            assert eng.last_geometry()["kernel"] == _lib.KERNEL_CHECK
        assert as_list(m) == want
        got.append(as_list(m))
    assert got[0] == got[1]
    for i, p in enumerate(b.parts):                  # every input byte unchanged
        host = dev.bufs[2 * i].cpu().numpy()
        base = lead & ~15
        for c in range(b.n):
            assert (host[base + c * dev.stride: base + c * dev.stride + p.shape[1]] == p[c]).all()


@gpu
def test_misaligned_map_is_refused_without_a_launch(oracle):
    import torch
    b = batch(oracle, "ec(8,2)")
    dev = Dev(b)
    out = torch.zeros(64 + 8 * b.n * b.pb, dtype=torch.uint8, device="cuda")
    for eng in (fused_engine(), generic_engine()):
        launches = eng.stats()["kernel_launches"]
        with pytest.raises(L.LzGpuError) as ei:
            eng.check_stripe_map_dev(b.goal, b.n, b.nb, dev.ptrs, dev.stride, dev.crcs, out.data_ptr() + 2)
        assert ei.value.status == _lib.ERR_ARG
        assert eng.stats()["kernel_launches"] == launches


@gpu
def test_deferred_mode_collects_the_crc_mismatch(oracle):
    b = batch(oracle, "ec(8,2)")
    b.corrupt(0, 4, 1)
    b.corrupt(0, 6, 0)
    want = as_list(expected_map(oracle, b, [0, 1]))
    b.crc[9][2, 1] ^= 1
    dev = Dev(b)
    for eng in (fused_engine(), generic_engine()):
        eng.set_deferred_verify(True)
        try:
            m = run_dev(eng, b, dev)                 # returns at once; the map is there once the stream has passed
            with pytest.raises(L.ChunkCrcError) as ei:
                eng.sync()
            assert ei.value.where == (2, 9, 1)
        finally:
            eng.set_deferred_verify(False)
        assert as_list(m) == want
        assert eng.status_slots()[1] == 0


@gpu
@pytest.mark.parametrize("cap", [1, 3])
@pytest.mark.parametrize("text", ["ec(8,2)", "xor3", "ec(8,4)", "ec(5,3)"])
def test_capped_grid_resets_the_stripe_bits_per_unit(oracle, text, cap):
    """eight chunks, several units per CTA: a stripe's bits must not leak into the next unit's"""
    b = batch(oracle, text, n=8, seed=5)
    for c in (0, 3, 7):
        b.corrupt(c, c % b.k, c % b.pb)
    b.corrupt(5, b.k, 2)
    b.corrupt(6, 0, b.pb - 1)
    want = as_list(expected_map(oracle, b, list(range(b.m))))
    dev = Dev(b)
    eng = engine(LZGPU_GRID_CAP=cap)
    m = as_list(run_dev(eng, b, dev))
    grid, units = eng.last_launch()
    assert eng.last_geometry()["kernel"] == _lib.KERNEL_CHECK
    assert eng.last_geometry()["grid"] == cap and units > 2 * cap
    assert m == want == as_list(run_dev(generic_engine(), b, dev)) == as_list(run_dev(fused_engine(), b, dev))


@gpu
def test_host_tiles_report_batch_wide_chunks():
    """ec(8,2), one-stripe chunks: 823 chunks take three tiles (as in test_gpu_stripe_check).  Faults in tiles 1 and 2."""
    goal, k, m, nb, n = L.SliceType("ec(8,2)"), 8, 2, 8, 823
    parts = [np.zeros((n, BLOCK), dtype=np.uint8) for _ in range(k + m)]
    crcs = [np.full((n, 1), ZERO_CRC, dtype=np.uint32) for _ in range(k + m)]
    for c, p in ((500, 3), (820, 9)):
        parts[p][c, 10:14] = 0xA5
        crcs[p][c, 0] = zlib.crc32(parts[p][c].tobytes())
    for eng in (fused_engine(), generic_engine()):
        before = eng.stats()["batches_timed"]
        got = eng.check_stripe_map(goal, nb, parts, crcs)
        assert eng.stats()["batches_timed"] - before == 3
        assert got.shape == (n, 1)
        bad = {c: tuple(int(x) for x in got[c, 0]) for c in range(n) if got[c, 0]["bad_rows"]}
        assert bad == {500: (3, 3), 820: (2, 9)}
        assert (got["suspect_part"][got["bad_rows"] == 0] == -1).all()
        crcs2 = [c.copy() for c in crcs]
        crcs2[5][700, 0] ^= 1
        crcs2[0][20, 0] ^= 1
        with pytest.raises(L.ChunkCrcError) as ei:
            eng.check_stripe_map(goal, nb, parts, crcs2)
        assert ei.value.where == (20, 0, 0)
        assert as_list(ei.value.map) == as_list(got)
        assert eng.status_slots()[1] == 0


def full_chunk(eng, goal, seed):
    """one 64 MiB chunk of a goal: parts [1, pb*64K] and stored CRCs [1, pb] per part"""
    k, m, nb = goal.k, goal.m, 1024
    pb = -(-nb // k)
    data = np.random.default_rng(seed).integers(0, 256, (1, nb * BLOCK), dtype=np.uint8)
    parity, crc = eng.encode_chunks(goal, data)
    padded = np.zeros((1, pb * k * BLOCK), dtype=np.uint8)
    padded[:, :nb * BLOCK] = data
    blocks = padded.reshape(1, pb, k, BLOCK)
    parts = [np.ascontiguousarray(blocks[:, :, j]).reshape(1, -1) for j in range(k)] + [np.ascontiguousarray(parity[:, r]) for r in range(m)]
    crcs = [np.array([[crc[0, s * k + j] if s * k + j < nb else ZERO_CRC for s in range(pb)]], dtype=np.uint32) for j in range(k)]
    crcs += [np.ascontiguousarray(crc[:, nb + r * pb: nb + (r + 1) * pb]) for r in range(m)]
    return parts, crcs


def corrupt_block(parts, crcs, part, s, offset, value=1):
    parts[part][0, s * BLOCK + offset] ^= value
    crcs[part][0, s] = zlib.crc32(parts[part][0, s * BLOCK:(s + 1) * BLOCK].tobytes())


@gpu
def test_one_full_size_chunk():
    goal = L.SliceType("ec(8,2)")
    parts, crcs = full_chunk(fused_engine(), goal, 11)
    for s, p in ((3, 1), (100, 5), (101, 5), (127, 9)):
        corrupt_block(parts, crcs, p, s, 65535 - s)
    maps = []
    for eng in (fused_engine(), generic_engine()):
        got = eng.check_stripe_map(goal, 1024, parts, crcs)
        invariant(got, eng.check_stripes(goal, 1024, parts, crcs))
        maps.append(as_list(got))
    assert fused_engine().last_geometry()["kernel"] == _lib.KERNEL_CHECK
    assert maps[0] == maps[1]
    bad = {s: e for s, e in enumerate(maps[0][0]) if e[0]}
    assert bad == {3: (3, 1), 100: (3, 5), 101: (3, 5), 127: (2, 9)}


@gpu
def test_repair_by_one_stripe_windows_restores_every_byte():
    """ec(8,2), one 64 MiB chunk, three bad stripes blaming three different parts: rebuilding any one part whole would read the
    corrupt blocks of the others, so each named block is rebuilt by a one-stripe window of lzgpu_recover_chunks_dev"""
    import torch
    goal, k, m, nb = L.SliceType("ec(8,2)"), 8, 2, 1024
    eng = fused_engine()
    parts, crcs = full_chunk(eng, goal, 12)
    original = [p.copy() for p in parts]
    for s, p in ((7, 2), (40, 6), (127, 8)):
        corrupt_block(parts, crcs, p, s, 4321, 0x3C)
    smap = eng.check_stripe_map(goal, nb, parts, crcs)
    bad = [(int(s), int(smap[0, s]["suspect_part"])) for s in np.nonzero(smap[0]["bad_rows"])[0]]
    assert bad == [(7, 2), (40, 6), (127, 8)]
    assert len({p for _, p in bad}) > 1                # the map's rule: not one part, so stripe by stripe
    dev = [torch.from_numpy(p[0]).cuda() for p in parts]
    out = torch.zeros(BLOCK, dtype=torch.uint8, device="cuda")
    for s, p in bad:
        window = [0 if i == p else dev[i].data_ptr() + s * BLOCK for i in range(k + m)]
        want = [1 if i == p else 0 for i in range(k + m)]
        d_out = [out.data_ptr() if i == p else 0 for i in range(k + m)]
        eng.recover_chunks_dev(goal, 1, min(k, nb - s * k), window, parts[0].shape[1], None, want, d_out)
        torch.cuda.synchronize()
        parts[p][0, s * BLOCK:(s + 1) * BLOCK] = out.cpu().numpy()
        crcs[p][0, s] = zlib.crc32(parts[p][0, s * BLOCK:(s + 1) * BLOCK].tobytes())
    for eng2 in (fused_engine(), generic_engine()):
        assert not eng2.check_stripe_map(goal, nb, parts, crcs)["bad_rows"].any()
    for p, o in zip(parts, original):
        assert (p == o).all()


def test_stripe_state_layout_matches_the_header(tmp_path):
    """(no GPU needed) the ctypes and numpy mirrors of lzgpu_stripe_state against sizeof / offsetof from include/lzgpu.h"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "s.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lzgpu.h"\nint main(void) { printf("%zu %zu %zu %zu\\n", '
                   'sizeof(lzgpu_stripe_state), _Alignof(lzgpu_stripe_state), offsetof(lzgpu_stripe_state, bad_rows), '
                   'offsetof(lzgpu_stripe_state, suspect_part)); return 0; }\n')
    subprocess.run(["gcc", "-std=c11", "-I", os.path.join(root, "include"), str(src), "-o", str(tmp_path / "s")], check=True)
    out = [int(x) for x in subprocess.run([str(tmp_path / "s")], capture_output=True, text=True, check=True).stdout.split()]
    cls = _lib.LzStripeState
    assert out[0] == ctypes.sizeof(cls) == STATE.itemsize == 8
    assert out[1] == ctypes.alignment(cls) == 4
    assert out[2:] == [getattr(cls, f).offset for f, _ in cls._fields_] == [STATE.fields[f][1] for f in STATE.names]
    assert [f for f, _ in cls._fields_] == list(STATE.names)
