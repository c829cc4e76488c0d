"""The one-pass encode for several slices (lzgpu_encode_slices*, fused_slices_kernel in csrc/slices_kernel.cuh) on the GPU.

For every xor/ec slice, parity and CRCs must equal lzgpu_encode_chunks for that slice on the same data, byte for byte; the standard
slice's CRCs must equal lzgpu_crc_blocks of the zero-extended blocks; and a sample of chunks must equal the oracle's encode.  Covered:
the goal sets of the issue that motivated the call (fused and refused ones), lengths from one block to 64 MiB, every fused geometry
of the plan table (tests/test_encode_slices_plan.py) checked against lzgpu_debug_last_geometry, several units per CTA
(LZGPU_GRID_CAP = 1 and 3), the per-slice route (LZGPU_DISABLE_FUSED=1), the _dev form at padded strides with offset buffers and
guard bytes, CRCs disabled, a host batch over three tiles, a two-context pool, argument refusals and the statistics."""
import os

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200.engine import LzGpuError
from tests.test_encode_slices_plan import PLAN_TABLE

pytestmark = pytest.mark.gpu
BLOCK = 65536
CHUNK = 1024 * BLOCK
FAKE_CRC = 0xFEDCBA98           # LZGPU_FAKE_CRC: every CRC with CRCs disabled

SETS = [
    ("xor2", "xor3"), ("ec(3,2)", "ec(8,2)"), ("std", "xor2", "xor3"), ("ec(8,2)", "ec(8,4)"), ("ec(5,3)", "ec(4,2)"),
    ("ec(8,3)", "ec(6,4)"), ("ec(7,2)", "ec(9,2)"), ("ec(8,2)",), ("std", "ec(8,2)"),
    ("ec(8,2)", "ec(9,2)"), ("ec(8,2)", "ec(10,5)"),          # refused: L = 72; a Cauchy slice
]

_engines = {}


def engine(kind):
    env = {"default": {}, "cap1": {"LZGPU_GRID_CAP": "1"}, "cap3": {"LZGPU_GRID_CAP": "3"}, "per_slice": {"LZGPU_DISABLE_FUSED": "1"}}[kind]
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


def lcm_of(names):
    out = 1
    for g in goals_of(names):
        if not g.is_std:
            out = out * g.k // np.gcd(out, g.k)
    return out


def rnd(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, size=shape, dtype=np.uint8)


def per_slice(eng, goals, data, chunk_len):
    """the reference: lzgpu_encode_chunks per xor/ec slice, lzgpu_crc_blocks of the zero-extended blocks for the standard slice"""
    out = []
    nb = -(-chunk_len // BLOCK)
    for g in goals:
        if g.is_std:
            padded = np.zeros((data.shape[0], nb * BLOCK), dtype=np.uint8)
            padded[:, :chunk_len] = data[:, :chunk_len]
            out.append((None, eng.crc_blocks(padded).reshape(data.shape[0], nb)))
        else:
            out.append(eng.encode_chunks(g, data, chunk_len=chunk_len))
    return out


def assert_same(got, want):
    assert len(got) == len(want)
    for i, ((gp, gc), (wp, wc)) in enumerate(zip(got, want)):
        assert (gp is None) == (wp is None), i
        if gp is not None:
            assert np.array_equal(gp, wp), f"slice {i}: parity differs"
        assert np.array_equal(gc, wc), f"slice {i}: CRCs differ"


def lengths(names):
    Lc = lcm_of(names)
    return [(2, CHUNK), (3, min(3 * Lc + 1, 1024) * BLOCK), (2, (2 * Lc) * BLOCK + 12345), (3, BLOCK), (12, Lc * BLOCK)]


CASES = [pytest.param(names, n, clen, id="+".join(names) + f"-n{n}-len{clen}") for names in SETS for n, clen in lengths(names)]


@pytest.mark.parametrize("names,n,chunk_len", CASES)
def test_goal_sets_match_per_slice_encode_and_oracle(oracle, names, n, chunk_len):
    eng = engine("default")
    goals = goals_of(names)
    data = rnd((n, chunk_len), n * 7 + chunk_len % 1000)
    got = eng.encode_slices(goals, data)
    assert_same(got, per_slice(eng, goals, data, chunk_len))
    for c in sorted({0} if chunk_len == CHUNK else {0, n - 1}):
        for g, (par, crc) in zip(goals, got):
            if g.is_std:
                continue
            p_ref, c_ref = oracle.encode_chunk(g.kind, g.k, g.m, data[c])
            assert np.array_equal(par[c].reshape(g.m, -1), p_ref) and np.array_equal(crc[c], c_ref)


@pytest.mark.parametrize("names", [s for s in SETS if len(s) > 1], ids="+".join)
def test_per_slice_route_gives_the_same_bytes(names):
    goals = goals_of(names)
    n, chunk_len = 3, (3 * lcm_of(names) + 1) * BLOCK + 999
    data = rnd((n, chunk_len), 5)
    assert_same(engine("default").encode_slices(goals, data), engine("per_slice").encode_slices(goals, data))


FUSED_TABLE = [e for e in PLAN_TABLE if e[3][0] == 1]


@pytest.mark.parametrize("ctx", ["default", "cap1", "cap3"])
@pytest.mark.parametrize("entry", FUSED_TABLE, ids=lambda e: "+".join(e[0]) + f"-n{e[1]}-nb{e[2]}")
def test_every_planned_geometry(entry, ctx):
    names, n, nb, plan = entry
    _, _, Lc, G, threads, stages, _, smem, units = plan
    eng = engine(ctx)
    goals = goals_of(names)
    data = rnd((n, nb * BLOCK), nb + n)
    d_data = torch.from_numpy(data).cuda()
    outs, par_ptr, par_stride, crc_ptr, crc_stride = [], [], [], [], []
    for g in goals:
        npb = -(-nb // g.k)
        m = 0 if g.is_std else g.m
        par = torch.full((n, max(m, 1) * npb * BLOCK), 0xA5, dtype=torch.uint8, device="cuda")
        crc = torch.zeros((n, nb + m * npb), dtype=torch.int32, device="cuda")
        outs.append((par, crc, m))
        par_ptr.append(0 if g.is_std else par.data_ptr())
        par_stride.append(0 if g.is_std else par.shape[1])
        crc_ptr.append(crc.data_ptr())
        crc_stride.append(crc.shape[1])
    eng.encode_slices_dev(goals, n, nb * BLOCK, d_data.data_ptr(), nb * BLOCK, par_ptr, par_stride, crc_ptr, crc_stride)
    torch.cuda.synchronize()
    geo = eng.last_geometry()
    cap = {"default": None, "cap1": 1, "cap3": 3}[ctx]
    assert (geo["kernel"], geo["G"], geo["threads"], geo["stages"], geo["smem_bytes"], geo["units"]) == \
        (_lib.KERNEL_ENCODE_SLICES, G, threads, stages, smem, units)
    if cap:
        assert geo["grid"] == min(cap, units)
    want = per_slice(engine("default"), goals, data, nb * BLOCK)
    got = [(None if m == 0 else par.cpu().numpy().reshape(n, m, -1), crc.cpu().numpy().view(np.uint32)) for par, crc, m in outs]
    assert_same(got, want)


def test_dev_form_at_padded_strides_with_guard_bytes():
    eng = engine("default")
    names = ("std", "ec(3,2)", "ec(8,2)")
    goals = goals_of(names)
    n, chunk_len = 3, 50 * BLOCK + 4321
    nb = 51
    data = rnd((n, chunk_len), 11)
    GUARD, OFF = 4096, 4096 + 48                                  # offset buffers (16-byte aligned, not 256), guard bytes around
    dstride = nb * BLOCK + 1024
    dbuf = torch.full((2 * GUARD + n * dstride,), 0x3C, dtype=torch.uint8, device="cuda")
    for c in range(n):
        dbuf[OFF + c * dstride: OFF + c * dstride + chunk_len] = torch.from_numpy(data[c]).cuda()
    bufs, par_ptr, par_stride, crc_ptr, crc_stride = [], [], [], [], []
    for g in goals:
        npb = -(-nb // g.k)
        m = 0 if g.is_std else g.m
        ps = m * npb * BLOCK + 2048
        cs = nb + m * npb + 5
        pbuf = torch.full((2 * GUARD + n * ps,), 0x5A, dtype=torch.uint8, device="cuda")
        cbuf = torch.full((2 * GUARD // 4 + n * cs,), 0x11223344, dtype=torch.int32, device="cuda")
        bufs.append((pbuf, ps, cbuf, cs, m, npb))
        par_ptr.append(0 if g.is_std else pbuf.data_ptr() + OFF)
        par_stride.append(ps)
        crc_ptr.append(cbuf.data_ptr() + OFF)
        crc_stride.append(cs)
    eng.encode_slices_dev(goals, n, chunk_len, dbuf.data_ptr() + OFF, dstride, par_ptr, par_stride, crc_ptr, crc_stride)
    torch.cuda.synchronize()
    want = per_slice(eng, goals, data, chunk_len)
    host = dbuf.cpu().numpy()
    assert (host[:OFF] == 0x3C).all() and (host[OFF + n * dstride:] == 0x3C).all()
    for c in range(n):
        row = host[OFF + c * dstride: OFF + (c + 1) * dstride]
        assert np.array_equal(row[:chunk_len], data[c]) and (row[chunk_len: nb * BLOCK] == 0).all() and (row[nb * BLOCK:] == 0x3C).all()
    for (pbuf, ps, cbuf, cs, m, npb), (wp, wc) in zip(bufs, want):
        ph, ch = pbuf.cpu().numpy(), cbuf.cpu().numpy().view(np.uint32)
        cw = OFF // 4
        if m:
            assert (ph[:OFF] == 0x5A).all() and (ph[OFF + n * ps:] == 0x5A).all()
        for c in range(n):
            if m:
                prow = ph[OFF + c * ps: OFF + (c + 1) * ps]
                assert np.array_equal(prow[: m * npb * BLOCK], wp[c].reshape(-1)) and (prow[m * npb * BLOCK:] == 0x5A).all()
            crow = ch[cw + c * cs: cw + (c + 1) * cs]
            assert np.array_equal(crow[: nb + m * npb], wc[c]) and (crow[nb + m * npb:] == 0x11223344).all()
        assert (ch[:cw] == 0x11223344).all() and (ch[cw + n * cs:] == 0x11223344).all()


def test_crcs_disabled():
    eng = engine("default")
    goals = goals_of(("std", "xor2", "ec(5,3)"))
    data = rnd((2, 31 * BLOCK + 5), 3)
    eng.lib.lzgpu_set_crc_enabled(0)
    try:
        got = eng.encode_slices(goals, data)
        want = per_slice(eng, goals, data, data.shape[1])
    finally:
        eng.lib.lzgpu_set_crc_enabled(1)
    for (gp, gc), (wp, _) in zip(got, want):
        assert (gc == FAKE_CRC).all()
        assert gp is None or np.array_equal(gp, wp)


def test_host_batch_over_three_tiles():
    eng = engine("default")
    goals = goals_of(("ec(3,2)", "ec(8,2)", "std"))
    data = rnd((5, CHUNK), 17)                                   # 128 MiB host tiles: two 64 MiB chunks per tile
    assert_same(eng.encode_slices(goals, data), per_slice(eng, goals, data, CHUNK))


def test_pool_of_two_contexts_on_one_device():
    pool = L.Pool([0, 0])
    try:
        goals = goals_of(("xor2", "xor3", "std"))
        data = rnd((7, 40 * BLOCK + 100), 23)
        assert_same(pool.encode_slices(goals, data), per_slice(engine("default"), goals, data, data.shape[1]))
    finally:
        pool.close()


def test_argument_refusals_launch_nothing():
    eng = engine("default")
    data = rnd((1, 8 * BLOCK), 1)
    before = eng.stats()["kernel_launches"]
    bad_sets = [goals_of(("xor2", "xor3", "xor4", "xor5", "xor6")), goals_of(("std",)), []]
    for goals in bad_sets:
        with pytest.raises(LzGpuError):
            eng.encode_slices(goals, data)
    d = torch.zeros(8 * BLOCK + 16, dtype=torch.uint8, device="cuda")
    p = torch.zeros(2 * 4 * BLOCK + 16, dtype=torch.uint8, device="cuda")
    c = torch.zeros(64, dtype=torch.int32, device="cuda")
    goals = goals_of(("xor2", "ec(4,2)"))
    args = dict(par=[p.data_ptr(), p.data_ptr()], ps=[4 * BLOCK, 8 * BLOCK], crc=[c.data_ptr(), c.data_ptr()], cs=[12, 12])
    for data_ptr, stride, ps in [(d.data_ptr() + 8, 8 * BLOCK, args["ps"]),          # data not 16-byte aligned
                                 (d.data_ptr(), 8 * BLOCK - 16, args["ps"]),         # chunk stride smaller than the blocks
                                 (d.data_ptr(), 8 * BLOCK, [4 * BLOCK, 4 * BLOCK - 16])]:  # parity stride too small
        with pytest.raises(LzGpuError):
            eng.encode_slices_dev(goals, 1, 8 * BLOCK, data_ptr, stride, args["par"], ps, args["crc"], args["cs"])
    with pytest.raises(LzGpuError):
        eng.encode_slices_dev(goals, 1, 8 * BLOCK, d.data_ptr(), 8 * BLOCK, [p.data_ptr(), 0], args["ps"], args["crc"], args["cs"])
    with pytest.raises(LzGpuError):                                                  # an empty batch is checked like any other, by the one-goal call too
        eng.encode_chunks_dev(goals[0], 0, 8 * BLOCK, d.data_ptr(), 8 * BLOCK - 16, p.data_ptr(), 4 * BLOCK, c.data_ptr(), 12)
    torch.cuda.synchronize()
    assert eng.stats()["kernel_launches"] == before


@pytest.mark.parametrize("ctx", ["default", "per_slice"])
def test_statistics(ctx):
    eng = engine(ctx)
    names = ("std", "ec(3,2)", "ec(8,2)")
    goals = goals_of(names)
    n, nb = 3, 1024
    d = torch.from_numpy(rnd((n, nb * BLOCK), 2)).cuda()
    outs = []
    for g in goals:
        npb = -(-nb // g.k)
        m = 0 if g.is_std else g.m
        outs.append((torch.empty((n, max(m, 1) * npb * BLOCK), dtype=torch.uint8, device="cuda"), torch.empty((n, nb + m * npb), dtype=torch.int32, device="cuda")))
    eng.lib.lzgpu_reset_stats(eng.h)
    eng.encode_slices_dev(goals, n, nb * BLOCK, d.data_ptr(), nb * BLOCK, [0 if g.is_std else p.data_ptr() for g, (p, _) in zip(goals, outs)],
                          [0 if g.is_std else p.shape[1] for g, (p, _) in zip(goals, outs)], [c.data_ptr() for _, c in outs],
                          [c.shape[1] for _, c in outs])
    torch.cuda.synchronize()
    s = eng.stats()
    # one pass: 64 MiB read, ec(3,2) 2 x 342 and ec(8,2) 2 x 128 parity blocks, the CRC arrays of all three slices (issue table row 1 + std)
    assert s["chunks_encoded"] == n
    assert s["batch_bytes_last"] == n * (128724656 + 4 * 1024)
