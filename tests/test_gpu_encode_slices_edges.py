"""The one-pass multi-slice encode (lzgpu_encode_slices*, fused_slices_kernel<M>) at the limits of its tables, on the GPU.

The rows are EDGE of tests/test_encode_slices_edges.py, whose literal plans are checked there against the planner and a plain-Python
restatement: 128 stripes per unit with 16 GF items per thread, 512 CRC streams, the shared memory 392 bytes under the cap, 336 staged
parity rows, four slices with parity, 12 GF warps beside parity rows, the standard slice in slots 1 and 3.  Each row runs at its
literal block count, at a ragged count whose last unit is partial (so that the last stripe of each slice is short or wholly past
pb_i) and with a chunk length that is not a block multiple, and at nb < L; each on the default context and with LZGPU_GRID_CAP = 1
and 2.

Every call is the _dev form at a different padded parity and CRC stride per slice, at 16-byte (not 256-byte) aligned bases, with
4 KiB guard bytes around every buffer; every byte outside the outputs must be unchanged and the partial block zero-filled in the
data buffer.  The expected bytes are the per-slice route (LZGPU_DISABLE_FUSED=1), which must equal lzgpu_encode_chunks per slice and
the oracle's encode_chunk (chunk 0 and the last at 64 MiB, every chunk below), and whose data CRCs must equal zlib.crc32 of the
zero-extended blocks.  The launch geometry must be the plan's.  Rows A, F and G also run through the host-pointer form, A and G
through a three-context pool, A and C with CRCs disabled."""
import os
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import _oracle as O
from tests.test_encode_slices_edges import EDGE, edge_goals, plan_lib, plan_model

pytestmark = pytest.mark.gpu
BLOCK = 65536
FAKE_CRC = 0xFEDCBA98           # LZGPU_FAKE_CRC: every CRC with CRCs disabled
GUARD, OFF = 4096, 4096 + 48    # guard bytes before and after every buffer; bases 16-byte but not 256-byte aligned
CTX = ["default", "cap1", "cap2"]
ROWS = {r[0]: r for r in EDGE}

_engines = {}


def engine(kind):
    env = {"default": {}, "cap1": {"LZGPU_GRID_CAP": "1"}, "cap2": {"LZGPU_GRID_CAP": "2"}, "per_slice": {"LZGPU_DISABLE_FUSED": "1"}}[kind]
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
    _want.clear()


def slice_types(names):
    return [L.SliceType(2, 1, 0) if n == "std" else L.SliceType(n) for n in names]


def cases(row):
    """(case id, blocks per chunk, chunk length): the row's literal count; a ragged count 2R + r whose last unit holds r < R blocks
    (r odd, so that a k = 2 slice's last stripe is short too), with a partial last block; nb < L"""
    rid, names, n, nb, plan = row
    out = [("nb%d" % nb, nb, nb * BLOCK)]
    if nb >= 1000:
        Lc, R = plan[2], plan[2] * plan[3]
        r = min((R // 2 + 1) | 1, R - 1) if R > 2 else 1
        out.append(("ragged", 2 * R + r, (2 * R + r - 1) * BLOCK + 12345))
        small = Lc - 1 if Lc > 2 else 1
        out.append(("small", small, small * BLOCK - 777))
    return out


def rnd(nbytes, seed):
    return np.frombuffer(bytearray(np.random.default_rng(seed).bytes(nbytes)), dtype=np.uint8)


_want = {}
_oracle_cache = {}


def want_of(rid, case):
    """(data, expected per slice) for a row and case, checked once: the per-slice route against lzgpu_encode_chunks per slice, the
    oracle's encode_chunk and zlib"""
    key = (rid, case[0])
    if key in _want:
        return _want[key]
    _want.clear()
    _oracle_cache.clear()
    _, names, n, _, _ = ROWS[rid]
    _, nb, chunk_len = case
    goals = slice_types(names)
    data = rnd(n * chunk_len, zlib.crc32(repr(key).encode())).reshape(n, chunk_len)
    want = engine("per_slice").encode_slices(goals, data)
    padded = np.zeros((n, nb * BLOCK), dtype=np.uint8)
    padded[:, :chunk_len] = data
    dcrc = np.array([[zlib.crc32(padded[c, b * BLOCK:(b + 1) * BLOCK]) for b in range(nb)] for c in range(n)], dtype=np.uint32)
    oracle = O.load_oracle()
    check = [0, n - 1] if nb == 1024 else range(n)
    for i, (g, (par, crc)) in enumerate(zip(goals, want)):
        assert np.array_equal(crc[:, :nb], dcrc), f"slice {i}: data CRCs differ from zlib"
        if g.is_std:
            assert par is None and crc.shape == (n, nb)
            continue
        p1, c1 = engine("default").encode_chunks(g, data)
        assert np.array_equal(p1, par) and np.array_equal(c1, crc), f"slice {i}: lzgpu_encode_chunks differs"
        for c in check:
            ok = (g.kind, g.k, g.m, c)
            if ok not in _oracle_cache:
                _oracle_cache[ok] = oracle.encode_chunk(g.kind, g.k, g.m, data[c])
            p_ref, c_ref = _oracle_cache[ok]
            assert np.array_equal(par[c].reshape(g.m, -1), p_ref) and np.array_equal(crc[c], c_ref), f"slice {i} chunk {c}: oracle"
    _want[key] = (data, want)
    return _want[key]


def assert_same(got, want):
    assert len(got) == len(want)
    for i, ((gp, gc), (wp, wc)) in enumerate(zip(got, want)):
        assert (gp is None) == (wp is None), i
        if gp is not None:
            assert np.array_equal(gp, wp), f"slice {i}: parity differs"
        assert np.array_equal(gc, wc), f"slice {i}: CRCs differ"


def check_geometry(eng, names, n, nb, ctx, whole_batch=True):
    """the context's last launch against the plan; whole_batch=False: a host-pointer call, whose last launch may cover only its last
    tile of chunks (units not compared)"""
    goals = edge_goals(names)
    plan = plan_lib(goals, n, nb)
    assert plan == plan_model(goals, n, nb) and plan[0] == 1
    _, _, _, G, threads, stages, _, smem, units = plan
    geo = eng.last_geometry()
    assert (geo["kernel"], geo["G"], geo["threads"], geo["stages"], geo["smem_bytes"]) == (_lib.KERNEL_ENCODE_SLICES, G, threads, stages, smem)
    assert geo["units"] == units or not whole_batch
    cap = {"default": None, "cap1": 1, "cap2": 2}[ctx]
    if cap:
        assert geo["grid"] == min(cap, units)
    return plan


DEV_CASES = [pytest.param(rid, case, ctx, id=f"{rid}-{case[0]}-{ctx}") for rid in ROWS for case in cases(ROWS[rid]) for ctx in CTX]


@pytest.mark.parametrize("rid,case,ctx", DEV_CASES)
def test_edge_row_dev_form(rid, case, ctx):
    _, names, n, _, _ = ROWS[rid]
    _, nb, chunk_len = case
    data, want = want_of(rid, case)
    eng = engine(ctx)
    goals = slice_types(names)
    dstride = nb * BLOCK + 1024
    dbuf = torch.full((2 * GUARD + n * dstride,), 0x3C, dtype=torch.uint8, device="cuda")
    for c in range(n):
        dbuf[OFF + c * dstride: OFF + c * dstride + chunk_len] = torch.from_numpy(data[c]).cuda()
    bufs, par_ptr, par_stride, crc_ptr, crc_stride = [], [], [], [], []
    for i, g in enumerate(goals):
        npb = -(-nb // g.k)
        m = 0 if g.is_std else g.m
        ps = m * npb * BLOCK + 2048 * (i + 1) if m else 0                   # a different padding per slice
        cs = nb + m * npb + 3 + 2 * i
        pbuf = torch.full((2 * GUARD + n * ps,), 0x5A + i, dtype=torch.uint8, device="cuda") if m else None
        cbuf = torch.full((2 * GUARD // 4 + n * cs,), 0x11223344 + i, dtype=torch.int32, device="cuda")
        bufs.append((pbuf, ps, cbuf, cs, m, npb))
        par_ptr.append(pbuf.data_ptr() + OFF if m else 0)
        par_stride.append(ps)
        crc_ptr.append(cbuf.data_ptr() + OFF)
        crc_stride.append(cs)
    before = eng.stats()["chunks_encoded"]
    torch.cuda.synchronize()        # the fills and copies above run on torch's stream; the call runs on the context's own stream
    eng.encode_slices_dev(goals, n, chunk_len, dbuf.data_ptr() + OFF, dstride, par_ptr, par_stride, crc_ptr, crc_stride)
    torch.cuda.synchronize()
    check_geometry(eng, names, n, nb, ctx)
    assert eng.stats()["chunks_encoded"] == before + n
    host = dbuf.cpu().numpy()
    assert (host[:OFF] == 0x3C).all() and (host[OFF + n * dstride:] == 0x3C).all()
    for c in range(n):
        row = host[OFF + c * dstride: OFF + (c + 1) * dstride]
        assert np.array_equal(row[:chunk_len], data[c]), f"chunk {c}: data changed"
        assert (row[chunk_len: nb * BLOCK] == 0).all(), f"chunk {c}: partial block not zero-filled"
        assert (row[nb * BLOCK:] == 0x3C).all(), f"chunk {c}: stride padding written"
    for i, ((pbuf, ps, cbuf, cs, m, npb), (wp, wc)) in enumerate(zip(bufs, want)):
        if m:
            ph = pbuf.cpu().numpy()
            assert (ph[:OFF] == 0x5A + i).all() and (ph[OFF + n * ps:] == 0x5A + i).all(), f"slice {i}: parity guard written"
            for c in range(n):
                prow = ph[OFF + c * ps: OFF + (c + 1) * ps]
                assert np.array_equal(prow[: m * npb * BLOCK], wp[c].reshape(-1)), f"slice {i} chunk {c}: parity differs"
                assert (prow[m * npb * BLOCK:] == 0x5A + i).all(), f"slice {i} chunk {c}: parity stride padding written"
        ch = cbuf.cpu().numpy().view(np.uint32)
        cw, fill = OFF // 4, 0x11223344 + i
        assert (ch[:cw] == fill).all() and (ch[cw + n * cs:] == fill).all(), f"slice {i}: CRC guard written"
        for c in range(n):
            crow = ch[cw + c * cs: cw + (c + 1) * cs]
            assert np.array_equal(crow[: nb + m * npb], wc[c]), f"slice {i} chunk {c}: CRCs differ"
            assert (crow[nb + m * npb:] == fill).all(), f"slice {i} chunk {c}: CRC stride padding written"


HOST_CASES = [pytest.param(rid, case, id=f"{rid}-{case[0]}") for rid in ("A", "F", "G") for case in cases(ROWS[rid])[:2]]


@pytest.mark.parametrize("rid,case", HOST_CASES)
def test_edge_row_host_form(rid, case):
    _, names, n, _, _ = ROWS[rid]
    data, want = want_of(rid, case)
    eng = engine("default")
    before = eng.stats()["chunks_encoded"]
    got = eng.encode_slices(slice_types(names), data)
    assert eng.stats()["chunks_encoded"] == before + n
    check_geometry(eng, names, n, case[1], "default", whole_batch=False)
    assert_same(got, want)


@pytest.mark.parametrize("rid", ["A", "G"])
def test_pool_of_three_contexts(rid):
    """seven chunks over three contexts on one device: shares of 3, 2 and 2 chunks"""
    _, names, _, _, _ = ROWS[rid]
    _, nb, chunk_len = cases(ROWS[rid])[1]
    goals = slice_types(names)
    data = rnd(7 * chunk_len, 41).reshape(7, chunk_len)
    pool = L.Pool([0, 0, 0])
    try:
        got = pool.encode_slices(goals, data)
        assert pool.stats()["chunks_encoded"] == 7
    finally:
        pool.close()
    assert_same(got, engine("per_slice").encode_slices(goals, data))


@pytest.mark.parametrize("rid", ["A", "C"])
def test_crcs_disabled(rid):
    _, names, n, _, _ = ROWS[rid]
    case = cases(ROWS[rid])[1]
    data, want = want_of(rid, case)
    eng = engine("default")
    eng.lib.lzgpu_set_crc_enabled(0)
    try:
        got = eng.encode_slices(slice_types(names), data)
        check_geometry(eng, names, n, case[1], "default", whole_batch=False)
    finally:
        eng.lib.lzgpu_set_crc_enabled(1)
    for (gp, gc), (wp, wc) in zip(got, want):
        assert gc.shape == wc.shape and (gc == FAKE_CRC).all()
        assert gp is None or np.array_equal(gp, wp)
