"""The chunkserver's block path at every byte-range class, across its staging tiles and with many requests per CTA.

Every chunkserver write goes through lzgpu_write_blocks / _dev (block_write_kernel), every block CRC through lzgpu_crc_blocks / _dev
/ lzgpu_pool_crc_blocks (crc_blocks_kernel, or the fused CRC route for dense 64 KiB blocks) and every scrub through
lzgpu_verify_blocks / _interleaved / _moosefs (verify_common: crc_compare_kernel, then sparse_confirm_kernel).  A wrong answer here
stores a bad CRC or calls good data damaged, and nothing above this path can notice.

References: zlib.crc32 (mycrc32 is the standard CRC-32) and `hdd_write` below, a plain restatement of the batched hdd_write contract
in include/lzgpu.h, itself checked against the oracle's transcription of hddspacemgr.cc (O.hdd_write_block, on the compiled
reference where oracle/_ref exists).  The oracle always applies the sparse rule, so the sparse_rule = 0 cases rest on the
restatement alone.

  - Writes: every offset / size class (around 4-byte words, 16-byte loads, the kernel's 256 payload segments, 4 KiB and the block
    end), the refused ranges, crossed with exists, sparse_rule, five stored states (valid, damaged, a hole stored with 0, a
    non-zero block stored with 0, a non-zero block with the zero block's CRC stored with 0) and right or corrupt packets; one call
    with five requests per CTA in which every CTA meets every outcome one after another, through the host and the _dev form; and
    8192 + 300 requests, so that the host form stages two tiles and must return the first failure in request order.
  - CRCs: every length regime of crc_blocks_kernel (words per lane, front padding, lane 0's byte tail), odd host strides, more
    blocks than warps, more than two 128 MiB host staging tiles, pool shares at odd strides, and CRCs disabled.
  - Scrubs: the sparse rule at short lengths (the zero CRC of the length, the byte tail of sparse_confirm_kernel), more holes
    than CTAs, the smallest failing index of the two kernels, a batch across the 1 GiB staging tile (host and pool forms), the
    MooseFS format at its largest block count for every data_parts, and CRCs disabled.

64 KiB blocks run on the fused and on the generic route (a context created with LZGPU_DISABLE_FUSED=1).  Argument refusals asked
of the library here are host-side checks made before any launch, and no _dev request names a block outside its device array."""
import ctypes as C
import functools
import os
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import _oracle as O

pytestmark = pytest.mark.gpu
BLOCK = 65536
ZERO64 = zlib.crc32(bytes(BLOCK))            # 0xD7978EEB
FAKE = 0xFEDCBA98                            # every CRC while CRCs are disabled (LZGPU_FAKE_CRC)
OK, ARG, CRC, DAMAGED = _lib.OK, _lib.ERR_ARG, _lib.ERR_CRC, _lib.ERR_DAMAGED
ORACLE_CODE = {0: OK, -1: ARG, -3: CRC, -4: DAMAGED}
LENGTHS = [1, 2, 3, 4, 5, 127, 128, 129, 131, 132, 4095, 4096, 4097, 65532, 65533, 65535, 65536]


# ---- references ------------------------------------------------------------------------------------------------------------------
POLY = 0xEDB88320


def mulmod(a, b):
    """a * b mod P, bit-reflected (bit 31 is x^0), as zlib's multmodp"""
    p, m = 0, 0x80000000
    while m:
        if a & m:
            p ^= b
        b = (b >> 1) ^ POLY if b & 1 else b >> 1
        m >>= 1
    return p


@functools.lru_cache(maxsize=None)
def xpow8(n):
    """x^(8n) mod P"""
    acc, sq = 0x80000000, 0x00800000
    while n:
        if n & 1:
            acc = mulmod(acc, sq)
        sq = mulmod(sq, sq)
        n >>= 1
    return acc


def combine(crc1, crc2, len2):
    """mycrc32_combine: CRC of A || B from CRC(A), CRC(B) and |B|"""
    return mulmod(crc1, xpow8(len2)) ^ crc2


def crc_of_zeros(n):
    return zlib.crc32(bytes(n))


def hdd_write(block, stored, offset, size, crc, payload, exists, sparse_rule):
    """One request of the batched hdd_write, restated from include/lzgpu.h: (status, block after, stored CRC after)."""
    if size > BLOCK or offset >= BLOCK or offset + size > BLOCK:
        return ARG, block, stored
    data = np.asarray(payload, dtype=np.uint8)[:size]
    if zlib.crc32(data.tobytes()) != crc:                     # the packet's own CRC
        return CRC, block, stored
    if offset == 0 and size == BLOCK:                         # whole block: the packet CRC is stored, nothing is read
        return OK, data.copy(), crc
    old = block if exists else np.zeros(BLOCK, dtype=np.uint8)  # a block beyond the end of the file is created as zeros
    end = offset + size
    pre, under, post = (zlib.crc32(old[a:b].tobytes()) for a, b in ((0, offset), (offset, end), (end, BLOCK)))
    if exists:
        have = stored
        if sparse_rule and have == 0 and not old.any():       # a hole stored with 0 counts as the zero block's CRC
            have = ZERO64
        if combine(combine(pre, under, size), post, BLOCK - end) != have:
            return DAMAGED, block, stored
    new = old.copy()
    new[offset:end] = data
    return OK, new, combine(combine(pre, crc, size), post, BLOCK - end)


def crcs_of(rows):
    return np.array([zlib.crc32(r.tobytes()) for r in rows], dtype=np.uint32)


def forge(block, free, target):
    """A copy of `block`, not all zero, whose bytes at the positions `free` are solved for so that its CRC-32 is `target`.
    The CRC is affine in those 8 * len(free) bits (32 equations); with more than 4 free bytes the solution is not unique, and a
    non-zero combination that leaves the CRC alone is added when the solution alone would give the zero block."""
    blk = np.array(block, dtype=np.uint8, copy=True)
    blk[free] = 0
    base = zlib.crc32(blk.tobytes())
    cols = []
    for p in free:
        for bit in range(8):
            blk[p] = 1 << bit
            cols.append(zlib.crc32(blk.tobytes()) ^ base)
        blk[p] = 0
    basis, kernel = {}, []                                    # leading bit -> (vector, unknowns that make it)
    for j, v in enumerate(cols):
        tag = 1 << j
        for lead in sorted(basis, reverse=True):
            if v >> lead & 1:
                v ^= basis[lead][0]
                tag ^= basis[lead][1]
        if v:
            basis[v.bit_length() - 1] = (v, tag)
        else:
            kernel.append(tag)
    want, x = target ^ base, 0
    for lead in sorted(basis, reverse=True):
        if want >> lead & 1:
            want ^= basis[lead][0]
            x ^= basis[lead][1]
    assert want == 0, "the free bytes cannot reach the target"
    if x == 0 and not blk.any():
        x = kernel[0]
    blk[free] = np.frombuffer(x.to_bytes(len(free), "little"), dtype=np.uint8)
    assert zlib.crc32(blk.tobytes()) == target and blk.any()
    return blk


FORGED64 = forge(np.random.default_rng(64).integers(1, 256, BLOCK, dtype=np.uint8), [BLOCK - 4 + i for i in range(4)], ZERO64)


# ---- contexts --------------------------------------------------------------------------------------------------------------------
def _engine(**env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        return L.Engine(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def engines():
    """the default context (fused CRC route for dense 64 KiB blocks) and one that always takes the generic route"""
    es = {"fused": _engine(), "generic": _engine(LZGPU_DISABLE_FUSED=1)}
    yield es
    for e in es.values():
        e.close()


@pytest.fixture(scope="module")
def pools():
    """pools of two and three slots: devices 0 and 1 where there are two, else device 0 several times"""
    two = torch.cuda.device_count() >= 2
    ps = {n: L.Pool(([0, 1, 0] if two else [0, 0, 0])[:n]) for n in (1, 2, 3)}
    yield ps
    for p in ps.values():
        p.close()


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def addr(a):
    return a.ctypes.data


# ---- block writes ----------------------------------------------------------------------------------------------------------------
def req(block, offset, data, exists=1, crc=None):
    data = np.asarray(data, dtype=np.uint8)
    return dict(block=int(block), offset=int(offset), size=int(data.size), data=data, exists=int(exists),
                crc=zlib.crc32(data.tobytes()) if crc is None else int(crc))


def pack(reqs):
    """lzgpu_block_write records (status preset to a value no request can return) and the payload they point into"""
    arr = (_lib.LzBlockWrite * len(reqs))()
    payload = np.concatenate([r["data"] for r in reqs] + [np.zeros(16, dtype=np.uint8)])
    pos = 0
    for i, r in enumerate(reqs):
        a = arr[i]
        a.block, a.offset, a.size, a.crc = r["block"], r["offset"], r["size"], r["crc"]
        a.payload_off, a.exists, a.status = pos, r["exists"], 12345
        pos += r["data"].size
    return arr, payload


def expected(blocks, stored, reqs, sparse_rule):
    status, eb, es = [], blocks.copy(), stored.copy()
    for r in reqs:
        b = r["block"]
        s, blk, crc = hdd_write(blocks[b], int(stored[b]), r["offset"], r["size"], r["crc"], r["data"], r["exists"], sparse_rule)
        status.append(s)
        if s == OK:
            eb[b], es[b] = blk, crc
    return status, eb, es


def write_host(lib, eng, blocks, stored, reqs, sparse_rule):
    """lzgpu_write_blocks on blocks / stored in place: (return code, per-request status)"""
    arr, payload = pack(reqs)
    rc = lib.lzgpu_write_blocks(eng.h, addr(blocks), addr(stored), blocks.shape[0], addr(payload), payload.size, arr, len(reqs), sparse_rule)
    return rc, [arr[i].status for i in range(len(reqs))]


def write_dev(lib, eng, blocks, stored, reqs, sparse_rule):
    """lzgpu_write_blocks_dev with blocks, CRCs, payload and records resident: (per-request status, blocks after, CRCs after)"""
    arr, payload = pack(reqs)
    d_blk = torch.from_numpy(blocks).cuda()
    d_crc = torch.from_numpy(stored.view(np.int32)).cuda()
    d_pay = torch.from_numpy(payload).cuda()
    d_wr = torch.from_numpy(np.frombuffer(bytes(arr), dtype=np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    rc = lib.lzgpu_write_blocks_dev(eng.h, d_blk.data_ptr(), d_crc.data_ptr(), d_pay.data_ptr(), d_wr.data_ptr(), len(reqs), sparse_rule, None)
    assert rc == OK, rc
    eng.sync()
    done = (_lib.LzBlockWrite * len(reqs)).from_buffer_copy(d_wr.cpu().numpy().tobytes())
    return [done[i].status for i in range(len(reqs))], d_blk.cpu().numpy(), d_crc.cpu().numpy().view(np.uint32)


def describe(r):
    return {k: v for k, v in r.items() if k != "data"}


def assert_outcome(name, reqs, status, want_status, blocks, want_blocks, stored, want_stored):
    wrong = [i for i in range(len(reqs)) if status[i] != want_status[i]]
    assert not wrong, (name, len(wrong), describe(reqs[wrong[0]]), status[wrong[0]], want_status[wrong[0]])
    diff = np.nonzero((blocks != want_blocks).any(axis=1) | (stored != want_stored))[0]
    by_block = {r["block"]: r for r in reqs}
    assert diff.size == 0, (name, diff.size, int(diff[0]), describe(by_block.get(int(diff[0]), {"block": int(diff[0]), "no request": 1})))


OFFSETS = [0, 1, 3, 4, 15, 16, 255, 256, 257, 4095, 4096, 32767, 65535]
SIZES = [0, 1, 3, 4, 255, 256, 257, 511, 512, 513, 4096]
BAD_RANGES = [(BLOCK, 0), (BLOCK, 1), (1, BLOCK), (BLOCK - 4, 5), (0, BLOCK + 1)]   # offset = 65536, offset + size = 65537, size = 65537
STATES = ["valid", "damaged", "hole", "nonzero0", "forged0"]


def byte_ranges():
    out = []
    for off in OFFSETS:
        for s in SIZES + [BLOCK - off]:
            r = (off, min(s, BLOCK - off))
            if r not in out:
                out.append(r)
    return out + BAD_RANGES


def set_state(blocks, stored, b, state, bit):
    if state == "damaged":
        stored[b] ^= 1 << bit
    elif state == "hole":
        blocks[b], stored[b] = 0, 0
    elif state == "nonzero0":
        stored[b] = 0
    elif state == "forged0":
        blocks[b], stored[b] = FORGED64, 0


@functools.lru_cache(maxsize=None)
def range_matrix():
    """every byte range x exists x stored state x packet, one request per block in a shuffled block order, and idle blocks"""
    rng = np.random.default_rng(1035)
    combos = [(1, s) for s in STATES] + [(0, "valid"), (0, "nonzero0"), (0, "hole")]
    cases = [(r, e, s, bad) for r in byte_ranges() for e, s in combos for bad in (False, True)]
    n = len(cases) + 24
    blocks = rng.integers(0, 256, (n, BLOCK), dtype=np.uint8)
    stored = crcs_of(blocks)
    where = rng.permutation(n)
    reqs = []
    for i, ((off, size), exists, state, bad_packet) in enumerate(cases):
        b = int(where[i])
        set_state(blocks, stored, b, state, i % 32)
        data = rng.integers(0, 256, size, dtype=np.uint8)
        crc = zlib.crc32(data.tobytes()) ^ ((1 << (7 * i % 32)) if bad_packet else 0)
        reqs.append(dict(req(b, off, data, exists, crc), state=state))
    blocks.flags.writeable = False
    stored.flags.writeable = False
    return blocks, stored, reqs


@pytest.mark.parametrize("sparse_rule", [0, 1])
def test_write_every_byte_range_class(engines, lib, oracle, ref, sparse_rule):
    blocks, stored, reqs = range_matrix()
    want, eb, es = expected(blocks, stored, reqs, sparse_rule)
    assert set(want) == {OK, ARG, CRC, DAMAGED}
    for r, s in zip(reqs, want):
        partial = not (r["offset"] == 0 and r["size"] == BLOCK)
        right = r["crc"] == zlib.crc32(r["data"].tobytes())
        if r["exists"] and right and r["offset"] + r["size"] <= BLOCK and r["offset"] < BLOCK:
            if not partial:
                assert s == OK                                          # over any stored state, no read-modify-write
            elif r["state"] in ("damaged", "nonzero0", "forged0") or (r["state"] == "hole" and not sparse_rule):
                assert s == DAMAGED, describe(r)
            else:
                assert s == OK, describe(r)
    if sparse_rule:
        # the restatement against the oracle's transcription of hdd_write (which always applies the sparse rule)
        checker = ref if ref is not None else oracle
        for r, s in zip(reqs, want):
            b = r["block"]
            rc, blk, crc = O.hdd_write_block(checker, blocks[b] if r["exists"] else None, int(stored[b]), r["offset"], r["size"], r["crc"],
                                             r["data"] if r["size"] else np.zeros(1, np.uint8))
            assert ORACLE_CODE[rc] == s, (describe(r), rc, s)
            if s == OK:
                assert (blk == eb[b]).all() and crc == es[b] == zlib.crc32(eb[b].tobytes()), describe(r)
    eng = engines["fused"]
    hb, hs = blocks.copy(), stored.copy()
    rc, status = write_host(lib, eng, hb, hs, reqs, sparse_rule)
    assert rc == next(s for s in want if s != OK)
    assert_outcome("host", reqs, status, want, hb, eb, hs, es)
    status, db, ds = write_dev(lib, eng, blocks.copy(), stored.copy(), reqs, sparse_rule)
    assert_outcome("dev", reqs, status, want, db, eb, ds, es)


KINDS = ["ok", "range", "packet", "damaged", "created"]


def test_write_several_requests_per_cta(engines, lib):
    """5 x 8 x SMs requests: CTA c takes requests c, c + grid, ... and meets the five outcomes one after another, each CTA in its
    own order; the host form (which stages a whole-block write with exists = 0) and the _dev form must agree with the restatement"""
    grid = 8 * sm_count()
    n = 5 * grid
    assert n >= 3 * grid
    rng = np.random.default_rng(2820)
    blocks = rng.integers(0, 256, (n + 16, BLOCK), dtype=np.uint8)
    stored = crcs_of(blocks)
    where = rng.permutation(n + 16)[:n]
    reqs, whole_over_damaged = [], []
    for i in range(n):
        cta, turn = i % grid, i // grid
        kind, variant = KINDS[(cta + turn) % 5], (cta // 5 + turn) % 3
        b = int(where[i])
        off = int(rng.integers(0, BLOCK))
        data = rng.integers(0, 256, int(rng.integers(0, min(BLOCK - off, 1500) + 1)), dtype=np.uint8)
        if kind == "ok":
            if variant == 1:
                set_state(blocks, stored, b, "hole", 0)
            elif variant == 2:
                set_state(blocks, stored, b, "damaged", i % 32)
                off, data = 0, rng.integers(0, 256, BLOCK, dtype=np.uint8)
                whole_over_damaged.append(i)
            reqs.append(req(b, off, data))
        elif kind == "range":
            size = max(data.size, 1)
            reqs.append(req(b, BLOCK if variant else BLOCK + 1 - size, rng.integers(0, 256, size, dtype=np.uint8)))
        elif kind == "packet":
            reqs.append(req(b, off, data, crc=zlib.crc32(data.tobytes()) ^ (1 << (i % 32))))
        elif kind == "damaged":
            set_state(blocks, stored, b, "forged0" if variant == 1 else "damaged", i % 32)
            reqs.append(req(b, off, data))
        else:
            reqs.append(req(b, off, data, exists=0))
    want, eb, es = expected(blocks, stored, reqs, 1)
    for c in range(0, grid, 97):
        assert {want[i] for i in range(c, n, grid)} == {OK, ARG, CRC, DAMAGED}
    assert whole_over_damaged and all(want[i] == OK for i in whole_over_damaged)
    eng = engines["fused"]
    hb, hs = blocks.copy(), stored.copy()
    rc, host_status = write_host(lib, eng, hb, hs, reqs, 1)
    assert rc == next(s for s in want if s != OK)
    dev_status, db, ds = write_dev(lib, eng, blocks.copy(), stored.copy(), reqs, 1)
    assert host_status == dev_status
    assert (hb == db).all() and (hs == ds).all()
    assert_outcome("host", reqs, host_status, want, hb, eb, hs, es)
    for i in whole_over_damaged:
        assert ds[reqs[i]["block"]] == reqs[i]["crc"]


def test_write_host_tiles_report_the_first_failure_in_request_order(engines, lib):
    """8192 + 300 requests: two host tiles.  The first failure in request order lies in the second tile, on the highest block; a
    later failure in that tile lies on block 3.  The call returns the first one's status."""
    n = 8192 + 300
    first, later = 8192 + 20, 8192 + 250
    rng = np.random.default_rng(2847)
    blocks = rng.integers(0, 256, (n, BLOCK), dtype=np.uint8)
    stored = crcs_of(blocks)
    where = list(rng.permutation(n))
    for i, b in ((first, n - 1), (later, 3)):
        j = where.index(b)
        where[i], where[j] = where[j], where[i]
    reqs = []
    for i in range(n):
        off = int(rng.integers(0, BLOCK - 64))
        data = rng.integers(0, 256, int(rng.integers(1, 65)), dtype=np.uint8)
        reqs.append(req(where[i], off, data, exists=int(i % 11 != 5), crc=zlib.crc32(data.tobytes()) ^ (8 if i == later else 0)))
    stored[n - 1] ^= 4                                                     # request `first` finds its stored block damaged
    want, eb, es = expected(blocks, stored, reqs, 1)
    assert [i for i, s in enumerate(want) if s != OK] == [first, later] and want[first] == DAMAGED and want[later] == CRC
    rc, status = write_host(lib, engines["fused"], blocks, stored, reqs, 1)
    assert rc == DAMAGED
    assert_outcome("host tiles", reqs, status, want, blocks, eb, stored, es)


# ---- block CRCs ------------------------------------------------------------------------------------------------------------------
def crc_host(lib, h, data, n, length, stride, fn="lzgpu_crc_blocks"):
    out = np.full(max(n, 1), 0x5A5A5A5A, dtype=np.uint32)
    rc = getattr(lib, fn)(h, addr(data), n, length, stride, addr(out))
    return rc, out[:n]


def strided(rng, n, length, stride, fill=0xA5):
    """n blocks of `length` random bytes every `stride` bytes, the gaps filled with `fill`; and the blocks themselves"""
    buf = np.full(max((n - 1) * stride + length, 1), fill, dtype=np.uint8)
    rows = rng.integers(0, 256, (n, length), dtype=np.uint8)
    for i in range(n):
        buf[i * stride: i * stride + length] = rows[i]
    return buf, rows


def route_engines(length):
    return ("fused", "generic") if length == BLOCK else ("fused",)


@pytest.mark.parametrize("length", LENGTHS)
def test_crc_blocks_every_length_and_host_stride(engines, lib, length):
    rng = np.random.default_rng(length)
    for extra in (0, 1, 3, 16):
        buf, rows = strided(rng, 37, length, length + extra)
        for name in route_engines(length):
            rc, out = crc_host(lib, engines[name].h, buf, 37, length, length + extra)
            assert rc == OK and (out == crcs_of(rows)).all(), (name, extra)


@pytest.mark.parametrize("length", LENGTHS)
def test_crc_blocks_dev_strides(engines, lib, length):
    """the _dev form at 4-byte-multiple strides; other strides are refused with LZGPU_ERR_ARG on the host before any launch"""
    rng = np.random.default_rng(length + 1)
    s4 = (length + 3) // 4 * 4
    n = 37
    for stride in (s4, s4 + 4, s4 + 16):
        buf, rows = strided(rng, n, length, stride)
        d = torch.from_numpy(buf).cuda()
        d_out = torch.zeros(n, dtype=torch.int32, device="cuda")
        for name in route_engines(length):
            d_out.zero_()
            assert lib.lzgpu_crc_blocks_dev(engines[name].h, d.data_ptr(), n, length, stride, d_out.data_ptr(), None) == OK
            engines[name].sync()
            assert (d_out.cpu().numpy().view(np.uint32) == crcs_of(rows)).all(), (name, stride)
    d = torch.zeros((n + 1) * (length + 16), dtype=torch.uint8, device="cuda")
    d_out = torch.zeros(n, dtype=torch.int32, device="cuda")
    for stride in sorted({length, length + 1, length + 3} - {s4, s4 + 4}):
        assert stride % 4
        for name in route_engines(length):
            assert lib.lzgpu_crc_blocks_dev(engines[name].h, d.data_ptr(), n, length, stride, d_out.data_ptr(), None) == ARG, stride


def test_crc_route_of_64k_blocks(engines):
    """the fused context CRCs dense 64 KiB blocks on the fused route (a persistent launch); the generic one never launches it"""
    rows = np.random.default_rng(9).integers(0, 256, (130, BLOCK), dtype=np.uint8)
    e = _engine()
    try:
        assert e.last_launch() == (0, 0)
        assert (e.crc_blocks(rows) == crcs_of(rows)).all()
        assert e.last_launch()[1] > 0
    finally:
        e.close()
    assert (engines["generic"].crc_blocks(rows) == crcs_of(rows)).all()
    assert engines["generic"].last_launch() == (0, 0)


@pytest.mark.parametrize("length", [4, 5, 131, 1000])
def test_crc_blocks_more_blocks_than_warps(engines, lib, length):
    """at least three times the grid's 8 x SMs x 8 warps: every warp walks several blocks"""
    n = 3 * 8 * sm_count() * 8 + 13
    rng = np.random.default_rng(n + length)
    rows = rng.integers(0, 256, (n, length), dtype=np.uint8)
    want = crcs_of(rows)
    rc, out = crc_host(lib, engines["fused"].h, rows, n, length, length)
    assert rc == OK and (out == want).all()
    stride = (length + 3) // 4 * 4
    buf = np.zeros((n, stride), dtype=np.uint8)
    buf[:, :length] = rows
    d, d_out = torch.from_numpy(buf).cuda(), torch.zeros(n, dtype=torch.int32, device="cuda")
    assert lib.lzgpu_crc_blocks_dev(engines["fused"].h, d.data_ptr(), n, length, stride, d_out.data_ptr(), None) == OK
    engines["fused"].sync()
    assert (d_out.cpu().numpy().view(np.uint32) == want).all()


def stamped(rng, n, length, distinct=5):
    """n blocks of `length` bytes built from a few random blocks, each stamped with its own index (so that every block differs)"""
    base = rng.integers(0, 256, (distinct, length), dtype=np.uint8)
    rows = base[np.arange(n) % distinct]
    rows[:, 8:16] = np.arange(n, dtype=np.uint64)[:, None].view(np.uint8)
    return rows


@pytest.mark.parametrize("length", [BLOCK, BLOCK - 1])
def test_crc_blocks_over_three_host_tiles(engines, lib, length):
    """2 x 2048 + 7 blocks: both staging slots of the 128 MiB tiles are used, the third tile is partial (a 65535-byte block is
    staged at a 65536-byte stride too)"""
    n = 2 * 2048 + 7
    rows = stamped(np.random.default_rng(length), n, length)
    want = crcs_of(rows)
    for name in ("fused", "generic"):
        rc, out = crc_host(lib, engines[name].h, rows, n, length, length)
        assert rc == OK
        wrong = np.nonzero(out != want)[0]
        assert wrong.size == 0, (name, wrong[:8])


@pytest.mark.parametrize("slots", [2, 3])
@pytest.mark.parametrize("length,stride", [(5, 7), (4097, 4099), (65535, 65537), (BLOCK, BLOCK + 3)])
def test_pool_crc_blocks_at_odd_strides(engines, pools, lib, slots, length, stride):
    rng = np.random.default_rng(length + slots)
    for n in (0, 1, 2, 7, 8):
        buf, rows = strided(rng, max(n, 1), length, stride)
        rc, out = crc_host(lib, pools[slots].h, buf, n, length, stride, "lzgpu_pool_crc_blocks")
        assert rc == OK and (out == crcs_of(rows[:n])).all(), n
        rc, one = crc_host(lib, engines["fused"].h, buf, n, length, stride)
        assert rc == OK and (one == out).all(), n
    empty = np.full(1, 0x5A5A5A5A, dtype=np.uint32)
    assert lib.lzgpu_pool_crc_blocks(pools[slots].h, addr(buf), 0, length, stride, addr(empty)) == OK and empty[0] == 0x5A5A5A5A


def test_crc_blocks_with_crcs_disabled(engines, pools, lib):
    rng = np.random.default_rng(41)
    lib.lzgpu_set_crc_enabled(0)
    try:
        for length in LENGTHS:
            n = 9
            buf, _ = strided(rng, n, length, length + 3)
            for name in route_engines(length):
                rc, out = crc_host(lib, engines[name].h, buf, n, length, length + 3)
                assert rc == OK and (out == FAKE).all(), (name, length)
            rc, out = crc_host(lib, pools[2].h, buf, n, length, length + 3, "lzgpu_pool_crc_blocks")
            assert rc == OK and (out == FAKE).all(), length
            s4 = (length + 3) // 4 * 4
            buf4, _ = strided(rng, n, length, s4)
            d, d_out = torch.from_numpy(buf4).cuda(), torch.zeros(n, dtype=torch.int32, device="cuda")
            for name in route_engines(length):
                assert lib.lzgpu_crc_blocks_dev(engines[name].h, d.data_ptr(), n, length, s4, d_out.data_ptr(), None) == OK
                engines[name].sync()
                assert (d_out.cpu().numpy().view(np.uint32) == FAKE).all(), (name, length)
    finally:
        lib.lzgpu_set_crc_enabled(1)
    assert lib.lzgpu_crc_enabled() == 1


# ---- scrubs ----------------------------------------------------------------------------------------------------------------------
def verify(lib, h, data, n, length, stride, stored, sparse_rule, fn="lzgpu_verify_blocks"):
    bad = C.c_int64(-2)
    rc = getattr(lib, fn)(h, addr(data), n, length, stride, addr(stored), sparse_rule, C.byref(bad))
    return rc, bad.value


def layout(rows, stride, fill=0xA5):
    n, length = rows.shape
    buf = np.full((n - 1) * stride + length, fill, dtype=np.uint8)
    for i in range(n):
        buf[i * stride: i * stride + length] = rows[i]
    return buf


def forged_body(length, seed):
    """a non-zero block with the CRC of `length` zero bytes whose non-zero bytes all lie in its 16-byte words"""
    body = length // 16 * 16
    blk = np.zeros(length, dtype=np.uint8)
    blk[:body] = np.random.default_rng(seed).integers(1, 256, body, dtype=np.uint8)
    return forge(blk, [body - 8, body - 7, body - 6, body - 5], crc_of_zeros(length))


def forged_tail(length):
    """a non-zero block with the CRC of `length` zero bytes whose non-zero bytes all lie in its last length % 16 bytes"""
    body = length // 16 * 16
    assert length - body >= 5
    return forge(np.zeros(length, dtype=np.uint8), list(range(body, length)), crc_of_zeros(length))


@pytest.mark.parametrize("length", [5, 17, 21, 4101, 65535])
def test_sparse_rule_at_short_lengths(engines, lib, length):
    rng = np.random.default_rng(length + 7)
    stride = length + 3
    n, holes = 11, [1, 4, 6]
    rows = rng.integers(0, 256, (n, length), dtype=np.uint8)
    rows[holes] = 0
    stored = crcs_of(rows)
    stored[holes] = 0
    forged = {}
    if length >= 16:
        forged["body"] = forged_body(length, length)
        assert not forged["body"][length // 16 * 16:].any()
    if length % 16 >= 5:
        forged["tail"] = forged_tail(length)
        assert not forged["tail"][: length // 16 * 16].any()
    assert forged
    for name in ("fused", "generic"):
        h = engines[name].h
        buf = layout(rows, stride)
        assert verify(lib, h, buf, n, length, stride, stored, 1) == (OK, -1), name        # holes stored with 0 are accepted
        s0 = stored.copy()
        for hole in holes:                                                                # ... and rejected without the rule
            assert verify(lib, h, buf, n, length, stride, s0, 0) == (CRC, hole), (name, hole)
            s0[hole] = crc_of_zeros(length)
        assert verify(lib, h, buf, n, length, stride, s0, 0) == (OK, -1), name
        for where, blk in forged.items():
            r = rows.copy()
            r[8] = blk
            s = stored.copy()
            s[8] = 0
            assert verify(lib, h, layout(r, stride), n, length, stride, s, 1) == (CRC, 8), (name, where)
            s[8] = crc_of_zeros(length)                                                   # its true CRC: fine either way
            assert verify(lib, h, layout(r, stride), n, length, stride, s, 1) == (OK, -1), (name, where)


@pytest.mark.parametrize("route", ["fused", "generic"])
def test_sparse_rule_with_more_holes_than_ctas(engines, lib, route):
    """3 x 8 x SMs + 40 candidate holes in one tile; the only non-zero one (the zero block's CRC, stored with 0) near the end"""
    n = 3 * 8 * sm_count() + 40
    rows = np.zeros((n, BLOCK), dtype=np.uint8)
    rows[:2] = np.random.default_rng(3).integers(0, 256, (2, BLOCK), dtype=np.uint8)
    stored = np.zeros(n, dtype=np.uint32)
    stored[:2] = crcs_of(rows[:2])
    h = engines[route].h
    assert verify(lib, h, rows, n, BLOCK, BLOCK, stored, 1) == (OK, -1)
    rows[n - 3] = FORGED64
    assert verify(lib, h, rows, n, BLOCK, BLOCK, stored, 1) == (CRC, n - 3)


@pytest.mark.parametrize("length", [BLOCK, 4101])
def test_smallest_failing_index_wins(engines, lib, length):
    """crc_compare_kernel and sparse_confirm_kernel lower the same word: a failing hole before a CRC mismatch is reported, and
    the other way round"""
    n = 64
    rng = np.random.default_rng(length + 11)
    forged = FORGED64 if length == BLOCK else forged_tail(length)
    for hole_at, mismatch_at in ((10, 40), (40, 10), (0, 63), (63, 0)):
        rows = rng.integers(0, 256, (n, length), dtype=np.uint8)
        rows[hole_at] = forged
        stored = crcs_of(rows)
        stored[hole_at] = 0
        stored[mismatch_at] ^= 0x100
        for name in ("fused", "generic"):
            assert verify(lib, engines[name].h, rows, n, length, length, stored, 1) == (CRC, min(hole_at, mismatch_at)), (name, hole_at)


def test_verify_across_the_1gib_tile(engines, pools, lib):
    """16384 + 3 blocks of 64 KiB: two 1 GiB staging tiles.  A bad block is reported at its index in the whole batch, and the
    first tile's bad block before the second's, by the host form on both routes and by pools of one and two slots"""
    n = 16384 + 3
    rows = stamped(np.random.default_rng(2718), n, BLOCK, distinct=3)
    stored = crcs_of(rows)
    calls = [(name, engines[name].h, "lzgpu_verify_blocks") for name in ("fused", "generic")]
    calls += [(f"pool{s}", pools[s].h, "lzgpu_pool_verify_blocks") for s in (1, 2)]
    for name, h, fn in calls:
        assert verify(lib, h, rows, n, BLOCK, BLOCK, stored, 0, fn) == (OK, -1), name
    late, early = 16384 + 1, 100
    rows[late, 333] ^= 0x20
    for name, h, fn in calls:
        assert verify(lib, h, rows, n, BLOCK, BLOCK, stored, 0, fn) == (CRC, late), name
    rows[early, 65535] ^= 1
    for name, h, fn in calls:
        assert verify(lib, h, rows, n, BLOCK, BLOCK, stored, 1, fn) == (CRC, early), name


def test_moosefs_at_the_block_limit_of_every_data_parts(engines, lib, oracle):
    rng = np.random.default_rng(1746)
    base = rng.integers(0, 256, (3, BLOCK), dtype=np.uint8)
    base_crc = crcs_of(base)
    for dp in range(1, 33):
        header = lib.lzgpu_moosefs_header_size(dp)
        assert header == O.moosefs_header_size(oracle, dp), dp
        n = -(-1024 // dp)
        img = np.zeros(header + (n + 1) * BLOCK, dtype=np.uint8)
        img[header:] = base[np.arange(n + 1) % 3].reshape(-1)
        img[1024: 1024 + 4 * n] = base_crc[np.arange(n) % 3].astype(">u4").view(np.uint8)
        for name in ("fused", "generic"):
            bad = C.c_int64(-2)
            assert lib.lzgpu_verify_moosefs(engines[name].h, dp, addr(img), n, C.byref(bad)) == OK, (name, dp)
            assert lib.lzgpu_verify_moosefs(engines[name].h, dp, addr(img), n + 1, C.byref(bad)) == ARG, (name, dp)
        img[header + (n - 1) * BLOCK + 4321] ^= 0x80
        assert O.scrub_moosefs(oracle, img, dp, n) == (-3, n - 1)
        for name in ("fused", "generic"):
            bad = C.c_int64(-2)
            assert lib.lzgpu_verify_moosefs(engines[name].h, dp, addr(img), n, C.byref(bad)) == CRC and bad.value == n - 1, (name, dp)


def interleaved(rows, stored):
    rec = np.zeros((rows.shape[0], 4 + BLOCK), dtype=np.uint8)
    rec[:, 4:] = rows
    rec[:, :4] = stored.astype(">u4").view(np.uint8).reshape(-1, 4)
    return rec


def test_scrubs_with_crcs_disabled(engines, lib):
    """stored 0xFEDCBA98 passes and the real CRC fails; with the sparse rule a hole stored with 0 still passes and a non-zero block
    stored with 0 still fails, also one with the zero block's CRC"""
    rng = np.random.default_rng(30)
    n = 12
    lib.lzgpu_set_crc_enabled(0)
    try:
        for length in (BLOCK, 4101):
            rows = rng.integers(0, 256, (n, length), dtype=np.uint8)
            rows[3] = 0
            forged = FORGED64 if length == BLOCK else forged_tail(length)
            for name in ("fused", "generic"):
                h = engines[name].h
                stored = np.full(n, FAKE, dtype=np.uint32)
                for sparse in (0, 1):
                    assert verify(lib, h, rows, n, length, length, stored, sparse) == (OK, -1), (name, length)
                s = stored.copy()
                s[7] = zlib.crc32(rows[7].tobytes())
                for sparse in (0, 1):
                    assert verify(lib, h, rows, n, length, length, s, sparse) == (CRC, 7), (name, length)
                s = stored.copy()
                s[3] = 0
                assert verify(lib, h, rows, n, length, length, s, 1) == (OK, -1), (name, length)
                assert verify(lib, h, rows, n, length, length, s, 0) == (CRC, 3), (name, length)
                for blk in (rows[5].copy(), forged):
                    r = rows.copy()
                    r[5] = blk
                    s5 = s.copy()
                    s5[5] = 0
                    assert verify(lib, h, r, n, length, length, s5, 1) == (CRC, 5), (name, length)
                if length == BLOCK:
                    for blk, crc5, want in ((rows[5], FAKE, (OK, -1)), (rows[5], 0, (CRC, 5)), (forged, 0, (CRC, 5)),
                                            (rows[5], zlib.crc32(rows[5].tobytes()), (CRC, 5))):
                        r = rows.copy()
                        r[5] = blk
                        s5 = s.copy()
                        s5[5] = crc5
                        rec, bad = interleaved(r, s5), C.c_int64(-2)
                        rc = lib.lzgpu_verify_interleaved(h, addr(rec), n, C.byref(bad))
                        assert (rc, bad.value) == want, (name, crc5)
    finally:
        lib.lzgpu_set_crc_enabled(1)
    assert lib.lzgpu_crc_enabled() == 1
