"""lzgpu_pool_check_stripes ... lzgpu_pool_verify_interleaved: the chunkserver's stripe consistency job and block scrub over every
device of a pool must return, for any input, exactly what the per-context call returns on one context for the whole batch.

Every case runs the same call on one Engine and on a pool, each on its own copy of the inputs, twice: through the C ABI with every
output buffer and `bad` filled with a sentinel first (return code, every result byte, bad / first_bad and every byte of the parts after
the call must be equal), and through the Python methods (result, exception type, status and .where equal).  A pool lists device 0
two or three times (one context and one pipeline each), or devices 0 and 1 when the box has two GPUs.  Batch sizes 0, 1 and 2 leave
slots idle, 7 and 8 cut the batch unevenly and evenly."""
import ctypes as C
import threading
import zlib

import numpy as np
import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200.engine import _p, _ptr_array

BLOCK = 65536
SIZES = (0, 1, 2, 7, 8)
gpu = pytest.mark.gpu

# call: (entry dtype, one entry per stripe (else per chunk), takes bad)
CALLS = {
    "check_stripes": (L.Engine.VERDICT_DTYPE, False, True),
    "check_stripe_map": (L.Engine.STRIPE_STATE_DTYPE, True, True),
    "correct_stripes": (L.Engine.STRIPE_FIX_DTYPE, True, True),
    "check_stripe_map_degraded": (L.Engine.STRIPE_STATE_DTYPE, True, True),
    "correct_stripes_degraded": (L.Engine.STRIPE_FIX_DTYPE, True, True),
    "repair_stripes": (L.Engine.STRIPE_REPAIR_DTYPE, True, False),
    "decode_stripes": (L.Engine.STRIPE_DECODE_DTYPE, True, False),
}
# (call, goal, lost parts): the check on xor3, ec(8,2), ec(8,4); the degraded map and correction on ec(8,3) with data part 2 lost;
# the repair on ec(8,2); the decode on ec(8,4) and ec(10,8) (a Cauchy generator: the generic route)
CASES = [(c, g, ()) for c in ("check_stripes", "check_stripe_map", "correct_stripes") for g in ("xor3", "ec(8,2)", "ec(8,4)")] + \
        [(c, "ec(8,3)", (2,)) for c in ("check_stripe_map_degraded", "correct_stripes_degraded")] + \
        [("repair_stripes", "ec(8,2)", ()), ("decode_stripes", "ec(8,4)", ()), ("decode_stripes", "ec(10,8)", ())]


def test_every_pool_call_refuses_a_null_pool():
    lib = _lib.load()
    g = L.SliceType("ec(8,2)")
    for call, (_, _, with_bad) in CALLS.items():
        args = [None, C.byref(g.c), 1, 16, None, 0, None, None] + ([None] if with_bad else [])
        assert getattr(lib, "lzgpu_pool_" + call)(*args) == _lib.ERR_ARG, call
    assert lib.lzgpu_pool_verify_blocks(None, None, 1, BLOCK, BLOCK, None, 0, None) == _lib.ERR_ARG
    assert lib.lzgpu_pool_verify_interleaved(None, None, 1, None) == _lib.ERR_ARG


@pytest.fixture(scope="module")
def eng():
    e = L.Engine(0)
    yield e
    e.close()


def _devices(n):
    import torch
    return [0, 1] if n == 2 and torch.cuda.device_count() >= 2 else [0] * n


@pytest.fixture(scope="module")
def pools():
    ps = {n: L.Pool(_devices(n)) for n in (2, 3)}
    yield ps
    for p in ps.values():
        p.close()


class Batch:
    """n chunks of nb blocks: every part [n, pb * 64 KiB] (short data parts zero-padded) and its stored CRCs [n, pb]"""

    def __init__(self, eng, text, n, nb, seed):
        self.goal = L.SliceType(text)
        self.k, self.m, self.n, self.nb = self.goal.k, self.goal.m, n, nb
        self.pb = -(-nb // self.k)
        data = np.random.default_rng(seed).integers(0, 256, size=(max(n, 1), nb * BLOCK), dtype=np.uint8)
        parity, _ = eng.encode_chunks(self.goal, data)
        parts = eng.split_chunks(self.goal, data, nb) + [np.ascontiguousarray(parity[:, r]) for r in range(self.m)]
        self.parts = [np.ascontiguousarray(p[:n]) for p in parts]
        self.crc = [np.ascontiguousarray(eng.crc_blocks(p).reshape(-1, self.pb)[:n]) for p in parts]

    def block(self, part, c, s):
        return self.parts[part][c, s * BLOCK:(s + 1) * BLOCK]

    def stale(self, part, c, s):
        """wrong bytes and a matching stored CRC: only the code sees it"""
        self.block(part, c, s)[100:104] ^= np.array([1, 22, 3, 44], dtype=np.uint8)
        self.crc[part][c, s] = zlib.crc32(self.block(part, c, s).tobytes())

    def rot(self, part, c, s):
        """wrong bytes under the old stored CRC"""
        self.block(part, c, s)[5000:5002] ^= np.array([7, 9], dtype=np.uint8)


def _raw(fn, name, h, b, given, crcs=True):
    """fn (the C function of call `name`, per context or pool) on copies of the given parts, every output byte and bad[] at a sentinel
    first: (rc, result bytes, bad, parts after)"""
    dtype, per_stripe, with_bad = CALLS[name]
    parts = [b.parts[i].copy() if i in given else None for i in range(b.k + b.m)]
    pc = _ptr_array([b.crc[i].copy() if i in given else None for i in range(b.k + b.m)]) if crcs else None
    shape = (b.n, b.pb) if per_stripe else (b.n,)
    out = np.full(int(np.prod(shape)) * dtype.itemsize, 0xA5, dtype=np.uint8)
    bad = (C.c_int64 * 3)(-7, -7, -7)
    args = [h, C.byref(b.goal.c), b.n, b.nb, _ptr_array(parts), b.pb * BLOCK, pc, _p(out)] + ([bad] if with_bad else [])
    rc = fn(*args)
    return rc, out.tobytes(), list(bad), parts


def _method(obj, name, b, given, crcs=True):
    """the Python method on copies: (status or 0, exception type name, .where, result array or None, parts after)"""
    parts = [b.parts[i].copy() if i in given else None for i in range(b.k + b.m)]
    pc = [b.crc[i].copy() if i in given else None for i in range(b.k + b.m)] if crcs else None
    try:
        out = getattr(obj, name)(b.goal, b.nb, parts, pc)
        return 0, None, None, out, parts
    except L.LzGpuError as e:
        res = next((getattr(e, a) for a in ("verdict", "map", "fix") if hasattr(e, a)), None)
        return e.status, type(e).__name__, getattr(e, "where", None), res, parts


def same(eng, pool, name, b, given=None, crcs=True):
    """the call on the engine and on the pool give the same everything; returns the C call's (rc, bad, parts after)"""
    given = set(range(b.k + b.m)) if given is None else set(given)
    lib = eng.lib
    e = _raw(getattr(lib, "lzgpu_" + name), name, eng.h, b, given, crcs)
    p = _raw(getattr(lib, "lzgpu_pool_" + name), name, pool.h, b, given, crcs)
    assert p[0] == e[0], (name, p[0], e[0], _lib.last_error())
    assert p[1] == e[1], "result entries differ"
    assert p[2] == e[2], ("bad differs", p[2], e[2])
    for i, (x, y) in enumerate(zip(p[3], e[3])):
        assert (x is None and y is None) or (x == y).all(), f"part {i} differs after the call"
    em, pm = _method(eng, name, b, given, crcs), _method(pool, name, b, given, crcs)
    assert pm[:3] == em[:3], (pm[:3], em[:3])
    assert (pm[3] is None) == (em[3] is None) and (em[3] is None or pm[3].tobytes() == em[3].tobytes())
    for x, y in zip(pm[4], em[4]):
        assert (x is None and y is None) or (x == y).all()
    return e[0], e[2], e[3]


@gpu
@pytest.mark.parametrize("fault", ["clean", "stale", "rot"])
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("case", CASES, ids=[f"{c}-{g}" for c, g, _ in CASES])
def test_pool_equals_one_context(eng, pools, case, n, fault):
    """faults in the first and the last share: stale blocks (valid CRCs) or rotten blocks, in a data and a parity part; the decode
    goals get two stale parts in one stripe of the last chunk (inside their radius)"""
    name, text, lost = case
    b = Batch(eng, text, n, 2 * L.SliceType(text).k + 3, seed=len(name) * 100 + n)
    given = [i for i in range(b.k + b.m) if i not in lost]
    if n and fault != "clean":
        hit = b.stale if fault == "stale" else b.rot
        hit(1, 0, 0)
        hit(b.k, n - 1, b.pb - 1)
        if name == "decode_stripes" and fault == "stale":
            hit(4, n - 1, 1)
            hit(b.k + 1, n - 1, 1)
    for pool in pools.values():
        same(eng, pool, name, b, given)


@gpu
@pytest.mark.parametrize("name,text", [("check_stripes", "ec(8,2)"), ("check_stripe_map", "ec(8,2)"), ("correct_stripes", "ec(8,2)"),
                                       ("check_stripe_map_degraded", "ec(8,3)"), ("correct_stripes_degraded", "ec(8,3)"),
                                       ("repair_stripes", "xor3"), ("decode_stripes", "xor3")])
def test_crc_failure_in_a_later_share_wins_over_an_inconsistent_earlier_one(eng, pools, name, text):
    """8 chunks over two slots: chunk 1 (share 0) is inconsistent, chunk 6 (share 1) has a block that fails its stored CRC.  One
    context returns LZGPU_ERR_CRC for the whole batch, so the pool must too.  The repair and the decode run on xor3, where a stale
    block stays UNEXPLAINED, with a wrong stored CRC in chunk 6 (CRC_ONLY)."""
    b = Batch(eng, text, 8, 2 * L.SliceType(text).k + 3, seed=11)
    b.stale(1, 1, 2)
    if name in ("repair_stripes", "decode_stripes"):
        b.crc[2][6, 1] ^= 0x10
    else:
        b.rot(b.k, 6, 1)
    given = [i for i in range(b.k + b.m) if not (b.m == 3 and i == 2)]
    rc, bad, _ = same(eng, pools[2], name, b, given)
    assert rc == _lib.ERR_CRC
    if CALLS[name][2]:
        assert bad[0] == 6


@gpu
@pytest.mark.parametrize("name", ["check_stripes", "check_stripe_map", "correct_stripes"])
def test_crc_failures_in_two_shares_report_the_lower_one(eng, pools, name):
    b = Batch(eng, "ec(8,4)", 8, 19, seed=12)
    b.rot(9, 7, 0)     # share 1 of a two-slot pool, share 2 of a three-slot pool
    b.rot(5, 3, 2)     # share 0 / 1
    b.rot(0, 4, 1)     # share 1 / 1: a lower part in a later chunk
    for pool in pools.values():
        rc, bad, _ = same(eng, pool, name, b)
        assert rc == _lib.ERR_CRC and bad == [3, 5, 2]


@gpu
@pytest.mark.parametrize("n", SIZES)
def test_refusals_write_nothing(eng, pools, n):
    """LZGPU_ERR_TOO_FEW_PARTS (a data part missing for the check, only k parts for the degraded calls), and the repair and the
    decode without stored CRCs: the same code, nothing written into the parts, the results or bad"""
    cases = [("check_stripes", "ec(8,2)", [i for i in range(10) if i != 3], True),
             ("correct_stripes", "ec(8,2)", [i for i in range(10) if i != 0], True),
             ("check_stripe_map_degraded", "ec(8,3)", [i for i in range(11) if i not in (2, 8, 9)], True),
             ("correct_stripes_degraded", "ec(8,3)", [i for i in range(11) if i not in (2, 8, 9)], True),
             ("repair_stripes", "ec(8,2)", list(range(10)), False),
             ("decode_stripes", "ec(8,4)", list(range(12)), False)]
    for name, text, given, crcs in cases:
        b = Batch(eng, text, n, 17, seed=13)
        if n:
            b.rot(1, n - 1, 0)
        dtype, per_stripe, _ = CALLS[name]
        for pool in pools.values():
            rc, bad, after = same(eng, pool, name, b, given, crcs)
            assert rc == (_lib.ERR_ARG if not crcs else _lib.ERR_TOO_FEW_PARTS), (name, rc)
            assert bad == [-7, -7, -7]
            for i in given:
                assert (after[i] == b.parts[i]).all()
            r = _raw(getattr(eng.lib, "lzgpu_pool_" + name), name, pool.h, b, set(given), crcs)
            assert r[1] == bytes([0xA5]) * len(r[1])


def _scrub_blocks(n, seed):
    rng = np.random.default_rng(seed)
    blocks = rng.integers(0, 256, size=(n, BLOCK), dtype=np.uint8)
    crc = np.array([zlib.crc32(x.tobytes()) for x in blocks], dtype=np.uint32)
    for i in range(0, n, 3):               # holes: all-zero blocks stored with CRC 0, which only the sparse rule accepts
        blocks[i] = 0
        crc[i] = 0
    return blocks, crc


def _interleaved(blocks, crc):
    rec = np.zeros((len(blocks), 4 + BLOCK), dtype=np.uint8)
    rec[:, :4] = crc.astype(">u4").view(np.uint8).reshape(-1, 4)
    rec[:, 4:] = blocks
    return rec


def _same_scrub(eng, pool, name, *args):
    """the raw call with first_bad at a sentinel, then the Python method: equal results; returns (rc, first_bad)"""
    out = []
    for fn, h in ((getattr(eng.lib, "lzgpu_" + name), eng.h), (getattr(eng.lib, "lzgpu_pool_" + name), pool.h)):
        bad = C.c_int64(-7)
        out.append((fn(h, *args, C.byref(bad)), bad.value))
    assert out[0] == out[1], out
    return out[0]


@gpu
@pytest.mark.parametrize("n", SIZES)
def test_scrub_with_the_sparse_rule(eng, pools, n):
    blocks, crc = _scrub_blocks(max(n, 1), 14)
    blocks, crc = np.ascontiguousarray(blocks[:n]), np.ascontiguousarray(crc[:n])
    for pool in pools.values():
        for sparse in (1, 0):
            rc, bad = _same_scrub(eng, pool, "verify_blocks", _p(blocks), n, BLOCK, BLOCK, _p(crc), sparse)
            assert rc == (_lib.ERR_CRC if n and not sparse else _lib.OK) and bad == (0 if n and not sparse else -1)
        rec = _interleaved(blocks, crc)
        assert _same_scrub(eng, pool, "verify_interleaved", _p(rec), n) == (_lib.OK, -1)
        if n:
            bad_blocks = blocks.copy()
            bad_blocks[n - 1, 77] ^= 1                 # the last share
            if n > 2:
                bad_blocks[2, 9] ^= 4                  # share 0: reported
            want = 2 if n > 2 else n - 1
            rc, bad = _same_scrub(eng, pool, "verify_blocks", _p(bad_blocks), n, BLOCK, BLOCK, _p(crc), 1)
            assert (rc, bad) == (_lib.ERR_CRC, want)
            rec = _interleaved(bad_blocks, crc)
            assert _same_scrub(eng, pool, "verify_interleaved", _p(rec), n) == (_lib.ERR_CRC, want)
            for obj in (eng, pool):
                with pytest.raises(L.ChunkCrcError) as e:
                    obj.verify_blocks(bad_blocks, crc, sparse_rule=True)
                assert e.value.where == (want,)
                with pytest.raises(L.ChunkCrcError) as e:
                    obj.verify_interleaved(rec)
                assert e.value.where == (want,)
        pool.verify_blocks(blocks, crc, sparse_rule=True)
        pool.verify_interleaved(_interleaved(blocks, crc))


@gpu
def test_scrub_refuses_device_memory(eng, pools):
    import torch
    blocks, crc = _scrub_blocks(4, 15)
    d_blocks = torch.from_numpy(blocks).cuda()
    d_crc = torch.from_numpy(crc.view(np.int32)).cuda()
    d_rec = torch.from_numpy(_interleaved(blocks, crc)).cuda()
    lib = eng.lib
    for pool in pools.values():
        for data, stored in ((d_blocks.data_ptr(), _p(crc)), (_p(blocks), d_crc.data_ptr())):
            bad = C.c_int64(-7)
            assert lib.lzgpu_pool_verify_blocks(pool.h, data, 4, BLOCK, BLOCK, stored, 1, C.byref(bad)) == _lib.ERR_ARG
            assert bad.value == -7 and "device memory" in _lib.last_error()
        bad = C.c_int64(-7)
        assert lib.lzgpu_pool_verify_interleaved(pool.h, d_rec.data_ptr(), 4, C.byref(bad)) == _lib.ERR_ARG and bad.value == -7
        assert lib.lzgpu_pool_verify_interleaved(pool.h, d_rec.data_ptr(), 0, C.byref(bad)) == _lib.ERR_ARG
    torch.cuda.synchronize()


@gpu
def test_two_threads_repair_through_one_pool_at_once(eng, pools):
    """two threads issue pool repairs at the same time, each on its own batch, several times: every result equals the one context's"""
    batches = []
    for t in range(2):
        b = Batch(eng, "ec(8,2)", 7, 19, seed=20 + t)
        for c in range(7):
            b.rot((c + t) % 10, c, c % 3)
        b.stale(4, 5, 1)
        batches.append(b)
    want = [_method(eng, "repair_stripes", b, set(range(10))) for b in batches]
    errors = []

    def worker(t):
        try:
            for _ in range(4):
                for pool in pools.values():
                    got = _method(pool, "repair_stripes", batches[t], set(range(10)))
                    assert got[:3] == want[t][:3] and got[3].tobytes() == want[t][3].tobytes()
                    assert all((x == y).all() for x, y in zip(got[4], want[t][4]))
        except Exception as exc:  # noqa: BLE001
            errors.append((t, repr(exc)))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
