"""lzgpu_pool_recover_slices: the recovery of a multi-slice goal from the parts of all its slices together, over every device of a pool,
must return for any input exactly what lzgpu_recover_slices returns on one context for the whole batch.

Every case runs on one Engine and on a pool, each on its own copy of the inputs, twice: through the C ABI with every output part (at an
out_stride that differs from part_stride), out CRC, image and bad[0..3] at a sentinel first (return code, every byte and bad must be
equal), and through the Python methods (result, exception type and .where equal).  A clean case is also checked against the original
data, lzgpu_encode_slices of it and zlib.crc32.  A pool lists device 0 two or three times (one context and one pipeline each), or
devices 0 and 1 when the box has two GPUs.  Batch sizes 0, 1 and 2 leave slots idle, 7 and 8 cut the batch unevenly and evenly."""
import ctypes as C
import threading
import zlib

import numpy as np
import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200.engine import _goal_array, _p, _ptr_array
from tests.test_recover_slices_plan import goalset, layout, ref_lost

BLOCK = 65536
SIZES = (0, 1, 2, 7, 8)
SENT, SENT_CRC = 0xA5, 0x5A5A5A5A
gpu = pytest.mark.gpu

# goal set: (slice names, given flags over the flat parts, nb with a tail combined stripe, nb < L)
SETS = {
    # xor2 parts 0, 1 and xor3 parts 0, 2 lost: neither slice has k parts, together they determine every block
    "xor2+xor3": (("xor2", "xor3"), [0, 0, 1, 0, 1, 0, 1], 13, 4),
    # 7 of 11 parts lost (ec(3,2) parts 0-3, ec(4,2) parts 0, 1, 3): only both slices together rebuild the chunk
    "ec(3,2)+ec(4,2)": (("ec(3,2)", "ec(4,2)"), [0, 0, 0, 0, 1, 0, 0, 1, 0, 1, 1], 29, 7),
    # the standard part and xor3 parts 1 and 3 lost, xor2 intact
    "std+xor2+xor3": (("std", "xor2", "xor3"), [0, 1, 1, 1, 1, 0, 1, 0], 13, 5),
    # ec(5,5) takes Cauchy rows (m >= 5): its data parts 1, 3 and parity rows 1, 2 given, xor2 only its parity: rescue only
    "ec(5,5)+xor2": (("ec(5,5)", "xor2"), [0, 1, 0, 1, 0, 0, 1, 1, 0, 0, 0, 0, 1], 23, 7),
}
RESCUE = SETS["ec(3,2)+ec(4,2)"]


def test_a_null_pool_and_null_goals_are_refused():
    lib = _lib.load()
    bad = (C.c_int64 * 4)(-7, -7, -7, -7)
    assert lib.lzgpu_pool_recover_slices(None, None, 2, 1, 16, None, None, None, None, None, None, None, None, 0, bad) == _lib.ERR_ARG
    assert list(bad) == [-7] * 4


def test_the_rescue_sets_are_lost_to_the_per_slice_rule():
    for name in ("xor2+xor3", "ec(3,2)+ec(4,2)", "ec(5,5)+xor2"):
        names, given, _, _ = SETS[name]
        assert ref_lost(goalset(names), given), name


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
    """n chunks of nb blocks of a goal set: the data, every flat part [n, pb_i * 64 KiB] (data parts split from the chunk, short ones
    zero-padded; parity parts from lzgpu_encode_slices) and its block CRCs [n, pb_i].  encode=False: zero parts and CRCs, for requests
    that are refused before anything is read."""

    def __init__(self, eng, names, given, n, nb, seed, encode=True):
        self.goals = goalset(names)
        self.lay, self.n_parts = layout(self.goals)
        self.slice_of = [i for i, (k, m, _, _) in enumerate(self.lay) for _ in range(k + m)]
        self.pbs = [-(-nb // k) for k, _, _, _ in self.lay]
        self.given, self.n, self.nb = list(given), n, nb
        self.parts = [np.zeros((n, self.pbs[self.slice_of[g]] * BLOCK), dtype=np.uint8) for g in range(self.n_parts)]
        self.crcs = [np.zeros((n, self.pbs[self.slice_of[g]]), dtype=np.uint32) for g in range(self.n_parts)]
        self.data = np.zeros((n, nb * BLOCK), dtype=np.uint8)
        if not encode:
            return
        data = np.random.default_rng(seed).integers(0, 256, size=(max(n, 1), nb * BLOCK), dtype=np.uint8)
        self.data = data[:n]
        g = 0
        for goal, (k, m, base, _), (par, crc) in zip(self.goals, self.lay, eng.encode_slices(self.goals, data)):
            if goal.is_std:
                self.parts[g], self.crcs[g] = np.ascontiguousarray(data[:n]), np.ascontiguousarray(crc[:n])
                g += 1
                continue
            pb = -(-nb // k)
            padded = np.zeros((data.shape[0], pb * k * BLOCK), dtype=np.uint8)
            padded[:, :nb * BLOCK] = data
            blocks = padded.reshape(-1, pb, k, BLOCK)
            for j in range(k):
                self.parts[g] = np.ascontiguousarray(blocks[:n, :, j, :]).reshape(n, pb * BLOCK)
                c = np.full((data.shape[0], pb), zlib.crc32(bytes(BLOCK)), dtype=np.uint32)
                idx = np.arange(pb) * k + j
                c[:, idx < nb] = crc[:, idx[idx < nb]]
                self.crcs[g] = np.ascontiguousarray(c[:n])
                g += 1
            for r in range(m):
                self.parts[g] = np.ascontiguousarray(par[:n, r])
                self.crcs[g] = np.ascontiguousarray(crc[:n, nb + r * pb: nb + (r + 1) * pb])
                g += 1

    def lost(self):
        return [0 if x else 1 for x in self.given]

    def where(self, chunk, g, block):
        """bad[0..3] of flat part g's block: (chunk, slice, part in the slice, block)"""
        i = self.slice_of[g]
        return (chunk, i, g - self.lay[i][2], block)


def _raw(fn, h, b, want, image, with_crc, crcs):
    """fn (lzgpu_recover_slices or lzgpu_pool_recover_slices) on copies of the given parts and CRCs, every output at a sentinel first:
    (rc, bad, outputs, output CRCs, image).  out_stride pads every part past part_stride, the image has a sentinel block past nb."""
    ns = len(b.goals)
    parts = [b.parts[g].copy() if b.given[g] else None for g in range(b.n_parts)]
    pc = None if crcs is None else _ptr_array([crcs[g].copy() if b.given[g] else None for g in range(b.n_parts)])
    pstride = (C.c_size_t * ns)(*[pb * BLOCK for pb in b.pbs])
    ostride = (C.c_size_t * ns)(*[pb * BLOCK + 4096 * (i + 1) for i, pb in enumerate(b.pbs)])
    outs = [np.full((b.n, ostride[b.slice_of[g]]), SENT, dtype=np.uint8) if want[g] else None for g in range(b.n_parts)]
    ocrc = [np.full((b.n, b.pbs[b.slice_of[g]]), SENT_CRC, dtype=np.uint32) if want[g] and with_crc else None for g in range(b.n_parts)]
    istride = (b.nb + 1) * BLOCK
    img = np.full((b.n, istride), SENT, dtype=np.uint8) if image else None
    bad = (C.c_int64 * 4)(-7, -7, -7, -7)
    w = np.asarray(want, dtype=np.uint8)
    rc = fn(h, _goal_array(b.goals), ns, b.n, b.nb, _ptr_array(parts), pstride, pc, _p(w), _ptr_array(outs), ostride,
            _ptr_array(ocrc) if with_crc else None, _p(img), istride, bad)
    return rc, list(bad), outs, ocrc, img


def _method(obj, b, want, image, with_crc, crcs):
    """the Python method on copies: (0, out, out_crc, image) or (status, exception type name, .where)"""
    parts = [b.parts[g].copy() if b.given[g] else None for g in range(b.n_parts)]
    pc = None if crcs is None else [crcs[g].copy() if b.given[g] else None for g in range(b.n_parts)]
    try:
        return (0,) + tuple(obj.recover_slices(b.goals, b.nb, parts, pc, want=want, chunk_image=image, with_crc=with_crc))
    except L.LzGpuError as e:
        return e.status, type(e).__name__, getattr(e, "where", None)


def _equal(x, y):
    return (x is None and y is None) or (x is not None and y is not None and np.array_equal(x, y))


def same(eng, pool, b, want=None, image=True, with_crc=True, crcs="stored"):
    """the call on the engine and on the pool give the same everything; returns the pool's raw result (rc, bad, outs, ocrc, img)"""
    want = b.lost() if want is None else want
    crcs = b.crcs if crcs == "stored" else crcs
    lib = eng.lib
    e = _raw(lib.lzgpu_recover_slices, eng.h, b, want, image, with_crc, crcs)
    p = _raw(lib.lzgpu_pool_recover_slices, pool.h, b, want, image, with_crc, crcs)
    assert p[0] == e[0], (p[0], e[0], _lib.last_error())
    assert p[1] == e[1], ("bad differs", p[1], e[1])
    if e[0] != _lib.ERR_CRC:                       # the outputs are undefined after a CRC mismatch
        for x, y in zip(p[2] + p[3] + [p[4]], e[2] + e[3] + [e[4]]):
            assert _equal(x, y), "an output differs"
    em, pm = _method(eng, b, want, image, with_crc, crcs), _method(pool, b, want, image, with_crc, crcs)
    assert pm[0] == em[0], (pm, em)
    if em[0] == 0:
        for xs, ys in zip(pm[1:3], em[1:3]):
            assert all(_equal(x, y) for x, y in zip(xs, ys))
        assert _equal(pm[3], em[3])
    else:
        assert pm[1:] == em[1:], (pm, em)
    return p


def check_clean(b, res, want, image, with_crc):
    """a clean call's outputs against the original data, the parts of lzgpu_encode_slices, their CRCs and zlib.crc32"""
    rc, bad, outs, ocrc, img = res
    assert rc == _lib.OK and (bad == [-1] * 4 if b.n else bad == [-7] * 4), (rc, bad)
    for g in range(b.n_parts):
        if not want[g]:
            assert outs[g] is None
            continue
        size = b.pbs[b.slice_of[g]] * BLOCK
        assert np.array_equal(outs[g][:, :size], b.parts[g]), g
        assert (outs[g][:, size:] == SENT).all(), g
        if with_crc:
            assert np.array_equal(ocrc[g], b.crcs[g]), g
            for c in {0, b.n - 1} if b.n else ():
                assert [zlib.crc32(outs[g][c, s * BLOCK:(s + 1) * BLOCK]) for s in range(size // BLOCK)] == list(ocrc[g][c]), g
    if image:
        assert np.array_equal(img[:, :b.nb * BLOCK], b.data) and (img[:, b.nb * BLOCK:] == SENT).all()


# (want every lost part or every lost part but the last, chunk image, output CRCs)
OPTS = {"image+crc": (False, True, True), "bare": (False, False, False), "subset": (True, False, True), "subset+image": (True, True, False)}


@gpu
@pytest.mark.parametrize("opts", list(OPTS))
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("shape", ["tail", "short"])
@pytest.mark.parametrize("name", list(SETS))
def test_pool_equals_one_context(eng, pools, name, shape, n, opts):
    names, given, nb_tail, nb_short = SETS[name]
    nb = nb_tail if shape == "tail" else nb_short
    b = Batch(eng, names, given, n, nb, seed=nb * 10 + n)
    subset, image, with_crc = OPTS[opts]
    want = b.lost()
    if subset:
        want[max(g for g in range(b.n_parts) if want[g])] = 0
    for pool in pools.values():
        check_clean(b, same(eng, pool, b, want, image, with_crc), want, image, with_crc)


@gpu
def test_a_full_64_mib_chunk_in_every_share(eng, pools):
    names, given, _, _ = RESCUE
    b = Batch(eng, names, given, 3, 1024, seed=5)
    for pool in pools.values():
        check_clean(b, same(eng, pool, b), b.lost(), True, True)


@gpu
@pytest.mark.parametrize("where", ["first_share", "last_share", "two_shares"])
def test_a_corrupt_stored_crc_is_reported_at_its_chunk_in_the_batch(eng, pools, where):
    """8 chunks: shares [0, 4) [4, 8) of a two-slot pool, [0, 3) [3, 6) [6, 8) of a three-slot pool.  Given flat parts 4 (ec(3,2)
    parity row 0), 7, 9 and 10 (ec(4,2) data part 2, parity rows 0 and 1).  With two, chunk 6 has the smaller (slice, part) but
    chunk 2 is reported."""
    names, given, nb, _ = RESCUE
    b = Batch(eng, names, given, 8, nb, seed=9)
    crcs = [c.copy() for c in b.crcs]
    hits = {"first_share": [(9, 1, 3)], "last_share": [(4, 7, 2)], "two_shares": [(4, 6, 0), (10, 2, 5)]}[where]
    for g, c, s in hits:
        crcs[g][c, s] ^= 1
    expect = min(b.where(c, g, s) for g, c, s in hits)
    for pool in pools.values():
        rc, bad, _, _, _ = same(eng, pool, b, crcs=crcs)
        assert rc == _lib.ERR_CRC and tuple(bad) == expect, (rc, bad, expect)
        with pytest.raises(L.ChunkCrcError) as e:
            pool.recover_slices(b.goals, b.nb, [p if x else None for p, x in zip(b.parts, given)], [c if x else None for c, x in zip(crcs, given)])
        assert e.value.where == expect


# refusals: (slice names, given, nb, wanted parts beyond the lost ones, code)
REFUSALS = {
    # one data part of xor2 alone: most positions are not determined
    "too_few_parts": (("xor2", "xor3"), [1, 0, 0, 0, 0, 0, 0], 13, [], _lib.ERR_TOO_FEW_PARTS),
    # a given part is also wanted
    "given_and_wanted": RESCUE[:2] + (RESCUE[2], [4], _lib.ERR_ARG),
    # L = lcm(9, 8) = 72 > 64
    "L_over_64": (("ec(9,2)", "ec(8,2)"), [1] * 9 + [0, 0] + [1] * 10, 75, [], _lib.ERR_ARG),
    # every data part given, every parity part wanted: 274 CRC streams per combined stripe, more than the kernel's 192
    "over_192_blocks": (("ec(3,2)", "ec(4,2)", "ec(5,2)"), [1, 1, 1, 0, 0, 1, 1, 1, 1, 0, 0, 1, 1, 1, 1, 1, 0, 0], 63, [], _lib.ERR_ARG),
}


@gpu
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", list(REFUSALS))
def test_refusals_write_nothing(eng, pools, kind, n):
    names, given, nb, extra, code = REFUSALS[kind]
    b = Batch(eng, names, given, n, nb, seed=0, encode=False)
    want = b.lost()
    for g in extra:
        want[g] = 1
    for pool in pools.values():
        rc, bad, outs, ocrc, img = same(eng, pool, b, want)
        assert rc == code and bad == [-7] * 4, (rc, bad)
        assert all((o == SENT).all() for o in outs if o is not None) and (img == SENT).all()
        assert all((c == SENT_CRC).all() for c in ocrc if c is not None)


@gpu
@pytest.mark.parametrize("n", [2, 7])
def test_every_share_launches_the_recovery_kernel(eng, n):
    """a fresh three-slot pool: every slot with a share reports the recovery kernel at the plan's G, an idle slot nothing; the
    chunks recovered are counted once"""
    names, given, nb, _ = RESCUE
    b = Batch(eng, names, given, n, nb, seed=n)
    pool = L.Pool(_devices(3))
    try:
        pool.recover_slices(b.goals, nb, [p if x else None for p, x in zip(b.parts, given)], [c if x else None for c, x in zip(b.crcs, given)])
        G = L.Engine.plan_recover_slices(b.goals, nb, given)["G"]
        lib = pool.lib
        for i in range(3):
            _, count = L.Pool.share(n, 3, i)
            geo = _lib.LzLaunchGeometry()
            assert lib.lzgpu_debug_last_geometry(lib.lzgpu_pool_ctx(pool.h, i), C.byref(geo)) == _lib.OK
            if count:
                assert (geo.kernel, geo.G) == (_lib.KERNEL_RECOVER_SLICES, G), i
            else:
                assert geo.kernel == _lib.KERNEL_NONE, i
        assert pool.stats()["chunks_recovered"] == n
    finally:
        pool.close()


@gpu
def test_two_threads_recover_through_one_pool_at_once(eng, pools):
    """two threads issue pool recoveries at the same time, each on its own batch, several times: every result equals the one
    context's"""
    batches = [Batch(eng, *SETS[name][:2], 7, SETS[name][2], seed=30 + t) for t, name in enumerate(("ec(3,2)+ec(4,2)", "std+xor2+xor3"))]
    want = [_method(eng, b, b.lost(), True, True, b.crcs) for b in batches]
    errors = []

    def worker(t):
        try:
            for _ in range(3):
                for pool in pools.values():
                    got = _method(pool, batches[t], batches[t].lost(), True, True, batches[t].crcs)
                    assert got[0] == want[t][0] == 0
                    assert all(_equal(x, y) for xs, ys in zip(got[1:3], want[t][1:3]) for x, y in zip(xs, ys))
                    assert _equal(got[3], want[t][3])
        except Exception as exc:  # noqa: BLE001
            errors.append((t, repr(exc)))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(2)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
