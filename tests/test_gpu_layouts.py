"""The device-pointer entry points at the layouts callers use: padded strides, chunk-major parts, offset base pointers.

Every *_dev call takes caller strides and per-part pointers.  The rest of the suite passes them at their dense values, where a
kernel that ignored a stride parameter and computed the dense one itself would still be right.  Here every buffer is a guarded
device allocation (`Guarded`): 4 KiB of guard before and after the region the call is given, and every byte of it, guards and
stride gaps included, seeded random.  After a call the whole allocation is downloaded and compared with what it must hold: the
oracle's answer (tests/_oracle.py) in the output regions, the original bytes everywhere else.  So a stray store into a gap, a
guard, an input or the buffer of a part nobody asked for fails, and so does a kernel that reads a gap as data (the gaps hold
random bytes, not zeros).  The dense layout is one of the layouts of every parametrisation, so each padded or offset layout is
also byte-identical to the dense call.

Each case asserts the route it means to test (the launch count of stats(), last_launch(), plan_encode, plan_convert), so a layout
that silently moved a call to another route fails instead of passing untested."""
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
GUARD = 4096
ZERO_CRC = 0xD7978EEB          # CRC of a 64 KiB zero block (the blocks a short data part does not have)
N = 3                          # chunks per batch

_engines = {}
_cache = {}
_scratch = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in _engines.values():
        e.close()
    _engines.clear()
    _cache.clear()
    _scratch.clear()


def engine(**env):
    """one context per set of switches; they are read when a context is created, so they are set around its creation only"""
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


def rnd(nbytes, seed):
    return np.frombuffer(np.random.default_rng(seed).bytes(nbytes), dtype=np.uint8).copy()


def u8(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(-1)


class Guarded:
    """One device allocation: GUARD bytes, `lead` more, the `nbytes` region a call is given, GUARD bytes; all seeded random.
    `put` writes input rows (into the initial image and the expected one), `expect` sets what rows must hold after the call,
    `undefined` excludes rows whose content the call leaves undefined; `check` compares every byte of the allocation."""

    def __init__(self, nbytes, seed, lead=0):
        self.lead = GUARD + lead
        self.init = rnd(self.lead + nbytes + GUARD, seed)
        self.want = self.init.copy()
        self.skip = None
        self.t = None

    @property
    def ptr(self):
        if self.t is None:
            self.t = torch.from_numpy(self.init).cuda()
        return self.t.data_ptr() + self.lead

    def _rows(self, arrs, byte0, stride, rows):
        for c, r in enumerate(rows):
            r = u8(r)
            o = self.lead + byte0 + c * stride
            for a in arrs:
                a[o:o + r.size] = r

    def put(self, byte0, stride, rows):
        assert self.t is None
        self._rows((self.init, self.want), byte0, stride, rows)

    def expect(self, byte0, stride, rows):
        self._rows((self.want,), byte0, stride, rows)

    def undefined(self, byte0, stride, n, length):
        if self.skip is None:
            self.skip = np.zeros(self.init.size, dtype=bool)
        self._rows((self.skip,), byte0, stride, [np.ones(length, dtype=bool)] * n)

    def check(self, what):
        if self.t is None:
            return                                      # never handed to the device
        got = self.t.cpu().numpy()
        diff = got != self.want
        if self.skip is not None:
            diff &= ~self.skip
        bad = np.flatnonzero(diff)
        assert bad.size == 0, f"{what}: {bad.size} bytes differ, the first at {int(bad[0]) - self.lead} from the region start"


class Parts:
    """n_parts part buffers of n chunks, part_bytes each, in one layout:
      dense / pad16 / pad64k   one allocation per part, stride part_bytes + 0 / 16 / 64 KiB + 48;
      chunk-major              the parts of a chunk next to each other in one allocation: part i of chunk c at
                               (c * n_parts + i) * part_bytes, stride n_parts * part_bytes;
      off16 / off48            one allocation per part, base pointer 16 / 48 bytes into it, stride + 16 / + 64 KiB + 48."""

    PAD = {"dense": 0, "pad16": 16, "pad64k": BLOCK + 48, "chunk-major": 0, "off16": 16, "off48": BLOCK + 48}
    LEAD = {"off16": 16, "off48": 48}

    def __init__(self, layout, n_parts, n, part_bytes, seed):
        self.layout, self.n = layout, n
        self.part_bytes = part_bytes
        if layout == "chunk-major":
            self.stride = n_parts * part_bytes
            g = Guarded(n * self.stride, seed)
            self.bufs = [(g, i * part_bytes) for i in range(n_parts)]
            self.allocs = [g]
        else:
            self.stride = part_bytes + self.PAD[layout]
            self.allocs = [Guarded((n - 1) * self.stride + part_bytes, seed + i, self.LEAD.get(layout, 0)) for i in range(n_parts)]
            self.bufs = [(g, 0) for g in self.allocs]

    def ptr(self, i):
        g, b = self.bufs[i]
        return g.ptr + b

    def put(self, i, rows):
        g, b = self.bufs[i]
        g.put(b, self.stride, rows)

    def expect(self, i, rows):
        g, b = self.bufs[i]
        g.expect(b, self.stride, rows)

    def undefined(self, i):
        g, b = self.bufs[i]
        g.undefined(b, self.stride, self.n, self.part_bytes)

    def gap(self, i, c):
        """(allocation, byte) of a byte in the stride gap after chunk c of part i, or None for a layout without gaps"""
        g, b = self.bufs[i]
        return None if self.stride == self.part_bytes or self.layout == "chunk-major" else (g, b + c * self.stride + self.part_bytes + 5)

    def check(self, what):
        for j, g in enumerate(self.allocs):
            g.check(f"{what} [{self.layout} allocation {j}]")


class Crcs:
    """per-part CRC arrays (n chunks x pb uint32, dense as the API has them) in guarded allocations, base 4 * lead bytes in"""

    def __init__(self, n_parts, n, pb, seed, lead=0):
        self.g = [Guarded(n * pb * 4, seed + i, 4 * lead) for i in range(n_parts)]

    def ptr(self, i):
        return self.g[i].ptr

    def check(self, what):
        for i, g in enumerate(self.g):
            g.check(f"{what} [CRC array {i}]")


def launches(e):
    return e.stats()["kernel_launches"]


def mark_launch(e):
    """a one-unit CRC launch first, so that last_launch() afterwards shows the launch of the call under test and nothing older"""
    if "blk" not in _scratch:
        _scratch["blk"] = torch.zeros(BLOCK, dtype=torch.uint8, device="cuda")
        _scratch["crc"] = torch.zeros(1, dtype=torch.int32, device="cuda")
    e.crc_blocks_dev(_scratch["blk"].data_ptr(), 1, _scratch["crc"].data_ptr())
    return e.last_launch()


def goal_tuple(goal):
    return (goal.kind, goal.k, goal.m)


def sliced(oracle, text, nb, n, seed):
    """chunks [n, nb*B], their k + m parts [n, pb*B] (data parts zero-padded) and each part's stored CRCs [n, pb]"""
    key = ("parts", text, nb, n, seed)
    if key not in _cache:
        goal = L.SliceType(text)
        k, m = goal.k, goal.m
        pb = -(-nb // k)
        data = rnd(n * nb * BLOCK, seed).reshape(n, nb * BLOCK)
        ref = [oracle.encode_chunk(goal.kind, k, m, data[c]) for c in range(n)]
        parity = np.stack([r[0] for r in ref])
        crc = np.stack([r[1] for r in ref])
        per = [O.split_parts(data[c], k)[0] for c in range(n)]
        parts = [np.stack([per[c][j] for c in range(n)]) for j in range(k)] + [np.ascontiguousarray(parity[:, r]) for r in range(m)]
        crcs = []
        for j in range(k):
            cj = np.full((n, pb), ZERO_CRC, dtype=np.uint32)
            mine = crc[:, j:nb:k]
            cj[:, : mine.shape[1]] = mine
            crcs.append(cj)
        crcs += [np.ascontiguousarray(crc[:, nb + r * pb: nb + (r + 1) * pb]) for r in range(m)]
        _cache[key] = (data, parts, crcs)
    return _cache[key]


# ---- encode --------------------------------------------------------------------------------------------------------------------

ENCODE = [
    # goal, blocks per chunk, bytes short of whole blocks (a partial last block), switches, route
    ("ec(8,2)", 61, 0, {}, "fused"),               # folded
    ("ec(8,2)", 61, 1000, {}, "fused"),
    ("xor2", 33, 0, {}, "fused"),
    ("ec(5,3)", 43, 7, {}, "fused"),               # three packed-byte rows
    ("ec(8,4)", 67, 0, {}, "fused"),               # bit-sliced, four rows
    ("ec(8,3)", 37, 4095, {}, "fused"),            # bit-sliced, three rows
    ("ec(7,2)", 31, 0, {}, "fused"),               # runtime k
    ("ec(21,4)", 50, 0, {}, "fused"),              # Cauchy rows
    ("ec(8,6)", 37, 100, {}, "fused"),             # two passes: rows 0-3, then 4-5 at 4 * pb blocks into each chunk's parity
    ("ec(8,2)", 61, 1000, dict(LZGPU_DISABLE_FUSED=1), "generic"),
]
# chunk stride pad, parity stride pad, CRC stride pad (elements), base offsets of data, parity, CRC (bytes)
ENCODE_LAYOUTS = {
    "dense": (0, 0, 0, 0, 0, 0),
    "pad16": (16, BLOCK + 48, 1, 0, 0, 0),
    "pad64k": (BLOCK + 48, 16, 5, 0, 0, 0),
    "off16": (16, 48, 1, 16, 48, 4),
    "off48": (BLOCK + 48, BLOCK + 16, 5, 48, 16, 8),
}


def _eid(case):
    env = ",".join(f"{k[6:]}={v}" for k, v in sorted(case[3].items()))
    return f"{case[0]}-{case[1]}-short{case[2]}" + (f"-{env}" if env else "")


@pytest.mark.parametrize("layout", list(ENCODE_LAYOUTS))
@pytest.mark.parametrize("case", ENCODE, ids=[_eid(c) for c in ENCODE])
def test_encode_at_strides(oracle, case, layout):
    text, nb, short, env, route = case
    goal = L.SliceType(text)
    m, pb = goal.m, -(-nb // goal.k)
    n_crc = nb + m * pb
    chunk_len = nb * BLOCK - short
    cpad, ppad, crcpad, dlead, plead, clead = ENCODE_LAYOUTS[layout]
    cs, ps, crs = nb * BLOCK + cpad, m * pb * BLOCK + ppad, n_crc + crcpad
    key = ("enc", text, nb, short)
    if key not in _cache:
        data = rnd(N * chunk_len, 100 + nb + short).reshape(N, chunk_len)
        ref = [oracle.encode_chunk(goal.kind, goal.k, m, data[c]) for c in range(N)]
        _cache[key] = (data, [r[0] for r in ref], [r[1] for r in ref])
    data, p_ref, c_ref = _cache[key]
    gd = Guarded((N - 1) * cs + nb * BLOCK, 11, dlead)
    gp = Guarded((N - 1) * ps + m * pb * BLOCK, 12, plead)
    gc = Guarded(((N - 1) * crs + n_crc) * 4, 13, clead)
    gd.put(0, cs, data)
    if short:
        gd.expect(chunk_len, cs, [np.zeros(short, np.uint8)] * N)     # the rest of the last block is zero-filled in place
    gp.expect(0, ps, p_ref)
    gc.expect(0, crs * 4, c_ref)
    e = engine(**env)
    plan = e.plan_encode(goal, N, nb, chunk_stride=cs)
    assert plan["fused"] == 1, plan                     # the build's route; LZGPU_DISABLE_FUSED=1 moves the call off it
    ptrs = (gd.ptr, gp.ptr, gc.ptr)
    torch.cuda.synchronize()
    before = mark_launch(e)
    e.encode_chunks_dev(goal, N, chunk_len, ptrs[0], cs, ptrs[1], ps, ptrs[2], crs)
    e.sync()
    if route == "fused":
        grid, units = e.last_launch()
        if plan["passes"] == 1:
            assert units == plan["units"], (units, plan)
        else:
            assert (grid, units) != before
    else:
        assert e.last_launch() == (0, 0)
    gd.check("data")
    gp.check("parity")
    gc.check("CRC")


# ---- degraded read -------------------------------------------------------------------------------------------------------------

RECOVER = [
    # name, goal, missing parts, wanted parts besides the missing data parts, blocks, switches, route
    ("k8", "ec(8,2)", (1, 4), (), 61, {}, "fused"),
    ("geo0", "ec(7,2)", (2,), (), 27, dict(LZGPU_RECOVER_GEO=0), "fused"),
    ("geo1", "ec(7,2)", (2, 5), (), 27, dict(LZGPU_RECOVER_GEO=1), "fused"),
    ("geo2", "ec(6,3)", (0, 2, 5), (), 29, dict(LZGPU_RECOVER_GEO=2, LZGPU_BS_RECOVER=0), "fused"),
    ("two", "ec(8,2)", (3,), (), 40, dict(LZGPU_RECOVER_TWO=1), "fused"),
    ("direct", "ec(8,6)", (0, 3), (), 37, dict(LZGPU_DIRECT_WIDE=0), "fused"),
    ("direct-wide", "ec(21,4)", (3, 9), (), 50, dict(LZGPU_DIRECT_WIDE=1), "fused"),
    ("bs3", "ec(5,3)", (0, 2, 4), (), 24, {}, "fused"),
    ("parity-wanted", "ec(8,2)", (1, 9), (9,), 61, {}, "generic"),
    ("unwanted-parity", "ec(8,2)", (1, 9), (), 61, {}, "fused"),    # parity part 9 is missing, not wanted, its buffer given
    ("fused-off", "ec(8,2)", (1, 4), (), 61, dict(LZGPU_DISABLE_FUSED=1), "off"),
]
LAYOUTS = ["dense", "pad16", "pad64k", "chunk-major", "off16", "off48"]
IMAGE_PAD = {"dense": 0, "pad16": BLOCK + 32, "pad64k": 16, "chunk-major": 32, "off16": 48, "off48": BLOCK + 16}


def check_route(e, route, before, n_launches):
    if route == "fused":          # one launch of the degraded-read kernel (it verifies in the same pass)
        grid, units = e.last_launch()
        assert n_launches == 1 and (grid, units) != before and units >= N, (n_launches, before, grid, units)
    elif route == "generic":      # GF dot product (not a persistent kernel), gather, CRC passes
        assert n_launches > 1 or e.last_launch() == before, (n_launches, before)
    else:
        assert e.last_launch() == (0, 0) and n_launches >= 1, n_launches


def run_recover(oracle, case, layout, verify, image, corrupt=None, gap=False):
    """one degraded read; corrupt = (chunk, part, block) of a flipped bit in an input part, gap: a flipped byte in a stride gap"""
    name, text, missing, extra, nb, env, route = case
    goal = L.SliceType(text)
    k, m = goal.k, goal.m
    pb = -(-nb // k)
    data, parts, crcs = sliced(oracle, text, nb, N, 300 + nb)
    want = [1 if (i in missing and i < k) or i in extra else 0 for i in range(k + m)]
    P = Parts(layout, k + m, N, pb * BLOCK, 20)
    for i in range(k + m):
        if i not in missing:
            rows = parts[i]
            if corrupt and corrupt[1] == i:
                rows = rows.copy()
                rows[corrupt[0], corrupt[2] * BLOCK + 333] ^= 0x10
            P.put(i, rows)
        elif want[i]:
            if corrupt:
                P.undefined(i)
            else:
                P.expect(i, parts[i])
    if gap:
        g, b = P.gap(next(i for i in range(k + m) if i not in missing), 1)
        g.init[g.lead + b] ^= 0xFF
        g.want[g.lead + b] ^= 0xFF
    C = None
    if verify:
        C = Crcs(k + m, N, pb, 40, 1 if layout.startswith("off") else 0)
        for i in range(k + m):
            if i not in missing:
                C.g[i].put(0, pb * 4, crcs[i])
    img, istride = None, nb * BLOCK + IMAGE_PAD[layout]
    if image:
        img = Guarded((N - 1) * istride + nb * BLOCK, 50, Parts.LEAD.get(layout, 0))
        if corrupt:
            img.undefined(0, istride, N, nb * BLOCK)
        else:
            img.expect(0, istride, data)
    e = engine(**env)
    d_parts = [0 if i in missing else P.ptr(i) for i in range(k + m)]
    d_out = [P.ptr(i) for i in range(k + m)]          # every part's buffer: only the wanted missing ones may change
    d_crc = [0 if i in missing else C.ptr(i) for i in range(k + m)] if verify else None
    d_img = img.ptr if image else None
    torch.cuda.synchronize()
    before = mark_launch(e)
    n0 = launches(e)
    where = None
    try:
        e.recover_chunks_dev(goal, N, nb, d_parts, P.stride, d_crc, want, d_out, d_img, istride if image else None)
    except L.ChunkCrcError as ex:
        where = ex.where
    e.sync()
    check_route(e, route, before, launches(e) - n0)
    what = f"{name} {layout} verify={verify} image={image}"
    P.check(what)
    if verify:
        C.check(what)
    if image:
        img.check(what + " image")
    return where


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("case", RECOVER, ids=[c[0] for c in RECOVER])
def test_recover_at_layouts(oracle, case, layout):
    for verify in (False, True):
        for image in (False, True):
            assert run_recover(oracle, case, layout, verify, image) is None


@pytest.mark.parametrize("layout", ["pad16", "chunk-major", "off48"])
@pytest.mark.parametrize("case", [RECOVER[0], RECOVER[7], RECOVER[10]], ids=["k8", "bs3", "fused-off"])
def test_recover_reports_a_corrupt_block_and_ignores_the_gaps(oracle, case, layout):
    """a flipped bit in a data block of an input part is reported at its (chunk, part, block); a flipped byte in a stride gap is
    not data: it changes nothing and is not reported"""
    missing, k = case[2], L.SliceType(case[1]).k
    part = next(i for i in range(k) if i not in missing)
    assert run_recover(oracle, case, layout, True, True, corrupt=(2, part, 1)) == (2, part, 1)
    if layout != "chunk-major":
        assert run_recover(oracle, case, layout, True, True, gap=True) is None


def test_full_chunks_chunk_major_recover_with_image(oracle):
    """two 64 MiB ec(8,2) chunks, chunk-major, data parts 1 and 4 lost, verified, with the chunk image at a padded stride"""
    goal = L.SliceType("ec(8,2)")
    n, nb, pb = 2, 1024, 128
    data, parts, crcs = sliced(oracle, "ec(8,2)", nb, n, 777)
    lost = (1, 4)
    P = Parts("chunk-major", 10, n, pb * BLOCK, 70)
    C = Crcs(10, n, pb, 80)
    for i in range(10):
        if i in lost:
            P.expect(i, parts[i])
        else:
            P.put(i, parts[i])
            C.g[i].put(0, pb * 4, crcs[i])
    istride = nb * BLOCK + 48
    img = Guarded((n - 1) * istride + nb * BLOCK, 90, 16)
    img.expect(0, istride, data)
    e = engine()
    before = mark_launch(e)
    n0 = launches(e)
    e.recover_chunks_dev(goal, n, nb, [0 if i in lost else P.ptr(i) for i in range(10)], P.stride,
                         [0 if i in lost else C.ptr(i) for i in range(10)], [1 if i in lost else 0 for i in range(10)],
                         [P.ptr(i) if i in lost else 0 for i in range(10)], img.ptr, istride)
    e.sync()
    assert launches(e) - n0 == 1 and e.last_launch() != before
    P.check("parts")
    C.check("stored CRCs")
    img.check("image")


# ---- slice conversion ----------------------------------------------------------------------------------------------------------

CONVERT = [
    # name, source, lost source parts, blocks, destination, switches, route
    ("one-pass", "ec(8,2)", (1, 4), 61, "ec(3,2)", {}, "one-pass"),
    ("split-encode", "ec(5,3)", (0, 2, 4), 24, "ec(3,2)", {}, "two-pass"),
    ("convert-fused-off", "ec(8,2)", (1, 4), 61, "ec(3,2)", dict(LZGPU_CONVERT_FUSED=0), "two-pass"),
    ("std-source", "std", (), 20, "ec(3,2)", {}, "two-pass"),
    ("std-destination", "ec(8,2)", (1,), 61, "std", {}, "image"),
]
# (source layout, destination layout): every pair has part_stride != out_stride
CONVERT_LAYOUTS = [("dense", "pad16"), ("pad16", "pad64k"), ("chunk-major", "off48"), ("off16", "chunk-major"), ("pad64k", "off16")]


def slice_of(text):
    return L.SliceType(2, 1, 0) if text == "std" else L.SliceType(text)


def convert_inputs(oracle, src_name, nb, seed):
    """source parts [n, pbs*B] and their stored CRCs [n, pbs]; a standard source is the chunk itself"""
    if src_name != "std":
        data, parts, crcs = sliced(oracle, src_name, nb, N, seed)
        return parts, crcs
    data = rnd(N * nb * BLOCK, seed).reshape(N, nb * BLOCK)
    crc = np.array([[zlib.crc32(data[c, b * BLOCK:(b + 1) * BLOCK].tobytes()) for b in range(nb)] for c in range(N)], dtype=np.uint32)
    return [data], [crc]


def run_convert(oracle, case, layouts, verify, corrupt=None):
    name, src_name, lost, nb, dst_name, env, route = case
    src, dst = slice_of(src_name), slice_of(dst_name)
    ns, nd = src.k + src.m, dst.k + dst.m
    pbs, pbd = -(-nb // src.k), -(-nb // dst.k)
    parts, crcs = convert_inputs(oracle, src_name, nb, 500 + nb)
    want = [1] * nd
    key = ("conv", name, nb)
    if key not in _cache:
        ref = [O.convert_chunk(oracle, goal_tuple(src), [None if i in lost else parts[i][c] for i in range(ns)],
                               [None if i in lost else crcs[i][c] for i in range(ns)], goal_tuple(dst), want, nb) for c in range(N)]
        assert all(r[0] == 0 for r in ref)
        _cache[key] = ([np.stack([r[1][i] for r in ref]) for i in range(nd)], [np.stack([r[2][i] for r in ref]) for i in range(nd)])
    want_out, want_crc = _cache[key]
    S = Parts(layouts[0], ns, N, pbs * BLOCK, 100)
    D = Parts(layouts[1], nd, N, pbd * BLOCK, 110)
    assert S.stride != D.stride
    for i in range(ns):
        if i not in lost:
            rows = parts[i]
            if corrupt and corrupt[1] == i:
                rows = rows.copy()
                rows[corrupt[0], corrupt[2] * BLOCK + 77] ^= 0x01
            S.put(i, rows)
    OC = Crcs(nd, N, pbd, 120, 1)
    for i in range(nd):
        if corrupt:
            D.undefined(i)
            OC.g[i].undefined(0, pbd * 4, N, pbd * 4)
        else:
            D.expect(i, want_out[i])
            OC.g[i].expect(0, pbd * 4, want_crc[i])
    SC = None
    if verify:
        SC = Crcs(ns, N, pbs, 130, 1 if layouts[0].startswith("off") else 0)
        for i in range(ns):
            if i not in lost:
                SC.g[i].put(0, pbs * 4, crcs[i])
    e = engine(**env)
    if src_name != "std" and dst_name != "std":
        plan = L.Engine.plan_convert(src, dst, [0 if i in lost else 1 for i in range(ns)], want)
        assert plan["one_pass"] == (name == "one-pass" or "CONVERT_FUSED" in str(env)), plan
    d_parts = [0 if i in lost else S.ptr(i) for i in range(ns)]
    d_out = [D.ptr(i) for i in range(nd)]
    torch.cuda.synchronize()
    before = mark_launch(e)
    n0 = launches(e)
    where = None
    try:
        e.convert_chunks_dev(src, dst, N, nb, d_parts, S.stride, want, d_out, D.stride,
                             d_part_crc=[0 if i in lost else SC.ptr(i) for i in range(ns)] if verify else None,
                             d_out_crc=[OC.ptr(i) for i in range(nd)])
    except L.ChunkCrcError as ex:
        where = ex.where
    e.sync()
    grid, units = e.last_launch()
    if route == "one-pass":           # the one-pass kernel, then the CRCs of the destination slice dealt out to its parts
        assert units == N * -(-nb // (plan["stripes_per_unit"] * dst.k)) and launches(e) - n0 == 2, (grid, units, plan)
    elif route == "two-pass":         # degraded read into the chunk image (none for a standard source), then split + encode
        assert launches(e) - n0 >= 2 and (grid, units) != before
    else:                             # a standard destination: the degraded read writes the image straight into d_out[0]
        assert (grid, units) != before
    what = f"{name} {layouts} verify={verify}"
    S.check(what + " source")
    D.check(what + " destination")
    OC.check(what + " destination")
    if verify:
        SC.check(what + " source")
    return where


@pytest.mark.parametrize("layouts", CONVERT_LAYOUTS, ids=["-to-".join(p) for p in CONVERT_LAYOUTS])
@pytest.mark.parametrize("case", CONVERT, ids=[c[0] for c in CONVERT])
def test_convert_at_layouts(oracle, case, layouts):
    for verify in (False, True):
        assert run_convert(oracle, case, layouts, verify) is None


@pytest.mark.parametrize("case", [CONVERT[0], CONVERT[2]], ids=["one-pass", "convert-fused-off"])
def test_convert_reports_a_corrupt_block(oracle, case):
    assert run_convert(oracle, case, ("pad16", "off48"), True, corrupt=(1, 2, 3)) == (1, 2, 3)


@pytest.mark.parametrize("layout", ["pad16", "chunk-major", "off48"])
def test_convert_same_slice_rebuild(oracle, layout):
    """src == dst: lost parts are rebuilt into their own slots, so the strides must be equal; unequal ones are refused"""
    goal = L.SliceType("ec(8,2)")
    nb, pb, lost = 45, 6, (1, 4)
    data, parts, crcs = sliced(oracle, "ec(8,2)", nb, N, 610)
    want = [1 if i in lost else 0 for i in range(10)]
    want[0] = 1                                     # an available part, its output buffer = its input buffer: nothing to do
    P = Parts(layout, 10, N, pb * BLOCK, 140)
    for i in range(10):
        (P.expect if i in lost else P.put)(i, parts[i])
    OC = Crcs(10, N, pb, 150)
    for i in range(10):
        if want[i]:
            OC.g[i].expect(0, pb * 4, crcs[i])
    e = engine()
    d_parts = [0 if i in lost else P.ptr(i) for i in range(10)]
    d_out = [P.ptr(i) if want[i] else 0 for i in range(10)]
    d_oc = [OC.ptr(i) if want[i] else 0 for i in range(10)]
    n0 = launches(e)
    with pytest.raises(L.LzGpuError) as ei:
        e.convert_chunks_dev(goal, goal, N, nb, d_parts, P.stride, want, d_out, P.stride + 16, d_out_crc=d_oc)
    assert ei.value.status == _lib.ERR_ARG and launches(e) == n0
    torch.cuda.synchronize()
    before = mark_launch(e)
    e.convert_chunks_dev(goal, goal, N, nb, d_parts, P.stride, want, d_out, P.stride, d_out_crc=d_oc)
    e.sync()
    assert e.last_launch() != before
    P.check("parts")
    OC.check("CRCs")


# ---- split, CRC, prefixes, block writes, fill ------------------------------------------------------------------------------------

@pytest.mark.parametrize("text,nb", [("ec(3,2)", 20), ("ec(8,2)", 61)])
def test_split_at_padded_strides(oracle, text, nb):
    """chunk order -> data parts at chunk stride + 48 (base + 16) and part stride + 64 KiB + 16; a NULL part is not written"""
    goal = L.SliceType(text)
    k, pb = goal.k, -(-nb // goal.k)
    data = rnd(N * nb * BLOCK, 700 + nb).reshape(N, nb * BLOCK)
    per = [O.split_parts(data[c], k)[0] for c in range(N)]
    cs, ps = nb * BLOCK + 48, pb * BLOCK + BLOCK + 16
    gd = Guarded((N - 1) * cs + nb * BLOCK, 160, 16)
    gd.put(0, cs, data)
    span = (N - 1) * ps + pb * BLOCK                   # all parts in one allocation, so the NULL part 1 lies between two others
    gp = Guarded(k * span, 170, 48)
    for j in range(k):
        if j != 1:
            gp.expect(j * span, ps, [per[c][j] for c in range(N)])
    e = engine()
    n0 = launches(e)
    e.split_chunks_dev(goal, N, nb, gd.ptr, cs, [0 if j == 1 else gp.ptr + j * span for j in range(k)], ps)
    e.sync()
    assert launches(e) - n0 == 1
    gd.check("chunks")
    gp.check("parts")


CRC_CASES = [
    # block length, stride, base offset (bytes past a 16-byte boundary)
    (65536, 65536, 0), (65536, 65540, 4), (65536, 65536 + 64, 0), (4096, 4100, 4), (1000, 1024, 12),
] + [(n, n + 4 - n % 4 + 8, 4) for n in (1, 2, 3, 4, 124, 127, 128, 129, 132, 4092, 4096, 4100, 65532, 65535)]


@pytest.mark.parametrize("block_len,stride,lead", CRC_CASES)
def test_crc_blocks_at_strides(block_len, stride, lead):
    """crc_blocks_dev against zlib: padded strides (64 KiB blocks at 65540 = the chunk-file record layout), a base that is only
    4-byte aligned, and block lengths of 32w - 1, 32w and 32w + 1 words around the warp tree of crc_blocks_kernel"""
    n = 150                                            # three units of the fused CRC kernel
    g = Guarded((n - 1) * stride + block_len, block_len + stride, lead)
    blocks = [g.init[g.lead + b * stride: g.lead + b * stride + block_len] for b in range(n)]
    ref = np.array([zlib.crc32(b.tobytes()) for b in blocks], dtype=np.uint32)
    out = Guarded(n * 4, 180, 4)
    out.expect(0, 0, [ref])
    e = engine()
    ptrs = (g.ptr, out.ptr)
    torch.cuda.synchronize()
    before = mark_launch(e)
    n0 = launches(e)
    e.crc_blocks_dev(ptrs[0], n, ptrs[1], block_len=block_len, block_stride=stride)
    e.sync()
    assert launches(e) - n0 == 1
    fused = (block_len, stride) == (BLOCK, BLOCK)
    assert (e.last_launch() != before) == fused            # whole dense blocks take the fused CRC kernel, the rest crc_blocks_kernel
    g.check("blocks")
    out.check("CRCs")


def test_write_data_prefixes_at_padded_crc_stride(oracle):
    goal = L.SliceType("ec(5,3)")
    k, m, nb = 5, 3, 23
    pb = -(-nb // k)
    n_crc = nb + m * pb
    crs = n_crc + 3
    crc = np.frombuffer(rnd(N * n_crc * 4, 190), dtype=np.uint32).reshape(N, n_crc)
    ids = np.array([0x0102030405060708, 0xFFEEDDCCBBAA9988, 7], dtype=np.uint64)
    gc = Guarded(((N - 1) * crs + n_crc) * 4, 191, 4)
    gc.put(0, crs * 4, crc)
    gi = Guarded(N * 8, 192, 8)
    gi.put(0, 0, [ids])
    go = Guarded(N * (k + m) * pb * 38, 193, 16)
    want = np.zeros((N, k + m, pb, 38), dtype=np.uint8)
    for c in range(N):
        for part in range(k + m):
            for s in range(pb):
                if part < k and s * k + part >= nb:
                    continue                                   # a block a short data part does not have: 38 zero bytes
                v = int(crc[c, s * k + part]) if part < k else int(crc[c, nb + (part - k) * pb + s])
                want[c, part, s] = O.write_data_prefix(oracle, int(ids[c]), 1000 + (c * (k + m) + part) * pb + s, s, 0, BLOCK, v)
    go.expect(0, 0, [want])
    e = engine()
    ptrs = (gc.ptr, gi.ptr, go.ptr)
    e.write_data_prefixes_dev(goal, N, nb, ptrs[0], crs, ptrs[1], ptrs[2], write_id_base=1000)
    e.sync()
    gc.check("CRCs")
    gi.check("chunk ids")
    go.check("prefixes")


def block_write_records(shapes, rng, payload_base):
    """lzgpu_block_write records for one write per block with the given (offset, size), payloads at odd offsets"""
    recs = (_lib.LzBlockWrite * len(shapes))()
    payloads, pos = [], payload_base
    for i, (off, size) in enumerate(shapes):
        data = np.frombuffer(rng.bytes(size), dtype=np.uint8)
        crc = zlib.crc32(data.tobytes())
        if i % 7 == 3:
            crc ^= 0x40                                         # a corrupt packet
        exists = i % 5 != 4 or (off == 0 and size == BLOCK)
        recs[i].block, recs[i].offset, recs[i].size, recs[i].crc = i, off, size, crc
        recs[i].payload_off, recs[i].exists, recs[i].status = pos, int(exists), 0
        payloads.append((pos, data))
        pos += size + 2 + size % 2                              # the next payload_off is odd again
    return recs, payloads, pos


def test_write_blocks_dev_with_odd_payload_offsets(oracle):
    """block_write_kernel called directly: payloads at odd offsets inside a guarded payload buffer, against hdd_write"""
    rng = np.random.default_rng(200)
    shapes = [(0, BLOCK), (0, 1), (1, 65535), (65535, 1), (100, 1000), (12345, 1), (7, 4097), (32768, 32768), (3, 0), (60000, 5536),
              (0, 4096), (65533, 3)]
    n = len(shapes)
    blocks = np.frombuffer(rng.bytes(n * BLOCK), dtype=np.uint8).reshape(n, BLOCK).copy()
    stored = np.array([zlib.crc32(b.tobytes()) for b in blocks], dtype=np.uint32)
    recs, payloads, total = block_write_records(shapes, rng, 1)
    assert all(recs[i].payload_off % 2 == 1 for i in range(n))
    gb = Guarded(n * BLOCK, 201, 16)
    gb.put(0, BLOCK, blocks)
    gs = Guarded(n * 4, 202, 4)
    gs.put(0, 0, [stored])
    gpay = Guarded(total, 203)
    for pos, data in payloads:
        gpay.put(pos, 0, [data])
    code = {0: 0, -3: _lib.ERR_CRC, -4: _lib.ERR_DAMAGED, -1: _lib.ERR_ARG}
    expect = []
    for i, (off, size) in enumerate(shapes):
        pos, data = payloads[i]
        rc, blk, new_crc = O.hdd_write_block(oracle, blocks[i] if recs[i].exists else None, int(stored[i]), off, size, recs[i].crc,
                                             data if size else np.zeros(1, np.uint8))
        expect.append(code[rc])
        if rc == 0:
            gb.expect(i * BLOCK, 0, [blk])
            gs.expect(i * 4, 0, [np.array([new_crc], dtype=np.uint32)])
    assert set(expect) == {0, _lib.ERR_CRC}
    d_wr = torch.from_numpy(np.frombuffer(bytes(recs), dtype=np.uint8).copy()).cuda()
    e = engine()
    ptrs = (gb.ptr, gs.ptr, gpay.ptr)
    e.write_blocks_dev(ptrs[0], ptrs[1], ptrs[2], d_wr.data_ptr(), n)
    e.sync()
    done = (_lib.LzBlockWrite * n).from_buffer_copy(d_wr.cpu().numpy().tobytes())
    assert [done[i].status for i in range(n)] == expect
    gb.check("blocks")
    gs.check("stored CRCs")
    gpay.check("payload")


def test_write_blocks_host_path_second_tile(oracle):
    """more than 8192 requests: the host path stages them in tiles of 8192, so the second tile (w0 > 0) runs"""
    n = 8192 + 300
    rng = np.random.default_rng(210)
    blocks = np.frombuffer(rng.bytes(n * BLOCK), dtype=np.uint8).reshape(n, BLOCK).copy()
    stored = np.array([zlib.crc32(b.tobytes()) for b in blocks], dtype=np.uint32)
    writes = []
    for i in range(n):
        off, size = (i * 37) % 60000, 1 + i % 300
        data = np.frombuffer(rng.bytes(size), dtype=np.uint8)
        crc = zlib.crc32(data.tobytes()) ^ (1 if i % 1000 == 999 else 0)
        writes.append(dict(block=(i * 7919) % n, offset=off, data=data, crc=crc))
    before_blocks, before_crc = blocks.copy(), stored.copy()
    status = engine().write_blocks(blocks, stored, writes)
    for i, w in enumerate(writes):
        b = w["block"]
        rc, blk, new_crc = O.hdd_write_block(oracle, before_blocks[b], int(before_crc[b]), w["offset"], w["data"].size, w["crc"], w["data"])
        assert status[i] == {0: 0, -3: _lib.ERR_CRC}[rc], (i, status[i], rc)
        assert (blocks[b] == blk).all() and stored[b] == new_crc, i
    assert status.count(_lib.ERR_CRC) == n // 1000


def test_fill_chunks_leaves_the_stride_gaps(oracle):
    n, clen, cs = 4, 3 * BLOCK + 104, 3 * BLOCK + 104 + 4096 + 8
    g = Guarded((n - 1) * cs + clen, 220, 8)
    g.expect(0, cs, [O.fill_chunk(oracle, clen, 4242, 5 + c) for c in range(n)])
    e = engine()
    e.fill_chunks_dev(g.ptr, n, clen, cs, 4242, first_chunk=5)
    e.sync()
    g.check("chunks")


# ---- misaligned pointers are refused before anything is enqueued ---------------------------------------------------------------

def _recover_args(kind):
    goal = L.SliceType("ec(3,2)")
    nb, pb = 6, 2
    buf = _scratch.setdefault("align", torch.zeros(48 * BLOCK, dtype=torch.uint8, device="cuda"))
    base = buf.data_ptr()
    part = [base + i * 2 * pb * BLOCK for i in range(5)]
    crc = [base + 12 * pb * BLOCK + i * 64 for i in range(5)]
    d_parts = [part[0], 0, part[2], part[3], part[4]]
    d_out = [0, part[1], 0, 0, 0]
    d_crc = [crc[0], 0, crc[2], crc[3], crc[4]]
    img = base + 14 * pb * BLOCK
    if kind == "part":
        d_parts[2] += 8
    elif kind == "out":
        d_out[1] += 8
    elif kind == "image":
        img += 8
    elif kind == "part_crc":
        d_crc[3] += 2
    return goal, nb, pb, d_parts, d_out, d_crc, img


@pytest.mark.parametrize("kind", ["part", "out", "image", "part_crc"])
def test_recover_refuses_misaligned_pointers(kind):
    goal, nb, pb, d_parts, d_out, d_crc, img = _recover_args(kind)
    e = engine()
    n0 = launches(e)
    with pytest.raises(L.LzGpuError) as ei:
        e.recover_chunks_dev(goal, 1, nb, d_parts, 2 * pb * BLOCK, d_crc, [0, 1, 0, 0, 0], d_out, img, nb * BLOCK)
    assert ei.value.status == _lib.ERR_ARG and "aligned" in str(ei.value)
    assert launches(e) == n0


@pytest.mark.parametrize("kind", ["part", "out", "part_crc", "out_crc"])
def test_convert_refuses_misaligned_pointers(kind):
    goal, nb, pb, d_parts, d_out, d_crc, img = _recover_args(kind if kind != "out_crc" else None)
    dst = L.SliceType("xor2")
    pbd = 3
    out = [img, img + pbd * BLOCK, img + 2 * pbd * BLOCK]
    ocrc = [d_crc[0] + 16 * i for i in range(3)]
    if kind == "out":
        out[2] += 8
    elif kind == "out_crc":
        ocrc[1] += 1
    e = engine()
    n0 = launches(e)
    with pytest.raises(L.LzGpuError) as ei:
        e.convert_chunks_dev(goal, dst, 1, nb, d_parts, 2 * pb * BLOCK, [1, 1, 1], out, pbd * BLOCK, d_part_crc=d_crc, d_out_crc=ocrc)
    assert ei.value.status == _lib.ERR_ARG and "aligned" in str(ei.value)
    assert launches(e) == n0


@pytest.mark.parametrize("kind", ["data", "part"])
def test_split_and_fill_refuse_misaligned_pointers(kind):
    goal, nb, pb, d_parts, d_out, d_crc, img = _recover_args(None)
    parts = [d_parts[0], d_parts[2], d_parts[3]]
    data = img
    if kind == "data":
        data += 8
    else:
        parts[1] += 4
    e = engine()
    n0 = launches(e)
    with pytest.raises(L.LzGpuError) as ei:
        e.split_chunks_dev(goal, 1, nb, data, nb * BLOCK, parts, 2 * pb * BLOCK)
    assert ei.value.status == _lib.ERR_ARG and "aligned" in str(ei.value)
    assert launches(e) == n0
    if kind == "data":
        with pytest.raises(L.LzGpuError) as ei:
            e.fill_chunks_dev(img + 4, 1, 64, 64, 1)
        assert ei.value.status == _lib.ERR_ARG
