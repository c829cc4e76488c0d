"""lzgpu_recover_slices (recover_slices_kernel) at the limits of its stripe tables, on the GPU.

The requests of EDGES and SMEM_EDGE (test_recover_slices_geometry.py, checked on the CPU against a restatement of rs_geometry) reach
192 reads, 192 writes and 192 CRC streams per combined stripe, 64 wanted parity blocks, L = 63 with 63 unknowns and 62 equations,
64 flat parts, Cauchy rows up to 15 (rows 8-15 beside known positions), Vandermonde rows up to 2, four striped slices and G = 2.  Each runs at nb < L, at a ragged nb
and (G > 1) with a partial last unit, two of them also at one full 64 MiB chunk, on the default context and with LZGPU_GRID_CAP = 1
and 3, through the host form and the _dev form (padded strides, offset buffers, guard bytes, an image sentinel past nb).  Every
expected byte is the original random data or the oracle's encode_chunk of every chunk, every expected CRC is zlib.crc32; the launch
is checked against the plan.  The requests past a cap refuse with nothing launched or written.  Then the paths the other file does
not take: rot in blocks read only to verify them, a mismatch at flat part 63, stored CRCs on some parts only, no output CRCs, the
CRC-disabled mode, a wanted subset, and the host pipeline over four tiles."""
import ctypes as C
import os
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200.engine import ChunkCrcError, Engine, LzGpuError
from tests import _oracle as O
from tests.test_recover_slices_geometry import EDGES, REFUSED, SMEM_EDGE, edge_id, goals_of, lcm_of, pattern, slices
from tests.test_recover_slices_plan import _debug_rows

pytestmark = pytest.mark.gpu
BLOCK = 65536
FAKE_CRC = 0xFEDCBA98
CAPS = {"default": None, "cap1": 1, "cap3": 3}

_engines = {}


def engine(kind):
    if kind not in _engines:
        old = os.environ.get("LZGPU_GRID_CAP")
        if CAPS[kind]:
            os.environ["LZGPU_GRID_CAP"] = str(CAPS[kind])
        try:
            _engines[kind] = L.Engine(0)
        finally:
            if old is None:
                os.environ.pop("LZGPU_GRID_CAP", None)
            else:
                os.environ["LZGPU_GRID_CAP"] = old
    return _engines[kind]


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in _engines.values():
        e.close()
    _engines.clear()


@pytest.fixture(scope="module")
def oracle():
    return O.load_oracle()


def zlib_crcs(part):
    n, size = part.shape
    return np.array([[zlib.crc32(part[c, b * BLOCK:(b + 1) * BLOCK]) for b in range(size // BLOCK)] for c in range(n)], dtype=np.uint32)


class Original:
    """n random chunks of nb blocks; every flat part: data parts split from the chunk (short parts zero-padded), parity parts from the
    oracle's encode_chunk of each chunk; block CRCs of every part by zlib"""

    def __init__(self, oracle, names, n, nb, seed):
        self.names, self.n, self.nb = names, n, nb
        self.goals = goals_of(names)
        self.lay, self.n_parts = slices(names)
        self.L = lcm_of(self.lay)
        self.data = np.frombuffer(np.random.default_rng(seed).bytes(n * nb * BLOCK), dtype=np.uint8).reshape(n, nb * BLOCK)
        self.parts, self.slice_of, self.pbs = [], [], []
        for i, (name, g, (k, m, base, _)) in enumerate(zip(names, self.goals, self.lay)):
            pb = -(-nb // k)
            self.pbs.append(pb)
            self.slice_of += [i] * (k + m)
            if name == "std":
                self.parts.append(self.data)
                continue
            padded = np.zeros((n, pb * k * BLOCK), dtype=np.uint8)
            padded[:, :nb * BLOCK] = self.data
            blocks = padded.reshape(n, pb, k, BLOCK)
            self.parts += [np.ascontiguousarray(blocks[:, :, j]).reshape(n, pb * BLOCK) for j in range(k)]
            par = [oracle.encode_chunk(g.kind, k, m, self.data[c])[0] for c in range(n)]
            self.parts += [np.ascontiguousarray(np.stack([par[c][r] for c in range(n)])) for r in range(m)]
        self.crcs = [zlib_crcs(p) for p in self.parts]

    def where(self, g):
        """(slice, part in the slice) of flat part g"""
        i = self.slice_of[g]
        return i, g - self.lay[i][2]


_orig = {}


def original(oracle, names, n, nb, seed):
    key = (names, n, nb, seed)
    if key not in _orig:
        _orig.clear()
        _orig[key] = Original(oracle, names, n, nb, seed)
    return _orig[key]


def writable(goals, nb, given):
    """(want, image): every lost part whose blocks are determined in each stripe shape the call has (the plan's masks), and the image
    when every position is"""
    p = Engine.plan_recover_slices(goals, nb, given)
    lay, n = slices(tuple(str(g) for g in goals))
    Lc, tail = p["L"], nb % p["L"]
    shapes = ([(Lc, p["determined"])] if nb >= Lc else []) + ([(tail, p["tail_determined"])] if tail else [])
    want = [0] * n
    for k, m, base, _ in lay:
        for q in range(k + m):
            if given[base + q]:
                continue
            ok = True
            for valid, det in shapes:
                for s in range(Lc // k):
                    if s * k >= valid:
                        continue
                    pos = [s * k + q] if q < k else range(s * k, s * k + k)
                    ok &= all((det >> x) & 1 for x in pos if x < valid)
            want[base + q] = int(ok)
    image = all(det == (1 << Lc) - 1 for _, det in shapes)
    return want, image


def check_geometry(e, ctx, goals, nb, n, given, host):
    p = Engine.plan_recover_slices(goals, nb, given)
    geo = e.last_geometry()
    assert p["ok"] == 1
    assert geo["kernel"] == _lib.KERNEL_RECOVER_SLICES
    assert (geo["G"], geo["threads"], geo["stages"], geo["smem_bytes"]) == (p["G"], p["threads"], p["stages"], p["smem_bytes"])
    upc = -(-(-(-nb // p["L"])) // p["G"])        # units per chunk
    if host:                                       # the host form may launch once per tile of chunks
        assert geo["units"] % upc == 0 and 0 < geo["units"] <= upc * n
    else:
        assert geo["units"] == upc * n
    assert 1 <= geo["grid"] <= geo["units"]
    if CAPS[ctx]:
        assert geo["grid"] <= CAPS[ctx]


def run_host(o, e, ctx, given, want, image, crc=True):
    inp = [p if given[g] else None for g, p in enumerate(o.parts)]
    incrc = [c if given[g] else None for g, c in enumerate(o.crcs)] if crc else None
    out, ocrc, img = e.recover_slices(o.goals, o.nb, inp, incrc, want=want, chunk_image=image)
    check_geometry(e, ctx, o.goals, o.nb, o.n, given, True)
    for g in range(o.n_parts):
        if not want[g]:
            assert out[g] is None and ocrc[g] is None
            continue
        assert np.array_equal(out[g], o.parts[g]), (g, o.where(g))
        assert np.array_equal(ocrc[g], o.crcs[g]), (g, o.where(g))
    if image:
        assert np.array_equal(img, o.data)


GUARD, OFF = 4096, 4096 + 48


def run_dev(o, e, ctx, given, want, image):
    """the _dev form at padded strides, every buffer offset into a guarded allocation; unwanted lost parts get buffers that must stay
    untouched; the image has a sentinel block past nb"""
    n, nb = o.n, o.nb
    pstride = [pb * BLOCK + 4096 + 16 * i for i, pb in enumerate(o.pbs)]
    ostride = [pb * BLOCK + 8192 + 32 * i for i, pb in enumerate(o.pbs)]
    keep, d_parts, d_crc, d_out, d_ocrc, outs = [], [], [], [], [], {}
    for g in range(o.n_parts):
        i = o.slice_of[g]
        size = o.pbs[i] * BLOCK
        if given[g]:
            h = np.full(2 * GUARD + n * pstride[i], 0x77, dtype=np.uint8)
            for c in range(n):
                h[OFF + c * pstride[i]: OFF + c * pstride[i] + size] = o.parts[g][c]
            b = torch.from_numpy(h).cuda()
            cr = torch.from_numpy(o.crcs[g].reshape(-1).view(np.int32).copy()).cuda()
            keep += [b, cr]
            d_parts.append(b.data_ptr() + OFF)
            d_crc.append(cr.data_ptr())
            d_out.append(0)
            d_ocrc.append(0)
            continue
        ob = torch.full((2 * GUARD + n * ostride[i],), 0x5A, dtype=torch.uint8, device="cuda")
        oc = torch.full((2 * GUARD // 4 + n * o.pbs[i],), 0x11223344, dtype=torch.int32, device="cuda")
        outs[g] = (ob, oc)
        d_parts.append(0)
        d_crc.append(0)
        d_out.append(ob.data_ptr() + OFF)
        d_ocrc.append(oc.data_ptr() + GUARD)
    istride = (nb + 1) * BLOCK
    img = torch.full((2 * GUARD + n * istride,), 0x3C, dtype=torch.uint8, device="cuda") if image else None
    e.recover_slices_dev(o.goals, n, nb, d_parts, pstride, d_crc, want, d_out, ostride, d_ocrc,
                         img.data_ptr() + OFF if image else None, istride if image else 0)
    torch.cuda.synchronize()
    check_geometry(e, ctx, o.goals, nb, n, given, False)
    for g, (ob, oc) in outs.items():
        i = o.slice_of[g]
        size = o.pbs[i] * BLOCK
        ho, hc = ob.cpu().numpy(), oc.cpu().numpy().view(np.uint32)
        if not want[g]:
            assert (ho == 0x5A).all() and (hc == 0x11223344).all(), g
            continue
        assert (ho[:OFF] == 0x5A).all() and (ho[OFF + (n - 1) * ostride[i] + size:] == 0x5A).all(), g
        for c in range(n):
            at = OFF + c * ostride[i]
            assert np.array_equal(ho[at: at + size], o.parts[g][c]), (g, o.where(g), c)
            assert (ho[at + size: at + ostride[i]] == 0x5A).all(), g
        g0 = GUARD // 4
        assert (hc[:g0] == 0x11223344).all() and (hc[g0 + n * o.pbs[i]:] == 0x11223344).all(), g
        assert np.array_equal(hc[g0: g0 + n * o.pbs[i]].reshape(n, o.pbs[i]), o.crcs[g]), (g, o.where(g))
    if image:
        hi = img.cpu().numpy()
        assert (hi[:OFF] == 0x3C).all() and (hi[OFF + n * istride:] == 0x3C).all()
        for c in range(n):
            at = OFF + c * istride
            assert np.array_equal(hi[at: at + nb * BLOCK], o.data[c]), c
            assert (hi[at + nb * BLOCK: at + istride] == 0x3C).all(), c      # the sentinel block past nb
    del keep


def edge_cases():
    rows = [(names, spec, nbs) for names, spec, _, nbs in EDGES] + [(SMEM_EDGE[0], SMEM_EDGE[1], (47, SMEM_EDGE[2]))]
    out = []
    for names, spec, nbs in rows:
        for nb in nbs:
            out.append(pytest.param(names, spec, nb, id=f"{edge_id((names, spec))}-nb{nb}"))
    return out


@pytest.mark.parametrize("names,spec,nb", edge_cases())
def test_edge_rows(oracle, names, spec, nb):
    goals = goals_of(names)
    given = pattern(names, spec)
    n = 1 if nb == 1024 else 2
    o = original(oracle, names, n, nb, seed=nb + len(names))
    want, image = writable(goals, nb, given)
    lost = [0 if given[g] else 1 for g in range(o.n_parts)]
    if names == ("ec(7,3)", "ec(9,5)") and nb >= o.L:
        # E = 62 < 63 unknowns in a full stripe: no part is determined, the call only verifies the given parts
        assert not any(want) and not image
    else:
        assert want == lost and image
    for ctx in CAPS:
        e = engine(ctx)
        run_host(o, e, ctx, given, want, image)
        run_dev(o, e, ctx, given, want, image)


def test_partial_last_unit_is_reached():
    """the G = 2 rows run a count of combined stripes that G does not divide"""
    for names, spec, lit, nbs in EDGES:
        if lit["G"] > 1:
            assert any(-(-nb // lit["L"]) % lit["G"] for nb in nbs), names


@pytest.mark.parametrize("names,spec,over", REFUSED, ids=[edge_id(r) for r in REFUSED])
def test_refused_requests_launch_and_write_nothing(oracle, names, spec, over):
    goals = goals_of(names)
    given = pattern(names, spec)
    lay, n_parts = slices(names)
    nb, n = lcm_of(lay) + 3, 1
    assert Engine.plan_recover_slices(goals, nb, given)["ok"] == 0
    want, image = writable(goals, nb, given)
    pbs = [-(-nb // g.k) for g in goals]
    slice_of = [i for i, (k, m, _, _) in enumerate(lay) for _ in range(k + m)]
    e = engine("default")
    before = e.stats()["kernel_launches"]
    src = torch.zeros(max(pbs) * BLOCK, dtype=torch.uint8, device="cuda")
    outs = {g: torch.full((pbs[slice_of[g]] * BLOCK,), 0x5A, dtype=torch.uint8, device="cuda") for g in range(n_parts) if want[g]}
    img = torch.full((nb * BLOCK,), 0x3C, dtype=torch.uint8, device="cuda")
    strides = [pb * BLOCK for pb in pbs]
    with pytest.raises(LzGpuError) as ex:
        e.recover_slices_dev(goals, n, nb, [src.data_ptr() if given[g] else 0 for g in range(n_parts)], strides, None, want,
                             [outs[g].data_ptr() if g in outs else 0 for g in range(n_parts)], strides, None,
                             img.data_ptr() if image else None, nb * BLOCK if image else 0)
    assert ex.value.status == _lib.ERR_ARG
    torch.cuda.synchronize()
    assert all(bool((t == 0x5A).all()) for t in outs.values()) and bool((img == 0x3C).all())
    host = [np.zeros((n, pbs[slice_of[g]] * BLOCK), dtype=np.uint8) if given[g] else None for g in range(n_parts)]
    with pytest.raises(LzGpuError) as ex:
        e.recover_slices(goals, nb, host, want=want, chunk_image=image)
    assert ex.value.status == _lib.ERR_ARG
    assert e.stats()["kernel_launches"] == before


# ------------------------------------------------------------------------------------------------------------------------------
# the paths test_gpu_recover_slices.py does not take, on ec(3,2) + ec(4,2) and on an edge row
# ------------------------------------------------------------------------------------------------------------------------------
MID = ("ec(3,2)", "ec(4,2)")
WIDE = ("ec(16,16)", "ec(8,16)", "ec(4,4)")


def rot(parts, g, c, blk, at=12345):
    out = list(parts)
    out[g] = parts[g].copy()
    out[g][c, blk * BLOCK + at] ^= 0x40
    return out


def expect_crc_error(o, e, given, parts, crcs, want, where):
    inp = [p if given[g] else None for g, p in enumerate(parts)]
    incrc = [c if given[g] else None for g, c in enumerate(crcs)]
    with pytest.raises(ChunkCrcError) as ex:
        e.recover_slices(o.goals, o.nb, inp, incrc, want=want)
    assert tuple(ex.value.where) == where
    strides = [pb * BLOCK for pb in o.pbs]
    d_parts = [torch.from_numpy(p).cuda() if given[g] else None for g, p in enumerate(parts)]
    d_crc = [torch.from_numpy(c.view(np.int32)).cuda() if given[g] else None for g, c in enumerate(crcs)]
    outs = {g: torch.zeros(parts[g].size, dtype=torch.uint8, device="cuda") for g in range(o.n_parts) if want[g]}
    with pytest.raises(ChunkCrcError) as ex:
        e.recover_slices_dev(o.goals, o.n, o.nb, [t.data_ptr() if t is not None else 0 for t in d_parts], strides,
                             [t.data_ptr() if t is not None else 0 for t in d_crc], want,
                             [outs[g].data_ptr() if g in outs else 0 for g in range(o.n_parts)], strides)
    assert tuple(ex.value.where) == where


@pytest.mark.parametrize("ctx", ["default", "cap1"])
def test_rot_in_blocks_read_only_to_verify(oracle, ctx):
    """every data part of every slice given: the data blocks of the later slices are second copies, read only for their stored CRCs,
    and the parity blocks of a slice without unknowns are no equation.  Rot there (stored CRC kept) is found, and reported before
    rot in a staged block of a later chunk"""
    e = engine(ctx)
    # ec(3,2) + ec(4,2): the data of both and the parity of ec(4,2) given, the parity of ec(3,2) rebuilt
    o = original(oracle, MID, 3, 29, 5)
    given = pattern(MID, "data")
    given[9] = given[10] = 1
    want = [0, 0, 0, 1, 1] + [0] * 6
    staged = rot(o.parts, 1, 1, 0)                        # ec(3,2) data part 1, chunk 1: a staged first copy
    expect_crc_error(o, e, given, rot(staged, 7, 0, 3), o.crcs, want, (0, 1, 2, 3))     # ec(4,2) data part 2: a second copy
    expect_crc_error(o, e, given, rot(staged, 9, 0, 5), o.crcs, want, (0, 1, 4, 5))     # ec(4,2) parity row 0: no equation
    # the 64-part set with its data parts given: the data of ec(8,16) and ec(4,4) are second copies
    o = original(oracle, WIDE, 2, 41, 6)
    given = pattern(WIDE, "data")
    want = [0 if given[g] else 1 for g in range(64)]
    staged = rot(o.parts, 5, 1, 2)
    expect_crc_error(o, e, given, rot(staged, 59, 0, 9), o.crcs, want, (0, 2, 3, 9))    # ec(4,4) data part 3, flat part 59


@pytest.mark.parametrize("ctx", ["default", "cap3"])
def test_mismatch_at_flat_part_63(oracle, ctx):
    """the 64-part set with its parity parts given: 16 unknowns from the 16 Cauchy rows of ec(16,16), so the parity of ec(8,16) and
    ec(4,4) is read only to verify it; rot in flat part 63 (the last parity part of ec(4,4)) is reported as slice 2, part 7"""
    e = engine(ctx)
    o = original(oracle, WIDE, 2, 41, 7)
    given = pattern(WIDE, "parity")
    nu, ne, unk, es, er, est, rows, det = _debug_rows(o.goals, given, 16)
    assert (nu, ne) == (16, 16) and not es[:ne].any()
    want = [0 if given[g] else 1 for g in range(64)]
    expect_crc_error(o, e, given, rot(rot(o.parts, 16, 1, 0), 63, 0, 10), o.crcs, want, (0, 2, 7, 10))
    bad = [c.copy() for c in o.crcs]
    bad[63][1, 3] ^= 1
    bad[40][1, 4] ^= 1                                     # ec(8,16) parity row 0, the smaller flat part
    expect_crc_error(o, e, given, o.parts, bad, want, (1, 1, 8, 4))


def test_stored_crcs_on_some_parts_and_none(oracle):
    """only the parts with stored CRCs are verified: rot in a second copy without them is neither reported nor used; without any
    stored CRC the bytes are the same"""
    e = engine("default")
    for names, nb, rotten in [(MID, 29, 6), (WIDE, 41, 57)]:
        o = original(oracle, names, 2, nb, 8)
        given = pattern(names, "data")
        k0 = o.lay[0][0]
        want = [0 if given[g] else 1 for g in range(o.n_parts)]
        parts = rot(o.parts, rotten, 1, 1)
        inp = [p if given[g] else None for g, p in enumerate(parts)]
        incrc = [o.crcs[g] if g < k0 else None for g in range(o.n_parts)]    # the data parts of slice 0 only
        for pc in (incrc, None):
            out, ocrc, img = e.recover_slices(o.goals, nb, inp, pc, want=want, chunk_image=True)
            assert np.array_equal(img, o.data)
            for g in range(o.n_parts):
                if want[g]:
                    assert np.array_equal(out[g], o.parts[g]) and np.array_equal(ocrc[g], o.crcs[g]), (names, g)


def test_without_output_crcs(oracle):
    e = engine("default")
    for names, spec, nb in [(MID, [0, 1, 9], 31), (("ec(7,4)", "ec(9,4)"), "data", 143)]:
        o = original(oracle, names, 2, nb, 9)
        given = pattern(names, spec)
        want, image = writable(o.goals, nb, given)
        inp = [p if given[g] else None for g, p in enumerate(o.parts)]
        incrc = [c if given[g] else None for g, c in enumerate(o.crcs)]
        out, ocrc, _ = e.recover_slices(o.goals, nb, inp, incrc, want=want, with_crc=False)
        assert any(want) and all(c is None for c in ocrc)
        for g in range(o.n_parts):
            if want[g]:
                assert np.array_equal(out[g], o.parts[g]), (names, g)


def test_crc_disabled_mode(oracle):
    """as lzgpu_recover_chunks: every output CRC is LZGPU_FAKE_CRC, stored CRCs equal to it pass and any other fails, the bytes are
    unchanged"""
    lib = _lib.load()
    e = engine("default")
    try:
        lib.lzgpu_set_crc_enabled(0)
        for names, spec, nb in [(MID, [0, 1, 9, 10], 31), (WIDE, "parity", 41)]:
            o = original(oracle, names, 2, nb, 10)
            given = pattern(names, spec)
            want, image = writable(o.goals, nb, given)
            inp = [p if given[g] else None for g, p in enumerate(o.parts)]
            fake = [np.full_like(c, FAKE_CRC) if given[g] else None for g, c in enumerate(o.crcs)]
            out, ocrc, img = e.recover_slices(o.goals, nb, inp, fake, want=want, chunk_image=image)
            if image:
                assert np.array_equal(img, o.data)
            for g in range(o.n_parts):
                if want[g]:
                    assert np.array_equal(out[g], o.parts[g]) and (ocrc[g] == FAKE_CRC).all(), (names, g)
            g = max(g for g in range(o.n_parts) if given[g])
            fake[g] = o.crcs[g]                                   # a real CRC is a mismatch in this mode
            with pytest.raises(ChunkCrcError) as ex:
                e.recover_slices(o.goals, nb, inp, fake, want=want)
            assert tuple(ex.value.where) == (0,) + o.where(g) + (0,)
    finally:
        lib.lzgpu_set_crc_enabled(1)
    assert lib.lzgpu_crc_enabled() == 1


def host_call(e, o, parts, want, outs, ocrcs, img):
    """lzgpu_recover_slices on caller buffers"""
    lib = _lib.load()
    ns = len(o.goals)
    ptrs = lambda arrs: (C.c_void_p * len(arrs))(*[a.ctypes.data if a is not None else None for a in arrs])  # noqa: E731
    strides = (C.c_size_t * ns)(*[pb * BLOCK for pb in o.pbs])
    w = np.asarray(want, dtype=np.uint8)
    bad = (C.c_int64 * 4)(-1, -1, -1, -1)
    arr = (_lib.LzGoal * ns)(*[g.c for g in o.goals])
    return lib.lzgpu_recover_slices(e.h, arr, ns, o.n, o.nb, ptrs(parts), strides, None, w.ctypes.data_as(C.c_void_p), ptrs(outs), strides,
                                    ptrs(ocrcs), img.ctypes.data_as(C.c_void_p) if img is not None else None, o.nb * BLOCK, bad)


def test_wanted_subset_on_the_host_form(oracle):
    """a subset of the determined lost parts: the others get no output; one more part whose positions are not all determined refuses
    with LZGPU_ERR_TOO_FEW_PARTS and nothing written.  ec(7,3) + ec(9,5) from its parity: every position of a 62-block chunk, none
    of a data part in a full stripe"""
    e = engine("default")
    for names, spec, nb_yes, nb_no in [(MID, [0, 1, 9], 31, 31), (("ec(7,3)", "ec(9,5)"), "parity", 62, 125)]:
        given = pattern(names, spec)
        o = original(oracle, names, 2, nb_yes, 11)
        able, _ = writable(o.goals, nb_yes, given)
        yes = [g for g in range(o.n_parts) if able[g]]
        assert len(yes) >= 2
        want = [1 if g == yes[-1] else 0 for g in range(o.n_parts)]
        inp = [p if given[g] else None for g, p in enumerate(o.parts)]
        out, ocrc, _ = e.recover_slices(o.goals, nb_yes, inp, want=want)
        assert np.array_equal(out[yes[-1]], o.parts[yes[-1]]) and np.array_equal(ocrc[yes[-1]], o.crcs[yes[-1]])
        assert all(out[g] is None for g in range(o.n_parts) if g != yes[-1])
        o = original(oracle, names, 2, nb_no, 11)
        able, image = writable(o.goals, nb_no, given)
        no = [g for g in range(o.n_parts) if not given[g] and not able[g]]
        assert no and not image
        want = [1 if able[g] and g == yes[-1] else 0 for g in range(o.n_parts)]
        want[no[0]] = 1
        inp = [p if given[g] else None for g, p in enumerate(o.parts)]
        outs = [np.full(o.parts[g].shape, 0x5A, dtype=np.uint8) if want[g] else None for g in range(o.n_parts)]
        ocrcs = [np.full(o.crcs[g].shape, 0x11223344, dtype=np.uint32) if want[g] else None for g in range(o.n_parts)]
        before = e.stats()["kernel_launches"]
        assert host_call(e, o, inp, want, outs, ocrcs, None) == _lib.ERR_TOO_FEW_PARTS
        assert e.stats()["kernel_launches"] == before
        assert all((a == 0x5A).all() for a in outs if a is not None) and all((c == 0x11223344).all() for c in ocrcs if c is not None)


def test_host_pipeline_over_four_tiles(oracle):
    """four 64 MiB chunks of xor2 + xor3, one chunk per staging tile: every chunk correct, a stored-CRC mismatch in tile 2 reported at
    its chunk index in the batch, then a correct call on the same context"""
    e = engine("default")
    names = ("xor2", "xor3")
    o = original(oracle, names, 4, 1024, 12)
    given = [1, 0, 1, 0, 0, 0, 0]                          # xor2 data part 0 and parity: everything else rebuilt
    want, image = writable(o.goals, 1024, given)
    assert image and sum(want) == 5
    run_host(o, e, "default", given, want, True)
    assert e.last_geometry()["units"] == 1024 // 6 + 1     # one chunk per launch: 171 units of G = 1 combined stripe
    bad = [c.copy() for c in o.crcs]
    bad[2][2, 300] ^= 1
    inp = [p if given[g] else None for g, p in enumerate(o.parts)]
    with pytest.raises(ChunkCrcError) as ex:
        e.recover_slices(o.goals, 1024, inp, [c if given[g] else None for g, c in enumerate(bad)], want=want, chunk_image=True)
    assert tuple(ex.value.where) == (2, 0, 2, 300)
    run_host(o, e, "default", given, want, True)
