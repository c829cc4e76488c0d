"""Recovery of a chunk of a multi-slice goal from the given parts of every slice together (lzgpu_recover_slices*, recover_slices_kernel
in csrc/recover_slices_kernel.cuh) on the GPU.

Every wanted part, its block CRCs and the chunk image are compared with the original data (the data parts and the image), with
lzgpu_encode_slices (parity), with the oracle's per-slice encode of the first chunk, and with zlib.crc32.  Covered, for each goal
set: loss patterns the per-slice rule loses but the given parts of all slices determine; patterns where one slice survives, against
lzgpu_convert_chunks from that slice; patterns that must refuse, where nothing is written.  Batch shapes: ragged nb, nb < L, a
partial last unit, one full 64 MiB chunk.  The _dev form with guard bytes around padded buffers and unwanted outputs; two corrupt
stored CRCs reported at the smaller (chunk, slice, part, block) on both forms.  Each case runs on the default context and with
LZGPU_GRID_CAP=2, and the launch is checked through lzgpu_debug_last_geometry against the plan."""
import os
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from lizardfs_b200.engine import ChunkCrcError, LzGpuError
from tests import _oracle as O
from tests.test_recover_slices_plan import layout, lcm_of, model, ref_lost

pytestmark = pytest.mark.gpu
BLOCK = 65536

_engines = {}


def engine(kind):
    env = {"default": {}, "cap2": {"LZGPU_GRID_CAP": "2"}}[kind]
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


@pytest.fixture(scope="module")
def oracle():
    return O.load_oracle()


def goals_of(names):
    return [L.SliceType(n) for n in names]


def original(goals, n, nb, seed):
    """data [n, nb * 64K] and every flat part [n, pb_i * 64K] with its block CRCs [n, pb_i], encoded by lzgpu_encode_slices"""
    rng = np.random.default_rng(seed)
    data = rng.integers(0, 256, size=(n, nb * BLOCK), dtype=np.uint8)
    enc = engine("default").encode_slices(goals, data)
    parts, crcs = [], []
    for g, (par, crc) in zip(goals, enc):
        if g.is_std:
            parts.append(data)
            crcs.append(crc)
            continue
        k, pb = g.k, -(-nb // g.k)
        padded = np.zeros((n, pb * k * BLOCK), dtype=np.uint8)
        padded[:, :nb * BLOCK] = data
        blocks = padded.reshape(n, pb, k, BLOCK)
        for j in range(k):
            parts.append(np.ascontiguousarray(blocks[:, :, j, :]).reshape(n, pb * BLOCK))
            c = np.full((n, pb), zlib.crc32(bytes(BLOCK)), dtype=np.uint32)
            idx = np.arange(pb) * k + j
            c[:, idx < nb] = crc[:, idx[idx < nb]]
            crcs.append(c)
        for r in range(g.m):
            parts.append(np.ascontiguousarray(par[:, r]))
            crcs.append(np.ascontiguousarray(crc[:, nb + r * pb: nb + (r + 1) * pb]))
    return data, parts, crcs


def zlib_crcs(part):
    n, size = part.shape
    return np.array([[zlib.crc32(part[c, b * BLOCK:(b + 1) * BLOCK].tobytes()) for b in range(size // BLOCK)] for c in range(n)],
                    dtype=np.uint32)


def check_oracle(oracle, goals, data, parts):
    """the first chunk's parity parts against the oracle's per-slice encode"""
    g0 = 0
    for g in goals:
        n_p = 1 if g.is_std else g.k + g.m
        if not g.is_std:
            par, _ = oracle.encode_chunk(g.kind, g.k, g.m, data[0])
            for r in range(g.m):
                if parts[g0 + g.k + r] is not None:
                    assert np.array_equal(parts[g0 + g.k + r][0], par[r])
        g0 += n_p


def check_geometry(e, goals, nb, n, given):
    p = e.plan_recover_slices(goals, nb, given)
    geo = e.last_geometry()
    n_cs = -(-nb // p["L"])
    assert geo["kernel"] == _lib.KERNEL_RECOVER_SLICES
    assert (geo["G"], geo["threads"], geo["stages"], geo["smem_bytes"]) == (p["G"], p["threads"], p["stages"], p["smem_bytes"])
    upc = -(-n_cs // p["G"])                      # units per chunk; the host form may launch once per tile of chunks
    assert geo["units"] % upc == 0 and 0 < geo["units"] <= upc * n
    if e is engine("cap2"):
        assert geo["grid"] <= 2


def run_and_check(oracle, e, goals, nb, n, given, seed, image=True):
    data, parts, crcs = original(goals, n, nb, seed)
    inp = [p if given[g] else None for g, p in enumerate(parts)]
    incrc = [c if given[g] else None for g, c in enumerate(crcs)]
    out, ocrc, img = e.recover_slices(goals, nb, inp, incrc, chunk_image=image)
    check_geometry(e, goals, nb, n, given)
    for g in range(len(parts)):
        if given[g]:
            assert out[g] is None
            continue
        assert np.array_equal(out[g], parts[g]), g
        assert np.array_equal(ocrc[g], crcs[g]), g
        assert np.array_equal(ocrc[g][:1], zlib_crcs(out[g][:1])), g
    if image:
        assert np.array_equal(img, data)
    check_oracle(oracle, goals, data, out)
    return data, parts, crcs, out, ocrc


def rescue_patterns(goals, limit):
    """loss patterns the per-slice rule loses and the given parts of all slices fully determine (the plan agrees, checked on the CPU)"""
    _, n = layout(goals)
    Lc = lcm_of(goals)
    found = []
    for bits in range(1 << n):
        given = [(bits >> g) & 1 for g in range(n)]
        if ref_lost(goals, given) and model(goals, given, Lc)[1] == (1 << Lc) - 1:
            found.append(given)
    step = max(1, len(found) // limit)
    return found[::step][:limit]


SETS = [("xor2", "xor3"), ("ec(3,2)", "ec(2,2)"), ("ec(3,2)", "ec(4,2)"), ("std", "xor2", "xor3")]


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names", SETS, ids="+".join)
def test_rescue_patterns(oracle, names, ctx):
    goals = goals_of(names)
    Lc = lcm_of(goals)
    for i, given in enumerate(rescue_patterns(goals, 3)):
        # a full stripe batch and a ragged one (a tail stripe), two chunks each
        for nb in (4 * Lc, 3 * Lc + Lc // 2 + 1 if Lc > 2 else 7):
            run_and_check(oracle, engine(ctx), goals, nb, 2, given, seed=100 + i)


def survivor_patterns(goals):
    """for each xor/ec slice: exactly k of its parts given (the first data part lost where m allows), every other slice empty"""
    lay, n = layout(goals)
    for i, (k, m, base, _) in enumerate(lay):
        if m == 0:
            continue
        keep = list(range(base + 1, base + k + 1)) if m >= 1 else list(range(base, base + k))
        yield i, [1 if g in keep else 0 for g in range(n)]


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names", SETS, ids="+".join)
def test_one_slice_survives_equals_convert(oracle, names, ctx):
    goals = goals_of(names)
    e = engine(ctx)
    nb = 37
    lay, n = layout(goals)
    for si, given in survivor_patterns(goals):
        data, parts, crcs, out, ocrc = run_and_check(oracle, e, goals, nb, 2, given, seed=7 + si)
        src = goals[si]
        k, m, base, _ = lay[si]
        src_parts = [parts[base + j] if given[base + j] else None for j in range(k + m)]
        src_crc = [crcs[base + j] if given[base + j] else None for j in range(k + m)]
        for di, dst in enumerate(goals):
            dk, dm, dbase, _ = lay[di]
            nd = dk + dm
            want = [0 if given[dbase + j] else 1 for j in range(nd)]
            if not any(want):
                continue
            cout, ccrc = e.convert_chunks(src, dst, nb, src_parts, want, part_crc=src_crc)
            for j in range(nd):
                if want[j]:
                    assert np.array_equal(cout[j], out[dbase + j]), (names, si, di, j)
                    assert np.array_equal(ccrc[j], ocrc[dbase + j]), (names, si, di, j)


@pytest.mark.parametrize("names", SETS, ids="+".join)
def test_undetermined_patterns_refuse_and_write_nothing(names):
    goals = goals_of(names)
    lay, n = layout(goals)
    Lc = lcm_of(goals)
    e = engine("default")
    nb = 2 * Lc + 1
    # one data part of the first xor/ec slice and nothing else: most positions are unknown and no equation exists
    first = next(base for k, m, base, _ in lay if m)
    given = [1 if g == first else 0 for g in range(n)]
    assert model(goals, given, Lc)[1] != (1 << Lc) - 1
    data, parts, crcs = original(goals, 1, nb, 5)
    d_parts = [torch.from_numpy(p).cuda() if given[g] else None for g, p in enumerate(parts)]
    outs = [torch.full((parts[g].size,), 0x5A, dtype=torch.uint8, device="cuda") for g in range(n)]
    img = torch.full((nb * BLOCK,), 0x3C, dtype=torch.uint8, device="cuda")
    strides = [-(-nb // (1 if g.is_std else g.k)) * BLOCK for g in goals]
    want = [0 if given[g] else 1 for g in range(n)]
    with pytest.raises(LzGpuError) as ex:
        e.recover_slices_dev(goals, 1, nb, [t.data_ptr() if t is not None else 0 for t in d_parts], strides, None, want,
                             [o.data_ptr() for o in outs], strides, None, img.data_ptr(), nb * BLOCK)
    assert ex.value.status == _lib.ERR_TOO_FEW_PARTS
    torch.cuda.synchronize()
    assert all(bool((o == 0x5A).all()) for o in outs)
    assert bool((img == 0x3C).all())
    with pytest.raises(LzGpuError) as ex:
        e.recover_slices(goals, nb, [p if given[g] else None for g, p in enumerate(parts)])
    assert ex.value.status == _lib.ERR_TOO_FEW_PARTS


@pytest.mark.parametrize("ctx", ["default", "cap2"])
@pytest.mark.parametrize("names,nb,n", [
    (("xor2", "xor3"), 1, 3),             # nb < L
    (("xor2", "xor3"), 1023, 2),          # ragged
    (("ec(3,2)", "ec(4,2)"), 7, 2),       # nb < L = 12
    (("ec(3,2)", "ec(8,2)"), 50, 2),      # L = 24, a tail of 2
    (("xor2", "ec(2,2)"), 11, 3),         # L = 2, G = 4: a partial last unit
    (("std", "xor2", "xor3"), 1024, 1),   # one full 64 MiB chunk
])
def test_batch_shapes(oracle, names, nb, n, ctx):
    goals = goals_of(names)
    # the first xor/ec slice keeps k of its parts (its data part 0 lost), every other slice is lost: each of its parts is rebuilt
    _, given = next(survivor_patterns(goals))
    run_and_check(oracle, engine(ctx), goals, nb, n, given, seed=nb)
    if names == ("xor2", "xor3"):
        run_and_check(oracle, engine(ctx), goals, nb, n, rescue_patterns(goals, 1)[0], seed=nb + 1)


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_dev_form_guard_bytes_sentinel_and_unwanted_outputs(ctx):
    e = engine(ctx)
    goals = goals_of(("ec(3,2)", "ec(4,2)"))
    lay, n_parts = layout(goals)
    nb, n = 29, 2
    given = rescue_patterns(goals, 1)[0]
    data, parts, crcs = original(goals, n, nb, 21)
    GUARD, OFF = 4096, 4096 + 48
    pbs = [-(-nb // g.k) for g in goals]
    slice_of = [i for i, g in enumerate(goals) for _ in range(g.k + g.m)]
    pstride = [pb * BLOCK + 4096 for pb in pbs]                  # padded strides
    bufs, d_parts, d_crc, d_out, d_ocrc, obufs, cbufs = [], [], [], [], [], [], []
    for g in range(n_parts):
        i = slice_of[g]
        if given[g]:
            b = torch.full((2 * GUARD + n * pstride[i],), 0x77, dtype=torch.uint8, device="cuda")
            for c in range(n):
                b[OFF + c * pstride[i]: OFF + c * pstride[i] + parts[g][c].size] = torch.from_numpy(parts[g][c]).cuda()
            cr = torch.from_numpy(np.ascontiguousarray(crcs[g]).view(np.int32).copy()).cuda()
            bufs += [b, cr]
            d_parts.append(b.data_ptr() + OFF)
            d_crc.append(cr.data_ptr())
            d_out.append(0)
            d_ocrc.append(0)
        else:
            d_parts.append(0)
            d_crc.append(0)
        if not given[g]:
            ob = torch.full((2 * GUARD + n * pstride[i],), 0x5A, dtype=torch.uint8, device="cuda")
            oc = torch.full((2 * GUARD // 4 + n * pbs[i],), 0x11223344, dtype=torch.int32, device="cuda")
            obufs.append((g, ob))
            cbufs.append((g, oc))
            d_out.append(ob.data_ptr() + OFF)
            d_ocrc.append(oc.data_ptr() + GUARD)
    # want every lost part but the last one: its buffers are passed and must stay untouched
    lost = [g for g in range(n_parts) if not given[g]]
    want = [1 if (g in lost and g != lost[-1]) else 0 for g in range(n_parts)]
    istride = (nb + 1) * BLOCK
    img = torch.full((2 * GUARD + n * istride,), 0x3C, dtype=torch.uint8, device="cuda")
    e.recover_slices_dev(goals, n, nb, d_parts, pstride, d_crc, want, d_out, pstride, d_ocrc, img.data_ptr() + OFF, istride)
    torch.cuda.synchronize()
    check_geometry(e, goals, nb, n, given)
    hi = img.cpu().numpy()
    assert (hi[:OFF] == 0x3C).all() and (hi[OFF + (n - 1) * istride + nb * BLOCK:] == 0x3C).all()
    for c in range(n):
        at = OFF + c * istride
        assert np.array_equal(hi[at: at + nb * BLOCK], data[c])
        assert (hi[at + nb * BLOCK: at + istride] == 0x3C).all()          # the sentinel block past nb
    for (g, ob), (_, oc) in zip(obufs, cbufs):
        i = slice_of[g]
        ho, hc = ob.cpu().numpy(), oc.cpu().numpy().view(np.uint32)
        size = pbs[i] * BLOCK
        if not want[g]:
            assert (ho == 0x5A).all() and (hc == 0x11223344).all()
            continue
        assert (ho[:OFF] == 0x5A).all() and (ho[OFF + (n - 1) * pstride[i] + size:] == 0x5A).all()
        for c in range(n):
            at = OFF + c * pstride[i]
            assert np.array_equal(ho[at: at + size], parts[g][c])
            assert (ho[at + size: at + pstride[i]] == 0x5A).all()
        g0 = GUARD // 4
        assert (hc[:g0] == 0x11223344).all() and (hc[g0 + n * pbs[i]:] == 0x11223344).all()
        assert np.array_equal(hc[g0: g0 + n * pbs[i]].reshape(n, pbs[i]), crcs[g])


@pytest.mark.parametrize("ctx", ["default", "cap2"])
def test_two_corrupt_stored_crcs_report_the_smaller(ctx):
    e = engine(ctx)
    goals = goals_of(("xor2", "xor3"))
    nb, n = 13, 3
    given = rescue_patterns(goals, 1)[0]
    data, parts, crcs = original(goals, n, nb, 33)
    lay, n_parts = layout(goals)
    g_hi = max(g for g in range(n_parts) if given[g])
    g_lo = min(g for g in range(n_parts) if given[g])
    bad_crcs = [c.copy() for c in crcs]
    bad_crcs[g_hi][1, 0] ^= 1         # chunk 1, the later part
    bad_crcs[g_lo][1, 2] ^= 1         # chunk 1, the earlier part: the smaller (chunk, slice, part, block)
    slice_of = [(i, g - base) for i, (k, m, base, _) in enumerate(lay) for g in range(base, base + k + m)]
    expect = (1, slice_of[g_lo][0], slice_of[g_lo][1], 2)
    inp = [p if given[g] else None for g, p in enumerate(parts)]
    incrc = [c if given[g] else None for g, c in enumerate(bad_crcs)]
    with pytest.raises(ChunkCrcError) as ex:
        e.recover_slices(goals, nb, inp, incrc)
    assert tuple(ex.value.where) == expect
    pbs = [-(-nb // g.k) for g in goals]
    d_parts = [torch.from_numpy(p).cuda() if given[g] else None for g, p in enumerate(parts)]
    d_crc = [torch.from_numpy(c.view(np.int32)).cuda() if given[g] else None for g, c in enumerate(bad_crcs)]
    outs = {g: torch.zeros(parts[g].size, dtype=torch.uint8, device="cuda") for g in range(n_parts) if not given[g]}
    strides = [pb * BLOCK for pb in pbs]
    with pytest.raises(ChunkCrcError) as ex:
        e.recover_slices_dev(goals, n, nb, [t.data_ptr() if t is not None else 0 for t in d_parts], strides,
                             [t.data_ptr() if t is not None else 0 for t in d_crc], [0 if given[g] else 1 for g in range(n_parts)],
                             [outs[g].data_ptr() if g in outs else 0 for g in range(n_parts)], strides)
    assert tuple(ex.value.where) == expect


def test_argument_refusals_launch_nothing():
    e = engine("default")
    goals = goals_of(("xor2", "xor3"))
    nb = 6
    data, parts, crcs = original(goals, 1, nb, 1)
    before = e.stats()["kernel_launches"]
    with pytest.raises(LzGpuError) as ex:
        e.recover_slices(goals_of(("xor2", "xor2")), nb, parts[:3] + parts[:3])
    assert ex.value.status == _lib.ERR_ARG
    with pytest.raises(LzGpuError) as ex:   # a given part wanted
        e.recover_slices(goals, nb, parts, want=[1] + [0] * 6)
    assert ex.value.status == _lib.ERR_ARG
    assert e.stats()["kernel_launches"] == before
