"""Persistent kernels with several work units per CTA.

Every streaming kernel (fused encode and CRC, fused_recover_kernel in its three geometries and its DIRECT form, bs_recover3_kernel,
fused_convert_kernel) is a loop over work units: CTA b takes units b, b + grid, b + 2 grid, ...  State runs from one unit into the
next: the refill of the next unit's first stages while the current one finishes, the stage / phase counters of the mbarrier rings,
the double-buffered block-CRC scratch, the bit-sliced GF warps' own unit loop, the atomicMin of the first CRC mismatch.  On the
default grid (one or two CTAs per SM) the small batches of the other tests give every CTA one unit, so none of that runs there.

Here every context is created with LZGPU_GRID_CAP = 1, 2, 3 or 7, and every batch has more than twice as many units as CTAs; the
odd caps give CTAs different unit counts and put the ragged last unit of a chunk in the middle of a CTA's walk.
lzgpu_debug_last_launch (Engine.last_launch) shows the grid and unit count of each launch, so a call that took another route, or a
launch site that ignores the cap, fails instead of passing without testing anything.  Every byte and CRC is compared with the oracle
(tests/_oracle.py) or with the original data a rebuilt part was withheld from."""
import math
import os
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from tests import _oracle as O

pytestmark = pytest.mark.gpu
BLOCK = 65536
CAPS = (1, 2, 3, 7)
N = 16                         # chunks per batch: at least one unit each, so every capped grid has units >= 2 * grid + 1
ZERO_CRC = 0xD7978EEB          # CRC of a 64 KiB zero block (the blocks a short data part does not have)

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


def engine(cap=None, **env):
    """one context per (cap, switches); the switches are read when a context is created, so they are set around its creation only"""
    env = {k: str(v) for k, v in env.items() if v is not None}
    if cap is not None:
        env["LZGPU_GRID_CAP"] = str(cap)
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


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def ptr(t):
    return 0 if t is None else t.data_ptr()


def host(t, dtype=np.uint8):
    return t.cpu().numpy().view(dtype)


def rnd(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, size=shape, dtype=np.uint8)


def mark_launch(e):
    """a one-unit CRC launch first, so that last_launch() afterwards shows the launch of the call under test and nothing older"""
    if "blk" not in _scratch:
        _scratch["blk"] = torch.zeros(BLOCK, dtype=torch.uint8, device="cuda")
        _scratch["crc"] = torch.zeros(1, dtype=torch.int32, device="cuda")
    e.crc_blocks_dev(ptr(_scratch["blk"]), 1, ptr(_scratch["crc"]))
    assert e.last_launch() == (1, 1)


def assert_walks(e, cap):
    """the launch that just ran had `cap` CTAs (fewer only with fewer units), each of them over two units or more"""
    grid, units = e.last_launch()
    assert grid == min(cap, units) and units >= 2 * grid + 1, (cap, grid, units)
    return units


def goal_tuple(goal):
    return (goal.kind, goal.k, goal.m)


# ---- inputs and the oracle's answers, computed once per shape -----------------------------------------------------------------

def encoded(oracle, text, nb, n, stride_blocks, seed):
    """data [n, stride] (nb meaningful blocks per chunk) with the oracle's parity [n, m, pb*B] and CRCs [n, nb + m*pb]"""
    key = ("enc", text, nb, n, stride_blocks, seed)
    if key not in _cache:
        goal = L.SliceType(text)
        data = rnd((n, stride_blocks * BLOCK), seed)
        ref = [oracle.encode_chunk(goal.kind, goal.k, goal.m, data[c, : nb * BLOCK]) for c in range(n)]
        _cache[key] = (data, np.stack([r[0] for r in ref]), np.stack([r[1] for r in ref]))
    return _cache[key]


def sliced(oracle, text, nb, n, seed):
    """chunks [n, nb*B], their k + m parts [n, pb*B] (data parts zero-padded) and each part's stored CRCs [n, pb]"""
    key = ("parts", text, nb, n, seed)
    if key not in _cache:
        goal = L.SliceType(text)
        k, m = goal.k, goal.m
        data, parity, crc = encoded(oracle, text, nb, n, nb, seed)
        pb = -(-nb // k)
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
    # goal, blocks per chunk, chunks, chunk stride in blocks, switches, the encoder instantiation (lzgpu_debug_encoder_kernels index;
    # the last pass for m > 4) — ragged shapes (nb % k != 0) where the unit mode allows them
    ("ec(8,2)", 61, 14, 61, dict(LZGPU_STRIPED=0), 25),         # per-chunk units, folded (k, G) = (8, 7): two units per chunk, one of them ragged
    ("ec(8,2)", 61, 14, 61, dict(LZGPU_STRIPED=1), 43),         # striped units, folded
    ("ec(8,2)", 61, 14, 64, {}, 43),                            # automatic (striped: per-chunk units would waste slots), padded stride
    ("ec(8,2)", 16, 56, 16, {}, 25),                            # flat units across chunk boundaries
    ("xor2", 65, 8, 65, dict(LZGPU_STRIPED=0), 26),             # folded (2, 32)
    ("xor3", 62, 8, 62, dict(LZGPU_STRIPED=0), 27),             # folded (3, 20)
    ("ec(3,2)", 50, 8, 50, dict(LZGPU_STRIPED=0), 28),          # folded (3, 16)
    ("ec(3,2)", 50, N, 50, dict(LZGPU_STRIPED=1), 46),          # striped, folded
    ("ec(5,3)", 43, 8, 43, dict(LZGPU_STRIPED=0), 31),          # folded (5, 8), packed-byte three rows
    ("ec(5,3)", 43, 16, 43, dict(LZGPU_STRIPED=1), 47),         # striped, folded
    ("ec(8,4)", 67, 8, 67, dict(LZGPU_STRIPED=0, LZGPU_BITSLICE=0), 33),  # folded (8, 8) on the packed-byte route
    ("ec(7,2)", 31, N, 31, dict(LZGPU_STRIPED=0), 2),           # runtime k
    ("ec(11,3)", 40, N, 40, dict(LZGPU_STRIPED=0, LZGPU_BITSLICE=0), 3),  # runtime k, packed-byte three rows
    ("ec(8,3)", 37, N, 37, dict(LZGPU_STRIPED=0), 58),          # bit-sliced, three rows, folded
    ("ec(11,3)", 40, N, 40, dict(LZGPU_STRIPED=0), 49),         # bit-sliced, three rows, runtime k
    ("ec(8,3)", 37, 2 * N, 37, dict(LZGPU_STRIPED=1), 51),      # bit-sliced striped, three rows
    ("ec(8,4)", 67, 8, 67, dict(LZGPU_STRIPED=0), 53),          # bit-sliced, four rows, folded
    ("ec(7,4)", 30, N, 30, dict(LZGPU_STRIPED=0), 50),          # bit-sliced, four rows, runtime k
    ("ec(8,4)", 67, N, 67, dict(LZGPU_STRIPED=1), 62),          # bit-sliced striped instantiation, folded (8, 8)
    ("ec(21,4)", 50, 8, 50, dict(LZGPU_STRIPED=0), 12),         # Cauchy rows on the generic-coefficient kernel
    ("ec(21,4)", 50, N, 50, {}, 24),                            # the same, automatic unit mode
    ("ec(8,6)", 37, N, 37, {}, 7),                              # m > 4: two passes (four rows, then two)
    ("ec(31,3)", 70, 8, 70, dict(LZGPU_BITSLICE=0), 10),        # Vandermonde rows that fit only the generic-coefficient CTA
]


def _id(case):
    env = ",".join(f"{k[6:]}={v}" for k, v in sorted(case[4].items()))
    return "-".join(str(x) for x in case[:4]) + (f"-{env}" if env else "")


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("case", ENCODE, ids=[_id(c) for c in ENCODE])
def test_encode_with_several_units_per_cta(oracle, case, cap):
    text, nb, n, stride, env, kernel = case
    goal = L.SliceType(text)
    m, pb = goal.m, -(-nb // goal.k)
    n_crc = nb + m * pb
    data, p_ref, c_ref = encoded(oracle, text, nb, n, stride, 7000 + nb + n)
    e = engine(cap, **env)
    d_data = dev(data)
    d_par = torch.full((n, m * pb * BLOCK), 0xA5, dtype=torch.uint8, device="cuda")
    d_crc = torch.full((n, n_crc), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    mark_launch(e)
    e.encode_chunks_dev(goal, n, nb * BLOCK, ptr(d_data), stride * BLOCK, ptr(d_par), m * pb * BLOCK, ptr(d_crc), n_crc)
    assert_walks(e, cap)
    assert e.last_encoder()[0] == kernel, (e.last_encoder(), L.encoder_kernels()[kernel])
    e.sync()
    parity = host(d_par).reshape(n, m, pb * BLOCK)
    crc = host(d_crc, np.uint32)
    for c in range(n):
        assert (parity[c] == p_ref[c]).all(), (c, [r for r in range(m) if (parity[c, r] != p_ref[c, r]).any()])
        assert (crc[c] == c_ref[c]).all(), (c, np.flatnonzero(crc[c] != c_ref[c])[:8])


# ---- CRC-only passes -----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cap", CAPS)
def test_crc_blocks_with_several_units_per_cta(oracle, cap):
    """lzgpu_crc_blocks_dev: one run of blocks, 64 blocks per unit (the last unit ragged)"""
    n = 64 * 15 + 17
    data = rnd((n, BLOCK), 31337)
    ref = np.array([zlib.crc32(data[b].tobytes()) for b in range(n)], dtype=np.uint32)
    assert all(oracle.crc32(0, data[b]) == ref[b] for b in (0, 64, n - 1))
    e = engine(cap)
    d_data = dev(data)
    d_out = torch.zeros(n, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    mark_launch(e)
    e.crc_blocks_dev(ptr(d_data), n, ptr(d_out))
    assert_walks(e, cap)
    e.sync()
    got = host(d_out, np.uint32)
    assert (got == ref).all(), np.flatnonzero(got != ref)[:8]


@pytest.mark.parametrize("cap", CAPS)
def test_generic_recover_verifies_parts_with_several_units_per_cta(oracle, cap):
    """a lost parity part is rebuilt by the generic kernels, which verify every part they read with the fused CRC kernel in its
    flat single-block-stripe form (parts of 15 blocks, contiguous: K = 1, 64 blocks per unit across part boundaries); a clean
    batch must pass and two corrupt blocks must be reported at the smaller (chunk, part, block)"""
    text, nb, n = "ec(2,1)", 30, 64
    goal = L.SliceType(text)
    data, parts, crcs = sliced(oracle, text, nb, n, 404)
    pb = parts[0].shape[1] // BLOCK
    e = engine(cap)
    d_parts = [dev(parts[0]), dev(parts[1]), None]
    d_crcs = [dev(crcs[0].view(np.int32)), dev(crcs[1].view(np.int32)), None]
    out = torch.zeros((n, pb * BLOCK), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    mark_launch(e)
    e.recover_chunks_dev(goal, n, nb, [ptr(t) for t in d_parts], pb * BLOCK, [ptr(t) for t in d_crcs], [0, 0, 1], [0, 0, ptr(out)])
    units = assert_walks(e, cap)
    assert units == math.ceil(n * pb / 64)
    e.sync()
    assert (host(out).reshape(n, -1) == parts[2]).all()
    bad = [parts[0].copy(), parts[1].copy()]
    bad[0][50, 9 * BLOCK + 3] ^= 0x01
    bad[1][40, 3 * BLOCK + 77] ^= 0x80
    d_bad = [dev(bad[0]), dev(bad[1]), None]
    torch.cuda.synchronize()
    with pytest.raises(L.ChunkCrcError) as ei:
        e.recover_chunks_dev(goal, n, nb, [ptr(t) for t in d_bad], pb * BLOCK, [ptr(t) for t in d_crcs], [0, 0, 1], [0, 0, ptr(out)])
    assert ei.value.where == (40, 1, 3)


# ---- degraded read -------------------------------------------------------------------------------------------------------------

RECOVER = [
    # goal, missing parts (data parts first; a missing parity part moves the rows in use), blocks per chunk
    ("ec(8,2)", (1,), 77),          # one lost, parity row 0: the k = 8 instantiation
    ("ec(8,2)", (1, 4), 77),        # two lost, rows 0, 1: the k = 8 instantiation
    ("ec(8,2)", (1, 8), 61),        # one lost, row 1 alone
    ("ec(3,2)", (1,), 14),          # k = 3 instantiations on the 16-warp geometry (runtime k with LZGPU_RECOVER_K3=0 or the other geometries)
    ("ec(3,2)", (0, 2), 17),
    ("ec(3,2)", (1, 3), 16),        # row 1 alone
    ("ec(4,2)", (0, 3), 19),        # k = 4
    ("ec(5,3)", (0, 3), 23),        # k = 5, two lost
    ("ec(5,3)", (0, 2, 4), 24),     # k = 5, three lost, rows 0, 1, 2
    ("ec(5,3)", (1, 2, 5), 22),     # two lost, rows 1, 2
    ("ec(6,3)", (1, 4), 29),        # k = 6
    ("ec(6,3)", (0, 2, 5), 27),
    ("ec(6,4)", (0, 1, 2, 6), 26),  # three lost, rows 1, 2, 3
    ("ec(6,4)", (0, 2, 3, 5), 25),  # four lost
    ("ec(7,2)", (2,), 27),          # runtime k
]
GEOMETRIES = [dict(LZGPU_RECOVER_GEO=0), dict(LZGPU_RECOVER_GEO=1), dict(LZGPU_RECOVER_GEO=2),
              dict(LZGPU_RECOVER_GEO=2, LZGPU_RECOVER_K3=0)]


def run_recover(e, cap, goal, nb, n, data, parts, crcs, missing, verify, image):
    k, m = goal.k, goal.m
    pb = parts[0].shape[1] // BLOCK
    lost = [i for i in missing if i < k]
    d_parts = [None if i in missing else dev(parts[i]) for i in range(k + m)]
    d_crcs = [None if i in missing else dev(crcs[i].view(np.int32)) for i in range(k + m)] if verify else None
    outs = [torch.zeros((n, pb * BLOCK), dtype=torch.uint8, device="cuda") if i in lost else None for i in range(k + m)]
    img = torch.full((n, nb * BLOCK), 0xA5, dtype=torch.uint8, device="cuda") if image else None
    torch.cuda.synchronize()
    mark_launch(e)
    e.recover_chunks_dev(goal, n, nb, [ptr(t) for t in d_parts], pb * BLOCK, None if d_crcs is None else [ptr(t) for t in d_crcs],
                         [1 if i in lost else 0 for i in range(k + m)], [ptr(t) for t in outs], ptr(img), nb * BLOCK if image else None)
    assert_walks(e, cap)
    e.sync()
    for i in lost:
        got = host(outs[i]).reshape(n, -1)
        assert (got == parts[i]).all(), (i, verify, image, [c for c in range(n) if (got[c] != parts[i][c]).any()])
    if image:
        got = host(img).reshape(n, -1)
        assert (got == data).all(), (verify, [c for c in range(n) if (got[c] != data[c]).any()])


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("geo", GEOMETRIES, ids=["geo0", "geo1", "geo2", "geo2-k3off"])
@pytest.mark.parametrize("text,missing,nb", RECOVER)
def test_recover_with_several_units_per_cta(oracle, text, missing, nb, geo, cap):
    """fused_recover_kernel (three lost data parts on it too: LZGPU_BS_RECOVER=0), with and without verification and chunk image"""
    goal = L.SliceType(text)
    data, parts, crcs = sliced(oracle, text, nb, N, 9000 + nb)
    e = engine(cap, LZGPU_BS_RECOVER=0, **geo)
    for verify in (True, False):
        for image in (True, False):
            run_recover(e, cap, goal, nb, N, data, parts, crcs, missing, verify, image)


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("wide", [0, 1])
@pytest.mark.parametrize("text,missing,nb", [
    ("ec(8,6)", (0,), 37), ("ec(8,6)", (0, 3), 37), ("ec(8,6)", (0, 3, 5), 35), ("ec(8,6)", (1, 2, 4, 7), 33),
    ("ec(8,6)", (2, 8), 37), ("ec(8,6)", (2, 6, 8, 10), 31),                 # parity rows not from 0 / not consecutive
    ("ec(21,4)", (3,), 50), ("ec(21,4)", (0, 5, 10, 20), 47), ("ec(21,4)", (4, 9, 21), 44)])
def test_recover_direct_with_several_units_per_cta(oracle, text, missing, nb, wide, cap):
    """DIRECT form (Cauchy generators: rows of the inverted k x k system), 4-byte items and wide items"""
    goal = L.SliceType(text)
    data, parts, crcs = sliced(oracle, text, nb, N, 9500 + nb)
    e = engine(cap, LZGPU_DIRECT_WIDE=wide)
    for verify in (True, False):
        for image in (True, False):
            run_recover(e, cap, goal, nb, N, data, parts, crcs, missing, verify, image)


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("text,missing,nb", [("ec(8,3)", (1, 4, 6), 37), ("ec(8,3)", (0, 1, 7), 40), ("ec(6,3)", (0, 2, 5), 29),
                                              ("ec(5,3)", (1, 2, 4), 23)])
def test_recover_three_lost_bit_sliced_with_several_units_per_cta(oracle, text, missing, nb, cap):
    """bs_recover3_kernel: its stream warps exist only when stored CRCs are given, so both ways"""
    goal = L.SliceType(text)
    data, parts, crcs = sliced(oracle, text, nb, N, 9700 + nb)
    e = engine(cap)
    for verify in (True, False):
        for image in (True, False):
            run_recover(e, cap, goal, nb, N, data, parts, crcs, missing, verify, image)


# ---- one-pass slice conversion -------------------------------------------------------------------------------------------------

CONVERT = [
    # source, lost source parts, blocks per chunk, destination
    ("xor2", (), 41, "ec(5,3)"),         # e = 0, three destination parity parts
    ("ec(8,2)", (), 50, "ec(3,2)"),      # e = 0, k_dst = 3 instantiation
    ("ec(3,2)", (1,), 40, "xor3"),       # e = 1, one destination parity part, k_dst = 3
    ("ec(3,2)", (1,), 31, "ec(5,3)"),    # e = 1, three
    ("ec(8,2)", (1, 4), 61, "ec(3,2)"),  # e = 2, k_dst = 3
    ("ec(5,3)", (0, 3), 23, "xor2"),     # e = 2, one
    ("ec(3,2)", (0, 2), 31, "ec(8,2)"),  # e = 2, two
]


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("src_name,lost,nb,dst_name", CONVERT)
def test_convert_with_several_units_per_cta(oracle, src_name, lost, nb, dst_name, cap):
    """fused_convert_kernel against the oracle's SliceRecoveryPlanner restatement and against the two-pass route"""
    src, dst = L.SliceType(src_name), L.SliceType(dst_name)
    ns, nd = src.k + src.m, dst.k + dst.m
    pbs, pbd = -(-nb // src.k), -(-nb // dst.k)
    data, parts, crcs = sliced(oracle, src_name, nb, N, 9900 + nb)
    key = ("conv", src_name, lost, nb, dst_name)
    if key not in _cache:
        ref = [O.convert_chunk(oracle, goal_tuple(src), [None if i in lost else parts[i][c] for i in range(ns)],
                               [None if i in lost else crcs[i][c] for i in range(ns)], goal_tuple(dst), [1] * nd, nb) for c in range(N)]
        assert all(r[0] == 0 for r in ref)
        _cache[key] = ([np.stack([r[1][i] for r in ref]) for i in range(nd)], [np.stack([r[2][i] for r in ref]) for i in range(nd)])
    want_out, want_crc = _cache[key]
    plan = L.Engine.plan_convert(src, dst, [0 if i in lost else 1 for i in range(ns)], [1] * nd)
    assert plan["one_pass"] == 1
    units = N * -(-nb // (plan["stripes_per_unit"] * dst.k))
    d_parts = [None if i in lost else dev(parts[i]) for i in range(ns)]
    d_crcs = [None if i in lost else dev(crcs[i].view(np.int32)) for i in range(ns)]
    e1, e2 = engine(cap), engine(cap, LZGPU_CONVERT_FUSED=0)
    for verify in (True, False):
        results = []
        for e in (e1, e2):
            outs = [torch.full((N, pbd * BLOCK), 0xA5, dtype=torch.uint8, device="cuda") for _ in range(nd)]
            ocrc = [torch.full((N, pbd), 0x5A5A5A5A, dtype=torch.int32, device="cuda") for _ in range(nd)]
            torch.cuda.synchronize()
            mark_launch(e)
            e.convert_chunks_dev(src, dst, N, nb, [ptr(t) for t in d_parts], pbs * BLOCK, [1] * nd, [ptr(t) for t in outs], pbd * BLOCK,
                                 d_part_crc=[ptr(t) for t in d_crcs] if verify else None, d_out_crc=[ptr(t) for t in ocrc])
            if e is e1:
                assert assert_walks(e, cap) == units    # the one-pass kernel (the two-pass route launches capped kernels too)
            e.sync()
            results.append(([host(t).reshape(N, -1) for t in outs], [host(t, np.uint32).reshape(N, -1) for t in ocrc]))
        for out, ocrc in results:
            for i in range(nd):
                assert (out[i] == want_out[i]).all(), (verify, i, [c for c in range(N) if (out[i][c] != want_out[i][c]).any()])
                assert (ocrc[i] == want_crc[i]).all(), (verify, i, [c for c in range(N) if (ocrc[i][c] != want_crc[i][c]).any()])


# ---- the first of several CRC mismatches ---------------------------------------------------------------------------------------
# With a cap of 2 CTAs, CTA 0 takes units 0, 2, 4, ... and CTA 1 units 1, 3, 5, ...; units are numbered chunk by chunk, stripe group
# by stripe group.  Each test corrupts three blocks of chunk 0: a larger (part, block) in unit 0, the smallest one in unit 2 (CTA 0
# reaches it after unit 0) and one in unit 1 (CTA 1).  The reported mismatch must be the smallest, and the same on the generic route.

def test_recover_reports_the_smallest_of_several_mismatches(oracle):
    text, nb, n = "ec(8,2)", 8 * 24 - 3, 4
    goal = L.SliceType(text)
    data, parts, crcs = sliced(oracle, text, nb, n, 555)
    lost = (1, 4)
    G = 8                                           # stripes per unit of the k = 8 kernel on the one-CTA geometry (checked below)
    bad = [None if i in lost else parts[i].copy() for i in range(10)]
    bad[7][0, 1 * BLOCK + 10] ^= 0x01               # unit 0
    bad[2][0, (2 * G + 1) * BLOCK + 20] ^= 0x02     # unit 2: the smallest
    bad[5][0, (G + 1) * BLOCK + 30] ^= 0x04         # unit 1
    acrc = [None if i in lost else crcs[i] for i in range(10)]
    want = [1 if i in lost else 0 for i in range(10)]
    capped = engine(2, LZGPU_RECOVER_GEO=0)
    for e in (capped, engine(None, LZGPU_DISABLE_FUSED=1)):
        if e is capped:
            mark_launch(e)
        for image in (True, False):
            with pytest.raises(L.ChunkCrcError) as ei:
                e.recover_chunks(goal, nb, bad, part_crc=acrc, want=want, chunk_image=image)
            assert ei.value.where == (0, 2, 2 * G + 1), (e is capped, image)
            if e is capped:
                assert e.last_launch() == (2, n * 3)


def test_convert_reports_the_smallest_of_several_mismatches(oracle):
    src_name, dst_name, lost = "ec(8,2)", "ec(3,2)", (1, 4)
    src, dst = L.SliceType(src_name), L.SliceType(dst_name)
    avail = [0 if i in lost else 1 for i in range(10)]
    plan = L.Engine.plan_convert(src, dst, avail, [1] * 5)
    assert plan["one_pass"] == 1
    R, T = plan["stripes_per_unit"] * dst.k, plan["source_stripes_per_unit"]   # chunk blocks / source stripes per unit
    nb, n = 3 * R - 1, 3
    pbs = -(-nb // src.k)
    assert 2 * T < pbs
    data, parts, crcs = sliced(oracle, src_name, nb, n, 556)
    bad = [None if i in lost else parts[i].copy() for i in range(10)]
    bad[7][0, 0 * BLOCK + 11] ^= 0x01               # unit 0
    bad[2][0, (2 * T) * BLOCK + 21] ^= 0x02         # unit 2: the smallest
    bad[5][0, T * BLOCK + 31] ^= 0x04               # unit 1
    acrc = [None if i in lost else crcs[i] for i in range(10)]
    capped = engine(2)
    for e in (capped, engine(None, LZGPU_DISABLE_FUSED=1)):
        if e is capped:
            mark_launch(e)
        with pytest.raises(L.ChunkCrcError) as ei:
            e.convert_chunks(src, dst, nb, bad, [1] * 5, part_crc=acrc)
        assert ei.value.where == (0, 2, 2 * T), e is capped
        if e is capped:
            assert e.last_launch() == (2, n * 3)


def test_verify_blocks_reports_the_smallest_of_several_mismatches():
    """lzgpu_verify_blocks: 64 blocks per unit of the CRC kernel, corrupt blocks in units 1 (CTA 1), 2 and 4 (CTA 0)"""
    n = 64 * 5
    data = rnd((n, BLOCK), 557)
    stored = np.array([zlib.crc32(data[b].tobytes()) for b in range(n)], dtype=np.uint32)
    bad = data.copy()
    for b in (64 + 7, 128 + 3, 256 + 1):
        bad[b, 100] ^= 0x10
    capped = engine(2)
    for e in (capped, engine(None, LZGPU_DISABLE_FUSED=1)):
        e.verify_blocks(data, stored)
        with pytest.raises(L.ChunkCrcError) as ei:
            e.verify_blocks(bad, stored)
        assert ei.value.where == (64 + 7,), e is capped
        if e is capped:
            assert e.last_launch() == (2, 5)


# ---- the default grid ----------------------------------------------------------------------------------------------------------

def test_uncapped_grid_with_several_units_per_cta(oracle):
    """no cap: a resident ec(8,2) batch of full 64 MiB chunks large enough that the default grid (two CTAs per SM for the encode,
    one for the degraded read) still has more than two units per CTA; every chunk against the oracle and the original data"""
    goal = L.SliceType("ec(8,2)")
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    nb, pb = 1024, 128
    n = math.ceil((4 * sm + 1) * 7 / 128)           # flat units of 7 stripes: more than 2 x (2 x sm) of them
    e = engine(None)
    d_data = torch.empty((n, nb * BLOCK), dtype=torch.uint8, device="cuda")
    chunks = [rnd(nb * BLOCK, 60000 + c) for c in range(n)]
    for c in range(n):
        d_data[c] = dev(chunks[c])
    d_par = torch.zeros((n, 2 * pb * BLOCK), dtype=torch.uint8, device="cuda")
    d_crc = torch.zeros((n, nb + 2 * pb), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    mark_launch(e)
    e.encode_chunks_dev(goal, n, nb * BLOCK, ptr(d_data), nb * BLOCK, ptr(d_par), 2 * pb * BLOCK, ptr(d_crc), nb + 2 * pb)
    grid, units = e.last_launch()
    assert grid == min(units, 2 * sm) and units > 2 * grid, (grid, units, sm)
    e.sync()
    part_crcs = []
    for c in range(n):
        p_ref, c_ref = oracle.encode_chunk(goal.kind, 8, 2, chunks[c])
        assert (host(d_par[c]).reshape(2, -1) == p_ref).all(), c
        assert (host(d_crc[c], np.uint32) == c_ref).all(), c
        part_crcs.append(c_ref)
    # degraded read of the same batch: data parts 1 and 4 lost, verified, with the chunk image
    lost = (1, 4)
    d_parts = []
    for j in range(8):
        d_parts.append(None if j in lost else d_data.view(n, pb, 8, BLOCK)[:, :, j].contiguous())
    d_parts += [d_par[:, r * pb * BLOCK:(r + 1) * pb * BLOCK].contiguous() for r in range(2)]
    crc_np = np.stack(part_crcs)
    d_pcrc = [None if j in lost else dev(np.ascontiguousarray(crc_np[:, j:nb:8]).view(np.int32)) for j in range(8)]
    d_pcrc += [dev(np.ascontiguousarray(crc_np[:, nb + r * pb: nb + (r + 1) * pb]).view(np.int32)) for r in range(2)]
    outs = [torch.zeros((n, pb * BLOCK), dtype=torch.uint8, device="cuda") if j in lost else None for j in range(10)]
    img = torch.zeros((n, nb * BLOCK), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    mark_launch(e)
    e.recover_chunks_dev(goal, n, nb, [ptr(t) for t in d_parts], pb * BLOCK, [ptr(t) for t in d_pcrc], [1 if j in lost else 0 for j in range(10)],
                         [ptr(t) for t in outs], ptr(img), nb * BLOCK)
    grid, units = e.last_launch()
    assert grid == min(units, sm) and units > 2 * grid, (grid, units, sm)
    e.sync()
    for c in range(n):
        blocks = chunks[c].reshape(pb, 8, BLOCK)
        for j in lost:
            assert (host(outs[j][c]).reshape(pb, BLOCK) == blocks[:, j]).all(), (c, j)
        assert (host(img[c]) == chunks[c]).all(), c
