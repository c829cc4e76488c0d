"""The bit-sliced kernels at every geometry their tuning switches select.

The CTA shapes, stage depths and GF-warp counts of the bit-sliced encoder (fused_stream_kernel with W = 8) and of
bs_recover3_kernel are runtime parameters, and the switches LZGPU_BS_GFW, LZGPU_BS_STAGES, LZGPU_BS_SMEM_KB and
LZGPU_BS_RECOVER_GFW move them far from the defaults the rest of the suite runs:
- stage rings of 5 to 11 stages, which meet the unit boundary (128 steps) in the middle of the ring, so the cross-unit refill
  and the stage / phase counters run out of step with the units;
- 9 or 10 stripes per unit on the encoder (5 GF warps), 1 or 2 at a small shared-memory budget, and 18 to 32 stripes with 9 to 16
  GF warps on bs_recover3_kernel;
- 230 136 bytes of dynamic shared memory (ec(4,4), 11 stages), next to the 227 KiB a CTA can have;
- no bit-sliced plan at all (ec(32,3) at 64 KiB), where the packed-word kernel takes the call.
LZGPU_EVICT_FIRST and LZGPU_L2_PROMO change the TMA loads and the tensor maps but no geometry.

Every case runs with LZGPU_GRID_CAP 1 and 3, so that each CTA walks several units, and asserts the whole geometry of the launch
(lzgpu_debug_last_geometry) against the table below, worked out from the host planner (fused_plan.h, the bs_recover3 G loop in
fused.cu): a switch that is ignored, or a planner change that no longer reaches the geometry, fails instead of running the default
twice.  Every parity byte and CRC is compared with the oracle (tests/_oracle.py), every rebuilt part and image with the original
data.  Shapes are ragged: nb % k != 0 and pb % G != 0 wherever G > 1."""
import os

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import _oracle as O

pytestmark = pytest.mark.gpu
BLOCK = 65536
CAPS = (1, 3)
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
    """a one-unit CRC launch first, so that the geometry read afterwards is that of the call under test and nothing older"""
    if "blk" not in _scratch:
        _scratch["blk"] = torch.zeros(BLOCK, dtype=torch.uint8, device="cuda")
        _scratch["crc"] = torch.zeros(1, dtype=torch.int32, device="cuda")
    e.crc_blocks_dev(ptr(_scratch["blk"]), 1, ptr(_scratch["crc"]))
    assert e.last_launch() == (1, 1)


def assert_geometry(e, cap, want):
    """the launch that just ran had the geometry `want` (kernel, threads, G, stages, gf_warps, smem_bytes, units) and `cap` CTAs,
    each of them over two units or more; returns the geometry"""
    g = e.last_geometry()
    assert (g["grid"], g["units"]) == e.last_launch()
    got = {k: g[k] for k in want}
    assert got == want, (got, want)
    assert g["grid"] == min(cap, g["units"]) and g["units"] >= 2 * g["grid"] + 1, (cap, g)
    return g


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


def units_of(mode, n, pb, G):
    """work units of an encode: G stripes of one chunk ("chunk"), or G stripes of the batch's run of stripes ("striped", "flat")"""
    return n * -(-pb // G) if mode == "chunk" else -(-(n * pb) // G)


def run_encode(oracle, e, cap, text, nb, n, stride, want=None, seed=0):
    """encode_chunks_dev of n chunks (stride blocks apart) on `e`; parity and CRCs against the oracle; returns (geometry, parity, CRCs)"""
    goal = L.SliceType(text)
    m, pb = goal.m, -(-nb // goal.k)
    n_crc = nb + m * pb
    data, p_ref, c_ref = encoded(oracle, text, nb, n, stride, 11000 + 7 * nb + n + seed)
    d_data = dev(data)
    d_par = torch.full((n, m * pb * BLOCK), 0xA5, dtype=torch.uint8, device="cuda")
    d_crc = torch.full((n, n_crc), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    mark_launch(e)
    e.encode_chunks_dev(goal, n, nb * BLOCK, ptr(d_data), stride * BLOCK, ptr(d_par), m * pb * BLOCK, ptr(d_crc), n_crc)
    g = assert_geometry(e, cap, want) if want is not None else e.last_geometry()
    e.sync()
    parity = host(d_par).reshape(n, m, pb * BLOCK)
    crc = host(d_crc, np.uint32)
    for c in range(n):
        assert (parity[c] == p_ref[c]).all(), (c, [r for r in range(m) if (parity[c, r] != p_ref[c, r]).any()])
        assert (crc[c] == c_ref[c]).all(), (c, np.flatnonzero(crc[c] != c_ref[c])[:8])
    return g, parity, crc


# ---- bit-sliced encoder ----------------------------------------------------------------------------------------------------------

BS = _lib.KERNEL_ENCODE_BITSLICE
ENCODE = [
    # goal, blocks per chunk, chunks, unit mode ("chunk": LZGPU_STRIPED=0, "striped": LZGPU_STRIPED=1, "flat": contiguous whole
    # stripes), switches, then the expected geometry: kernel, threads, G, stages, GF warps, shared memory bytes
    # LZGPU_BS_GFW: more or fewer GF warps, so more or fewer stripes per unit (default: four GF warps, G = 8)
    ("ec(4,4)", 41, 4, "chunk", dict(LZGPU_BS_GFW=1), (BS, 512, 2, 4, 1, 29320)),        # off the folded (4, 4, 8)
    ("ec(4,4)", 41, 4, "chunk", dict(LZGPU_BS_GFW=2), (BS, 512, 4, 4, 2, 57992)),
    ("ec(4,4)", 41, 4, "chunk", dict(LZGPU_BS_GFW=3), (BS, 512, 6, 4, 3, 86664)),
    ("ec(4,4)", 41, 4, "chunk", dict(LZGPU_BS_GFW=5), (BS, 512, 10, 4, 5, 144008)),      # G = 10: items 128..159 on a fifth GF warp
    ("ec(6,4)", 61, 4, "chunk", dict(LZGPU_BS_GFW=5), (BS, 512, 9, 4, 5, 168584)),       # G = 9: the fifth GF warp half empty
    ("ec(5,3)", 61, 4, "chunk", dict(LZGPU_BS_GFW=5, LZGPU_BITSLICE=7), (BS, 512, 10, 4, 5, 144008)),
    ("ec(10,4)", 53, 4, "chunk", dict(LZGPU_BS_GFW=2), (BS, 512, 4, 4, 2, 107144)),      # off the folded (4, 10, 6)
    ("ec(8,4)", 67, 4, "chunk", dict(LZGPU_BS_GFW=3), (BS, 512, 6, 4, 3, 135816)),       # off the folded (4, 8, 8)
    ("ec(8,3)", 67, 4, "chunk", dict(LZGPU_BS_GFW=3), (BS, 512, 6, 4, 3, 123528)),       # off the folded (3, 8, 8)
    # LZGPU_BS_STAGES: rings whose depth does not divide the 128 steps of a unit (below 4 has no effect: the ring has at least 4)
    ("ec(4,4)", 41, 4, "chunk", dict(LZGPU_BS_STAGES=2), (BS, 512, 8, 4, 4, 115336)),
    ("ec(4,4)", 41, 4, "chunk", dict(LZGPU_BS_STAGES=5), (BS, 512, 8, 5, 4, 131736)),
    ("ec(4,4)", 41, 4, "chunk", dict(LZGPU_BS_STAGES=7), (BS, 512, 8, 7, 4, 164536)),
    ("ec(4,4)", 41, 4, "chunk", dict(LZGPU_BS_STAGES=16), (BS, 512, 8, 9, 4, 197336)),  # as many as fit 200 KiB
    ("ec(11,3)", 60, 4, "chunk", dict(LZGPU_BS_STAGES=7), (BS, 512, 4, 7, 2, 174776)),  # runtime k, three rows
    ("ec(11,3)", 60, 4, "chunk", dict(LZGPU_BS_STAGES=16), (BS, 512, 4, 8, 2, 197320)),
    ("ec(5,3)", 61, 4, "chunk", dict(LZGPU_BS_STAGES=16, LZGPU_BITSLICE=7), (BS, 512, 8, 8, 4, 197320)),
    # the folded instantiations (the bit-sliced entries of kEncoders, csrc/fused.cu) with deeper rings
    ("ec(12,4)", 70, 4, "chunk", dict(LZGPU_BS_STAGES=16), (BS, 512, 5, 5, 3, 187032)),
    ("ec(10,4)", 71, 4, "chunk", dict(LZGPU_BS_STAGES=16), (BS, 512, 6, 5, 3, 191128)),
    ("ec(6,4)", 61, 4, "chunk", dict(LZGPU_BS_STAGES=16), (BS, 512, 8, 6, 4, 197288)),
    ("ec(8,3)", 67, 4, "chunk", dict(LZGPU_BS_STAGES=16), (BS, 512, 8, 5, 4, 197272)),
    ("ec(9,3)", 64, 4, "chunk", dict(LZGPU_BS_STAGES=7), (BS, 512, 6, 6, 3, 191144)),
    ("ec(10,3)", 71, 4, "chunk", dict(LZGPU_BS_STAGES=16), (BS, 512, 6, 5, 3, 178840)),
    ("ec(12,3)", 70, 4, "chunk", dict(LZGPU_BS_STAGES=16), (BS, 512, 5, 5, 3, 174744)),
    # LZGPU_BS_SMEM_KB (with LZGPU_BS_STAGES=16): G and depth from the budget
    ("ec(16,4)", 37, 4, "chunk", dict(LZGPU_BS_SMEM_KB=64, LZGPU_BS_STAGES=16), (BS, 512, 1, 6, 1, 58024)),
    ("ec(7,3)", 33, 4, "chunk", dict(LZGPU_BS_SMEM_KB=64, LZGPU_BS_STAGES=16), (BS, 512, 2, 7, 1, 59064)),
    ("ec(8,4)", 67, 4, "chunk", dict(LZGPU_BS_SMEM_KB=96, LZGPU_BS_STAGES=16), (BS, 512, 4, 4, 2, 90760)),
    ("ec(4,4)", 41, 4, "chunk", dict(LZGPU_BS_SMEM_KB=226, LZGPU_BS_STAGES=16), (BS, 512, 8, 11, 4, 230136)),  # near the 227 KiB limit
    # no bit-sliced plan fits 64 KiB: the packed-word kernel (8 warps, two CTAs per SM, 3 stages)
    ("ec(32,3)", 37, 4, "chunk", dict(LZGPU_BS_SMEM_KB=64, LZGPU_BS_STAGES=16), (_lib.KERNEL_ENCODE, 256, 1, 3, 0, 53880)),
    # striped units (one TMA box per stripe, refilled by a whole warp): the folded striped (4, 8, 8) and the runtime-k forms
    ("ec(8,4)", 67, 8, "striped", dict(LZGPU_BS_SMEM_KB=226, LZGPU_BS_STAGES=16), (BS, 512, 8, 5, 4, 213656)),
    ("ec(4,4)", 41, 8, "striped", dict(LZGPU_BS_GFW=5, LZGPU_BS_STAGES=7), (BS, 512, 10, 6, 5, 185000)),
    ("ec(11,3)", 60, 8, "striped", dict(LZGPU_BS_STAGES=16), (BS, 512, 4, 8, 2, 197320)),
    # flat units: contiguous chunks of whole stripes (nb % k == 0), units across chunk boundaries
    ("ec(4,4)", 40, 5, "flat", dict(LZGPU_BS_STAGES=7), (BS, 512, 8, 7, 4, 164536)),
]


def _id(case):
    env = ",".join(f"{k[6:]}={v}" for k, v in sorted(case[4].items()))
    return f"{case[0]}-{case[1]}x{case[2]}-{case[3]}-{env}"


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("case", ENCODE, ids=[_id(c) for c in ENCODE])
def test_bit_sliced_encode_at_switched_geometry(oracle, case, cap):
    text, nb, n, mode, env, (kernel, threads, G, stages, gf_warps, smem) = case
    goal = L.SliceType(text)
    pb = -(-nb // goal.k)
    assert mode == "flat" or (nb % goal.k and (G == 1 or pb % G)), "ragged shapes"
    e = engine(cap, LZGPU_STRIPED=1 if mode == "striped" else 0, **env)
    want = dict(kernel=kernel, threads=threads, G=G, stages=stages, gf_warps=gf_warps, smem_bytes=smem, units=units_of(mode, n, pb, G))
    run_encode(oracle, e, cap, text, nb, n, nb, want)


# ---- bs_recover3_kernel ----------------------------------------------------------------------------------------------------------

RECOVER_GOALS = [
    # goal, lost data parts, blocks per chunk (37 stripes: pb % G != 0 for every even G)
    ("ec(3,3)", (0, 1, 2), 109),
    ("ec(4,4)", (0, 1, 3), 145),      # parity row 3 is not among the first k available parts
    ("ec(5,3)", (0, 2, 4), 181),      # the KT = 5 instance
    ("ec(6,3)", (1, 2, 5), 217),      # runtime k
    ("ec(8,3)", (4, 5, 7), 289),      # the KT = 8 instance; first lost part past 3: A S0, A^2 S0 as masked products
]
RECOVER_GFW = (1, 3, 9, 12, 16)
# (k, LZGPU_BS_RECOVER_GFW, stored CRCs given) -> (G, stages, GF warps, shared memory bytes).  With stored CRCs the k G 4 input rows
# need stream warps too: at most 16 warps in all.
BS3_GEOMETRY = {
    (3, 1, False): (2, 6, 1, 18592), (3, 1, True): (2, 6, 1, 18592),
    (3, 3, False): (6, 6, 3, 55456), (3, 3, True): (6, 6, 3, 55456),
    (3, 9, False): (18, 6, 9, 166048), (3, 9, True): (18, 6, 9, 166048),
    (3, 12, False): (24, 5, 12, 184464), (3, 12, True): (18, 6, 9, 166048),
    (3, 16, False): (32, 4, 16, 196736), (3, 16, True): (18, 6, 9, 166048),
    (4, 1, False): (2, 6, 1, 24736), (4, 1, True): (2, 6, 1, 24736),
    (4, 3, False): (6, 6, 3, 73888), (4, 3, True): (6, 6, 3, 73888),
    (4, 9, False): (18, 5, 9, 184464), (4, 9, True): (16, 6, 8, 196768),
    (4, 12, False): (24, 4, 12, 196736), (4, 12, True): (16, 6, 8, 196768),
    (4, 16, False): (32, 3, 16, 196720), (4, 16, True): (16, 6, 8, 196768),
    (5, 1, False): (2, 6, 1, 30880), (5, 1, True): (2, 6, 1, 30880),
    (5, 3, False): (6, 6, 3, 92320), (5, 3, True): (6, 6, 3, 92320),
    (5, 9, False): (18, 4, 9, 184448), (5, 9, True): (14, 5, 7, 179344),
    (5, 12, False): (24, 3, 12, 184432), (5, 12, True): (14, 5, 7, 179344),
    (5, 16, False): (26, 3, 13, 199792), (5, 16, True): (14, 5, 7, 179344),
    (6, 1, False): (2, 6, 1, 37024), (6, 1, True): (2, 6, 1, 37024),
    (6, 3, False): (6, 6, 3, 110752), (6, 3, True): (6, 6, 3, 110752),
    (6, 9, False): (18, 3, 9, 166000), (6, 9, True): (12, 5, 6, 184464),
    (6, 12, False): (22, 3, 11, 202864), (6, 12, True): (12, 5, 6, 184464),
    (6, 16, False): (22, 3, 11, 202864), (6, 16, True): (12, 5, 6, 184464),
    (8, 1, False): (2, 6, 1, 49312), (8, 1, True): (2, 6, 1, 49312),
    (8, 3, False): (6, 6, 3, 147616), (8, 3, True): (6, 6, 3, 147616),
    (8, 9, False): (16, 3, 8, 196720), (8, 9, True): (8, 6, 4, 196768),
    (8, 12, False): (16, 3, 8, 196720), (8, 12, True): (8, 6, 4, 196768),
    (8, 16, False): (16, 3, 8, 196720), (8, 16, True): (8, 6, 4, 196768),
}
N_RECOVER = 4


def run_recover(e, cap, goal, nb, n, data, parts, crcs, missing, verify, image, want=None):
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
    g = assert_geometry(e, cap, want) if want is not None else e.last_geometry()
    e.sync()
    got = {}
    for i in lost:
        got[i] = host(outs[i]).reshape(n, -1)
        assert (got[i] == parts[i]).all(), (i, verify, image, [c for c in range(n) if (got[i][c] != parts[i][c]).any()])
    if image:
        got["image"] = host(img).reshape(n, -1)
        assert (got["image"] == data).all(), (verify, [c for c in range(n) if (got["image"][c] != data[c]).any()])
    return g, got


@pytest.mark.parametrize("cap", CAPS, ids=[f"cap{c}" for c in CAPS])
@pytest.mark.parametrize("gfw", RECOVER_GFW, ids=[f"gfw{g}" for g in RECOVER_GFW])
@pytest.mark.parametrize("text,missing,nb", RECOVER_GOALS, ids=[f"{t}-lost{','.join(map(str, x))}" for t, x, _ in RECOVER_GOALS])
def test_bs_recover3_at_switched_geometry(oracle, text, missing, nb, gfw, cap):
    """three lost data parts (parity rows 0, 1, 2 in use) with and without stored CRCs, with and without the chunk image"""
    goal = L.SliceType(text)
    pb = -(-nb // goal.k)
    assert nb % goal.k and pb == 37
    data, parts, crcs = sliced(oracle, text, nb, N_RECOVER, 13000 + nb)
    e = engine(cap, LZGPU_BS_RECOVER_GFW=gfw)
    for verify in (True, False):
        G, stages, gf_warps, smem = BS3_GEOMETRY[(goal.k, gfw, verify)]
        want = dict(kernel=_lib.KERNEL_RECOVER_BS3, threads=512, G=G, stages=stages, gf_warps=gf_warps, smem_bytes=smem,
                    units=N_RECOVER * -(-pb // G))
        for image in (True, False):
            run_recover(e, cap, goal, nb, N_RECOVER, data, parts, crcs, missing, verify, image, want)


@pytest.mark.parametrize("cap", CAPS)
def test_bs_recover3_reports_a_corrupt_stored_crc_at_its_block(oracle, cap):
    """ec(3,3) at 18 stripes per unit (9 GF warps, 7 stream warps): one corrupt stored CRC in the second unit of chunk 2 is reported at
    its (chunk, part, block), with and without the image"""
    text, missing, nb = RECOVER_GOALS[0]
    goal = L.SliceType(text)
    data, parts, crcs = sliced(oracle, text, nb, N_RECOVER, 13000 + nb)
    bad = [c.copy() for c in crcs]
    bad[4][2, 25] ^= 0x00010000                      # part 4 (parity row 1), chunk 2, block 25
    e = engine(cap, LZGPU_BS_RECOVER_GFW=9)
    k, m = goal.k, goal.m
    pb = parts[0].shape[1] // BLOCK
    d_parts = [None if i in missing else dev(parts[i]) for i in range(k + m)]
    d_crcs = [None if i in missing else dev(bad[i].view(np.int32)) for i in range(k + m)]
    outs = [torch.zeros((N_RECOVER, pb * BLOCK), dtype=torch.uint8, device="cuda") if i in missing else None for i in range(k + m)]
    for image in (True, False):
        img = torch.zeros((N_RECOVER, nb * BLOCK), dtype=torch.uint8, device="cuda") if image else None
        torch.cuda.synchronize()
        mark_launch(e)
        with pytest.raises(L.ChunkCrcError) as ei:
            e.recover_chunks_dev(goal, N_RECOVER, nb, [ptr(t) for t in d_parts], pb * BLOCK, [ptr(t) for t in d_crcs],
                                 [1 if i in missing else 0 for i in range(k + m)], [ptr(t) for t in outs], ptr(img), nb * BLOCK if image else None)
        assert ei.value.where == (2, 4, 25), image
        assert_geometry(e, cap, dict(kernel=_lib.KERNEL_RECOVER_BS3, G=18, stages=6, gf_warps=9, units=N_RECOVER * 3))


# ---- switches that change no geometry ------------------------------------------------------------------------------------------

NEUTRAL = [dict(LZGPU_EVICT_FIRST=1), dict(LZGPU_L2_PROMO=0), dict(LZGPU_L2_PROMO=1), dict(LZGPU_L2_PROMO=2)]


def _neutral_id(env):
    return ",".join(f"{k[6:]}={v}" for k, v in env.items())


def same_geometry(g, g_default, kernel):
    assert g["kernel"] == kernel, g
    assert g == g_default, (g, g_default)


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("env", NEUTRAL, ids=[_neutral_id(x) for x in NEUTRAL])
@pytest.mark.parametrize("text,nb,n,kernel", [("ec(8,2)", 61, 4, _lib.KERNEL_ENCODE), ("ec(8,4)", 67, 4, _lib.KERNEL_ENCODE_BITSLICE)])
def test_encode_with_neutral_switches(oracle, text, nb, n, kernel, env, cap):
    """packed-word and bit-sliced encode (per-chunk units: the loads that LZGPU_EVICT_FIRST switches) against the oracle and against
    a context without the switch"""
    results = [run_encode(oracle, engine(cap, LZGPU_STRIPED=0, **x), cap, text, nb, n, nb) for x in (env, {})]
    (g, parity, crc), (g0, parity0, crc0) = results
    assert g["units"] >= 2 * g["grid"] + 1 and g["grid"] == cap, g
    same_geometry(g, g0, kernel)
    assert (parity == parity0).all() and (crc == crc0).all()


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("env", NEUTRAL, ids=[_neutral_id(x) for x in NEUTRAL])
@pytest.mark.parametrize("text,missing,nb,kernel", [("ec(8,2)", (1, 4), 77, _lib.KERNEL_RECOVER_GEO0),
                                                    ("ec(5,3)", (0, 2, 4), 181, _lib.KERNEL_RECOVER_BS3)])
def test_degraded_read_with_neutral_switches(oracle, text, missing, nb, kernel, env, cap):
    """degraded read, verified, with the chunk image, against the original data and a context without the switch"""
    goal = L.SliceType(text)
    data, parts, crcs = sliced(oracle, text, nb, N_RECOVER, 13000 + nb)
    (g, got), (g0, got0) = [run_recover(engine(cap, **x), cap, goal, nb, N_RECOVER, data, parts, crcs, missing, True, True) for x in (env, {})]
    assert g["units"] >= 2 * g["grid"] + 1 and g["grid"] == cap, g
    same_geometry(g, g0, kernel)
    assert got.keys() == got0.keys() and all((got[x] == got0[x]).all() for x in got)


@pytest.mark.parametrize("cap", CAPS)
@pytest.mark.parametrize("env", NEUTRAL, ids=[_neutral_id(x) for x in NEUTRAL])
def test_convert_with_neutral_switches(oracle, env, cap):
    """one-pass conversion ec(8,2) with data parts 1 and 4 lost -> ec(3,2), verified, against the oracle's SliceRecoveryPlanner
    restatement and a context without the switch"""
    src_name, lost, nb, dst_name, n = "ec(8,2)", (1, 4), 61, "ec(3,2)", N_RECOVER
    src, dst = L.SliceType(src_name), L.SliceType(dst_name)
    ns, nd = src.k + src.m, dst.k + dst.m
    pbs, pbd = -(-nb // src.k), -(-nb // dst.k)
    data, parts, crcs = sliced(oracle, src_name, nb, n, 13000 + nb)
    key = ("conv", src_name, lost, nb, dst_name)
    if key not in _cache:
        ref = [O.convert_chunk(oracle, (src.kind, src.k, src.m), [None if i in lost else parts[i][c] for i in range(ns)],
                               [None if i in lost else crcs[i][c] for i in range(ns)], (dst.kind, dst.k, dst.m), [1] * nd, nb) for c in range(n)]
        assert all(r[0] == 0 for r in ref)
        _cache[key] = ([np.stack([r[1][i] for r in ref]) for i in range(nd)], [np.stack([r[2][i] for r in ref]) for i in range(nd)])
    want_out, want_crc = _cache[key]
    plan = L.Engine.plan_convert(src, dst, [0 if i in lost else 1 for i in range(ns)], [1] * nd)
    assert plan["one_pass"] == 1
    d_parts = [None if i in lost else dev(parts[i]) for i in range(ns)]
    d_crcs = [None if i in lost else dev(crcs[i].view(np.int32)) for i in range(ns)]
    geos = []
    for x in (env, {}):
        e = engine(cap, **x)
        outs = [torch.full((n, pbd * BLOCK), 0xA5, dtype=torch.uint8, device="cuda") for _ in range(nd)]
        ocrc = [torch.full((n, pbd), 0x5A5A5A5A, dtype=torch.int32, device="cuda") for _ in range(nd)]
        torch.cuda.synchronize()
        mark_launch(e)
        e.convert_chunks_dev(src, dst, n, nb, [ptr(t) for t in d_parts], pbs * BLOCK, [1] * nd, [ptr(t) for t in outs], pbd * BLOCK,
                             d_part_crc=[ptr(t) for t in d_crcs], d_out_crc=[ptr(t) for t in ocrc])
        geos.append(assert_geometry(e, cap, dict(kernel=_lib.KERNEL_CONVERT, threads=256, G=plan["stripes_per_unit"], stages=plan["stages"],
                                                 gf_warps=plan["rebuild_warps"], smem_bytes=plan["smem_bytes"],
                                                 units=n * -(-nb // (plan["stripes_per_unit"] * dst.k)))))
        e.sync()
        for i in range(nd):
            got = host(outs[i]).reshape(n, -1)
            assert (got == want_out[i]).all(), (x, i, [c for c in range(n) if (got[c] != want_out[i][c]).any()])
            got = host(ocrc[i], np.uint32).reshape(n, -1)
            assert (got == want_crc[i]).all(), (x, i, [c for c in range(n) if (got[c] != want_crc[i][c]).any()])
    assert geos[0] == geos[1]
