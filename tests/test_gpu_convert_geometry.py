"""The one-pass slice conversion (fused_convert_kernel<M, E, KD>, csrc/convert_kernel.cuh) at every unit geometry its planner
(convert_plan, csrc/fused_plan.h) selects.

convert_plan() picks the unit geometry at run time: G destination stripes = T source stripes per unit, R = G * k_dst <= 64 chunk
blocks, slot regions of 4 T rows rounded up to 8, a ring of 2-4 stages, 3-8 worker warps and the rest rebuild warps; the kernel
branches on all of these, on the compile-time k_dst = 3 walk, and with two lost data parts on how 2^x0 * S0 is formed (x0
doublings for x0 <= 4, a multiply by w[0] otherwise).  CASES below holds one request per feature value the planner's space has
(test_convert_geometry_table_covers_the_planner_space enumerates that space on the CPU and fails when a table entry is missing
or its literal plan no longer matches), plus requests at the edge that must take the two-pass route.

Every case runs at a ragged block count (nb % R, nb % k_src, nb % k_dst != 0, three units per chunk) and at nb < R (one partial
unit); three also at nb = 1024 (64 MiB chunks).  Each conversion runs on three contexts: the default one, LZGPU_GRID_CAP=2 (several
units per CTA: the stage ring wraps from one unit into the next) and LZGPU_CONVERT_FUSED=0 (the two-pass route).  Outputs start
as 0xA5 bytes and 0x5A5A5A5A CRC words; every byte of every destination part and every destination CRC must equal the oracle's
restatement of SliceRecoveryPlanner (tests/_oracle.py convert_chunk) and the two-pass route's answer, unwanted parts must keep
the sentinel, and lzgpu_debug_last_geometry must show the planned geometry.  Five pairs are also pinned to the compiled
reference's SliceRecoveryPlanner (digests recorded in tests/golden/reference_digests.json by gen_golden.py)."""
import math
import os
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import _oracle as O

BLOCK = 65536
N, N_CAP = 3, 5                 # chunks per call; under the cap of 2 CTAs, 5 chunks give more than 2 x 2 units at nb < R as well
ZERO_CRC = 0xD7978EEB           # CRC of a 64 KiB zero block (the blocks a short data part does not have)
SENTINEL, SENTINEL_CRC = 0xA5, 0x5A5A5A5A
PLAN_KEYS = ("one_pass", "stripes_per_unit", "source_stripes_per_unit", "stages", "worker_warps", "rebuild_warps")
TWO_PASS = (0, 0, 0, 0, 0, 0)

CASES = [
    # source, lost source parts (data parts first, then parity rows), block counts (ragged with three units per chunk, nb < R),
    # destination, plan: one_pass, G, T, stages, worker warps, rebuild warps (R = G * k_dst)
    ("ec(8,2)", (1, 4), (49, 11), "ec(3,2)", (1, 8, 3, 4, 5, 3)),       # the geometry bench.py measures; x0 = 1 by doublings, KD = 3
    ("ec(8,2)", (5, 6), (49, 11), "ec(3,2)", (1, 8, 3, 4, 5, 3)),       # the same geometry, x0 = 5: 2^x0 S0 by the multiply with w[0]
    ("ec(7,2)", (5, 6), (43, 10), "xor7", (1, 3, 3, 4, 4, 4)),          # k_src = k_dst, multiply branch, last part lost
    ("ec(8,3)", (6, 7), (49, 12), "ec(8,2)", (1, 3, 3, 4, 5, 3)),       # k_src = k_dst with fewer destination parity parts
    ("ec(8,2)", (), (97, 23), "ec(8,3)", (1, 6, 6, 3, 8, 0)),           # k_src = k_dst with more, e = 0
    ("ec(12,2)", (0, 1), (25, 5), "ec(2,3)", (1, 6, 1, 4, 4, 4)),       # T = 1
    ("ec(6,2)", (0, 1), (25, 5), "ec(2,3)", (1, 6, 2, 4, 4, 4)),        # T = 2
    ("ec(16,2)", (9, 15), (65, 15), "ec(8,2)", (1, 4, 2, 4, 5, 3)),     # T = 2, x0 = 9, last part lost
    ("ec(32,2)", (30, 31), (65, 15), "ec(16,2)", (1, 2, 1, 3, 5, 3)),   # T = 1, 3 stages, k_src = 32
    ("ec(15,2)", (0, 1), (91, 22), "ec(9,2)", (1, 5, 3, 2, 7, 1)),      # 2-stage ring, e = 2
    ("ec(22,1)", (0,), (45, 11), "ec(2,3)", (1, 11, 1, 2, 6, 2)),       # 2-stage ring, e = 1, T = 1
    ("ec(2,2)", (0, 1), (21, 5), "ec(10,2)", (1, 1, 5, 4, 3, 5)),       # G = 1, 5 rebuild warps next to 3 worker warps
    ("ec(2,2)", (0, 1), (25, 5), "xor3", (1, 4, 6, 4, 3, 5)),           # 5 rebuild warps, KD = 3
    ("xor2", (), (129, 31), "ec(2,1)", (1, 32, 32, 3, 8, 0)),           # R = 64, xor -> ec part numbering with the same k
    ("ec(9,2)", (), (127, 31), "ec(7,1)", (1, 9, 7, 3, 8, 0)),          # R = 63
    ("ec(16,4)", (3, 12), (65, 15), "ec(8,3)", (1, 4, 2, 4, 6, 2)),     # source parity rows 2 and 3 present, not used
    ("ec(8,3)", (2, 10), (81, 19), "ec(4,2)", (1, 10, 5, 3, 7, 1)),     # data part 2 and parity row 2 lost: row 0 alone is needed
    ("xor3", (2,), (49, 11), "xor8", (1, 3, 8, 4, 4, 4)),               # e = 1, even T, k_src < k_dst, xor -> xor
    ("ec(16,1)", (), (65, 15), "ec(32,2)", (1, 1, 2, 4, 8, 0)),         # e = 0, G = 1, T = 2
    ("ec(18,1)", (0,), (73, 17), "xor3", (1, 12, 2, 4, 5, 3)),          # e = 1, T = 2, KD = 3
    ("xor9", (), (91, 22), "ec(3,2)", (1, 15, 5, 2, 8, 0)),             # e = 0, 2-stage ring, KD = 3
    ("xor7", (0,), (99, 24), "ec(7,1)", (1, 7, 7, 3, 7, 1)),            # e = 1, R = 49, xor -> ec with the same k
    ("xor7", (0,), (29, 5), "ec(2,3)", (1, 7, 2, 4, 4, 4)),             # e = 1, R = 14
    ("xor2", (0,), (37, 9), "ec(18,3)", (1, 1, 9, 4, 4, 4)),            # e = 1, G = 1
    ("ec(18,1)", (), (37, 9), "ec(2,3)", (1, 9, 1, 4, 8, 0)),           # e = 0, T = 1
    ("ec(25,2)", (0, 1), (101, 23), "xor2", (1, 25, 2, 4, 7, 1)),       # e = 2, R = 50
    ("ec(3,1)", (1,), (73, 17), "xor3", (1, 12, 12, 4, 6, 2)),          # ec -> xor with the same k
    # the two-pass route
    ("ec(7,2)", (5, 6), (40, 10), "ec(9,3)", TWO_PASS),                 # refused on rows: R * 4 + e T 4 + G (m_dst - 1) 4 > 224
    ("ec(8,2)", (), (37, 11), "ec(8,4)", TWO_PASS),                     # four destination parity parts
    ("ec(10,5)", (), (43, 13), "ec(8,2)", TWO_PASS),                    # Cauchy source
    ("ec(8,2)", (), (45, 13), "ec(22,4)", TWO_PASS),                    # Cauchy destination
    ("ec(8,3)", (1, 4, 6), (37, 13), "ec(4,2)", TWO_PASS),              # three data parts lost
    ("ec(8,3)", (0, 8), (37, 13), "ec(4,2)", TWO_PASS),                 # data part 0 and parity row 0 lost: row 1 alone
]
FULL_SIZE = [("ec(8,2)", (5, 6), "ec(3,2)"), ("ec(12,2)", (0, 1), "ec(2,3)"), ("ec(15,2)", (0, 1), "ec(9,2)")]   # also at nb = 1024
REF_PINNED = [("ec(8,2)", (5, 6), "ec(3,2)"), ("ec(12,2)", (0, 1), "ec(2,3)"), ("ec(7,2)", (5, 6), "xor7"), ("xor2", (), "ec(2,1)"),
              ("ec(16,4)", (3, 12), "ec(8,3)")]
CONTEXTS = ("default", "cap", "two_pass")


def _case_id(case, nb):
    src, lost, _, dst, _ = case
    return f"{src}-lost{''.join(map(str, lost)) or '-'}-{dst}-nb{nb}"


def _params(full_size=False):
    """(case, nb) for the `inp` fixture; the 64 MiB runs last, so that every test's list starts with the same entries and pytest
    runs the tests of one input set one after the other (the input fixture is built once per set)"""
    out = [pytest.param((case, nb), id=_case_id(case, nb)) for case in CASES for nb in case[2]]
    if full_size:
        out += [pytest.param((case, 1024), id=_case_id(case, 1024)) for case in CASES if (case[0], case[1], case[3]) in FULL_SIZE]
    return out


def plan_of(src, lost, dst, want=None):
    s, d = L.SliceType(src), L.SliceType(dst)
    avail = [0 if i in lost else 1 for i in range(s.k + s.m)]
    return L.Engine.plan_convert(s, d, avail, want if want is not None else [1] * (d.k + d.m))


# ---- the planner's space, on the CPU ---------------------------------------------------------------------------------------------

def _goals():
    return [L.SliceType(f"xor{k}") for k in range(2, 10)] + [L.SliceType(f"ec({k},{m})") for k in range(2, 33) for m in range(1, 5)]


def _losses(k, m):
    """no loss, each single data loss, and pairs: first / last, adjacent at both ends and in the middle, x0 <= 4 and >= 5"""
    out = [()] + [(j,) for j in range(k)]
    if m >= 2:
        pairs = {(0, k - 1), (0, 1), (k - 2, k - 1), (k // 2 - 1, k // 2), (1, 4), (min(4, k - 2), k - 1), (5, 6), (5, k - 1)}
        out += sorted(p for p in pairs if 0 <= p[0] < p[1] < k)
    return out


def features(ks, kd, md, lost, plan):
    """the values of the geometry and loss features the kernel branches on, alone and paired with e"""
    e = plan["lost_data_parts"]
    G, T, R = plan["stripes_per_unit"], plan["source_stripes_per_unit"], plan["stripes_per_unit"] * kd
    f = {("T", T if T <= 2 else ("odd >= 3" if T % 2 else "even >= 4")), ("stages", plan["stages"]), ("rebuild warps", plan["rebuild_warps"]),
         ("G", "1" if G == 1 else ("> worker warps" if G > plan["worker_warps"] else "<= worker warps")),
         ("R", "<= 16" if R <= 16 else ("17-48" if R <= 48 else "> 48")), ("m_dst", md), ("KD = 3", md <= 2 and kd == 3),
         ("k_src vs k_dst", "<" if ks < kd else ("=" if ks == kd else ">")), ("e", e)}
    data_lost = [x for x in lost if x < ks]
    if e == 2:
        f |= {("x0 >= 5", data_lost[0] >= 5), ("adjacent", data_lost[1] == data_lost[0] + 1)}
    if e >= 1:
        f.add(("last data part lost", data_lost[-1] == ks - 1))
    return f | {(e,) + x for x in f}


REFUSALS = ("Cauchy source", "Cauchy destination", "four destination parity parts", "three data parts lost",
            "parity rows in use other than 0 .. e-1", "no unit geometry fits")


def refusal(src, lost, dst):
    """why a request takes the two-pass route"""
    s, d = L.SliceType(src), L.SliceType(dst)
    cauchy = lambda g: g.m >= 5 or (g.m == 4 and g.k > 20)       # noqa: E731  (reed_solomon.h: Cauchy rows beyond Vandermonde's)
    used = [i for i in range(s.k + s.m) if i not in lost][:s.k]
    e = sum(1 for i in range(s.k) if i in lost)
    if cauchy(s):
        return REFUSALS[0]
    if cauchy(d):
        return REFUSALS[1]
    if d.m > 3:
        return REFUSALS[2]
    if e > 2:
        return REFUSALS[3]
    if [i - s.k for i in used if i >= s.k] != list(range(e)):
        return REFUSALS[4]
    return REFUSALS[5]


def test_convert_geometry_table_covers_the_planner_space():
    """every feature value, and every (e, feature value), that some one-pass request of the planner's space has also occurs in
    CASES; every literal plan of CASES is the planner's; the block counts are ragged / partial as the GPU tests assume"""
    space = set()
    goals = _goals()
    dsts = [d for d in goals if d.m <= 3]
    all_wanted = {}
    for s in goals:
        for lost in _losses(s.k, s.m):
            avail = [0 if i in lost else 1 for i in range(s.k + s.m)]
            for d in dsts:
                if (s.kind, s.k, s.m) == (d.kind, d.k, d.m):
                    continue
                want = all_wanted.setdefault(d.k + d.m, [1] * (d.k + d.m))
                p = L.Engine.plan_convert(s, d, avail, want)
                if p["one_pass"]:
                    space |= features(s.k, d.k, d.m, lost, p)
    table = set()
    for src, lost, nbs, dst, want in CASES:
        p = plan_of(src, lost, dst)
        assert tuple(p[k] for k in PLAN_KEYS) == want, (src, lost, dst, p)
        s, d = L.SliceType(src), L.SliceType(dst)
        ragged, small = nbs
        assert ragged % s.k and ragged % d.k and small < ragged, (src, dst, nbs)
        if p["one_pass"]:
            table |= features(s.k, d.k, d.m, lost, p)
            R = p["stripes_per_unit"] * d.k
            assert ragged % R and ragged > 2 * R and small < R, (src, dst, nbs, R)
    assert not space - table, sorted(space - table, key=str)
    assert ("ec(8,2)", (1, 4), (49, 11), "ec(3,2)", (1, 8, 3, 4, 5, 3)) in CASES    # bench.py's geometry stays put
    assert {refusal(c[0], c[1], c[3]) for c in CASES if not c[4][0]} == set(REFUSALS)
    for src, lost, dst in FULL_SIZE + REF_PINNED:
        assert any(c[0] == src and c[1] == lost and c[3] == dst and c[4][0] == 1 for c in CASES), (src, lost, dst)


# ---- GPU: contexts, inputs, one call -------------------------------------------------------------------------------------------

_engines = {}
_scratch = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in _engines.values():
        e.close()
    _engines.clear()
    _scratch.clear()


def engine(ctx):
    """one context per kind; the switches are read when a context is created, so they are set around its creation only"""
    env = {"default": {}, "cap": {"LZGPU_GRID_CAP": "2"}, "two_pass": {"LZGPU_CONVERT_FUSED": "0"}}[ctx]
    if ctx not in _engines:
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            _engines[ctx] = L.Engine(0)
        finally:
            for k, v in old.items():
                if v is None:
                    del os.environ[k]
                else:
                    os.environ[k] = v
    return _engines[ctx]


@pytest.fixture(scope="module")
def eng():
    return engine("default")


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t, dtype=np.uint8):
    return t.cpu().numpy().view(dtype)


def inputs(oracle, case, nb):
    """N_CAP chunks (N at 64 MiB, which already gives more than 2 x 2 units) of random data, the k + m parts of the source slice (data
    parts zero-padded) with their stored CRCs, on the host and the device, and the oracle's destination parts and CRCs per chunk"""
    src_name, lost, _, dst_name, _ = case
    src, dst = L.SliceType(src_name), L.SliceType(dst_name)
    k, m = src.k, src.m
    n = N if nb == 1024 else N_CAP
    pb = -(-nb // k)
    rng = np.random.default_rng(zlib.crc32(repr((src_name, lost, dst_name, nb)).encode()))
    data = rng.integers(0, 256, size=(n, nb * BLOCK), dtype=np.uint8)
    enc = [oracle.encode_chunk(src.kind, k, m, data[c]) for c in range(n)]
    per = [O.split_parts(data[c], k)[0] for c in range(n)]
    parts = [np.stack([per[c][j] for c in range(n)]) for j in range(k)] + [np.stack([enc[c][0][r] for c in range(n)]) for r in range(m)]
    crc = np.stack([enc[c][1] for c in range(n)])
    crcs = []
    for j in range(k):
        cj = np.full((n, pb), ZERO_CRC, dtype=np.uint32)
        mine = crc[:, j:nb:k]
        cj[:, : mine.shape[1]] = mine
        crcs.append(cj)
    crcs += [np.ascontiguousarray(crc[:, nb + r * pb: nb + (r + 1) * pb]) for r in range(m)]
    nd = dst.k + dst.m
    ref = [O.convert_chunk(oracle, (src.kind, k, m), [None if i in lost else parts[i][c] for i in range(k + m)],
                           [None if i in lost else crcs[i][c] for i in range(k + m)], (dst.kind, dst.k, dst.m), [1] * nd, nb)
           for c in range(n)]
    assert all(r[0] == 0 for r in ref)
    return dict(case=case, src=src, dst=dst, lost=lost, nb=nb, n_cap=n, parts=parts, crcs=crcs,
                d_parts=[None if i in lost else dev(parts[i]) for i in range(k + m)],
                d_crcs=[None if i in lost else dev(crcs[i].view(np.int32)) for i in range(k + m)],
                want_out=[np.stack([r[1][i] for r in ref]) for i in range(nd)],
                want_crc=[np.stack([r[2][i] for r in ref]) for i in range(nd)])


@pytest.fixture(scope="module")
def inp(request, oracle):
    """the inputs of one (case, nb), built once for every test that takes them (pytest groups those tests)"""
    case, nb = request.param
    return inputs(oracle, case, nb)


def mark_launch(e):
    """a one-unit CRC launch first, so that last_geometry() afterwards shows the launch of the call under test and nothing older"""
    if "blk" not in _scratch:
        _scratch["blk"] = torch.zeros(BLOCK, dtype=torch.uint8, device="cuda")
        _scratch["crc"] = torch.zeros(1, dtype=torch.int32, device="cuda")
    e.crc_blocks_dev(_scratch["blk"].data_ptr(), 1, _scratch["crc"].data_ptr())
    assert e.last_launch() == (1, 1)


def run(ctx, inp, want, verify=True, d_crcs=None):
    """convert_chunks_dev on the context `ctx` over N chunks (all of them under the cap); every destination part and CRC array has a
    sentinel-filled buffer, wanted or not.  Returns the host copies of all of them."""
    e = engine(ctx)
    n = inp["n_cap"] if ctx == "cap" else N
    src, dst, nb = inp["src"], inp["dst"], inp["nb"]
    pbs, pbd, nd = -(-nb // src.k), -(-nb // dst.k), dst.k + dst.m
    outs = [torch.full((n, pbd * BLOCK), SENTINEL, dtype=torch.uint8, device="cuda") for _ in range(nd)]
    ocrc = [torch.full((n, pbd), SENTINEL_CRC, dtype=torch.int32, device="cuda") for _ in range(nd)]
    crcs = d_crcs if d_crcs is not None else inp["d_crcs"]
    torch.cuda.synchronize()
    mark_launch(e)
    try:
        e.convert_chunks_dev(src, dst, n, nb, [0 if t is None else t.data_ptr() for t in inp["d_parts"]], pbs * BLOCK, want,
                             [t.data_ptr() for t in outs], pbd * BLOCK,
                             d_part_crc=[0 if t is None else t.data_ptr() for t in crcs] if verify else None,
                             d_out_crc=[t.data_ptr() for t in ocrc])
    finally:
        check_route(ctx, inp, n, want)
    e.sync()
    return [host(t).reshape(n, -1) for t in outs], [host(t, np.uint32).reshape(n, -1) for t in ocrc]


def check_route(ctx, inp, n, want):
    """the call that just ran launched the one-pass kernel with the planned geometry, or (two-pass route) did not launch it"""
    src, dst, nb = inp["src"], inp["dst"], inp["nb"]
    plan = L.Engine.plan_convert(src, dst, [0 if i in inp["lost"] else 1 for i in range(src.k + src.m)], want)
    e = engine(ctx)
    g = e.last_geometry()
    assert (g["grid"], g["units"]) == e.last_launch()
    if ctx == "two_pass" or not plan["one_pass"]:
        assert g["kernel"] != _lib.KERNEL_CONVERT, g
        return
    R = plan["stripes_per_unit"] * dst.k
    expect = dict(kernel=_lib.KERNEL_CONVERT, threads=256, G=plan["stripes_per_unit"], stages=plan["stages"], gf_warps=plan["rebuild_warps"],
                  smem_bytes=plan["smem_bytes"], units=n * math.ceil(nb / R))
    assert {k: g[k] for k in expect} == expect, (g, expect)
    if ctx == "cap":
        assert g["grid"] == 2 and g["units"] > 2 * g["grid"], g
    else:
        sm = torch.cuda.get_device_properties(0).multi_processor_count
        assert g["grid"] == min(g["units"], 2 * sm), (g, sm)


def assert_outputs(inp, out, ocrc, want, what):
    n = out[0].shape[0]
    for i, w in enumerate(want):
        if w:
            assert (out[i] == inp["want_out"][i][:n]).all(), (what, i, [c for c in range(n) if (out[i][c] != inp["want_out"][i][c]).any()])
            bad = np.argwhere(ocrc[i] != inp["want_crc"][i][:n])
            assert bad.size == 0, (what, i, bad[:4].tolist())
        else:
            assert (out[i] == SENTINEL).all() and (ocrc[i] == SENTINEL_CRC).all(), (what, "unwanted part written", i)


# ---- GPU: every byte and CRC, three contexts -------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("inp", _params(full_size=True), indirect=True)
def test_convert_geometry_vs_oracle_and_two_passes(inp):
    nd = inp["dst"].k + inp["dst"].m
    want = [1] * nd
    for verify in (True, False):
        got = {}
        for ctx in CONTEXTS:
            got[ctx] = run(ctx, inp, want, verify)
            assert_outputs(inp, *got[ctx], want, (ctx, verify))
        for ctx in ("default", "cap"):
            for i in range(nd):
                assert (got[ctx][0][i][:N] == got["two_pass"][0][i]).all(), (ctx, verify, i)
                assert (got[ctx][1][i][:N] == got["two_pass"][1][i]).all(), (ctx, verify, i)


@pytest.mark.gpu
@pytest.mark.parametrize("inp", _params(), indirect=True)
def test_convert_geometry_wanted_subsets(inp):
    """only the last destination parity part (a replication job), and the data parts with parity row 0"""
    kd, md = inp["dst"].k, inp["dst"].m
    for name, want in (("last parity part", [0] * (kd + md - 1) + [1]), ("data + parity row 0", [1] * (kd + 1) + [0] * (md - 1))):
        for ctx in CONTEXTS:
            out, ocrc = run(ctx, inp, want)
            assert_outputs(inp, out, ocrc, want, (ctx, name))


@pytest.mark.gpu
@pytest.mark.parametrize("inp", _params(), indirect=True)
def test_convert_geometry_reports_stored_crc_errors(inp):
    """a wrong stored CRC word of the last source parity part in use, in the ragged last unit of chunk 1; in a separate call a wrong
    word of a read data part (a parity part where every data part is lost) in a middle unit of chunk 1 plus one in chunk 2: each
    reported at the (chunk, part, block) of the first mismatch, on both routes"""
    case, nb, src, dst = inp["case"], inp["nb"], inp["src"], inp["dst"]
    ks, lost = src.k, inp["lost"]
    pbs = -(-nb // ks)
    used = [i for i in range(ks + src.m) if i not in lost][:ks]
    par = [i for i in used if i >= ks]
    read = [i for i in used if i < min(ks, nb)] or par     # parts read that have blocks (data part i has none when i >= nb)
    plan = plan_of(case[0], lost, case[3])
    j = read[-1]
    last = (nb - 1 - j) // ks if j < ks else pbs - 1    # the last stripe at which part j has a block
    if plan["one_pass"]:
        T, units = plan["source_stripes_per_unit"], math.ceil(nb / (plan["stripes_per_unit"] * dst.k))
        mid = min((units // 2) * T + T // 2, last)
        assert units < 3 or units // 2 * T <= mid < (units // 2 + 1) * T
    else:
        mid = last // 2
    calls = []
    if par:
        calls.append(([(1, par[-1], pbs - 1)], (1, par[-1], pbs - 1)))
    calls.append(([(2, read[0], 0), (1, j, mid)], (1, j, mid)))
    want = [1] * (dst.k + dst.m)
    for words, where in calls:
        d_crcs = list(inp["d_crcs"])
        bad = {}
        for c, part, blk in words:
            bad.setdefault(part, inp["crcs"][part].copy())[c, blk] ^= 0x00010000
        for part, words_of_part in bad.items():
            d_crcs[part] = dev(words_of_part.view(np.int32))
        for ctx in CONTEXTS:
            with pytest.raises(L.ChunkCrcError) as ei:
                run(ctx, inp, want, True, d_crcs)
            assert ei.value.where == where, (ctx, words)


# ---- GPU: the compiled reference's SliceRecoveryPlanner ------------------------------------------------------------------------

@pytest.mark.gpu
def test_convert_geometry_vs_reference_planner(eng, oracle):
    """five of the one-pass pairs above straight against the reference's SliceRecoveryPlanner + post-processing executed in memory
    (oracle/ref_plans.cc), or its answers recorded in tests/golden/reference_digests.json; one chunk at the ragged block count"""
    from tests.test_oracle_plans import make_slice, ref_sources, true_blocks
    for src_name, lost, dst_name in REF_PINNED:
        nb = next(c[2][0] for c in CASES if (c[0], c[1], c[3]) == (src_name, lost, dst_name))
        s, d = L.SliceType(src_name), L.SliceType(dst_name)
        src, dst = (s.kind, s.k, s.m), (d.kind, d.k, d.m)
        chunk = O.fill_chunk(oracle, nb * BLOCK, 41, 0)
        sparts, _ = make_slice(oracle, src, chunk)
        parts = [None if i in lost else sparts[i][None, :] for i in range(len(sparts))]
        nd = d.k + d.m
        out, ocrc = eng.convert_chunks(s, d, nb, parts, [1] * nd)
        sources = ref_sources(src, sparts, nb, lost)
        for i in range(nd):
            nblk = true_blocks(dst, i, nb)
            if nblk == 0:
                continue
            want = O.ref_digest(f"gpu_convert/{src_name}/{list(lost)}/{nb}/{dst_name}/{i}", lambda ref: O.plan_recover_part(
                ref, sources, O.slice_type(*dst), O.ref_part_number(dst[0], dst[1], i), 0, nblk) or (None,))
            assert O.digest(out[i][0][: nblk * BLOCK], ocrc[i][0][:nblk].view(np.uint32)) == want, (src_name, dst_name, i)
