"""The fused encode (fused_stream_kernel, csrc/fused_kernel.cuh) at every kernel instantiation and unit mode its launcher selects.

Each launch of the encoder family picks one of the compiled instantiations (lzgpu_debug_encoder_kernels lists them, KERNELS below
writes them out): fused_run / find_encoder (csrc/fused.cu) choose by the parity rows M (0: the CRC-only form), Vandermonde or generic
coefficients, bit-sliced or packed items, the unit mode (per-chunk, flat, striped), the SPLIT conversion form and whether (K, G) has
a constant-folded entry; a generic entry's 4-byte-item twin is taken when G leaves fewer than three warps of 16-byte items.
lzgpu_debug_last_encoder reports which instantiation and unit mode a launch ran, so a route that silently moves to another kernel
(a folded (K, G) that falls through to the run-time-k kernel, say) fails here even though its bytes stay right.

The CPU half restates the launcher in plain Python (route(): lz_fused_encode, lz_fused_encode_split, lz_fused_crc, fused_run,
find_encoder, with pick_group / fused_plan from csrc/fused_plan.h and the H100's 232 448 bytes of opt-in shared memory), enumerates
it over every goal, a set of batch shapes, the striped policies and the tuning switches, and checks that
  - every instantiation is reached with the default switches, or is in SWITCH_ONLY (with a switch set that reaches it), or is in
    UNREACHED (with the reason);
  - CASES holds every reachable (instantiation, unit mode) pair once, at a shape where that mode breaks, with the restatement's
    instantiation and geometry written out;
  - the restatement agrees with lzgpu_plan_encode, the planner's own copy of the route, for every enumerated plain encode.
The GPU half runs every row of CASES uncapped and with LZGPU_GRID_CAP=2 (several units per CTA), checks last_encoder() and
last_geometry() against the row, and every output byte against the oracle (encode, SPLIT) or zlib.crc32 (the CRC-only form), with
sentinels in the stride padding and in every output the call does not own."""
import collections
import functools
import os
import zlib

import numpy as np
import pytest
import torch

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import _oracle as O

BLOCK = 65536
SMEM_OPTIN = 232448               # cudaDevAttrMaxSharedMemoryPerBlockOptin of the H100
SMEM_CAP = 113 * 1024             # kSmemCap: two CTAs per SM
SENTINEL, SENTINEL_CRC, GARBAGE = 0xA5, 0x5A5A5A5A, 0x5C
ENCODE, BITSLICE = _lib.KERNEL_ENCODE, _lib.KERNEL_ENCODE_BITSLICE

# every compiled instantiation, in kEncoders order with a generic entry's narrow twin right after it:
# (m, generic, bitsliced, striped, split, kt, gt, item_bytes)
KERNELS = [
    (0, 0, 0, 0, 0, 0, 0, 16), (1, 0, 0, 0, 0, 0, 0, 16), (2, 0, 0, 0, 0, 0, 0, 16), (3, 0, 0, 0, 0, 0, 0, 16),   # 0-3
    (4, 0, 0, 0, 0, 0, 0, 8),                                                                                       # 4
    (1, 1, 0, 0, 0, 0, 0, 16), (1, 1, 0, 0, 0, 0, 0, 4), (2, 1, 0, 0, 0, 0, 0, 16), (2, 1, 0, 0, 0, 0, 0, 4),       # 5-8
    (3, 1, 0, 0, 0, 0, 0, 16), (3, 1, 0, 0, 0, 0, 0, 4), (4, 1, 0, 0, 0, 0, 0, 16), (4, 1, 0, 0, 0, 0, 0, 4),       # 9-12
    (1, 0, 0, 0, 1, 0, 0, 16), (2, 0, 0, 0, 1, 0, 0, 16), (3, 0, 0, 0, 1, 0, 0, 16), (4, 0, 0, 0, 1, 0, 0, 8),       # 13-16 SPLIT
    (4, 1, 0, 0, 1, 0, 0, 16), (4, 1, 0, 0, 1, 0, 0, 4),                                                            # 17-18
    (1, 0, 0, 1, 0, 0, 0, 16), (2, 0, 0, 1, 0, 0, 0, 16), (3, 0, 0, 1, 0, 0, 0, 16), (4, 0, 0, 1, 0, 0, 0, 8),       # 19-22 striped
    (4, 1, 0, 1, 0, 0, 0, 16), (4, 1, 0, 1, 0, 0, 0, 4),                                                            # 23-24
    (2, 0, 0, 0, 0, 8, 7, 16), (1, 0, 0, 0, 0, 2, 32, 16), (1, 0, 0, 0, 0, 3, 20, 16), (2, 0, 0, 0, 0, 3, 16, 16),  # 25-28 folded
    (2, 0, 0, 0, 0, 4, 12, 16), (2, 0, 0, 0, 0, 6, 9, 16), (3, 0, 0, 0, 0, 5, 8, 16), (3, 0, 0, 0, 0, 6, 8, 16),    # 29-32
    (4, 0, 0, 0, 0, 8, 8, 8), (3, 0, 0, 0, 0, 8, 6, 16), (1, 0, 0, 0, 0, 4, 16, 16), (2, 0, 0, 0, 0, 5, 10, 16),     # 33-36
    (2, 0, 0, 0, 0, 10, 5, 16), (3, 0, 0, 0, 0, 4, 8, 16), (4, 0, 0, 0, 0, 10, 6, 8), (4, 0, 0, 0, 0, 12, 5, 8),     # 37-40
    (4, 0, 0, 0, 0, 6, 8, 8), (4, 0, 0, 0, 0, 4, 8, 8),                                                              # 41-42
    (2, 0, 0, 1, 0, 8, 7, 16), (1, 0, 0, 1, 0, 2, 32, 16), (1, 0, 0, 1, 0, 3, 20, 16), (2, 0, 0, 1, 0, 3, 16, 16),  # 43-46 striped folded
    (3, 0, 0, 1, 0, 5, 8, 16), (4, 0, 0, 1, 0, 8, 8, 8),                                                             # 47-48
    (3, 0, 1, 0, 0, 0, 0, 32), (4, 0, 1, 0, 0, 0, 0, 32), (3, 0, 1, 1, 0, 0, 0, 32), (4, 0, 1, 1, 0, 0, 0, 32),      # 49-52 bit-sliced
    (4, 0, 1, 0, 0, 8, 8, 32), (4, 0, 1, 0, 0, 10, 6, 32), (4, 0, 1, 0, 0, 12, 5, 32), (4, 0, 1, 0, 0, 6, 8, 32),    # 53-56
    (4, 0, 1, 0, 0, 4, 8, 32), (3, 0, 1, 0, 0, 8, 8, 32), (3, 0, 1, 0, 0, 9, 6, 32), (3, 0, 1, 0, 0, 10, 6, 32),     # 57-60
    (3, 0, 1, 0, 0, 12, 5, 32), (4, 0, 1, 1, 0, 8, 8, 32),                                                           # 61-62
]

# ---- the launcher, restated -----------------------------------------------------------------------------------------------------

Switches = collections.namedtuple("Switches", "striped bitslice bs_gfw bs_stages bs_smem")
DEFAULT_SWITCHES = Switches(striped=-1, bitslice=3, bs_gfw=4, bs_stages=4, bs_smem=200 * 1024)


@functools.lru_cache(maxsize=None)
def switches(env):
    """what lz_fused_init reads from the environment (env: "NAME=value" strings), as the restatement's switches"""
    sw = DEFAULT_SWITCHES._asdict()
    for item in env:
        name, value = item.split("=")
        v = int(value)
        if name == "LZGPU_STRIPED":
            sw["striped"] = v
        elif name == "LZGPU_BITSLICE":
            sw["bitslice"] = v
        elif name == "LZGPU_BS_GFW":
            sw["bs_gfw"] = max(1, min(12, v))
        elif name == "LZGPU_BS_STAGES":
            sw["bs_stages"] = max(2, min(16, v))
        elif name == "LZGPU_BS_SMEM_KB":
            sw["bs_smem"] = max(64, min(226, v)) * 1024
        else:
            assert name in ("LZGPU_CONVERT_FUSED",), name      # (the conversion's route, not the encoder's)
    return Switches(**sw)


def cauchy(k, m):
    return m >= 5 or (m == 4 and k > 20)


def threads(m, generic, bs=False):
    return 512 if bs else 288 if generic else 256 if m <= 3 else 512


def item_words(m, generic):
    return 4 if generic else 2 if m == 4 else 4


def ctas_per_sm(m, generic, bs=False):
    return 1 if threads(m, generic, bs) > 320 else 2


def n_stages(m, generic, bs=False):
    return 4 if ctas_per_sm(m, generic, bs) == 1 else 3


def smem_cap(m, generic):
    return 200 * 1024 if ctas_per_sm(m, generic) == 1 else SMEM_CAP


def smem_bytes(rows, prows, nst, npst=4):
    return nst * rows * 128 + npst * ((prows * 128 + 1023) & ~1023) + 520 + 8 * (2 * nst + 2 * npst)


@functools.lru_cache(maxsize=None)
def pick_group(K, PC, cap, thr, m, generic, bs, bs_gfw):
    best = 0
    per_stripe = 16 if bs else 128 // item_words(m, generic)
    for g in range(1, 65):
        gf_warps = (g * per_stripe + 31) // 32 if bs else 0
        if bs:
            if gf_warps > bs_gfw:
                break
        elif (thr > 288 or m >= 3) and m > 0 and best and g * per_stripe > thr:
            break
        rows, prows = g * K * 4, g * PC * 4
        if rows > 256 or rows + prows > thr - 32 * gf_warps or prows > 128 or g * K > 64:
            break
        if rows % 8:
            continue
        if smem_bytes(rows, prows, n_stages(m, generic, bs)) > cap:
            break
        best = g
    return best


@functools.lru_cache(maxsize=None)
def fused_plan(M, generic, K, n, nb, stride, cap, policy, bs=False, bs_stages=4, bs_gfw=4):
    """fused_plan (csrc/fused_plan.h): None where the fused kernel does not take the shape"""
    PC = 0 if M == 0 else (M if generic else M - 1)
    thr = threads(M, generic, bs)
    G = pick_group(K, PC, cap, thr, M, generic, bs, bs_gfw)
    if G == 0 or stride % 16:
        return None
    pb = -(-nb // K)
    flat = n > 1 and stride == nb * BLOCK and nb % K == 0 and n * pb < 2 ** 31 and n * nb * 4 < 2 ** 31
    mode = 1 if flat else 0
    if not flat and M > 0 and n * pb < 2 ** 31:
        wasteful = -(-pb // G) * G * n * 100 > n * pb * 112
        if policy == 1 or (policy < 0 and wasteful):
            mode = 2
    units = -(-(n * pb) // G) if mode else -(-pb // G) * n
    if units > 0x7FFFFFFF:
        return None
    rows, prows = G * K * 4, G * PC * 4
    nst = n_stages(M, generic, bs)
    while bs and nst < bs_stages and smem_bytes(rows, prows, nst + 1) <= cap:
        nst += 1
    return dict(G=G, pb=pb, mode=mode, units=units, threads=thr, rows=rows, stages=nst, smem=smem_bytes(rows, prows, nst), bs=bs)


def bitslice(m, generic, mask, k):
    return not generic and ((m == 4 and mask & 1) or (m == 3 and ((mask & 2 and k >= 7) or mask & 4)))


def find_encoder(M, generic, K, G, striped, split, bs):
    """the folded entry of (M, K, G) where there is one, else the run-time-k one (indices into KERNELS; narrow twins skipped)"""
    runtime_k = None
    for i, (m, gen, b, st, sp, kt, gt, ib) in enumerate(KERNELS):
        if gen and ib == 4:
            continue
        if (m, gen, b, st, sp) != (M, generic, bs, striped, split):
            continue
        if (kt, gt) == (K, G):
            return i
        if kt == 0:
            runtime_k = i
    return runtime_k


@functools.lru_cache(maxsize=None)
def fused_run(sw, M, generic, K, n, nb, stride, split=False, policy=None):
    """fused_run: the launch (index, mode and geometry), or None (LZGPU_NOT_HANDLED)"""
    spol = 0 if split else (sw.striped if policy is None else policy)
    pl = None
    if not split and bitslice(M, generic, sw.bitslice, K):
        pl = fused_plan(M, generic, K, n, nb, stride, min(SMEM_OPTIN, sw.bs_smem), spol, True, sw.bs_stages, sw.bs_gfw)
    if pl is None:
        pl = fused_plan(M, generic, K, n, nb, stride, min(SMEM_OPTIN, smem_cap(M, generic)), spol)
    if pl is None:
        return None
    G, bs = pl["G"], pl["bs"]
    i = find_encoder(M, generic, K, G, pl["mode"] == 2, split, bs)
    if i is None:
        return None
    if generic and 32 * G < 96:
        i += 1                    # fused_generic_item_words(G) == 1: the 4-byte-item twin
    geo = (BITSLICE if bs else ENCODE, G, pl["threads"], pl["stages"], (16 * G + 31) // 32 if bs else 0, pl["smem"], pl["units"])
    return dict(index=i, mode=pl["mode"], geo=geo, plan=pl)


def route(sw, form, goal, n, nb, stride):
    """the encoder launches of one call, in order; None: no fused launch (the generic kernels take the call).
    form "encode": lz_fused_encode (goal = (kind, k, m)); "split": lz_fused_encode_split (goal = the destination); "crc":
    lz_fused_crc of n runs of nb blocks at `stride` (goal unused)"""
    if form == "crc":
        contiguous = n > 1 and stride == nb * BLOCK
        K = 1 if (contiguous and nb % 64) else 64
        r = fused_run(sw, 0, False, K, n, nb, stride if n > 1 else nb * BLOCK)
        return None if r is None else [r]
    kind, K, M = goal
    if form == "split":
        if M > 4:
            return None
        r = fused_run(sw, 4, True, K, n, nb, stride, split=True) if cauchy(K, M) else fused_run(sw, M, False, K, n, nb, stride, split=True)
        return None if r is None else [r]
    if cauchy(K, M):
        if M == 4:
            r = fused_run(sw, 4, True, K, n, nb, stride)
            return None if r is None else [r]
        for rows in (4, M % 4):
            if rows and fused_plan(rows, True, K, n, nb, stride, min(SMEM_OPTIN, smem_cap(rows, True)), 0) is None:
                return None
        return [fused_run(sw, min(4, M - r0), True, K, n, nb, stride, policy=0) for r0 in range(0, M, 4)]
    if M > 4:
        return None
    r = fused_run(sw, M, False, K, n, nb, stride)
    if r is None and kind == 1:
        r = fused_run(sw, M, True, K, n, nb, stride, policy=0)   # the nine-warp generic-coefficient CTA (ec(31,3) on packed items)
    return None if r is None else [r]


# ---- the space the restatement is enumerated over --------------------------------------------------------------------------------

GOALS = [(0, k, 1) for k in range(2, 10)] + [(1, k, m) for k in range(2, 33) for m in range(1, 33)]
SWITCH_SETS = [(), ("LZGPU_STRIPED=0",), ("LZGPU_STRIPED=1",)] + [(f"LZGPU_BITSLICE={b}",) for b in (0, 1, 2, 4, 7)] + [
    ("LZGPU_BS_SMEM_KB=64",), ("LZGPU_BS_GFW=2",), ("LZGPU_BS_GFW=8",), ("LZGPU_BS_STAGES=8",), ("LZGPU_BITSLICE=0", "LZGPU_STRIPED=1"),
    ("LZGPU_BITSLICE=0", "LZGPU_STRIPED=0"), ("LZGPU_BITSLICE=7", "LZGPU_STRIPED=1")]
PAD = 4096                        # stride padding of the padded shapes


def shapes(k):
    """(n_chunks, nb, stride) batch shapes: one and several chunks; nb = 1, < k, k, ragged, 64 and 1024; dense and padded"""
    out = set()
    for nb in {1, max(1, k - 1), k, 2 * k + 1, 3 * k, 64, 1024}:
        for n in (1, 3):
            out |= {(n, nb, nb * BLOCK), (n, nb, nb * BLOCK + PAD)}
    return sorted(out)


@functools.lru_cache(maxsize=None)
def enumerate_routes():
    """{switch set: {(index, mode): a call that records it}} over the whole space, and the set of indices each switch set launches
    (every pass of a multi-pass encode counts)"""
    recorded, launched = {}, {}
    for env in SWITCH_SETS:
        sw = switches(env)
        rec, lau = {}, set()

        def add(calls, key):
            if calls:
                rec.setdefault((calls[-1]["index"], calls[-1]["mode"]), key)
                lau.update(c["index"] for c in calls)
        for goal in GOALS:
            for n, nb, stride in shapes(goal[1]):
                add(route(sw, "encode", goal, n, nb, stride), ("encode", goal, n, nb, stride))
                if goal[2] <= 4:
                    add(route(sw, "split", goal, n, nb, stride), ("split", goal, n, nb, stride))
        for n, nb, stride in ((1, 64, 64 * BLOCK), (1, 5, 5 * BLOCK), (3, 64, 64 * BLOCK), (3, 7, 7 * BLOCK), (3, 7, 7 * BLOCK + PAD)):
            add(route(sw, "crc", None, n, nb, stride), ("crc", None, n, nb, stride))
        recorded[env], launched[env] = rec, lau
    return recorded, launched


# ---- what the enumeration found ----------------------------------------------------------------------------------------------------

# reached only under a switch: the packed four-row kernels (every Vandermonde ec(k,4) is bit-sliced by default, and the bit-sliced
# plan fits every one of them), and the packed folded ec(8,3) (three rows with k >= 7 are bit-sliced by default)
SWITCH_ONLY = [
    (4, ("LZGPU_BITSLICE=0",)), (22, ("LZGPU_BITSLICE=0", "LZGPU_STRIPED=1")), (33, ("LZGPU_BITSLICE=0",)), (34, ("LZGPU_BITSLICE=0",)),
    (39, ("LZGPU_BITSLICE=0",)), (40, ("LZGPU_BITSLICE=0",)), (41, ("LZGPU_BITSLICE=0",)), (42, ("LZGPU_BITSLICE=0",)),
    (48, ("LZGPU_BITSLICE=0", "LZGPU_STRIPED=1")),
]
# never launched: the generic four-row SPLIT and striped forms serve only a Cauchy ec(k,4), k > 20, whose G is at most 2 (k G 4 data
# rows and 16 G parity rows on 288 threads), so fused_generic_item_words always takes the 4-byte-item twin
UNREACHED = [
    (17, "generic SPLIT, 16-byte items: only Cauchy ec(k,4) with k > 20 take it, and their G <= 2 selects the narrow twin"),
    (23, "generic striped, 16-byte items: only Cauchy ec(k,4) with k > 20 take it, and their G <= 2 selects the narrow twin"),
]


def test_encoder_kernel_list_is_the_compiled_one():
    got = L.encoder_kernels()
    assert [tuple(e[f] for f in ("m", "generic", "bitsliced", "striped", "split", "kt", "gt", "item_bytes")) for e in got] == KERNELS
    lib = _lib.load()
    assert lib.lzgpu_debug_encoder_kernels(None, 0) == len(KERNELS) == 63
    few = (_lib.LzEncoderKernel * 2)()
    assert lib.lzgpu_debug_encoder_kernels(few, 2) == 63 and (few[1].m, few[1].kt) == (1, 0)   # capacity bounds the writes only


def test_every_instantiation_is_reached_or_accounted_for():
    recorded, launched = enumerate_routes()
    default = launched[()]
    switch_only = dict(SWITCH_ONLY)
    unreached = dict(UNREACHED)
    assert not set(switch_only) & set(unreached)
    for i in range(len(KERNELS)):
        if i in unreached:
            assert all(i not in lau for lau in launched.values()), (i, unreached[i])
        elif i in switch_only:
            assert i not in default, i
            assert i in launched[switch_only[i]], (i, switch_only[i])
        else:
            assert i in default, i
    assert len(default) == 52 and len(SWITCH_ONLY) == 9 and len(UNREACHED) == 2
    # the reason given for UNREACHED: every Cauchy ec(k,4) has G <= 2 on the generic CTA
    for k in range(21, 33):
        assert pick_group(k, 4, SMEM_CAP, 288, 4, True, False, 4) <= 2, k


def test_restatement_matches_the_plan():
    """with the default switches, the restatement's first launch is lzgpu_plan_encode's plan for every enumerated plain encode"""
    import ctypes as C
    lib, out = _lib.load(), _lib.LzEncodePlan()

    def eng_plan(g, n, nb, stride, policy):
        assert lib.lzgpu_plan_encode(C.byref(g.c), n, nb, stride, policy, C.byref(out)) == 0
        return {f: getattr(out, f) for f, _ in _lib.LzEncodePlan._fields_}
    for goal in GOALS:
        g = L.SliceType(*goal)
        for n, nb, stride in shapes(goal[1]):
            for policy in (-1, 0, 1):
                calls = route(switches((f"LZGPU_STRIPED={policy}",)), "encode", goal, n, nb, stride)
                p = eng_plan(g, n, nb, stride, policy)
                if calls is None:
                    assert not p["fused"], (goal, n, nb, stride, policy, p)
                    continue
                first = calls[0]["plan"]
                got = dict(fused=1, mode=first["mode"], stripes_per_unit=first["G"], threads_per_cta=first["threads"], units=first["units"],
                           stage_rows=first["rows"], smem_bytes=first["smem"], passes=len(calls))
                assert {k: p[k] for k in got} == got, (goal, n, nb, stride, policy)


# ---- the GPU case table ------------------------------------------------------------------------------------------------------------

CONVERT_TWO_PASS = ("LZGPU_CONVERT_FUSED=0",)
CASES = [
    # form, goal (the destination for "split" / "crc_parts"), chunks, blocks per chunk, bytes the chunk is short of nb whole blocks,
    # stride padding in bytes, switches, instantiation (index into KERNELS), unit mode, geometry: (kernel, G, threads, stages,
    # gf_warps, smem_bytes, units).  "encode": lzgpu_encode_chunks_dev; "split": the conversion of a standard chunk into the goal
    # (two-pass route: the SPLIT encode of the image); "crc_blocks" / "verify": lzgpu_crc_blocks_dev / lzgpu_verify_blocks over
    # nb blocks; "crc_parts": the conversion wanting only the data parts, with their CRCs (crc_of_parts over each data part).
    # Per-chunk rows: nb % k != 0, pb % G != 0 and two or more units per chunk; flat rows: nb % k == 0, n pb % G != 0 (units
    # straddle chunk boundaries) and three or more units; striped rows: a padded stride, a ragged tail and three or more units;
    # per family one row with nb < k (a single partial stripe).
    ("encode", "xor5", 2, 106, 1000, 0, (), 1, 0, (1, 12, 256, 3, 0, 92792, 4)),
    ("encode", "xor5", 2, 65, 0, 0, (), 1, 1, (1, 12, 256, 3, 0, 92792, 3)),
    ("encode", "ec(2,2)", 2, 75, 1000, 0, (), 2, 0, (1, 21, 256, 3, 0, 110200, 4)),
    ("encode", "ec(2,2)", 2, 44, 0, 0, (), 2, 1, (1, 21, 256, 3, 0, 110200, 3)),
    ("encode", "ec(2,3)", 2, 29, 1000, 0, (), 3, 0, (1, 8, 256, 3, 0, 57976, 4)),
    ("encode", "ec(2,3)", 2, 18, 0, 0, (), 3, 1, (1, 8, 256, 3, 0, 57976, 3)),
    ("encode", "ec(2,4)", 2, 17, 1000, 0, ('LZGPU_BITSLICE=0', 'LZGPU_STRIPED=0'), 4, 0, (1, 8, 512, 4, 0, 82568, 4)),
    ("encode", "ec(2,4)", 2, 18, 0, 0, ('LZGPU_BITSLICE=0',), 4, 1, (1, 8, 512, 4, 0, 82568, 3)),
    ("encode", "ec(2,5)", 2, 45, 1000, 0, (), 5, 0, (1, 22, 288, 3, 0, 113272, 4)),
    ("encode", "ec(2,5)", 3, 30, 0, 0, (), 5, 1, (1, 22, 288, 3, 0, 113272, 3)),
    ("encode", "ec(17,5)", 2, 35, 1000, 0, (), 6, 0, (1, 2, 288, 3, 0, 56952, 4)),
    ("encode", "ec(17,5)", 3, 51, 0, 0, (), 6, 1, (1, 2, 288, 3, 0, 56952, 5)),
    ("encode", "ec(2,6)", 2, 33, 1000, 0, (), 7, 0, (1, 16, 288, 3, 0, 115320, 4)),
    ("encode", "ec(2,6)", 3, 22, 0, 0, (), 7, 1, (1, 16, 288, 3, 0, 115320, 3)),
    ("encode", "ec(17,6)", 2, 35, 1000, 0, (), 8, 0, (1, 2, 288, 3, 0, 61048, 4)),
    ("encode", "ec(17,6)", 3, 51, 0, 0, (), 8, 1, (1, 2, 288, 3, 0, 61048, 5)),
    ("encode", "ec(2,7)", 2, 19, 1000, 0, (), 9, 0, (1, 9, 288, 3, 0, 85624, 4)),
    ("encode", "ec(2,7)", 2, 20, 0, 0, (), 9, 1, (1, 9, 288, 3, 0, 85624, 3)),
    ("encode", "ec(15,7)", 2, 31, 1000, 0, (), 10, 0, (1, 2, 288, 3, 0, 59000, 4)),
    ("encode", "ec(15,7)", 3, 45, 0, 0, (), 10, 1, (1, 2, 288, 3, 0, 59000, 5)),
    ("encode", "ec(2,8)", 2, 17, 1000, 0, (), 11, 0, (1, 8, 288, 3, 0, 90744, 4)),
    ("encode", "ec(2,8)", 2, 18, 0, 0, (), 11, 1, (1, 8, 288, 3, 0, 90744, 3)),
    ("encode", "ec(15,8)", 2, 31, 1000, 0, (), 12, 0, (1, 2, 288, 3, 0, 63096, 4)),
    ("encode", "ec(15,8)", 3, 45, 0, 0, (), 12, 1, (1, 2, 288, 3, 0, 63096, 5)),
    ("split", "xor2", 2, 65, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 13, 0, (1, 32, 256, 3, 0, 98936, 4)),
    ("split", "xor2", 2, 66, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 13, 1, (1, 32, 256, 3, 0, 98936, 3)),
    ("split", "ec(2,2)", 2, 43, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 14, 0, (1, 21, 256, 3, 0, 110200, 4)),
    ("split", "ec(2,2)", 2, 44, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 14, 1, (1, 21, 256, 3, 0, 110200, 3)),
    ("split", "ec(2,3)", 2, 17, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 15, 0, (1, 8, 256, 3, 0, 57976, 4)),
    ("split", "ec(2,3)", 2, 18, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 15, 1, (1, 8, 256, 3, 0, 57976, 3)),
    ("split", "ec(2,4)", 2, 17, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 16, 0, (1, 8, 512, 4, 0, 82568, 4)),
    ("split", "ec(2,4)", 2, 18, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 16, 1, (1, 8, 512, 4, 0, 82568, 3)),
    ("split", "ec(21,4)", 2, 43, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 18, 0, (1, 2, 288, 3, 0, 81528, 4)),
    ("split", "ec(21,4)", 3, 63, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 18, 1, (1, 2, 288, 3, 0, 81528, 5)),
    ("encode", "xor4", 3, 41, 1000, 4096, (), 19, 2, (1, 16, 256, 3, 0, 98936, 3)),
    ("encode", "ec(2,2)", 2, 43, 1000, 4096, (), 20, 2, (1, 21, 256, 3, 0, 110200, 3)),
    ("encode", "ec(2,3)", 3, 11, 1000, 4096, (), 21, 2, (1, 8, 256, 3, 0, 57976, 3)),
    ("encode", "ec(2,4)", 3, 11, 1000, 4096, ('LZGPU_BITSLICE=0',), 22, 2, (1, 8, 512, 4, 0, 82568, 3)),
    ("encode", "ec(21,4)", 2, 43, 1000, 4096, (), 24, 2, (1, 2, 288, 3, 0, 81528, 3)),
    ("encode", "ec(8,2)", 2, 97, 1000, 0, (), 25, 0, (1, 7, 256, 3, 0, 103032, 4)),
    ("encode", "ec(8,2)", 3, 40, 0, 0, (), 25, 1, (1, 7, 256, 3, 0, 103032, 3)),
    ("encode", "xor2", 2, 115, 1000, 0, (), 26, 0, (1, 32, 256, 3, 0, 98936, 4)),
    ("encode", "xor2", 2, 66, 0, 0, (), 26, 1, (1, 32, 256, 3, 0, 98936, 3)),
    ("encode", "xor3", 2, 106, 1000, 0, (), 27, 0, (1, 20, 256, 3, 0, 92792, 4)),
    ("encode", "xor3", 2, 63, 0, 0, (), 27, 1, (1, 20, 256, 3, 0, 92792, 3)),
    ("encode", "ec(3,2)", 2, 85, 1000, 0, (), 28, 0, (1, 16, 256, 3, 0, 107128, 4)),
    ("encode", "ec(3,2)", 3, 33, 0, 0, (), 28, 1, (1, 16, 256, 3, 0, 107128, 3)),
    ("encode", "ec(4,2)", 2, 85, 1000, 0, (), 29, 0, (1, 12, 256, 3, 0, 98936, 4)),
    ("encode", "ec(4,2)", 2, 52, 0, 0, (), 29, 1, (1, 12, 256, 3, 0, 98936, 3)),
    ("encode", "ec(6,2)", 2, 97, 1000, 0, (), 30, 0, (1, 9, 256, 3, 0, 104056, 4)),
    ("encode", "ec(6,2)", 2, 60, 0, 0, (), 30, 1, (1, 9, 256, 3, 0, 104056, 3)),
    ("encode", "ec(5,3)", 2, 71, 1000, 0, (), 31, 0, (1, 8, 256, 3, 0, 94840, 4)),
    ("encode", "ec(5,3)", 2, 45, 0, 0, (), 31, 1, (1, 8, 256, 3, 0, 94840, 3)),
    ("encode", "ec(6,3)", 2, 85, 1000, 0, (), 32, 0, (1, 8, 256, 3, 0, 107128, 4)),
    ("encode", "ec(6,3)", 2, 54, 0, 0, (), 32, 1, (1, 8, 256, 3, 0, 107128, 3)),
    ("encode", "ec(8,4)", 2, 65, 1000, 0, ('LZGPU_BITSLICE=0', 'LZGPU_STRIPED=0'), 33, 0, (1, 8, 512, 4, 0, 180872, 4)),
    ("encode", "ec(8,4)", 2, 72, 0, 0, ('LZGPU_BITSLICE=0',), 33, 1, (1, 8, 512, 4, 0, 180872, 3)),
    ("encode", "ec(8,3)", 2, 49, 1000, 0, ('LZGPU_BITSLICE=0', 'LZGPU_STRIPED=0'), 34, 0, (1, 6, 256, 3, 0, 98936, 4)),
    ("encode", "ec(8,3)", 2, 56, 0, 0, ('LZGPU_BITSLICE=0',), 34, 1, (1, 6, 256, 3, 0, 98936, 3)),
    ("encode", "xor4", 2, 113, 1000, 0, (), 35, 0, (1, 16, 256, 3, 0, 98936, 4)),
    ("encode", "xor4", 3, 44, 0, 0, (), 35, 1, (1, 16, 256, 3, 0, 98936, 3)),
    ("encode", "ec(5,2)", 2, 86, 1000, 0, (), 36, 0, (1, 10, 256, 3, 0, 97912, 4)),
    ("encode", "ec(5,2)", 3, 35, 0, 0, (), 36, 1, (1, 10, 256, 3, 0, 97912, 3)),
    ("encode", "ec(10,2)", 2, 81, 1000, 0, (), 37, 0, (1, 5, 256, 3, 0, 89720, 4)),
    ("encode", "ec(10,2)", 2, 60, 0, 0, (), 37, 1, (1, 5, 256, 3, 0, 89720, 3)),
    ("encode", "ec(4,3)", 2, 57, 1000, 0, (), 38, 0, (1, 8, 256, 3, 0, 82552, 4)),
    ("encode", "ec(4,3)", 2, 36, 0, 0, (), 38, 1, (1, 8, 256, 3, 0, 82552, 3)),
    ("encode", "ec(10,4)", 2, 61, 1000, 0, ('LZGPU_BITSLICE=0', 'LZGPU_STRIPED=0'), 39, 0, (1, 6, 512, 4, 0, 160392, 4)),
    ("encode", "ec(10,4)", 2, 70, 0, 0, ('LZGPU_BITSLICE=0',), 39, 1, (1, 6, 512, 4, 0, 160392, 3)),
    ("encode", "ec(12,4)", 2, 61, 1000, 0, ('LZGPU_BITSLICE=0', 'LZGPU_STRIPED=0'), 40, 0, (1, 5, 512, 4, 0, 156296, 4)),
    ("encode", "ec(12,4)", 2, 72, 0, 0, ('LZGPU_BITSLICE=0',), 40, 1, (1, 5, 512, 4, 0, 156296, 3)),
    ("encode", "ec(6,4)", 2, 49, 1000, 0, ('LZGPU_BITSLICE=0', 'LZGPU_STRIPED=0'), 41, 0, (1, 8, 512, 4, 0, 148104, 4)),
    ("encode", "ec(6,4)", 2, 54, 0, 0, ('LZGPU_BITSLICE=0',), 41, 1, (1, 8, 512, 4, 0, 148104, 3)),
    ("encode", "ec(4,4)", 2, 33, 1000, 0, ('LZGPU_BITSLICE=0', 'LZGPU_STRIPED=0'), 42, 0, (1, 8, 512, 4, 0, 115336, 4)),
    ("encode", "ec(4,4)", 2, 36, 0, 0, ('LZGPU_BITSLICE=0',), 42, 1, (1, 8, 512, 4, 0, 115336, 3)),
    ("encode", "ec(8,2)", 3, 33, 1000, 4096, (), 43, 2, (1, 7, 256, 3, 0, 103032, 3)),
    ("encode", "xor2", 3, 43, 1000, 4096, (), 44, 2, (1, 32, 256, 3, 0, 98936, 3)),
    ("encode", "xor3", 3, 40, 1000, 4096, (), 45, 2, (1, 20, 256, 3, 0, 92792, 3)),
    ("encode", "ec(3,2)", 3, 31, 1000, 4096, (), 46, 2, (1, 16, 256, 3, 0, 107128, 3)),
    ("encode", "ec(5,3)", 3, 26, 1000, 4096, (), 47, 2, (1, 8, 256, 3, 0, 94840, 3)),
    ("encode", "ec(8,4)", 3, 41, 1000, 4096, ('LZGPU_BITSLICE=0',), 48, 2, (1, 8, 512, 4, 0, 180872, 3)),
    ("encode", "ec(7,3)", 2, 99, 1000, 0, (), 49, 0, (2, 8, 512, 4, 4, 148104, 4)),
    ("encode", "ec(7,3)", 2, 63, 0, 0, (), 49, 1, (2, 8, 512, 4, 4, 148104, 3)),
    ("encode", "ec(2,4)", 2, 29, 1000, 0, (), 50, 0, (2, 8, 512, 4, 4, 82568, 4)),
    ("encode", "ec(2,4)", 2, 18, 0, 0, (), 50, 1, (2, 8, 512, 4, 4, 82568, 3)),
    ("encode", "ec(11,3)", 3, 23, 1000, 4096, (), 51, 2, (2, 4, 512, 4, 2, 107144, 3)),
    ("encode", "ec(2,4)", 3, 11, 1000, 4096, (), 52, 2, (2, 8, 512, 4, 4, 82568, 3)),
    ("encode", "ec(8,4)", 2, 113, 1000, 0, (), 53, 0, (2, 8, 512, 4, 4, 180872, 4)),
    ("encode", "ec(8,4)", 2, 72, 0, 0, (), 53, 1, (2, 8, 512, 4, 4, 180872, 3)),
    ("encode", "ec(10,4)", 2, 101, 1000, 0, (), 54, 0, (2, 6, 512, 4, 3, 160392, 4)),
    ("encode", "ec(10,4)", 2, 70, 0, 0, (), 54, 1, (2, 6, 512, 4, 3, 160392, 3)),
    ("encode", "ec(12,4)", 2, 97, 1000, 0, (), 55, 0, (2, 5, 512, 4, 3, 156296, 4)),
    ("encode", "ec(12,4)", 2, 72, 0, 0, (), 55, 1, (2, 5, 512, 4, 3, 156296, 3)),
    ("encode", "ec(6,4)", 2, 85, 1000, 0, (), 56, 0, (2, 8, 512, 4, 4, 148104, 4)),
    ("encode", "ec(6,4)", 2, 54, 0, 0, (), 56, 1, (2, 8, 512, 4, 4, 148104, 3)),
    ("encode", "ec(4,4)", 2, 57, 1000, 0, (), 57, 0, (2, 8, 512, 4, 4, 115336, 4)),
    ("encode", "ec(4,4)", 2, 36, 0, 0, (), 57, 1, (2, 8, 512, 4, 4, 115336, 3)),
    ("encode", "ec(8,3)", 2, 113, 1000, 0, (), 58, 0, (2, 8, 512, 4, 4, 164488, 4)),
    ("encode", "ec(8,3)", 2, 72, 0, 0, (), 58, 1, (2, 8, 512, 4, 4, 164488, 3)),
    ("encode", "ec(9,3)", 2, 91, 1000, 0, (), 59, 0, (2, 6, 512, 4, 3, 135816, 4)),
    ("encode", "ec(9,3)", 2, 63, 0, 0, (), 59, 1, (2, 6, 512, 4, 3, 135816, 3)),
    ("encode", "ec(10,3)", 2, 101, 1000, 0, (), 60, 0, (2, 6, 512, 4, 3, 148104, 4)),
    ("encode", "ec(10,3)", 2, 70, 0, 0, (), 60, 1, (2, 6, 512, 4, 3, 148104, 3)),
    ("encode", "ec(12,3)", 2, 97, 1000, 0, (), 61, 0, (2, 5, 512, 4, 3, 144008, 4)),
    ("encode", "ec(12,3)", 2, 72, 0, 0, (), 61, 1, (2, 5, 512, 4, 3, 144008, 3)),
    ("encode", "ec(8,4)", 3, 41, 1000, 4096, (), 62, 2, (2, 8, 512, 4, 4, 180872, 3)),
    ("encode", "xor5", 2, 4, 1000, 0, (), 19, 2, (1, 12, 256, 3, 0, 92792, 1)),
    ("encode", "ec(2,5)", 2, 1, 1000, 0, (), 5, 0, (1, 22, 288, 3, 0, 113272, 2)),
    ("split", "xor2", 2, 1, 0, 0, ("LZGPU_CONVERT_FUSED=0",), 13, 0, (1, 32, 256, 3, 0, 98936, 2)),
    ("encode", "ec(7,3)", 2, 6, 1000, 0, (), 51, 2, (2, 8, 512, 4, 4, 148104, 1)),
    ("crc_blocks", None, 1, 130, 0, 0, (), 0, 0, (1, 1, 256, 3, 0, 98936, 3)),
    ("crc_blocks", None, 1, 5, 0, 0, (), 0, 0, (1, 1, 256, 3, 0, 98936, 1)),
    ("verify", None, 1, 70, 0, 0, (), 0, 0, (1, 1, 256, 3, 0, 98936, 2)),
    ("crc_parts", "xor2", 3, 90, 0, 0, ('LZGPU_CONVERT_FUSED=0',), 0, 1, (1, 64, 256, 3, 0, 98936, 3)),
    ("crc_parts", "xor2", 2, 128, 0, 0, ('LZGPU_CONVERT_FUSED=0',), 0, 1, (1, 1, 256, 3, 0, 98936, 2)),
    ("crc_parts", "xor2", 3, 90, 0, 4096, ('LZGPU_CONVERT_FUSED=0',), 0, 0, (1, 1, 256, 3, 0, 98936, 3)),
]
FAMILIES = ("packed", "generic", "bitsliced", "split", "crc")


def goal_of(text):
    g = L.SliceType(text)
    return (g.kind, g.k, g.m)


def family(index):
    m, generic, bs, striped, split, kt, gt, ib = KERNELS[index]
    return "crc" if m == 0 else "split" if split else "bitsliced" if bs else "generic" if generic else "packed"


def restated(case):
    """the launches of the row's call, as route() restates them"""
    form, goal, n, nb, tail, pad, env = case[:7]
    sw = switches(env)
    if form in ("crc_blocks", "verify"):
        return route(sw, "crc", None, 1, nb, nb * BLOCK)
    if form == "crc_parts":
        pbd = -(-nb // goal_of(goal)[1])
        return route(sw, "crc", None, n, pbd, pbd * BLOCK + pad)
    return route(sw, form, goal_of(goal), n, nb, nb * BLOCK + pad)


def _case_id(case):
    form, goal, n, nb, tail, pad, env, index, mode = case[:9]
    sw = "-".join(e.replace("LZGPU_", "") for e in env if e not in CONVERT_TWO_PASS)
    return f"{form}-{goal or 'blocks'}-n{n}-nb{nb}{'-tail' if tail else ''}{'-padded' if pad else ''}{'-' + sw if sw else ''}-k{index}-mode{mode}"


def test_cases_cover_every_reachable_instantiation_and_mode():
    """every row is what the restated launcher does with it, at a shape where its unit mode breaks; together the rows hold every
    (instantiation, unit mode) pair that some call of the enumerated space records, each once"""
    recorded, _ = enumerate_routes()
    reachable = set().union(*recorded.values())
    keys = set()
    partial = {f: False for f in FAMILIES}
    short = {f: False for f in FAMILIES if f not in ("split", "crc")}
    for case in CASES:
        form, goal, n, nb, tail, pad, env, index, mode, geo = case
        calls = restated(case)
        assert calls and (calls[-1]["index"], calls[-1]["mode"], calls[-1]["geo"]) == (index, mode, geo), (case, calls and calls[-1])
        if form in ("split", "crc_parts"):
            assert "LZGPU_CONVERT_FUSED=0" in env, case
        G, units = geo[1], geo[6]
        K = 64 if form in ("crc_blocks", "verify") or (form == "crc_parts" and G == 1) else 1 if form == "crc_parts" else goal_of(goal)[1]
        rows = -(-nb // goal_of(goal)[1]) if form == "crc_parts" else nb        # blocks per run of the launch
        pb = -(-rows // K)
        fam = family(index)
        partial[fam] |= rows < K
        if fam in short:
            short[fam] |= tail > 0
        if rows >= K and form not in ("crc_blocks", "verify"):
            if mode == 0:
                assert rows % K and pb > G and (G == 1 or pb % G) or form == "crc_parts", case
            elif mode == 1:
                assert rows % K == 0 and not pad and n * pb % G and (G == 1 or pb % G) and units >= 3 or K == 64, case
            else:
                assert pad and rows % K and units >= 3, case
        key = (form, index, mode, G, rows < K)
        assert key not in keys, ("redundant row", case)
        keys.add(key)
    table = {(c[7], c[8]) for c in CASES}
    assert table == reachable, (sorted(reachable - table), sorted(table - reachable))
    assert all(partial.values()) and all(short.values()), (partial, short)
    crc = {(c[0], c[8], c[9][1]) for c in CASES if c[7] == 0}
    assert {("crc_blocks", 0, 1), ("verify", 0, 1), ("crc_parts", 1, 64), ("crc_parts", 1, 1), ("crc_parts", 0, 1)} <= crc, crc


# ---- GPU: contexts, inputs, checks -------------------------------------------------------------------------------------------------

_engines, _cache = {}, {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in _engines.values():
        e.close()
    _engines.clear()
    _cache.clear()


def engine(env):
    """one context per switch set; the switches are read when a context is created, so they are set around its creation only"""
    if env not in _engines:
        values = dict(item.split("=") for item in env)
        old = {k: os.environ.get(k) for k in values}
        os.environ.update(values)
        try:
            _engines[env] = L.Engine(0)
        finally:
            for k, v in old.items():
                if v is None:
                    del os.environ[k]
                else:
                    os.environ[k] = v
    return _engines[env]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t, dtype=np.uint8):
    return t.cpu().numpy().view(dtype)


def sentinel(shape, value=SENTINEL):
    if value == SENTINEL:
        return torch.full(shape, SENTINEL, dtype=torch.uint8, device="cuda")
    return torch.full(shape, value, dtype=torch.int32, device="cuda")


def crcs(blocks):
    return np.array([zlib.crc32(b.tobytes()) for b in blocks.reshape(-1, BLOCK)], dtype=np.uint32)


def mark(e):
    """a one-unit stripe check (a persistent launch that is no encoder kernel) first: last_encoder() must then read (-1, 0), and after
    the call under test it shows that call's launch and nothing older"""
    if "parts" not in _cache:
        _cache["parts"] = torch.zeros((3, BLOCK), dtype=torch.uint8, device="cuda")
        _cache["verdict"] = torch.zeros(16, dtype=torch.int32, device="cuda")
    parts = _cache["parts"]
    e.check_stripes_dev(L.SliceType("xor2"), 1, 2, [parts[i].data_ptr() for i in range(3)], BLOCK, None, _cache["verdict"].data_ptr())
    assert e.last_encoder() == (-1, 0) and e.last_geometry()["kernel"] == _lib.KERNEL_CHECK


def check_launch(e, case, cap):
    index, mode, (kernel, G, thr, stages, gf_warps, smem, units) = case[7:]
    assert e.last_encoder() == (index, mode), (e.last_encoder(), KERNELS[index])
    g = e.last_geometry()
    want = dict(kernel=kernel, G=G, threads=thr, stages=stages, gf_warps=gf_warps, smem_bytes=smem, units=units)
    assert {k: g[k] for k in want} == want, (g, want)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    assert g["grid"] == min(units, 2 if cap else sm * (1 if thr > 320 else 2)), (g, cap)


def contexts(case):
    return [(case[6], False), (case[6] + ("LZGPU_GRID_CAP=2",), True)]


def rnd(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, size=shape, dtype=np.uint8)


def run_encode(oracle, case):
    form, text, n, nb, tail, pad = case[:6]
    goal = L.SliceType(text)
    k, m = goal.k, goal.m
    pb, chunk_len, stride = -(-nb // k), nb * BLOCK - tail, nb * BLOCK + pad
    data = rnd((n, stride), zlib.crc32(repr(case).encode()))
    data[:, chunk_len:] = GARBAGE
    ref = [oracle.encode_chunk(goal.kind, k, m, data[c, :chunk_len]) for c in range(n)]
    par_bytes, n_crc = m * pb * BLOCK, nb + m * pb
    par_stride, crc_stride = par_bytes + PAD, n_crc + 5
    for env, cap in contexts(case):
        e = engine(env)
        d_data, d_par, d_crc = dev(data), sentinel((n, par_stride)), sentinel((n, crc_stride), SENTINEL_CRC)
        torch.cuda.synchronize()
        mark(e)
        before = e.stats()["kernel_launches"]
        e.encode_chunks_dev(goal, n, chunk_len, d_data.data_ptr(), stride, d_par.data_ptr(), par_stride, d_crc.data_ptr(), crc_stride)
        assert e.stats()["kernel_launches"] - before == len(restated(case))        # every pass on the fused route, nothing else
        check_launch(e, case, cap)
        e.sync()
        par, crc, img = host(d_par).reshape(n, par_stride), host(d_crc, np.uint32).reshape(n, crc_stride), host(d_data).reshape(n, stride)
        for c in range(n):
            bad = [r for r in range(m) if (par[c, r * pb * BLOCK:(r + 1) * pb * BLOCK] != ref[c][0][r]).any()]
            assert not bad, (cap, c, "parity rows", bad)
            assert (crc[c, :n_crc] == ref[c][1]).all(), (cap, c, np.flatnonzero(crc[c, :n_crc] != ref[c][1])[:8])
        assert (par[:, par_bytes:] == SENTINEL).all() and (crc[:, n_crc:] == SENTINEL_CRC).all(), (cap, "stride padding written")
        assert (img[:, :chunk_len] == data[:, :chunk_len]).all(), cap
        assert (img[:, chunk_len:nb * BLOCK] == 0).all(), (cap, "the trailing partial block is not zero-filled")
        assert (img[:, nb * BLOCK:] == GARBAGE).all(), (cap, "data stride padding written")


def convert(e, dst, image, n, nb, pad, want, out_pad=0, fused=True):
    """the conversion of n standard chunks (image [n, nb * B + pad]) into dst: every destination part and CRC array sentinel-filled,
    wanted or not (fused = False: a context that launches no persistent kernel).  Returns their host copies."""
    nd, pbd = dst.k + dst.m, -(-nb // dst.k)
    outs = [sentinel((n, pbd * BLOCK + out_pad)) for _ in range(nd)]
    ocrc = [sentinel((n, pbd), SENTINEL_CRC) for _ in range(nd)]
    d_img = dev(image)
    torch.cuda.synchronize()
    if fused:
        mark(e)
    e.convert_chunks_dev(L.SliceType(2, 1, 0), dst, n, nb, [d_img.data_ptr()], nb * BLOCK + pad, want, [t.data_ptr() for t in outs],
                         pbd * BLOCK + out_pad, d_out_crc=[t.data_ptr() for t in ocrc])
    e.sync()
    return [host(t).reshape(n, -1) for t in outs], [host(t, np.uint32).reshape(n, -1) for t in ocrc]


def expected_parts(oracle, dst, image, nb):
    """per destination part [n, pbd * B] and its block CRCs [n, pbd]: the oracle's split (zero-padded data parts) and encode"""
    n, kd, md = image.shape[0], dst.k, dst.m
    per = [O.split_parts(image[c, :nb * BLOCK], kd)[0] + list(oracle.encode_chunk(dst.kind, kd, md, image[c, :nb * BLOCK])[0]) for c in range(n)]
    parts = [np.stack([per[c][i] for c in range(n)]) for i in range(kd + md)]
    return parts, [np.stack([crcs(p[c]) for c in range(n)]) for p in parts]


def assert_parts(got, want, parts, pcrc, what, out_pad=0):
    out, ocrc = got
    for i, w in enumerate(want):
        if w:
            assert (out[i][:, :parts[i].shape[1]] == parts[i]).all(), (what, "part", i)
            assert (out[i][:, parts[i].shape[1]:] == SENTINEL).all(), (what, "stride padding of part", i)
            assert (ocrc[i] == pcrc[i]).all(), (what, "CRCs of part", i, np.argwhere(ocrc[i] != pcrc[i])[:4].tolist())
        else:
            assert (out[i] == SENTINEL).all() and (ocrc[i] == SENTINEL_CRC).all(), (what, "unwanted part written", i)


def run_split(oracle, case):
    form, text, n, nb, tail, pad = case[:6]
    dst = L.SliceType(text)
    kd, nd = dst.k, dst.k + dst.m
    image = rnd((n, nb * BLOCK + pad), zlib.crc32(repr(case).encode()))
    parts, pcrc = expected_parts(oracle, dst, image, nb)
    every = [1] * nd
    subset = [1 if (i < kd and i % 2 == 0) or i == nd - 1 else 0 for i in range(nd)]   # a parity part must be wanted
    plain = convert(engine(CONVERT_TWO_PASS + ("LZGPU_DISABLE_FUSED=1",)), dst, image, n, nb, pad, every, fused=False)
    assert_parts(plain, every, parts, pcrc, "generic route")
    for env, cap in contexts(case):
        e = engine(env)
        for want in (every, subset):
            got = convert(e, dst, image, n, nb, pad, want)
            check_launch(e, case, cap)
            assert_parts(got, want, parts, pcrc, (cap, want))
            if want is every:
                assert all((g == p).all() for g, p in zip(got[0] + got[1], plain[0] + plain[1])), cap


def run_crc(oracle, case):
    form, text, n, nb, tail, pad = case[:6]
    for env, cap in contexts(case):
        e = engine(env)
        seed = zlib.crc32(repr(case).encode())
        if form == "crc_parts":
            dst = L.SliceType(text)
            image = rnd((n, nb * BLOCK), seed)
            parts, pcrc = expected_parts(oracle, dst, image, nb)
            want = [1] * dst.k + [0] * dst.m
            got = convert(e, dst, image, n, nb, 0, want, out_pad=pad)
            check_launch(e, case, cap)
            assert_parts(got, want, parts, pcrc, cap, out_pad=pad)
            continue
        data = rnd((nb, BLOCK), seed)
        ref = crcs(data)
        if form == "crc_blocks":
            d_data, d_out = dev(data), sentinel((nb + 4,), SENTINEL_CRC)
            torch.cuda.synchronize()
            mark(e)
            e.crc_blocks_dev(d_data.data_ptr(), nb, d_out.data_ptr())
            check_launch(e, case, cap)
            e.sync()
            out = host(d_out, np.uint32)
            assert (out[:nb] == ref).all() and (out[nb:] == SENTINEL_CRC).all(), (cap, np.flatnonzero(out[:nb] != ref)[:8])
        else:
            mark(e)
            e.verify_blocks(data, ref)
            check_launch(e, case, cap)
            bad = ref.copy()
            bad[nb // 2] ^= 0x00000100
            with pytest.raises(L.ChunkCrcError):
                e.verify_blocks(data, bad)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_case_id(c) for c in CASES])
def test_encoder_instantiation_vs_oracle(oracle, case):
    {"encode": run_encode, "split": run_split}.get(case[0], run_crc)(oracle, case)
