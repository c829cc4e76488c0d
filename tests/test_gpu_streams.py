"""Every device-pointer entry point keeps to its caller's stream: gated streams, many threads on one context, deferred verification.

include/lzgpu.h promises, for the *_dev calls: all work of a call is enqueued on the caller's `stream` (the call waits only to
report a stored-CRC verdict); any number of threads may call them on one context at once; in deferred mode the verdicts are
collected by lzgpu_dev_sync.  A test that calls with stream=None and then synchronises the device cannot see a launch, memset,
temporary or result copy that went to the context's stream instead, so here:

  - ROWS is one table of every *_dev entry point: a small seeded request of a few chunks with ragged block counts, its input and
    output buffers (each a device allocation with random guard bytes around it), and the oracle's answer where the suite has one.
    The stripe rows carry planted faults, so that the correction, repair and decode really write into the parts.
  - The baseline of a request is the call on a context of its own, inputs synchronised, stream=None; it must equal the oracle and
    leave every guard and every input it does not write as it was.
  - Gated: the buffers hold a decoy (another seed, with matching CRCs; other sentinels in the outputs), a fresh stream sleeps
    GATE_MS and then copies the real inputs and sentinels in, the call is made on that stream, and copies of every buffer are
    enqueued behind it.  Work that ran on any other stream reads the decoy or is overwritten by the sentinels, so each copy must
    equal the baseline byte for byte.  A call that does not wait must return while the gate still holds its stream; one that
    verifies stored CRCs must block until the gate has passed.
  - Threads: eight threads share one context, each on its own stream, walking the table in its own order with its own goals and
    seeds, with host-pointer calls mixed in and one planted stored-CRC mismatch per round.
  - Deferred: mismatches are reported once, by one lzgpu_dev_sync, also when the call that found one was enqueued by another thread
    while that sync was already waiting for the device, and when the call's stream was destroyed before the sync.

Every case runs on the default context and on one with LZGPU_DISABLE_FUSED=1 (the generic route: the most launches, memsets and
temporaries per call)."""
import ctypes
import os
import threading
import time
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
N = 3                      # chunks per request
GATE_MS = 100              # how long a gate holds its stream
SENTINEL, DECOY_SENTINEL = 0xA5, 0x5A
CONTEXTS = {"default": {}, "generic": {"LZGPU_DISABLE_FUSED": "1"}}

_engines = {}
_base = {}
_gate = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in _engines.values():
        e.close()
    _engines.clear()
    _base.clear()


def new_engine(ctx):
    """a context of its own; the switches are read when a context is created, so they are set around its creation only"""
    env = CONTEXTS[ctx]
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return L.Engine(0)
    finally:
        for k, v in old.items():
            if v is None:
                del os.environ[k]
            else:
                os.environ[k] = v


def engine(ctx, role):
    if (ctx, role) not in _engines:
        _engines[(ctx, role)] = new_engine(ctx)
    return _engines[(ctx, role)]


def rnd(nbytes, seed):
    return np.frombuffer(np.random.default_rng(seed).bytes(nbytes), dtype=np.uint8).copy()


def u8(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(-1)


def block_crcs(a):
    """zlib CRC of every 64 KiB block of every row of a [n, blocks * 64 KiB] array"""
    return np.array([[zlib.crc32(r[b * BLOCK:(b + 1) * BLOCK].tobytes()) for b in range(r.size // BLOCK)] for r in a], dtype=np.uint32)


def gate_cycles():
    """GPU clock cycles of torch.cuda._sleep that take GATE_MS, measured with CUDA events"""
    if "cycles" not in _gate:
        s = torch.cuda.Stream()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(s):
            torch.cuda._sleep(1_000_000)
            e0.record()
            torch.cuda._sleep(50_000_000)
            e1.record()
        e1.synchronize()
        _gate["cycles"] = int(50_000_000 / e0.elapsed_time(e1) * GATE_MS)
    return _gate["cycles"]


def gate(stream, ms=GATE_MS):
    with torch.cuda.stream(stream):
        torch.cuda._sleep(gate_cycles() * ms // GATE_MS)


# ---- the table -----------------------------------------------------------------------------------------------------------------

class Req:
    """One request: its buffers (name -> initial region bytes, None for an output; size; whether the call may write it), the call
    (call(engine, ptr, stream) with ptr(name) = the device address of a buffer's region), the oracle's answer for the regions it
    knows (expect), whether the call verifies stored CRCs (and so waits for its stream), and one stored CRC to corrupt with the
    position the mismatch is reported at (site = (buffer, element, where), where_deferred as lzgpu_last_bad reports it)."""

    def __init__(self):
        self.bufs, self.expect = {}, {}
        self.call, self.check = None, None
        self.verifies, self.site, self.where_deferred = False, None, None

    def inp(self, name, arr, written=False, expect=None):
        b = u8(arr).copy()
        self.bufs[name] = (b, b.size, written)
        if expect is not None:
            self.expect[name] = u8(expect)

    def out(self, name, nbytes, expect=None):
        self.bufs[name] = (None, nbytes, True)
        if expect is not None:
            self.expect[name] = u8(expect)

    def region(self, name, decoy=None):
        data, size, _ = self.bufs[name]
        if data is None:
            return np.full(size, SENTINEL if decoy is None else DECOY_SENTINEL, dtype=np.uint8)
        return data if decoy is None else decoy.bufs[name][0]

    def corrupted(self):
        """the same request with the stored CRC at `site` off by one bit"""
        name, elem, _ = self.site
        r = Req()
        r.__dict__.update(self.__dict__)
        r.bufs = dict(self.bufs)
        data = self.bufs[name][0].copy()
        data[4 * elem] ^= 0x01
        r.bufs[name] = (data,) + self.bufs[name][1:]
        return r


def coded(oracle, text, data):
    """the k + m parts [n, pb * 64K] of chunks data [n, nb * 64K] (data parts zero-padded) and their block CRCs [n, pb]"""
    goal = L.SliceType(2, 1, 0) if text == "std" else L.SliceType(text)
    if goal.is_std:
        return goal, [data], [block_crcs(data)]
    k, m = goal.k, goal.m
    enc = [oracle.encode_chunk(goal.kind, k, m, data[c]) for c in range(len(data))]
    per = [O.split_parts(data[c], k)[0] for c in range(len(data))]
    parts = [np.stack([per[c][j] for c in range(len(data))]) for j in range(k)]
    parts += [np.stack([enc[c][0][r] for c in range(len(data))]) for r in range(m)]
    return goal, parts, [block_crcs(p) for p in parts]


def chunks(nb, seed):
    return rnd(N * nb * BLOCK, seed).reshape(N, nb * BLOCK)


def stale(parts, crcs, p, c, s):
    """block s of part p in chunk c rewritten, with a stored CRC that matches the new bytes (a stale part)"""
    parts[p][c, s * BLOCK + 100: s * BLOCK + 108] ^= np.arange(1, 9, dtype=np.uint8)
    crcs[p][c, s] = zlib.crc32(parts[p][c, s * BLOCK:(s + 1) * BLOCK].tobytes())


def rot(parts, p, c, s):
    """block s of part p in chunk c rewritten under its old stored CRC (bit rot)"""
    parts[p][c, s * BLOCK + 321: s * BLOCK + 324] ^= 0xFF


def part_site(crcs, lost, pb, c=1, b=1, first=1):
    """a stored CRC of the first given part from `first` on, at chunk c, block b"""
    p = next(i for i in range(first, len(crcs)) if i not in lost)
    return (f"c{p}", c * pb + b, (c, p, b))


def given_parts(r, parts, crcs, lost, written=False, expect=None):
    for i in range(len(parts)):
        if i not in lost:
            r.inp(f"p{i}", parts[i], written, None if expect is None else expect[i])
            r.inp(f"c{i}", crcs[i])


def ptrs(p, prefix, n, skip=()):
    return [0 if i in skip else p(f"{prefix}{i}") for i in range(n)]


def row_encode(oracle, v, seed):
    text, nb, short = [("ec(8,2)", 13, 1000), ("ec(5,3)", 11, 0)][v]
    goal = L.SliceType(text)
    k, m, pb = goal.k, goal.m, -(-nb // goal.k)
    clen, n_crc = nb * BLOCK - short, nb + m * pb
    data = chunks(nb, seed)
    filled = data.copy()
    filled[:, clen:] = 0                               # the rest of a partial last block is zero-filled in place
    enc = [oracle.encode_chunk(goal.kind, k, m, data[c, :clen]) for c in range(N)]
    r = Req()
    r.inp("data", data, written=short > 0, expect=filled)
    r.out("parity", N * m * pb * BLOCK, np.stack([e[0] for e in enc]))
    r.out("crc", N * n_crc * 4, np.stack([e[1] for e in enc]))
    r.call = lambda e, p, s: e.encode_chunks_dev(goal, N, clen, p("data"), nb * BLOCK, p("parity"), m * pb * BLOCK, p("crc"), n_crc,
                                                 stream=s)
    return r


def row_encode_slices(oracle, v, seed):
    names, nb = [(("std", "xor2", "xor3"), 14), (("ec(3,2)", "ec(8,2)"), 26)][v]
    data = chunks(nb, seed)
    r = Req()
    r.inp("data", data)
    goals, pst, cst = [], [], []
    for i, text in enumerate(names):
        goal, parts, crcs = coded(oracle, text, data)
        goals.append(goal)
        if goal.is_std:
            r.out(f"crc{i}", N * nb * 4, crcs[0])
            pst.append(0)
            cst.append(nb)
            continue
        k, m, pb = goal.k, goal.m, -(-nb // goal.k)
        r.out(f"par{i}", N * m * pb * BLOCK, np.concatenate(parts[k:], axis=1))
        chunk_crcs = block_crcs(data)
        r.out(f"crc{i}", N * (nb + m * pb) * 4, np.concatenate([chunk_crcs] + crcs[k:], axis=1))
        pst.append(m * pb * BLOCK)
        cst.append(nb + m * pb)
    par = lambda p: [0 if g.is_std else p(f"par{i}") for i, g in enumerate(goals)]
    r.call = lambda e, p, s: e.encode_slices_dev(goals, N, nb * BLOCK, p("data"), nb * BLOCK, par(p), pst,
                                                 [p(f"crc{i}") for i in range(len(goals))], cst, stream=s)
    return r


def row_recover(oracle, v, seed):
    text, lost, nb = [("ec(8,2)", (1, 4), 21), ("ec(5,3)", (0, 2), 17)][v]
    data = chunks(nb, seed)
    goal, parts, crcs = coded(oracle, text, data)
    n, pb = goal.k + goal.m, -(-nb // goal.k)
    r = Req()
    given_parts(r, parts, crcs, lost)
    for i in lost:
        r.out(f"o{i}", N * pb * BLOCK, parts[i])
    r.out("image", N * nb * BLOCK, data)
    r.verifies, r.site = True, part_site(crcs, lost, pb)
    r.where_deferred = r.site[2]
    want = [int(i in lost) for i in range(n)]
    r.call = lambda e, p, s: e.recover_chunks_dev(goal, N, nb, ptrs(p, "p", n, lost), pb * BLOCK, ptrs(p, "c", n, lost), want,
                                                  [p(f"o{i}") if i in lost else 0 for i in range(n)], p("image"), nb * BLOCK, stream=s)
    return r


def row_recover_slices(oracle, v, seed):
    names, given, nb = [(("xor2", "xor3"), (0, 1, 3, 5), 13), (("xor2", "xor3"), (1, 2, 3, 4), 17)][v]
    data = chunks(nb, seed)
    goals, parts, crcs, slice_of, pbs = [], [], [], [], []
    for i, text in enumerate(names):
        goal, pp, cc = coded(oracle, text, data)
        goals.append(goal)
        parts += pp
        crcs += cc
        slice_of += [i] * len(pp)
        pbs.append(-(-nb // goal.k))
    n = len(parts)
    lost = [g for g in range(n) if g not in given]
    assert L.Engine.plan_recover_slices(goals, nb, [int(g in given) for g in range(n)])["ok"] == 1
    r = Req()
    given_parts(r, parts, crcs, lost)
    for g in lost:
        r.out(f"o{g}", N * pbs[slice_of[g]] * BLOCK, parts[g])
        r.out(f"oc{g}", N * pbs[slice_of[g]] * 4, crcs[g])
    r.out("image", N * nb * BLOCK, data)
    g = given[2]
    first = slice_of.index(slice_of[g])
    r.verifies = True
    r.site = (f"c{g}", 2 * pbs[slice_of[g]] + 1, (2, slice_of[g], g - first, 1))
    r.where_deferred = (2, g, 1)
    stride = [pb * BLOCK for pb in pbs]
    want = [int(g in lost) for g in range(n)]
    r.call = lambda e, p, s: e.recover_slices_dev(goals, N, nb, ptrs(p, "p", n, lost), stride, ptrs(p, "c", n, lost), want,
                                                  [p(f"o{g}") if g in lost else 0 for g in range(n)], stride,
                                                  [p(f"oc{g}") if g in lost else 0 for g in range(n)], p("image"), nb * BLOCK, stream=s)
    return r


def convert_row(oracle, src_text, lost, nb, dst_text, seed, one_pass):
    data = chunks(nb, seed)
    src, parts, crcs = coded(oracle, src_text, data)
    dst = L.SliceType(dst_text)
    ns, nd = src.k + src.m, dst.k + dst.m
    pbs, pbd = -(-nb // src.k), -(-nb // dst.k)
    want = [1] * nd
    if not src.is_std:
        assert L.Engine.plan_convert(src, dst, [int(i not in lost) for i in range(ns)], want)["one_pass"] == one_pass
    ref = [O.convert_chunk(oracle, (src.kind, src.k, src.m), [None if i in lost else parts[i][c] for i in range(ns)],
                           [None if i in lost else crcs[i][c] for i in range(ns)], (dst.kind, dst.k, dst.m), want, nb) for c in range(N)]
    assert all(x[0] == 0 for x in ref)
    r = Req()
    given_parts(r, parts, crcs, lost)
    for i in range(nd):
        r.out(f"o{i}", N * pbd * BLOCK, np.stack([x[1][i] for x in ref]))
        r.out(f"oc{i}", N * pbd * 4, np.stack([x[2][i] for x in ref]))
    r.verifies = True
    r.site = part_site(crcs, lost, pbs, first=0 if src.is_std else 1)
    r.where_deferred = r.site[2]
    r.call = lambda e, p, s: e.convert_chunks_dev(src, dst, N, nb, ptrs(p, "p", ns, lost), pbs * BLOCK, want, ptrs(p, "o", nd), pbd * BLOCK,
                                                  d_part_crc=ptrs(p, "c", ns, lost), d_out_crc=ptrs(p, "oc", nd), stream=s)
    return r


def row_convert_one_pass(oracle, v, seed):
    return convert_row(oracle, *[("ec(8,2)", (1, 4), 25, "ec(3,2)"), ("ec(8,2)", (3,), 19, "ec(3,2)")][v], seed, one_pass=1)


def row_convert_two_pass(oracle, v, seed):
    return convert_row(oracle, *[("ec(5,3)", (0, 2, 4), 24, "ec(3,2)"), ("std", (), 20, "ec(3,2)")][v], seed, one_pass=0)


# stripe rows: (goal, lost parts, blocks, stale blocks, rotten blocks), each block (part, chunk, stripe)
CHECKED = [("ec(5,3)", (), 17, [(2, 1, 1)], []), ("ec(8,3)", (), 29, [(9, 0, 2)], [])]
DEGRADED = [("ec(5,3)", (1,), 17, [(3, 2, 0)], []), ("ec(8,4)", (2,), 29, [(5, 0, 1)], [])]
REPAIRED = [("ec(8,2)", (), 21, [], [(3, 1, 1)]), ("xor3", (), 13, [], [(1, 2, 0)])]
DECODED = [("ec(8,4)", (), 21, [(2, 0, 1), (6, 0, 1)], []), ("ec(8,3)", (), 29, [(1, 2, 0)], [(5, 2, 0)])]


def stripe_row(oracle, case, seed, result, entry, status=None, in_place=False, verifies=True):
    """a batch with planted faults.  result(e) = the Engine method, entry = bytes per map / fix entry (per chunk for the verdicts);
    an in-place call must leave the pristine parts and the status `status` in the faulted stripe's entry, CLEAN elsewhere"""
    text, lost, nb, stale_blocks, rotten = case
    data = chunks(nb, seed)
    goal, parts, crcs = coded(oracle, text, data)
    n, pb = goal.k + goal.m, -(-nb // goal.k)
    pristine = [q.copy() for q in parts]
    for f in stale_blocks:
        stale(parts, crcs, *f)
    for f in rotten:
        rot(parts, *f)
    r = Req()
    given_parts(r, parts, crcs, lost, written=in_place, expect=pristine if in_place else None)
    per_chunk = entry == 12
    r.out("res", N * (1 if per_chunk else pb) * entry)
    faults = stale_blocks + rotten
    p0, c0, s0 = faults[0]

    def check(got):
        res = got["res"].view(np.int32).reshape(N, -1, entry // 4)
        if per_chunk:                          # verdicts: first_bad_stripe, bad_rows, suspect_part
            assert [int(x) for x in res[:, 0, 0]] == [s0 if c == c0 else -1 for c in range(N)], res[:, 0]
            assert res[c0, 0, 2] == p0, res[c0]
            return
        if status is None:                     # map: bad_rows, suspect_part
            assert res[c0, s0, 1] == p0 and res[c0, s0, 0] != 0, res[c0, s0]
        else:
            assert res[c0, s0, 2] == status, res[c0, s0]
        bad = res[..., 0] != 0
        bad[c0, s0] = False
        assert not bad.any(), np.argwhere(bad)

    r.check = check
    if verifies:
        r.verifies, r.site = True, part_site(crcs, lost, pb, c=2, b=1, first=0)
        r.where_deferred = r.site[2]
    r.call = lambda e, p, s: result(e)(goal, N, nb, ptrs(p, "p", n, lost), pb * BLOCK, ptrs(p, "c", n, lost), p("res"), stream=s)
    return r


def row_check_stripes(oracle, v, seed):
    return stripe_row(oracle, CHECKED[v], seed, lambda e: e.check_stripes_dev, 12)


def row_check_stripe_map(oracle, v, seed):
    return stripe_row(oracle, CHECKED[v], seed, lambda e: e.check_stripe_map_dev, 8)


def row_correct_stripes(oracle, v, seed):
    return stripe_row(oracle, CHECKED[v], seed, lambda e: e.correct_stripes_dev, 16, _lib.FIX_CORRECTED, in_place=True)


def row_check_stripe_map_degraded(oracle, v, seed):
    return stripe_row(oracle, DEGRADED[v], seed, lambda e: e.check_stripe_map_degraded_dev, 8)


def row_correct_stripes_degraded(oracle, v, seed):
    return stripe_row(oracle, DEGRADED[v], seed, lambda e: e.correct_stripes_degraded_dev, 16, _lib.FIX_CORRECTED, in_place=True)


def row_repair_stripes(oracle, v, seed):
    return stripe_row(oracle, REPAIRED[v], seed, lambda e: e.repair_stripes_dev, 24, _lib.FIX_REBUILT, in_place=True, verifies=False)


def row_decode_stripes(oracle, v, seed):
    return stripe_row(oracle, DECODED[v], seed, lambda e: e.decode_stripes_dev, 40, _lib.FIX_DECODED, in_place=True, verifies=False)


def row_split(oracle, v, seed):
    text, nb = [("ec(3,2)", 20), ("ec(8,2)", 19)][v]
    data = chunks(nb, seed)
    goal, parts, _ = coded(oracle, text, data)
    k, pb = goal.k, -(-nb // goal.k)
    r = Req()
    r.inp("data", data)
    for j in range(k):
        r.out(f"o{j}", N * pb * BLOCK, parts[j])
    r.call = lambda e, p, s: e.split_chunks_dev(goal, N, nb, p("data"), nb * BLOCK, ptrs(p, "o", k), pb * BLOCK, stream=s)
    return r


def row_prefixes(oracle, v, seed):
    text, nb = [("ec(5,3)", 23), ("xor3", 10)][v]
    goal = L.SliceType(text)
    k, m, pb = goal.k, goal.m, -(-nb // goal.k)
    n_crc, base = nb + m * pb, 1000 + 7 * v
    crc = np.frombuffer(rnd(N * n_crc * 4, seed), dtype=np.uint32).reshape(N, n_crc)
    ids = np.frombuffer(rnd(N * 8, seed + 1), dtype=np.uint64)
    want = np.zeros((N, k + m, pb, _lib.WRITE_PREFIX_SIZE), dtype=np.uint8)
    for c in range(N):
        for part in range(k + m):
            for s in range(pb):
                if part < k and s * k + part >= nb:
                    continue                           # a block a short data part does not have: 38 zero bytes
                x = int(crc[c, s * k + part]) if part < k else int(crc[c, nb + (part - k) * pb + s])
                want[c, part, s] = O.write_data_prefix(oracle, int(ids[c]), base + (c * (k + m) + part) * pb + s, s, 0, BLOCK, x)
    r = Req()
    r.inp("crc", crc)
    r.inp("ids", ids)
    r.out("out", want.size, want)
    r.call = lambda e, p, s: e.write_data_prefixes_dev(goal, N, nb, p("crc"), n_crc, p("ids"), p("out"), write_id_base=base, stream=s)
    return r


def row_crc_blocks(oracle, v, seed):
    block_len, stride, n = [(BLOCK, BLOCK, 40), (4000, 4100, 60)][v]
    blocks = rnd((n - 1) * stride + block_len, seed)
    r = Req()
    r.inp("blocks", blocks)
    r.out("crc", n * 4, np.array([zlib.crc32(blocks[b * stride: b * stride + block_len].tobytes()) for b in range(n)], dtype=np.uint32))
    r.call = lambda e, p, s: e.crc_blocks_dev(p("blocks"), n, p("crc"), block_len=block_len, block_stride=stride, stream=s)
    return r


def row_write_blocks(oracle, v, seed):
    shapes = [[(0, BLOCK), (0, 1), (1, 65535), (100, 1000), (7, 4097), (32768, 32768), (65533, 3)],
              [(12345, 1), (0, 4096), (60000, 5536), (0, BLOCK), (3, 0)]][v]
    rng = np.random.default_rng(seed)
    n = len(shapes)
    blocks = np.frombuffer(rng.bytes(n * BLOCK), dtype=np.uint8).reshape(n, BLOCK).copy()
    stored = block_crcs(blocks.reshape(1, -1))[0]
    recs = (_lib.LzBlockWrite * n)()
    payload, pos = [], 1
    for i, (off, size) in enumerate(shapes):
        data = np.frombuffer(rng.bytes(size), dtype=np.uint8)
        recs[i].block, recs[i].offset, recs[i].size = i, off, size
        recs[i].crc = zlib.crc32(data.tobytes()) ^ (0x40 if i == 3 else 0)        # request 3 carries a corrupt packet
        recs[i].payload_off, recs[i].exists, recs[i].status = pos, int(i != 0), 0
        payload.append((pos, data))
        pos += size + 3
    pay = rnd(pos, seed + 1)
    for p0, data in payload:
        pay[p0:p0 + data.size] = data
    new_blocks, new_stored = blocks.copy(), stored.copy()
    done = (_lib.LzBlockWrite * n).from_buffer_copy(bytes(recs))
    code = {0: 0, -3: _lib.ERR_CRC, -4: _lib.ERR_DAMAGED, -1: _lib.ERR_ARG}
    for i, (off, size) in enumerate(shapes):
        rc, blk, crc = O.hdd_write_block(oracle, blocks[i] if recs[i].exists else None, int(stored[i]), off, size, recs[i].crc,
                                         payload[i][1] if size else np.zeros(1, np.uint8))
        done[i].status = code[rc]
        if rc == 0:
            new_blocks[i], new_stored[i] = blk, crc
    r = Req()
    r.inp("blocks", blocks, written=True, expect=new_blocks)
    r.inp("stored", stored, written=True, expect=new_stored)
    r.inp("payload", pay)
    r.inp("writes", np.frombuffer(bytes(recs), dtype=np.uint8), written=True, expect=np.frombuffer(bytes(done), dtype=np.uint8))
    r.call = lambda e, p, s: e.write_blocks_dev(p("blocks"), p("stored"), p("payload"), p("writes"), n, stream=s)
    return r


def row_fill(oracle, v, seed):
    n, clen, gap = [(4, 3 * BLOCK + 104, 4104), (2, 5 * BLOCK, 8)][v]
    cs = clen + gap
    want = np.full((n - 1) * cs + clen, SENTINEL, dtype=np.uint8)           # the stride gaps are not written
    for c in range(n):
        want[c * cs: c * cs + clen] = O.fill_chunk(oracle, clen, seed, 5 + c)
    r = Req()
    r.out("chunks", want.size, want)
    r.call = lambda e, p, s: e.fill_chunks_dev(p("chunks"), n, clen, cs, seed, first_chunk=5, stream=s)
    return r


ROWS = {
    "encode_chunks": row_encode, "encode_slices": row_encode_slices, "recover_chunks": row_recover, "recover_slices": row_recover_slices,
    "convert_one_pass": row_convert_one_pass, "convert_two_pass": row_convert_two_pass, "check_stripes": row_check_stripes,
    "check_stripe_map": row_check_stripe_map, "correct_stripes": row_correct_stripes,
    "check_stripe_map_degraded": row_check_stripe_map_degraded, "correct_stripes_degraded": row_correct_stripes_degraded,
    "repair_stripes": row_repair_stripes, "decode_stripes": row_decode_stripes, "split_chunks": row_split,
    "write_data_prefixes": row_prefixes, "crc_blocks": row_crc_blocks, "write_blocks": row_write_blocks, "fill_chunks": row_fill,
}
VERIFYING = ["recover_chunks", "recover_slices", "convert_one_pass", "convert_two_pass", "check_stripes", "check_stripe_map",
             "correct_stripes", "check_stripe_map_degraded", "correct_stripes_degraded"]
# the verifying rows whose chunk counters do not depend on the verdict (the two-pass conversion may stop after its first pass)
CORRUPTIBLE = [n for n in VERIFYING if not n.startswith("convert")]


# ---- running a request ---------------------------------------------------------------------------------------------------------

def guard_bytes(name, end):
    return rnd(GUARD, zlib.crc32(f"{name}/{end}".encode()))


class Bufs:
    """the device allocations of one call: per buffer GUARD random bytes, the region, GUARD random bytes, made on the current stream"""

    def __init__(self, req, decoy=None):
        self.t = {}
        for name, (_, size, _) in req.bufs.items():
            a = np.concatenate([guard_bytes(name, 0), req.region(name, decoy), guard_bytes(name, 1)])
            self.t[name] = torch.from_numpy(a).cuda()

    def ptr(self, name):
        return self.t[name].data_ptr() + GUARD

    def region(self, name):
        return self.t[name][GUARD:-GUARD]


def run(e, req, stream):
    """the call on `stream` (None: the context's stream, then lzgpu_dev_sync): (every allocation as a numpy array, ChunkCrcError.where
    or None)"""
    with torch.cuda.stream(stream or torch.cuda.current_stream()):
        b = Bufs(req)
        if stream is None:
            torch.cuda.synchronize()
        where = None
        try:
            req.call(e, b.ptr, None if stream is None else stream.cuda_stream)
        except L.ChunkCrcError as ex:
            where = ex.where
        if stream is None:
            e.sync()
        return {n: t.cpu().numpy() for n, t in b.t.items()}, where


def baseline(ctx, name, v, seed, oracle):
    """(request, the allocations after the ungated call, its chunks_encoded / chunks_recovered), checked against the oracle once"""
    key = (ctx, name, v, seed)
    if key not in _base:
        req = ROWS[name](oracle, v, seed)
        e = engine(ctx, "baseline")
        s0 = e.stats()
        got, where = run(e, req, None)
        s1 = e.stats()
        assert where is None, (name, v, where)
        regions = {}
        for n, (data, size, written) in req.bufs.items():
            a = got[n]
            assert (a[:GUARD] == guard_bytes(n, 0)).all() and (a[-GUARD:] == guard_bytes(n, 1)).all(), f"{name}: guard of {n} written"
            regions[n] = a[GUARD:-GUARD]
            if not written:
                assert (regions[n] == data).all(), f"{name}: input {n} written"
            if n in req.expect:
                bad = np.flatnonzero(regions[n] != req.expect[n])
                assert bad.size == 0, f"{name} v{v} ({ctx}): {n} differs from the oracle at {bad.size} bytes, the first at {bad[0]}"
        if req.check:
            req.check(regions)
        counts = (s1["chunks_encoded"] - s0["chunks_encoded"], s1["chunks_recovered"] - s0["chunks_recovered"])
        _base[key] = (req, got, counts)
    return _base[key]


def differences(got, want):
    out = []
    for n, a in want.items():
        bad = np.flatnonzero(got[n] != a)
        if bad.size:
            out.append(f"{n}: {bad.size} bytes, the first at {int(bad[0]) - GUARD} from the region start")
    return out


# ---- B: one call behind a gate on its stream -------------------------------------------------------------------------------------

@pytest.mark.parametrize("ctx", list(CONTEXTS))
@pytest.mark.parametrize("name", list(ROWS))
def test_gated_stream(oracle, name, ctx):
    """the decoy is in every buffer until the gate opens; every byte the call leaves must be the baseline's"""
    req, want, _ = baseline(ctx, name, 0, 1, oracle)
    decoy = ROWS[name](oracle, 0, 2)
    e = engine(ctx, "gated")
    b = Bufs(req, decoy)
    real = {n: torch.from_numpy(req.region(n)).cuda() for n in req.bufs}
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    t0 = time.monotonic()
    gate(s)
    with torch.cuda.stream(s):
        for n, t in real.items():
            b.region(n).copy_(t, non_blocking=True)
    req.call(e, b.ptr, s.cuda_stream)
    t1 = time.monotonic()
    held = not s.query()
    with torch.cuda.stream(s):
        snap = {n: t.clone() for n, t in b.t.items()}
    s.synchronize()
    if req.verifies:
        assert t1 - t0 >= 0.9 * GATE_MS / 1000, f"{name}: returned {1000 * (t1 - t0):.1f} ms after the gate of {GATE_MS} ms was enqueued"
    else:
        assert held, f"{name}: the gate of {GATE_MS} ms had passed when the call returned (too short a gate, or the call waited)"
    diff = differences({n: t.cpu().numpy() for n, t in snap.items()}, want)
    assert not diff, f"{name} ({ctx}) behind a gate: " + "; ".join(diff)


# ---- C: many threads on one context --------------------------------------------------------------------------------------------

THREADS, ROUNDS = 8, 3


def host_request(oracle, t):
    goal = L.SliceType(["ec(3,2)", "xor2", "ec(5,3)", "ec(8,2)"][t % 4])
    data = rnd(2 * (5 + t) * BLOCK, 900 + t).reshape(2, -1)
    return goal, data, [oracle.encode_chunk(goal.kind, goal.k, goal.m, data[c]) for c in range(2)]


@pytest.mark.parametrize("ctx", list(CONTEXTS))
def test_threads_on_one_context(oracle, ctx):
    """eight threads, each on its own stream, walk the table in their own order, three rounds, host-pointer calls between; in each
    round one thread's verifying call carries a corrupt stored CRC and must get it reported at its position, and nothing else"""
    inst = lambda t: (t % 2, 10 + t % 4)                 # goal variant and seed of thread t
    for t in range(4):
        for name in ROWS:
            baseline(ctx, name, *inst(t), oracle)
    host = [host_request(oracle, t) for t in range(THREADS)]
    he = engine(ctx, "baseline")
    s0 = he.stats()["chunks_encoded"]
    he.encode_chunks(host[0][0], host[0][1])
    host_count = he.stats()["chunks_encoded"] - s0
    orders = [[list(np.random.default_rng(100 * t + r).permutation(list(ROWS))) for r in range(ROUNDS)] for t in range(THREADS)]
    corrupt = {}
    for r in range(ROUNDS):
        t = (3 * r + 1) % THREADS
        corrupt[(t, r)] = next(n for n in orders[t][r] if n in CORRUPTIBLE)
    e = new_engine(ctx)
    errors, expected = [], [0, 0]
    lock = threading.Lock()

    def worker(t):
        try:
            s = torch.cuda.Stream()
            goal, data, ref = host[t]
            for r in range(ROUNDS):
                for i, name in enumerate(orders[t][r]):
                    req, want, counts = _base[(ctx, name, *inst(t))]
                    with lock:
                        expected[0] += counts[0]
                        expected[1] += counts[1]
                    if corrupt.get((t, r)) == name:
                        _, where = run(e, req.corrupted(), s)
                        if where != req.site[2]:
                            errors.append((t, r, name, "planted mismatch reported at", where, "not", req.site[2]))
                        continue
                    got, where = run(e, req, s)
                    diff = differences(got, want)
                    if where is not None or diff:
                        errors.append((t, r, name, where, diff))
                    if i % 6 == 5:                      # a host-pointer call now and then
                        par, crc = e.encode_chunks(goal, data)
                        with lock:
                            expected[0] += host_count
                        if not all((par[c] == ref[c][0]).all() and (crc[c] == ref[c][1]).all() for c in range(2)):
                            errors.append((t, r, "host encode_chunks"))
                        got_crc = e.crc_blocks(data[1])
                        if not (got_crc == ref[1][1][:got_crc.size]).all():
                            errors.append((t, r, "host crc_blocks"))
        except Exception as exc:  # noqa: BLE001
            errors.append((t, repr(exc)))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(THREADS)]
    try:
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        assert not errors, errors[:5]
        st = e.stats()
        assert (st["chunks_encoded"], st["chunks_recovered"]) == tuple(expected)
        assert e.status_slots()[1] == 0
    finally:
        e.close()


# ---- D: deferred verification across threads ------------------------------------------------------------------------------------

class Gated:
    """A request's buffers and the tensors for their copies, made on stream s up front, so that a call later allocates nothing
    and waits for nothing but its own stream (the device may be held by another thread's gate or sync).  call(): a gate of `ms`,
    the call, copies of every buffer behind it; snap(): the copies, once the device has passed them."""

    def __init__(self, req, s):
        self.req, self.s = req, s
        with torch.cuda.stream(s):
            self.b = Bufs(req)
            self.copies = {n: torch.empty_like(t) for n, t in self.b.t.items()}

    def call(self, e, ms):
        gate(self.s, ms)
        self.req.call(e, self.b.ptr, self.s.cuda_stream)
        with torch.cuda.stream(self.s):
            for n, t in self.b.t.items():
                self.copies[n].copy_(t, non_blocking=True)

    def snap(self):
        return {n: x.cpu().numpy() for n, x in self.copies.items()}


def sync_report(e):
    """lzgpu_dev_sync: None, or the (chunk, part, block) lzgpu_last_bad names"""
    try:
        e.sync()
        return None
    except L.ChunkCrcError as ex:
        return ex.where


@pytest.mark.parametrize("ctx", list(CONTEXTS))
def test_deferred_calls_from_several_threads(oracle, ctx):
    """four threads, each behind its own gate, make deferred verifying calls (they return at once); one planted mismatch is reported
    by the next lzgpu_dev_sync at its position, a second sync reports nothing, and every clean call's results are the baseline's"""
    reqs = [baseline(ctx, "recover_chunks", t % 2, 20 + t, oracle) for t in range(4)]
    e = new_engine(ctx)
    try:
        e.set_deferred_verify(True)
        errors = []
        streams = [torch.cuda.Stream() for _ in range(4)]
        calls = [Gated(reqs[t][0].corrupted() if t == 2 else reqs[t][0], streams[t]) for t in range(4)]

        def worker(t):
            try:
                calls[t].call(e, 60 + 30 * t)
                if streams[t].query():
                    errors.append((t, "the deferred call waited for its stream (or the gate was too short)"))
            except Exception as exc:  # noqa: BLE001
                errors.append((t, repr(exc)))

        threads = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        assert not errors, errors
        assert sync_report(e) == reqs[2][0].where_deferred
        assert sync_report(e) is None
        for t in (0, 1, 3):
            diff = differences(calls[t].snap(), reqs[t][1])
            assert not diff, (t, diff)
        again = [Gated(reqs[t][0], streams[t]) for t in range(4)]       # and once more, all clean
        for g in again:
            g.call(e, 20)
        assert sync_report(e) is None
        assert e.status_slots()[1] == 0
    finally:
        e.close()


@pytest.mark.parametrize("ctx", list(CONTEXTS))
@pytest.mark.parametrize("prior", ["clean", "mismatch"])
def test_deferred_call_made_during_another_threads_sync(oracle, ctx, prior):
    """Thread A makes a deferred call behind a gate on S1, then calls lzgpu_dev_sync.  While that sync waits, B makes a deferred call
    behind a longer gate on S2, and C a verifying call on S3 with deferred mode off.  The result slots hold a `prior` verdict from the
    calls before, so a verdict read before its call has run shows up: B's mismatch (prior clean) must still be reported, once, by A's
    sync or a later one; a clean B (prior mismatch) must never be reported; C must not see B's verdict."""
    (ra, want_a, _), (rb, want_b, _), (rc, want_c, _) = [baseline(ctx, "recover_chunks", v, 30 + v, oracle) for v in (0, 0, 1)]
    rb_call = rb.corrupted() if prior == "clean" else rb
    e = new_engine(ctx)
    try:
        e.set_deferred_verify(True)
        s1, s2, s3 = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
        primers = [Gated(ra.corrupted() if prior == "mismatch" else ra, s) for s in (s1, s2)]
        for g in primers:                                # two slots on top of the free list now hold the prior verdict
            g.call(e, 1)
        assert sync_report(e) == (ra.where_deferred if prior == "mismatch" else None)
        calls = {"a": Gated(ra, s1), "b": Gated(rb_call, s2), "c": Gated(rc, s3)}
        syncing, out = threading.Event(), {}

        def thread_a():
            try:
                calls["a"].call(e, 150)
                out["a0"] = time.monotonic()
                syncing.set()
                out["a"] = sync_report(e)
                out["a1"] = time.monotonic()
            except Exception as exc:  # noqa: BLE001
                out["error"] = repr(exc)
                syncing.set()

        th = threading.Thread(target=thread_a)
        th.start()
        try:
            assert syncing.wait(10)
            time.sleep(0.02)
            out["b0"] = time.monotonic()
            calls["b"].call(e, 400)
            out["b1"] = time.monotonic()
            e.set_deferred_verify(False)
            try:
                c_where = None
                calls["c"].call(e, 300)
            except L.ChunkCrcError as ex:
                c_where = ex.where
            finally:
                e.set_deferred_verify(True)
        finally:
            th.join()
        assert "error" not in out, out["error"]
        assert out["a0"] < out["b0"] and out["b1"] < out["a1"], f"B's call was not made during A's sync: {out}"
        later = sync_report(e)
        reports = [x for x in (out["a"], later) if x is not None]
        assert reports == ([rb.where_deferred] if prior == "clean" else []), (out["a"], later)
        assert c_where is None, f"C reported {c_where}"
        for key, want in (("a", want_a), ("c", want_c)) + ((("b", want_b),) if prior == "mismatch" else ()):
            diff = differences(calls[key].snap(), want)
            assert not diff, (key, diff)
        assert sync_report(e) is None
        assert e.status_slots()[1] == 0
    finally:
        e.close()


@pytest.mark.parametrize("ctx", list(CONTEXTS))
def test_deferred_call_whose_stream_is_gone_by_the_sync(oracle, ctx):
    """a caller may destroy its stream right after a deferred call (the queued work still runs): the sync still reports the call's
    mismatch, since it waits for the call's result copy, not for the stream"""
    cudart = ctypes.CDLL("libcudart.so.12")
    cudart.cudaStreamDestroy.argtypes = [ctypes.c_void_p]
    req = baseline(ctx, "recover_chunks", 0, 40, oracle)[0].corrupted()
    e = new_engine(ctx)
    try:
        e.set_deferred_verify(True)
        b = Bufs(req)
        torch.cuda.synchronize()
        h = ctypes.c_void_p()
        assert cudart.cudaStreamCreateWithFlags(ctypes.byref(h), 1) == 0          # cudaStreamNonBlocking
        s = torch.cuda.ExternalStream(h.value)
        gate(s, 50)
        req.call(e, b.ptr, h.value)
        held = not s.query()
        assert cudart.cudaStreamDestroy(h) == 0
        assert held, "the gate of 50 ms had passed when the deferred call returned"
        assert sync_report(e) == req.where_deferred
        assert sync_report(e) is None
        assert e.status_slots()[1] == 0
    finally:
        e.close()
