"""lzgpu_check_stripes / _dev: do the parts of every stripe still form a codeword, and which part is to blame?

Parts and stored CRCs come from the oracle's encode (tests/_oracle.py).  Faults are injected into part bytes with the stored CRC of
the block recomputed (zlib.crc32 == mycrc32), so only the stripe check can see them.  The expected verdict of a faulty chunk comes
from the oracle too: its data parts are re-encoded and the recomputed parity compared with the stored parity per stripe and row;
the suspect is the part the fault was put in.  Every case runs on the fused route and, with LZGPU_DISABLE_FUSED=1, on the generic
route; both must give the same verdicts, and the route is asserted through last_geometry()."""
import os
import subprocess
import zlib

import numpy as np
import pytest

import lizardfs_b200 as L
from lizardfs_b200 import _lib
from tests import _oracle as O

BLOCK = 65536
ZERO_CRC = 0xD7978EEB
CLEAN = (-1, 0, -1)

GOALS = ["xor2", "xor3", "ec(3,2)", "ec(5,3)", "ec(8,2)", "ec(4,4)", "ec(8,4)", "ec(6,5)", "ec(22,4)"]
_engines = {}


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for e in _engines.values():
        e.close()
    _engines.clear()


def engine(**env):
    """one context per set of switches (read when a context is created)"""
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


def fused_engine():
    return engine()


def generic_engine():
    return engine(LZGPU_DISABLE_FUSED=1)


class Batch:
    """n chunks of a goal: data parts, oracle parity, per-part stored CRCs"""

    def __init__(self, oracle, text, n, nb, seed, tail=1000):
        self.goal = L.SliceType(text)
        self.k, self.m = self.goal.k, self.goal.m
        self.kind = 0 if text.startswith("xor") else 1
        self.n, self.nb = n, nb
        self.pb = (nb + self.k - 1) // self.k
        self.oracle = oracle
        rng = np.random.default_rng(seed)
        chunks = rng.integers(0, 256, (n, nb * BLOCK), dtype=np.uint8)
        chunks[:, nb * BLOCK - tail:] = 0          # partial last block: zero-extended
        self.parts = [np.zeros((n, self.pb * BLOCK), dtype=np.uint8) for _ in range(self.k + self.m)]
        self.crc = [np.zeros((n, self.pb), dtype=np.uint32) for _ in range(self.k + self.m)]
        for c in range(n):
            parity, crc = oracle.encode_chunk(self.kind, self.k, self.m, chunks[c])
            data, _ = O.split_parts(chunks[c], self.k)
            for j in range(self.k):
                self.parts[j][c] = data[j]
                self.crc[j][c] = [crc[s * self.k + j] if s * self.k + j < nb else ZERO_CRC for s in range(self.pb)]
            for r in range(self.m):
                self.parts[self.k + r][c] = parity[r]
                self.crc[self.k + r][c] = crc[nb + r * self.pb: nb + (r + 1) * self.pb]
        self.faulty = set()

    def corrupt(self, c, part, stripe, offset=777, length=5):
        """flip bytes of a part block and recompute its stored CRC: only the stripe check sees it"""
        blk = self.parts[part][c, stripe * BLOCK:(stripe + 1) * BLOCK]
        blk[offset:offset + length] ^= np.arange(1, length + 1, dtype=np.uint8) * 37
        self.crc[part][c, stripe] = zlib.crc32(blk.tobytes())
        self.faulty.add(c)

    def expected(self, rows):
        """verdicts from the oracle: re-encode the data parts of each faulty chunk, compare with the stored parity rows `rows`"""
        out = [CLEAN] * self.n
        for c in sorted(self.faulty):
            blocks = np.stack([self.parts[j][c].reshape(self.pb, BLOCK) for j in range(self.k)], axis=1).reshape(-1, BLOCK)
            parity, _ = self.oracle.encode_chunk(self.kind, self.k, self.m, np.ascontiguousarray(blocks[:self.nb]).reshape(-1))
            diff = {r: (parity[r] != self.parts[self.k + r][c]).reshape(self.pb, BLOCK).any(axis=1) for r in rows}
            bad = [s for s in range(self.pb) if any(diff[r][s] for r in rows)]
            if bad:
                out[c] = (bad[0], sum(1 << r for r in rows if diff[r][bad[0]]), None)
        return out


def given_parts(b, skip=()):
    return [None if i in skip else b.parts[i] for i in range(b.k + b.m)]


def as_tuples(v):
    return [(int(x["first_bad_stripe"]), int(x["bad_rows"]), int(x["suspect_part"])) for x in v]


def run_both(b, parts, crcs, expect_fused):
    """the host call on both routes; returns the (identical) verdicts"""
    results = []
    for eng, fused in ((fused_engine(), expect_fused), (generic_engine(), False)):
        before = eng.last_geometry()
        v = as_tuples(eng.check_stripes(b.goal, b.nb, parts, crcs))
        geo = eng.last_geometry()
        if fused:
            assert geo["kernel"] == _lib.KERNEL_CHECK
            assert geo["units"] == b.n * -(-b.pb // geo["G"])
        else:
            assert geo["kernel"] != _lib.KERNEL_CHECK or geo == before
        assert eng.status_slots()[1] == 0
        results.append(v)
    assert results[0] == results[1], "fused and generic routes disagree"
    return results[0]


def check(got, want, suspects):
    for c, (g, w) in enumerate(zip(got, want)):
        if w == CLEAN:
            assert g == CLEAN, c
        else:
            assert g[:2] == w[:2], (c, g, w)
            assert g[2] == suspects[c], (c, g, suspects[c])


def fused_goal(text):
    g = L.SliceType(text)
    return not (g.m >= 5 or (g.m == 4 and g.k > 20))


def nb_for(k):
    return 2 * k + 1 if k > 1 else 5          # ragged: nb % k != 0, three stripes


_batches = {}


def batch(oracle, text, n=3, seed=1):
    key = (text, n, seed)
    if key not in _batches:
        g = L.SliceType(text)
        _batches[key] = Batch(oracle, text, n, nb_for(g.k), seed)
    b = _batches[key]
    fresh = Batch.__new__(Batch)
    fresh.__dict__.update(b.__dict__)
    fresh.parts = [p.copy() for p in b.parts]
    fresh.crc = [c.copy() for c in b.crc]
    fresh.faulty = set()
    return fresh


gpu = pytest.mark.gpu


@gpu
@pytest.mark.parametrize("text", GOALS)
@pytest.mark.parametrize("with_crc", [True, False])
def test_clean_batches_are_codewords(oracle, text, with_crc):
    b = batch(oracle, text)
    v = run_both(b, given_parts(b), b.crc if with_crc else None, fused_goal(text))
    assert v == [CLEAN] * b.n


@gpu
@pytest.mark.parametrize("text", GOALS)
def test_data_faults_name_the_part(oracle, text):
    b = batch(oracle, text)
    rows = list(range(b.m))
    b.corrupt(0, 0, b.pb - 1)                  # the last, ragged stripe (data part 0 has a block there)
    b.corrupt(2, b.k - 1, 1)
    v = run_both(b, given_parts(b), b.crc, fused_goal(text))
    want = b.expected(rows)
    assert want[0][0] == b.pb - 1 and want[2][0] == 1
    assert want[0][1] == want[2][1] == (1 << b.m) - 1     # every row sees a data fault
    multi = b.m >= 2
    check(v, want, {0: 0 if multi else -1, 2: b.k - 1 if multi else -1})


@gpu
@pytest.mark.parametrize("text", GOALS)
def test_parity_fault_names_its_row(oracle, text):
    b = batch(oracle, text)
    r = b.m - 1
    b.corrupt(1, b.k + r, 0)
    v = run_both(b, given_parts(b), b.crc, fused_goal(text))
    want = b.expected(list(range(b.m)))
    assert want[1][:2] == (0, 1 << r)
    check(v, want, {1: b.k + r if b.m >= 2 else -1})


@gpu
@pytest.mark.parametrize("text", ["ec(5,3)", "ec(4,4)", "ec(8,4)", "ec(6,5)"])
def test_two_corrupt_parts_in_one_stripe_have_no_suspect(oracle, text):
    b = batch(oracle, text)
    b.corrupt(1, 0, 1, offset=100)
    b.corrupt(1, 1, 1, offset=100)             # the same bytes: the syndromes combine two columns
    b.corrupt(2, 0, 1, offset=100)
    b.corrupt(2, b.k, 1, offset=5000)          # different bytes: each byte names its own part
    v = run_both(b, given_parts(b), b.crc, fused_goal(text))
    check(v, b.expected(list(range(b.m))), {1: -1, 2: -1})


@gpu
@pytest.mark.parametrize("text", ["ec(8,2)", "ec(5,3)", "xor3"])
def test_faults_in_two_stripes_report_the_lower(oracle, text):
    b = batch(oracle, text)
    b.corrupt(1, 0, 2)
    b.corrupt(1, b.k, 1)
    v = run_both(b, given_parts(b), b.crc, fused_goal(text))
    want = b.expected(list(range(b.m)))
    assert want[1][0] == 1
    check(v, want, {1: b.k if b.m >= 2 else -1})


@gpu
@pytest.mark.parametrize("text,skip,x", [("ec(5,3)", (6,), 2), ("ec(8,4)", (8,), 3), ("ec(8,4)", (9, 11), 5), ("ec(8,2)", (8,), 4),
                                         ("ec(4,4)", (4, 5, 6), 1)])
def test_missing_parity_rows_are_not_checked(oracle, text, skip, x):
    b = batch(oracle, text)
    rows = [r for r in range(b.m) if b.k + r not in skip]
    b.corrupt(0, x, 1)
    b.corrupt(2, b.k + rows[-1], 2)
    for p in skip:                             # a fault in a part that is not given is not seen
        b.corrupt(1, p, 0)
    v = run_both(b, given_parts(b, skip), b.crc, fused_goal(text))
    want = b.expected(rows)
    assert want[0][1] == sum(1 << r for r in rows) and want[1] == CLEAN
    check(v, want, {0: x if len(rows) >= 2 else -1, 2: b.k + rows[-1] if len(rows) >= 2 else -1})


@gpu
def test_missing_parts_are_refused(oracle):
    b = batch(oracle, "ec(5,3)")
    for eng in (fused_engine(), generic_engine()):
        launches = eng.stats()["kernel_launches"]
        for skip in ((0,), (5, 6, 7)):
            with pytest.raises(L.LzGpuError) as ei:
                eng.check_stripes(b.goal, b.nb, given_parts(b, skip), b.crc)
            assert ei.value.status == _lib.ERR_TOO_FEW_PARTS
        assert eng.stats()["kernel_launches"] == launches


@gpu
@pytest.mark.parametrize("text", ["ec(8,2)", "ec(5,3)", "xor3", "ec(6,5)"])
def test_stored_crc_failure_keeps_the_verdicts(oracle, text):
    b = batch(oracle, text)
    b.corrupt(2, 1, 1)
    want = b.expected(list(range(b.m)))
    crcs = [c.copy() for c in b.crc]
    crcs[b.k][1, 1] ^= 0x40                    # (chunk 1, parity part 0, block 1)
    crcs[0][2, 0] ^= 0x40                      # a later chunk: not the first mismatch
    results = []
    for eng in (fused_engine(), generic_engine()):
        with pytest.raises(L.ChunkCrcError) as ei:
            eng.check_stripes(b.goal, b.nb, given_parts(b), crcs)
        assert ei.value.where == (1, b.k, 1)
        v = as_tuples(ei.value.verdict)
        check(v, want, {2: 1 if b.m >= 2 else -1})
        results.append(v)
        assert eng.status_slots()[1] == 0
    assert results[0] == results[1]


class Dev:
    """the batch resident on the device (torch), parts at part_stride from an offset base"""

    def __init__(self, b, pad=0, lead=0):
        import torch
        self.torch = torch
        self.stride = b.pb * BLOCK + pad
        self.bufs, self.ptrs, self.crcs = [], [], []
        for p, c in zip(b.parts, b.crc):
            host = np.random.default_rng(7).integers(0, 256, lead + b.n * self.stride, dtype=np.uint8)
            for i in range(b.n):
                host[lead + i * self.stride: lead + i * self.stride + p.shape[1]] = p[i]
            t = torch.from_numpy(host).cuda()
            ct = torch.from_numpy(c.view(np.int32).copy()).cuda()
            self.bufs += [t, ct]
            self.ptrs.append(t.data_ptr() + lead)
            self.crcs.append(ct.data_ptr())


def run_dev(eng, b, dev, skip=(), crcs=True, guard=4096, lead=0):
    torch = dev.torch
    init = np.random.default_rng(3).integers(0, 256, 2 * guard + lead + 12 * b.n, dtype=np.uint8)
    t = torch.from_numpy(init.copy()).cuda()
    parts = [None if i in skip else p for i, p in enumerate(dev.ptrs)]
    eng.check_stripes_dev(b.goal, b.n, b.nb, parts, dev.stride, dev.crcs if crcs else None, t.data_ptr() + guard + lead)
    torch.cuda.synchronize()
    after = t.cpu().numpy()
    o = guard + lead
    assert (after[:o] == init[:o]).all() and (after[o + 12 * b.n:] == init[o + 12 * b.n:]).all(), "write outside d_verdict"
    return as_tuples(after[o:o + 12 * b.n].copy().view(L.Engine.VERDICT_DTYPE))


@gpu
@pytest.mark.parametrize("text", ["ec(8,2)", "ec(5,3)", "xor2", "ec(22,4)"])
@pytest.mark.parametrize("pad,lead", [(0, 0), (16, 16), (65536 + 48, 48)])
def test_dev_layouts_write_only_the_verdicts(oracle, text, pad, lead):
    b = batch(oracle, text)
    b.corrupt(1, 2, 1)
    want = b.expected(list(range(b.m)))
    dev = Dev(b, pad, lead)
    got = []
    for eng, fused in ((fused_engine(), fused_goal(text)), (generic_engine(), False)):
        v = run_dev(eng, b, dev, lead=lead % 64)
        if fused:
            assert eng.last_geometry()["kernel"] == _lib.KERNEL_CHECK
        check(v, want, {1: 2 if b.m >= 2 else -1})
        got.append(v)
    assert got[0] == got[1]
    # every input byte unchanged
    for i, p in enumerate(b.parts):
        host = dev.bufs[2 * i].cpu().numpy()
        for c in range(b.n):
            assert (host[lead + c * dev.stride: lead + c * dev.stride + p.shape[1]] == p[c]).all()


@gpu
def test_misaligned_pointers_are_refused_without_a_launch(oracle):
    import torch
    b = batch(oracle, "ec(8,2)")
    dev = Dev(b)
    out = torch.zeros(64 + 12 * b.n, dtype=torch.uint8, device="cuda")
    for eng in (fused_engine(), generic_engine()):
        launches = eng.stats()["kernel_launches"]
        bad_parts = list(dev.ptrs)
        bad_parts[3] += 8
        bad_crcs = list(dev.crcs)
        bad_crcs[9] += 2
        for parts, crcs, ver in ((bad_parts, dev.crcs, out.data_ptr()), (dev.ptrs, bad_crcs, out.data_ptr()),
                                 (dev.ptrs, dev.crcs, out.data_ptr() + 2)):
            with pytest.raises(L.LzGpuError) as ei:
                eng.check_stripes_dev(b.goal, b.n, b.nb, parts, dev.stride, crcs, ver)
            assert ei.value.status == _lib.ERR_ARG
        assert eng.stats()["kernel_launches"] == launches


@gpu
def test_deferred_mode_collects_the_crc_mismatch(oracle):
    b = batch(oracle, "ec(8,2)")
    b.corrupt(0, 4, 1)
    want = b.expected([0, 1])
    b.crc[9][2, 1] ^= 1
    dev = Dev(b)
    for eng in (fused_engine(), generic_engine()):
        eng.set_deferred_verify(True)
        try:
            v = run_dev(eng, b, dev)           # returns at once; the verdicts are there once the stream has passed
            with pytest.raises(L.ChunkCrcError) as ei:
                eng.sync()
            assert ei.value.where == (2, 9, 1)
        finally:
            eng.set_deferred_verify(False)
        check(v, want, {0: 4})
        assert eng.status_slots()[1] == 0


@gpu
@pytest.mark.parametrize("cap", [1, 3])
@pytest.mark.parametrize("text", ["ec(8,2)", "xor3", "ec(8,4)", "ec(5,3)"])
def test_capped_grid_walks_several_units_per_cta(oracle, text, cap):
    b = batch(oracle, text, n=8, seed=5)
    for c in (0, 3, 7):
        b.corrupt(c, c % b.k, c % b.pb)
    b.corrupt(5, b.k, 2)
    want = b.expected(list(range(b.m)))
    dev = Dev(b)
    eng = engine(LZGPU_GRID_CAP=cap)
    v = run_dev(eng, b, dev)
    grid, units = eng.last_launch()
    assert eng.last_geometry()["kernel"] == _lib.KERNEL_CHECK
    assert grid == cap and units > 2 * cap
    assert v == run_dev(generic_engine(), b, dev) == run_dev(fused_engine(), b, dev)
    multi = b.m >= 2
    check(v, want, {0: 0 if multi else -1, 3: 3 % b.k if multi else -1, 7: 7 % b.k if multi else -1, 5: b.k if multi else -1})


@gpu
def test_host_tiles_report_batch_wide_chunks():
    """ec(8,2), one-stripe chunks: 409 chunks fill a 256 MiB tile of ten parts, so 823 chunks take three tiles.  All-zero chunks are
    codewords with the CRC of a zero block everywhere; faults in tiles 1 and 2."""
    goal, k, m, nb, n = L.SliceType("ec(8,2)"), 8, 2, 8, 823
    parts = [np.zeros((n, BLOCK), dtype=np.uint8) for _ in range(k + m)]
    crcs = [np.full((n, 1), ZERO_CRC, dtype=np.uint32) for _ in range(k + m)]
    for c, p in ((500, 3), (820, 9)):
        parts[p][c, 10:14] = 0xA5
        crcs[p][c, 0] = zlib.crc32(parts[p][c].tobytes())
    for eng in (fused_engine(), generic_engine()):
        before = eng.stats()["batches_timed"]
        v = as_tuples(eng.check_stripes(goal, nb, parts, crcs))
        assert eng.stats()["batches_timed"] - before == 3
        bad = {c: x for c, x in enumerate(v) if x != CLEAN}
        assert bad == {500: (0, 3, 3), 820: (0, 2, 9)}
        assert eng.status_slots()[1] == 0
        crcs2 = [c.copy() for c in crcs]
        crcs2[5][700, 0] ^= 1
        crcs2[0][20, 0] ^= 1
        with pytest.raises(L.ChunkCrcError) as ei:
            eng.check_stripes(goal, nb, parts, crcs2)
        assert ei.value.where == (20, 0, 0)
        assert {c: x for c, x in enumerate(as_tuples(ei.value.verdict)) if x != CLEAN} == bad
        assert eng.status_slots()[1] == 0


@gpu
def test_full_size_chunks():
    goal, k, m, nb = L.SliceType("ec(8,2)"), 8, 2, 1024
    enc = fused_engine()
    data = np.random.default_rng(11).integers(0, 256, (2, nb * BLOCK), dtype=np.uint8)
    parity, crc = enc.encode_chunks(goal, data)
    blocks = data.reshape(2, nb // k, k, BLOCK)
    parts = [np.ascontiguousarray(blocks[:, :, j]).reshape(2, -1) for j in range(k)] + [np.ascontiguousarray(parity[:, r]) for r in range(m)]
    crcs = [np.ascontiguousarray(crc[:, :nb].reshape(2, nb // k, k)[:, :, j]) for j in range(k)]
    crcs += [np.ascontiguousarray(crc[:, nb + r * 128: nb + (r + 1) * 128]) for r in range(m)]
    assert run_plain(goal, nb, parts, crcs) == [CLEAN, CLEAN]
    parts[5][1, 100 * BLOCK + 65535] ^= 1
    crcs[5][1, 100] = zlib.crc32(parts[5][1, 100 * BLOCK:101 * BLOCK].tobytes())
    parts[9][0, 127 * BLOCK] ^= 1
    crcs[9][0, 127] = zlib.crc32(parts[9][0, 127 * BLOCK:].tobytes())
    assert run_plain(goal, nb, parts, crcs) == [(127, 2, 9), (100, 3, 5)]


def run_plain(goal, nb, parts, crcs):
    got = [as_tuples(eng.check_stripes(goal, nb, parts, crcs)) for eng in (fused_engine(), generic_engine())]
    assert got[0] == got[1]
    assert fused_engine().last_geometry()["kernel"] == _lib.KERNEL_CHECK
    return got[0]


def test_verdict_struct_layout_matches_the_header(tmp_path):
    """(no GPU needed) the ctypes and numpy mirrors of lzgpu_stripe_verdict against sizeof / offsetof from include/lzgpu.h"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "v.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "lzgpu.h"\nint main(void) { printf("%zu %zu %zu %zu %d %d\\n", '
                   'sizeof(lzgpu_stripe_verdict), offsetof(lzgpu_stripe_verdict, first_bad_stripe), offsetof(lzgpu_stripe_verdict, bad_rows), '
                   'offsetof(lzgpu_stripe_verdict, suspect_part), LZGPU_ERR_INCONSISTENT, LZGPU_KERNEL_CHECK); return 0; }\n')
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(root, "include"), str(src), "-o", str(tmp_path / "v")], check=True)
    out = [int(x) for x in subprocess.run([str(tmp_path / "v")], capture_output=True, text=True, check=True).stdout.split()]
    cls = _lib.LzStripeVerdict
    assert out[0] == C_sizeof(cls) == L.Engine.VERDICT_DTYPE.itemsize
    assert out[1:4] == [getattr(cls, f).offset for f, _ in cls._fields_] == [L.Engine.VERDICT_DTYPE.fields[f][1] for f in L.Engine.VERDICT_DTYPE.names]
    assert out[4] == _lib.ERR_INCONSISTENT and out[5] == _lib.KERNEL_CHECK


def C_sizeof(cls):
    import ctypes
    return ctypes.sizeof(cls)
