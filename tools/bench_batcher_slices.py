"""Time the call shape of lzgpu::StripeBatcher over several slices (include/lzgpu_stripe_batcher.hpp) against the alternatives.

A flush of n complete combined stripes (L = lcm(k_i) blocks each) can be passed to lzgpu_encode_slices as
  (a) n chunks of L blocks (one combined stripe per chunk),
  (b) the batcher's packed pseudo-chunks: q = ceil(n / floor(1024 / L)) chunks of s = ceil(n / q) stripes, zero padding at the end,
  (c) one call per slice on the n chunks of L blocks (lzgpu_encode_chunks per xor/ec slice, lzgpu_crc_blocks for a standard slice).
The three alternate in one run, after a warm-up of each, on resident buffers (the _dev calls, CUDA events around each) and from
pinned host buffers (the host calls, which return when the results are in host memory).  The goal sets and stripe counts are those
of DESIGN.md §5 (1 GiB of data each).  A one-slice batcher keeps passing n chunks of k blocks; the packed form of ec(8,2) is timed
against it as well.  After the timing, the outputs of (b) and (c) are remapped to stripe order and compared with (a).  The card's
name and power limit are read in the same run.

    python tools/bench_batcher_slices.py [--iters 10] [--host-iters 2] [--rounds 3] [--out results/bench_batcher_slices.json]
"""
import argparse
import ctypes as C
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lizardfs_b200 as L  # noqa: E402
from bench_slices import card, time_ms  # noqa: E402  (tools/ is this script's directory)

BLOCK = 65536
CASES = [(("std", "xor2", "xor3"), 2730), (("ec(3,2)", "ec(8,2)"), 682)]
SINGLE = ("ec(8,2)", 2048)


def lcm_k(goals):
    out = 1
    for g in goals:
        a, b = out, g.k
        while b:
            a, b = b, a % b
        out = out // a * g.k
    return out


def packing(n, per_chunk):
    q = -(-n // per_chunk)
    return q, -(-n // q)


class Shape:
    """the outputs of one call shape, `chunks` chunks of `stripes` combined stripes, one parity / CRC buffer per slice"""

    def __init__(self, goals, lc, chunks, stripes, pinned):
        self.goals, self.lc, self.chunks, self.stripes = goals, lc, chunks, stripes
        self.chunk_len = stripes * lc * BLOCK
        dev = None if pinned else "cuda"
        self.out = []
        for g in goals:
            m = 0 if g.is_std else g.m
            pb = stripes * lc // g.k
            par = torch.empty((chunks, m * pb * BLOCK if m else 1), dtype=torch.uint8, device=dev)
            crc = torch.empty((chunks, stripes * lc + m * pb), dtype=torch.int32, device=dev)
            self.out.append((par.pin_memory() if pinned else par, crc.pin_memory() if pinned else crc, m, pb))
        ns = len(goals)
        self.garr = (L.engine.LzGoal * ns)(*[g.c for g in goals])
        self.pp = [p.data_ptr() if m else 0 for p, _, m, _ in self.out]
        self.ps = [m * pb * BLOCK for _, _, m, pb in self.out]
        self.cp = [c.data_ptr() for _, c, _, _ in self.out]
        self.cs = [c.shape[1] for _, c, _, _ in self.out]

    def dev(self, eng, data, stream):
        eng.encode_slices_dev(self.goals, self.chunks, self.chunk_len, data.data_ptr(), self.chunk_len, self.pp, self.ps, self.cp, self.cs, stream)

    def host(self, eng, data):
        ns = len(self.goals)
        rc = eng.lib.lzgpu_encode_slices(eng.h, self.garr, ns, self.chunks, self.chunk_len, data.data_ptr(), self.chunk_len,
                                         (C.c_void_p * ns)(*[p or None for p in self.pp]), (C.c_size_t * ns)(*self.ps),
                                         (C.c_void_p * ns)(*self.cp), (C.c_size_t * ns)(*self.cs))
        assert rc == 0, eng.lib.lzgpu_last_error()

    def per_slice_dev(self, eng, data, stream):
        for g, (p, c, m, pb) in zip(self.goals, self.out):
            if g.is_std:
                eng.crc_blocks_dev(data.data_ptr(), self.chunks * self.stripes * self.lc, c.data_ptr(), stream=stream)
            else:
                eng.encode_chunks_dev(g, self.chunks, self.chunk_len, data.data_ptr(), self.chunk_len, p.data_ptr(), m * pb * BLOCK,
                                      c.data_ptr(), c.shape[1], stream)

    def per_slice_host(self, eng, data):
        for g, (p, c, m, pb) in zip(self.goals, self.out):
            if g.is_std:
                rc = eng.lib.lzgpu_crc_blocks(eng.h, data.data_ptr(), self.chunks * self.stripes * self.lc, BLOCK, BLOCK, c.data_ptr())
            else:
                rc = eng.lib.lzgpu_encode_chunks(eng.h, C.byref(g.c), self.chunks, self.chunk_len, data.data_ptr(), self.chunk_len,
                                                 p.data_ptr(), m * pb * BLOCK, c.data_ptr(), c.shape[1])
            assert rc == 0, eng.lib.lzgpu_last_error()

    def by_stripe(self, n):
        """per slice: parity [n, m, per blocks], data CRCs [n, L], parity CRCs [n, m, per] in combined-stripe order"""
        q, s = self.chunks, self.stripes
        res = []
        for g, (p, c, m, pb) in zip(self.goals, self.out):
            per = self.lc // g.k
            par = p[:, :m * pb * BLOCK].reshape(q, m, s, per * BLOCK).permute(0, 2, 1, 3).reshape(q * s, m, per * BLOCK)[:n]
            cd = c[:, :s * self.lc].reshape(q * s, self.lc)[:n]
            cp = c[:, s * self.lc:].reshape(q, m, s, per).permute(0, 2, 1, 3).reshape(q * s, m, per)[:n]
            res.append((par, cd, cp))
        return res


def same(x, y):
    return all(torch.equal(a, b) for sx, sy in zip(x, y) for a, b in zip(sx, sy))


def rotate(fns, iters, rounds, sync):
    for f in fns.values():      # warm-up of every shape
        f()
        f()
    sync()
    times = {k: [] for k in fns}
    for _ in range(rounds):
        for k, f in fns.items():
            times[k].append(time_ms(f, iters))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--host-iters", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batcher_slices: no CUDA device")
    info = card()
    print(f"# {info}", flush=True)
    eng = L.Engine(0)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    st = stream.cuda_stream
    rows = []

    def report(kind, name, n, times, shapes, ok):
        best = {k: min(v) for k, v in times.items()}
        r = dict(kind=kind, slices=name, stripes=n, shapes=shapes, ms=times, best_ms=best, same_bytes=ok)
        rows.append(r)
        print(f"{kind:8s} {name:16s} n={n:5d}  " + "  ".join(f"{k} {best[k]:8.3f} ms {times[k]}" for k in times) + f"  same={ok}", flush=True)

    for names, n in CASES + [((SINGLE[0],), SINGLE[1])]:
        goals = [L.SliceType(x) for x in names]
        lc = lcm_k(goals)
        q, s = packing(n, 1024 // lc)
        name = "+".join(names)
        shapes = dict(a=f"{n} x {lc} blocks", b=f"{q} x {s * lc} blocks")
        for pinned in (False, True):
            data = torch.randint(0, 256, (q * s * lc * BLOCK,), dtype=torch.uint8, device=None if pinned else "cuda")
            data[n * lc * BLOCK:] = 0                   # the zero padding stripes of the last pseudo-chunk
            if pinned:
                data = data.pin_memory()
            fa = Shape(goals, lc, n, 1, pinned)
            fb = Shape(goals, lc, q, s, pinned)
            if pinned:
                fns = {"a": lambda: fa.host(eng, data), "b": lambda: fb.host(eng, data)}
            else:
                fns = {"a": lambda: fa.dev(eng, data, st), "b": lambda: fb.dev(eng, data, st)}
            fc = None
            if len(goals) > 1:
                fc = Shape(goals, lc, n, 1, pinned)
                fns["c"] = (lambda: fc.per_slice_host(eng, data)) if pinned else (lambda: fc.per_slice_dev(eng, data, st))
            times = rotate(fns, a.host_iters if pinned else a.iters, a.rounds, torch.cuda.synchronize)
            ref = fa.by_stripe(n)
            ok = same(ref, fb.by_stripe(n)) and (fc is None or same(ref, fc.by_stripe(n)))
            report("host" if pinned else "resident", name, n, times, shapes, ok)
            del data, fa, fb, fc
            torch.cuda.empty_cache()
    eng.close()
    result = dict(card=info, rows=rows)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(dict(card=info, rows=[{k: r[k] for k in ("kind", "slices", "best_ms", "same_bytes")} for r in rows])))


if __name__ == "__main__":
    main()
