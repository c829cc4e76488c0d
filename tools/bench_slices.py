"""Time the one-pass encode for several slices (lzgpu_encode_slices_dev) against one call per slice on the same buffers.

Rows (resident 64 MiB chunks on the device): each goal set below, one lzgpu_encode_slices_dev call against lzgpu_encode_chunks_dev per
xor/ec slice plus lzgpu_crc_blocks_dev for the standard slice; the two alternate twice after a warm-up, CUDA events around each.
Also: the batched shape of one combined stripe per chunk (chunk_len = L x 64 KiB), and the host forms (lzgpu_encode_slices against
the per-slice host calls) on pinned buffers.  Reports GiB/s of chunk data and the fraction of 3.35 TB/s (H100 SXM HBM3) the one-pass
algorithmic bytes (SURVEY.md §8(d), the data read once) reach, with the card's name and power limit read in the same run.  The
outputs of both forms are compared after the timing.

    python tools/bench_slices.py [--chunks 16] [--iters 10] [--out results/bench_slices.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lizardfs_b200 as L  # noqa: E402

BLOCK = 65536
HBM = 3.35e12
SETS = [("ec(3,2)", "ec(8,2)"), ("xor2", "xor3"), ("std", "xor2", "xor3"), ("ec(8,2)", "ec(8,4)")]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        out = torch.cuda.get_device_name(0) + ", power limit unknown"
    return out


def alg_bytes(goals, n, chunk_len):
    nb = -(-chunk_len // BLOCK)
    total = chunk_len
    for g in goals:
        m = 0 if g.is_std else g.m
        pb = -(-nb // g.k)
        total += m * pb * BLOCK + 4 * (nb + m * pb)
    return n * total


class Buffers:
    """the data and one parity / CRC buffer per slice for each form, all resident"""

    def __init__(self, goals, n, chunk_len, seed=1):
        self.goals, self.n, self.chunk_len = goals, n, chunk_len
        self.nb = -(-chunk_len // BLOCK)
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.data = torch.randint(0, 256, (n, self.nb * BLOCK), dtype=torch.uint8, device="cuda", generator=g)
        self.data[:, chunk_len:] = 0
        self.out = {form: [self._slice_out(s) for s in goals] for form in ("one", "per")}

    def _slice_out(self, g):
        m = 0 if g.is_std else g.m
        pb = -(-self.nb // g.k)
        par = torch.empty((self.n, max(m, 1) * pb * BLOCK), dtype=torch.uint8, device="cuda")
        crc = torch.empty((self.n, self.nb + m * pb), dtype=torch.int32, device="cuda")
        return par, crc, m

    def one(self, eng):
        o = self.out["one"]
        st = torch.cuda.current_stream().cuda_stream
        eng.encode_slices_dev(self.goals, self.n, self.chunk_len, self.data.data_ptr(), self.nb * BLOCK,
                              [0 if m == 0 else p.data_ptr() for p, _, m in o], [0 if m == 0 else p.shape[1] for p, _, m in o],
                              [c.data_ptr() for _, c, _ in o], [c.shape[1] for _, c, _ in o], st)

    def per(self, eng):
        st = torch.cuda.current_stream().cuda_stream
        for g, (p, c, m) in zip(self.goals, self.out["per"]):
            if g.is_std:
                eng.crc_blocks_dev(self.data.data_ptr(), self.n * self.nb, c.data_ptr(), stream=st)
            else:
                eng.encode_chunks_dev(g, self.n, self.chunk_len, self.data.data_ptr(), self.nb * BLOCK, p.data_ptr(), p.shape[1], c.data_ptr(),
                                      c.shape[1], st)

    def same(self):
        for (p1, c1, m), (p2, c2, _) in zip(self.out["one"], self.out["per"]):
            if m and not torch.equal(p1, p2):
                return False
            if not torch.equal(c1, c2):
                return False
        return True


def time_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def alternate(fa, fb, iters, rounds=2):
    for _ in range(2):   # warm-up of both shapes
        fa()
        fb()
    torch.cuda.synchronize()
    ta, tb = [], []
    for _ in range(rounds):
        ta.append(time_ms(fa, iters))
        tb.append(time_ms(fb, iters))
    return ta, tb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=16)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_slices: no CUDA device")
    eng = L.Engine(0)
    stream = torch.cuda.Stream()          # a stream of its own: the *_dev calls and the events are ordered on it
    torch.cuda.set_stream(stream)
    rows = []
    info = card()
    print(f"# {info}")

    def row(kind, names, n, chunk_len, ta, tb, ok):
        goals = [L.SliceType(x) for x in names]
        data_bytes = n * chunk_len
        one, per = min(ta), min(tb)
        r = dict(kind=kind, slices="+".join(names), chunks=n, chunk_len=chunk_len, one_pass_ms=ta, per_slice_ms=tb,
                 one_pass_gibps=data_bytes / one / 1e-3 / 2**30, per_slice_gibps=data_bytes / per / 1e-3 / 2**30,
                 one_pass_hbm_fraction=alg_bytes(goals, n, chunk_len) / (one * 1e-3) / HBM, speedup=per / one, same_bytes=ok)
        rows.append(r)
        print(f"{kind:9s} {r['slices']:22s} n={n:5d} len={chunk_len:9d}  one pass {one:8.3f} ms ({r['one_pass_gibps']:6.1f} GiB/s, "
              f"{100 * r['one_pass_hbm_fraction']:5.1f} % of 3.35 TB/s)  per slice {per:8.3f} ms ({r['per_slice_gibps']:6.1f} GiB/s)  "
              f"x{r['speedup']:.2f}  same={ok}", flush=True)

    for names in SETS:
        goals = [L.SliceType(x) for x in names]
        b = Buffers(goals, a.chunks, 1024 * BLOCK)
        ta, tb = alternate(lambda: b.one(eng), lambda: b.per(eng), a.iters)
        row("resident", names, a.chunks, 1024 * BLOCK, ta, tb, b.same())
        del b
    for names in (("ec(3,2)", "ec(8,2)"), ("std", "xor2", "xor3")):
        goals = [L.SliceType(x) for x in names]
        Lc = int(np.lcm.reduce([g.k for g in goals if not g.is_std]))
        n = (a.chunks * 1024) // Lc
        b = Buffers(goals, n, Lc * BLOCK)
        ta, tb = alternate(lambda: b.one(eng), lambda: b.per(eng), a.iters)
        row("stripe", names, n, Lc * BLOCK, ta, tb, b.same())
        del b
    # host forms: data and every output in pinned memory, through the C ABI
    for names in (("ec(3,2)", "ec(8,2)"), ("std", "xor2", "xor3")):
        goals = [L.SliceType(x) for x in names]
        n, clen, nb = a.chunks, 1024 * BLOCK, 1024
        host = torch.randint(0, 256, (n, clen), dtype=torch.uint8).pin_memory()
        outs = {}
        for form in ("one", "per"):
            outs[form] = []
            for g in goals:
                m = 0 if g.is_std else g.m
                pb = -(-nb // g.k)
                outs[form].append((torch.empty((n, max(m, 1) * pb * BLOCK), dtype=torch.uint8).pin_memory(),
                                   torch.empty((n, nb + m * pb), dtype=torch.int32).pin_memory(), m))
        lib = eng.lib
        ns = len(goals)
        garr = (L.engine.LzGoal * ns)(*[g.c for g in goals])
        o = outs["one"]
        pp = (C.c_void_p * ns)(*[p.data_ptr() if m else None for p, _, m in o])
        ps = (C.c_size_t * ns)(*[p.shape[1] if m else 0 for p, _, m in o])
        cp = (C.c_void_p * ns)(*[c.data_ptr() for _, c, _ in o])
        cs = (C.c_size_t * ns)(*[c.shape[1] for _, c, _ in o])

        def one():
            assert lib.lzgpu_encode_slices(eng.h, garr, ns, n, clen, host.data_ptr(), clen, pp, ps, cp, cs) == 0

        def per():
            for g, (p, c, m) in zip(goals, outs["per"]):
                if g.is_std:
                    assert lib.lzgpu_crc_blocks(eng.h, host.data_ptr(), n * nb, BLOCK, BLOCK, c.data_ptr()) == 0
                else:
                    assert lib.lzgpu_encode_chunks(eng.h, C.byref(g.c), n, clen, host.data_ptr(), clen, p.data_ptr(), p.shape[1], c.data_ptr(),
                                                   c.shape[1]) == 0
        ta, tb = alternate(one, per, 1)
        ok = all((m == 0 or torch.equal(p1, p2)) and torch.equal(c1, c2) for (p1, c1, m), (p2, c2, _) in zip(outs["one"], outs["per"]))
        row("host", names, n, clen, ta, tb, ok)
    eng.close()
    result = dict(card=info, rows=rows)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(dict(card=info, rows=[{k: v for k, v in r.items() if k in ("kind", "slices", "speedup", "same_bytes")} for r in rows])))


if __name__ == "__main__":
    main()
