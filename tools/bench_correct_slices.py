"""Time the correction of a multi-slice goal's chunks (lzgpu_correct_slices_dev) against the consistency map alone
(lzgpu_check_slices_dev) on the same inputs.

Resident 64 MiB chunks on the device, every part given, stored CRCs verified, new CRCs written, for ec(3,2) + ec(4,2) and
std + xor2 + xor3:
  clean     the correction and the check alternate after a warm-up, CUDA events around each.  Every entry must be CLEAN and no part
            may change.
  stale     one block of the last part rewritten in one combined stripe of every chunk (its stored CRC recomputed), so that the locate
            pass and correct_slices_kernel run on one entry per chunk.  The stale block is restored from a copy before every call,
            outside the events.  Every chunk's entry for that stripe must be CORRECTED with that part named, and the corrected part
            must equal the encoded original.
Reports milliseconds per batch and GiB/s of chunk data, with the card's name and power limit read in the same run.

    python tools/bench_correct_slices.py [--chunks 16] [--iters 10] [--out results/bench_correct_slices.json]
"""
import argparse
import json
import os
import sys
import zlib

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lizardfs_b200 as L  # noqa: E402
from lizardfs_b200 import _lib  # noqa: E402
from tools.bench_check_slices import SETS  # noqa: E402
from tools.bench_recover_slices import BLOCK, NB, card, flat_parts, timed  # noqa: E402


def timed_each(fn, before, iters):
    """mean milliseconds of fn() over iters calls, with before() run outside the events ahead of each"""
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    for _ in range(iters):
        before()
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        total += s.elapsed_time(e)
    return total / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=16)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n = a.chunks
    eng = L.Engine(0)
    chunk_gib = n * NB * BLOCK / 2**30
    rows = []
    for name, goals in SETS.items():
        parts, crcs, pbs = flat_parts(eng, goals, n)
        n_parts = len(parts)
        Lc = L.Engine.plan_check_slices(goals, NB, [1] * n_parts)["L"]
        n_cs = -(-NB // Lc)
        strides, base = [], 0
        for g in goals:
            strides.append(pbs[base] * BLOCK)
            base += g.k + g.m
        dmap = torch.zeros(n * n_cs * 2, dtype=torch.int64, device="cuda")
        dfix = torch.zeros(n * n_cs * 4, dtype=torch.int64, device="cuda")
        new_crc = [torch.zeros_like(c) for c in crcs]

        def ptrs(ts):
            return [t.data_ptr() for t in ts]

        def check():
            eng.check_slices_dev(goals, n, NB, ptrs(parts), strides, ptrs(crcs), dmap.data_ptr())

        def correct():
            eng.correct_slices_dev(goals, n, NB, ptrs(parts), strides, ptrs(crcs), ptrs(new_crc), dfix.data_ptr())

        def fix():
            torch.cuda.synchronize()
            return dfix.cpu().numpy().view(L.Engine.SLICES_FIX_DTYPE).reshape(n, n_cs)

        row = {"goals": name, "chunks": n, "card": card()}
        g = n_parts - 1
        orig = parts[g].clone()
        for f in (check, correct):
            timed(f, 2)
        t1, t2 = [], []
        for _ in range(3):
            t1.append(timed(correct, a.iters))
            t2.append(timed(check, a.iters))
        m = fix()
        assert (m["status"] == _lib.FIX_CLEAN).all() and (m["changed"] == 0).all(), "a clean batch has an entry that is not CLEAN"
        assert torch.equal(parts[g], orig), "a clean batch was changed"
        row.update(clean_correct_ms=min(t1), clean_check_ms=min(t2), clean_correct_gibs=chunk_gib / (min(t1) / 1e3),
                   clean_check_gibs=chunk_gib / (min(t2) / 1e3))
        # stale: block 3 of the last part rewritten in every chunk, with its stored CRC recomputed
        pb = pbs[g]
        host = orig.cpu().numpy().reshape(n, pb * BLOCK).copy()
        host[:, 3 * BLOCK + 100:3 * BLOCK + 164] ^= 0x5A
        hc = crcs[g].cpu().numpy().view(np.uint32).reshape(n, pb).copy()
        hc[:, 3] = [zlib.crc32(host[c, 3 * BLOCK:4 * BLOCK].tobytes()) for c in range(n)]
        stale = torch.from_numpy(host.reshape(-1)).cuda()
        crcs[g] = torch.from_numpy(hc.reshape(-1).view(np.int32)).cuda()

        def restore():
            parts[g].copy_(stale)

        timed_each(correct, restore, 2)
        t = min(timed_each(correct, restore, a.iters) for _ in range(3))
        m = fix()
        cs = 3 * goals[-1].k // Lc
        assert (m["status"][:, cs] == _lib.FIX_CORRECTED).all() and (m["suspect_part"][:, cs] == g).all(), "the stale part is not corrected"
        assert (m["status"] == _lib.FIX_CORRECTED).sum() == n, "an entry other than the stale one was corrected"
        assert torch.equal(parts[g], orig), "the corrected part differs from the original"
        restore()
        ts = min(timed(check, a.iters) for _ in range(3))
        row.update(stale_correct_ms=t, stale_check_ms=ts, stale_correct_gibs=chunk_gib / (t / 1e3))
        print(json.dumps(row))
        rows.append(row)
        del parts, crcs, new_crc
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
