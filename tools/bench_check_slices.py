"""Time the consistency map of a multi-slice goal's chunks (lzgpu_check_slices_dev) against lzgpu_recover_slices_dev on the same inputs.

Resident 64 MiB chunks on the device, every part given, stored CRCs verified, for ec(3,2) + ec(4,2) and std + xor2 + xor3:
  clean     the check, and lzgpu_recover_slices_dev writing the chunk image from the same parts; the two calls alternate after a
            warm-up, CUDA events around each.  Every entry must be {0, -1, 0}.
  stale     one block of the last part rewritten in one combined stripe of every chunk (its stored CRC recomputed), so that the locate
            pass runs on one entry per chunk.  Every chunk's entry for that stripe must name that part, and no other entry may be bad.
Reports milliseconds per batch and GiB/s of chunk data, with the card's name and power limit read in the same run.

    python tools/bench_check_slices.py [--chunks 16] [--iters 10] [--out results/bench_check_slices.json]
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
from tools.bench_recover_slices import BLOCK, NB, card, flat_parts, timed  # noqa: E402

SETS = {"ec(3,2)+ec(4,2)": [L.SliceType("ec(3,2)"), L.SliceType("ec(4,2)")],
        "std+xor2+xor3": [L.SliceType(2, 1, 0), L.SliceType("xor2"), L.SliceType("xor3")]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=16)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n = a.chunks
    eng = L.Engine(0)
    chunk_gib = n * NB * BLOCK / 2**30
    img = torch.zeros(n * NB * BLOCK, dtype=torch.uint8, device="cuda")
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

        def ptrs(ts):
            return [t.data_ptr() for t in ts]

        def check():
            eng.check_slices_dev(goals, n, NB, ptrs(parts), strides, ptrs(crcs), dmap.data_ptr())

        def recover():
            eng.recover_slices_dev(goals, n, NB, ptrs(parts), strides, ptrs(crcs), [0] * n_parts, [0] * n_parts, strides, None,
                                   img.data_ptr(), NB * BLOCK)

        def entries():
            torch.cuda.synchronize()
            return dmap.cpu().numpy().view(L.Engine.SLICES_CHECK_DTYPE).reshape(n, n_cs)

        row = {"goals": name, "chunks": n, "card": card()}
        for f in (check, recover):
            timed(f, 2)
        t1, t2 = [], []
        for _ in range(3):
            t1.append(timed(check, a.iters))
            t2.append(timed(recover, a.iters))
        m = entries()
        assert (m["bad_checks"] == 0).all() and (m["suspect_part"] == -1).all(), "a clean batch has a bad entry"
        row.update(clean_check_ms=min(t1), recover_image_ms=min(t2), clean_check_gibs=chunk_gib / (min(t1) / 1e3),
                   recover_image_gibs=chunk_gib / (min(t2) / 1e3))
        # stale: block 3 of the last part's chunk c, rewritten with its stored CRC recomputed, in every chunk
        g = n_parts - 1
        pb = pbs[g]
        host = parts[g].cpu().numpy().reshape(n, pb * BLOCK)
        host[:, 3 * BLOCK + 100:3 * BLOCK + 164] ^= 0x5A
        hc = crcs[g].cpu().numpy().view(np.uint32).reshape(n, pb)
        hc[:, 3] = [zlib.crc32(host[c, 3 * BLOCK:4 * BLOCK].tobytes()) for c in range(n)]
        parts[g] = torch.from_numpy(host.reshape(-1)).cuda()
        crcs[g] = torch.from_numpy(hc.reshape(-1).view(np.int32)).cuda()
        timed(check, 2)
        t = min(timed(check, a.iters) for _ in range(3))
        m = entries()
        cs = 3 * (goals[-1].k) // Lc
        bad = m["bad_checks"] != 0
        assert bad[:, cs].all() and bad.sum() == n, "the stale stripe is not the only bad entry"
        assert (m["suspect_part"][:, cs] == g).all(), "the stale part is not named"
        row.update(stale_check_ms=t, stale_check_gibs=chunk_gib / (t / 1e3))
        print(json.dumps(row))
        rows.append(row)
        del parts, crcs
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
