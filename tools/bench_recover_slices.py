"""Time the recovery of a multi-slice goal from the parts of all its slices together (lzgpu_recover_slices_dev).

Goal set ec(3,2) + ec(4,2), resident 64 MiB chunks on the device, stored CRCs verified and the CRCs of every rebuilt part written:
  survivor  ec(4,2) keeps parts 1..5 (its data part 0 lost), ec(3,2) is lost: every lost part of both slices is rebuilt.  Timed
            against lzgpu_convert_chunks_dev from the surviving slice (ec(4,2) -> ec(3,2) for the five parts, ec(4,2) -> ec(4,2) for
            its part 0), which writes the same bytes; the two forms alternate after a warm-up, CUDA events around each, and their
            outputs are compared after the timing.
  rescue    ec(3,2) parts 0-3 and ec(4,2) parts 0, 1, 3 lost (7 of 11 parts): no slice has k parts, so only this call can rebuild
            the chunk.
Reports milliseconds per batch and GiB/s of chunk data, with the card's name and power limit read in the same run.

    python tools/bench_recover_slices.py [--chunks 16] [--iters 10] [--out results/bench_recover_slices.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lizardfs_b200 as L  # noqa: E402

BLOCK = 65536
NB = 1024


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def flat_parts(eng, goals, n):
    """every flat part of n identical chunks on the device, with its stored CRCs: (parts, crcs, pb per flat part)"""
    rng = np.random.default_rng(1)
    data = rng.integers(0, 256, size=(1, NB * BLOCK), dtype=np.uint8)
    enc = eng.encode_slices(goals, data)
    parts, crcs, pbs = [], [], []
    for g, (par, crc) in zip(goals, enc):
        k, pb = g.k, -(-NB // g.k)
        padded = np.zeros((pb * k * BLOCK,), dtype=np.uint8)
        padded[:NB * BLOCK] = data[0]
        blocks = padded.reshape(pb, k, BLOCK)
        zero_crc = np.uint32(0xD7978EEB)
        for j in range(k):
            c = np.full(pb, zero_crc, dtype=np.uint32)
            idx = np.arange(pb) * k + j
            c[idx < NB] = crc[0, idx[idx < NB]]
            parts.append(np.ascontiguousarray(blocks[:, j, :]).reshape(-1))
            crcs.append(c)
            pbs.append(pb)
        for r in range(g.m):
            parts.append(par[0, r].copy())
            crcs.append(crc[0, NB + r * pb: NB + (r + 1) * pb].copy())
            pbs.append(pb)
    dev = [torch.from_numpy(p).cuda().repeat(n) for p in parts]
    dcrc = [torch.from_numpy(c.view(np.int32)).cuda().repeat(n) for c in crcs]
    return dev, dcrc, pbs


def timed(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=16)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n = a.chunks
    eng = L.Engine(0)
    goals = [L.SliceType("ec(3,2)"), L.SliceType("ec(4,2)")]
    parts, crcs, pbs = flat_parts(eng, goals, n)
    strides = [pbs[0] * BLOCK, pbs[5] * BLOCK]
    chunk_gib = n * NB * BLOCK / 2**30
    rows = []

    def outputs(want):
        o = [torch.zeros(n * pbs[g] * BLOCK, dtype=torch.uint8, device="cuda") if want[g] else None for g in range(11)]
        c = [torch.zeros(n * pbs[g], dtype=torch.int32, device="cuda") if want[g] else None for g in range(11)]
        return o, c

    def ptrs(ts):
        return [t.data_ptr() if t is not None else 0 for t in ts]

    for name, given in (("survivor", [0] * 5 + [0, 1, 1, 1, 1, 1]), ("rescue", [0, 0, 0, 0, 1, 0, 0, 1, 0, 1, 1])):
        want = [0 if x else 1 for x in given]
        d_in = [p if x else None for p, x in zip(parts, given)]
        d_c = [c if x else None for c, x in zip(crcs, given)]
        out, ocrc = outputs(want)

        def one():
            eng.recover_slices_dev(goals, n, NB, ptrs(d_in), strides, ptrs(d_c), want, ptrs(out), strides, ptrs(ocrc))

        row = {"pattern": name, "chunks": n, "card": card()}
        if name == "survivor":
            src = goals[1]
            s_in, s_c = d_in[5:], d_c[5:]
            cout, ccrc = outputs(want)

            def per():
                eng.convert_chunks_dev(src, goals[0], n, NB, ptrs(s_in), strides[1], want[:5], ptrs(cout[:5]), strides[0], ptrs(s_c),
                                       ptrs(ccrc[:5]))
                eng.convert_chunks_dev(src, goals[1], n, NB, ptrs(s_in), strides[1], want[5:], ptrs(cout[5:]), strides[1], ptrs(s_c),
                                       ptrs(ccrc[5:]))

            for f in (one, per):
                timed(f, 2)
            t1, t2 = [], []
            for _ in range(2):
                t1.append(timed(one, a.iters))
                t2.append(timed(per, a.iters))
            same = all(torch.equal(x, y) for x, y in zip(out + ocrc, cout + ccrc) if x is not None)
            row.update(recover_slices_ms=min(t1), convert_ms=min(t2), same_bytes=same,
                       recover_slices_gibs=chunk_gib / (min(t1) / 1e3), convert_gibs=chunk_gib / (min(t2) / 1e3))
        else:
            timed(one, 2)
            t = min(timed(one, a.iters) for _ in range(2))
            row.update(recover_slices_ms=t, recover_slices_gibs=chunk_gib / (t / 1e3))
        print(json.dumps(row))
        rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
