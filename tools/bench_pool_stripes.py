"""The chunkserver's stripe consistency job over a pool of devices against one context: lzgpu_pool_repair_stripes and
lzgpu_pool_check_stripe_map against lzgpu_repair_stripes and lzgpu_check_stripe_map on the same host batch.

Workload: `--chunks` full 64 MiB chunks of ec(8,2) and of ec(8,4), every part and its stored CRCs in page-locked host memory (what a
chunkserver's block pool registers), with one rotten block (bytes changed, stored CRC kept) in part 3 of every fourth chunk.  The
repair rebuilds those blocks in place, so before every timed repair they are rotten again (host byte flips, outside the timed
region).  Each call is timed with a host clock (the host-pointer calls return when every result is in the caller's buffers); the one
context and the pool alternate, `--reps` times each after a warm-up, and the median is reported as GiB/s of chunk data.  The pool has
one slot per visible device, or [0, 0] (two contexts, two host pipelines on one GPU) when there is one; then the line says that
multi-GPU scaling is not shown.  The pool's map and repair entries and repaired bytes must equal the one context's.  The device names
and power limits are read in the same run and printed with every line.

    python tools/bench_pool_stripes.py [--chunks 16] [--reps 5]      (one JSON line per measurement)
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lizardfs_b200 as L  # noqa: E402

BLOCK = 65536
NB = 1024


def cards():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 else [torch.cuda.get_device_name(d) for d in range(torch.cuda.device_count())]


def pinned(shape, dtype):
    return torch.empty(shape, dtype=dtype, pin_memory=True).numpy()


def batch(eng, text, n):
    """every part [n, pb * 64 KiB] and its stored CRCs [n, pb], page-locked; the encode runs a chunk at a time"""
    goal = L.SliceType(text)
    k, m = goal.k, goal.m
    pb = NB // k
    parts = [pinned((n, pb * BLOCK), torch.uint8) for _ in range(k + m)]
    crcs = [pinned((n, pb), torch.int32).view(np.uint32) for _ in range(k + m)]
    rng = np.random.default_rng(7)
    for c in range(n):
        data = rng.integers(0, 256, size=(1, NB * BLOCK), dtype=np.uint8)
        parity, _ = eng.encode_chunks(goal, data)
        for j, p in enumerate(eng.split_chunks(goal, data, NB) + [parity[:, r] for r in range(m)]):
            parts[j][c] = p.reshape(-1)
            crcs[j][c] = eng.crc_blocks(parts[j][c])
    return goal, parts, crcs


def rot(parts, n):
    """flip two bytes of block 5 of part 3 in every fourth chunk (twice = restored)"""
    for c in range(0, n, 4):
        parts[3][c, 5 * BLOCK + 100:5 * BLOCK + 102] ^= np.array([0x21, 0x42], dtype=np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=16)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    n_dev = torch.cuda.device_count()
    devices = list(range(n_dev)) if n_dev > 1 else [0, 0]
    info = {"devices": cards(), "pool": devices,
            "note": None if n_dev > 1 else "one visible device: the pool is two contexts on it, multi-GPU scaling is not shown"}
    eng = L.Engine(0)
    pool = L.Pool(devices)
    for text in ("ec(8,2)", "ec(8,4)"):
        goal, parts, crcs = batch(eng, text, args.chunks)
        pristine = [p.copy() for p in parts]
        rot(parts, args.chunks)
        chunk_bytes = args.chunks * NB * BLOCK
        for what in ("check_stripe_map", "repair_stripes"):
            times = {"context": [], "pool": []}
            results = {}
            for rep in range(args.reps + 1):
                for name, obj in (("context", eng), ("pool", pool)):
                    t0 = time.perf_counter()
                    try:
                        out = getattr(obj, what)(goal, NB, parts, crcs)
                    except L.ChunkCrcError as e:     # the map reports the rotten blocks; its entries are written all the same
                        out = e.map if hasattr(e, "map") else e.fix
                    dt = time.perf_counter() - t0
                    if what == "repair_stripes":
                        assert all((p == q).all() for p, q in zip(parts, pristine)), "the repair did not restore the parts"
                        rot(parts, args.chunks)      # rotten again for the next call, outside the timed region
                    if rep:
                        times[name].append(dt)
                    results[name] = out.tobytes()
            assert results["pool"] == results["context"], "the pool's entries differ from the one context's"
            t_ctx, t_pool = statistics.median(times["context"]), statistics.median(times["pool"])
            print(json.dumps({"what": what, "goal": text, "chunks": args.chunks, "chunk_mib": NB * BLOCK >> 20,
                              "rotten_blocks": len(range(0, args.chunks, 4)),
                              "context_gib_s": round(chunk_bytes / t_ctx / 2**30, 2), "pool_gib_s": round(chunk_bytes / t_pool / 2**30, 2),
                              "pool_over_context": round(t_ctx / t_pool, 3), "context_s": round(t_ctx, 4), "pool_s": round(t_pool, 4),
                              "results_equal": True, **info}), flush=True)
        del parts, crcs, pristine
    pool.close()
    eng.close()


if __name__ == "__main__":
    main()
