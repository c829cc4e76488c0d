"""The recovery of a multi-slice goal from the parts of all its slices together over a pool of devices against one context:
lzgpu_pool_recover_slices against lzgpu_recover_slices on the same host batch.

Workload: ec(3,2) + ec(4,2), `--chunks` batches (16 and 64) of full 64 MiB chunks, the two patterns of DESIGN.md §5:
  survivor  ec(4,2) keeps parts 1..5 (its data part 0 lost), ec(3,2) is lost: every lost part of both slices is rebuilt;
  rescue    ec(3,2) parts 0-3 and ec(4,2) parts 0, 1, 3 lost (7 of 11 parts): no slice has k parts.
Every given part and its stored CRCs (verified by the call), every lost part and its block CRCs (written by the call) are in
page-locked host memory (what a chunkserver's block pool registers); the context and the pool read the same inputs and write their
own outputs.  Each call is timed with a host clock (a host-pointer call returns when every output is in the caller's buffers); the
one context and the pool alternate, `--reps` times each after a warm-up, and the median is reported as ms and GiB/s of chunk data.
The pool has one slot per visible device, or [0, 0] (two contexts, two host pipelines on one GPU) when there is one; then the line
says that multi-GPU scaling is not shown.  Before a line is printed the pool's outputs must equal the one context's, and every
chunk's outputs the original parts (every chunk of the batch is a copy of one encoded chunk).  The device names and power limits are read in the same run and printed with every line.

    python tools/bench_pool_recover_slices.py [--chunks 16,64] [--reps 5]      (one JSON line per measurement)
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time
import zlib

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lizardfs_b200 as L  # noqa: E402
from lizardfs_b200 import _lib  # noqa: E402
from lizardfs_b200.engine import _goal_array, _p, _ptr_array  # noqa: E402

BLOCK = 65536
NB = 1024
NAMES = ("ec(3,2)", "ec(4,2)")
PATTERNS = {"survivor": [0] * 5 + [0, 1, 1, 1, 1, 1], "rescue": [0, 0, 0, 0, 1, 0, 0, 1, 0, 1, 1]}


def cards():
    q = subprocess.run(["nvidia-smi", "--query-gpu=index,name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 else [torch.cuda.get_device_name(d) for d in range(torch.cuda.device_count())]


class Pinned:
    """numpy arrays page-locked with cudaHostRegister (exact sizes; torch's pinned allocator rounds up to a power of two)"""

    def __init__(self):
        self.arrays = []

    def __call__(self, shape, dtype):
        a = np.empty(shape, dtype=dtype)
        torch.cuda.check_error(torch.cuda.cudart().cudaHostRegister(a.ctypes.data, a.nbytes, 0))
        self.arrays.append(a)
        return a

    def release(self):
        for a in self.arrays:
            torch.cuda.check_error(torch.cuda.cudart().cudaHostUnregister(a.ctypes.data))
        self.arrays.clear()


def original(eng, goals):
    """one random chunk's flat parts [pb_g * 64 KiB] and their block CRCs [pb_g], from lzgpu_encode_slices"""
    data = np.random.default_rng(1).integers(0, 256, size=(1, NB * BLOCK), dtype=np.uint8)
    parts, crcs = [], []
    for g, (par, crc) in zip(goals, eng.encode_slices(goals, data)):
        k, pb = g.k, -(-NB // g.k)
        padded = np.zeros(pb * k * BLOCK, dtype=np.uint8)
        padded[:NB * BLOCK] = data[0]
        blocks = padded.reshape(pb, k, BLOCK)
        for j in range(k):
            c = np.full(pb, zlib.crc32(bytes(BLOCK)), dtype=np.uint32)
            idx = np.arange(pb) * k + j
            c[idx < NB] = crc[0, idx[idx < NB]]
            parts.append(np.ascontiguousarray(blocks[:, j]).reshape(-1))
            crcs.append(c)
        for r in range(g.m):
            parts.append(par[0, r].copy())
            crcs.append(crc[0, NB + r * pb: NB + (r + 1) * pb].copy())
    return parts, crcs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", default="16,64")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    sizes = [int(x) for x in args.chunks.split(",")]
    n_dev = torch.cuda.device_count()
    devices = list(range(n_dev)) if n_dev > 1 else [0, 0]
    info = {"devices": cards(), "pool": devices,
            "note": None if n_dev > 1 else "one visible device: the pool is two contexts on it, multi-GPU scaling is not shown"}
    eng = L.Engine(0)
    pool = L.Pool(devices)
    lib = eng.lib
    goals = [L.SliceType(n) for n in NAMES]
    garr = _goal_array(goals)
    pbs = [-(-NB // g.k) for g in goals]
    slice_of = [i for i, g in enumerate(goals) for _ in range(g.k + g.m)]
    strides = (C.c_size_t * 2)(*[pb * BLOCK for pb in pbs])
    src, src_crc = original(eng, goals)
    n_max = max(sizes)
    for pattern, given in PATTERNS.items():
        pin = Pinned()
        want = np.array([0 if x else 1 for x in given], dtype=np.uint8)
        size = [pbs[slice_of[g]] for g in range(11)]
        parts = [None] * 11
        crcs = [None] * 11
        for g in range(11):
            if given[g]:
                parts[g] = pin((n_max, size[g] * BLOCK), np.uint8)
                parts[g][:] = src[g]
                crcs[g] = pin((n_max, size[g]), np.uint32)
                crcs[g][:] = src_crc[g]
        outs = {who: ([pin((n_max, size[g] * BLOCK), np.uint8) if want[g] else None for g in range(11)],
                      [pin((n_max, size[g]), np.uint32) if want[g] else None for g in range(11)]) for who in ("context", "pool")}
        calls = {"context": (lib.lzgpu_recover_slices, eng.h), "pool": (lib.lzgpu_pool_recover_slices, pool.h)}
        for n in sizes:
            times = {"context": [], "pool": []}
            for rep in range(args.reps + 1):
                for who, (fn, h) in calls.items():
                    o, oc = outs[who]
                    bad = (C.c_int64 * 4)(-1, -1, -1, -1)
                    t0 = time.perf_counter()
                    rc = fn(h, garr, 2, n, NB, _ptr_array(parts), strides, _ptr_array(crcs), _p(want), _ptr_array(o), strides, _ptr_array(oc),
                            None, 0, bad)
                    dt = time.perf_counter() - t0
                    assert rc == _lib.OK, (who, rc, _lib.last_error())
                    if rep:
                        times[who].append(dt)
            for g in range(11):
                if not want[g]:
                    continue
                for (x, y, ref) in ((outs["pool"][0][g], outs["context"][0][g], src[g]), (outs["pool"][1][g], outs["context"][1][g], src_crc[g])):
                    assert np.array_equal(x[:n], y[:n]), f"the pool's part {g} differs from the one context's"
                    assert (x[:n] == ref).all(), f"part {g} differs from the original"     # every chunk of the batch is the same chunk
            t_ctx, t_pool = statistics.median(times["context"]), statistics.median(times["pool"])
            chunk_gib = n * NB * BLOCK / 2**30
            print(json.dumps({"pattern": pattern, "goals": "+".join(NAMES), "chunks": n, "chunk_mib": NB * BLOCK >> 20,
                              "context_ms": round(t_ctx * 1e3, 2), "pool_ms": round(t_pool * 1e3, 2),
                              "context_gib_s": round(chunk_gib / t_ctx, 2), "pool_gib_s": round(chunk_gib / t_pool, 2),
                              "pool_over_context": round(t_ctx / t_pool, 3), "outputs_equal": True, **info}), flush=True)
        pin.release()
        del parts, crcs, outs
    pool.close()
    eng.close()


if __name__ == "__main__":
    main()
