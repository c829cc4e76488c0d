"""Time the salvage of the determined blocks of a multi-slice goal's chunks (lzgpu_salvage_slices_dev).

Goal set ec(3,2) + ec(4,2), resident 64 MiB chunks on the device, stored CRCs verified, the image's block CRCs and map written:
  whole     ec(3,2) parts 0-3 and ec(4,2) parts 0, 1, 3 lost: every block is determined.  Timed against lzgpu_recover_slices_dev
            writing the chunk image only (no wanted part) on the same batch; the two calls alternate after a warm-up, CUDA events
            around each, and their images are compared after the timing.
  partial   the same with one more part lost, chosen so that some blocks are holes and some are still solved from parity blocks:
            lzgpu_recover_slices refuses it, so the salvage is timed alone.
Reports milliseconds per batch and GiB/s of chunk data (image bytes), with the card's name and power limit read in the same run.

    python tools/bench_salvage_slices.py [--chunks 16] [--iters 10] [--out results/bench_salvage_slices.json]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import lizardfs_b200 as L  # noqa: E402
from tools.bench_recover_slices import BLOCK, NB, card, flat_parts, timed  # noqa: E402

WHOLE = [0, 0, 0, 0, 1, 0, 0, 1, 0, 1, 1]


def partial_pattern(goals):
    """WHOLE with one more given part lost: the first such pattern that leaves holes and still solves a block from parity"""
    for g in range(len(WHOLE)):
        if not WHOLE[g]:
            continue
        given = [0 if h == g else x for h, x in enumerate(WHOLE)]
        p = L.Engine.plan_salvage_slices(goals, NB, given)
        if p["determined"] != (1 << p["L"]) - 1 and p["determined"] & ~p["known"]:
            return given
    raise RuntimeError("no partial pattern with solved blocks")


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
    img = torch.zeros(n * NB * BLOCK, dtype=torch.uint8, device="cuda")
    icrc = torch.zeros(n * NB, dtype=torch.int32, device="cuda")
    smap = torch.zeros(n * NB, dtype=torch.uint8, device="cuda")
    rimg = torch.zeros_like(img)
    rows = []

    def ptrs(ts):
        return [t.data_ptr() if t is not None else 0 for t in ts]

    for name, given in (("whole", WHOLE), ("partial", partial_pattern(goals))):
        d_in = [p if x else None for p, x in zip(parts, given)]
        d_c = [c if x else None for c, x in zip(crcs, given)]

        def salvage():
            eng.salvage_slices_dev(goals, n, NB, ptrs(d_in), strides, ptrs(d_c), img.data_ptr(), NB * BLOCK, icrc.data_ptr(), smap.data_ptr())

        def recover():
            eng.recover_slices_dev(goals, n, NB, ptrs(d_in), strides, ptrs(d_c), [0] * 11, [0] * 11, strides, None, rimg.data_ptr(),
                                   NB * BLOCK)

        row = {"pattern": name, "given": given, "chunks": n, "card": card()}
        if name == "whole":
            for f in (salvage, recover):
                timed(f, 2)
            t1, t2 = [], []
            for _ in range(3):
                t1.append(timed(salvage, a.iters))
                t2.append(timed(recover, a.iters))
            row.update(salvage_ms=min(t1), recover_image_ms=min(t2), same_image=bool(torch.equal(img, rimg)),
                       salvage_gibs=chunk_gib / (min(t1) / 1e3), recover_image_gibs=chunk_gib / (min(t2) / 1e3))
        else:
            timed(salvage, 2)
            t = min(timed(salvage, a.iters) for _ in range(3))
            counts = torch.bincount(smap.long(), minlength=4).tolist()
            row.update(salvage_ms=t, salvage_gibs=chunk_gib / (t / 1e3), blocks_hole_known_solved_withheld=counts)
        print(json.dumps(row))
        rows.append(row)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)
    eng.close()


if __name__ == "__main__":
    main()
