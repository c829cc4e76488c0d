#!/usr/bin/env python
"""Mixed-goal sweep (BASELINE.json configs[1], [3], [4]): GiB/s of chunk data and fraction of the measured HBM
peak for encode+CRC over goals x chunk sizes, and for degraded-read recover, inputs resident in HBM, one GPU.
Prints a markdown table (and writes it to --out when given).  Not the headline bench — that is bench.py."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lizardfs_b200 as L  # noqa: E402

BLOCK = 65536
GIB = float(1 << 30)


def alg_bytes_encode(k, m, chunk_len):
    nb = (chunk_len + BLOCK - 1) // BLOCK
    pb = (nb + k - 1) // k
    return chunk_len + m * pb * BLOCK + 4 * (nb + m * pb)


ENGINE = None
NVML = None


def sm_clock():
    """current SM clock (MHz) right after a timed loop: long sweeps run into the power cap and the kernels that are not purely
    DRAM-bound follow the clock — the column attributes row-to-row differences of the same shape"""
    global NVML
    try:
        import pynvml
        if NVML is None:
            pynvml.nvmlInit()
            NVML = pynvml.nvmlDeviceGetHandleByIndex(0)
        return pynvml.nvmlDeviceGetClockInfo(NVML, pynvml.NVML_CLOCK_SM)
    except Exception:
        return 0


LAST = {"mhz": 0}


def time_steps(fn, steps, warmup, stream):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record(stream)
    for _ in range(steps):
        fn()
    ev[1].record(stream)
    for _ in range(2):
        fn()            # keep the device busy while the clock is read
    LAST["mhz"] = sm_clock()
    torch.cuda.synchronize()
    if ENGINE is not None:
        ENGINE.sync()   # raises if a deferred verification failed
    return ev[0].elapsed_time(ev[1]) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", help="also write the table to this file")
    ap.add_argument("--bytes", type=int, default=8 << 30, help="chunk data per launch")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--full-size-only", action="store_true", help="all goals, 64 MiB chunks only")
    ap.add_argument("--sections", default="enc,scrub,rec,conv,bw", help="comma list of enc,scrub,rec,conv,bw")
    ap.add_argument("--goals", default="", help="comma-free list separated by ';' of encode goals, e.g. 'ec(8,4);ec(5,3)'")
    ap.add_argument("--rec", default="", help="recover cases 'goal:lost,lost;...' e.g. 'ec(5,3):0,1,4;ec(3,2):0,2'")
    ap.add_argument("--rec-variants", default="both", choices=["both", "plain", "full"])
    args = ap.parse_args()
    sections = set(args.sections.split(","))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    eng = L.Engine(0)
    # the timed launches are issued back to back: verdicts of the verifying calls are collected by eng.sync() after each loop
    eng.set_deferred_verify(True)
    global ENGINE
    ENGINE = eng
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    sp = stream.cuda_stream
    peaks = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(peaks):
        peak, peak_src = float(json.load(open(peaks))["hbm_gbs"]), "measured HBM copy peak"
    else:
        peak, peak_src = 3350.0, "H100 SXM data-sheet HBM3 bandwidth, not measured"
    lines = [f"# Mixed-goal sweep, 1 x {torch.cuda.get_device_name()}, inputs resident in HBM", "",
             f"`python tools/sweep.py` — {args.bytes / GIB:.0f} GiB of chunk data per launch, {args.steps} timed launches, CUDA events; "
             f"frac = algorithmic bytes / time / {peak:.1f} GB/s ({peak_src}).", "",
             "## encode + per-block CRC32", "", "| goal | chunk | chunks/launch | ms | GiB/s data | GB/s algorithmic | frac of measured HBM | SM MHz |", "|---|---|---|---|---|---|---|---|"]
    goals = ["xor2", "xor3", "ec(3,2)", "ec(5,3)", "ec(8,2)", "ec(8,4)"]
    sizes = [1 << 20, 4 << 20, 16 << 20, 64 << 20, (37 << 20) + 5 * BLOCK]
    if args.quick:
        goals, sizes = ["ec(3,2)", "ec(8,2)"], [64 << 20]
    if args.full_size_only:
        sizes = [64 << 20]
    if args.goals:
        goals = [g for g in args.goals.split(";") if g]
    if "enc" not in sections:
        goals = []
    d_data = torch.empty(args.bytes, dtype=torch.uint8, device=dev)
    eng.fill_chunks_dev(d_data.data_ptr(), args.bytes // (64 << 20), 64 << 20, 64 << 20, seed=12345, stream=sp)
    for text in goals:
        g = L.SliceType(text)
        for clen in sizes:
            nb = (clen + BLOCK - 1) // BLOCK
            pb = (nb + g.k - 1) // g.k
            stride = nb * BLOCK
            n = args.bytes // stride
            par_stride, crc_stride = g.m * pb * BLOCK, nb + g.m * pb
            d_par = torch.empty(n * par_stride, dtype=torch.uint8, device=dev)
            d_crc = torch.empty(n * crc_stride, dtype=torch.int32, device=dev)
            ms = time_steps(lambda: eng.encode_chunks_dev(g, n, clen, d_data.data_ptr(), stride, d_par.data_ptr(), par_stride,
                                                          d_crc.data_ptr(), crc_stride, stream=sp), args.steps, args.warmup, stream)
            gibs = n * clen / GIB / (ms / 1e3)
            gbs = n * alg_bytes_encode(g.k, g.m, clen) / (ms / 1e3) / 1e9
            label = f"{clen / (1 << 20):.2f} MiB"
            lines.append(f"| {text} | {label} | {n} | {ms:.3f} | {gibs:.0f} | {gbs:.0f} | {gbs / peak:.3f} | {LAST['mhz']} |")
            del d_par, d_crc
    # scrub: CRC32 of every 64 KiB block of the resident buffer (hdd_int_test, hddspacemgr.cc:2174-2190)
    nblk = args.bytes // BLOCK
    if "scrub" in sections:
        d_c = torch.empty(nblk, dtype=torch.int32, device=dev)
        ms = time_steps(lambda: eng.crc_blocks_dev(d_data.data_ptr(), nblk, d_c.data_ptr(), stream=sp), args.steps, args.warmup, stream)
        gbs = (args.bytes + 4 * nblk) / (ms / 1e3) / 1e9
        lines += ["", "## scrub (CRC32 of 64 KiB blocks, fused kernel with M = 0)", "", "| blocks | ms | GiB/s | GB/s algorithmic | frac |", "|---|---|---|---|---|",
                  f"| {nblk} | {ms:.3f} | {args.bytes / GIB / (ms / 1e3):.0f} | {gbs:.0f} | {gbs / peak:.3f} |"]
        del d_c
    # degraded read: ec(8,2), data parts 1 and 4 lost (BASELINE configs[3]); also ec(3,2) / ec(5,3) / xor3
    lines += ["", "## degraded-read recover (stored CRCs verified, chunk-order image written)", "",
              "| goal | lost parts | chunks/launch | variant | ms | GiB/s chunk data | GB/s algorithmic | frac | SM MHz |", "|---|---|---|---|---|---|---|---|---|"]
    cases = [("ec(8,2)", (1, 4)), ("ec(8,2)", (0,)), ("ec(3,2)", (0, 2)), ("ec(5,3)", (0, 1, 4)), ("xor3", (1,))]
    if args.quick:
        cases = cases[:1]
    if args.rec:
        cases = [(c.split(":")[0], tuple(int(x) for x in c.split(":")[1].split(","))) for c in args.rec.split(";") if c]
    if "rec" not in sections and "conv" not in sections:
        cases = []
    elif "rec" not in sections:
        cases = [("ec(8,2)", (1, 4))]
    variants_sel = {"both": (0, 1), "plain": (0,), "full": (1,)}[args.rec_variants]
    conv_src = None
    clen = 64 << 20
    nb = clen // BLOCK
    for text, lost in cases:
        g = L.SliceType(text)
        k, m = g.k, g.m
        pb = (nb + k - 1) // k
        n = min(args.bytes // clen, 64)
        part_stride = pb * BLOCK
        # build part-major parts from an encode of the resident data (parity) + a gather of the data parts on the host side of torch
        d_par = torch.empty(n * m * part_stride, dtype=torch.uint8, device=dev)
        d_crc = torch.empty(n * (nb + m * pb), dtype=torch.int32, device=dev)
        eng.encode_chunks_dev(g, n, clen, d_data.data_ptr(), clen, d_par.data_ptr(), m * part_stride, d_crc.data_ptr(), nb + m * pb, stream=sp)
        torch.cuda.synchronize()
        chunks = d_data[: n * clen].view(n, nb, BLOCK)
        parts, pcrc = [], []
        crc_all = d_crc.view(n, nb + m * pb)
        for j in range(k):
            pj = torch.zeros((n, pb, BLOCK), dtype=torch.uint8, device=dev)
            blk = chunks[:, j::k]
            pj[:, : blk.shape[1]] = blk
            parts.append(pj.contiguous())
            cj = torch.full((n, pb), -0x28687115, dtype=torch.int32, device=dev)  # 0xD7978EEB as int32 (zero padding blocks)
            cj[:, : blk.shape[1]] = crc_all[:, j:nb:k]
            pcrc.append(cj.contiguous())
        for r in range(m):
            parts.append(d_par.view(n, m, part_stride)[:, r].contiguous())
            pcrc.append(crc_all[:, nb + r * pb: nb + (r + 1) * pb].contiguous())
        outs = [torch.empty((n, part_stride), dtype=torch.uint8, device=dev) if i in lost else None for i in range(k + m)]
        img = torch.empty((n, nb * BLOCK), dtype=torch.uint8, device=dev)
        dp = [0 if i in lost else parts[i].data_ptr() for i in range(k + m)]
        dc = [0 if i in lost else pcrc[i].data_ptr() for i in range(k + m)]
        do = [outs[i].data_ptr() if i in lost else 0 for i in range(k + m)]
        want = [1 if i in lost else 0 for i in range(k + m)]
        e = len([i for i in lost if i < k])
        for vi, (variant, crcs, image) in enumerate([("recover only", None, None), ("verify + recover + image", dc, img)]):
            if vi not in variants_sel:
                continue
            ms = time_steps(lambda: eng.recover_chunks_dev(g, n, nb, dp, part_stride, crcs, want, do, image.data_ptr() if image is not None else None,
                                                           nb * BLOCK, stream=sp), args.steps, args.warmup, stream)
            alg = k * pb * BLOCK + e * pb * BLOCK + (4 * k * pb + nb * BLOCK if crcs is not None else 0)
            gibs = n * clen / GIB / (ms / 1e3)
            gbs = n * alg / (ms / 1e3) / 1e9
            lines.append(f"| {text} | {list(lost)} | {n} | {variant} | {ms:.3f} | {gibs:.0f} | {gbs:.0f} | {gbs / peak:.3f} | {LAST['mhz']} |")
        # correctness spot check of the timed outputs
        torch.cuda.synchronize()
        for i in lost:
            if i < k:
                assert torch.equal(outs[i].view(n, pb, BLOCK), parts[i]), (text, i)
        if 1 in variants_sel:
            assert torch.equal(img.view(n, nb, BLOCK), chunks)
        if text == "ec(8,2)" and lost == (1, 4) or args.quick:
            conv_src = (g, n, nb, pb, dp, dc)
            conv_keep = (parts, pcrc)
        del parts, pcrc, outs, img, d_par, d_crc

    # ---- replication: slice-type conversion (SliceRecoveryPlanner) --------------------------------------------------
    lines += ["", "## slice-type conversion for replication (source CRCs verified, destination block CRCs produced)", "",
              "| source | destination parts | chunks/launch | ms | GiB/s chunk data | GB/s algorithmic | frac |", "|---|---|---|---|---|---|---|"]
    conv_cases = [("ec(3,2)", "all"), ("ec(3,2)", "one parity"), ("std", "all"), ("xor3", "all")]
    if "conv" not in sections or conv_src is None:
        conv_cases = []
    else:
        g, n, nb, pb, dp, dc = conv_src
    for dst_text, want_parts in conv_cases:
        d = L.SliceType(dst_text)
        nd = d.k + d.m
        pbd = (nb + d.k - 1) // d.k
        want = [1] * nd if want_parts == "all" else [0] * (nd - 1) + [1]
        outs = [torch.empty((n, pbd * BLOCK), dtype=torch.uint8, device=dev) if want[i] else None for i in range(nd)]
        ocrc = [torch.empty((n, pbd), dtype=torch.int32, device=dev) if want[i] else None for i in range(nd)]
        ms = time_steps(lambda: eng.convert_chunks_dev(g, d, n, nb, dp, pb * BLOCK, want, [o.data_ptr() if o is not None else 0 for o in outs], pbd * BLOCK,
                                                       d_part_crc=dc, d_out_crc=[o.data_ptr() if o is not None else 0 for o in ocrc], stream=sp),
                        args.steps, args.warmup, stream)
        # algorithmic bytes (DESIGN 4.5): the k source parts that are read + their stored CRCs, every wanted destination part + its CRCs, once
        alg = n * (g.k * pb * (BLOCK + 4) + sum(want) * pbd * (BLOCK + 4))
        gbs = alg / (ms / 1e3) / 1e9
        lines.append(f"| ec(8,2), data parts 1 and 4 lost | {dst_text}: {want_parts} | {n} | {ms:.3f} | {n * clen / GIB / (ms / 1e3):.0f} | {gbs:.0f} | {gbs / peak:.3f} |")
        torch.cuda.synchronize()
        if dst_text == "std":
            assert torch.equal(outs[0].view(n, nb, BLOCK), chunks)
        del outs, ocrc
    conv_keep = None

    # ---- chunkserver block writes (hdd_write) -------------------------------------------------------------------------
    lines += ["", "## batched chunkserver block writes (packet CRC check + stored-block check + new CRC)", "",
              "| requests | bytes per request | ms | requests/s | GB/s of stored blocks read |", "|---|---|---|---|---|"]
    import ctypes as C
    import zlib
    import numpy as np
    from lizardfs_b200 import _lib
    nreq = 16384
    for size in ((4096, 65535) if "bw" in sections else ()):
        blocks = d_data[: nreq * BLOCK]
        crc_t = torch.empty(nreq, dtype=torch.int32, device=dev)
        eng.crc_blocks_dev(blocks.data_ptr(), nreq, crc_t.data_ptr(), stream=sp)
        payload_h = np.random.default_rng(1).integers(0, 256, size, dtype=np.uint8)
        pcrc = zlib.crc32(payload_h.tobytes())
        payload = torch.from_numpy(payload_h).to(dev)
        arr = (_lib.LzBlockWrite * nreq)()
        for i in range(nreq):
            arr[i].block, arr[i].offset, arr[i].size, arr[i].crc, arr[i].payload_off, arr[i].exists = i, (i * 37) % (BLOCK - size + 1), size, pcrc, 0, 1
        d_wr = torch.empty(C.sizeof(arr), dtype=torch.uint8, device=dev)
        d_wr.copy_(torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8))
        torch.cuda.synchronize()
        # every launch re-applies the same payload: the first one changes the blocks, later ones find them already patched (the stored
        # CRC was updated by the first), so each timed launch does the full read-check-update work
        ms = time_steps(lambda: _lib.load().lzgpu_write_blocks_dev(eng.h, blocks.data_ptr(), crc_t.data_ptr(), payload.data_ptr(), d_wr.data_ptr(), nreq, 1,
                                                                  sp), args.steps, args.warmup, stream)
        st = np.frombuffer(d_wr.cpu().numpy().tobytes(), dtype=np.int32).reshape(nreq, 8)[:, 7]
        assert (st == 0).all(), st[:8]
        lines.append(f"| {nreq} | {size} | {ms:.3f} | {nreq / (ms / 1e3):.3g} | {nreq * BLOCK / (ms / 1e3) / 1e9:.0f} |")
    eng.fill_chunks_dev(d_data.data_ptr(), args.bytes // (64 << 20), 64 << 20, 64 << 20, seed=12345, stream=sp)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        open(args.out, "w").write("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
