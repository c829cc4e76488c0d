"""Throughput of the stripe check (lzgpu_check_stripes_dev) on resident 64 MiB chunks with stored CRCs.

For each goal: full chunks are generated on the device (lzgpu_fill_chunks_dev), split into parts and encoded in a chunk-major layout
(part i of chunk c at base + (c*(k+m) + i)*pb*64K), and every part block's CRC is stored per part.  The check is then timed with CUDA
events around `--iters` back-to-back calls after `--warmup` calls (deferred verification, so no call waits for the host).  Reported:
GiB/s of chunk data, and algorithmic bytes (every part read, its stored CRCs read, 12 bytes of verdict written) over time against the
H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s.  The ec(8,2) degraded read of the same batch (data parts 1 and 4 rebuilt, the eight
parts read verified) is timed in the same run as the streaming reference point.  On each goal's timed buffers one byte is then flipped
(its block CRC restored) and the fused and the generic route must return identical verdicts naming it.

The stripe map (lzgpu_check_stripe_map_dev) is timed next to the check on the same resident batch, alternating the two calls, in three
cases: a clean batch, one bad stripe per chunk (data part 3, stripe 5), and every stripe of every chunk bad (one byte of data part 0
per stripe).  Clean stripes cost the one pass; a bad one is re-read by a CTA of its own to name its suspect.  In every case the maps of
both routes must be identical and each chunk's lowest bad stripe must equal both routes' verdicts.

The stripe correction (lzgpu_correct_stripes_dev) is timed against the map on the same resident batch in the same three cases, with
CUDA events around each call only.  A correction repairs the batch, so before every timed call the faulty bytes are put back by device
copies on the same stream, outside the timed region.  With one bad stripe per chunk the existing route is timed too: the map, the map
back on the host, then one lzgpu_recover_chunks_dev call per bad stripe over a one-stripe window, writing the suspect's block in place.
In every case the fix entries of both routes must be identical and the corrected bytes must be the original ones.

The degraded map (lzgpu_check_stripe_map_degraded_dev) runs on the same kind of batch with data parts missing: ec(8,2) without part 1
(one spare), ec(5,3) without part 1, ec(8,3) without parts 1 and 4, ec(8,4) without part 1 and without parts 1 and 4.  Each row times
it on the fused and the generic route and times the full-parts map of the same goal, alternating the three calls twice.  Algorithmic
bytes are the given parts, their stored CRCs and the 8-byte map entries.  Both routes must return identical maps, clean and with one
stale input block per chunk, which they must name when there are two spares or more.

The stripe repair (lzgpu_repair_stripes_dev) runs on the same kind of batch for ec(8,2), ec(8,4) and xor3, in three cases, each
timed as the correction is (the rotten bytes put back before every call, outside the events): a clean batch, against
lzgpu_correct_stripes_dev; one rotten block (bytes changed, stored CRC kept) in each of the first k stripes of part 3 of every chunk,
against today's alternative, dropping part 3 and rebuilding it whole with lzgpu_recover_chunks_dev; and m rotten blocks in every
stripe, the worst case, alone.  Both routes must return identical entries, and the rebuilt bytes must be the original ones.

The stripe decode (lzgpu_decode_stripes_dev) is timed against the repair and the map on the same batch, alternated, as the repair is:
clean for ec(8,3), ec(8,4) and ec(10,5); two stale parts (bytes changed, stored CRCs recomputed) in each of the first k stripes of
every chunk (ec(8,4)); one stale and one rotten block there (ec(8,3)); two stale parts in every stripe (ec(8,4)).  The repair leaves
those stripes unfixed.  The cost per decoded stripe, (decode - repair) / decoded stripes, is reported next to the map's locate cost,
(map - clean map) / bad stripes.  Both routes must return identical entries, and the rewritten bytes must be the original ones.

    python tools/bench_check.py [--chunks 16] [--iters 20] [--warmup 3] [--only degraded|repair|decode]      (one JSON line per measurement)
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lizardfs_b200 as L  # noqa: E402
from lizardfs_b200 import _lib  # noqa: E402

BLOCK = 65536
NB = 1024
HBM_TBPS = 3.35
GOALS = ["ec(8,2)", "ec(5,3)", "ec(8,4)", "xor3", "ec(10,5)"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip().splitlines()[0] if q.returncode == 0 else None}


class Resident:
    """n full chunks of a goal on the device, chunk-major parts, per-part stored CRCs"""

    def __init__(self, eng, text, n, seed=1):
        self.goal = L.SliceType(text)
        k, m = self.goal.k, self.goal.m
        self.k, self.m, self.n = k, m, n
        self.pb = (NB + k - 1) // k
        self.part_bytes = self.pb * BLOCK
        self.stride = (k + m) * self.part_bytes
        data = torch.empty(n * NB * BLOCK, dtype=torch.uint8, device="cuda")
        eng.fill_chunks_dev(data.data_ptr(), n, NB * BLOCK, NB * BLOCK, seed)
        self.buf = torch.empty(n * self.stride, dtype=torch.uint8, device="cuda")
        base = self.buf.data_ptr()
        self.ptrs = [base + i * self.part_bytes for i in range(k + m)]
        eng.split_chunks_dev(self.goal, n, NB, data.data_ptr(), NB * BLOCK, self.ptrs[:k], self.stride)
        crc = torch.empty(n * (NB + m * self.pb), dtype=torch.int32, device="cuda")
        eng.encode_chunks_dev(self.goal, n, NB * BLOCK, data.data_ptr(), NB * BLOCK, self.ptrs[k], self.stride, crc.data_ptr(), NB + m * self.pb)
        del data, crc
        self.crc = torch.empty((k + m, n, self.pb), dtype=torch.int32, device="cuda")
        for i in range(k + m):
            for c in range(n):
                eng.crc_blocks_dev(self.ptrs[i] + c * self.stride, self.pb, self.crc[i, c].data_ptr())
        self.crc_ptrs = [self.crc[i].data_ptr() for i in range(k + m)]
        torch.cuda.synchronize()

    def alg_bytes(self):
        return self.n * ((self.k + self.m) * (self.part_bytes + 4 * self.pb) + 12)


def timed(call, iters, warmup, stream):
    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(iters):
        call()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3 / iters


def verdicts(eng, r, out):
    eng.check_stripes_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out.data_ptr())
    torch.cuda.synchronize()
    return out.cpu().numpy().view(L.Engine.VERDICT_DTYPE).copy()


def stripe_map(eng, r, out):
    eng.check_stripe_map_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out.data_ptr())
    torch.cuda.synchronize()
    return out.cpu().numpy().view(L.Engine.STRIPE_STATE_DTYPE).reshape(r.n, r.pb).copy()


def flip(eng, r, part, stripes, offset):
    """flip one byte of `part` in each of `stripes` of every chunk, and restore the stored CRCs of those blocks"""
    idx = torch.tensor([c * r.stride + part * r.part_bytes + s * BLOCK + offset for c in range(r.n) for s in stripes], device="cuda")
    r.buf[idx] ^= 0x5A
    for c in range(r.n):
        eng.crc_blocks_dev(r.ptrs[part] + c * r.stride, r.pb, r.crc[part, c].data_ptr())
    torch.cuda.synchronize()


def map_rows(eng, generic, r, text, args, stream, info):
    """time the map next to the check in the three cases, and check it against both routes' verdicts"""
    st = stream.cuda_stream
    out_v = torch.empty(12 * r.n, dtype=torch.uint8, device="cuda")
    out_m = torch.empty(8 * r.n * r.pb, dtype=torch.uint8, device="cuda")
    cases = [("clean", None), ("one_bad_stripe_per_chunk", (3, [5], 777)), ("every_stripe_bad", (0, range(r.pb), 4242))]
    for case, fault in cases:
        if fault:
            flip(eng, r, *fault)
        t_check = t_map = 0.0
        for _ in range(2):               # alternate the calls, twice: other work shares the card
            t_check += timed(lambda: eng.check_stripes_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_v.data_ptr(), stream=st),
                             args.iters, args.warmup, stream) / 2
            t_map += timed(lambda: eng.check_stripe_map_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_m.data_ptr(), stream=st),
                           args.iters, args.warmup, stream) / 2
        eng.sync()
        route = "fused" if eng.last_geometry()["kernel"] == _lib.KERNEL_CHECK else "generic"
        m_fused, m_generic = stripe_map(eng, r, out_m), stripe_map(generic, r, out_m)
        assert (m_fused == m_generic).all(), "fused and generic maps differ"
        for e in (eng, generic):
            v = verdicts(e, r, out_v)
            for c in range(r.n):
                bad = m_fused[c]["bad_rows"].nonzero()[0]
                first = (int(bad[0]), int(m_fused[c, bad[0]]["bad_rows"]), int(m_fused[c, bad[0]]["suspect_part"])) if len(bad) else (-1, 0, -1)
                assert first == tuple(int(x) for x in v[c]), (c, first, v[c])
        n_bad = int((m_fused["bad_rows"] != 0).sum())
        assert n_bad == {"clean": 0, "one_bad_stripe_per_chunk": r.n, "every_stripe_bad": r.n * r.pb}[case]
        if r.m >= 2 and fault:
            assert (m_fused["suspect_part"][m_fused["bad_rows"] != 0] == fault[0]).all()
        print(json.dumps({"what": "check_stripe_map_dev", "goal": text, "case": case, "route": route, "chunks": r.n,
                          "chunk_mib": NB * BLOCK >> 20, "bad_stripes": n_bad, "ms_per_call": round(t_map * 1e3, 3),
                          "check_stripes_ms_per_call": round(t_check * 1e3, 3), "map_over_check": round(t_map / t_check, 3),
                          "chunk_gib_s": round(r.n * NB * BLOCK / t_map / 2**30, 1), "routes_agree": True, **info}), flush=True)
        if fault:
            flip(eng, r, *fault)         # flipped back: the next case starts from a clean batch


def timed_each(call, restore, iters, warmup, stream):
    """mean time of one call, CUDA events around the call only; restore() runs on `stream` before each call, outside the events"""
    for _ in range(warmup):
        restore()
        call()
    torch.cuda.synchronize()
    evs = []
    for _ in range(iters):
        restore()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        call()
        e1.record(stream)
        evs.append((e0, e1))
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in evs) / 1e3 / iters


def window_repair(eng, r, out_m, stream):
    """the route before lzgpu_correct_stripes: the map, back on the host, then a one-stripe recover_chunks_dev window per bad stripe"""
    st = stream.cuda_stream
    eng.check_stripe_map_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_m.data_ptr(), stream=st)
    with torch.cuda.stream(stream):
        smap = out_m.cpu().numpy().view(L.Engine.STRIPE_STATE_DTYPE).reshape(r.n, r.pb)
    n = r.k + r.m
    for c, s in zip(*smap["bad_rows"].nonzero()):
        p = int(smap[c, s]["suspect_part"])
        if p < 0:
            continue
        off = int(c) * r.stride + int(s) * BLOCK
        window = [0 if i == p else r.ptrs[i] + off for i in range(n)]
        d_out = [r.ptrs[p] + off if i == p else 0 for i in range(n)]
        eng.recover_chunks_dev(r.goal, 1, min(r.k, NB - int(s) * r.k), window, r.stride, None, [int(i == p) for i in range(n)], d_out,
                               stream=st)


def correct_rows(eng, generic, r, text, args, stream, info):
    """time the correction against the map (and, with one bad stripe per chunk, against map + one-stripe windows); check both routes"""
    st = stream.cuda_stream
    out_m = torch.empty(8 * r.n * r.pb, dtype=torch.uint8, device="cuda")
    out_f = torch.empty(16 * r.n * r.pb, dtype=torch.uint8, device="cuda")
    cases = [("clean", None), ("one_bad_stripe_per_chunk", (3, [5], 777)), ("every_stripe_bad", (0, range(r.pb), 4242))]
    for case, fault in cases:
        idx = good = faulty = None
        if fault:
            part, stripes, offset = fault
            idx = torch.tensor([c * r.stride + part * r.part_bytes + s * BLOCK + offset for c in range(r.n) for s in stripes], device="cuda")
            good = r.buf[idx].clone()
            flip(eng, r, *fault)         # the stored CRCs now match the faulty blocks: only the stripe check sees them
            faulty = r.buf[idx].clone()

        def restore():
            if idx is not None:
                with torch.cuda.stream(stream):
                    r.buf[idx] = faulty

        def correct():
            eng.correct_stripes_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_f.data_ptr(), stream=st)

        def smap():
            eng.check_stripe_map_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_m.data_ptr(), stream=st)

        t_corr = t_map = t_win = 0.0
        for _ in range(2):               # alternate the calls, twice: other work shares the card
            t_corr += timed_each(correct, restore, args.iters, args.warmup, stream) / 2
            t_map += timed_each(smap, restore, args.iters, args.warmup, stream) / 2
            if case == "one_bad_stripe_per_chunk":
                t_win += timed_each(lambda: window_repair(eng, r, out_m, stream), restore, args.iters, args.warmup, stream) / 2
        eng.sync()
        fixes = []
        for e in (eng, generic):
            restore()
            torch.cuda.synchronize()
            e.correct_stripes_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_f.data_ptr())
            torch.cuda.synchronize()
            fixes.append(out_f.cpu().numpy().view(L.Engine.STRIPE_FIX_DTYPE).reshape(r.n, r.pb).copy())
            if idx is not None and r.m >= 2:
                assert (r.buf[idx] == good).all(), "a corrected block differs from the original"
        assert (fixes[0] == fixes[1]).all(), "fused and generic fix entries differ"
        n_fixed = int((fixes[0]["status"] == _lib.FIX_CORRECTED).sum())
        n_bad = int((fixes[0]["bad_rows"] != 0).sum())
        assert n_bad == {"clean": 0, "one_bad_stripe_per_chunk": r.n, "every_stripe_bad": r.n * r.pb}[case]
        assert n_fixed == (n_bad if r.m >= 2 else 0)
        row = {"what": "correct_stripes_dev", "goal": text, "case": case, "chunks": r.n, "chunk_mib": NB * BLOCK >> 20, "bad_stripes": n_bad,
               "corrected": n_fixed, "ms_per_call": round(t_corr * 1e3, 3), "check_stripe_map_ms_per_call": round(t_map * 1e3, 3),
               "correct_over_map": round(t_corr / t_map, 3)}
        if t_win:
            row.update({"map_and_windows_ms": round(t_win * 1e3, 3), "correct_over_map_and_windows": round(t_corr / t_win, 3)})
        print(json.dumps({**row, "routes_agree": True, **info}), flush=True)
        if fault:                        # the original bytes and their CRCs: the next case starts from a clean batch
            r.buf[idx] = good
            for c in range(r.n):
                eng.crc_blocks_dev(r.ptrs[fault[0]] + c * r.stride, r.pb, r.crc[fault[0], c].data_ptr())
            torch.cuda.synchronize()


def repair_rows(eng, generic, args, stream, info):
    """time the repair against the correction (clean), a whole-part recover (one rotten block in k stripes of part 3 per chunk) and
    alone (m rotten blocks in every stripe); check both routes and the rebuilt bytes"""
    st = stream.cuda_stream
    for text in ("ec(8,2)", "ec(8,4)", "xor3"):
        r = Resident(eng, text, args.chunks)
        n = r.k + r.m
        out_f = torch.empty(24 * r.n * r.pb, dtype=torch.uint8, device="cuda")
        rebuilt = torch.empty(r.n * r.stride, dtype=torch.uint8, device="cuda")
        cases = [("clean", []), ("one_rotten_block_in_k_stripes", [(3 % n, s) for s in range(r.k)]),
                 ("m_rotten_blocks_in_every_stripe", [(p, s) for s in range(r.pb) for p in range(r.m)])]
        for case, blocks in cases:
            idx = good = faulty = None
            if blocks:                   # the stored CRCs stay the original ones: every rotten block fails its own
                idx = torch.tensor([c * r.stride + p * r.part_bytes + s * BLOCK + 777 + 64 * p for c in range(r.n) for p, s in blocks],
                                   device="cuda")
                good = r.buf[idx].clone()
                faulty = good ^ 0x5A

            def restore():
                if idx is not None:
                    with torch.cuda.stream(stream):
                        r.buf[idx] = faulty

            def repair(e=eng):
                e.repair_stripes_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_f.data_ptr(), stream=st)

            def correct():
                eng.correct_stripes_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_f.data_ptr(), stream=st)

            def recover_part():          # today's alternative: drop part 3 and rebuild it whole from k others
                lost = 3 % n
                parts = [0 if i == lost else p for i, p in enumerate(r.ptrs)]
                crcs = [0 if i == lost else p for i, p in enumerate(r.crc_ptrs)]
                eng.recover_chunks_dev(r.goal, r.n, NB, parts, r.stride, crcs, [int(i == lost) for i in range(n)],
                                       [rebuilt.data_ptr() if i == lost else 0 for i in range(n)], stream=st)

            other = {"clean": ("correct_stripes_dev", correct), "one_rotten_block_in_k_stripes": ("recover_chunks_dev_whole_part", recover_part)}.get(case)
            t_rep = t_other = 0.0
            for _ in range(2):           # alternate the calls, twice: other work shares the card
                t_rep += timed_each(repair, restore, args.iters, args.warmup, stream) / 2
                if other:
                    t_other += timed_each(other[1], restore, args.iters, args.warmup, stream) / 2
            eng.sync()
            fixes = []
            for e in (eng, generic):
                restore()
                torch.cuda.synchronize()
                repair(e)
                torch.cuda.synchronize()
                fixes.append(out_f.cpu().numpy().view(L.Engine.STRIPE_REPAIR_DTYPE).reshape(r.n, r.pb).copy())
                if idx is not None:
                    assert (r.buf[idx] == good).all(), "a rebuilt block differs from the original"
            assert (fixes[0] == fixes[1]).all(), "fused and generic repair entries differ"
            n_rebuilt = int((fixes[0]["status"] == _lib.FIX_REBUILT).sum())
            assert n_rebuilt == r.n * len({s for _, s in blocks}), (case, n_rebuilt)
            assert int((fixes[0]["status"] == _lib.FIX_CLEAN).sum()) == r.n * r.pb - n_rebuilt
            row = {"what": "repair_stripes_dev", "goal": text, "case": case, "chunks": r.n, "chunk_mib": NB * BLOCK >> 20,
                   "rotten_blocks": len(blocks) * r.n, "rebuilt_stripes": n_rebuilt, "ms_per_call": round(t_rep * 1e3, 3)}
            if other:
                row.update({f"{other[0]}_ms_per_call": round(t_other * 1e3, 3), f"repair_over_{other[0]}": round(t_rep / t_other, 3)})
            print(json.dumps({**row, "routes_agree": True, **info}), flush=True)
        del r, out_f, rebuilt
        torch.cuda.empty_cache()


def decode_rows(eng, generic, args, stream, info):
    """time the decode against the repair on the same batch: clean, two stale parts in each of the first k stripes (ec(8,4)), one
    stale and one rotten block there (ec(8,3)), two stale parts in every stripe (ec(8,4)); next to it the map, clean and on the same
    batch, for the locate cost per bad stripe; check both routes and the rewritten bytes"""
    st = stream.cuda_stream
    cases = [("ec(8,3)", "clean", [], []), ("ec(8,4)", "clean", [], []), ("ec(10,5)", "clean", [], []),
             ("ec(8,4)", "two_stale_in_k_stripes", [(p, s) for s in range(8) for p in (1, 9)], []),
             ("ec(8,3)", "stale_and_rotten_in_k_stripes", [(5, s) for s in range(8)], [(3, s) for s in range(8)]),
             ("ec(8,4)", "two_stale_in_every_stripe", [(p, s) for s in range(128) for p in (1, 9)], [])]
    r, resident, clean_map = None, None, {}
    for text, case, stale, rotten in cases:
        if resident != text:
            del r
            torch.cuda.empty_cache()
            r, resident = Resident(eng, text, args.chunks), text
        out_f = torch.empty(40 * r.n * r.pb, dtype=torch.uint8, device="cuda")
        out_r = torch.empty(24 * r.n * r.pb, dtype=torch.uint8, device="cuda")
        out_m = torch.empty(8 * r.n * r.pb, dtype=torch.uint8, device="cuda")
        blocks = stale + rotten
        idx = good = faulty = None
        if blocks:                       # stale blocks get their CRCs recomputed, rotten ones keep the original
            idx = torch.tensor([c * r.stride + p * r.part_bytes + s * BLOCK + 777 + 64 * p for c in range(r.n) for p, s in blocks],
                               device="cuda")
            good = r.buf[idx].clone()
            faulty = good ^ 0x5A
            r.buf[idx] = faulty
            for p in {p for p, _ in stale}:
                for c in range(r.n):
                    eng.crc_blocks_dev(r.ptrs[p] + c * r.stride, r.pb, r.crc[p, c].data_ptr())
            torch.cuda.synchronize()

        def restore():
            if idx is not None:
                with torch.cuda.stream(stream):
                    r.buf[idx] = faulty

        def decode(e=eng):
            e.decode_stripes_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_f.data_ptr(), stream=st)

        def repair():
            eng.repair_stripes_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_r.data_ptr(), stream=st)

        def smap():
            eng.check_stripe_map_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out_m.data_ptr(), stream=st)

        t_dec = t_rep = t_map = 0.0
        for _ in range(2):               # alternate the calls, twice: other work shares the card
            t_dec += timed_each(decode, restore, args.iters, args.warmup, stream) / 2
            t_rep += timed_each(repair, restore, args.iters, args.warmup, stream) / 2
            t_map += timed_each(smap, restore, args.iters, args.warmup, stream) / 2
        try:
            eng.sync()
        except L.ChunkCrcError:          # the map's deferred verdict on the rotten blocks
            assert rotten
        fixes = []
        for e in (eng, generic):
            restore()
            torch.cuda.synchronize()
            decode(e)
            torch.cuda.synchronize()
            fixes.append(out_f.cpu().numpy().view(L.Engine.STRIPE_DECODE_DTYPE).reshape(r.n, r.pb).copy())
            if idx is not None:
                assert (r.buf[idx] == good).all(), "a decoded block differs from the original"
        assert fixes[0].tobytes() == fixes[1].tobytes(), "fused and generic decode entries differ"
        n_dec = int((fixes[0]["status"] == _lib.FIX_DECODED).sum())
        assert n_dec == r.n * len({s for _, s in blocks}), (case, n_dec)
        assert int((fixes[0]["status"] == _lib.FIX_CLEAN).sum()) == r.n * r.pb - n_dec
        row = {"what": "decode_stripes_dev", "goal": text, "case": case, "chunks": r.n, "chunk_mib": NB * BLOCK >> 20,
               "decoded_stripes": n_dec, "ms_per_call": round(t_dec * 1e3, 3), "repair_stripes_dev_ms_per_call": round(t_rep * 1e3, 3),
               "decode_over_repair": round(t_dec / t_rep, 3), "check_stripe_map_dev_ms_per_call": round(t_map * 1e3, 3)}
        if case == "clean":
            clean_map[text] = t_map
        else:
            row.update({"decode_us_per_decoded_stripe": round((t_dec - t_rep) / n_dec * 1e6, 2),
                        "map_locate_us_per_bad_stripe": round((t_map - clean_map[text]) / n_dec * 1e6, 2)})
        print(json.dumps({**row, "routes_agree": True, **info}), flush=True)
        if idx is not None:              # the original bytes and CRCs: the next case starts from a clean batch
            r.buf[idx] = good
            for p in {p for p, _ in stale}:
                for c in range(r.n):
                    eng.crc_blocks_dev(r.ptrs[p] + c * r.stride, r.pb, r.crc[p, c].data_ptr())
            torch.cuda.synchronize()
        del out_f, out_r, out_m
    del r
    torch.cuda.empty_cache()


DEGRADED = [("ec(8,2)", (1,)), ("ec(5,3)", (1,)), ("ec(8,3)", (1, 4)), ("ec(8,4)", (1,)), ("ec(8,4)", (1, 4))]


def degraded_rows(eng, generic, args, stream, info):
    """the degraded map on both routes and the full-parts map of the same goal, same resident batch"""
    st = stream.cuda_stream
    for text, lost in DEGRADED:
        r = Resident(eng, text, args.chunks)
        n = r.k + r.m
        out = torch.empty(8 * r.n * r.pb, dtype=torch.uint8, device="cuda")
        parts = [0 if i in lost else p for i, p in enumerate(r.ptrs)]
        crcs = [0 if i in lost else p for i, p in enumerate(r.crc_ptrs)]

        def degraded(e):
            e.check_stripe_map_degraded_dev(r.goal, r.n, NB, parts, r.stride, crcs, out.data_ptr(), stream=st)

        def full():
            eng.check_stripe_map_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out.data_ptr(), stream=st)

        t_fused = t_generic = t_full = 0.0
        for _ in range(2):               # alternate the calls, twice: other work shares the card
            t_fused += timed(lambda: degraded(eng), args.iters, args.warmup, stream) / 2
            eng.sync()
            geo = eng.last_geometry()
            t_generic += timed(lambda: degraded(generic), args.iters, args.warmup, stream) / 2
            generic.sync()
            t_full += timed(full, args.iters, args.warmup, stream) / 2
            eng.sync()
        assert geo["kernel"] == _lib.KERNEL_CHECK_DEGRADED, geo
        given = [i for i in range(n) if i not in lost]
        spares = given[r.k:]
        stale = 3                        # an input data part in every goal here
        maps = []
        for fault in (None, (stale, [5], 777)):
            if fault:
                flip(eng, r, *fault)
            got = []
            for e in (eng, generic):
                degraded(e)
                e.sync()
                got.append(out.cpu().numpy().view(L.Engine.STRIPE_STATE_DTYPE).reshape(r.n, r.pb).copy())
            assert (got[0] == got[1]).all(), "fused and generic degraded maps differ"
            maps.append(got[0])
            if fault:
                flip(eng, r, *fault)
        assert not maps[0]["bad_rows"].any()
        bad = maps[1]["bad_rows"] != 0
        assert bad.sum() == r.n and bad[:, 5].all()
        assert (maps[1]["suspect_part"][:, 5] == (stale if len(spares) >= 2 else -1)).all()
        deg_bytes = r.n * (len(given) * (r.part_bytes + 4 * r.pb) + 8 * r.pb)
        full_bytes = r.n * (n * (r.part_bytes + 4 * r.pb) + 8 * r.pb)
        rate = lambda b, t: round(b / t / 1e12, 3)
        print(json.dumps({"what": "check_stripe_map_degraded_dev", "goal": text, "lost": list(lost), "spares": len(spares),
                          "chunks": r.n, "chunk_mib": NB * BLOCK >> 20, "fused_ms": round(t_fused * 1e3, 3),
                          "generic_ms": round(t_generic * 1e3, 3), "full_parts_map_ms": round(t_full * 1e3, 3),
                          "fused_alg_tb_s": rate(deg_bytes, t_fused), "fused_of_hbm": round(deg_bytes / t_fused / 1e12 / HBM_TBPS, 3),
                          "generic_alg_tb_s": rate(deg_bytes, t_generic), "generic_of_hbm": round(deg_bytes / t_generic / 1e12 / HBM_TBPS, 3),
                          "full_parts_alg_tb_s": rate(full_bytes, t_full), "full_parts_of_hbm": round(full_bytes / t_full / 1e12 / HBM_TBPS, 3),
                          "fused_chunk_gib_s": round(r.n * NB * BLOCK / t_fused / 2**30, 1), "geometry": geo, "routes_agree": True,
                          **info}), flush=True)
        del r, out
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=16)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", choices=["degraded", "repair", "decode"], default=None,
                    help="run only the degraded-map rows, the repair rows or the decode rows")
    args = ap.parse_args()
    info = card()
    eng = L.Engine(0)
    os.environ["LZGPU_DISABLE_FUSED"] = "1"
    generic = L.Engine(0)
    del os.environ["LZGPU_DISABLE_FUSED"]
    stream = torch.cuda.Stream()        # the calls and the events share one stream
    st = stream.cuda_stream
    eng.set_deferred_verify(True)
    generic.set_deferred_verify(True)
    if args.only in (None, "degraded"):
        degraded_rows(eng, generic, args, stream, info)
    if args.only in (None, "repair"):
        repair_rows(eng, generic, args, stream, info)
    if args.only in (None, "decode"):
        decode_rows(eng, generic, args, stream, info)
    generic.set_deferred_verify(False)
    for text in (GOALS if args.only is None else []):
        r = Resident(eng, text, args.chunks)
        out = torch.empty(12 * r.n, dtype=torch.uint8, device="cuda")
        t = timed(lambda: eng.check_stripes_dev(r.goal, r.n, NB, r.ptrs, r.stride, r.crc_ptrs, out.data_ptr(), stream=st),
                  args.iters, args.warmup, stream)
        eng.sync()
        geo = eng.last_geometry()
        route = "fused" if geo["kernel"] == _lib.KERNEL_CHECK else "generic"
        clean = verdicts(eng, r, out)
        assert (clean["first_bad_stripe"] == -1).all(), "a clean batch reported a bad stripe"
        # one injected fault: chunk n/2, data part 3, stripe 5; its block CRC restored so only the check sees it
        c, part, s = r.n // 2, 3, 5
        off = c * r.stride + part * r.part_bytes + s * BLOCK + 1234
        r.buf[off] ^= 0x5A
        eng.crc_blocks_dev(r.ptrs[part] + c * r.stride + s * BLOCK, 1, r.crc[part, c, s:].data_ptr())
        eng.sync()
        v_fused, v_generic = verdicts(eng, r, out), verdicts(generic, r, out)
        assert (v_fused == v_generic).all(), "fused and generic verdicts differ"
        bad = [(i, tuple(int(x) for x in v_fused[i])) for i in range(r.n) if v_fused[i]["first_bad_stripe"] >= 0]
        want_rows = (1 << r.m) - 1
        assert bad == [(c, (s, want_rows, part if r.m >= 2 else -1))], bad
        print(json.dumps({"what": "check_stripes_dev", "goal": text, "route": route, "chunks": r.n, "chunk_mib": NB * BLOCK >> 20,
                          "ms_per_call": round(t * 1e3, 3), "chunk_gib_s": round(r.n * NB * BLOCK / t / 2**30, 1),
                          "alg_tb_s": round(r.alg_bytes() / t / 1e12, 3), "of_hbm": round(r.alg_bytes() / t / 1e12 / HBM_TBPS, 3),
                          "geometry": geo, "fault_verdict": bad[0][1], "routes_agree": True, **info}), flush=True)
        if text == "ec(8,2)":
            r.buf[off] ^= 0x5A   # restore the byte: the degraded read runs on valid parts
            eng.crc_blocks_dev(r.ptrs[part] + c * r.stride + s * BLOCK, 1, r.crc[part, c, s:].data_ptr())
            lost = (1, 4)
            outs = {j: torch.empty(r.n * r.stride, dtype=torch.uint8, device="cuda") for j in lost}
            parts = [0 if i in lost else p for i, p in enumerate(r.ptrs)]
            crcs = [0 if i in lost else p for i, p in enumerate(r.crc_ptrs)]
            want = [1 if i in lost else 0 for i in range(r.k + r.m)]
            d_out = [outs[i].data_ptr() if i in lost else 0 for i in range(r.k + r.m)]
            t_rec = timed(lambda: eng.recover_chunks_dev(r.goal, r.n, NB, parts, r.stride, crcs, want, d_out, stream=st), args.iters, args.warmup, stream)
            eng.sync()
            rec_bytes = r.n * (r.k * (r.part_bytes + 4 * r.pb) + 2 * r.part_bytes)
            print(json.dumps({"what": "recover_chunks_dev (reference point)", "goal": text, "lost": list(lost), "chunks": r.n,
                              "ms_per_call": round(t_rec * 1e3, 3), "chunk_gib_s": round(r.n * NB * BLOCK / t_rec / 2**30, 1),
                              "alg_tb_s": round(rec_bytes / t_rec / 1e12, 3), "of_hbm": round(rec_bytes / t_rec / 1e12 / HBM_TBPS, 3),
                              "geometry": eng.last_geometry(), **info}), flush=True)
            del outs
        if text != "ec(8,2)":   # the map cases start from a clean batch (the ec(8,2) branch restored the byte already)
            r.buf[off] ^= 0x5A
            eng.crc_blocks_dev(r.ptrs[part] + c * r.stride + s * BLOCK, 1, r.crc[part, c, s:].data_ptr())
            torch.cuda.synchronize()
        map_rows(eng, generic, r, text, args, stream, info)
        correct_rows(eng, generic, r, text, args, stream, info)
        del r, out
        torch.cuda.empty_cache()
    eng.set_deferred_verify(False)
    generic.close()
    eng.close()


if __name__ == "__main__":
    main()
