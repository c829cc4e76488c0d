# compute-sanitizer passes over a small encode + recover + scrub through the C ABI (run on a GPU machine).
# Full reports land in gpurun_out/sanitize_<tool>.log.
mkdir -p gpurun_out
cat > /tmp/san_case.py <<'PY'
import numpy as np, sys
sys.path.insert(0, '.')
import lizardfs_b200 as L
from tests import _oracle as O
o = O.load_oracle()
eng = L.Engine(0)
for text, nblk in [("ec(8,2)", 24), ("ec(3,2)", 7), ("xor3", 9)]:
    g = L.SliceType(text)
    data = np.stack([O.fill_chunk(o, nblk * 65536, 3, c) for c in range(2)])
    par, crc = eng.encode_chunks(g, data)
    for c in range(2):
        p_ref, c_ref = o.encode_chunk(g.kind, g.k, g.m, data[c])
        assert (par[c] == p_ref).all() and (crc[c] == c_ref).all()
    parts = [np.stack([O.split_parts(data[c], g.k)[0][j] for c in range(2)]) for j in range(g.k)] + [np.ascontiguousarray(par[:, r]) for r in range(g.m)]
    avail = [None if i == 1 else parts[i] for i in range(g.k + g.m)]
    out, img = eng.recover_chunks(g, nblk, avail, chunk_image=True)
    assert (out[1] == parts[1]).all() and (img == data).all()
eng.verify_blocks(data.reshape(-1), eng.crc_blocks(data.reshape(-1)))
# round-1 additions: striped units (ragged small chunks), the two-CTA recover geometry, slice conversion, both scrub formats
# with the exact sparse rule, batched block writes
import os, zlib
for mode in ("1", "0"):
    os.environ["LZGPU_STRIPED"] = mode; os.environ["LZGPU_RECOVER_TWO"] = mode
    e2 = L.Engine(0)
    for text, nblk, n in [("ec(5,3)", 11, 7), ("xor3", 7, 9), ("ec(8,2)", 13, 5)]:
        g = L.SliceType(text)
        data = np.stack([O.fill_chunk(o, nblk * 65536, 5, c) for c in range(n)])
        par, crc = e2.encode_chunks(g, data)
        for c in range(n):
            p_ref, c_ref = o.encode_chunk(g.kind, g.k, g.m, data[c])
            assert (par[c] == p_ref).all() and (crc[c] == c_ref).all()
        parts = [np.stack([O.split_parts(data[c], g.k)[0][j] for c in range(n)]) for j in range(g.k)] + [np.ascontiguousarray(par[:, r]) for r in range(g.m)]
        avail = [None if i == 0 else parts[i] for i in range(g.k + g.m)]
        out, img = e2.recover_chunks(g, nblk, avail, chunk_image=True)
        assert (out[0] == parts[0]).all() and (img == data).all()
        out2, ocrc = e2.convert_chunks(g, L.SliceType("ec(3,2)"), nblk, avail, [1] * 5)
        p32, c32 = e2.encode_chunks(L.SliceType("ec(3,2)"), data)
        assert (out2[3] == p32[:, 0]).all() and (out2[4] == p32[:, 1]).all()
rec = np.zeros((5, 4 + 65536), dtype=np.uint8)
for i in range(5):
    rec[i, 4:] = O.fill_chunk(o, 65536, 9, i)
    rec[i, :4] = np.frombuffer(zlib.crc32(rec[i, 4:].tobytes()).to_bytes(4, "big"), dtype=np.uint8)
rec[2] = 0
eng.verify_interleaved(rec)
hdr = eng.moosefs_header_size(3)
img = np.zeros(hdr + 3 * 65536, dtype=np.uint8)
for b in range(3):
    img[hdr + b * 65536: hdr + (b + 1) * 65536] = rec[b, 4:]
    img[1024 + 4 * b: 1028 + 4 * b] = rec[b, :4]
img[1024 + 8: 1024 + 12] = np.frombuffer((0xD7978EEB).to_bytes(4, "big"), dtype=np.uint8)
eng.verify_moosefs(img, 3, 3)
blocks = np.stack([O.fill_chunk(o, 65536, 11, i) for i in range(6)])
stored = np.array([zlib.crc32(b.tobytes()) for b in blocks], dtype=np.uint32)
ws = []
for i, (off, size) in enumerate([(0, 65536), (1, 1), (100, 4097), (65535, 1), (0, 3), (32768, 32768)]):
    d = O.fill_chunk(o, max(size, 8), 13, i)[:size]
    ws.append(dict(block=i, offset=off, data=d, crc=zlib.crc32(d.tobytes()), exists=i != 4))
st = eng.write_blocks(blocks, stored, ws)
assert st == [0] * 6 and all(stored[i] == zlib.crc32(blocks[i].tobytes()) for i in range(6))
# round-2 additions: the 16-warp CTA with 8-byte items (four parity rows), Cauchy rows in passes and with narrow items, the
# nine-warp generic CTA (ec(31,3)), the 16-warp recover geometry incl. the three-unknown elimination, the SPLIT encode of the
# slice conversion, a pool of two contexts
os.environ.pop("LZGPU_STRIPED", None); os.environ.pop("LZGPU_RECOVER_TWO", None)
for geo in ("2", "0"):
    os.environ["LZGPU_RECOVER_GEO"] = geo
    e3 = L.Engine(0)
    for text, nblk, n, lost in [("ec(8,4)", 21, 3, (0, 5)), ("ec(8,6)", 19, 2, (1,)), ("ec(21,4)", 45, 2, (3,)), ("ec(31,3)", 62, 2, (0, 7, 30)),
                                ("ec(5,3)", 23, 4, (0, 1, 4)), ("ec(3,2)", 11, 5, (0, 2))]:
        g = L.SliceType(text)
        data = np.stack([O.fill_chunk(o, nblk * 65536, 17, c) for c in range(n)])
        par, crc = e3.encode_chunks(g, data)
        for c in range(n):
            p_ref, c_ref = o.encode_chunk(g.kind, g.k, g.m, data[c])
            assert (par[c] == p_ref).all() and (crc[c] == c_ref).all(), text
        if geo == "0" and g.m > 4:
            continue
        parts = [np.stack([O.split_parts(data[c], g.k)[0][j] for c in range(n)]) for j in range(g.k)] + [np.ascontiguousarray(par[:, r]) for r in range(g.m)]
        avail = [None if i in lost else parts[i] for i in range(g.k + g.m)]
        out, img = e3.recover_chunks(g, nblk, avail, chunk_image=True)
        assert all((out[i] == parts[i]).all() for i in lost) and (img == data).all(), text
    e3.close()
os.environ.pop("LZGPU_RECOVER_GEO", None)
# round 2, later: the one-pass slice conversion (convert_kernel.cuh: dedicated rebuild warps, table-driven block addressing) and the
# DIRECT form of the degraded read for Cauchy goals, both with CRC verification
def slice_parts(eng_, g, data, nblk):
    par, crc = eng_.encode_chunks(g, data)
    n = data.shape[0]
    parts = [np.stack([O.split_parts(data[c], g.k)[0][j] for c in range(n)]) for j in range(g.k)] + [np.ascontiguousarray(par[:, r]) for r in range(g.m)]
    pb = parts[0].shape[1] // 65536
    crcs = []
    for j in range(g.k):
        cj = np.full((n, pb), 0xD7978EEB, dtype=np.uint32)
        mine = crc[:, j:nblk:g.k]
        cj[:, : mine.shape[1]] = mine
        crcs.append(cj)
    crcs += [np.ascontiguousarray(crc[:, nblk + r * pb: nblk + (r + 1) * pb]) for r in range(g.m)]
    return parts, crcs, par, crc
e4 = L.Engine(0)
for src, lost, nblk, dst in [("ec(8,2)", (1, 4), 29, "ec(3,2)"), ("ec(3,2)", (0,), 10, "ec(5,3)"), ("xor3", (), 13, "xor2"), ("ec(5,3)", (0, 3), 23, "ec(8,2)")]:
    gs, gd = L.SliceType(src), L.SliceType(dst)
    data = np.stack([O.fill_chunk(o, nblk * 65536, 23, c) for c in range(3)])
    parts, crcs, _, _ = slice_parts(e4, gs, data, nblk)
    avail = [None if i in lost else parts[i] for i in range(gs.k + gs.m)]
    acrc = [None if i in lost else crcs[i] for i in range(gs.k + gs.m)]
    out, ocrc = e4.convert_chunks(gs, gd, nblk, avail, [1] * (gd.k + gd.m), part_crc=acrc)
    dparts, dcrcs, _, _ = slice_parts(e4, gd, data, nblk)
    for i in range(gd.k + gd.m):
        assert (out[i] == dparts[i]).all(), (src, dst, i)
        nreal = gd.part_blocks(i, nblk)
        assert (ocrc[i][:, :nreal] == dcrcs[i][:, :nreal]).all(), (src, dst, i)
for text, nblk, lost in [("ec(8,6)", 19, (2,)), ("ec(4,5)", 9, (0, 3)), ("ec(21,4)", 43, (5,))]:
    g = L.SliceType(text)
    data = np.stack([O.fill_chunk(o, nblk * 65536, 29, c) for c in range(2)])
    parts, crcs, _, _ = slice_parts(e4, g, data, nblk)
    avail = [None if i in lost else parts[i] for i in range(g.k + g.m)]
    acrc = [None if i in lost else crcs[i] for i in range(g.k + g.m)]
    out, img = e4.recover_chunks(g, nblk, avail, part_crc=acrc, want=[1 if i in lost else 0 for i in range(g.k + g.m)], chunk_image=True)
    assert all((out[i] == parts[i]).all() for i in lost) and (img == data).all(), text
e4.close()
pool = L.Pool([0, 0])
g = L.SliceType("ec(8,2)")
data = np.stack([O.fill_chunk(o, 16 * 65536, 19, c) for c in range(5)])
par, crc = pool.encode_chunks(g, data)
for c in range(5):
    p_ref, c_ref = o.encode_chunk(g.kind, g.k, g.m, data[c])
    assert (par[c] == p_ref).all() and (crc[c] == c_ref).all()
pool.close()
# the salvage of a multi-slice chunk (recover_slices_kernel, SALVAGE form): xor2 + xor3 with xor2's parity and xor3's data part 0
# given (positions 1, 2 solved, 4, 5 holes), a tail stripe, and one corrupt byte in xor3 part 0 so that its dependents are withheld
goals = [L.SliceType("xor2"), L.SliceType("xor3")]
nblk = 14
data = np.stack([O.fill_chunk(o, nblk * 65536, 31, c) for c in range(2)])
enc = eng.encode_slices(goals, data)
sparts = []
for g, (par, crc) in zip(goals, enc):
    pb = -(-nblk // g.k)
    padded = np.zeros((2, pb * g.k * 65536), dtype=np.uint8)
    padded[:, :nblk * 65536] = data
    sparts += [np.ascontiguousarray(padded.reshape(2, pb, g.k, 65536)[:, :, j]).reshape(2, -1) for j in range(g.k)] + [par[:, 0]]
given = [0, 0, 1, 1, 0, 0, 0]
img, icrc, smap = eng.salvage_slices(goals, nblk, [p if x else None for p, x in zip(sparts, given)])
assert (smap == 2).any() and (smap == 0).any()
rot = sparts[3].copy()
rot[1, 70000] ^= 1
scrc = [eng.crc_blocks(p.reshape(-1)).reshape(2, -1) if x else None for p, x in zip(sparts, given)]
try:
    eng.salvage_slices(goals, nblk, [rot if g == 3 else (p if x else None) for g, (p, x) in enumerate(zip(sparts, given))], scrc)
    raise AssertionError("the corrupt block passed")
except L.ChunkCrcError as e:
    assert (e.map == 3).any()
# the correction of several slices (recover_slices_kernel CORRECT form, locate, correct_slices_kernel): xor2 + xor3 with every part
# given, a stale byte in xor3's parity in the tail combined stripe, corrected back with its new CRC
full = [p.copy() for p in sparts]
full[6][0, 4 * 65536 + 9] ^= 0x41
fcrc = [eng.crc_blocks(p.reshape(-1)).reshape(2, -1) for p in full]
fix, ncrc = eng.correct_slices(goals, nblk, full, fcrc)
assert (fix["status"] == 1).sum() == 1 and all((a == b).all() for a, b in zip(full, sparts))
assert ncrc[6][0, 4] == eng.crc_blocks(sparts[6][0, 4 * 65536:5 * 65536])[0]
# the same at the limits of the tables (tests/test_slices_check_edges.py): A, ec(8,8) + ec(16,32) with all 64 parts, 64 checks, a
# stale flat part 63 in combined stripe 1; C, std + ec(31,1) + ec(2,1) with ec(2,1) lost, L = 62, the whole std copy of stripe 1
# stale: a 62-block correction in correct_slices_kernel's largest shared memory
for names, given, nblk, stale in [(("ec(8,8)", "ec(16,32)"), [1] * 64, 32, (63, [1])),
                                  (("std", "ec(31,1)", "ec(2,1)"), [1] * 33 + [0] * 3, 124, (0, list(range(62, 124))))]:
    goals = [L.SliceType(2, 1, 0) if x == "std" else L.SliceType(x) for x in names]
    data = np.stack([O.fill_chunk(o, nblk * 65536, 37, 0)])
    enc = eng.encode_slices(goals, data)
    eparts = []
    for g, (par, crc) in zip(goals, enc):
        if g.is_std:
            eparts.append(data.copy())
            continue
        pb = -(-nblk // g.k)
        padded = np.zeros((1, pb * g.k * 65536), dtype=np.uint8)
        padded[:, :nblk * 65536] = data
        eparts += [np.ascontiguousarray(padded.reshape(1, pb, g.k, 65536)[:, :, j]).reshape(1, -1) for j in range(g.k)]
        eparts += [np.ascontiguousarray(par[:, r]) for r in range(g.m)]
    part, blks = stale
    bad = [p.copy() for p in eparts]
    for b in blks:
        bad[part][0, b * 65536 + 77] ^= 0x3C
    inp = [p if x else None for p, x in zip(bad, given)]
    bcrc = [eng.crc_blocks(p.reshape(-1)).reshape(1, -1) if x else None for p, x in zip(bad, given)]
    m = eng.check_slices(goals, nblk, inp, bcrc)
    assert m[0, 1]["suspect_part"] == part and m[0, 1]["bad_checks"] != 0
    fix, _ = eng.correct_slices(goals, nblk, inp, bcrc)
    assert fix[0, 1]["status"] == 1 and bin(int(fix[0, 1]["changed"])).count("1") == len(blks)
    assert all(a is None or (a == b).all() for a, b in zip(inp, eparts))
# the one-pass encode of several slices at the limits of its tables (tests/test_encode_slices_edges.py): A, xor2 x 3 + ec(2,3) with
# 128 stripes per unit, 16 GF items per thread and 512 CRC streams; F, ec(2,4) + ec(21,3) with the shared memory 392 bytes under the
# cap; two chunks each, the last unit partial and the last block short
for names, nblk in [(("xor2", "xor2", "xor2", "ec(2,3)"), 67), (("ec(2,4)", "ec(21,3)"), 43)]:
    goals = [L.SliceType(x) for x in names]
    data = np.stack([O.fill_chunk(o, nblk * 65536 - 999, 41, c) for c in range(2)])
    enc = eng.encode_slices(goals, data)
    for g, (par, crc) in zip(goals, enc):
        for c in range(2):
            p_ref, c_ref = o.encode_chunk(g.kind, g.k, g.m, data[c])
            assert (par[c] == p_ref).all() and (crc[c] == c_ref).all(), names
print("sanitizer case OK")
PY
for tool in ${TOOLS:-memcheck racecheck synccheck}; do
  echo "== $tool"; timeout 900 compute-sanitizer --tool $tool --print-limit 8 python /tmp/san_case.py > gpurun_out/sanitize_$tool.log 2>&1
  grep -E "SUMMARY|sanitizer case OK|Error|error" gpurun_out/sanitize_$tool.log | head -5
done
