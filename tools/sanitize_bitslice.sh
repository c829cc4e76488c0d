# compute-sanitizer memcheck over the bit-sliced three- / four-parity-row encoders only (on a GPU machine; the long case list is tools/sanitize.sh).
mkdir -p gpurun_out
cat > /tmp/san_bs.py <<'PY'
import os, sys
import numpy as np
sys.path.insert(0, '.')
import lizardfs_b200 as L
from tests import _oracle as O
o = O.load_oracle()
# dedicated GF warps (csrc/bitslice.cuh): per-chunk units with a tail stripe, flat units, striped units; then the packed-byte route
for bs, striped in (("7", "0"), ("7", "1"), ("0", "0")):
    os.environ["LZGPU_BITSLICE"] = bs; os.environ["LZGPU_STRIPED"] = striped
    e = L.Engine(0)
    for text, nblk, n in [("ec(8,4)", 19, 3), ("ec(8,4)", 16, 5), ("ec(5,4)", 11, 4), ("ec(12,4)", 25, 2), ("ec(5,3)", 11, 4), ("ec(8,3)", 16, 3), ("ec(31,3)", 63, 2)]:
        g = L.SliceType(text)
        data = np.stack([O.fill_chunk(o, nblk * 65536, 17, c) for c in range(n)])
        par, crc = e.encode_chunks(g, data)
        for c in range(n):
            p_ref, c_ref = o.encode_chunk(g.kind, g.k, g.m, data[c])
            assert (par[c] == p_ref).all() and (crc[c] == c_ref).all(), (text, bs, striped)
    e.close()
    print("three / four parity rows, bitslice", bs, "striped", striped, "OK")
# degraded read with three lost data parts on bit planes (bs_recover_kernel.cuh): verification + image, first unknown at 0 and at 4
os.environ.pop("LZGPU_BITSLICE", None); os.environ.pop("LZGPU_STRIPED", None)
e = L.Engine(0)
for text, nblk, lost in [("ec(5,3)", 11, (0, 1, 4)), ("ec(8,3)", 19, (4, 5, 7)), ("ec(12,3)", 25, (0, 5, 11))]:
    g = L.SliceType(text)
    n = 2
    data = np.stack([O.fill_chunk(o, nblk * 65536, 21, c) for c in range(n)])
    par, crc = e.encode_chunks(g, data)
    parts = [np.stack([O.split_parts(data[c], g.k)[0][j] for c in range(n)]) for j in range(g.k)] + [np.ascontiguousarray(par[:, r]) for r in range(g.m)]
    pb = parts[0].shape[1] // 65536
    crcs = []
    for j in range(g.k):
        cj = np.full((n, pb), 0xD7978EEB, dtype=np.uint32)
        mine = crc[:, j:nblk:g.k]
        cj[:, : mine.shape[1]] = mine
        crcs.append(cj)
    crcs += [np.ascontiguousarray(crc[:, nblk + r * pb: nblk + (r + 1) * pb]) for r in range(g.m)]
    avail = [None if i in lost else parts[i] for i in range(g.k + g.m)]
    acrc = [None if i in lost else crcs[i] for i in range(g.k + g.m)]
    out, img = e.recover_chunks(g, nblk, avail, part_crc=acrc, want=[1 if i in lost else 0 for i in range(g.k + g.m)], chunk_image=True)
    assert all((out[i] == parts[i]).all() for i in lost) and (img == data).all(), text
    print("three lost on bit planes", text, lost, "OK")
e.close()
print("sanitizer case OK")
PY
for tool in ${TOOLS:-memcheck}; do
  echo "== $tool"; timeout ${SAN_TIMEOUT:-300} compute-sanitizer --tool $tool --print-limit 8 python /tmp/san_bs.py > gpurun_out/sanitize_bs_$tool.log 2>&1
  grep -E "SUMMARY|sanitizer case OK|Error|error" gpurun_out/sanitize_bs_$tool.log | head -5
done
