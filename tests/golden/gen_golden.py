"""Generate tests/golden/vectors.json from the UNMODIFIED reference (oracle/_ref/liblzref.so,
built by oracle/Makefile from the reference sources), and tests/golden/reference_digests.json: the
digests of the reference's answers to the calls the tests make (tests/_oracle.py ref_digest).  Run
where oracle/_ref is built:

    python tests/golden/gen_golden.py

Inputs are the deterministic splitmix64 stream (oracle lzo_fill_chunk; DESIGN.md §6), so the
fixture only stores outputs: per-block CRCs, a SHA-256 of every parity part and its first bytes.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import _oracle as O  # noqa: E402

BLOCK = 65536
CASES = [  # (goal text, kind, k, m, chunk_len bytes, seed)
    ("xor2", 0, 2, 1, 5 * BLOCK, 11),
    ("xor3", 0, 3, 1, 7 * BLOCK + 12345, 12),
    ("xor9", 0, 9, 1, 19 * BLOCK, 13),
    ("ec(3,2)", 1, 3, 2, 10 * BLOCK, 14),
    ("ec(5,3)", 1, 5, 3, 11 * BLOCK + 1, 15),
    ("ec(8,2)", 1, 8, 2, 17 * BLOCK, 16),
    ("ec(8,4)", 1, 8, 4, 16 * BLOCK, 17),
    ("ec(2,1)", 1, 2, 1, 3 * BLOCK, 18),
    ("ec(4,5)", 1, 4, 5, 9 * BLOCK, 19),     # Cauchy generator (m >= 5)
    ("ec(21,4)", 1, 21, 4, 43 * BLOCK, 20),  # Cauchy generator (m == 4, k > 20)
    ("ec(32,32)", 1, 32, 32, 33 * BLOCK, 21),
]


def main():
    oracle = O.load_oracle()
    ref = O.load_ref()
    assert ref is not None, "oracle/_ref/liblzref.so missing (needs /root/reference)"
    out = {"generator": "tests/golden/gen_golden.py", "source": "oracle/_ref/liblzref.so (unmodified reference)", "cases": []}
    for text, kind, k, m, clen, seed in CASES:
        chunk = O.fill_chunk(oracle, clen, seed, 0)
        parity, crc = ref.encode_chunk(kind, k, m, chunk)
        nb = (clen + BLOCK - 1) // BLOCK
        out["cases"].append({
            "goal": text, "kind": kind, "k": k, "m": m, "chunk_len": clen, "seed": seed, "nb": nb,
            "crc": [int(x) for x in crc],
            "parity_sha256": [hashlib.sha256(p.tobytes()).hexdigest() for p in parity],
            "parity_head": [p[:16].tobytes().hex() for p in parity],
        })
    # matrices and scalar known answers straight from the reference
    mats = {}
    for k, m in [(8, 2), (5, 3), (8, 4), (4, 5), (21, 4), (32, 32)]:
        cauchy = m >= 5 or (m == 4 and k > 20)
        g = ref.gen_cauchy1_matrix(k + m, k) if cauchy else ref.gen_rs_matrix(k + m, k)
        mats[f"{k},{m}"] = g[k:].tolist()
    out["generator_parity_rows"] = mats
    out["crc_kat"] = {str(n): int(ref.crc32(0, np.full(n, ord("a"), dtype=np.uint8))) for n in [1, 2, 4, 8, 16, 32, 64, 65536]}
    out["crc_zero_block"] = int(ref.crc32_zeroblock(0, BLOCK))
    out["crc_combine"] = [[a, b, n, int(ref.crc32_combine(a, b, n))] for a, b, n in
                          [(0x12345678, 0x9ABCDEF0, 1), (0xDEADBEEF, 0x01020304, 65535), (0xFFFFFFFF, 0, 65536), (1, 2, 65537), (0xCAFEBABE, 0x0BADF00D, 1 << 26)]]
    out["write_data_prefix"] = [[list(a), O.write_data_prefix(ref, *a).tobytes().hex()] for a in
                                [(0x1122334455667788, 7, 3, 0, 65536, 0xAABBCCDD), (1, 0xFFFFFFFF, 1023, 4096, 61440, 0), (2**63 + 5, 12, 0, 0, 1, 0xD7978EEB)]]
    # planner-level rows: the reference's own ChunkReadPlanner / SliceRecoveryPlanner executed in memory (oracle/ref_plans.cc)
    from tests.test_oracle_plans import GOALS, make_slice, ref_sources, true_blocks
    plans = []
    for src_name, lost, nb, dst_name, seed in [("ec(3,2)", (0, 2), 10, "ec(8,2)", 31), ("ec(8,2)", (1, 4), 19, "ec(3,2)", 32), ("xor3", (1,), 10, "ec(5,3)", 33),
                                               ("std", (), 9, "xor2", 34), ("ec(5,3)", (0, 1, 4), 11, "std", 35), ("ec(8,2)", (8,), 16, "ec(8,2)", 36)]:
        src, dst = GOALS[src_name], GOALS[dst_name]
        chunk = O.fill_chunk(oracle, nb * BLOCK, seed, 0)
        parts, _ = make_slice(oracle, src, chunk)
        sources = ref_sources(src, parts, nb, lost)
        case = {"src": src_name, "lost": list(lost), "nb": nb, "dst": dst_name, "seed": seed, "parts": []}
        if src[0] != 2:
            image = O.plan_read_chunk(ref, sources, 0, nb)
            case["image_sha256"] = hashlib.sha256(image.tobytes()).hexdigest()
        for part in range(dst[1] + dst[2]):
            nblk = true_blocks(dst, part, nb)
            if nblk == 0:
                case["parts"].append(None)
                continue
            data, crc = O.plan_recover_part(ref, sources, O.slice_type(*dst), O.ref_part_number(dst[0], dst[1], part), 0, nblk)
            case["parts"].append({"blocks": nblk, "sha256": hashlib.sha256(data.tobytes()).hexdigest(), "crc": [int(x) for x in crc]})
        plans.append(case)
    out["planner_cases"] = plans
    with open(os.path.join(os.path.dirname(__file__), "vectors.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote vectors.json with", len(out["cases"]), "cases")
    record_reference_digests()


def record_reference_digests():
    """run the tests that compare with the reference with LZ_RECORD_REF_DIGESTS=1; the GPU one through a stand-in engine (the
    oracle's conversion), since only the reference's side of it is recorded"""
    import subprocess
    if os.path.exists(O.REF_DIGESTS):
        os.remove(O.REF_DIGESTS)
    env = dict(os.environ, LZ_RECORD_REF_DIGESTS="1")
    subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "tests/test_oracle.py", "tests/test_oracle_plans.py"],
                   cwd=ROOT, env=env, check=True)
    os.environ["LZ_RECORD_REF_DIGESTS"] = "1"
    from tests import test_gpu_convert_geometry as CG
    from tests import test_gpu_replication as R
    oracle = O.load_oracle()

    class OracleEngine:
        def convert_chunks(self, src, dst, nb, parts, want):
            sk = (src.kind, src.k, src.m)
            avail = [None if p is None else p[0] for p in parts]
            rc, out, ocrc, _ = O.convert_chunk(oracle, sk, avail, None, (dst.kind, dst.k, dst.m), want, nb)
            assert rc == 0
            return [o[None, :] for o in out], [c[None, :] for c in ocrc]
    R.test_convert_chunks_vs_reference_planner(OracleEngine(), oracle)
    CG.test_convert_geometry_vs_reference_planner(OracleEngine(), oracle)
    print("recorded", len(O._recorded), "answers of the reference (plus those of the pytest run) in", O.REF_DIGESTS)


if __name__ == "__main__":
    main()
