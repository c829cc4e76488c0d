"""The tile pipeline of the host-pointer calls over batches of at least four tiles: lzgpu_recover_chunks and lzgpu_convert_chunks
(erasure-coded and standard sources), on the fused and on the generic route.  Results against the original data, the oracle and an
independent encode; a stored-CRC mismatch reported at its (chunk, part, block) in the whole batch, whichever tile holds it and
whatever is still in flight; the next call on the context correct; every verification result slot back in the pool afterwards
(lzgpu_debug_status_slots), after a deferred-mode mismatch too."""
import os

import numpy as np
import pytest

import lizardfs_b200 as L
from tests import _oracle as O

pytestmark = pytest.mark.gpu
BLOCK = 65536
TILE_BYTES = 2 * (128 << 20)       # staged per tile by the recover and convert calls: input parts + output parts

K, M, NB = 8, 2, 24                # ec(8,2), 1.5 MiB chunks: three blocks per part
PB = NB // K
LOST = (1, 4)
USED = [i for i in range(K + M) if i not in LOST]                  # the k parts read
T_REC = TILE_BYTES // (K * PB * BLOCK)                             # 170 chunks per recover tile
N_REC = 3 * T_REC + 4                                              # four tiles, the last one short
KD, PBD = 3, NB // 3                                               # conversion to ec(3,2)
T_CONV = TILE_BYTES // (K * PB * BLOCK + (KD + 2) * PBD * BLOCK)   # 64 chunks per tile, from an ec(8,2) or a standard source
N_CONV = 3 * T_CONV + 4


@pytest.fixture(scope="module", params=["fused", "generic"])
def eng(request):
    if request.param == "generic":
        os.environ["LZGPU_DISABLE_FUSED"] = "1"
    try:
        e = L.Engine(0)
    finally:
        os.environ.pop("LZGPU_DISABLE_FUSED", None)
    yield e
    e.close()


class Batch:
    pass


@pytest.fixture(scope="module")
def batch():
    """N_REC random chunks, their ec(8,2) parts and per-part CRCs, and the ec(3,2) encode of the first N_CONV chunks"""
    e = L.Engine(0)
    b = Batch()
    b.chunks = np.random.default_rng(2024).integers(0, 256, (N_REC, NB * BLOCK), dtype=np.uint8)
    parity, crc = e.encode_chunks(L.SliceType("ec(8,2)"), b.chunks)
    blocks = b.chunks.reshape(N_REC, PB, K, BLOCK)
    b.parts = [np.ascontiguousarray(blocks[:, :, j]).reshape(N_REC, -1) for j in range(K)] + [np.ascontiguousarray(parity[:, r]) for r in range(M)]
    b.parity, b.crc = parity, crc
    b.pcrc = [np.ascontiguousarray(crc[:, :NB].reshape(N_REC, PB, K)[:, :, j]) for j in range(K)]
    b.pcrc += [np.ascontiguousarray(crc[:, NB + r * PB: NB + (r + 1) * PB]) for r in range(M)]
    b.p32, b.c32 = e.encode_chunks(L.SliceType("ec(3,2)"), b.chunks[:N_CONV])
    e.close()
    return b


def boundary_chunks(tile, n):
    return sorted({0, tile - 1, tile, 2 * tile - 1, 2 * tile, 3 * tile - 1, 3 * tile, n - 1})


def check_slots_returned(eng, allocated):
    assert eng.status_slots() == (allocated, 0)


def tiles_run(eng, call):
    before = eng.stats()["batches_timed"]
    result = call()
    return result, eng.stats()["batches_timed"] - before


def recover(eng, b, crcs):
    parts = [None if i in LOST else b.parts[i] for i in range(K + M)]
    return eng.recover_chunks(L.SliceType("ec(8,2)"), NB, parts, part_crc=crcs, chunk_image=True)


def check_recover(b, out, img):
    for i in LOST:
        assert (out[i] == b.parts[i]).all(), i
    assert (img == b.chunks).all()


def corrupt(crcs, *where):
    crcs = list(crcs)
    for c, p, blk in where:
        crcs[p] = crcs[p].copy()
        crcs[p][c, blk] ^= 0x10
    return crcs


@pytest.mark.parametrize("with_crc", [True, False])
def test_recover_over_four_tiles_matches_the_oracle(eng, batch, oracle, with_crc):
    allocated = eng.status_slots()[0]
    (out, img), tiles = tiles_run(eng, lambda: recover(eng, batch, batch.pcrc if with_crc else None))
    assert tiles == 4
    check_recover(batch, out, img)
    for c in boundary_chunks(T_REC, N_REC):
        p_ref, c_ref = oracle.encode_chunk(1, K, M, batch.chunks[c])
        assert (batch.parity[c] == p_ref).all() and (batch.crc[c] == c_ref).all(), c
        avail = [None if i in LOST else batch.parts[i][c] for i in range(K + M)]
        rc, ref_out, _ = oracle.recover_chunk(1, K, M, avail, [None if i in LOST else batch.pcrc[i][c] for i in range(K + M)],
                                              [1 if i in LOST else 0 for i in range(K + M)], PB)
        assert rc == 0
        for i in LOST:
            assert (out[i][c] == ref_out[i]).all(), (c, i)
    check_slots_returned(eng, allocated)


def test_recover_reports_the_first_mismatch_of_a_later_tile_at_its_batch_position(eng, batch):
    allocated = eng.status_slots()[0]
    first = (2 * T_REC + 5, USED[4], 2)
    crcs = corrupt(batch.pcrc, first, (3 * T_REC + 1, USED[0], 0))
    with pytest.raises(L.ChunkCrcError) as ei:
        recover(eng, batch, crcs)
    assert ei.value.where == first
    check_slots_returned(eng, allocated)


def test_recover_mismatch_in_tile_0_with_later_tiles_in_flight(eng, batch):
    allocated = eng.status_slots()[0]
    first = (5, USED[-1], 1)
    with pytest.raises(L.ChunkCrcError) as ei:
        recover(eng, batch, corrupt(batch.pcrc, first))
    assert ei.value.where == first
    check_slots_returned(eng, allocated)
    out, img = recover(eng, batch, batch.pcrc)                         # the next call on the context
    check_recover(batch, out, img)
    check_slots_returned(eng, allocated)


def convert(eng, b, source, crcs):
    want = [1] * (KD + 2)
    if source == "ec(8,2)":
        parts = [None if i in LOST else b.parts[i][:N_CONV] for i in range(K + M)]
        return eng.convert_chunks(L.SliceType("ec(8,2)"), L.SliceType("ec(3,2)"), NB, parts, want, part_crc=crcs)
    return eng.convert_chunks(L.SliceType("std"), L.SliceType("ec(3,2)"), NB, [b.chunks[:N_CONV]], want, part_crc=crcs)


def source_crcs(b, source):
    if source == "ec(8,2)":
        return [None if i in LOST else c[:N_CONV] for i, c in enumerate(b.pcrc)]
    return [np.ascontiguousarray(b.crc[:N_CONV, :NB])]


def check_convert(b, out, ocrc):
    blocks = b.chunks[:N_CONV].reshape(N_CONV, PBD, KD, BLOCK)
    for j in range(KD):
        assert (out[j] == blocks[:, :, j].reshape(N_CONV, -1)).all(), j
        assert (ocrc[j] == b.c32[:, :NB].reshape(N_CONV, PBD, KD)[:, :, j]).all(), j
    for r in range(2):
        assert (out[KD + r] == b.p32[:, r]).all(), r
        assert (ocrc[KD + r] == b.c32[:, NB + r * PBD: NB + (r + 1) * PBD]).all(), r


@pytest.mark.parametrize("source", ["ec(8,2)", "std"])
def test_convert_over_four_tiles_matches_the_oracle(eng, batch, oracle, source):
    allocated = eng.status_slots()[0]
    crcs = source_crcs(batch, source)
    (out, ocrc), tiles = tiles_run(eng, lambda: convert(eng, batch, source, crcs))
    assert tiles == 4
    check_convert(batch, out, ocrc)
    src = (1, K, M) if source == "ec(8,2)" else (2, 1, 0)
    for c in boundary_chunks(T_CONV, N_CONV):
        if source == "ec(8,2)":
            avail = [None if i in LOST else batch.parts[i][c] for i in range(K + M)]
        else:
            avail = [batch.chunks[c]]
        rc, ref_out, ref_crc, _ = O.convert_chunk(oracle, src, avail, [None if x is None else x[c] for x in crcs], (1, KD, 2), [1] * (KD + 2), NB)
        assert rc == 0
        for i in range(KD + 2):
            assert (out[i][c] == ref_out[i]).all() and (ocrc[i][c] == ref_crc[i]).all(), (c, i)
    check_slots_returned(eng, allocated)


@pytest.mark.parametrize("source", ["ec(8,2)", "std"])
def test_convert_reports_the_first_mismatch_of_a_later_tile_at_its_batch_position(eng, batch, source):
    allocated = eng.status_slots()[0]
    p0, p1 = (USED[5], USED[1]) if source == "ec(8,2)" else (0, 0)
    first = (2 * T_CONV + 9, p0, 2 if source == "ec(8,2)" else 17)
    crcs = corrupt(source_crcs(batch, source), first, (3 * T_CONV + 2, p1, 1))
    with pytest.raises(L.ChunkCrcError) as ei:
        convert(eng, batch, source, crcs)
    assert ei.value.where == first
    check_slots_returned(eng, allocated)


@pytest.mark.parametrize("source", ["ec(8,2)", "std"])
def test_convert_mismatch_in_tile_0_with_later_tiles_in_flight(eng, batch, source):
    allocated = eng.status_slots()[0]
    first = (3, USED[2], 0) if source == "ec(8,2)" else (3, 0, 23)
    with pytest.raises(L.ChunkCrcError) as ei:
        convert(eng, batch, source, corrupt(source_crcs(batch, source), first))
    assert ei.value.where == first
    check_slots_returned(eng, allocated)
    out, ocrc = convert(eng, batch, source, source_crcs(batch, source))
    check_convert(batch, out, ocrc)
    check_slots_returned(eng, allocated)


def test_deferred_mismatch_returns_every_slot_at_sync(eng, batch):
    """device-pointer calls in deferred mode hold their slots until lzgpu_dev_sync; after a mismatch there every slot is back"""
    import torch
    dev = torch.device("cuda", 0)
    n = 4
    allocated = eng.status_slots()[0]
    d_parts = [None if i in LOST else torch.from_numpy(batch.parts[i][:n]).to(dev) for i in range(K + M)]
    good = [None if i in LOST else torch.from_numpy(batch.pcrc[i][:n].view(np.int32)).to(dev) for i in range(K + M)]
    bad = list(good)
    bad_crc = batch.pcrc[USED[3]][:n].copy()
    bad_crc[2, 1] ^= 1
    bad[USED[3]] = torch.from_numpy(bad_crc.view(np.int32)).to(dev)
    outs = [torch.empty(n * PB * BLOCK, dtype=torch.uint8, device=dev) if i in LOST else None for i in range(K + M)]
    d32 = [torch.empty(n * PBD * BLOCK, dtype=torch.uint8, device=dev) for _ in range(KD + 2)]
    torch.cuda.synchronize()
    ptrs = lambda ts: [0 if t is None else t.data_ptr() for t in ts]  # noqa: E731

    def recover_dev(crcs):
        eng.recover_chunks_dev(L.SliceType("ec(8,2)"), n, NB, ptrs(d_parts), PB * BLOCK, ptrs(crcs), [1 if i in LOST else 0 for i in range(K + M)],
                               ptrs(outs))

    def convert_dev(crcs):
        eng.convert_chunks_dev(L.SliceType("ec(8,2)"), L.SliceType("ec(3,2)"), n, NB, ptrs(d_parts), PB * BLOCK, [1] * (KD + 2), ptrs(d32),
                               PBD * BLOCK, d_part_crc=ptrs(crcs))

    eng.set_deferred_verify(True)
    try:
        recover_dev(good); convert_dev(bad); recover_dev(bad); convert_dev(good)
        assert eng.status_slots()[1] == 4                               # one slot per verifying call, held until the sync
        with pytest.raises(L.ChunkCrcError) as ei:
            eng.sync()
        assert ei.value.where == (2, USED[3], 1)
        check_slots_returned(eng, allocated)
    finally:
        eng.set_deferred_verify(False)
    allocated = eng.status_slots()[0]
    with pytest.raises(L.ChunkCrcError):                                # immediate mode: the call reports and returns its slot
        convert_dev(bad)
    check_slots_returned(eng, allocated)
