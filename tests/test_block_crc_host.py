"""lzgpu_mycrc32_subrange (host scalar, no GPU needed) against zlib.crc32 of the range itself.

lzgpu::StripeBatcher CRCs every sub-block packet by running the whole 64 KiB block, zero outside the written range, through the
batched CRC kernel, and then asks lzgpu_mycrc32_subrange for the CRC of the range alone: each packet carries that value, and a
wrong one is a corrupt packet to every chunkserver that receives it."""
import zlib

import numpy as np
import pytest

from lizardfs_b200 import _lib

BLOCK = 65536


def subrange(block, lo, hi):
    return int(_lib.load().lzgpu_mycrc32_subrange(zlib.crc32(block.tobytes()), lo, hi))


def padded(rng, lo, hi):
    """a 64 KiB block that is zero outside [lo, hi) and random inside"""
    block = np.zeros(BLOCK, dtype=np.uint8)
    block[lo:hi] = rng.integers(0, 256, hi - lo, dtype=np.uint8)
    return block


@pytest.mark.parametrize("lo,hi", [(0, 1), (0, BLOCK), (BLOCK - 1, BLOCK), (1, BLOCK - 1), (32768, 32769), (0, 4), (3, 260), (65532, 65536)])
def test_subrange_edges(lo, hi):
    rng = np.random.default_rng(lo * 7 + hi)
    for _ in range(3):
        block = padded(rng, lo, hi)
        assert subrange(block, lo, hi) == zlib.crc32(block[lo:hi].tobytes()), (lo, hi)
    zeros = np.zeros(BLOCK, dtype=np.uint8)                          # the range itself may be zero too
    assert subrange(zeros, lo, hi) == zlib.crc32(bytes(hi - lo)), (lo, hi)


def test_subrange_random_ranges():
    rng = np.random.default_rng(162)
    for i in range(500):
        lo = int(rng.integers(0, BLOCK))
        # half the ranges short, so that both ends vary at the byte level near every position
        hi = lo + 1 + int(rng.integers(0, min(BLOCK - lo, 64) if i % 2 else BLOCK - lo))
        block = padded(rng, lo, hi)
        assert subrange(block, lo, hi) == zlib.crc32(block[lo:hi].tobytes()), (i, lo, hi)


def test_subrange_refusals_return_zero():
    lib = _lib.load()
    crc = zlib.crc32(bytes(BLOCK))
    for lo, hi in [(0, 0), (5, 5), (BLOCK, BLOCK), (7, 3), (BLOCK - 1, 0), (0, BLOCK + 1), (BLOCK, BLOCK + 1), (100, 0xFFFFFFFF)]:
        assert lib.lzgpu_mycrc32_subrange(crc, lo, hi) == 0, (lo, hi)
    assert lib.lzgpu_mycrc32_subrange(0x12345678, 1, 0) == 0
