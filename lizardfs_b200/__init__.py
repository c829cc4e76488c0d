"""lizardfs_b200 — H100-native erasure-coding + CRC32 engine behind LizardFS's
Goal / slice_traits / ReedSolomon / blockXor / mycrc32 interfaces.

The package is a thin host-side mirror (ctypes) over liblzgpu.so, the C-ABI library whose
kernels are hand-written CUDA for sm_90a.  No CPU fallback exists: importing the package
without the built library, or creating an Engine without an H100 (sm_90), fails loudly.
"""
from . import _lib  # noqa: F401
from ._lib import BLOCK_SIZE, BLOCKS_IN_CHUNK, CHUNK_SIZE  # noqa: F401
from .engine import (ChunkCrcError, Engine, LzGpuError, Pool, ReedSolomon, SliceType, blockXor, ec_encode_data,  # noqa: F401
                     ec_init_tables, encoder_kernels, gf_gen_cauchy1_matrix, gf_gen_rs_matrix, gf_inv, gf_invert_matrix, gf_mul,
                     mycrc32, mycrc32_combine, mycrc32_init, mycrc32_xorblocks, mycrc32_zeroblock,
                     mycrc32_zeroexpanded, recompute_crc_if_block_empty)

_lib.load()
