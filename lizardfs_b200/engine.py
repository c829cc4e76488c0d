"""Host-side mirror of the reference's interface for the erasure-coding + CRC hot path.

Names, argument meaning and error behaviour follow the reference (paths relative to the
lizardfs tree) so that the parity tests read like the reference's own unit tests:

  ReedSolomon(k, m).encode / .recover      src/common/reed_solomon.h:41-155
  mycrc32 / mycrc32_combine / mycrc32_zeroblock / mycrc32_zeroexpanded / mycrc32_xorblocks
                                           src/common/crc.h:25-36
  blockXor(dest, source)                   src/common/block_xor.h:33
  gf_gen_rs_matrix ... ec_encode_data      src/common/galois_field.h:35-88
  SliceType / part geometry                src/common/goal.h:99-177, slice_traits.h:96-349
  Engine.encode_chunks / recover_chunks    chunk-level batches behind ChunkWriter::startOperation
                                           (src/mount/chunk_writer.cc:475-547) and
                                           ReadPlan::postProcessData (src/common/read_plan.h:141-160)

Everything here is a thin ctypes veneer over the C ABI (include/lzgpu.h): all arithmetic on chunk
bytes happens in the CUDA kernels of liblzgpu.so.  numpy is used only to own host buffers.
"""
import ctypes as C
import math

import numpy as np

from . import _lib
from ._lib import BLOCK_SIZE, BLOCKS_IN_CHUNK, CHUNK_SIZE, LzGoal, LzStats


class LzGpuError(RuntimeError):
    def __init__(self, status, where):
        self.status = status
        super().__init__(f"{where}: status {status}: {_lib.last_error()}")


class ChunkCrcError(LzGpuError):
    """CRC mismatch — the analogue of ChunkCrcException (read_operation_executor.cc:262-264) /
    LIZARDFS_ERROR_CRC (hddspacemgr.cc:1918-1920).  `.where` = (chunk, part, block) or (block,)."""

    def __init__(self, status, where_txt, where):
        super().__init__(status, where_txt)
        self.where = where


def _check(rc, where):
    if rc != _lib.OK:
        raise LzGpuError(rc, where)


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _u8(a):
    a = np.asarray(a)
    if a.dtype != np.uint8 or not a.flags.c_contiguous:
        a = np.ascontiguousarray(a, dtype=np.uint8)
    return a


def _ptr_array(arrs):
    out = (C.c_void_p * len(arrs))()
    for i, a in enumerate(arrs):
        out[i] = None if a is None else a.ctypes.data
    out._arrays = arrs                  # the pointers stay valid as long as the array of them
    return out


def _dev_ptrs(ptrs, n):
    """C array of n device pointers (ints; 0 or None = absent), None for None"""
    return None if ptrs is None else (C.c_void_p * n)(*[p if p else None for p in ptrs])


def _host_parts(parts, part_crc, pb, in_place=False, crc_rows=False):
    """The parts of a host-pointer batch call, each None or [n_chunks, pb * 64 KiB] uint8 (in_place: the call writes into them, so
    each must already be a writeable C-contiguous uint8 array), and their stored CRCs (uint32, crc_rows: [n_chunks, pb] each).
    Returns (parts, n_chunks, C array of the CRC pointers or None)."""
    if in_place:
        for p in parts:
            if p is not None and not (isinstance(p, np.ndarray) and p.dtype == np.uint8 and p.flags.c_contiguous and p.flags.writeable):
                raise ValueError("correct_stripes corrects the parts in place: each must be a writeable C-contiguous uint8 array")
    parts = [None if p is None else (p if in_place else _u8(p)).reshape(-1, pb * BLOCK_SIZE) for p in parts]
    n = next(p.shape[0] for p in parts if p is not None)
    if part_crc is None:
        return parts, n, None
    crcs = [None if c is None else np.ascontiguousarray(c, dtype=np.uint32) for c in part_crc]
    if crc_rows:
        crcs = [None if c is None else c.reshape(n, pb) for c in crcs]
    return parts, n, _ptr_array(crcs)


def _check_crc(rc, where, bad, **result):
    """Raises ChunkCrcError on a stored-CRC mismatch (.where = bad; `result`, e.g. verdict=..., attached to it) and LzGpuError on
    any other failure.  A call that returns a `result` may also return ERR_INCONSISTENT: the result says where, it is no failure."""
    if rc == _lib.ERR_CRC:
        err = ChunkCrcError(rc, where, tuple(bad))
        for name, value in result.items():
            setattr(err, name, value)
        raise err
    if not (result and rc == _lib.ERR_INCONSISTENT):
        _check(rc, where)


def _name(fn):
    return fn.__name__.removeprefix("lzgpu_")


# the bodies of the batch calls that Engine and Pool share, `fn` the C function (the context or the pool as its first argument)
def _goal_array(goals):
    arr = (LzGoal * len(goals))()
    for i, g in enumerate(goals):
        arr[i] = g.c
    return arr


def _encode_slices(fn, h, goals, data, chunk_len, out=None):
    """one (parity or None, crc) per slice: parity [n, m, pb * 64 KiB] and crc [n, nb + m * pb] for an xor/ec slice, parity None and
    crc [n, nb] for the standard slice.  out: the caller's (parity, crc) per slice, C-contiguous arrays of those shapes that the
    call writes into; a None among them is allocated here."""
    data = _u8(data)
    if data.ndim == 1:
        data = data.reshape(1, -1)
    n, stride = data.shape
    if chunk_len is None:
        chunk_len = stride
    ns = len(goals)
    par_stride, crc_stride = (C.c_size_t * ns)(), (C.c_size_t * ns)()
    res = []
    for i, (g, (parity, crc)) in enumerate(zip(goals, out or [(None, None)] * ns)):
        nb, pb = Engine.geometry(g, chunk_len)
        m = 0 if g.is_std else g.m
        par_stride[i], crc_stride[i] = m * pb * BLOCK_SIZE, nb + m * pb
        if parity is None and m:
            parity = np.empty((n, m, pb * BLOCK_SIZE), dtype=np.uint8)
        if crc is None:
            crc = np.empty((n, nb + m * pb), dtype=np.uint32)
        res.append((parity, crc))
    _check(fn(h, _goal_array(goals), ns, n, chunk_len, _p(data), stride, _ptr_array([p for p, _ in res]), par_stride,
              _ptr_array([c for _, c in res]), crc_stride), _name(fn))
    return res


def _encode_chunks(fn, h, goal, data, chunk_len, parity=None, crc=None):
    """_encode_slices for one xor/ec slice through the one-goal C call: scalars where that takes one-entry arrays"""
    def one(h, goals, ns, n, chunk_len, data, stride, parity, par_stride, crc, crc_stride):
        return fn(h, goals, n, chunk_len, data, stride, parity[0], par_stride[0], crc[0], crc_stride[0])
    one.__name__ = fn.__name__
    return _encode_slices(one, h, [goal], data, chunk_len, [(parity, crc)])[0]


def _recover_chunks(fn, h, goal, nb, parts, part_crc, want, chunk_image):
    n_parts = goal.k + goal.m
    assert len(parts) == n_parts
    pb = (nb + goal.k - 1) // goal.k
    parts, n, crcs = _host_parts(parts, part_crc, pb)
    if want is None:
        want = [1 if (parts[i] is None and i < goal.k) else 0 for i in range(n_parts)]
    w = np.asarray(want, dtype=np.uint8)
    out = [np.zeros((n, pb * BLOCK_SIZE), dtype=np.uint8) if (w[i] and parts[i] is None) else None for i in range(n_parts)]
    img = np.zeros((n, nb * BLOCK_SIZE), dtype=np.uint8) if chunk_image else None
    bad = (C.c_int64 * 3)(-1, -1, -1)
    rc = fn(h, C.byref(goal.c), n, nb, _ptr_array(parts), pb * BLOCK_SIZE, crcs, _p(w), _ptr_array(out), _p(img), nb * BLOCK_SIZE, bad)
    _check_crc(rc, _name(fn), bad)
    return out, img


def _convert_chunks(fn, h, src, dst, nb, parts, want, part_crc, with_crc):
    ns, nd = src.k + src.m, dst.k + dst.m
    pbs, pbd = -(-nb // src.k), -(-nb // dst.k)
    arrs, n, crcs = _host_parts(parts, part_crc, pbs, crc_rows=True)
    w = np.asarray(want, dtype=np.uint8)
    assert len(arrs) == ns and w.size == nd
    out = [np.zeros((n, pbd * BLOCK_SIZE), dtype=np.uint8) if w[i] else None for i in range(nd)]
    ocrc = [np.zeros((n, pbd), dtype=np.uint32) if (w[i] and with_crc) else None for i in range(nd)]
    bad = (C.c_int64 * 3)(-1, -1, -1)
    rc = fn(h, C.byref(src.c), C.byref(dst.c), n, nb, _ptr_array(arrs), pbs * BLOCK_SIZE, crcs, _p(w), _ptr_array(out), pbd * BLOCK_SIZE,
            _ptr_array(ocrc) if with_crc else None, bad)
    _check_crc(rc, _name(fn), bad)
    return out, ocrc


def _n_flat(goals):
    """the flat parts of a multi-slice goal: slice i's k + m parts after those of the slices before it, one for the standard slice"""
    return sum(1 if g.is_std else g.k + g.m for g in goals)


def _slices_host(goals, nb, parts, part_crc, in_place=False):
    """The shared preamble of the multi-slice host-pointer calls.  parts: one entry per flat part, each None or [n_chunks, pb_i *
    64 KiB] uint8 (in_place: the call corrects them, so each must already be a writeable C-contiguous uint8 array).  Returns (parts,
    n_chunks, C array of the stored-CRC pointers or None, C array of the part strides per slice, pb per flat part, L); n_chunks is 0
    when no part is given, for the library to refuse the call."""
    pbs = [-(-nb // g.k) for g in goals]
    pb = [pbs[i] for i, g in enumerate(goals) for _ in range(1 if g.is_std else g.k + g.m)]
    assert len(parts) == len(pb)
    if in_place:
        for p in parts:
            if p is not None and not (isinstance(p, np.ndarray) and p.dtype == np.uint8 and p.flags.c_contiguous and p.flags.writeable):
                raise ValueError("correct_slices corrects the parts in place: each must be a writeable C-contiguous uint8 array")
    arrs = [None if p is None else (p if in_place else _u8(p)).reshape(-1, pb[j] * BLOCK_SIZE) for j, p in enumerate(parts)]
    n = next((a.shape[0] for a in arrs if a is not None), 0)
    crcs = None if part_crc is None else _ptr_array([None if c is None else np.ascontiguousarray(c, dtype=np.uint32) for c in part_crc])
    strides = (C.c_size_t * len(goals))(*[p * BLOCK_SIZE for p in pbs])
    return arrs, n, crcs, strides, pb, math.lcm(*[g.k for g in goals if not g.is_std])


def _recover_slices(fn, h, goals, nb, parts, part_crc, want, chunk_image, with_crc):
    arrs, n, crcs, strides, pb, _ = _slices_host(goals, nb, parts, part_crc)
    if want is None:
        want = [1 if a is None else 0 for a in arrs]
    w = np.asarray(want, dtype=np.uint8)
    out = [np.zeros((n, pb[j] * BLOCK_SIZE), dtype=np.uint8) if w[j] else None for j in range(len(arrs))]
    ocrc = [np.zeros((n, pb[j]), dtype=np.uint32) if (w[j] and with_crc) else None for j in range(len(arrs))]
    img = np.zeros((n, nb * BLOCK_SIZE), dtype=np.uint8) if chunk_image else None
    bad = (C.c_int64 * 4)(-1, -1, -1, -1)
    rc = fn(h, _goal_array(goals), len(goals), n, nb, _ptr_array(arrs), strides, crcs, _p(w), _ptr_array(out), strides,
            _ptr_array(ocrc) if with_crc else None, _p(img), nb * BLOCK_SIZE, bad)
    _check_crc(rc, _name(fn), bad)
    return out, ocrc, img


def _salvage_slices(fn, h, goals, nb, parts, part_crc, with_crc):
    arrs, n, crcs, strides, _, _ = _slices_host(goals, nb, parts, part_crc)
    img = np.zeros((n, nb * BLOCK_SIZE), dtype=np.uint8)
    icrc = np.zeros((n, nb), dtype=np.uint32) if with_crc else None
    smap = np.zeros((n, nb), dtype=np.uint8)
    bad = (C.c_int64 * 4)(-1, -1, -1, -1)
    rc = fn(h, _goal_array(goals), len(goals), n, nb, _ptr_array(arrs), strides, crcs, _p(img), nb * BLOCK_SIZE, _p(icrc), _p(smap), bad)
    _check_crc(rc, _name(fn), bad, image=img, image_crc=icrc, map=smap)
    return img, icrc, smap


SLICES_CHECK_DTYPE = np.dtype([("bad_checks", np.uint64), ("suspect_part", np.int32), ("zero", np.uint32)])


def _check_slices(fn, h, goals, nb, parts, part_crc):
    arrs, n, crcs, strides, _, L = _slices_host(goals, nb, parts, part_crc)
    out = np.zeros((n, -(-nb // L)), dtype=SLICES_CHECK_DTYPE)
    bad = (C.c_int64 * 4)(-1, -1, -1, -1)
    rc = fn(h, _goal_array(goals), len(goals), n, nb, _ptr_array(arrs), strides, crcs, _p(out), bad)
    _check_crc(rc, _name(fn), bad, map=out)
    return out


SLICES_FIX_DTYPE = np.dtype([("bad_checks", np.uint64), ("suspect_part", np.int32), ("status", np.int32), ("crc_failed", np.uint64),
                             ("changed", np.uint64)])


def _correct_slices(fn, h, goals, nb, parts, part_crc, with_crc):
    arrs, n, crcs, strides, pb, L = _slices_host(goals, nb, parts, part_crc, in_place=True)
    new_crc = [np.zeros((n, pb[j]), dtype=np.uint32) if (a is not None and with_crc) else None for j, a in enumerate(arrs)]
    fix = np.zeros((n, -(-nb // L)), dtype=SLICES_FIX_DTYPE)
    bad = (C.c_int64 * 4)(-1, -1, -1, -1)
    rc = fn(h, _goal_array(goals), len(goals), n, nb, _ptr_array(arrs), strides, crcs, _ptr_array(new_crc) if with_crc else None, _p(fix),
            bad)
    _check_crc(rc, _name(fn), bad, fix=fix, new_crc=new_crc if with_crc else None)
    return fix, (new_crc if with_crc else None)


def _part_batch(fn, h, goal, nb, parts, part_crc, result, attr, in_place=False):
    # the host-pointer check, map and correction: result(n_chunks, pb) makes the array the call fills, which is returned, and
    # attached to a ChunkCrcError as `attr`
    assert len(parts) == goal.k + goal.m
    pb = (nb + goal.k - 1) // goal.k
    parts, n, crcs = _host_parts(parts, part_crc, pb, in_place=in_place)
    out = result(n, pb)
    bad = (C.c_int64 * 3)(-1, -1, -1)
    rc = fn(h, C.byref(goal.c), n, nb, _ptr_array(parts), pb * BLOCK_SIZE, crcs, _p(out), bad)
    _check_crc(rc, _name(fn), bad, **{attr: out})
    return out


def _stripe_fix(fn, h, goal, nb, parts, part_crc, dtype):
    # the host-pointer repair and decode: the parts are rewritten in place, the entries of `dtype` [n_chunks, pb] are returned
    # and attached to a ChunkCrcError as .fix
    assert len(parts) == goal.k + goal.m
    pb = (nb + goal.k - 1) // goal.k
    parts, n, crcs = _host_parts(parts, part_crc, pb, in_place=True)
    out = np.empty((n, pb), dtype=dtype)
    rc = fn(h, C.byref(goal.c), n, nb, _ptr_array(parts), pb * BLOCK_SIZE, crcs, _p(out))
    _check_crc(rc, _name(fn), (-1, -1, -1), fix=out)
    return out


def _verify_blocks(fn, h, data, stored_crc, block_len, sparse_rule):
    data = _u8(data).reshape(-1)
    stored = np.ascontiguousarray(stored_crc, dtype=np.uint32)
    bad = C.c_int64(-1)
    rc = fn(h, _p(data), stored.size, block_len, block_len, _p(stored), int(sparse_rule), C.byref(bad))
    _check_crc(rc, _name(fn), (bad.value,))


def _verify_interleaved(fn, h, records):
    records = _u8(records).reshape(-1)
    n = records.size // (4 + BLOCK_SIZE)
    bad = C.c_int64(-1)
    rc = fn(h, _p(records), n, C.byref(bad))
    _check_crc(rc, _name(fn), (bad.value,))


# ------------------------------------------------------------------------------------------------
# goals / slice types
# ------------------------------------------------------------------------------------------------
class SliceType:
    """xorN / ec(k,m) slice type.  Part indices in this package: data 0..k-1, parity k..k+m-1."""

    def __init__(self, text_or_kind, k=None, m=None):
        lib = _lib.load()
        g = LzGoal()
        if text_or_kind == 2 and (k, m) == (1, 0):
            g.kind, g.k, g.m = 2, 1, 0      # standard slice: only Engine.convert_chunks accepts it
        elif isinstance(text_or_kind, str):
            if lib.lzgpu_goal_parse(text_or_kind.encode(), C.byref(g)) != 0:
                raise ValueError(f"bad goal {text_or_kind!r} (expected xorN with N in 2..9 or ec(K,M) with K in 2..32, M in 1..32)")
        else:
            g.kind, g.k, g.m = int(text_or_kind), int(k), int(m)
            if not lib.lzgpu_goal_valid(C.byref(g)):
                raise ValueError("invalid goal")
        self.c = g

    kind = property(lambda s: s.c.kind)
    k = property(lambda s: s.c.k)
    m = property(lambda s: s.c.m)
    is_xor = property(lambda s: s.c.kind == 0)
    is_std = property(lambda s: s.c.kind == 2)

    @classmethod
    def from_id(cls, type_id):
        g = LzGoal()
        if _lib.load().lzgpu_goal_from_slice_type(int(type_id), C.byref(g)) != 0:
            raise ValueError("not an xor/ec slice type id")
        return cls(g.kind, g.k, g.m)

    def type_id(self):
        if self.is_std:
            return 0                        # Goal::Slice::Type::kStandard (goal.h:108-120)
        return _lib.load().lzgpu_goal_slice_type(C.byref(self.c))

    def chunk_part_id(self, part):
        return _lib.load().lzgpu_chunk_part_id(C.byref(self.c), part)

    def ref_part_index(self, part):
        return _lib.load().lzgpu_ref_part_index(C.byref(self.c), part)

    def part_blocks(self, part, blocks_in_chunk=BLOCKS_IN_CHUNK):
        return _lib.load().lzgpu_part_blocks(C.byref(self.c), part, blocks_in_chunk)

    def part_length(self, part, chunk_length):
        return _lib.load().lzgpu_part_length(C.byref(self.c), part, chunk_length)

    def __str__(self):
        return "std" if self.is_std else f"xor{self.k}" if self.is_xor else f"ec({self.k},{self.m})"

    __repr__ = __str__


# ------------------------------------------------------------------------------------------------
# reference-shaped free functions
# ------------------------------------------------------------------------------------------------
def mycrc32(crc, block):
    block = _u8(block)
    return _lib.load().lzgpu_mycrc32(crc, _p(block), block.size)


def mycrc32_combine(crc1, crc2, leng2):
    return _lib.load().lzgpu_mycrc32_combine(crc1, crc2, leng2)


def mycrc32_zeroblock(crc, zeros):
    return _lib.load().lzgpu_mycrc32_zeroblock(crc, zeros)


def mycrc32_zeroexpanded(crc, block, zeros):
    block = _u8(block)
    return _lib.load().lzgpu_mycrc32_zeroexpanded(crc, _p(block), block.size, zeros)


def mycrc32_xorblocks(crc, crcblock1, crcblock2, leng):
    return _lib.load().lzgpu_mycrc32_xorblocks(crc, crcblock1, crcblock2, leng)


def mycrc32_init():
    _lib.load().lzgpu_mycrc32_init()


def recompute_crc_if_block_empty(block, crc):
    block = _u8(block)
    c = C.c_uint32(crc)
    _lib.load().lzgpu_recompute_crc_if_block_empty(_p(block), C.byref(c))
    return c.value


def blockXor(dest, source):
    """dest ^= source, in place (dest must be a writable contiguous uint8 array)."""
    assert dest.dtype == np.uint8 and dest.flags.c_contiguous and dest.flags.writeable
    source = _u8(source)
    assert source.size >= dest.size or source.size == dest.size
    _lib.load().lzgpu_block_xor(_p(dest), _p(source), min(dest.size, source.size))


def gf_mul(a, b):
    return _lib.load().gf_mul(a, b)


def gf_inv(a):
    return _lib.load().gf_inv(a)


def gf_gen_rs_matrix(m, k):
    a = np.zeros((m, k), dtype=np.uint8)
    _lib.load().gf_gen_rs_matrix(_p(a), m, k)
    return a


def gf_gen_cauchy1_matrix(m, k):
    a = np.zeros((m, k), dtype=np.uint8)
    _lib.load().gf_gen_cauchy1_matrix(_p(a), m, k)
    return a


def gf_invert_matrix(mat):
    mat = np.array(mat, dtype=np.uint8, copy=True)
    n = mat.shape[0]
    out = np.zeros((n, n), dtype=np.uint8)
    rc = _lib.load().gf_invert_matrix(_p(mat), _p(out), n)
    return rc, out


def ec_init_tables(k, rows, a):
    a = _u8(a)
    t = np.zeros(32 * k * rows, dtype=np.uint8)
    _lib.load().ec_init_tables(k, rows, _p(a), _p(t))
    return t


def ec_encode_data(length, tables, src, n_dest):
    """ISA-L shaped call: `tables` from ec_init_tables, `src` list of uint8 arrays; returns dest list."""
    src = [_u8(s) for s in src]
    dest = [np.zeros(length, dtype=np.uint8) for _ in range(n_dest)]
    tables = _u8(tables)
    _lib.load().ec_encode_data(length, len(src), n_dest, _p(tables), _ptr_array(src), _ptr_array(dest))
    return dest



class Pool:
    """Several GPUs behind one process (lzgpu_pool in include/lzgpu.h): one context and one worker thread per device, a batch is
    cut into one contiguous run of chunks per device and every run goes through that device's own host pipeline.  `devices`:
    None = every visible device, an int mask, or a list of device numbers (a device may appear twice)."""

    def __init__(self, devices=None):
        self.lib = _lib.load()
        h = C.c_void_p()
        if devices is None or isinstance(devices, int):
            rc = self.lib.lzgpu_pool_create(int(devices or 0), C.byref(h))
        else:
            arr = (C.c_int * len(devices))(*devices)
            rc = self.lib.lzgpu_pool_create_list(arr, len(devices), C.byref(h))
        if rc != _lib.OK:
            raise LzGpuError(rc, f"lzgpu_pool_create({devices})")
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.lzgpu_pool_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return self.lib.lzgpu_pool_size(self.h)

    @staticmethod
    def share(n_chunks, n_devices, i):
        """(first chunk, count) of device slot i — pure host logic, usable without a GPU"""
        first, count = C.c_uint32(), C.c_uint32()
        _lib.load().lzgpu_pool_share(n_chunks, n_devices, i, C.byref(first), C.byref(count))
        return first.value, count.value

    def stats(self):
        s = LzStats()
        self.lib.lzgpu_pool_get_stats(self.h, C.byref(s))
        return {f[0]: getattr(s, f[0]) for f in LzStats._fields_}

    def encode_chunks(self, goal, data, chunk_len=None, parity=None, crc=None):
        return _encode_chunks(self.lib.lzgpu_pool_encode_chunks, self.h, goal, data, chunk_len, parity, crc)

    def encode_slices(self, goals, data, chunk_len=None):
        """Engine.encode_slices over every device of the pool (lzgpu_pool_encode_slices)"""
        return _encode_slices(self.lib.lzgpu_pool_encode_slices, self.h, goals, data, chunk_len)

    def recover_chunks(self, goal, nb, parts, part_crc=None, want=None, chunk_image=False):
        return _recover_chunks(self.lib.lzgpu_pool_recover_chunks, self.h, goal, nb, parts, part_crc, want, chunk_image)

    def convert_chunks(self, src, dst, nb, parts, want, part_crc=None, with_crc=True):
        """Engine.convert_chunks over every device of the pool (lzgpu_pool_convert_chunks)"""
        return _convert_chunks(self.lib.lzgpu_pool_convert_chunks, self.h, src, dst, nb, parts, want, part_crc, with_crc)

    def recover_slices(self, goals, nb, parts, part_crc=None, want=None, chunk_image=False, with_crc=True):
        """Engine.recover_slices over every device of the pool (lzgpu_pool_recover_slices): the same arguments, results and errors for
        the whole batch; ChunkCrcError.where = (chunk in the batch, slice, part, block)"""
        return _recover_slices(self.lib.lzgpu_pool_recover_slices, self.h, goals, nb, parts, part_crc, want, chunk_image, with_crc)

    def salvage_slices(self, goals, nb, parts, part_crc=None, with_crc=True):
        """Engine.salvage_slices over every device of the pool (lzgpu_pool_salvage_slices): the same arguments, results and errors for
        the whole batch; ChunkCrcError.where = (chunk in the batch, slice, part, block)"""
        return _salvage_slices(self.lib.lzgpu_pool_salvage_slices, self.h, goals, nb, parts, part_crc, with_crc)

    def check_slices(self, goals, nb, parts, part_crc=None):
        """Engine.check_slices over every device of the pool (lzgpu_pool_check_slices): the same arguments, map and errors for the
        whole batch; ChunkCrcError.where = (chunk in the batch, slice, part, block)"""
        return _check_slices(self.lib.lzgpu_pool_check_slices, self.h, goals, nb, parts, part_crc)

    def correct_slices(self, goals, nb, parts, part_crc=None, with_crc=True):
        """Engine.correct_slices over every device of the pool (lzgpu_pool_correct_slices): the same arguments, results and errors
        as on one context."""
        return _correct_slices(self.lib.lzgpu_pool_correct_slices, self.h, goals, nb, parts, part_crc, with_crc)

    def crc_blocks(self, data, block_len=BLOCK_SIZE):
        data = _u8(data).reshape(-1, block_len)
        out = np.empty(data.shape[0], dtype=np.uint32)
        _check(self.lib.lzgpu_pool_crc_blocks(self.h, _p(data), data.shape[0], block_len, block_len, _p(out)), "pool_crc_blocks")
        return out

    # the chunkserver's stripe consistency job and block scrub: the Engine methods of the same names over every device of the pool,
    # the same arguments, results and errors for the whole batch (lzgpu_pool_check_stripes ... in include/lzgpu.h)
    def check_stripes(self, goal, nb, parts, part_crc=None):
        return _part_batch(self.lib.lzgpu_pool_check_stripes, self.h, goal, nb, parts, part_crc,
                           lambda n, pb: np.empty(n, dtype=Engine.VERDICT_DTYPE), "verdict")

    def check_stripe_map(self, goal, nb, parts, part_crc=None):
        return _part_batch(self.lib.lzgpu_pool_check_stripe_map, self.h, goal, nb, parts, part_crc,
                           lambda n, pb: np.empty((n, pb), dtype=Engine.STRIPE_STATE_DTYPE), "map")

    def correct_stripes(self, goal, nb, parts, part_crc=None):
        return _part_batch(self.lib.lzgpu_pool_correct_stripes, self.h, goal, nb, parts, part_crc,
                           lambda n, pb: np.empty((n, pb), dtype=Engine.STRIPE_FIX_DTYPE), "fix", in_place=True)

    def check_stripe_map_degraded(self, goal, nb, parts, part_crc=None):
        return _part_batch(self.lib.lzgpu_pool_check_stripe_map_degraded, self.h, goal, nb, parts, part_crc,
                           lambda n, pb: np.empty((n, pb), dtype=Engine.STRIPE_STATE_DTYPE), "map")

    def correct_stripes_degraded(self, goal, nb, parts, part_crc=None):
        return _part_batch(self.lib.lzgpu_pool_correct_stripes_degraded, self.h, goal, nb, parts, part_crc,
                           lambda n, pb: np.empty((n, pb), dtype=Engine.STRIPE_FIX_DTYPE), "fix", in_place=True)

    def repair_stripes(self, goal, nb, parts, part_crc):
        return _stripe_fix(self.lib.lzgpu_pool_repair_stripes, self.h, goal, nb, parts, part_crc, Engine.STRIPE_REPAIR_DTYPE)

    def decode_stripes(self, goal, nb, parts, part_crc):
        return _stripe_fix(self.lib.lzgpu_pool_decode_stripes, self.h, goal, nb, parts, part_crc, Engine.STRIPE_DECODE_DTYPE)

    def verify_blocks(self, data, stored_crc, block_len=BLOCK_SIZE, sparse_rule=False):
        """host memory only: the pool refuses device pointers (ERR_ARG)"""
        _verify_blocks(self.lib.lzgpu_pool_verify_blocks, self.h, data, stored_crc, block_len, sparse_rule)

    def verify_interleaved(self, records):
        _verify_interleaved(self.lib.lzgpu_pool_verify_interleaved, self.h, records)


class ReedSolomon:
    """Mirror of ReedSolomon<32,32> (src/common/reed_solomon.h:41-155)."""

    kMaxDataCount = 32
    kMaxParityCount = 32

    def __init__(self, k, m):
        assert 1 <= k <= self.kMaxDataCount and 1 <= m <= self.kMaxParityCount
        self.k, self.m = k, m

    def generator(self):
        g = np.zeros((self.k + self.m, self.k), dtype=np.uint8)
        _check(_lib.load().lzgpu_rs_generator(self.k, self.m, _p(g)), "rs_generator")
        return g

    def recovery_matrix(self, erased, wanted):
        e = np.asarray(erased, dtype=np.uint8)
        w = np.asarray(wanted, dtype=np.uint8)
        out = np.zeros((self.m, self.k), dtype=np.uint8)
        rows = _lib.load().lzgpu_rs_recovery_matrix(self.k, self.m, _p(e), _p(w), _p(out))
        if rows < 0:
            raise LzGpuError(rows, "rs_recovery_matrix")
        return out[:rows]

    def encode(self, data_fragments, data_size=None):
        """data_fragments: k arrays or None (None = all-zero part). Returns m parity arrays."""
        frags = [None if f is None else _u8(f) for f in data_fragments]
        assert len(frags) == self.k
        if data_size is None:
            data_size = next(f.size for f in frags if f is not None)
        parity = [np.zeros(data_size, dtype=np.uint8) for _ in range(self.m)]
        _check(_lib.load().lzgpu_rs_encode(self.k, self.m, _ptr_array(frags), _ptr_array(parity), data_size), "rs_encode")
        return parity

    def recover(self, input_fragments, erased, wanted=None, data_size=None):
        """input_fragments: k+m arrays/None; erased: k+m flags (exactly m set); wanted: flags of the
        erased parts to rebuild (default: all erased).  Returns a list with arrays at rebuilt indices."""
        n = self.k + self.m
        frags = [None if f is None else _u8(f) for f in input_fragments]
        assert len(frags) == n and len(erased) == n
        if wanted is None:
            wanted = erased
        if data_size is None:
            data_size = next(f.size for f in frags if f is not None)
        out = [np.zeros(data_size, dtype=np.uint8) if (erased[i] and wanted[i]) else None for i in range(n)]
        e = np.asarray(erased, dtype=np.uint8)
        ins = [None if erased[i] else frags[i] for i in range(n)]
        _check(_lib.load().lzgpu_rs_recover(self.k, self.m, _ptr_array(ins), _p(e), _ptr_array(out), data_size), "rs_recover")
        return out


# ------------------------------------------------------------------------------------------------
# batched engine
# ------------------------------------------------------------------------------------------------
def encoder_kernels():
    """every compiled fused_stream_kernel instantiation (lzgpu_debug_encoder_kernels; pure host logic, no GPU needed), in the order
    Engine.last_encoder() indexes: a list of dicts of m, generic, bitsliced, striped, split, kt, gt (0: read at run time), item_bytes"""
    lib = _lib.load()
    n = lib.lzgpu_debug_encoder_kernels(None, 0)
    out = (_lib.LzEncoderKernel * n)()
    _check(0 if lib.lzgpu_debug_encoder_kernels(out, n) == n else _lib.ERR_ARG, "debug_encoder_kernels")
    return [{f: getattr(e, f) for f, _ in _lib.LzEncoderKernel._fields_} for e in out]


class Engine:
    """One context on one GPU.  Host arrays in, host arrays out; the *_dev methods take raw device
    pointers (ints, e.g. torch.Tensor.data_ptr()) and are asynchronous on the given stream."""

    def __init__(self, device=0):
        self.lib = _lib.load()
        h = C.c_void_p()
        rc = self.lib.lzgpu_ctx_create(device, C.byref(h))
        if rc != _lib.OK:
            raise LzGpuError(rc, f"lzgpu_ctx_create(device={device})")
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.lzgpu_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def stats(self):
        s = LzStats()
        self.lib.lzgpu_get_stats(self.h, C.byref(s))
        return {f[0]: getattr(s, f[0]) for f in LzStats._fields_}

    def last_launch(self):
        """(grid, units) of this context's most recent persistent kernel launch: CTAs launched and work units they shared
        (lzgpu_debug_last_launch; (0, 0) before the first)"""
        grid, units = C.c_uint32(), C.c_uint32()
        _check(self.lib.lzgpu_debug_last_launch(self.h, C.byref(grid), C.byref(units)), "debug_last_launch")
        return grid.value, units.value

    def last_geometry(self):
        """geometry of the same launch as last_launch() (lzgpu_debug_last_geometry): a dict of kernel (_lib.KERNEL_*), grid, units,
        threads, G (stripes per unit), stages, gf_warps and smem_bytes"""
        g = _lib.LzLaunchGeometry()
        _check(self.lib.lzgpu_debug_last_geometry(self.h, C.byref(g)), "debug_last_geometry")
        return {f: getattr(g, f) for f, _ in _lib.LzLaunchGeometry._fields_}

    def last_encoder(self):
        """(index, mode) of the same launch as last_geometry() (lzgpu_debug_last_encoder): its position in encoder_kernels() and its
        unit mode (0 per-chunk, 1 flat, 2 striped); (-1, 0) when that launch was not a fused_stream_kernel instantiation"""
        index, mode = C.c_int32(), C.c_uint32()
        _check(self.lib.lzgpu_debug_last_encoder(self.h, C.byref(index), C.byref(mode)), "debug_last_encoder")
        return index.value, mode.value

    def status_slots(self):
        """(allocated, in_use) verification result slots of this context (lzgpu_debug_status_slots)"""
        allocated, in_use = C.c_uint32(), C.c_uint32()
        _check(self.lib.lzgpu_debug_status_slots(self.h, C.byref(allocated), C.byref(in_use)), "debug_status_slots")
        return allocated.value, in_use.value

    def sync(self):
        """waits for the device; in deferred-verification mode also collects the verdicts of the *_dev calls issued since the last
        sync and raises ChunkCrcError for the first mismatch"""
        rc = self.lib.lzgpu_dev_sync(self.h)
        if rc == _lib.ERR_CRC:
            bad = (C.c_int64 * 3)(-1, -1, -1)
            self.lib.lzgpu_last_bad(self.h, bad)
            _check_crc(rc, "dev_sync (deferred verification)", bad)
        _check(rc, "dev_sync")

    def set_deferred_verify(self, enabled):
        _check(self.lib.lzgpu_ctx_set_deferred_verify(self.h, 1 if enabled else 0), "set_deferred_verify")

    # ---- geometry helpers -------------------------------------------------------------------
    @staticmethod
    def geometry(goal, chunk_len):
        nb = (chunk_len + BLOCK_SIZE - 1) // BLOCK_SIZE
        pb = (nb + goal.k - 1) // goal.k
        return nb, pb

    # ---- encode ------------------------------------------------------------------------------
    def encode_chunks(self, goal, data, chunk_len=None):
        """data: uint8 array [n_chunks, stride] (chunk order). Returns (parity [n, m, pb*64K], crc [n, nb+m*pb])."""
        return _encode_chunks(self.lib.lzgpu_encode_chunks, self.h, goal, data, chunk_len)

    def encode_slices(self, goals, data, chunk_len=None):
        """Encode the batch for every slice of a goal in one pass (lzgpu_encode_slices): goals = up to four SliceTypes, the standard
        slice among them at most once in practice.  Returns one (parity, crc) per slice, each as encode_chunks returns it for an xor/ec
        slice; (None, the nb data-block CRCs per chunk) for the standard slice."""
        return _encode_slices(self.lib.lzgpu_encode_slices, self.h, goals, data, chunk_len)

    def encode_slices_dev(self, goals, n_chunks, chunk_len, d_data, chunk_stride, d_parity, parity_stride, d_crc, crc_stride, stream=None):
        """lzgpu_encode_slices_dev: d_parity / d_crc / parity_stride / crc_stride are lists, one entry per slice (device pointers as
        ints; 0 or None for the standard slice's parity)"""
        ns = len(goals)
        _check(self.lib.lzgpu_encode_slices_dev(self.h, _goal_array(goals), ns, n_chunks, chunk_len, d_data, chunk_stride, _dev_ptrs(d_parity, ns),
                                                (C.c_size_t * ns)(*parity_stride), _dev_ptrs(d_crc, ns), (C.c_size_t * ns)(*crc_stride), stream),
               "encode_slices_dev")

    @staticmethod
    def plan_encode_slices(goals, n_chunks, nb):
        """how encode_slices would run the batch (pure host logic, csrc/fused_plan.h slices_plan; no GPU needed): dict with fused,
        refusal (SLICES_* in _lib), L, G, threads, stages, crc_rows, smem_bytes, units"""
        out = _lib.LzSlicesPlan()
        _check(_lib.load().lzgpu_plan_encode_slices(_goal_array(goals), len(goals), n_chunks, nb, C.byref(out)), "plan_encode_slices")
        return {f: getattr(out, f) for f, _ in _lib.LzSlicesPlan._fields_}

    def encode_chunks_dev(self, goal, n_chunks, chunk_len, d_data, chunk_stride, d_parity, parity_stride, d_crc, crc_stride, stream=None):
        _check(self.lib.lzgpu_encode_chunks_dev(self.h, C.byref(goal.c), n_chunks, chunk_len, d_data, chunk_stride, d_parity,
                                                parity_stride, d_crc, crc_stride, stream), "encode_chunks_dev")

    # ---- recover -----------------------------------------------------------------------------
    def recover_chunks(self, goal, nb, parts, part_crc=None, want=None, chunk_image=False):
        """parts: list of k+m arrays [n_chunks, pb*64K] or None (unavailable).
        part_crc: optional list of arrays [n_chunks, pb] (uint32) or None per part.
        want: flags of requested parts (default: every unavailable data part).
        Returns (out_list, chunk_out or None); raises ChunkCrcError on a stored-CRC mismatch."""
        return _recover_chunks(self.lib.lzgpu_recover_chunks, self.h, goal, nb, parts, part_crc, want, chunk_image)

    def recover_slices(self, goals, nb, parts, part_crc=None, want=None, chunk_image=False, with_crc=True):
        """Recover a chunk of a multi-slice goal from the given parts of every slice together (lzgpu_recover_slices).  goals: up to
        four SliceTypes; parts: one entry per flat part (slice i's k + m parts after those of the slices before it, one for the
        standard slice), an array [n_chunks, pb_i * 64K] or None (lost); part_crc: None, or one [n_chunks, pb_i] uint32 array or None
        per flat part.  want: flags per flat part (default: every lost part).  Returns (out, out_crc, image): out[g] / out_crc[g] for
        every wanted part (else None), image [n_chunks, nb * 64K] or None.  Raises LzGpuError(ERR_TOO_FEW_PARTS) when a block it must
        write is not determined, ChunkCrcError (.where = chunk, slice, part, block) on a stored-CRC mismatch."""
        return _recover_slices(self.lib.lzgpu_recover_slices, self.h, goals, nb, parts, part_crc, want, chunk_image, with_crc)

    def _slices_dev(self, fn, goals, n_chunks, nb, d_parts, part_stride, d_part_crc, stream, *own):
        # the multi-slice device-pointer calls: goals, the flat parts with their stored CRCs and part_stride per slice, then the
        # call's own arguments
        ns, n = len(goals), _n_flat(goals)
        bad = (C.c_int64 * 4)(-1, -1, -1, -1)
        rc = fn(self.h, _goal_array(goals), ns, n_chunks, nb, _dev_ptrs(d_parts, n), (C.c_size_t * ns)(*part_stride), _dev_ptrs(d_part_crc, n),
                *own, bad, stream)
        _check_crc(rc, _name(fn), bad)

    def recover_slices_dev(self, goals, n_chunks, nb, d_parts, part_stride, d_part_crc, want, d_out, out_stride, d_out_crc=None,
                           d_chunk_out=None, chunk_out_stride=0, stream=None):
        """lzgpu_recover_slices_dev: d_parts / d_part_crc / d_out / d_out_crc are lists over the flat parts (device pointers as ints,
        0 or None = absent), part_stride / out_stride one entry per slice.  Raises ChunkCrcError (.where = chunk, slice, part, block)."""
        n, w = _n_flat(goals), np.asarray(want, dtype=np.uint8)
        self._slices_dev(self.lib.lzgpu_recover_slices_dev, goals, n_chunks, nb, d_parts, part_stride, d_part_crc, stream, _p(w),
                         _dev_ptrs(d_out, n), (C.c_size_t * len(goals))(*out_stride), _dev_ptrs(d_out_crc, n), d_chunk_out, chunk_out_stride)

    def salvage_slices(self, goals, nb, parts, part_crc=None, with_crc=True):
        """Salvage the blocks of lost chunks of a multi-slice goal that the given parts of every slice still determine
        (lzgpu_salvage_slices).  goals, parts, part_crc as in recover_slices.  Returns (image, image_crc, map): image [n_chunks, nb * 64K]
        with every determined block and zeros elsewhere, image_crc [n_chunks, nb] uint32 (None without with_crc), map [n_chunks, nb]
        of _lib.SALVAGE_* per block.  Raises LzGpuError(ERR_TOO_FEW_PARTS) when no part is given; on a stored-CRC mismatch
        ChunkCrcError (.where = chunk, slice, part, block) with the still complete results as .image, .image_crc and .map."""
        return _salvage_slices(self.lib.lzgpu_salvage_slices, self.h, goals, nb, parts, part_crc, with_crc)

    def salvage_slices_dev(self, goals, n_chunks, nb, d_parts, part_stride, d_part_crc, d_image, image_stride, d_image_crc, d_map,
                           stream=None):
        """lzgpu_salvage_slices_dev: d_parts / d_part_crc are lists over the flat parts (device pointers as ints, 0 or None = absent),
        part_stride one entry per slice; d_image_crc may be None.  Raises ChunkCrcError (.where = chunk, slice, part, block); the device
        results are then still complete."""
        self._slices_dev(self.lib.lzgpu_salvage_slices_dev, goals, n_chunks, nb, d_parts, part_stride, d_part_crc, stream, d_image,
                         image_stride, d_image_crc, d_map)

    SLICES_CHECK_DTYPE = SLICES_CHECK_DTYPE

    def check_slices(self, goals, nb, parts, part_crc=None):
        """Do the given parts of every slice describe one chunk, combined stripe by combined stripe (lzgpu_check_slices)?  goals, parts,
        part_crc as in recover_slices.  Returns a structured array [n_chunks, ceil(nb / L)] of SLICES_CHECK_DTYPE (bad_checks, 0 =
        consistent; suspect_part, the flat part to blame or -1), whether or not any entry is bad; raises ChunkCrcError (.where = chunk,
        slice, part, block) on a stored-CRC mismatch, with the map, written in full all the same, as .map."""
        return _check_slices(self.lib.lzgpu_check_slices, self.h, goals, nb, parts, part_crc)

    def check_slices_dev(self, goals, n_chunks, nb, d_parts, part_stride, d_part_crc, d_map, stream=None):
        """lzgpu_check_slices_dev: d_parts / d_part_crc are lists over the flat parts (device pointers as ints, 0 or None = absent),
        part_stride one entry per slice; n_chunks * ceil(nb / L) entries of 16 bytes go to d_map (8-byte aligned device memory).
        Raises ChunkCrcError (.where = chunk, slice, part, block); the map is then still complete."""
        self._slices_dev(self.lib.lzgpu_check_slices_dev, goals, n_chunks, nb, d_parts, part_stride, d_part_crc, stream, d_map)

    SLICES_FIX_DTYPE = SLICES_FIX_DTYPE

    def correct_slices(self, goals, nb, parts, part_crc=None, with_crc=True):
        """Check the given parts of every slice and correct in place each combined stripe that the check blames on one part
        (lzgpu_correct_slices).  goals, parts, part_crc as in check_slices, but every given part must be a writeable C-contiguous uint8
        array: the suspect's blocks are rewritten in it.  Returns (fix, new_crc): fix a structured array [n_chunks, ceil(nb / L)] of
        SLICES_FIX_DTYPE (bad_checks and suspect_part as check_slices had them before the call; status = _lib.FIX_CLEAN / _CORRECTED /
        _UNEXPLAINED / _CRC_CONFLICT / _UNDETERMINED; crc_failed, bit g: a block of flat part g fails its stored CRC; changed, bit s:
        the suspect's block s changed), whether or not an entry is left bad; new_crc[g] a [n_chunks, pb_g] uint32 array per given part
        (None without with_crc) holding the new CRC at every rewritten block and 0 elsewhere.  Raises ChunkCrcError (.where = chunk,
        slice, part, block) on a stored-CRC mismatch, with .fix and .new_crc complete and the corrections the rule allows made."""
        return _correct_slices(self.lib.lzgpu_correct_slices, self.h, goals, nb, parts, part_crc, with_crc)

    def correct_slices_dev(self, goals, n_chunks, nb, d_parts, part_stride, d_part_crc, d_new_crc, d_fix, stream=None):
        """lzgpu_correct_slices_dev: d_parts / d_part_crc / d_new_crc are lists over the flat parts (device pointers as ints, 0 or
        None = absent; d_new_crc may be None), part_stride one entry per slice; n_chunks * ceil(nb / L) entries of 32 bytes go to d_fix
        (8-byte aligned device memory).  Raises ChunkCrcError (.where = chunk, slice, part, block); the entries are then still complete."""
        self._slices_dev(self.lib.lzgpu_correct_slices_dev, goals, n_chunks, nb, d_parts, part_stride, d_part_crc, stream,
                         _dev_ptrs(d_new_crc, _n_flat(goals)), d_fix)

    @staticmethod
    def plan_correct_slices(goals, nb, given):
        """what correct_slices corrects with the given flat parts (pure host logic, csrc/slices_check.h; no GPU needed): the dict of
        plan_check_slices, with correctable and tail_correctable (bit g: flat part g is corrected when named)"""
        out = _lib.LzSlicesCorrectPlan()
        g = np.asarray(given, dtype=np.uint8)
        _check(_lib.load().lzgpu_plan_correct_slices(_goal_array(goals), len(goals), nb, _p(g), C.byref(out)), "plan_correct_slices")
        d = {f: getattr(out.check, f) for f, _ in _lib.LzSlicesCheckPlan._fields_}
        d.update(correctable=out.correctable, tail_correctable=out.tail_correctable)
        return d

    @staticmethod
    def debug_correct_slices_rows(goals, given, valid, part):
        """the left inverse P_g of one stripe shape (csrc/slices_check.h; no GPU needed): (blk_s [n], rows [n, 64]), rows[j, h] the
        coefficient of syndrome S_h in the error of the part's block blk_s[j].  Raises LzGpuError(ERR_ARG) when the part is not
        correctable there."""
        n = C.c_uint32()
        blk_s, rows = np.zeros(64, dtype=np.uint8), np.zeros((64, 64), dtype=np.uint8)
        g = np.asarray(given, dtype=np.uint8)
        _check(_lib.load().lzgpu_debug_correct_slices_rows(_goal_array(goals), len(goals), _p(g), valid, part, C.byref(n), _p(blk_s),
                                                            _p(rows)), "debug_correct_slices_rows")
        return blk_s[:n.value].copy(), rows[:n.value].copy()

    @staticmethod
    def plan_check_slices(goals, nb, given):
        """what check_slices checks with the given flat parts (pure host logic, csrc/slices_check.h; no GPU needed): dict with L,
        tail_blocks, n_checks, tail_n_checks, checked, tail_checked, locatable, tail_locatable (bit g: flat part g), ok and the launch
        geometry G, threads, stages, smem_bytes"""
        out = _lib.LzSlicesCheckPlan()
        g = np.asarray(given, dtype=np.uint8)
        _check(_lib.load().lzgpu_plan_check_slices(_goal_array(goals), len(goals), nb, _p(g), C.byref(out)), "plan_check_slices")
        return {f: getattr(out, f) for f, _ in _lib.LzSlicesCheckPlan._fields_}

    @staticmethod
    def debug_check_slices_rows(goals, given, valid):
        """the checks of one stripe shape (csrc/slices_check.h; no GPU needed): (check_part [n], check_stripe [n], coef [n, 64, 64]),
        coef[h, g, s] the coefficient of block s of flat part g in check h.  Raises LzGpuError(ERR_ARG) with more than 64 checks."""
        n = C.c_uint32()
        part, stripe = np.zeros(64, dtype=np.uint8), np.zeros(64, dtype=np.uint8)
        coef = np.zeros((64, 64, 64), dtype=np.uint8)
        g = np.asarray(given, dtype=np.uint8)
        _check(_lib.load().lzgpu_debug_check_slices_rows(_goal_array(goals), len(goals), _p(g), valid, C.byref(n), _p(part), _p(stripe),
                                                          _p(coef)), "debug_check_slices_rows")
        return part[:n.value].copy(), stripe[:n.value].copy(), coef[:n.value].copy()

    @staticmethod
    def plan_salvage_slices(goals, nb, given):
        """what salvage_slices writes from the given flat parts (pure host logic, csrc/slices_solve.h; no GPU needed): dict with known,
        determined, tail_known, tail_determined (bit q: combined-stripe position q), L, tail_blocks, ok and the launch geometry G,
        threads, stages, smem_bytes"""
        out = _lib.LzSlicesSalvagePlan()
        g = np.asarray(given, dtype=np.uint8)
        _check(_lib.load().lzgpu_plan_salvage_slices(_goal_array(goals), len(goals), nb, _p(g), C.byref(out)), "plan_salvage_slices")
        return {f: getattr(out, f) for f, _ in _lib.LzSlicesSalvagePlan._fields_}

    @staticmethod
    def plan_recover_slices(goals, nb, given):
        """what recover_slices can rebuild from the given flat parts (pure host logic, csrc/slices_solve.h; no GPU needed): dict with
        known, determined, tail_determined (bit q: combined-stripe position q), L, tail_blocks, unknowns, equations, tail_unknowns,
        tail_equations, ok and the launch geometry G, threads, stages, smem_bytes"""
        out = _lib.LzSlicesRecoverPlan()
        g = np.asarray(given, dtype=np.uint8)
        _check(_lib.load().lzgpu_plan_recover_slices(_goal_array(goals), len(goals), nb, _p(g), C.byref(out)), "plan_recover_slices")
        return {f: getattr(out, f) for f, _ in _lib.LzSlicesRecoverPlan._fields_}

    def recover_chunks_dev(self, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, want, d_out, d_chunk_out=None,
                           chunk_out_stride=None, stream=None):
        """Device-pointer degraded read.  With d_part_crc the call waits for its stream and raises ChunkCrcError on a
        mismatch (the library never lets a failed verification pass); without it the call only enqueues."""
        n_parts = goal.k + goal.m
        if d_chunk_out and chunk_out_stride is None:
            raise ValueError("recover_chunks_dev: chunk_out_stride is required with d_chunk_out")
        chunk_out_stride = chunk_out_stride or 0
        w = np.asarray(want, dtype=np.uint8)
        bad = (C.c_int64 * 3)(-1, -1, -1)
        rc = self.lib.lzgpu_recover_chunks_dev(self.h, C.byref(goal.c), n_chunks, nb, _dev_ptrs(d_parts, n_parts), part_stride,
                                               _dev_ptrs(d_part_crc, n_parts), _p(w), _dev_ptrs(d_out, n_parts), d_chunk_out,
                                               chunk_out_stride, bad, stream)
        _check_crc(rc, "recover_chunks_dev", bad)

    def _part_batch_dev(self, fn, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_result, stream):
        # the device-pointer check, map and correction: the same arguments, the result (verdicts, map or fix entries) on the device
        n_parts = goal.k + goal.m
        bad = (C.c_int64 * 3)(-1, -1, -1)
        rc = fn(self.h, C.byref(goal.c), n_chunks, nb, _dev_ptrs(d_parts, n_parts), part_stride, _dev_ptrs(d_part_crc, n_parts), d_result,
                bad, stream)
        _check_crc(rc, _name(fn), bad)

    def _stripe_fix_dev(self, fn, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, stream):
        # the device-pointer repair and decode: the check's arguments without `bad`, as the call only enqueues
        n_parts = goal.k + goal.m
        rc = fn(self.h, C.byref(goal.c), n_chunks, nb, _dev_ptrs(d_parts, n_parts), part_stride, _dev_ptrs(d_part_crc, n_parts), d_fix,
                stream)
        _check(rc, _name(fn))

    # ---- stripe check ------------------------------------------------------------------------
    VERDICT_DTYPE = np.dtype([("first_bad_stripe", np.int32), ("bad_rows", np.uint32), ("suspect_part", np.int32)])

    def check_stripes(self, goal, nb, parts, part_crc=None):
        """Do the parts of every stripe still form a codeword (lzgpu_check_stripes)?  parts: list of k+m arrays [n_chunks, pb*64K];
        every data part is required, None for a parity part = that row is not checked.  part_crc: as in recover_chunks.
        Returns the verdicts, a structured array [n_chunks] of VERDICT_DTYPE (first_bad_stripe, bad_rows, suspect_part; -1 = none),
        whether or not any chunk is inconsistent; raises ChunkCrcError on a stored-CRC mismatch (its .verdict holds the verdicts,
        which are written for every chunk all the same)."""
        return _part_batch(self.lib.lzgpu_check_stripes, self.h, goal, nb, parts, part_crc,
                           lambda n, pb: np.empty(n, dtype=self.VERDICT_DTYPE), "verdict")

    def check_stripes_dev(self, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_verdict, stream=None):
        """Device-pointer stripe check: the verdicts go to d_verdict (n_chunks x 12 bytes, device memory).  With d_part_crc the
        call waits for its stream and raises ChunkCrcError on a mismatch; without it the call only enqueues."""
        self._part_batch_dev(self.lib.lzgpu_check_stripes_dev, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_verdict, stream)

    STRIPE_STATE_DTYPE = np.dtype([("bad_rows", np.uint32), ("suspect_part", np.int32)])

    def check_stripe_map(self, goal, nb, parts, part_crc=None):
        """The state of every stripe of every chunk (lzgpu_check_stripe_map); parts and part_crc as in check_stripes.  Returns a
        structured array [n_chunks, pb] of STRIPE_STATE_DTYPE (bad_rows, 0 = a codeword; suspect_part, -1 = none), whether or not
        any stripe is bad; raises ChunkCrcError on a stored-CRC mismatch (its .map holds the map, written in full all the same).
        For each chunk the lowest bad stripe and its entry equal check_stripes' verdict."""
        return _part_batch(self.lib.lzgpu_check_stripe_map, self.h, goal, nb, parts, part_crc,
                           lambda n, pb: np.empty((n, pb), dtype=self.STRIPE_STATE_DTYPE), "map")

    def check_stripe_map_dev(self, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_map, stream=None):
        """Device-pointer stripe map: n_chunks * pb entries of 8 bytes go to d_map (device memory).  With d_part_crc the call waits
        for its stream and raises ChunkCrcError on a mismatch; without it the call only enqueues."""
        self._part_batch_dev(self.lib.lzgpu_check_stripe_map_dev, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_map, stream)

    STRIPE_FIX_DTYPE = np.dtype([("bad_rows", np.uint32), ("suspect_part", np.int32), ("status", np.int32), ("crc", np.uint32)])

    def correct_stripes(self, goal, nb, parts, part_crc=None):
        """Check every stripe and correct in place each one that names a suspect part (lzgpu_correct_stripes).  parts and part_crc
        as in check_stripe_map, but every given part must be a writeable C-contiguous uint8 array: a corrected block is written
        into it.  part_crc is not changed: the new CRC of a corrected block is in its entry.  Returns a structured array [n_chunks,
        pb] of STRIPE_FIX_DTYPE (bad_rows and suspect_part as the map had them before the call; status = _lib.FIX_*; crc of the
        corrected block), whether or not a stripe is left bad; raises ChunkCrcError on a stored-CRC mismatch (its .fix holds the
        entries, written in full all the same, and the corrections the rule allowed are made)."""
        return _part_batch(self.lib.lzgpu_correct_stripes, self.h, goal, nb, parts, part_crc,
                           lambda n, pb: np.empty((n, pb), dtype=self.STRIPE_FIX_DTYPE), "fix", in_place=True)

    def correct_stripes_dev(self, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, stream=None):
        """Device-pointer stripe correction: the corrected blocks are written into d_parts, n_chunks * pb entries of 16 bytes go to
        d_fix (device memory).  With d_part_crc the call waits for its stream and raises ChunkCrcError on a mismatch; without it
        the call only enqueues."""
        self._part_batch_dev(self.lib.lzgpu_correct_stripes_dev, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, stream)

    def check_stripe_map_degraded(self, goal, nb, parts, part_crc=None):
        """The stripe map of chunks that have lost parts (lzgpu_check_stripe_map_degraded), to take before a lost part is rebuilt.
        parts and part_crc as in check_stripe_map, but any part may be None as long as k + 1 are given: the first k given parts are
        the inputs, the others (parity parts) are checked against their re-encoding from the inputs, and bad_rows bit r is spare part
        k + r.  With every data part given the result is check_stripe_map's."""
        return _part_batch(self.lib.lzgpu_check_stripe_map_degraded, self.h, goal, nb, parts, part_crc,
                           lambda n, pb: np.empty((n, pb), dtype=self.STRIPE_STATE_DTYPE), "map")

    def check_stripe_map_degraded_dev(self, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_map, stream=None):
        """Device-pointer form of check_stripe_map_degraded, as check_stripe_map_dev"""
        self._part_batch_dev(self.lib.lzgpu_check_stripe_map_degraded_dev, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_map,
                             stream)

    def correct_stripes_degraded(self, goal, nb, parts, part_crc=None):
        """correct_stripes on the map of check_stripe_map_degraded (lzgpu_correct_stripes_degraded): every stripe that names a
        suspect has its block rewritten in place from the first k given parts other than it; a missing part is never written"""
        return _part_batch(self.lib.lzgpu_correct_stripes_degraded, self.h, goal, nb, parts, part_crc,
                           lambda n, pb: np.empty((n, pb), dtype=self.STRIPE_FIX_DTYPE), "fix", in_place=True)

    def correct_stripes_degraded_dev(self, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, stream=None):
        """Device-pointer form of correct_stripes_degraded, as correct_stripes_dev"""
        self._part_batch_dev(self.lib.lzgpu_correct_stripes_degraded_dev, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix,
                             stream)

    STRIPE_REPAIR_DTYPE = np.dtype([("bad_rows", np.uint32), ("suspect_part", np.int32), ("status", np.int32), ("crc", np.uint32),
                                    ("crc_failed", np.uint64)])

    def repair_stripes(self, goal, nb, parts, part_crc):
        """correct_stripes_degraded, plus every block that fails its stored CRC rebuilt in place as an erasure (lzgpu_repair_stripes).
        parts as in correct_stripes_degraded; part_crc is required for every given part.  Returns a structured array [n_chunks, pb]
        of STRIPE_REPAIR_DTYPE (crc_failed: bit p = the block of part p failed its stored CRC before the call; status = _lib.FIX_*,
        REBUILT and CRC_ONLY included), whether or not a stripe is left bad; raises ChunkCrcError when a block still fails its stored
        CRC after the call (its .fix holds the entries, and every repair the rule allowed is made)."""
        return _stripe_fix(self.lib.lzgpu_repair_stripes, self.h, goal, nb, parts, part_crc, self.STRIPE_REPAIR_DTYPE)

    def repair_stripes_dev(self, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, stream=None):
        """Device-pointer form of repair_stripes: the rewritten blocks go into d_parts, n_chunks * pb entries of 24 bytes to d_fix
        (device memory, 8-byte aligned).  The call only enqueues, with or without failing CRCs: the entries report them."""
        self._stripe_fix_dev(self.lib.lzgpu_repair_stripes_dev, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, stream)

    STRIPE_DECODE_DTYPE = np.dtype([("bad_rows", np.uint32), ("suspect_part", np.int32), ("status", np.int32), ("crc", np.uint32),
                                    ("crc_failed", np.uint64), ("located", np.uint64), ("located_crc", np.uint32, (2,))])

    def decode_stripes(self, goal, nb, parts, part_crc):
        """repair_stripes, then errors-and-erasures decoding up to the code's radius where the repair gives up (lzgpu_decode_stripes):
        up to two located blocks (valid CRC, wrong bytes) per stripe beside the failing ones.  Arguments as in repair_stripes.
        Returns a structured array [n_chunks, pb] of STRIPE_DECODE_DTYPE (the first five fields as repair_stripes returns them unless
        status == _lib.FIX_DECODED; located: bit p = part p's block was located and rewritten; located_crc: their new CRCs,
        ascending part); raises ChunkCrcError when a block still fails its stored CRC after the call (its .fix holds the entries)."""
        return _stripe_fix(self.lib.lzgpu_decode_stripes, self.h, goal, nb, parts, part_crc, self.STRIPE_DECODE_DTYPE)

    def decode_stripes_dev(self, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, stream=None):
        """Device-pointer form of decode_stripes: the rewritten blocks go into d_parts, n_chunks * pb entries of 40 bytes to d_fix
        (device memory, 8-byte aligned).  The call only enqueues, as repair_stripes_dev."""
        self._stripe_fix_dev(self.lib.lzgpu_decode_stripes_dev, goal, n_chunks, nb, d_parts, part_stride, d_part_crc, d_fix, stream)

    # ---- wire format --------------------------------------------------------------------------
    def write_data_prefixes(self, goal, nb, crc, chunk_ids, write_id_base=0):
        """LIZ_CLTOCS_WRITE_DATA prefixes (cltocs.h:116-137) for every block of every part: uint8 [n, k+m, pb, 38]
        from the CRC array returned by encode_chunks."""
        crc = np.ascontiguousarray(crc, dtype=np.uint32)
        n, stride = crc.shape
        ids = np.ascontiguousarray(chunk_ids, dtype=np.uint64)
        assert ids.size == n
        pb = (nb + goal.k - 1) // goal.k
        out = np.zeros((n, goal.k + goal.m, pb, _lib.WRITE_PREFIX_SIZE), dtype=np.uint8)
        _check(self.lib.lzgpu_write_data_prefixes(self.h, C.byref(goal.c), n, nb, _p(crc), stride, _p(ids), write_id_base, _p(out)),
               "write_data_prefixes")
        return out

    def write_data_prefixes_dev(self, goal, n_chunks, nb, d_crc, crc_stride, d_chunk_ids, d_out, write_id_base=0, stream=None):
        """device-pointer form of write_data_prefixes: crc_stride in uint32 elements, d_out receives n_chunks*(k+m)*pb prefixes"""
        _check(self.lib.lzgpu_write_data_prefixes_dev(self.h, C.byref(goal.c), n_chunks, nb, d_crc, crc_stride, d_chunk_ids, write_id_base,
                                                      d_out, stream), "write_data_prefixes_dev")

    # ---- slice conversion ---------------------------------------------------------------------
    def split_chunks(self, goal, data, nb=None):
        """chunk order [n, nb*64K] -> list of k part-major data parts [n, pb*64K] (BlockConverter,
        src/chunkserver/slice_recovery_planner.h:41-57)."""
        data = _u8(data)
        if data.ndim == 1:
            data = data.reshape(1, -1)
        n, stride = data.shape
        if nb is None:
            nb = stride // BLOCK_SIZE
        pb = (nb + goal.k - 1) // goal.k
        parts = [np.empty((n, pb * BLOCK_SIZE), dtype=np.uint8) for _ in range(goal.k)]
        _check(self.lib.lzgpu_split_chunks(self.h, C.byref(goal.c), n, nb, _p(data), stride, _ptr_array(parts), pb * BLOCK_SIZE), "split_chunks")
        return parts

    def split_chunks_dev(self, goal, n_chunks, nb, d_data, chunk_stride, d_parts, part_stride, stream=None):
        _check(self.lib.lzgpu_split_chunks_dev(self.h, C.byref(goal.c), n_chunks, nb, d_data, chunk_stride, _dev_ptrs(d_parts, goal.k), part_stride,
                                               stream), "split_chunks_dev")

    def plan_encode(self, goal, n_chunks, nb, chunk_stride=None, striped_policy=-1):
        """how encode_chunks_dev would lay the batch out (pure host logic, csrc/fused_plan.h): dict with fused, mode
        (0 per-chunk / 1 flat / 2 striped units), stripes_per_unit, threads_per_cta, units, stage_rows, smem_bytes"""
        out = _lib.LzEncodePlan()
        stride = nb * BLOCK_SIZE if chunk_stride is None else chunk_stride
        _check(self.lib.lzgpu_plan_encode(C.byref(goal.c), n_chunks, nb, stride, striped_policy, C.byref(out)), "plan_encode")
        return {f: getattr(out, f) for f, _ in _lib.LzEncodePlan._fields_}

    # ---- replication / slice-type conversion ----------------------------------------------------
    @staticmethod
    def plan_convert(src, dst, available, want):
        """how convert_chunks would serve the request (pure host logic, csrc/fused_plan.h convert_plan; no GPU needed): dict with
        one_pass (1 = ONE kernel from the source parts to the wanted destination parts), lost_data_parts, stripes_per_unit, ..."""
        out = _lib.LzConvertPlan()
        a = np.asarray(available, dtype=np.uint8)
        w = np.asarray(want, dtype=np.uint8)
        assert a.size == src.k + src.m and w.size == dst.k + dst.m
        _check(_lib.load().lzgpu_plan_convert(C.byref(src.c), C.byref(dst.c), _p(a), _p(w), C.byref(out)), "plan_convert")
        return {f: getattr(out, f) for f, _ in _lib.LzConvertPlan._fields_}

    @staticmethod
    def plan_recover(goal, available, want, verify, image, switches=None):
        """how recover_chunks* would serve the degraded read (pure host logic, csrc/fused_plan.h recover_plan; no GPU needed): dict
        with fused, refusal (_lib.RECOVER_REFUSED_*), kernel (_lib.KERNEL_RECOVER_*), lost_data_parts, kt (compile-time k, 0 =
        runtime), rows, item_bytes, solve, doublings, G, stages, threads, gf_warps, smem_bytes.  switches: a dict of
        lzgpu_recover_switches fields that differ from the build's defaults (_lib.RECOVER_SWITCHES_DEFAULT), None = the defaults."""
        out = _lib.LzRecoverPlan()
        a = np.asarray(available, dtype=np.uint8)
        w = np.asarray(want, dtype=np.uint8)
        assert a.size == goal.k + goal.m and w.size == goal.k + goal.m
        sw = None
        if switches is not None:
            unknown = set(switches) - set(_lib.RECOVER_SWITCHES_DEFAULT)
            assert not unknown, unknown
            sw = C.byref(_lib.LzRecoverSwitches(**{**_lib.RECOVER_SWITCHES_DEFAULT, **switches}))
        rc = _lib.load().lzgpu_plan_recover(C.byref(goal.c), _p(a), _p(w), int(bool(verify)), int(bool(image)), sw, C.byref(out))
        if rc != _lib.ERR_TOO_FEW_PARTS:
            _check(rc, "plan_recover")
        return {f: getattr(out, f) for f, _ in _lib.LzRecoverPlan._fields_}

    @staticmethod
    def plan_check(goal, given):
        """how check_stripes / check_stripe_map / correct_stripes would check the batch (pure host logic, csrc/fused_plan.h
        check_plan; no GPU needed): dict with fused (0 = the generic route), rows (checked parity rows), consecutive (rows 0 .. R-1),
        G, stages, threads, item_passes, smem_bytes.  given: k+m flags, part i given; a missing data part or no parity part raises
        LzGpuError (ERR_TOO_FEW_PARTS), as the calls do."""
        out = _lib.LzCheckPlan()
        g = np.asarray(given, dtype=np.uint8)
        assert g.size == goal.k + goal.m
        _check(_lib.load().lzgpu_plan_check(C.byref(goal.c), _p(g), C.byref(out)), "plan_check")
        return {f: getattr(out, f) for f, _ in _lib.LzCheckPlan._fields_}

    @staticmethod
    def plan_check_degraded(goal, given):
        """how check_stripe_map_degraded / correct_stripes_degraded would check the batch (lzgpu_plan_check_degraded): the dict of
        plan_check; any part may be missing, fewer than k + 1 given parts raise LzGpuError (ERR_TOO_FEW_PARTS), as the calls do"""
        out = _lib.LzCheckPlan()
        g = np.asarray(given, dtype=np.uint8)
        assert g.size == goal.k + goal.m
        _check(_lib.load().lzgpu_plan_check_degraded(C.byref(goal.c), _p(g), C.byref(out)), "plan_check_degraded")
        return {f: getattr(out, f) for f, _ in _lib.LzCheckPlan._fields_}

    def convert_chunks(self, src, dst, nb, parts, want, part_crc=None, with_crc=True):
        """Rebuild the `want`ed parts of slice type `dst` from the available `parts` of slice type `src`
        (SliceRecoveryPlanner, slice_recovery_planner.h:87-204).  parts[i]: (n_chunks, pb_src*65536) uint8 or None.
        Returns (out, out_crc): lists indexed by destination part (None where not wanted)."""
        return _convert_chunks(self.lib.lzgpu_convert_chunks, self.h, src, dst, nb, parts, want, part_crc, with_crc)

    def convert_chunks_dev(self, src, dst, n_chunks, nb, d_parts, part_stride, want, d_out, out_stride, d_part_crc=None, d_out_crc=None, stream=None):
        ns, nd = src.k + src.m, dst.k + dst.m
        w = np.asarray(want, dtype=np.uint8)
        bad = (C.c_int64 * 3)(-1, -1, -1)
        rc = self.lib.lzgpu_convert_chunks_dev(self.h, C.byref(src.c), C.byref(dst.c), n_chunks, nb, _dev_ptrs(d_parts, ns), part_stride,
                                               _dev_ptrs(d_part_crc, ns), _p(w), _dev_ptrs(d_out, nd), out_stride, _dev_ptrs(d_out_crc, nd),
                                               bad, stream)
        _check_crc(rc, "convert_chunks_dev", bad)

    # ---- CRC ---------------------------------------------------------------------------------
    def crc_blocks(self, data, block_len=BLOCK_SIZE, block_stride=None):
        data = _u8(data).reshape(-1)
        if block_stride is None:
            block_stride = block_len
        n = (data.size - block_len) // block_stride + 1 if data.size >= block_len else 0
        out = np.zeros(n, dtype=np.uint32)
        _check(self.lib.lzgpu_crc_blocks(self.h, _p(data), n, block_len, block_stride, _p(out)), "crc_blocks")
        return out

    def crc_blocks_dev(self, d_data, n_blocks, d_out, block_len=BLOCK_SIZE, block_stride=BLOCK_SIZE, stream=None):
        _check(self.lib.lzgpu_crc_blocks_dev(self.h, d_data, n_blocks, block_len, block_stride, d_out, stream), "crc_blocks_dev")

    def verify_blocks(self, data, stored_crc, block_len=BLOCK_SIZE, sparse_rule=False):
        _verify_blocks(self.lib.lzgpu_verify_blocks, self.h, data, stored_crc, block_len, sparse_rule)

    def verify_interleaved(self, records):
        """records: on-disk layout, n x (4-byte big-endian CRC + 65536 data bytes) (chunk.h:40)."""
        _verify_interleaved(self.lib.lzgpu_verify_interleaved, self.h, records)

    def verify_interleaved_ptr(self, ptr, n_blocks):
        """same, `ptr` = raw address of the records: host memory or a device buffer of this engine's device"""
        bad = C.c_int64(-1)
        rc = self.lib.lzgpu_verify_interleaved(self.h, ptr, n_blocks, C.byref(bad))
        _check_crc(rc, "verify_interleaved", (bad.value,))

    def moosefs_header_size(self, data_parts=1):
        return int(self.lib.lzgpu_moosefs_header_size(data_parts))

    def verify_moosefs(self, file_image, n_blocks, data_parts=1):
        """file_image: MooseFS-format chunk file (chunk.cc:126-190): signature, big-endian CRC table at 1024, data after the header."""
        img = _u8(file_image).reshape(-1)
        bad = C.c_int64(-1)
        rc = self.lib.lzgpu_verify_moosefs(self.h, data_parts, _p(img), n_blocks, C.byref(bad))
        _check_crc(rc, "verify_moosefs", (bad.value,))

    # ---- chunkserver block writes ----------------------------------------------------------------
    def write_blocks(self, blocks, stored_crc, writes, sparse_rule=True):
        """Batched hdd_write (hddspacemgr.cc:1898-2008).  blocks: uint8 [n, 65536], stored_crc: uint32 [n], both updated in place.
        writes: list of dicts {block, offset, data (uint8 array), crc, exists (default True)}.  Returns the list of per-request
        status codes (0, ERR_CRC = corrupt packet, ERR_DAMAGED = the stored block fails its CRC, ERR_ARG = bad range)."""
        assert blocks.dtype == np.uint8 and blocks.flags.c_contiguous and stored_crc.dtype == np.uint32 and stored_crc.flags.c_contiguous
        n = len(writes)
        arr = (_lib.LzBlockWrite * max(n, 1))()
        payload = np.concatenate([_u8(w["data"]).reshape(-1) for w in writes]) if n else np.zeros(0, dtype=np.uint8)
        pos = 0
        for i, w in enumerate(writes):
            size = int(np.asarray(w["data"]).size)
            arr[i].block, arr[i].offset, arr[i].size, arr[i].crc = int(w["block"]), int(w["offset"]), size, int(w["crc"])
            arr[i].payload_off, arr[i].exists, arr[i].status = pos, int(w.get("exists", True)), 0
            pos += size
        payload = np.ascontiguousarray(payload)
        rc = self.lib.lzgpu_write_blocks(self.h, _p(blocks), _p(stored_crc), blocks.size // BLOCK_SIZE, _p(payload) if payload.size else None,
                                         payload.size, arr, n, int(sparse_rule))
        if rc not in (_lib.OK, _lib.ERR_CRC, _lib.ERR_DAMAGED, _lib.ERR_ARG) or (rc == _lib.ERR_ARG and all(arr[i].status == 0 for i in range(n))):
            _check(rc, "write_blocks")
        return [arr[i].status for i in range(n)]

    def write_blocks_dev(self, d_blocks, d_stored_crc, d_payload, d_writes, n_writes, sparse_rule=True, stream=None):
        """device-pointer form of write_blocks: d_writes holds n_writes lzgpu_block_write records (_lib.LzBlockWrite) whose status
        fields the kernel fills in; asynchronous, the per-request statuses are valid once the stream has passed the call"""
        _check(self.lib.lzgpu_write_blocks_dev(self.h, d_blocks, d_stored_crc, d_payload, d_writes, n_writes, int(sparse_rule), stream),
               "write_blocks_dev")

    # ---- device helpers ----------------------------------------------------------------------
    def fill_chunks_dev(self, d_data, n_chunks, chunk_len, chunk_stride, seed, first_chunk=0, stream=None):
        _check(self.lib.lzgpu_fill_chunks_dev(self.h, d_data, n_chunks, chunk_len, chunk_stride, seed, first_chunk, stream), "fill_chunks_dev")

    def dev_alloc(self, nbytes):
        p = C.c_void_p()
        _check(self.lib.lzgpu_dev_alloc(self.h, nbytes, C.byref(p)), "dev_alloc")
        return p.value

    def dev_free(self, ptr):
        _check(self.lib.lzgpu_dev_free(self.h, ptr), "dev_free")

    def upload(self, d_dst, arr):
        arr = np.ascontiguousarray(arr)
        _check(self.lib.lzgpu_dev_upload(self.h, d_dst, _p(arr), arr.nbytes), "dev_upload")

    def download(self, d_src, nbytes, dtype=np.uint8):
        out = np.empty(nbytes // np.dtype(dtype).itemsize, dtype=dtype)
        _check(self.lib.lzgpu_dev_download(self.h, _p(out), d_src, nbytes), "dev_download")
        return out
