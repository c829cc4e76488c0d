"""lzgpu_repair_stripes without a GPU: the host build of the per-stripe row derivation the repair kernel runs (csrc/repair_rows.h)
against lzgpu_rs_recovery_matrix for every given set and every set F of failing blocks the rule rebuilds, and the layout of
lzgpu_stripe_repair against the header."""
import ctypes as C
import itertools
import os
import subprocess

import numpy as np
import pytest

from lizardfs_b200 import _lib
from lizardfs_b200.engine import Engine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _device_rows(lib, k, m, inputs, wanted):
    ins = np.array(inputs, dtype=np.uint8)
    w = np.array(wanted, dtype=np.uint8)
    rows = np.zeros((len(wanted), k), dtype=np.uint8)
    rc = lib.lzgpu_debug_repair_rows(k, m, _p(ins), _p(w), len(wanted), _p(rows))
    return rc, rows


def _host_rows(lib, k, m, inputs, wanted):
    erased = np.ones(k + m, dtype=np.uint8)
    erased[list(inputs)] = 0
    want = np.zeros(k + m, dtype=np.uint8)
    want[list(wanted)] = 1
    rows = np.zeros((m, k), dtype=np.uint8)
    rc = lib.lzgpu_rs_recovery_matrix(k, m, _p(erased), _p(want), _p(rows))
    return rc, rows[:max(rc, 0)]


# xor3, ec(3,2), ec(5,3), ec(8,4) (Vandermonde) and ec(4,5) (Cauchy: m >= 5)
@pytest.mark.parametrize("k,m", [(3, 1), (3, 2), (5, 3), (8, 4), (4, 5)])
def test_rows_equal_the_recovery_matrix_for_every_pattern(k, m):
    """Every given set of at least k + 1 parts and every F the rule rebuilds (1 <= |F| <= given - k): the inputs are the first k
    given parts outside F; the rows of F over them must be lzgpu_rs_recovery_matrix's, byte for byte (or both singular)."""
    lib = _lib.load()
    n = k + m
    seen = set()
    for size in range(k + 1, n + 1):
        for given in itertools.combinations(range(n), size):
            for nf in range(1, size - k + 1):
                for f in itertools.combinations(given, nf):
                    inputs = tuple(p for p in given if p not in f)[:k]
                    if (inputs, f) in seen:
                        continue
                    seen.add((inputs, f))
                    rc_d, rows_d = _device_rows(lib, k, m, inputs, f)
                    rc_h, rows_h = _host_rows(lib, k, m, inputs, f)
                    if rc_h < 0:
                        assert rc_d == _lib.ERR_ARG, (inputs, f)
                        continue
                    assert rc_d == rc_h == nf, (inputs, f)
                    assert (rows_d == rows_h).all(), (inputs, f, rows_d, rows_h)
    assert seen


def test_rows_refuse_bad_arguments():
    lib = _lib.load()
    assert _device_rows(lib, 3, 2, (0, 1, 2), (0,))[0] == _lib.ERR_ARG       # a wanted part is an input
    assert _device_rows(lib, 3, 2, (1, 0, 2), (3,))[0] == _lib.ERR_ARG       # inputs not ascending
    assert _device_rows(lib, 3, 2, (0, 1, 2), (5,))[0] == _lib.ERR_ARG       # no such part
    assert _device_rows(lib, 3, 2, (0, 1, 2), (3, 4, 3))[0] == _lib.ERR_ARG  # more wanted than m


def test_stripe_repair_layout_matches_the_header(tmp_path):
    fields = [f for f, _ in _lib.LzStripeRepair._fields_]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(['#include <stdio.h>', '#include <stddef.h>', '#include "lzgpu.h"', 'int main(void) {',
                              'printf("%zu %zu", sizeof(lzgpu_stripe_repair), _Alignof(lzgpu_stripe_repair));'] +
                             [f'printf(" %zu", offsetof(lzgpu_stripe_repair, {f}));' for f in fields] +
                             ['printf(" %d %d\\n", LZGPU_FIX_REBUILT, LZGPU_FIX_CRC_ONLY);', 'return 0; }']))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    size, align, *rest = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    offsets, consts = rest[:len(fields)], rest[len(fields):]
    assert size == 24 == C.sizeof(_lib.LzStripeRepair) == Engine.STRIPE_REPAIR_DTYPE.itemsize
    assert align == 8
    assert offsets == [getattr(_lib.LzStripeRepair, f).offset for f in fields]
    assert offsets == [Engine.STRIPE_REPAIR_DTYPE.fields[f][1] for f in fields]
    assert consts == [_lib.FIX_REBUILT, _lib.FIX_CRC_ONLY]
