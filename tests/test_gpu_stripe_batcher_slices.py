"""lzgpu::StripeBatcher over goals of several slices (include/lzgpu_stripe_batcher.hpp): the mount write path batched by combined
stripe, every block the sink receives checked against the reference's contract and the CPU oracle inside the C++ test
(tests/cpp/test_stripe_batcher_slices.cc).  The GPU build also checks that a fused flush is one launch of the one-pass kernel at the
geometry of the packed pseudo-chunks; the CPU build runs the same host logic against tests/cpp/oracle_backend.cc."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "cpp", "build")
GPU_BIN = os.path.join(BUILD, "test_stripe_batcher_slices")
CPU_BIN = os.path.join(BUILD, "test_stripe_batcher_slices_cpu")


def _built(exe):
    if not os.path.exists(exe):
        subprocess.run(["make", "-s", "-C", os.path.join(ROOT, "tests", "cpp"), "-f", "slices.mk"], check=True)
    assert os.path.exists(exe), f"{os.path.basename(exe)} was not built"
    return exe


def _run(exe):
    r = subprocess.run([_built(exe)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "all tests passed" in r.stdout


def test_gpu_binary_links_the_library():
    out = subprocess.run(["ldd", _built(GPU_BIN)], capture_output=True, text=True).stdout
    assert "liblzgpu.so" in out and "liboracle.so" in out and "not found" not in out


def test_stripe_batcher_slices_host_logic_on_cpu():
    _run(CPU_BIN)


@pytest.mark.gpu
def test_stripe_batcher_slices_cpp():
    _run(GPU_BIN)
