"""CPU tier: the SHIPPED device function csdrb::wrap_phase_pm_pi (csdr_b200/csrc/common.cuh) compiled for the host (tests/host_shim/
wrap_host.cpp maps the CUDA intrinsics onto the same IEEE single-precision operations) and compared bit for bit with the reference's
`while (ph > PI) ph -= 2*PI; while (ph < -PI) ph += 2*PI;` loop (libcsdr_gpl.c:49-50) across every binade it has a special case for."""
import ctypes as C
import shutil
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
CUDA_INC = Path("/usr/local/cuda/include")


@pytest.fixture(scope="module")
def wrap(tmp_path_factory):
    if not shutil.which("g++") or not (CUDA_INC / "cuda_runtime.h").exists():
        pytest.skip("needs g++ and the CUDA headers")
    so = tmp_path_factory.mktemp("wrap") / "wrap_host.so"
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", f"-I{CUDA_INC}",
                    str(ROOT / "tests" / "host_shim" / "wrap_host.cpp"), "-o", str(so)], check=True, capture_output=True)
    L = C.CDLL(str(so))
    L.wrap_compare.argtypes = [C.c_void_p, C.c_long, C.POINTER(C.c_float)]; L.wrap_compare.restype = C.c_long
    L.wrap_fast.argtypes = [C.c_float]; L.wrap_fast.restype = C.c_float
    L.wrap_loop.argtypes = [C.c_float]; L.wrap_loop.restype = C.c_float
    return L


def test_fast_forward_equals_the_loop_in_every_binade(wrap):
    rng = np.random.default_rng(0)
    total = 0
    for E in range(-4, 26):
        lo, hi = np.float32(2.0 ** E), np.float32(2.0 ** (E + 1))
        count = int(min(20_000, max(24, 3e7 / 2.0 ** E)))              # the loop costs |ph|/2pi iterations per value
        x = rng.uniform(lo, hi, count).astype(np.float32)
        edge = np.array([lo, np.nextafter(lo, np.float32(0)), np.nextafter(hi, np.float32(0)), np.nextafter(lo, hi)], np.float32)
        x = np.concatenate([x, -x, edge, -edge]).astype(np.float32)
        bad = C.c_float(0)
        assert wrap.wrap_compare(x.ctypes.data, x.size, C.byref(bad)) == 0, (E, bad.value)
        total += x.size
    assert total > 300_000


def test_phase_sums_of_real_streams(wrap):
    """the values the kernels actually wrap: phase + rate*PI*n for CLI chunk sizes, both signs"""
    rng = np.random.default_rng(1)
    PI = np.float32(3.14159265358979323846)
    rates = rng.uniform(-1.0, 1.0, 4000).astype(np.float32)
    ph = rng.uniform(-3.2, 3.2, 4000).astype(np.float32)
    for n in (1, 37, 1000, 1024, 4096, 16384, 262144):
        x = (ph + (rates * PI) * np.float32(n)).astype(np.float32)
        bad = C.c_float(0)
        assert wrap.wrap_compare(x.ctypes.data, x.size, C.byref(bad)) == 0, (n, bad.value)


def test_special_values(wrap):
    for v in (0.0, -0.0, 3.1415927, 3.1415929, -3.1415927, -3.1415929, float("inf"), float("-inf"), 6.7e7, -6.7e7, 2.0 ** 26, 1e30, -1e30):
        a, b = np.float32(wrap.wrap_fast(v)), np.float32(wrap.wrap_loop(v))
        assert a.view(np.uint32) == b.view(np.uint32), (v, a, b)
    assert np.isnan(wrap.wrap_fast(float("nan")))


def test_wraps_landing_on_zero(wrap):
    """a phase the loop wraps exactly onto zero ends at +0 from either side (fl(-2 pi + 2 pi) = +0), as the reference's loop leaves it; only
    an input of -0.0, which no step touches, stays -0.0"""
    two_pi = np.float32(2) * np.float32(3.14159265358979323846)
    x = (two_pi * np.arange(1, 2000, dtype=np.float32)).astype(np.float32)
    x = np.concatenate([x, -x]).astype(np.float32)
    zeros = [v for v in x if wrap.wrap_loop(float(v)) == 0]
    assert any(v < 0 for v in zeros) and any(v > 0 for v in zeros), zeros
    bad = C.c_float(0)
    assert wrap.wrap_compare(x.ctypes.data, x.size, C.byref(bad)) == 0, bad.value
