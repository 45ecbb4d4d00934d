"""CPU tier: the FFT twiddle tables belong to one device.  fft.cu runs under the emulator with two pretend devices (CUDA_EMUL_DEVICES=2): the
row-FFT table and the r2c split table of one size are separate allocations on device 0 and device 1, the same allocation again on a repeat call
on one device, and hold the same values on both.  (A table shared by the whole process would hand device 1 a pointer into device 0's memory.)"""
import ctypes as C
import os
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "host_shim"))
import emul_build  # noqa: E402

SET_DEVICE = 'extern "C" int emul_set_device(int d) { return (int)cudaSetDevice(d); }\n'


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    old = os.environ.get("CUDA_EMUL_DEVICES")
    os.environ["CUDA_EMUL_DEVICES"] = "2"
    try:
        L, _ = emul_build.build_file(tmp_path_factory.mktemp("emul_fft_tables"), "fft.cu", extra=SET_DEVICE)
        L.emul_set_device.argtypes = [C.c_int]
        yield L
        L.emul_set_device(0)
    finally:
        if old is None:
            del os.environ["CUDA_EMUL_DEVICES"]
        else:
            os.environ["CUDA_EMUL_DEVICES"] = old


def table(lib, fn, n, device):
    assert lib.emul_set_device(device) == 0
    p = C.c_void_p()
    assert fn(n, C.byref(p)) == 0, lib.emul_last_error()
    return p.value


def check_per_device(lib, fn, n, entries):
    p0, p1 = table(lib, fn, n, 0), table(lib, fn, n, 1)
    assert p0 and p1 and p0 != p1, "one table serves both devices"
    assert table(lib, fn, n, 1) == p1 and table(lib, fn, n, 0) == p0, "a repeat call on one device made a new table"
    v0, v1 = ((C.c_uint32 * (2 * entries)).from_address(p) for p in (p0, p1))
    assert np.array_equal(np.frombuffer(v0, np.uint32), np.frombuffer(v1, np.uint32))


@pytest.mark.parametrize("n", [16, 32, 4096])
def test_row_fft_table_is_per_device(lib, n):
    """radix-8 planes (3n entries) below 32 points, radix-16 planes (4n) from 32 on"""
    check_per_device(lib, lib.emul_row_fft_twiddles, n, (4 if n >= 32 else 3) * n)


@pytest.mark.parametrize("m", [2, 1024])
def test_rfft_split_table_is_per_device(lib, m):
    check_per_device(lib, lib.emul_get_rfft_twiddles, m, m // 2 + 1)
