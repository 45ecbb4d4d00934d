"""Exact comparison helpers shared by the reference modules of the bank tests (tests/ddc_ref.py, tests/fir_ref.py)."""
import numpy as np

U = 2.0 ** -24                                                       # unit roundoff of binary32
SENTINEL = np.uint32(0x7FC0DEAD)                                     # a NaN the kernels never produce: padding must keep it


def bits(a):
    """the bit patterns of a float32 / complex64 array (NaN-safe exact comparison)"""
    a = np.ascontiguousarray(a)
    return a.view(np.uint32) if a.dtype in (np.float32, np.complex64) else a


def assert_bits_equal(a, b, what):
    a, b = bits(a), bits(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    if not np.array_equal(a, b):
        bad = np.argwhere(a != b)
        raise AssertionError(f"{what}: {len(bad)} of {a.size} words differ, first at {tuple(bad[0])}")
