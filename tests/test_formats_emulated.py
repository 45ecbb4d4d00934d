"""CPU tier for the sample-format conversions (csdr_b200/csrc/elementwise.cu) through the C ABI of the whole emulated library: convert_s8_f,
convert_f_s8, convert_f_u8, convert_s24_f and convert_f_s24 bit for bit against the restatements of tests/formats/formats.py and the compiled
reference (all 256 s8 codes, an edge-heavy subset of the s24 codes in both byte orders, +-0, subnormals, every truncation boundary, the wrap
region, |s| at 2^31, +-Inf and NaN; lengths 1..40 at odd offsets); the refusals; the libcsdr drop-ins on unaligned host buffers."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "formats"))
import emul_build  # noqa: E402
import formats as M  # noqa: E402

needs_ref = pytest.mark.skipif(not M.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built")
CASES = [(k, be) for k in M.KINDS for be in ((0, 1) if M.KINDS[k][2] else (0,))]


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    return M.EmulDev(C.CDLL(str(lib)))


def test_the_build_constants():
    """the reciprocals the build multiplies by, and that multiplying is not dividing for s8"""
    assert M.S8_RECIP == np.float32(1) / np.float32(127) and M.S24_RECIP == np.float32(1) / np.float32(2147483392.0)
    assert np.float32(2 ** 31 - 1 - 256) == np.float32(2147483392.0)
    b = np.arange(-128, 128).astype(np.float32)
    assert np.any((b / np.float32(127)).astype(np.float32) != (b * M.S8_RECIP).astype(np.float32))


@pytest.mark.parametrize("kind,bigendian", CASES)
def test_restatement(dev, kind, bigendian):
    x = M.inputs(kind, np.random.default_rng(1))
    M.check_against(dev, kind, x, bigendian, with_ref=M.have_ref())


@needs_ref
@pytest.mark.parametrize("kind,bigendian", CASES)
def test_lengths_and_offsets_against_the_build(dev, kind, bigendian):
    rng = np.random.default_rng(2)
    x = M.inputs(kind, rng)
    item = M.KINDS[kind][0]
    if item == 4:                                                     # specials first, then straddled boundaries, shuffled into 40 values
        x = np.concatenate([x[:20], rng.permutation(x)[:20]])
    else:
        x = rng.permutation(x.reshape(-1, item))[:40].reshape(-1)
    M.check_lengths_and_offsets(dev, kind, x, bigendian)


def test_round_trips(dev):
    """convert_f_s24 | convert_s24_f and convert_f_s8 | convert_s8_f in either byte order give the restatement's values"""
    x = np.random.default_rng(3).uniform(-1, 1, 1001).astype(np.float32)
    for be in (0, 1):
        b = M.run(dev, "f_s24", x, be)
        y = M.run(dev, "s24_f", b, be).view(np.float32)
        assert M.same(y, M.s24_f(M.f_s24(x, be), be)) and np.abs(y - x).max() < 2.0 ** -22
        assert not M.same(M.run(dev, "s24_f", b, 1 - be), y)              # the other order reads other values
    y = M.run(dev, "s8_f", M.run(dev, "f_s8", x)).view(np.float32)
    assert M.same(y, M.s8_f(M.f_s8(x))) and np.abs(y - x).max() < 1 / 127


def test_refusals_launch_nothing(dev):
    assert M.refusals(dev) == []


@needs_ref
def test_dropins_on_unaligned_host_buffers(dev):
    L = dev.L
    rng = np.random.default_rng(4)
    for kind, be in CASES:
        i, o, takes_be = M.KINDS[kind]
        x = np.ascontiguousarray(M.inputs(kind, rng)).view(np.uint8).reshape(-1)
        for n in (0, 1, 7, min(1000, x.size // i)):
            src = np.zeros(n * i + 1, np.uint8)[1:]; src[:] = x[:n * i]          # odd addresses on both sides
            dst = np.full(n * o + 2, M.SENTINEL, np.uint8)
            f = getattr(L, "convert_" + kind)
            args = (src.ctypes.data, dst.ctypes.data + 1, n) + ((be,) if takes_be else ())
            f(*args)
            assert dst[0] == M.SENTINEL and dst[-1] == M.SENTINEL, (kind, n)
            part = src.view(np.float32) if i == 4 else src
            assert M.same(dst[1:-1], np.asarray(M.ref_call(kind, part, be)).view(np.uint8)), (kind, be, n)
