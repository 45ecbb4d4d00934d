"""ctypes front-end of tone_oracle.c (the CPU restatement of apply_fir_cc and bfsk_demod_cf), bindings to the same functions and to
firdes_add_peak_c of the compiled reference (oracle/_ref/libcsdr_ref.so), the per-output bound between bfsk_demod_cf summed in two orders,
and a seeded RTTY FSK signal.  TEST INFRASTRUCTURE: the C file is compiled once per process into a temporary directory."""
from __future__ import annotations

import ctypes as C
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF_SO = ROOT / "oracle" / "_ref" / "libcsdr_ref.so"
sys.path.insert(0, str(ROOT / "tests" / "rtty"))

HAMMING = 2
_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        out = Path(tempfile.mkdtemp(prefix="tone_oracle_")) / "libtone_oracle.so"
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(out),
                        str(HERE / "tone_oracle.c"), "-lm"], check=True)
        L = C.CDLL(str(out))
        vp, it = C.c_void_p, C.c_int
        L.tone_oracle_apply_fir_cc.argtypes = [vp, vp, it, vp, it]
        L.tone_oracle_bfsk_demod_cf.argtypes = [vp, vp, it, vp, vp, it]
        _lib = L
    return _lib


def _c(x):
    return np.ascontiguousarray(x, np.complex64)


def apply_fir_cc(x, taps):
    x, taps = _c(x), _c(taps)
    out = np.zeros(max(x.size - taps.size + 1, 1), np.complex64)
    m = lib().tone_oracle_apply_fir_cc(x.ctypes.data, out.ctypes.data, x.size, taps.ctypes.data, taps.size)
    return out[:m]


def bfsk_demod_cf(x, mark, space):
    x, mark, space = _c(x), _c(mark), _c(space)
    out = np.zeros(max(x.size - mark.size + 1, 1), np.float32)
    m = lib().tone_oracle_bfsk_demod_cf(x.ctypes.data, out.ctypes.data, x.size, mark.ctypes.data, space.ctypes.data, mark.size)
    return out[:m]


# ---- the compiled reference ---------------------------------------------------------------------------------------------------------
def have_ref() -> bool:
    return REF_SO.exists()


def ref():
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_SO))
        vp, it = C.c_void_p, C.c_int
        L.firdes_add_peak_c.argtypes = [vp, it, C.c_float, it, it, it]
        L.apply_fir_cc.argtypes = [vp, vp, it, vp, it]; L.apply_fir_cc.restype = it
        L.bfsk_demod_cf.argtypes = [vp, vp, it, vp, vp, it]; L.bfsk_demod_cf.restype = it
        _ref = L
    return _ref


def ref_peak(rate, length, window=HAMMING, into=None, add=0, normalize=1):
    t = np.zeros(max(length, 1), np.complex64) if into is None else into
    ref().firdes_add_peak_c(t.ctypes.data, length, rate, window, add, normalize)
    return t[:length]


def ref_apply_fir_cc(x, taps):
    x, taps = _c(x), _c(taps)
    out = np.zeros(max(x.size - taps.size + 1, 1), np.complex64)
    m = ref().apply_fir_cc(x.ctypes.data, out.ctypes.data, x.size, taps.ctypes.data, taps.size)
    return out[:m]


def ref_bfsk_demod_cf(x, mark, space):
    x, mark, space = _c(x), _c(mark), _c(space)
    out = np.zeros(max(x.size - mark.size + 1, 1), np.float32)
    m = ref().bfsk_demod_cf(x.ctypes.data, out.ctypes.data, x.size, mark.ctypes.data, space.ctypes.data, mark.size)
    return out[:max(m, 0)]


def bfsk_taps(spacing, length, peak=None):
    """the taps `csdr bfsk_demod_cf spacing length` designs (csdr.c:3283-3286): Hamming peaks at +spacing/2 (mark) and -spacing/2 (space)"""
    peak = peak or ref_peak
    half = np.float32(np.float32(spacing) / np.float32(2))
    return peak(float(half), length), peak(float(-half), length)


# ---- the bound between two summation orders of bfsk_demod_cf ---------------------------------------------------------------------
U = 2.0 ** -24


def gamma(k):
    return k * U / (1 - k * U)


def bfsk_bound(x, mark, space):
    """per output, the most two float evaluations of bfsk_demod_cf that differ only in the order of the `ti` sums can differ by.
    Each accumulator (mark or space, real or imaginary part) is a sum of 2L rounded products, so in any order it lies within
    d = gamma(2L) * P of its exact value a, P being the sum of the products' magnitudes (Higham, Accuracy and Stability, 3.1).  Then
    |a'^2 - a^2| <= d (2|a| + d), and the squares, their sums and the final difference add rounding errors of at most gamma(3) times
    sum (|a| + d)^2.  Each evaluation is within E = sum d (2|a| + d) + gamma(3) sum (|a| + d)^2 of the exact value; two within 2E of each
    other.  a and P are computed in float64 (their own error, below 2^-40 of P, is covered by a factor 1.001), plus an absolute
    8L * 2^-149 for products that underflow."""
    x = np.asarray(x, np.complex128)
    L = len(mark)
    g = gamma(2 * L) * 1.001
    e = np.zeros(x.size - L + 1)
    for t in (np.asarray(mark, np.complex128), np.asarray(space, np.complex128)):
        a = np.correlate(x, np.conj(t), "valid")
        p_re = np.correlate(np.abs(x.real), np.abs(t.real), "valid") + np.correlate(np.abs(x.imag), np.abs(t.imag), "valid")
        p_im = np.correlate(np.abs(x.real), np.abs(t.imag), "valid") + np.correlate(np.abs(x.imag), np.abs(t.real), "valid")
        for v, p in ((np.abs(a.real), p_re), (np.abs(a.imag), p_im)):
            d = g * p
            e += d * (2 * v + d) + gamma(3) * (v + d) ** 2
    return 2 * e + 8 * L * 2.0 ** -149


# ---- a seeded RTTY FSK signal ------------------------------------------------------------------------------------------------------
def rtty_signal(text, spb, rng, freq=0.0, noise=0.01, **kw):
    """rtty.modulate: ITA2 at spb samples per bit, 170 Hz shift at 45.45 Bd, continuous phase, complex Gaussian noise"""
    import rtty
    return rtty.modulate(text, spb, rng, freq=freq, noise=noise, **kw)
