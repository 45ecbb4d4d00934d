"""The checker side of the transmit blocks: fir_interpolate_cc restated in numpy in the kernel's summation order (tap order, every product and sum
rounded to float, no FMA), the float64 per-output bound between two summation orders of it, the fmmod_fc phase chain of the reference build
(its disassembly: the wrap loops test the value before the step against fl(3*PI)), and bindings to the compiled reference
(oracle/_ref/libcsdr_ref.so).  TEST INFRASTRUCTURE."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
REF_SO = ROOT / "oracle" / "_ref" / "libcsdr_ref.so"
U = 2.0 ** -24
_ref = None


def groups(n, I, T):
    return max(n - (T - 1 + I - 1) // I, 0)


def fir_interpolate_cc(x, I, taps):
    """the kernel's order: output i*I + ip = sum over si, ascending, of x[i+si] * taps[(I-ip) + si*I] while that index is below T"""
    x = np.asarray(x, np.complex64)
    taps = np.asarray(taps, np.float32)
    T = taps.size
    G = groups(x.size, I, T)
    xr, xq = x.real.astype(np.float32), x.imag.astype(np.float32)
    out = np.zeros((G, I), np.complex64)
    for ip in range(I):
        ai = np.zeros(G, np.float32); aq = np.zeros(G, np.float32)
        si = 0
        for ti in range(I - ip, T, I):
            t = taps[ti]
            ai = (ai + xr[si:si + G] * t).astype(np.float32)
            aq = (aq + xq[si:si + G] * t).astype(np.float32)
            si += 1
        out[:, ip] = ai + 1j * aq
    return out.reshape(-1)


def interp_bound(x, I, taps):
    """per output and component, how far two float evaluations of the same sum in different orders can lie apart: each is within
    gamma(k) * sum |x t| of the exact sum, k the number of terms (Higham, Accuracy and Stability, 3.1), plus k * 2^-149 for underflow"""
    x = np.asarray(x, np.complex128)
    taps = np.asarray(taps, np.float64)
    T = taps.size
    G = groups(x.size, I, T)
    bi = np.zeros((G, I)); bq = np.zeros((G, I))
    for ip in range(I):
        tis = list(range(I - ip, T, I))
        k = len(tis)
        if not k:
            continue
        g = k * U / (1 - k * U) * 1.001
        pi = sum(np.abs(x.real[si:si + G]) * abs(taps[ti]) for si, ti in enumerate(tis))
        pq = sum(np.abs(x.imag[si:si + G]) * abs(taps[ti]) for si, ti in enumerate(tis))
        bi[:, ip] = 2 * g * pi + 2 * k * 2.0 ** -149
        bq[:, ip] = 2 * g * pq + 2 * k * 2.0 ** -149
    return bi.reshape(-1), bq.reshape(-1)


PI = np.float32(np.pi)
TWO_PI = np.float32(2) * PI
THREE_PI = np.float32(3 * np.float64(PI))


def fmmod_phases(x, phase=0.0):
    """the reference build's phase after every sample"""
    ph = np.float32(phase)
    out = np.empty(len(x), np.float32)
    for k, v in enumerate(np.asarray(x, np.float32)):
        ph = np.float32(ph + np.float32(v * PI))
        if ph > PI:
            while True:
                old = ph; ph = np.float32(ph - TWO_PI)
                if not old > THREE_PI:
                    break
        elif ph <= -PI:
            while True:
                old = ph; ph = np.float32(ph + TWO_PI)
                if not old <= -THREE_PI:
                    break
        out[k] = ph
    return out


# ---- the compiled reference ---------------------------------------------------------------------------------------------------------
def have_ref() -> bool:
    return REF_SO.exists()


def ref():
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_SO))
        vp, it = C.c_void_p, C.c_int
        L.fir_interpolate_cc.argtypes = [vp, vp, it, it, vp, it]; L.fir_interpolate_cc.restype = it
        L.fmmod_fc.argtypes = [vp, vp, it, C.c_float]; L.fmmod_fc.restype = C.c_float
        L.firdes_lowpass_f.argtypes = [vp, it, C.c_float, it]
        L.firdes_filter_len.argtypes = [C.c_float]; L.firdes_filter_len.restype = it
        _ref = L
    return _ref


def ref_fir_interpolate_cc(x, I, taps):
    x = np.ascontiguousarray(x, np.complex64); taps = np.ascontiguousarray(taps, np.float32)
    out = np.zeros(max(x.size * I, 1), np.complex64)
    m = ref().fir_interpolate_cc(x.ctypes.data, out.ctypes.data, x.size, I, taps.ctypes.data, taps.size)
    return out[:m]


def ref_fmmod_fc(x, phase=0.0):
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros(max(x.size, 1), np.complex64)
    ph = ref().fmmod_fc(x.ctypes.data, out.ctypes.data, x.size, float(phase))
    return out[:x.size], np.float32(ph)


def ref_fmmod_phases(x, phase=0.0):
    """the reference's phase after every sample, one call per sample (the carried phase is its return value)"""
    ph, out = np.float32(phase), np.empty(len(x), np.float32)
    for k in range(len(x)):
        _, ph = ref_fmmod_fc(np.asarray(x[k:k + 1], np.float32), ph)
        out[k] = ph
    return out


def ref_lowpass(T, cutoff, window=2):
    t = np.zeros(T, np.float32)
    ref().firdes_lowpass_f(t.ctypes.data, T, cutoff, window)
    return t
