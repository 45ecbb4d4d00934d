"""The checker side of the amplitude modulator banks (csdr_b200/csrc/modulate.cu): numpy restatements of gain_ff, dsb_fc, add_dcoffset_cc (as the
reference build runs it) and fixed_amplitude_cc (the source's sqrt/division form), the float64 bound of fixed_amplitude_cc, bindings to the
compiled reference (oracle/_ref/libcsdr_ref.so), and the checks both tiers run through the C ABI.  TEST INFRASTRUCTURE.

fixed_amplitude_cc bound.  y = A*x/|x| exactly; u = 2^-24.  The kernel: s = fl(fl(i*i) + fl(q*q)) has relative error <= 3u (three roundings of
non-negative terms), sqrt halves it and rounds (<= 2.5u), the division adds one rounding (<= 3.5u), the product one more: each component within
4.6u*|A*x_k|/|x| <= 4.6u*|A|.  The build replaces sqrt and division by rsqrtss (relative error <= 1.5*2^-12) and one Newton step, which leaves
1.5*(1.5*2^-12)^2 = 2e-7 = 3.4u, plus six roundings.  Both are held to 10u*|A| per component (measured: build 5.2u, kernel 3.4u) wherever s is a
finite normal float; where s is zero both give a zero, compared by value."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
REF_SO = ROOT / "oracle" / "_ref" / "libcsdr_ref.so"
U = 2.0 ** -24
BOUND_U = 10
F = np.float32
_ref = None


# ---- restatements ------------------------------------------------------------------------------------------------------------------------
def gain_ff(x, gain):
    with np.errstate(all="ignore"):
        return (np.asarray(x, F) * F(gain)).astype(F)


def dsb_fc(x, q_value=0.0):
    x = np.asarray(x, F)
    out = np.empty(x.shape + (2,), F)
    out[..., 0] = x; out[..., 1] = F(q_value)
    return out.view(np.complex64)[..., 0]


def add_dcoffset_cc(x):
    v = np.asarray(x, np.complex64).view(F).reshape(np.shape(x) + (2,))
    out = np.empty_like(v)
    with np.errstate(all="ignore"):
        out[..., 0] = (v[..., 0] + F(1)) * F(0.5)
        out[..., 1] = v[..., 1] * F(0.5)
    return out.view(np.complex64)[..., 0]


def fixed_amplitude_cc(x, amplitude):
    v = np.asarray(x, np.complex64).view(F).reshape(np.shape(x) + (2,))
    i, q = v[..., 0], v[..., 1]
    with np.errstate(all="ignore"):
        now = np.sqrt((i * i + q * q).astype(F)).astype(F)
        g = np.where(now > 0, (F(amplitude) / np.where(now > 0, now, F(1))).astype(F), F(0)).astype(F)
        out = np.stack([(i * g).astype(F), (q * g).astype(F)], axis=-1)
    return np.ascontiguousarray(out).view(np.complex64)[..., 0]


def same_bits(a, b):
    """equal float32 bits, NaN for NaN (a GPU's NaN results carry the canonical payload)"""
    fa, fb = np.asarray(a).view(F), np.asarray(b).view(F)
    na, nb = np.isnan(fa), np.isnan(fb)
    return fa.shape == fb.shape and np.array_equal(na, nb) and np.array_equal(fa[~na].view(np.uint32), fb[~nb].view(np.uint32))


def fixed_amplitude_ok(got, x, amplitude, want_ref=None):
    """got (and want_ref, the build's output, when given) within the float64 bound where s = i*i + q*q is a finite normal float; zeros where s
    is zero; returns the worst error in units of u*|A|"""
    x = np.asarray(x, np.complex64)
    i, q = x.real.astype(F), x.imag.astype(F)
    with np.errstate(all="ignore"):
        s = (i * i + q * q).astype(F)
    normal = np.isfinite(s) & (s >= np.finfo(F).tiny)
    zero = s == 0
    xd = x.astype(np.complex128)[normal]
    exact = float(amplitude) * xd / np.abs(xd)
    worst = 0.0
    for y in [got] + ([want_ref] if want_ref is not None else []):
        y = np.asarray(y, np.complex64)
        e = np.maximum(np.abs(y[normal].real.astype(np.float64) - exact.real), np.abs(y[normal].imag.astype(np.float64) - exact.imag))
        if e.size:
            worst = max(worst, float(e.max()) / (U * abs(float(amplitude)) or 1.0))
        assert np.all(e <= BOUND_U * U * abs(float(amplitude)) + 1e-45), float(e.max()) if e.size else 0
        assert np.all(y[zero] == 0), "s == 0 must give a zero"
    return worst


# ---- test vectors ----------------------------------------------------------------------------------------------------------------------------
SPECIAL = np.array([0.0, -0.0, 1e-45, -1e-45, 3e-39, -1.1e-38, 1.5e-38, np.inf, -np.inf, np.nan, 1.0, -1.0, 0.5, 3.4e38, -3.4e38, 1e-20, 7.0,
                    -0.25], F)


def real_rows(rng, ch, n):
    """uniform samples with the special values scattered in"""
    x = rng.uniform(-1, 1, (ch, n)).astype(F)
    k = min(n, SPECIAL.size)
    for c in range(ch):
        pos = rng.choice(n, k, replace=False) if n else []
        x[c, pos] = rng.choice(SPECIAL, k)
    return x


def complex_rows(rng, ch, n):
    return np.ascontiguousarray(np.stack([real_rows(rng, ch, n), real_rows(rng, ch, n)], axis=-1)).view(np.complex64)[..., 0]


def magnitude_rows(rng, ch, n):
    """fixed_amplitude_cc inputs spanning 12 decades of magnitude at every angle"""
    mag = 10.0 ** rng.uniform(-6, 6, (ch, n))
    ang = rng.uniform(-np.pi, np.pi, (ch, n))
    return (mag * np.exp(1j * ang)).astype(np.complex64)


# ---- the C ABI, on host memory (the emulated library) or device memory ---------------------------------------------------------------------
BANKS = {  # name: (input dtype, output dtype, takes a scalar)
    "gain": (F, F, True),
    "dsb": (F, np.complex64, True),
    "add_dcoffset": (np.complex64, np.complex64, False),
    "fixed_amplitude": (np.complex64, np.complex64, True),
}


def bind(L):
    vp, lg, it, fl = C.c_void_p, C.c_long, C.c_int, C.c_float
    L.csdrb_gain_bank_ff.argtypes = [vp, lg, vp, lg, it, it, fl, vp]
    L.csdrb_dsb_bank_fc.argtypes = [vp, lg, vp, lg, it, it, fl, vp]
    L.csdrb_add_dcoffset_bank_cc.argtypes = [vp, lg, vp, lg, it, it, vp]
    L.csdrb_fixed_amplitude_bank_cc.argtypes = [vp, lg, vp, lg, it, it, fl, vp]
    L.gain_ff.argtypes = [vp, vp, it, fl]
    L.add_dcoffset_cc.argtypes = [vp, vp, it]
    L.fixed_amplitude_cc.argtypes = [vp, vp, it, fl]
    L.csdrb_kernel_launches.restype = C.c_long
    return L


def call(L, name, d_in, in_stride, d_out, out_stride, channels, n, arg=0.0, stream=None):
    f = {"gain": L.csdrb_gain_bank_ff, "dsb": L.csdrb_dsb_bank_fc, "add_dcoffset": L.csdrb_add_dcoffset_bank_cc,
         "fixed_amplitude": L.csdrb_fixed_amplitude_bank_cc}[name]
    if BANKS[name][2]:
        return f(d_in, in_stride, d_out, out_stride, channels, n, arg, stream)
    return f(d_in, in_stride, d_out, out_stride, channels, n, stream)


def restate(name, x, arg):
    return {"gain": lambda: gain_ff(x, arg), "dsb": lambda: dsb_fc(x, arg), "add_dcoffset": lambda: add_dcoffset_cc(x),
            "fixed_amplitude": lambda: fixed_amplitude_cc(x, arg)}[name]()


def rows_for(name, rng, ch, n):
    return real_rows(rng, ch, n) if BANKS[name][0] is F else complex_rows(rng, ch, n)


ARGS = {"gain": [0.5, -3.0, 1e-30, 0.0, 2.5e38], "dsb": [0.0, 0.3, -1e-40], "add_dcoffset": [0.0], "fixed_amplitude": [1.0, 2.0, 0.3]}


def refusals(L, h_in, h_out):
    """every refusal returns -1; the pointers point at host (emulated) or device buffers of at least 64 elements"""
    bad = []
    for name in BANKS:
        for args in ((h_in, 8, h_out, 8, 1, -1), (h_in, 8, h_out, 8, -1, 8), (h_in, 7, h_out, 8, 1, 8), (h_in, 8, h_out, 7, 1, 8),
                     (None, 8, h_out, 8, 1, 8), (h_in, 8, None, 8, 1, 8), (h_in, 8, h_in, 16, 2, 8)):
            if call(L, name, *args, 1.0) != -1:
                bad.append((name, args))
        if call(L, name, None, 0, None, 0, 1, 0, 1.0) != 0 or call(L, name, None, 8, None, 8, 0, 8, 1.0) != 8:   # no work: no pointer needed
            bad.append((name, "no work"))
    if call(L, "dsb", h_in, 8, h_in, 8, 1, 8, 1.0) != -1:                                                  # dsb_fc is never in place
        bad.append(("dsb", "in place"))
    return bad


# ---- the compiled reference ------------------------------------------------------------------------------------------------------------------
def have_ref() -> bool:
    return REF_SO.exists()


def ref():
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_SO))
        vp, it = C.c_void_p, C.c_int
        L.gain_ff.argtypes = [vp, vp, it, C.c_float]
        L.add_dcoffset_cc.argtypes = [vp, vp, it]
        L.fixed_amplitude_cc.argtypes = [vp, vp, it, C.c_float]
        _ref = L
    return _ref


def ref_call(name, x, arg=0.0):
    """the reference library on one row; dsb_fc has no library function and is restated"""
    x = np.ascontiguousarray(x)
    if name == "dsb":
        return dsb_fc(x, arg)
    out = np.zeros_like(x)
    if name == "gain":
        ref().gain_ff(x.ctypes.data, out.ctypes.data, x.size, arg)
    elif name == "add_dcoffset":
        ref().add_dcoffset_cc(x.ctypes.data, out.ctypes.data, x.size)
    else:
        ref().fixed_amplitude_cc(x.ctypes.data, out.ctypes.data, x.size, arg)
    return out
