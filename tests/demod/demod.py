"""The checker side of the demodulator banks (csdr_b200/csrc/demod.cu, the dcblock recursion of audio.cu and K4's novect form): numpy restatements
of fmdemod_atan_cf, fmdemod_quadri_novect_cf, amdemod_estimator_cf and dcblock_ff as the reference build computes them, bindings to the compiled
reference (oracle/_ref/libcsdr_ref.so), and the checks both tiers run through the C ABI.  TEST INFRASTRUCTURE.

The atan rounding rule.  The phase is (float)atan2((double)Q, (double)I).  On the host both sides call glibc's atan2, so the emulated banks give
the reference's bits.  CUDA's double atan2 is within 2 ulp (double) of the exact value, so its float rounding can differ from glibc's only where
the double value lies that close to a float rounding midpoint.  atan_near_midpoint() marks the samples whose float64 phase (numpy's arctan2, the
same libm as the build) lies within 4 ulp (double) of one; there the phase may be one float ulp off.  Phase k enters outputs k and k+1 as one
operand of a float subtraction in [-2pi, 2pi], so each of them may move by at most ATAN_NEAR_BOUND (one ulp of pi for the phase, one ulp of 2pi
for the subtraction's rounding, scaled by 1/pi, plus the product's rounding); the wrap by 2pi may then flip, which moves the output by 2 more.
Everywhere else the bits must be the reference's."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
REF_SO = ROOT / "oracle" / "_ref" / "libcsdr_ref.so"
F = np.float32
PI = F(np.pi)
INV_PI = F(float.fromhex("0x1.45f306p-2"))                             # the float reciprocal of PI the build multiplies by
K = 0.340447550238101026565118445432744920253753662109375
EST_ALPHA, EST_BETA = F(0.947543636291), F(0.392485425092)
ATAN_NEAR_BOUND = 2.0 ** -21
_ref = None


# ---- restatements ------------------------------------------------------------------------------------------------------------------------
def _iq(x):
    v = np.ascontiguousarray(x, np.complex64).view(F).reshape(np.shape(x) + (2,))
    return v[..., 0], v[..., 1]


def atan_phase(x):
    i, q = _iq(x)
    with np.errstate(all="ignore"):
        return np.arctan2(q.astype(np.float64), i.astype(np.float64)).astype(F)


def fmdemod_atan_from_phase(ph, last=0.0):
    ph = np.asarray(ph, F)
    prev = np.concatenate([[F(last)], ph[:-1]]).astype(F)
    with np.errstate(all="ignore"):
        d = (ph - prev).astype(F)
        d = np.where(d < -PI, (d + F(2) * PI).astype(F), np.where(d > PI, (d - F(2) * PI).astype(F), d)).astype(F)
        return (d * INV_PI).astype(F)


def fmdemod_atan_cf(x, last=0.0):
    """(y, the last sample's phase) of one call"""
    ph = atan_phase(x)
    return fmdemod_atan_from_phase(ph, last), (F(ph[-1]) if ph.size else F(last))


def fmdemod_quadri_novect_cf(x, last=0j):
    """(y, the last sample) of one call as the build computes it: the numerator as I*(Q-Qp) + Q*(Ip-I) (fmdemod_quadri_cf's form
    I*(Q-Qp) - Q*(I-Ip) gives the other sign of a zero where consecutive samples are equal and I < 0), and a zero den divided by"""
    x = np.asarray(x, np.complex64)
    i, q = _iq(x)
    prev = np.concatenate([[np.complex64(last)], x[:-1]])
    pi_, pq = _iq(prev)
    with np.errstate(all="ignore"):
        num = ((i * (q - pq).astype(F)).astype(F) + (q * (pi_ - i).astype(F)).astype(F)).astype(F)
        den = ((i * i).astype(F) + (q * q).astype(F)).astype(F)
        y = (K * num.astype(np.float64) / den.astype(np.float64)).astype(F)
    return y, (complex(x[-1]) if x.size else last)


def amdemod_estimator_cf(x, alpha=0.0, beta=0.0):
    """one call on the samples x"""
    if F(alpha) == 0:
        alpha, beta = EST_ALPHA, EST_BETA
    i, q = _iq(x)
    ai, aq = np.abs(i), np.abs(q)
    with np.errstate(all="ignore"):
        if np.size(x) >= 2:                                            # the build's SSE loops: maxps/minps(|I|, |Q|), a NaN takes |Q|
            mx = np.where(ai > aq, ai, aq)
            mn = np.where(ai < aq, ai, aq)
        else:                                                          # its scalar loop for a call of one sample: a NaN takes |I|
            mx = np.where(aq > ai, aq, ai)
            mn = np.where(aq < ai, aq, ai)
        return ((F(alpha) * mx).astype(F) + (F(beta) * mn).astype(F)).astype(F)


def dcblock_rows(x, a=0.0, state=None):
    """dcblock_ff over rows x [C, n] at once (the recursion runs along n, vectorised over channels): (y, state [C, 2])"""
    x = np.atleast_2d(np.asarray(x, F))
    a = F(0.999) if F(a) == 0 else F(a)
    st = np.zeros((x.shape[0], 2), F) if state is None else np.array(state, F).reshape(x.shape[0], 2)
    last_in, last_out = st[:, 0].copy(), st[:, 1].copy()
    y = np.empty_like(x)
    with np.errstate(all="ignore"):
        for k in range(x.shape[1]):
            last_out = ((x[:, k] - last_in).astype(F) + (a * last_out).astype(F)).astype(F)
            last_in = x[:, k]
            y[:, k] = last_out
    return y, np.stack([last_in, last_out], axis=1).astype(F)


def same_bits(a, b):
    """equal float32 bits, NaN for NaN (a GPU's NaN results carry the canonical payload)"""
    fa, fb = np.asarray(a, F).ravel(), np.asarray(b, F).ravel()
    na, nb = np.isnan(fa), np.isnan(fb)
    return fa.shape == fb.shape and np.array_equal(na, nb) and np.array_equal(fa[~na].view(np.uint32), fb[~nb].view(np.uint32))


# ---- the atan rounding rule ----------------------------------------------------------------------------------------------------------------
def atan_near_midpoint(x):
    """samples whose float64 phase lies within 4 ulp (double) of a float32 rounding midpoint"""
    i, q = _iq(x)
    with np.errstate(all="ignore"):
        p = np.arctan2(q.astype(np.float64), i.astype(np.float64))
        f = p.astype(F)
        up = np.nextafter(f, F(np.inf)).astype(np.float64)
        dn = np.nextafter(f, F(-np.inf)).astype(np.float64)
        f64 = f.astype(np.float64)
        dist = np.minimum(np.abs(p - (f64 + up) / 2), np.abs(p - (f64 + dn) / 2))
        return np.isfinite(p) & (dist <= 4 * np.spacing(np.abs(p)))


def atan_matches(got, want, x):
    """got equals want bit for bit except at outputs k and k+1 of samples k near a midpoint, which are held to ATAN_NEAR_BOUND (or that
    plus a flipped wrap of 2).  Returns (near samples, outputs that differ)."""
    got, want = np.asarray(got, F), np.asarray(want, F)
    near = atan_near_midpoint(x)
    touched = near.copy()
    touched[1:] |= near[:-1]
    diff = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    assert not np.any(diff & ~touched), f"{int(np.sum(diff & ~touched))} outputs differ away from a rounding midpoint, e.g. at " \
                                        f"{np.flatnonzero(diff & ~touched)[:5]}"
    e = np.abs(got[diff].astype(np.float64) - want[diff].astype(np.float64))
    assert np.all((e <= ATAN_NEAR_BOUND) | (np.abs(e - 2) <= ATAN_NEAR_BOUND)), float(e.max())
    return int(near.sum()), int(diff.sum())


# ---- test vectors ----------------------------------------------------------------------------------------------------------------------------
SPECIAL = np.array([0.0, -0.0, 1e-45, -1e-45, 3e-39, -1.1e-38, 1.5e-38, np.inf, -np.inf, np.nan, 1.0, -1.0, 0.5, 3.4e38, -3.4e38, 1e-20, 7.0,
                    -0.25, 1e-23, -2e-23], F)


def complex_rows(rng, ch, n, special=True):
    """uniform I and Q in [-1, 1), the special values scattered into I, Q or both (edge_row() has every edge case once)"""
    v = rng.uniform(-1, 1, (ch, n, 2)).astype(F)
    if special and n:
        for c in range(ch):
            k = min(n, SPECIAL.size)
            pos = rng.choice(n, k, replace=False)
            which = rng.integers(0, 3, k)
            vals = rng.choice(SPECIAL, (k, 2))
            for p, w, (a, b) in zip(pos, which, vals):
                if w == 0: v[c, p, 0] = a
                elif w == 1: v[c, p, 1] = b
                else: v[c, p] = (a, b)
    return np.ascontiguousarray(v).view(np.complex64)[..., 0]


def edge_row():
    """the atan2 quadrant edges (+-0 against +-0, which give +-pi or +-0), +-Inf pairs, NaN in I, Q and both, subnormals, and quadri's den = 0"""
    z, nz, inf, nan, sub = 0.0, -0.0, np.inf, np.nan, 1e-45
    pairs = [(z, z), (nz, z), (z, nz), (nz, nz), (z, 1.0), (nz, -1.0), (-1.0, z), (-1.0, nz), (inf, inf), (-inf, inf), (inf, -inf), (-inf, -inf),
             (inf, 1.0), (-inf, 1.0), (1.0, inf), (1.0, -inf), (nan, 1.0), (1.0, nan), (nan, nan), (0.5, 0.5), (sub, sub), (-sub, sub),
             (sub, -sub), (1e-23, 1e-23), (-1e-23, 2e-23), (3e-39, -3e-39), (1.0, z), (z, z), (-1.0, z), (z, z), (1.0, 1e-30), (-1.0, -1e-30)]
    return np.array([complex(a, b) for a, b in pairs], np.complex64)


def quantised_rows(rng, ch, n):
    """an 8-bit receiver's samples (u8 levels through convert_u8_f's arithmetic): a slowly turning carrier, so consecutive samples repeat, in
    every quadrant -- where fmdemod_quadri_novect_cf's numerator is a zero whose sign depends on the form the build computes"""
    ph = np.cumsum(rng.uniform(0.0, 0.02, (ch, n)), axis=1) + rng.uniform(0, 2 * np.pi, (ch, 1))
    z = 0.6 * np.exp(1j * ph)
    v = np.stack([z.real, z.imag], axis=-1)
    u8 = np.clip(np.floor(v * 127.5 + 128), 0, 255)
    f = (u8.astype(F) / F(127.5) - F(1)).astype(F)
    return np.ascontiguousarray(f).view(np.complex64)[..., 0]


def real_rows(rng, ch, n):
    x = rng.uniform(-1, 1, (ch, n)).astype(F)
    for c in range(ch):
        k = min(n, SPECIAL.size)
        if k:
            x[c, rng.choice(n, k, replace=False)] = rng.choice(SPECIAL, k)
    return x


# ---- the C ABI on host memory (the emulated library) or device memory ----------------------------------------------------------------------
class DcBlock(C.Structure):
    _fields_ = [("last_input", C.c_float), ("last_output", C.c_float)]


class CF(C.Structure):
    _fields_ = [("i", C.c_float), ("q", C.c_float)]


def bind(L):
    vp, lg, it, fl = C.c_void_p, C.c_long, C.c_int, C.c_float
    L.csdrb_fmdemod_atan_bank_cf.argtypes = [vp, lg, vp, lg, it, it, vp, vp, vp]
    L.csdrb_fmdemod_quadri_novect_bank_cf.argtypes = [vp, lg, vp, lg, it, it, vp, vp, vp]
    L.csdrb_fmdemod_quadri_bank_cf.argtypes = [vp, lg, vp, lg, it, it, vp, vp, vp]
    L.csdrb_amdemod_estimator_bank_cf.argtypes = [vp, lg, vp, lg, it, it, fl, fl, vp]
    L.csdrb_dcblock_bank_ff.argtypes = [vp, lg, vp, lg, it, it, fl, vp, vp]
    L.fmdemod_atan_cf.argtypes = [vp, vp, it, fl]; L.fmdemod_atan_cf.restype = fl
    L.fmdemod_quadri_novect_cf.argtypes = [vp, vp, it, CF]; L.fmdemod_quadri_novect_cf.restype = CF
    L.amdemod_estimator_cf.argtypes = [vp, vp, it, fl, fl]
    L.dcblock_ff.argtypes = [vp, vp, it, fl, DcBlock]; L.dcblock_ff.restype = DcBlock
    L.csdrb_last_error.restype = C.c_char_p
    L.csdrb_kernel_launches.restype = C.c_long
    return L


def refusals(L, d_cf, d_f, d_state):
    """every refusal returns a negative code and launches nothing; the pointers point at host (emulated) or device buffers of at least 64
    elements (d_cf complexf, d_f float, d_state two dcblock_preserve_t / four floats)"""
    bad = []
    before = L.csdrb_kernel_launches()
    banks = {  # name: (its input buffer, the input's alignment, the call)
        "atan": (d_cf, 8, lambda i, si, o, so, ch, n: L.csdrb_fmdemod_atan_bank_cf(i, si, o, so, ch, n, d_state, d_state + 8, None)),
        "estimator": (d_cf, 8, lambda i, si, o, so, ch, n: L.csdrb_amdemod_estimator_bank_cf(i, si, o, so, ch, n, 0.0, 0.0, None)),
        "dcblock": (d_f, 4, lambda i, si, o, so, ch, n: L.csdrb_dcblock_bank_ff(i, si, o, so, ch, n, 0.0, d_state, None)),
    }
    for name, (src, align, f) in banks.items():
        for args in ((src, 8, d_f, 8, 1, -1), (src, 8, d_f, 8, -1, 8), (src, 8, d_f, 8, 70000, 8), (src, 7, d_f, 8, 2, 8), (src, 8, d_f, 7, 2, 8),
                     (None, 8, d_f, 8, 1, 8), (src, 8, None, 8, 1, 8), (src + align // 2, 8, d_f, 8, 1, 8), (src, 8, d_f + 2, 8, 1, 8)):
            if f(*args) >= 0:
                bad.append((name, args))
    if L.csdrb_fmdemod_atan_bank_cf(d_cf, 8, d_f, 8, 1, 8, d_state, d_state, None) >= 0:
        bad.append(("atan", "aliased phases"))
    if L.csdrb_fmdemod_atan_bank_cf(d_cf, 8, d_cf, 8, 1, 8, None, None, None) >= 0:
        bad.append(("atan", "in place"))
    if L.csdrb_amdemod_estimator_bank_cf(d_cf, 8, d_cf, 8, 1, 8, 0.0, 0.0, None) >= 0:
        bad.append(("estimator", "in place"))
    if L.csdrb_dcblock_bank_ff(d_f, 8, d_f, 16, 2, 8, 0.0, d_state, None) >= 0:
        bad.append(("dcblock", "in place with different strides"))
    if L.csdrb_dcblock_bank_ff(d_f, 8, d_f + 256, 8, 1, 8, 0.0, None, None) >= 0:
        bad.append(("dcblock", "null state"))
    if L.csdrb_fmdemod_quadri_novect_bank_cf(None, 8, d_f, 8, 1, 8, None, None, None) >= 0:
        bad.append(("novect", "null input"))
    if L.csdrb_fmdemod_quadri_novect_bank_cf(d_cf, 8, d_f, 8, 1, 8, d_state, d_state, None) >= 0:
        bad.append(("novect", "aliased carries"))
    if not L.csdrb_last_error():
        bad.append(("no message", None))
    if L.csdrb_kernel_launches() != before:
        bad.append(("launches", L.csdrb_kernel_launches() - before))
    return bad


# ---- the compiled reference ------------------------------------------------------------------------------------------------------------------
def have_ref() -> bool:
    return REF_SO.exists()


def ref():
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_SO))
        vp, it, fl = C.c_void_p, C.c_int, C.c_float
        L.fmdemod_atan_cf.argtypes = [vp, vp, it, fl]; L.fmdemod_atan_cf.restype = fl
        L.fmdemod_quadri_novect_cf.argtypes = [vp, vp, it, CF]; L.fmdemod_quadri_novect_cf.restype = CF
        L.amdemod_estimator_cf.argtypes = [vp, vp, it, fl, fl]
        L.dcblock_ff.argtypes = [vp, vp, it, fl, DcBlock]; L.dcblock_ff.restype = DcBlock
        _ref = L
    return _ref


def ref_atan(x, last=0.0):
    x = np.ascontiguousarray(x, np.complex64); y = np.empty(x.size, F)
    r = ref().fmdemod_atan_cf(x.ctypes.data, y.ctypes.data, x.size, last)
    return y, F(r)


def ref_novect(x, last=0j):
    x = np.ascontiguousarray(x, np.complex64); y = np.empty(x.size, F)
    r = ref().fmdemod_quadri_novect_cf(x.ctypes.data, y.ctypes.data, x.size, CF(F(last.real), F(last.imag)))
    return y, complex(r.i, r.q)


def ref_estimator(x, alpha=0.0, beta=0.0):
    x = np.ascontiguousarray(x, np.complex64); y = np.empty(x.size, F)
    ref().amdemod_estimator_cf(x.ctypes.data, y.ctypes.data, x.size, alpha, beta)
    return y


def ref_dcblock(x, a=0.0, state=(0.0, 0.0)):
    x = np.ascontiguousarray(x, F); y = np.empty(x.size, F)
    r = ref().dcblock_ff(x.ctypes.data, y.ctypes.data, x.size, a, DcBlock(*state))
    return y, (F(r.last_input), F(r.last_output))
