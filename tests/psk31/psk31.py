"""ctypes front-end of psk31_oracle.c (the CPU restatement of simple_agc_cc, timing_recovery_cc, dbpsk_decoder_c_u8 and the varicode
decoder), bindings to the same four blocks of the compiled reference (oracle/_ref/libcsdr_ref.so), and a seeded BPSK31 test signal.
TEST INFRASTRUCTURE: the C file is compiled once per process into a temporary directory."""
from __future__ import annotations

import ctypes as C
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
REF_SO = ROOT / "oracle" / "_ref" / "libcsdr_ref.so"
REF_CLI = ROOT / "oracle" / "_ref" / "csdr_ref"

GARDNER, EARLYLATE = 0, 1

_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        out = Path(tempfile.mkdtemp(prefix="psk31_oracle_")) / "libpsk31_oracle.so"
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(out),
                        str(HERE / "psk31_oracle.c"), "-lm"], check=True)
        L = C.CDLL(str(out))
        vp, fl, it = C.c_void_p, C.c_float, C.c_int
        L.psk31_oracle_simple_agc_cc.argtypes = [vp, vp, it, fl, fl, fl, vp]
        L.psk31_oracle_timing_recovery_cc.argtypes = [vp, vp, it, vp, vp, it, it, it, fl, fl, vp]
        L.psk31_oracle_dbpsk_decoder_c_u8.argtypes = [vp, vp, it, vp]
        L.psk31_oracle_varicode_code.argtypes = [it, vp]
        L.psk31_oracle_varicode_decode.argtypes = [vp, it, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def _cf(x):
    return np.ascontiguousarray(x, np.complex64)


# ---- the checker --------------------------------------------------------------------------------------------------------------------
def simple_agc_cc(x, rate=0.001, reference=0.5, max_gain=65535.0, gain=1.0):
    """one call: (y, gain)"""
    x = _cf(x); y = np.empty_like(x); g = np.array([gain], np.float32)
    lib().psk31_oracle_simple_agc_cc(_p(x), _p(y), x.size, rate, reference, max_gain, _p(g))
    return y, float(g[0])


def timing_recovery_cc(x, algorithm, decimation, use_q=True, loop_gain=0.5, max_error=2.0, last_correction_offset=0):
    """one call: (y, error, indexes, (last_correction_offset, input_processed, output_size))"""
    x = _cf(x); n = x.size
    y = np.zeros(max(n, 1), np.complex64); e = np.zeros(max(n, 1), np.float32); ix = np.zeros(max(n, 1), np.int32)
    st = np.array([last_correction_offset, 0, 0], np.int32)
    lib().psk31_oracle_timing_recovery_cc(_p(x), _p(y), n, _p(e), _p(ix), algorithm, decimation, int(use_q), loop_gain, max_error, _p(st))
    m = int(st[2])
    return y[:m], e[:m], ix[:m], tuple(int(v) for v in st)


def dbpsk_decoder_c_u8(x, last=0j):
    """(bits, last sample)"""
    x = _cf(x); out = np.empty(x.size, np.uint8); l = np.array([last.real, last.imag], np.float32)
    lib().psk31_oracle_dbpsk_decoder_c_u8(_p(x), _p(out), x.size, _p(l))
    return out, complex(l[0], l[1])


def varicode_decode(bits, hist=0):
    """(bytes of the non-zero characters, shift register)"""
    b = np.ascontiguousarray(bits, np.uint8); out = np.empty(max(b.size, 1), np.uint8); h = np.array([hist], np.uint64)
    n = lib().psk31_oracle_varicode_decode(_p(b), b.size, _p(out), _p(h))
    return out[:n].tobytes(), int(h[0])


def varicode_table():
    """[(code, bits)] for ASCII 0..127 as the checker states it"""
    out = []
    for a in range(128):
        b = C.c_int(0)
        code = lib().psk31_oracle_varicode_code(a, C.byref(b))
        out.append((code, b.value))
    return out


def timing_stream(x, algorithm, decimation, calls, **kw):
    """the stream x cut into timing_recovery_cc calls at the given sizes; each call re-presents the unconsumed input (csdr.c:2621-2636).
    Returns (y, error, absolute indexes, final state)."""
    x = _cf(x); pos = 0; co = 0; ys, es, ixs = [], [], []
    st = (0, 0, 0)
    for size in calls:
        y, e, ix, st = timing_recovery_cc(x[pos:pos + size], algorithm, decimation, last_correction_offset=co, **kw)
        ys.append(y); es.append(e); ixs.append(ix + pos)
        co = st[0]; pos += st[1]
    return np.concatenate(ys), np.concatenate(es), np.concatenate(ixs), st


def chain(x, sps, agc_ref=0.5):
    """simple_agc_cc 0.001 R | timing_recovery_cc GARDNER sps 0.5 2 --add_q | dbpsk_decoder_c_u8 | psk31_varicode_decoder_u8_u8 over the
    whole stream x in one call per block (the timing recovery's result does not depend on how the stream is cut)"""
    a, _ = simple_agc_cc(x, 0.001, agc_ref)
    s, _, _, _ = timing_recovery_cc(a, GARDNER, sps, True, 0.5, 2.0)
    bits, _ = dbpsk_decoder_c_u8(s)
    text, _ = varicode_decode(bits)
    return text


# ---- the compiled reference ---------------------------------------------------------------------------------------------------------
class _TR(C.Structure):                  # timing_recovery_state_t (libcsdr.h:322-336)
    _fields_ = [("algorithm", C.c_int), ("decimation_rate", C.c_int), ("output_size", C.c_int), ("input_processed", C.c_int),
                ("use_q", C.c_int), ("debug_phase", C.c_int), ("debug_every_nth", C.c_int), ("debug_writefiles_path", C.c_char_p),
                ("last_correction_offset", C.c_int), ("earlylate_ratio", C.c_float), ("loop_gain", C.c_float), ("max_error", C.c_float)]


def have_ref() -> bool:
    return REF_SO.exists()


def ref():
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_SO))
        vp, fl, it = C.c_void_p, C.c_float, C.c_int
        L.simple_agc_cc.argtypes = [vp, vp, it, fl, fl, fl, vp]
        L.timing_recovery_init.argtypes = [it, it, it, fl, fl, it, C.c_char_p]; L.timing_recovery_init.restype = _TR
        L.timing_recovery_cc.argtypes = [vp, vp, it, vp, vp, C.POINTER(_TR)]
        L.dbpsk_decoder_c_u8.argtypes = [vp, vp, it]
        L.psk31_varicode_decoder_push.argtypes = [C.POINTER(C.c_ulonglong), C.c_ubyte]; L.psk31_varicode_decoder_push.restype = C.c_ubyte
        L.psk31_varicode_encoder_u8_u8.argtypes = [vp, vp, it, it, C.POINTER(it), C.POINTER(it)]
        _ref = L
    return _ref


def ref_simple_agc_cc(x, rate=0.001, reference=0.5, max_gain=65535.0, gain=1.0):
    x = _cf(x); y = np.empty_like(x); g = np.array([gain], np.float32)
    ref().simple_agc_cc(_p(x), _p(y), x.size, rate, reference, max_gain, _p(g))
    return y, float(g[0])


def ref_timing_recovery_cc(x, algorithm, decimation, use_q=True, loop_gain=0.5, max_error=2.0, last_correction_offset=0):
    x = _cf(x); n = x.size
    y = np.zeros(max(n, 1), np.complex64); e = np.zeros(max(n, 1), np.float32); ix = np.zeros(max(n, 1), np.int32)
    st = ref().timing_recovery_init(algorithm, decimation, int(use_q), loop_gain, max_error, -1, None)
    st.last_correction_offset = last_correction_offset
    ref().timing_recovery_cc(_p(x), _p(y), n, _p(e), _p(ix), C.byref(st))
    m = st.output_size
    return y[:m], e[:m], ix[:m], (st.last_correction_offset, st.input_processed, st.output_size)


def ref_dbpsk_decoder_c_u8(x, last=0j):
    """the reference keeps its previous sample in a static: one call on [last] sets it first"""
    x = _cf(x); pre = np.array([last], np.complex64); junk = np.empty(1, np.uint8); out = np.empty(x.size, np.uint8)
    ref().dbpsk_decoder_c_u8(_p(pre), _p(junk), 1)
    ref().dbpsk_decoder_c_u8(_p(x), _p(out), x.size)
    return out


def ref_varicode_decode(bits, hist=0):
    h = C.c_ulonglong(hist); out = bytearray()
    for b in np.asarray(bits, np.uint8):
        c = ref().psk31_varicode_decoder_push(C.byref(h), int(b))
        if c:
            out.append(c)
    return bytes(out), h.value


def ref_varicode_encode(text: bytes):
    """psk31_varicode_encoder_u8_u8 of the compiled reference: one byte (0/1) per bit"""
    t = np.frombuffer(text, np.uint8).copy(); cap = 16 * t.size + 16
    out = np.zeros(cap, np.uint8); ip = C.c_int(0); os_ = C.c_int(0)
    ref().psk31_varicode_encoder_u8_u8(_p(t), _p(out), t.size, cap, C.byref(ip), C.byref(os_))
    assert ip.value == t.size
    return out[:os_.value].copy()


# ---- a seeded BPSK31 signal ---------------------------------------------------------------------------------------------------------
def modulate(bits, sps, rng, freq=0.0, noise=0.02, amplitude=0.3, lead=32, tail=32):
    """differential BPSK at sps samples per symbol: a 0 bit reverses the phase, a 1 keeps it (PSK31); `lead`/`tail` idle reversals around
    the bits, raised-cosine transitions, a carrier offset of `freq` cycles per sample and complex Gaussian noise"""
    allbits = np.concatenate([np.zeros(lead, np.uint8), np.asarray(bits, np.uint8), np.zeros(tail, np.uint8)])
    sym = np.empty(allbits.size + 1, np.float64); sym[0] = 1.0
    for k, b in enumerate(allbits):
        sym[k + 1] = sym[k] if b else -sym[k]
    t = np.arange(sps) / sps
    ramp = 0.5 - 0.5 * np.cos(np.pi * t)                                   # 0 -> 1 over one symbol
    base = np.concatenate([sym[k] + (sym[k + 1] - sym[k]) * ramp for k in range(sym.size - 1)])
    n = base.size
    z = amplitude * base * np.exp(2j * np.pi * freq * np.arange(n) + 1j * rng.uniform(0, 2 * np.pi))
    z = z + noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return z.astype(np.complex64)
