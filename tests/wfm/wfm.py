"""Checker and drivers for the WFM audio bank csdrb_wfm_audio_bank_f_s16 (csdr_b200/csrc/audio.cu).  TEST INFRASTRUCTURE.

The bank's contract is the CLI pipe `fractional_decimator_ff R 12 | deemphasis_wfm_ff SR TAU | convert_f_s16` with buffer size B on every row.
The checker is the oracle's composition of the same three steps: the decimator in the CLI's B-sample calls (oracle.fractional_decimator_ff with
block=B, complete calls only), the de-emphasis in B-sample calls from stream start, and convert_f_s16.  The bank runs through a `Dev` of
tests/spectrum/spectrum.py: the emulated library (numpy buffers as device memory) or the real one on a GPU (torch CUDA tensors), so the CPU
and GPU tiers run the same bodies.  replay() is a brute-force float32 restatement of the reference's call loop (libcsdr.c:751-793 driven as
csdr.c:1510-1522 drives it), used to check the bank's output counts and its refusals."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT / "tests" / "spectrum"))
import spectrum as S  # noqa: E402

POINTS = 12


class Params(C.Structure):
    _fields_ = [("rate", C.c_float), ("bufsize", C.c_int), ("tau", C.c_float), ("sample_rate", C.c_int)]


class State(C.Structure):
    _fields_ = [("where", C.c_float), ("audio", C.c_longlong)]


def setup(L):
    vp, lg, it = C.c_void_p, C.c_long, C.c_int
    L.csdrb_wfm_audio_bank_outputs.argtypes = [C.POINTER(Params), C.POINTER(State), it, C.POINTER(it)]
    L.csdrb_wfm_audio_bank_f_s16.argtypes = [vp, lg, it, it, C.POINTER(Params), C.POINTER(State), vp, vp, lg, C.POINTER(it), vp]
    return L


def emul_dev(L):
    d = S.EmulDev(L); setup(d.L); return d


def cuda_dev():
    d = S.CudaDev(); setup(d.L); return d


def checker(oracle, x, rate, bufsize, tau=50e-6, sample_rate=48000, last=0.0):
    """one row: the oracle's composition over the complete decimator calls"""
    y = oracle.fractional_decimator_ff(np.ascontiguousarray(x, np.float32), rate, POINTS, None, bufsize)
    a, _ = oracle.deemphasis_wfm_ff(y, tau, sample_rate, last=last, block=bufsize)
    return oracle.convert_f_s16(a)


def replay(rate, bufsize, n, where=None):
    """the reference's calls over n samples in float32: (outputs, consumed, where) or None when a call would consume nothing or more than B"""
    r, w = np.float32(rate), np.float32(5.0 if where is None else where)
    at = m = 0
    while n - at >= bufsize:
        while True:
            high = int(np.ceil(w))
            if not high + POINTS < bufsize:
                break
            m += 1
            w = np.float32(w + r)
        processed = high - 1 - (POINTS // 2 - 1)
        if processed < 1 or processed > bufsize:
            return None
        w = np.float32(w - np.float32(processed))
        at += processed
    return m, at, float(w)


def outputs(dev, p, s, n):
    consumed = C.c_int(-7)
    m = dev.L.csdrb_wfm_audio_bank_outputs(C.byref(p), C.byref(s), n, C.byref(consumed))
    return m, consumed.value


def bank(dev, x, p, cuts=(), pad=0, last=None, starts=None):
    """x [rows, T] float32 through the bank in calls cut at `cuts`, each re-presenting the unconsumed rest at the row start, rows `pad` floats
    apart beyond their length; returns ([rows, m] int16, final State, final carry).  `starts`, a list, gets the audio index each call starts at."""
    x = np.asarray(x, np.float32)
    rows, T = x.shape
    s = State(0.0, 0)
    d_last = dev.put(np.zeros(rows, np.float32) if last is None else np.asarray(last, np.float32))
    rest = np.zeros((rows, 0), np.float32)
    parts = []
    for a, b in zip((0,) + tuple(cuts), tuple(cuts) + (T,)):
        cur = np.concatenate([rest, x[:, a:b]], axis=1)
        n = cur.shape[1]
        stride = n + pad
        buf = np.zeros((rows, max(stride, 1)), np.float32); buf[:, :n] = cur
        m, _ = outputs(dev, p, s, n)
        assert m >= 0, dev.L.csdrb_last_error()
        if starts is not None:
            starts.append(s.audio)
        ostride = m + pad + 1
        d_in, d_out = dev.put(buf), dev.alloc(2 * rows * ostride)
        consumed = C.c_int(-1)
        got = dev.L.csdrb_wfm_audio_bank_f_s16(dev.ptr(d_in), stride, rows, n, C.byref(p), C.byref(s), dev.ptr(d_last), dev.ptr(d_out), ostride,
                                               C.byref(consumed), dev.stream)
        assert got == m, (got, m, dev.L.csdrb_last_error())
        parts.append(dev.get(d_out, np.int16).reshape(rows, ostride)[:, :m])
        rest = cur[:, consumed.value:]
        assert rest.shape[1] < p.bufsize
    return np.concatenate(parts, axis=1), s, dev.get(d_last, np.float32)


def signal(rng, rows, T, hot=True):
    """discriminator-like rows: tones and a little noise within +-1, with (hot) a few samples far past full scale where s16 wraps"""
    t = np.arange(T)
    f = rng.uniform(0.001, 0.05, (rows, 1))
    x = 0.5 * np.sin(2 * np.pi * f * t) + 0.05 * rng.standard_normal((rows, T))
    if hot:
        x[:, rng.integers(0, T, 8)] = rng.choice([-40.0, 40.0], (rows, 8))
    return x.astype(np.float32)
