"""ctypes front-end of rtty_oracle.c (the CPU restatement of serial_line_decoder_f_u8 and rtty_baudot_decoder_lookup), bindings to the same
functions of the compiled reference (oracle/_ref/libcsdr_ref.so), and a seeded RTTY signal: ITA2 at 45.45 Bd, 170 Hz shift, continuous-phase
FSK, 1.5 stop bits.  TEST INFRASTRUCTURE: the C file is compiled once per process into a temporary directory."""
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
REF_CLI = ROOT / "oracle" / "_ref" / "csdr_ref"
sys.path.insert(0, str(ROOT))

FIGS, LTRS = 27, 31
BAUD, SHIFT = 45.45, 170.0

_lib = None
_ref = None
_ora = None


def lib():
    global _lib
    if _lib is None:
        out = Path(tempfile.mkdtemp(prefix="rtty_oracle_")) / "librtty_oracle.so"
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(out),
                        str(HERE / "rtty_oracle.c"), "-lm"], check=True)
        L = C.CDLL(str(out))
        vp, fl, it = C.c_void_p, C.c_float, C.c_int
        L.rtty_oracle_serial_line_decoder.argtypes = [vp, vp, it, fl, it, fl, fl, vp]
        L.rtty_oracle_baudot_lookup.argtypes = [C.POINTER(C.c_ubyte), C.c_ubyte]
        L.rtty_oracle_baudot_decode.argtypes = [vp, it, vp, C.POINTER(C.c_ubyte)]
        _lib = L
    return _lib


def _p(a):
    return C.c_void_p(a.ctypes.data)


def _f(x):
    return np.ascontiguousarray(x, np.float32)


def max_outputs(n, spb, databits, stopbits):
    """the characters n samples can hold at most: n / floor(all_bits*spb) + 1, all_bits*spb in float as the decoder forms it"""
    span = np.float32(spb) * (np.float32(1 + databits) + np.float32(stopbits))
    return int(n) // int(span) + 1


# ---- the checker --------------------------------------------------------------------------------------------------------------------
def serial_line_decoder(x, spb, databits=8, stopbits=1.0, ratio=0.4):
    """one call: (codes, input_used)"""
    x = _f(x); n = x.size
    out = np.zeros(max(n, 1), np.uint8); st = np.zeros(2, np.int32)
    xp = _p(x) if n else _p(np.zeros(1, np.float32))
    lib().rtty_oracle_serial_line_decoder(xp, _p(out), n, spb, databits, stopbits, ratio, _p(st))
    return out[:st[0]].tobytes(), int(st[1])


def serial_stream(x, spb, databits=8, stopbits=1.0, ratio=0.4, bufsize=16384, start=0, end=None):
    """calls of exactly bufsize samples over x[start:end] while at least bufsize remain, each starting where the previous one's input_used
    ends (the CLI's memmove-and-refill framing): (codes, new start, stuck)"""
    x = _f(x); end = x.size if end is None else end
    codes, pos = b"", start
    while end - pos >= bufsize:
        c, used = serial_line_decoder(x[pos:pos + bufsize], spb, databits, stopbits, ratio)
        if used == 0:
            return codes, pos, True
        codes += c; pos += used
    return codes, pos, False


def baudot_lookup(code, fig_mode=0):
    m = C.c_ubyte(fig_mode)
    ch = lib().rtty_oracle_baudot_lookup(C.byref(m), code)
    return ch, m.value


def baudot_decode(codes, fig_mode=0):
    """(text, fig_mode)"""
    b = np.frombuffer(bytes(codes), np.uint8).copy() if not isinstance(codes, np.ndarray) else np.ascontiguousarray(codes, np.uint8)
    out = np.zeros(max(b.size, 1), np.uint8); m = C.c_ubyte(fig_mode)
    n = lib().rtty_oracle_baudot_decode(_p(b) if b.size else None, b.size, _p(out), C.byref(m))
    return out[:n].tobytes(), m.value


def oracle():
    global _ora
    if _ora is None:
        from oracle.pyoracle import Oracle
        _ora = Oracle()
    return _ora


def discriminator(z):
    """fmdemod_quadri_cf of the checker (oracle/oracle.c) over the whole stream"""
    return oracle().fmdemod_quadri_cf(np.ascontiguousarray(z, np.complex64))[0]


def chain(z, spb, databits=5, stopbits=1.5, bufsize=16384):
    """fmdemod_quadri_cf | serial_line_decoder_f_u8 spb databits stopbits | rtty_baudot2ascii_u8_u8 over the stream z, the decoder
    framed in calls of bufsize samples"""
    codes, _, _ = serial_stream(discriminator(z), spb, databits, stopbits, 0.4, bufsize)
    return baudot_decode(codes)[0]


# ---- the compiled reference ---------------------------------------------------------------------------------------------------------
class _Serial(C.Structure):              # serial_line_t (libcsdr.h:278-286)
    _fields_ = [("samples_per_bits", C.c_float), ("databits", C.c_int), ("stopbits", C.c_float), ("output_size", C.c_int),
                ("input_used", C.c_int), ("bit_sampling_width_ratio", C.c_float)]


def have_ref() -> bool:
    return REF_SO.exists()


def ref():
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_SO))
        L.serial_line_decoder_f_u8.argtypes = [C.POINTER(_Serial), C.c_void_p, C.c_void_p, C.c_int]
        L.rtty_baudot_decoder_lookup.argtypes = [C.POINTER(C.c_ubyte), C.c_ubyte]; L.rtty_baudot_decoder_lookup.restype = C.c_ubyte
        _ref = L
    return _ref


def ref_serial_line_decoder(x, spb, databits=8, stopbits=1.0, ratio=0.4):
    x = _f(x); n = x.size
    out = np.zeros(max(n, 1), np.uint8)
    s = _Serial(spb, databits, stopbits, 0, 0, ratio)
    ref().serial_line_decoder_f_u8(C.byref(s), _p(x) if n else _p(np.zeros(1, np.float32)), _p(out), n)
    return out[:s.output_size].tobytes(), s.input_used


def ref_baudot_lookup(code, fig_mode=0):
    m = C.c_ubyte(fig_mode)
    ch = ref().rtty_baudot_decoder_lookup(C.byref(m), code)
    return ch, m.value


# ---- a seeded RTTY signal -----------------------------------------------------------------------------------------------------------
_LETTERS = "\0T\rO HNM\nLRGIPCVEZDBSYFXAWJ\0UQK\0"
_FIGURES = "\x005\r9 $,.\n)4*80:=3+#?'6@/-2\a\x0071(\0"
assert len(_LETTERS) == 32 and len(_FIGURES) == 32


def ita2_encode(text: bytes):
    """ITA2 codes for text (upper case letters, digits, punctuation, space, CR, LF), with LTRS/FIGS shifts where the mode changes; a LTRS
    first, like a transmitter starting up"""
    codes, fig = [LTRS], False
    for ch in text.decode("ascii"):
        in_l, in_f = ch in _LETTERS[1:27] + _LETTERS[28:31], ch in _FIGURES[1:27] + _FIGURES[28:31]
        if not (in_l or in_f):
            raise ValueError(f"{ch!r} has no ITA2 code")
        if in_l and in_f:                                                   # space, CR, LF: either mode
            codes.append(_LETTERS.index(ch))
        elif in_l:
            if fig:
                codes.append(LTRS); fig = False
            codes.append(_LETTERS.index(ch))
        else:
            if not fig:
                codes.append(FIGS); fig = True
            codes.append(_FIGURES.index(ch))
    return codes


def bits_of_codes(codes, stopbits=1.5, gap=0.0):
    """(level, length in bits) runs: start bit 0, five data bits first-sent-most-significant (the order the decoder assembles), stop 1 for
    stopbits + gap bits"""
    runs = []
    for c in codes:
        runs.append((0, 1.0))
        runs += [((c >> (4 - k)) & 1, 1.0) for k in range(5)]
        runs.append((1, stopbits + gap))
    return runs


def modulate(text: bytes, spb, rng, freq=0.0, noise=0.01, amplitude=0.3, lead_bits=20.0, tail_bits=20.0, stopbits=1.5, gap=2.0):
    """continuous-phase FSK at spb samples per bit: mark (1) at +shift/2, space (0) at -shift/2, the shift 170/45.45 bit rates; an idle
    mark of lead_bits before the text and tail_bits after it; a carrier offset of `freq` cycles per sample and complex Gaussian noise.
    `gap` samples of mark follow every stop bit: serial_line_decoder_f_u8 consumes exactly (1 + 5 + stopbits)*spb samples from the first
    negative sample of a start bit, so without a gap the next start bit's first negative sample is the first sample of what remains, where
    the decoder's edge search (from its second sample) cannot see it (DESIGN.md section 7)"""
    runs = [(1, lead_bits)] + bits_of_codes(ita2_encode(text), stopbits, gap / spb) + [(1, tail_bits)]
    edges = np.round(np.cumsum([0.0] + [r[1] * spb for r in runs])).astype(np.int64)
    level = np.empty(edges[-1], np.float64)
    for (b, _), a, e in zip(runs, edges[:-1], edges[1:]):
        level[a:e] = 1.0 if b else -1.0
    dev = 0.5 * SHIFT / BAUD / spb                                          # cycles per sample
    phase = 2 * np.pi * np.cumsum(freq + dev * level) + rng.uniform(0, 2 * np.pi)
    n = level.size
    z = amplitude * np.exp(1j * phase) + noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return z.astype(np.complex64)
