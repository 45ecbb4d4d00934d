"""The two CPU checkers of rational_resampler_ff (TEST INFRASTRUCTURE):

* ``Oracle`` -> resampler_oracle.c, the strict-IEEE restatement in the reference's loop order (compiled once per process into a temporary
  directory), bit-exact target of the GPU bank;
* ``Ref``    -> the compiled, unmodified reference library oracle/_ref/libcsdr_ref.so (vectorised under -ffast-math: not bit-exact with the
  sequential order, compared within 1e-5 relative RMS).

Both return (y, state) for one call, state = (input_processed, output_size, last_taps_delay), and replay the CLI loop (csdr.c:1448-1461) with
``stream``.
"""
from __future__ import annotations

import ctypes as C
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
WINDOWS = {"BOXCAR": 0, "BLACKMAN": 1, "HAMMING": 2}


class _State(C.Structure):              # libcsdr.h:132-137
    _fields_ = [("input_processed", C.c_int), ("output_size", C.c_int), ("last_taps_delay", C.c_int)]


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def lowpass(oracle, T, I, D, window="HAMMING"):
    """rational_resampler_get_lowpass_f (libcsdr.c:665-673) on the oracle's firdes_lowpass_f"""
    cutoff = min(np.float32(1.0 / I), np.float32(1.0 / D))
    return oracle.firdes_lowpass_f(T, float(np.float32(cutoff / np.float32(2))), window)


class _Base:
    def rational_resampler_ff(self, x, I, D, taps, ltd=0):
        x = np.ascontiguousarray(x, np.float32); taps = np.ascontiguousarray(taps, np.float32)
        y = np.zeros(max(x.size * I // D, 1), np.float32)
        st = self._call(x, y, x.size, I, D, taps, ltd)
        return y[:st[1]].copy(), st

    def stream(self, x, I, D, taps, block):
        """the CLI loop over x: first call on `block` samples, later ones on the unconsumed tail plus input_processed new samples; complete reads only"""
        x = np.ascontiguousarray(x, np.float32); taps = np.ascontiguousarray(taps, np.float32)
        buf = np.zeros(block, np.float32); out = np.zeros(max(block * I // D, 1), np.float32)
        ip, ltd, pos, outs = 0, 0, 0, []
        while True:
            need = block if ip == 0 else ip
            if ip:
                buf[:block - ip] = buf[ip:].copy()
            if pos + need > x.size:
                break
            buf[block - need:] = x[pos:pos + need]; pos += need
            ip, n, ltd = self._call(buf, out, block, I, D, taps, ltd)
            outs.append(out[:n].copy())
        return np.concatenate(outs) if outs else np.zeros(0, np.float32)


class Oracle(_Base):
    name = "oracle"
    _lib = None

    def __init__(self):
        if Oracle._lib is None:
            so = Path(tempfile.mkdtemp(prefix="resampler_oracle_")) / "libresampler_oracle.so"
            subprocess.run(["gcc", "-std=gnu99", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(so),
                            str(HERE / "resampler_oracle.c")], check=True)
            L = C.CDLL(str(so))
            fp = C.POINTER(C.c_float)
            L.rs_oracle_rational_resampler_ff.argtypes = [fp, fp, C.c_int, C.c_int, C.c_int, fp, C.c_int, C.c_int, C.POINTER(C.c_int)]
            L.rs_oracle_cap_endings.argtypes = [C.c_int] * 4; L.rs_oracle_cap_endings.restype = C.c_long
            Oracle._lib = L

    def _call(self, x, y, n, I, D, taps, ltd):
        st = (C.c_int * 3)()
        self._lib.rs_oracle_rational_resampler_ff(_fp(x), _fp(y), n, I, D, _fp(taps), taps.size, ltd, st)
        return tuple(st)


    def cap_endings(self, I, D, T, n_max):
        """calls of 0..n_max inputs (every last_taps_delay) that end on the output cap, from the reference loop on indices"""
        return int(self._lib.rs_oracle_cap_endings(I, D, T, n_max))


class Ref(_Base):
    name = "reference"
    SO = ROOT / "oracle" / "_ref" / "libcsdr_ref.so"

    def __init__(self):
        if not self.SO.exists():
            raise FileNotFoundError(f"{self.SO} missing (built where the reference sources are available)")
        L = self.L = C.CDLL(str(self.SO))
        fp = C.POINTER(C.c_float)
        L.rational_resampler_ff.argtypes = [fp, fp, C.c_int, C.c_int, C.c_int, fp, C.c_int, C.c_int]
        L.rational_resampler_ff.restype = _State
        L.rational_resampler_get_lowpass_f.argtypes = [fp, C.c_int, C.c_int, C.c_int, C.c_int]

    def _call(self, x, y, n, I, D, taps, ltd):
        st = self.L.rational_resampler_ff(_fp(x), _fp(y), n, I, D, _fp(taps), taps.size, ltd)
        return st.input_processed, st.output_size, st.last_taps_delay

    def lowpass(self, T, I, D, window="HAMMING"):
        t = np.empty(T, np.float32)
        self.L.rational_resampler_get_lowpass_f(_fp(t), T, I, D, WINDOWS[window]); return t


def have_ref() -> bool:
    return Ref.SO.exists()
