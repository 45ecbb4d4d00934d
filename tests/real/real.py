"""Checkers of the real-input shift: ctypes front-end of real_oracle.c (oracle_shift_addition_fc, our C restatement) and a binding of the same
function in the compiled reference (oracle/_ref/libcsdr_ref.so).  TEST INFRASTRUCTURE: the C file is compiled once per process into a temporary
directory."""
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
sys.path.insert(0, str(ROOT))


class _Shift(C.Structure):
    _fields_ = [("sindelta", C.c_float), ("cosdelta", C.c_float), ("rate", C.c_float)]


_libs = {}


def _oracle_lib():
    if "oracle" not in _libs:
        out = Path(tempfile.mkdtemp(prefix="real_oracle_")) / "libreal_oracle.so"
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(out),
                        str(HERE / "real_oracle.c"), "-lm"], check=True)
        L = C.CDLL(str(out))
        L.oracle_shift_addition_fc.argtypes = [C.c_void_p, C.c_void_p, C.c_int, _Shift, C.c_float, C.c_int]
        L.oracle_shift_addition_fc.restype = C.c_float
        _libs["oracle"] = L
    return _libs["oracle"]


def have_ref() -> bool:
    return REF_SO.exists()


def _ref_lib():
    if "ref" not in _libs:
        L = C.CDLL(str(REF_SO))
        L.shift_addition_init.argtypes = [C.c_float]; L.shift_addition_init.restype = _Shift
        L.shift_addition_fc.argtypes = [C.c_void_p, C.c_void_p, C.c_int, _Shift, C.c_float]; L.shift_addition_fc.restype = C.c_float
        _libs["ref"] = L
    return _libs["ref"]


def shift_init(rate):
    """the deltas the product computes on the host (shift_addition_init, bit for bit the reference's: tests/test_oracle.py)"""
    from oracle.pyoracle import Oracle
    s, c, r = Oracle().shift_addition_init(float(rate))
    return _Shift(s, c, r)


def shift_addition_fc(x, rate, phase=0.0, chunk=None, ref=False, build_seed=False):
    """real x -> (complex64 y, float32 phase): one shift_addition_fc call per `chunk` samples (None: one call), by the C restatement or the reference.
    The restatement seeds every call with cos/sin in double (the source, the banks) or, with build_seed, with sincosf (the reference build, the drop-in)."""
    x = np.ascontiguousarray(x, np.float32)
    y = np.empty(x.size, np.complex64)
    if ref:
        L = _ref_lib(); fn = L.shift_addition_fc; d = L.shift_addition_init(float(rate))
    else:
        o = _oracle_lib().oracle_shift_addition_fc; d = shift_init(rate)
        fn = lambda a, b, n, d, ph: o(a, b, n, d, ph, 1 if build_seed else 0)
    chunk = chunk or max(x.size, 1)
    ph = float(phase)
    for s in range(0, x.size, chunk):
        n = min(chunk, x.size - s)
        ph = fn(x[s:].ctypes.data, y[s:].ctypes.data, n, d, ph)
    return y, np.float32(ph)


def cli_stream(x, rate, block=16384, call=1024):
    """what `csdr shift_addition_fc RATE` (and the reference CLI) writes for the real stream x: blocks of `block` samples, each cut into calls of `call`; a short last
    block is processed whole, its tail the previous block's stale samples (the reference reads into the same buffer and tests EOF before the read)"""
    x = np.ascontiguousarray(x, np.float32)
    buf = np.zeros(block, np.float32)
    out = []
    ph = np.float32(0.0)
    for s in range(0, x.size, block):
        part = x[s:s + block]
        buf[:part.size] = part
        y, ph = shift_addition_fc(buf, rate, ph, call, build_seed=True)
        out.append(y)
    return np.concatenate(out) if out else np.zeros(0, np.complex64)
