"""ctypes front-end of am_ssb_oracle.c (the CPU restatement of amdemod_cf, fastdcblock_ff and agc_ff) plus the stream drivers
the reference CLI applies to them.  TEST INFRASTRUCTURE: the C file is compiled once per process into a temporary directory."""
from __future__ import annotations

import ctypes as C
import subprocess
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent

# agc_ff CLI defaults, csdr.c:1342-1361: hang_time, reference, attack_rate, decay_rate, max_gain, attack_wait, filter_alpha
AGC_DEFAULTS = dict(hang_time=200, reference=0.2, attack_rate=0.01, decay_rate=0.0001, max_gain=65536.0, attack_wait=0, alpha=0.999)

_lib = None


def lib():
    global _lib
    if _lib is None:
        out = Path(tempfile.mkdtemp(prefix="am_ssb_oracle_")) / "libam_ssb_oracle.so"
        subprocess.run(["gcc", "-std=gnu99", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-shared", "-o", str(out),
                        str(HERE / "am_ssb_oracle.c"), "-lm"], check=True)
        L = C.CDLL(str(out))
        fp = C.POINTER(C.c_float)
        L.am_oracle_amdemod_cf.argtypes = [fp, fp, C.c_int]
        L.am_oracle_fastdcblock_ff.argtypes = [fp, fp, C.c_int, C.c_float]; L.am_oracle_fastdcblock_ff.restype = C.c_float
        L.am_oracle_agc_ff.argtypes = [fp, fp, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_short, C.c_short, C.c_float, C.c_float]
        L.am_oracle_agc_ff.restype = C.c_float
        _lib = L
    return _lib


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def amdemod_cf(x):
    x = np.ascontiguousarray(x, np.complex64); y = np.empty(x.size, np.float32)
    lib().am_oracle_amdemod_cf(_fp(x.view(np.float32)), _fp(y), x.size); return y


def fastdcblock_ff(x, last_dc=0.0):
    """one call on one block: (y, avg)"""
    x = np.ascontiguousarray(x, np.float32); y = np.empty_like(x)
    avg = lib().am_oracle_fastdcblock_ff(_fp(x), _fp(y), x.size, last_dc); return y, float(np.float32(avg))


def fastdcblock_stream(x, block=1024, last_dc=0.0):
    """the CLI loop (csdr.c:952-968) over the whole blocks of x: (y, last_dc)"""
    x = np.ascontiguousarray(x, np.float32); nb = x.size // block
    y = np.empty(nb * block, np.float32)
    for b in range(nb):
        y[b * block:(b + 1) * block], last_dc = fastdcblock_ff(x[b * block:(b + 1) * block], last_dc)
    return y, last_dc


def agc_ff(x, last_gain=1.0, **kw):
    """one call: (y, gain)"""
    p = dict(AGC_DEFAULTS, **kw)
    x = np.ascontiguousarray(x, np.float32); y = np.empty_like(x)
    g = lib().am_oracle_agc_ff(_fp(x), _fp(y), x.size, p["reference"], p["attack_rate"], p["decay_rate"], p["max_gain"],
                               p["hang_time"], p["attack_wait"], p["alpha"], last_gain)
    return y, float(np.float32(g))


def agc_stream(x, chunk=1024, last_gain=1.0, **kw):
    """the CLI loop (csdr.c:1363-1372): one agc_ff call per `chunk` samples from stream start (the last one may be short): (y, gain)"""
    x = np.ascontiguousarray(x, np.float32); y = np.empty_like(x)
    for s in range(0, x.size, chunk):
        y[s:s + chunk], last_gain = agc_ff(x[s:s + chunk], last_gain, **kw)
    return y, last_gain


def agc_tail(x, oracle, chunk=1024, limit=0.0, s16=False, **kw):
    """[realpart_cf |] agc_ff [| limit_ff limit] [| convert_f_s16] on one channel; complex input takes the real part"""
    x = np.asarray(x)
    if np.iscomplexobj(x):
        x = np.ascontiguousarray(x.real, np.float32)
    y, _ = agc_stream(x, chunk, **kw)
    if limit > 0:
        y = oracle.limit_ff(y, limit)
    return oracle.convert_f_s16(y) if s16 else y


def am_front(iq, block=1024, last_dc=0.0):
    """amdemod_cf | fastdcblock_ff block over the whole blocks of one channel: (y, last_dc)"""
    return fastdcblock_stream(amdemod_cf(iq), block, last_dc)
