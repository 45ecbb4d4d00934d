"""CPU tier: csdr-bankd's AM and SSB tails on the emulated library, with two pretend devices for --devices -- the test bodies of
tests/test_gpu_zzz_bankd_am_ssb.py.  The usb/lsb bandpass reference is the emulated library's own csdrb_bandpass_fir_fft_bank_cc."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_am_ssb as g  # noqa: E402

_emul = {}


def emul_bandpass(bb, lo, hi):
    L = _emul["lib"]
    vp = C.c_void_p
    T = L.firdes_filter_len(C.c_float(g.SSB_BW))
    N = 1 << (T - 1).bit_length()
    if N - T < 200:
        N <<= 1
    isz = N - T + 1
    taps = np.zeros(N, np.complex64)
    L.firdes_bandpass_c.argtypes = [vp, C.c_int, C.c_float, C.c_float, C.c_int]
    L.firdes_bandpass_c(taps.ctypes.data, T, lo, hi, 2)                       # WINDOW_HAMMING
    tf = np.zeros(N, np.complex64)
    L.csdrb_fft_c2c_batch.argtypes = [vp, C.c_long, vp, C.c_long, C.c_int, C.c_int, C.c_int, vp]
    assert L.csdrb_fft_c2c_batch(taps.ctypes.data, N, tf.ctypes.data, N, N, 1, 0, None) >= 0
    ch, nb = bb.shape[0], bb.shape[1] // isz
    x = np.ascontiguousarray(bb[:, :nb * isz]); y = np.zeros_like(x); tail = np.zeros((ch, N), np.complex64)
    L.csdrb_bandpass_fir_fft_bank_cc.argtypes = [vp, C.c_long, vp, C.c_long, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_long, vp, vp]
    assert L.csdrb_bandpass_fir_fft_bank_cc(x.ctypes.data, x.shape[1], y.ctypes.data, y.shape[1], ch, N, isz, nb, tf.ctypes.data, 0, tail.ctypes.data, None) >= 0
    return y


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(base, "MULTI_DEVICES", lambda: ["0", "0,1"]), (_emul, "lib", C.CDLL(str(lib))),
                                                                             (g, "BANDPASS", emul_bandpass)])


test_am_ssb_tails_equal_the_oracle_on_the_banks_baseband = g.test_am_ssb_tails_equal_the_oracle_on_the_banks_baseband
test_am_ssb_tails_over_several_devices = g.test_am_ssb_tails_over_several_devices
