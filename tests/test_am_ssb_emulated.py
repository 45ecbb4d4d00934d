"""CPU tier for the AM / SSB receiver kernels (csdr_b200/csrc/agc.cu): the shipped kernels and launchers run thread by thread under
tests/host_shim/cuda_emul.h (see tests/test_kernels_emulated.py) and must equal the CPU restatement tests/am_ssb/am_ssb_oracle.c bit for
bit -- channel counts that are not multiples of 32, row strides, block sizes with remainders mod 4, and streams cut into calls of random
sizes, which must equal one long call.  Every test runs under three fiber scheduling orders."""
import ctypes as C
import os
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "am_ssb"))
import am_ssb  # noqa: E402
import emul_build  # noqa: E402

ORDERS = ["alternate", "reverse", "random"]
_built = {}
GUARD = 256


@pytest.fixture(scope="module", params=ORDERS)
def agc(request, tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    if "agc" not in _built:
        lib, names = emul_build.build_file(tmp_path_factory.mktemp("emul_agc"), "agc.cu")
        _built["agc"] = (Path(lib._name), names, lib)
    so, names, proto = _built["agc"]
    copy = so.with_name(f"{so.stem}_{request.param}.so")
    if not copy.exists():
        shutil.copy(so, copy)
    os.environ["CUDA_EMUL_ORDER"] = request.param
    lib = C.CDLL(str(copy))
    for n in names:
        f, g = getattr(lib, "emul_" + n), getattr(proto, "emul_" + n)
        f.argtypes, f.restype = g.argtypes, g.restype
    lib.emul_last_error.restype = C.c_char_p
    return lib


class Guarded:
    """a zeroed array with canary bytes before and after it, 16-byte aligned; check() fails on an out-of-bounds write"""

    def __init__(self, shape, dtype):
        self.n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        self.raw = np.full(self.n + 2 * GUARD + 16, 0xA5, np.uint8)
        off = GUARD + (-(self.raw.ctypes.data + GUARD) % 16)
        self.off = off
        self.raw[off:off + self.n] = 0
        self.a = self.raw[off:off + self.n].view(dtype).reshape(shape)

    def check(self):
        assert np.all(self.raw[:self.off] == 0xA5) and np.all(self.raw[self.off + self.n:] == 0xA5), "write outside the array"


def P(a):
    return a.ctypes.data


def agc_params(chunk=1024, **kw):
    p = dict(am_ssb.AGC_DEFAULTS, **kw)
    return np.array([(p["reference"], p["attack_rate"], p["decay_rate"], p["max_gain"], p["hang_time"], p["attack_wait"], p["alpha"], chunk)],
                    dtype=[("r", "<f4"), ("a", "<f4"), ("d", "<f4"), ("m", "<f4"), ("h", "<i4"), ("w", "<i4"), ("al", "<f4"), ("c", "<i4")])


def agc_state0(ch):
    st = np.zeros((ch, 5), np.int32)
    st[:, 0] = np.array([1.0], np.float32).view(np.int32)[0]
    return st


def test_amdemod_elementwise(agc):
    rng = np.random.default_rng(3)
    n = 1237
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64) * np.float32(50)
    x[:3] = [0, -0.0, 3 + 4j]
    y = Guarded(n, np.float32)
    assert agc.emul_launch_amdemod_cf(P(x), P(y.a), n) >= 0
    y.check()
    assert np.array_equal(y.a, am_ssb.amdemod_cf(x))


@pytest.mark.parametrize("block,cf32", [(1, True), (3, False), (5, True), (6, False), (7, True), (64, True), (1024, True), (1027, False)])
def test_fastdcblock_bank_stream(agc, block, cf32):
    """two bank calls (8 + 11 blocks: runs of 8 with the lead-in block) equal the CLI loop over all 19 blocks; rows have a stride"""
    rng = np.random.default_rng(block)
    ch, nb = 5, 19
    n = nb * block
    stride = n + 9
    if cf32:
        x = (rng.standard_normal((ch, stride)) + 1j * rng.standard_normal((ch, stride))).astype(np.complex64) + np.complex64(0.3 + 0.1j)
    else:
        x = (rng.standard_normal((ch, stride)) + 2.0).astype(np.float32)
    x[:, 2 * block: 2 * block + 7] = 0
    out = Guarded((ch, stride + 3), np.float32)
    last = Guarded(ch, np.float32)
    last.a[:] = np.linspace(-1, 1, ch, dtype=np.float32)
    want = []
    for c in range(ch):
        src = am_ssb.amdemod_cf(x[c, :n]) if cf32 else x[c, :n]
        want.append(am_ssb.fastdcblock_stream(src, block, float(last.a[c])))
    esz = x.itemsize
    for b0, nbl in ((0, 8), (8, 11)):
        rc = agc.emul_launch_fastdcblock_bank(P(x) + b0 * block * esz, stride, int(cf32), P(out.a) + b0 * block * 4, stride + 3, ch, block, nbl, P(last.a))
        assert rc >= 0, agc.emul_last_error()
    out.check(); last.check()
    for c in range(ch):
        assert np.array_equal(out.a[c, :n].view(np.int32), want[c][0].view(np.int32)), c
        assert np.float32(want[c][1]).view(np.int32) == last.a[c:c + 1].view(np.int32)[0]
        assert np.all(out.a[c, n:] == 0)


AGC_CASES = [
    dict(),
    dict(attack_rate=0.2, decay_rate=0.01, attack_wait=5, hang_time=30, alpha=0.9),
    dict(max_gain=40.0, decay_rate=0.05, hang_time=1500),
]


@pytest.mark.parametrize("case", range(len(AGC_CASES)))
@pytest.mark.parametrize("chunk", [1024, 100, 1])
def test_agc_bank_split_stream(agc, case, chunk):
    """37 channels (two CTAs, the second one partly empty), a stream cut into calls of random sizes, equals agc_ff's CLI loop"""
    rng = np.random.default_rng(case * 10 + chunk)
    ch, n = 37, 3111
    stride = n + 5
    x = np.zeros((ch, stride), np.float32)
    for c in range(ch):
        x[c, :n] = am_ssb_signal(rng, n, c)
    kw = AGC_CASES[case]
    p = agc_params(chunk, **kw)
    st = Guarded((ch, 5), np.int32); st.a[:] = agc_state0(ch)
    out = Guarded((ch, stride), np.float32)
    cuts = np.sort(rng.choice(np.arange(1, n), 6, replace=False))
    for s0, s1 in zip(np.r_[0, cuts], np.r_[cuts, n]):
        rc = agc.emul_launch_agc_bank(P(x) + int(s0) * 4, stride, 0, P(out.a) + int(s0) * 4, stride, 0, ch, int(s1 - s0), P(p), P(st.a), 0.0)
        assert rc >= 0, agc.emul_last_error()
    out.check(); st.check()
    for c in range(ch):
        want, g = am_ssb.agc_stream(x[c, :n], chunk, **kw)
        assert np.array_equal(out.a[c, :n].view(np.int32), want.view(np.int32)), (c, int(np.argmax(out.a[c, :n] != want)))
        assert st.a[c, 0] == np.array([g], np.float32).view(np.int32)[0]
        assert st.a[c, 4] == n % chunk


@pytest.mark.parametrize("limit,s16", [(0.0, True), (0.5, True), (0.5, False)])
def test_agc_bank_ssb_tail(agc, oracle, limit, s16):
    """realpart_cf | agc_ff | limit_ff | convert_f_s16 from cf32 rows (the SSB tail), one call"""
    rng = np.random.default_rng(11)
    ch, n = 33, 2500
    x = np.zeros((ch, n), np.complex64)
    for c in range(ch):
        x[c] = am_ssb_signal(rng, n, c) + 1j * rng.standard_normal(n).astype(np.float32)
    p = agc_params(1024)
    st = agc_state0(ch)
    out = Guarded((ch, n), np.int16 if s16 else np.float32)
    assert agc.emul_launch_agc_bank(P(x), n, 1, P(out.a), n, int(s16), ch, n, P(p), P(st), limit) >= 0, agc.emul_last_error()
    out.check()
    for c in range(ch):
        want = am_ssb.agc_tail(x[c], oracle, 1024, limit, s16)
        assert np.array_equal(out.a[c].view(np.uint8), want.view(np.uint8)), c


def am_ssb_signal(rng, n, c):
    t = np.arange(n)
    x = (0.2 * (1 + (c % 5)) * np.sin(2 * np.pi * t / (17.0 + c)) * (1 + 0.8 * np.sin(2 * np.pi * t / 900.0))).astype(np.float32)
    x += (0.003 * rng.standard_normal(n)).astype(np.float32)
    x[n // 4: n // 4 + 400] = 0.0
    x[n // 2: n // 2 + 150] *= 30.0
    x[rng.integers(0, n, n // 40)] = 0.0
    if c == 3:
        x[100] = np.nan; x[200] = np.inf
    return x
