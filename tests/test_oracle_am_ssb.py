"""Pins the CPU restatement of amdemod_cf, fastdcblock_ff and agc_ff (tests/am_ssb/am_ssb_oracle.c) against the compiled, unmodified
reference (oracle/_ref/libcsdr_ref.so, its -O3 -ffast-math build): bit for bit for agc_ff and fastdcblock_ff, within a measured ulp bound
for amdemod_cf (the reference build takes that square root with rsqrtps + one Newton step, whose bits depend on the CPU vendor)."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent / "am_ssb"))
import am_ssb  # noqa: E402

# amdemod_cf: largest distance, in float32 ulp, between the reference build and the correctly rounded sqrt(i*i + q*q), measured on
# an x86-64 CPU over 10^6 random samples spanning 2^-60 .. 2^60 in magnitude: 61 % equal, 37 % 1 ulp, 1.8 % 2 ulp, 0.02 % 3 ulp,
# none further, at every scale tried (2^-8..2^8, 2^-20..2^20, 2^-60..2^60)
AMDEMOD_ULP = 3


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


@pytest.fixture(scope="module")
def R(ref):
    L = ref.L
    fp = C.POINTER(C.c_float)
    L.amdemod_cf.argtypes = [fp, fp, C.c_int]; L.amdemod_cf.restype = None
    L.fastdcblock_ff.argtypes = [fp, fp, C.c_int, C.c_float]; L.fastdcblock_ff.restype = C.c_float
    L.agc_ff.argtypes = [fp, fp, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_short, C.c_short, C.c_float, C.c_float]
    L.agc_ff.restype = C.c_float
    return L


def ref_agc_stream(R, x, chunk, last_gain=1.0, **kw):
    p = dict(am_ssb.AGC_DEFAULTS, **kw)
    x = np.ascontiguousarray(x, np.float32); y = np.empty_like(x)
    for s in range(0, x.size, chunk):
        n = min(chunk, x.size - s)
        last_gain = R.agc_ff(_fp(x[s:]), _fp(y[s:]), n, p["reference"], p["attack_rate"], p["decay_rate"], p["max_gain"],
                             p["hang_time"], p["attack_wait"], p["alpha"], last_gain)
    return y, float(np.float32(last_gain))


def ulp_distance(a, b):
    ia = a.view(np.int32).astype(np.int64); ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7fffffff), ia); ib = np.where(ib < 0, -(ib & 0x7fffffff), ib)
    return np.abs(ia - ib)


def test_amdemod_within_ulp_bound(R):
    rng = np.random.default_rng(1)
    n = 1_000_003
    mag = np.exp2(rng.uniform(-60, 60, n)); ph = rng.uniform(0, 2 * np.pi, n)
    iq = (mag * np.exp(1j * ph)).astype(np.complex64)
    iq[:7] = [0, 1, 1j, -3 + 4j, 1e-30, 3e18 + 4e18j, -0.0]
    want = np.empty(n, np.float32)
    R.amdemod_cf(_fp(iq.view(np.float32)), _fp(want), n)
    got = am_ssb.amdemod_cf(iq)
    d = ulp_distance(got, want)
    assert d.max() <= AMDEMOD_ULP, (d.max(), int(np.argmax(d)))
    # the oracle is the correctly rounded sqrt of the float32 sum of float32 products (numpy's float32 ops are IEEE round-to-nearest)
    i, q = iq.real.astype(np.float32), iq.imag.astype(np.float32)
    assert np.array_equal(got, np.sqrt(i * i + q * q))


@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 6, 7, 8, 9, 13, 1023, 1024, 1025, 1026, 1027, 4096, 777])
@pytest.mark.parametrize("inplace", [False, True])
def test_fastdcblock_bit_exact(R, n, inplace):
    rng = np.random.default_rng(n)
    last = np.float32(0.0)
    for rep in range(4):
        x = (rng.standard_normal(n) * (10.0 ** rep) + rng.uniform(-5, 5)).astype(np.float32)
        if rep == 3:
            x[::3] = 0.0
        want_in = x.copy(); want = want_in if inplace else np.empty_like(x)
        avg_ref = R.fastdcblock_ff(_fp(want_in), _fp(want), n, float(last))
        got, avg = am_ssb.fastdcblock_ff(x, float(last))
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), (n, rep)
        assert np.float32(avg_ref).view(np.int32) == np.float32(avg).view(np.int32)
        last = np.float32(avg)


AGC_CASES = {
    "defaults": {},
    "fast_attack_wait": dict(attack_rate=0.2, decay_rate=0.01, attack_wait=5, hang_time=30),
    "max_gain_hit": dict(max_gain=40.0, decay_rate=0.05),
    "long_hang": dict(hang_time=1500, attack_rate=0.05),
    "alpha_small": dict(alpha=0.05, reference=0.7),
    "negative_counts": dict(hang_time=-3, attack_wait=-2),
}


def agc_signal(rng, n):
    """bursts, silence (exact zeros), a slow fade and a spike: drives the gain to max_gain and back"""
    t = np.arange(n)
    x = (0.3 * np.sin(2 * np.pi * t / 37.0) * (1 + 0.9 * np.sin(2 * np.pi * t / 5000.0))).astype(np.float32)
    x += (0.01 * rng.standard_normal(n)).astype(np.float32)
    x[n // 5: n // 5 + 3000] = 0.0                                  # silence: gain climbs to max_gain
    x[n // 2: n // 2 + 400] *= 40.0                                  # burst
    x[n // 2 + 2000] = 7.0                                           # spike
    x[n // 3: n // 3 + 800] *= 1e-4                                  # deep fade
    x[rng.integers(0, n, n // 50)] = 0.0                             # isolated zero samples
    return x


@pytest.mark.parametrize("case", sorted(AGC_CASES))
@pytest.mark.parametrize("chunk", [1024, 1000, 257])
def test_agc_bit_exact(R, case, chunk):
    rng = np.random.default_rng(len(case) * 1000 + chunk)
    x = agc_signal(rng, 23_457)
    kw = AGC_CASES[case]
    want, gw = ref_agc_stream(R, x, chunk, **kw)
    got, gg = am_ssb.agc_stream(x, chunk, **kw)
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), (case, chunk, int(np.argmax(got.view(np.int32) != want.view(np.int32))))
    assert np.float32(gw).view(np.int32) == np.float32(gg).view(np.int32)


def test_agc_special_values(R):
    """NaN and infinities go through the same branches as in the reference build; gain 0 makes last_peak infinite"""
    rng = np.random.default_rng(7)
    x = agc_signal(rng, 5000)
    x[100] = np.nan; x[200] = np.inf; x[300] = -np.inf; x[301:305] = -0.0
    for lg in (1.0, 0.0, 3.5):
        want, gw = ref_agc_stream(R, x, 1024, last_gain=lg, max_gain=100.0)
        got, gg = am_ssb.agc_stream(x, 1024, last_gain=lg, max_gain=100.0)
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), lg


def test_agc_gain_reaches_max(R):
    """silence drives the gain to max_gain: the clamp is active in the pinned run"""
    x = np.zeros(20_000, np.float32); x[:50] = 0.1; x[-50:] = 0.1
    y, g = am_ssb.agc_stream(x, 1024, max_gain=200.0, decay_rate=0.01, alpha=0.9)
    want, gw = ref_agc_stream(R, x, 1024, max_gain=200.0, decay_rate=0.01, alpha=0.9)
    assert np.array_equal(y.view(np.int32), want.view(np.int32))
    assert g > 200.0                                                 # the fixed point of the zero-input path is max_gain / alpha
