"""CPU tier for the transmit banks (csdr_b200/csrc/interpolate.cu): the shipped kernels and launchers run thread by thread under
tests/host_shim/cuda_emul.h.  fir_interpolate_cc must equal the kernel's summation order restated in tests/tx/tx.py bit for bit and lie within the
float64 per-output bound derived there of the compiled reference; fmmod_fc's phases must equal the reference build's bit for bit, its samples
within one float ulp of the build's sincosf.  Covered: I in {1, 2, 3, 5, 50, 256}, T from 1 past the shared-memory tap tile, the unused tap 0,
n below one group, odd strides and several rows, calls cut with the carry, NaN/Inf locality, the refusals, and the drop-ins of the whole
emulated library."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "tx"))
import emul_build  # noqa: E402
import tx  # noqa: E402

needs_ref = pytest.mark.skipif(not tx.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built")
ULP1 = 2.0 ** -24                                                   # one float ulp of a value in [0.5, 1), more than that of any smaller one


@pytest.fixture(scope="module")
def K(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _ = emul_build.build_file(tmp_path_factory.mktemp("emul_tx"), "interpolate.cu")
    return lib


def P(a):
    return a.ctypes.data


def same_bits(a, b):
    fa, fb = np.asarray(a).view(np.float32), np.asarray(b).view(np.float32)
    na, nb = np.isnan(fa), np.isnan(fb)
    return fa.shape == fb.shape and np.array_equal(na, nb) and np.array_equal(fa[~na].view(np.uint32), fb[~nb].view(np.uint32))


def rows(rng, ch, n):
    return ((rng.standard_normal((ch, n)) + 1j * rng.standard_normal((ch, n))) * 10.0 ** rng.uniform(-3, 3, (ch, 1))).astype(np.complex64)


def interp(K, x, n, I, taps, stride=None, out_stride=None):
    ch = x.shape[0]
    stride = stride or max(n, 1)
    xin = np.zeros((ch, stride), np.complex64); xin[:, :n] = x[:, :n]
    m = tx.groups(n, I, len(taps)) * I
    ostride = out_stride or max(m, 1)
    out = np.full((ch, ostride), np.nan, np.complex64)
    t = np.ascontiguousarray(taps, np.float32)
    rc = K.emul_launch_fir_interpolate_bank_cc(P(xin), stride, P(out), ostride, ch, n, I, P(t), len(t))
    assert rc == m, (rc, m, K.emul_last_error())
    return out[:, :m]


GEOMS = [(1, 1, 40), (1, 7, 300), (2, 2, 5), (2, 81, 500), (3, 1, 9), (3, 81, 700), (5, 4, 3), (5, 801, 900), (50, 401, 120), (50, 49, 60),
         (50, 2001, 100), (256, 81, 30), (256, 2049, 40), (3, 9001, 3500), (50, 8193, 300)]             # the last two: taps past the 8192 staged


def test_interp_bank_equals_restatement(K):
    rng = np.random.default_rng(1)
    for I, T, n in GEOMS:
        ch = 3
        x = rows(rng, ch, n)
        taps = rng.standard_normal(T).astype(np.float32)
        got = interp(K, x, n, I, taps, stride=n + int(rng.integers(0, 4)) | 1, out_stride=tx.groups(n, I, T) * I + int(rng.integers(0, 3)) * 2 + 1)
        for c in range(ch):
            assert same_bits(got[c], tx.fir_interpolate_cc(x[c], I, taps)), (I, T, n, c)


def test_tap_zero_is_never_used_and_short_rows_give_nothing(K):
    rng = np.random.default_rng(2)
    x = rows(rng, 2, 50)
    for I, T in ((1, 5), (3, 10), (50, 120)):
        taps = rng.standard_normal(T).astype(np.float32)
        other = taps.copy(); other[0] = 1e30
        assert same_bits(interp(K, x, 50, I, taps), interp(K, x, 50, I, other)), (I, T)
    for I, T, n in ((3, 10, 3), (50, 401, 8), (1, 5, 4), (5, 6, 0)):
        assert tx.groups(n, I, T) == 0
        out = np.full(4, 7.0, np.complex64)
        assert K.emul_launch_fir_interpolate_bank_cc(P(x), 50, P(out), 0, 2, n, I, P(np.ones(T, np.float32)), T) == 0
        assert np.all(out == 7.0)


@needs_ref
def test_interp_bank_within_bound_of_reference(K):
    rng = np.random.default_rng(3)
    for I, T, n in GEOMS[:13]:
        x = rows(rng, 2, n)
        taps = tx.ref_lowpass(T, 0.5 / I)
        got = interp(K, x, n, I, taps)
        for c in range(2):
            want = tx.ref_fir_interpolate_cc(x[c], I, taps)
            bi, bq = tx.interp_bound(x[c], I, taps)
            assert want.size == got[c].size, (I, T, n)
            assert np.all(np.abs(got[c].real.astype(np.float64) - want.real) <= bi), (I, T, n)
            assert np.all(np.abs(got[c].imag.astype(np.float64) - want.imag) <= bq), (I, T, n)


def test_interp_calls_with_carry_equal_one_call(K):
    """a stream cut into calls, each starting with the inputs the previous one did not consume, gives the bits of one call"""
    rng = np.random.default_rng(4)
    for I, T in ((3, 81), (50, 401), (1, 2)):
        n = 900
        x = rows(rng, 2, n)
        taps = rng.standard_normal(T).astype(np.float32)
        whole = interp(K, x, n, I, taps)
        pieces, pos, keep = [], 0, (T - 1 + I - 1) // I
        while pos + keep < n:
            k = min(n - pos, keep + int(rng.integers(1, 200)))
            part = interp(K, np.ascontiguousarray(x[:, pos:pos + k]), k, I, taps)
            pieces.append(part)
            pos += part.shape[1] // I
        assert same_bits(np.concatenate(pieces, axis=1), whole), (I, T)


def test_interp_nan_and_inf_stay_in_their_windows(K):
    rng = np.random.default_rng(5)
    I, T, n = 5, 41, 300
    x = rows(rng, 3, n)
    taps = rng.uniform(0.1, 1, T).astype(np.float32)
    clean = interp(K, x, n, I, taps)
    bad = x.copy(); spots = {0: (100, np.nan), 1: (150, np.inf), 2: (200, -np.inf)}
    for c, (i, v) in spots.items():
        bad[c, i] = v
    got = interp(K, bad, n, I, taps)
    G = tx.groups(n, I, T)
    for c, (i, v) in spots.items():
        hit = np.zeros((G, I), bool); hit[max(0, i - (T - 1) // I):i + 1] = True
        hit = hit.reshape(-1)
        assert same_bits(got[c][~hit], clean[c][~hit]), c
        assert same_bits(got[c], tx.fir_interpolate_cc(bad[c], I, taps)), c
        assert not np.all(np.isfinite(got[c][hit].view(np.float32))), c


def test_interp_refusals_launch_nothing(K):
    x = np.zeros(64, np.complex64); t = np.ones(8, np.float32); out = np.full(640, 7.0, np.complex64)
    for I, T, n, stride, ostride in ((0, 8, 64, 64, 640), (2, 0, 64, 64, 640), (2, 8, 64, 63, 640), (2, 8, 64, 64, 113)):
        assert K.emul_launch_fir_interpolate_bank_cc(P(x), stride, P(out), ostride, 1, n, I, P(t), T) == -1, (I, T, stride, ostride)
    assert np.all(out == 7.0)


# ---- fmmod_fc --------------------------------------------------------------------------------------------------------------------------
def fmmod(K, x, n, phase, stride=None, out_stride=None):
    ch = x.shape[0]
    stride = stride or max(n, 1)
    xin = np.zeros((ch, stride), np.float32); xin[:, :n] = x[:, :n]
    ostride = out_stride or max(n, 1)
    out = np.full((ch, ostride), np.nan, np.complex64)
    ph = np.ascontiguousarray(phase, np.float32).copy()
    assert K.emul_launch_fmmod_bank_fc(P(xin), stride, P(out), ostride, ch, n, P(ph)) == n, K.emul_last_error()
    return out[:, :n], ph


def fm_inputs(rng, n):
    t = np.arange(n)
    return np.stack([np.linspace(-1, 1, n), np.where(t % 7 < 3, 1.0, -1.0), rng.uniform(-1, 1, n),
                     rng.uniform(-9, 9, n) * (t % 5 == 0), 0.3 * np.sin(2 * np.pi * t / 37.0)]).astype(np.float32)


def test_fmmod_phases_equal_the_build(K):
    """phases bit for bit against the restated build, over ramps, +-1 full scale, and values that wrap several times; each row carries on from
    its own starting phase"""
    rng = np.random.default_rng(6)
    n = 300
    x = fm_inputs(rng, n)
    start = np.array([0, 3.1, -3.14159, 1.0, -2.5], np.float32)
    # row r with its first k samples replaced by zeros after the prefix: the carried phase after a call of k samples is the k-th phase
    for k in (1, 2, 31, 32, 33, 299, 300):
        _, ph = fmmod(K, np.ascontiguousarray(x[:, :k]), k, start)
        for r in range(x.shape[0]):
            assert ph[r] == tx.fmmod_phases(x[r, :k], start[r])[-1], (k, r)


@needs_ref
def test_fmmod_against_reference(K):
    rng = np.random.default_rng(7)
    n = 400
    x = fm_inputs(rng, n)
    got, ph = fmmod(K, x, n, np.zeros(x.shape[0], np.float32), stride=n + 3, out_stride=n + 1)
    for r in range(x.shape[0]):
        phases = tx.ref_fmmod_phases(x[r])
        assert np.array_equal(phases.view(np.uint32), tx.fmmod_phases(x[r]).view(np.uint32)), r
        want, last = tx.ref_fmmod_fc(x[r])
        assert ph[r] == last, r
        assert np.abs(got[r].real - want.real).max() <= ULP1 and np.abs(got[r].imag - want.imag).max() <= ULP1, r
        exact = np.exp(1j * phases.astype(np.float64))
        assert np.abs(got[r] - exact).max() < 1e-7, r


@needs_ref
def test_fmmod_wraps_huge_phases_like_the_reference(K):
    """x*PI in [2^26, 2^27): the float spacing is 8 there, a step of 2*PI still moves the phase (to ph - 8), and the reference's loop ends"""
    x = np.array([[3.0e7, 0.5, -2.2e7, -0.25, 4.1e7, 1.0]], np.float32)
    assert all(2.0 ** 26 <= abs(float(v) * np.pi) < 2.0 ** 27 for v in x[0, [0, 2, 4]])
    want, last = tx.ref_fmmod_fc(x[0])
    got, ph = fmmod(K, x, x.shape[1], np.zeros(1, np.float32))
    assert ph[0] == last and abs(last) <= np.pi
    assert np.abs(got[0].view(np.float32) - want.view(np.float32)).max() <= ULP1


def test_fmmod_phase_carries_over_any_cut(K):
    rng = np.random.default_rng(8)
    n = 500
    x = fm_inputs(rng, n)
    whole, ph_whole = fmmod(K, x, n, np.zeros(5, np.float32))
    pos, ph, parts = 0, np.zeros(5, np.float32), []
    while pos < n:
        k = min(n - pos, int(rng.integers(0, 70)))
        part, ph = fmmod(K, np.ascontiguousarray(x[:, pos:pos + k]), k, ph)
        parts.append(part); pos += k
    assert same_bits(np.concatenate(parts, axis=1), whole) and np.array_equal(ph, ph_whole)


def test_fmmod_nan_stays_in_its_row_and_inf_ends(K):
    x = np.zeros((3, 40), np.float32); x[0, 10] = np.nan; x[1, 5] = np.inf; x[2] = 0.25
    got, ph = fmmod(K, x, 40, np.zeros(3, np.float32))
    assert np.all(np.isnan(got[0, 10:].view(np.float32))) and np.all(np.isfinite(got[0, :10].view(np.float32)))
    assert np.isinf(ph[1]) and np.isfinite(ph[2])                     # the reference never returns from an Inf; the bank carries it on
    assert same_bits(got[2], fmmod(K, x[2:], 40, np.zeros(1, np.float32))[0][0])
    out = np.full(8, 7.0, np.complex64)
    assert K.emul_launch_fmmod_bank_fc(P(x), 39, P(out), 40, 1, 40, P(np.zeros(1, np.float32))) == -1
    assert K.emul_launch_fmmod_bank_fc(P(x), 40, P(out), 39, 1, 40, P(np.zeros(1, np.float32))) == -1
    assert np.all(out == 7.0)


# ---- the drop-ins on the whole emulated library ------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    L = C.CDLL(str(lib))
    vp, it = C.c_void_p, C.c_int
    L.fir_interpolate_cc.argtypes = [vp, vp, it, it, vp, it]; L.fir_interpolate_cc.restype = it
    L.fmmod_fc.argtypes = [vp, vp, it, C.c_float]; L.fmmod_fc.restype = C.c_float
    return L


@needs_ref
def test_dropins_against_reference(full):
    rng = np.random.default_rng(9)
    for I, T, n in ((1, 81, 200), (3, 81, 1024), (50, 401, 60), (5, 81, 10)):
        x = rows(rng, 1, n)[0]
        taps = tx.ref_lowpass(T, 0.5 / I)
        out = np.zeros(max(n * I, 1), np.complex64)
        m = full.fir_interpolate_cc(P(x), P(out), n, I, P(taps), T)
        want = tx.ref_fir_interpolate_cc(x, I, taps)
        assert m == want.size and same_bits(out[:m], tx.fir_interpolate_cc(x, I, taps)), (I, T, n)
    x = fm_inputs(rng, 700)[2]
    out = np.zeros(700, np.complex64)
    ph = full.fmmod_fc(P(x), P(out), 700, 0.5)
    want, last = tx.ref_fmmod_fc(x, 0.5)
    assert np.float32(ph) == last and np.abs(out - want).max() <= 2 * ULP1
