"""CPU tier for the tone filter banks (csdr_b200/csrc/tone.cu): the shipped kernels and launchers run thread by thread under
tests/host_shim/cuda_emul.h.  apply_fir_cc must equal the checker tests/tone/tone_oracle.c and the compiled reference bit for bit;
bfsk_demod_cf must equal the checker bit for bit and lie within the per-output bound of tests/tone/tone.py (bfsk_bound, derived there)
of the reference, whose build sums in another order.  Covered: random L in 2..4096, ragged n, row strides and channel counts; a stream
cut into calls with the L - 1 carry; NaN and Inf kept inside their own windows; the -1 and -2 refusals, which launch nothing; and
firdes_add_peak_c and the drop-ins of the whole emulated library against the reference."""
import ctypes as C
import os
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "tone"))
import emul_build  # noqa: E402
import tone  # noqa: E402

_built = {}
needs_ref = pytest.mark.skipif(not tone.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built")


@pytest.fixture(scope="module", params=["alternate", "random"])
def K(request, tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    if "tone" not in _built:
        lib, names = emul_build.build_file(tmp_path_factory.mktemp("emul_tone"), "tone.cu")
        _built["tone"] = (Path(lib._name), names, lib)
    so, names, proto = _built["tone"]
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


def P(a):
    return a.ctypes.data


def rows_of(rng, ch, n, kind="noise"):
    z = (rng.standard_normal((ch, n)) + 1j * rng.standard_normal((ch, n))) * 0.5
    if kind == "heavy":
        z *= 10.0 ** rng.uniform(-6, 6, (ch, n))
    return z.astype(np.complex64)


def bank(K, kind, x, n, taps, stride=None, out_stride=None):
    """x [ch, >= n] complex64 -> the bank's rows; taps: one set (apply) or (mark, space)"""
    ch = x.shape[0]
    stride = stride or n
    xin = np.zeros((ch, stride), np.complex64)
    xin[:, :n] = x[:, :n]
    L = len(taps) if kind == "apply" else len(taps[0])
    m = n - L + 1
    ostride = out_stride or max(m, 1)
    if kind == "apply":
        out = np.full((ch, ostride), np.nan, np.complex64)
        t = np.ascontiguousarray(taps, np.complex64)
        rc = K.emul_launch_apply_fir_bank_cc(P(xin), stride, P(out), ostride, ch, n, P(t), L)
    else:
        out = np.full((ch, ostride), np.nan, np.float32)
        mk, sp = (np.ascontiguousarray(t, np.complex64) for t in taps)
        rc = K.emul_launch_bfsk_demod_bank_cf(P(xin), stride, P(out), ostride, ch, n, P(mk), P(sp), L)
    assert rc == m, (rc, K.emul_last_error())
    return out[:, :m]


def oracle(kind, x, taps):
    return tone.apply_fir_cc(x, taps) if kind == "apply" else tone.bfsk_demod_cf(x, *taps)


def random_taps(rng, kind, L):
    t = lambda: ((rng.standard_normal(L) + 1j * rng.standard_normal(L)) / L).astype(np.complex64)   # noqa: E731
    return t() if kind == "apply" else (t(), t())


def same_bits(a, b):
    """equal bit for bit, except that any NaN equals any NaN (the GPU writes the canonical NaN, a CPU keeps an input's payload)"""
    fa, fb = np.asarray(a).view(np.float32), np.asarray(b).view(np.float32)
    na, nb = np.isnan(fa), np.isnan(fb)
    return fa.shape == fb.shape and np.array_equal(na, nb) and np.array_equal(fa[~na].view(np.uint32), fb[~nb].view(np.uint32))


@pytest.mark.parametrize("kind", ["apply", "bfsk"])
def test_bank_equals_checker(K, kind):
    rng = np.random.default_rng(1 if kind == "apply" else 2)
    geoms = [(2, 3, 1), (3, 9, 2), (7, 900, 3), (44, 2000, 5), (255, 1170, 2), (int(rng.integers(8, 700)), 1500, 3),
             (int(rng.integers(700, 2100)), 2500, 2), (4096, 4096 + 130, 1), (int(rng.integers(2100, 4096)), 4300, 1)]
    for L, n, ch in geoms:
        x = rows_of(rng, ch, n, "heavy" if L % 2 else "noise")
        taps = random_taps(rng, kind, L)
        got = bank(K, kind, x, n, taps, stride=n + int(rng.integers(0, 5)), out_stride=n - L + 1 + int(rng.integers(0, 3)))
        for c in range(ch):
            assert same_bits(got[c], oracle(kind, x[c], taps)), (L, n, c)


@needs_ref
def test_apply_bank_equals_reference_bit_for_bit(K):
    rng = np.random.default_rng(3)
    for L, n in ((2, 40), (5, 300), (44, 1000), (301, 1300), (1024, 1500)):
        x = rows_of(rng, 2, n, "heavy")
        taps = tone.ref_peak(float(rng.uniform(-0.5, 0.5)), L)
        got = bank(K, "apply", x, n, taps)
        for c in range(2):
            assert same_bits(got[c], tone.ref_apply_fir_cc(x[c], taps)), (L, c)


@needs_ref
def test_bfsk_bank_within_bound_of_reference(K):
    """the reference's build vectorises the sum: the bank equals it within bfsk_bound, and most outputs bit for bit is not required"""
    rng = np.random.default_rng(4)
    worst = 0.0
    for L, n, spacing in ((2, 50, 0.2), (5, 200, 0.1), (44, 900, 0.085), (255, 1400, 0.02), (1023, 1600, 0.01)):
        z = tone.rtty_signal(b"RYRY CQ", 44.0, rng, noise=0.05)[:n]
        x = np.stack([z, rows_of(rng, 1, n, "heavy")[0]])
        mark, space = tone.bfsk_taps(spacing, L)
        got = bank(K, "bfsk", x, n, (mark, space))
        for c in range(2):
            want = tone.ref_bfsk_demod_cf(x[c], mark, space)
            bound = tone.bfsk_bound(x[c], mark, space)
            err = np.abs(got[c].astype(np.float64) - want)
            assert np.all(err <= bound), (L, c, float(np.max(err / bound)))
            worst = max(worst, float(np.max(err / bound)))
    assert worst > 0.0                                                  # the two orders do differ somewhere


@pytest.mark.parametrize("kind", ["apply", "bfsk"])
def test_calls_with_carry_equal_one_call(K, kind):
    """a stream cut into calls of any size, each starting with the previous call's last L - 1 inputs, gives the bits of one call"""
    rng = np.random.default_rng(5)
    for L in (2, 44, 255):
        n = 3000
        x = rows_of(rng, 3, n)
        taps = random_taps(rng, kind, L)
        whole = bank(K, kind, x, n, taps)
        pieces, pos = [], 0
        while pos + L - 1 < n:
            k = min(n - pos, L - 1 + int(rng.integers(1, 700)))
            pieces.append(bank(K, kind, np.ascontiguousarray(x[:, pos:pos + k]), k, taps))
            pos += k - (L - 1)
        assert same_bits(np.concatenate(pieces, axis=1), whole), L


@pytest.mark.parametrize("kind", ["apply", "bfsk"])
def test_nan_and_inf_stay_in_their_windows(K, kind):
    rng = np.random.default_rng(6)
    L, n = 37, 1200
    x = rows_of(rng, 3, n)
    taps = random_taps(rng, kind, L)
    clean = bank(K, kind, x, n, taps)
    bad = x.copy()
    spots = {0: (100, np.nan), 1: (640, np.inf), 2: (1100, -np.inf)}
    for c, (i, v) in spots.items():
        bad[c, i] = v + (1j * 0 if c != 1 else 0)
    got = bank(K, kind, bad, n, taps)
    for c, (i, v) in spots.items():
        hit = np.zeros(n - L + 1, bool)
        hit[max(0, i - L + 1):i + 1] = True
        assert same_bits(got[c][~hit], clean[c][~hit]), c
        assert same_bits(got[c], oracle(kind, bad[c], taps)), c
        g = got[c][hit].view(np.float32) if kind == "apply" else got[c][hit]
        assert not np.all(np.isfinite(g)), c


def test_refusals_launch_nothing(K):
    x = np.zeros(64, np.complex64); t = np.ones(4097, np.complex64)
    out = np.full(64, 7.0, np.complex64); outf = np.full(64, 7.0, np.float32)
    for L, n, stride, ostride, want in ((1, 64, 64, 64, -2), (4097, 5000, 5000, 5000, -2), (0, 64, 64, 64, -2), (8, 7, 64, 64, -1),
                                        (8, 64, 63, 64, -1), (8, 64, 64, 56, -1)):
        assert K.emul_launch_apply_fir_bank_cc(P(x), stride, P(out), ostride, 1, n, P(t), L) == want, (L, n)
        assert K.emul_launch_bfsk_demod_bank_cf(P(x), stride, P(outf), ostride, 1, n, P(t), P(t), L) == want, (L, n)
    assert np.all(out == 7.0) and np.all(outf == 7.0)


# ---- filter design and the drop-ins on the whole emulated library -----------------------------------------------------------------
@pytest.fixture(scope="module")
def full(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    L = C.CDLL(str(lib))
    vp, it = C.c_void_p, C.c_int
    L.firdes_add_peak_c.argtypes = [vp, it, C.c_float, it, it, it]
    L.apply_fir_cc.argtypes = [vp, vp, it, vp, it]; L.apply_fir_cc.restype = it
    L.bfsk_demod_cf.argtypes = [vp, vp, it, vp, vp, it]; L.bfsk_demod_cf.restype = it
    return L


def ours_peak(L):
    def peak(rate, length, window=tone.HAMMING, into=None, add=0, normalize=1):
        t = np.zeros(max(length, 1), np.complex64) if into is None else into
        L.firdes_add_peak_c(t.ctypes.data, length, rate, window, add, normalize)
        return t[:length]
    return peak


@needs_ref
def test_firdes_add_peak_c_equals_reference(full):
    peak = ours_peak(full)
    rng = np.random.default_rng(7)
    rates = [0.0, 0.0425, -0.0425, 0.25, -0.5, 0.5, 0.49999, 1e-6, 0.3333333, -0.1234567, 0.75, -1.3] + list(rng.uniform(-0.5, 0.5, 12))
    for window in (0, 1, 2):
        for length in (2, 3, 4, 5, 44, 45, 101, 255, 1000, 4096):
            for rate in rates:
                a, b = peak(float(rate), length, window), tone.ref_peak(float(rate), length, window)
                if window == 1:
                    # Blackman at |x| = 1 is 0.42 - 0.5 cos 2pi + 0.08 cos 4pi, about 1e-17, which the product's window kernel (shared with
                    # firdes_lowpass_f) rounds differently from the build; those end taps differ below 1e-16 of the largest tap, the rest agree
                    ends = np.abs(np.arange(length) - length // 2) == length // 2
                    assert same_bits(a[~ends], b[~ends]), (rate, length)
                    assert np.all(np.abs(a[ends] - b[ends]) <= 1e-16 * np.max(np.abs(b))), (rate, length)
                else:
                    assert same_bits(a, b), (rate, length, window)
    # several peaks added up, normalised after the last (peaks_fir_cc)
    for length in (45, 301):
        a = np.zeros(length, np.complex64); b = np.zeros(length, np.complex64)
        for k, rate in enumerate((0.1, -0.2, 0.33)):
            peak(rate, length, 2, into=a, add=1, normalize=int(k == 2)); tone.ref_peak(rate, length, 2, into=b, add=1, normalize=int(k == 2))
        assert same_bits(a, b), length


@needs_ref
def test_dropins_against_reference(full):
    rng = np.random.default_rng(8)
    for L, n in ((2, 2), (44, 43), (44, 1024), (255, 3000)):
        x = rows_of(rng, 1, n)[0]
        taps = tone.ref_peak(0.1, L)
        out = np.zeros(max(n, 1), np.complex64)
        m = full.apply_fir_cc(x.ctypes.data, out.ctypes.data, n, taps.ctypes.data, L)
        want = tone.ref_apply_fir_cc(x, taps)
        assert m == max(n - L + 1, 0) and same_bits(out[:m], want), (L, n)
        mark, space = tone.bfsk_taps(0.085, L)
        outf = np.zeros(max(n, 1), np.float32)
        m = full.bfsk_demod_cf(x.ctypes.data, outf.ctypes.data, n, mark.ctypes.data, space.ctypes.data, L)
        assert m == n - L + 1, (L, n, m)                                  # the reference's count, negative when n < L - 1
        if m > 0:
            assert same_bits(outf[:m], tone.bfsk_demod_cf(x, mark, space))
            assert np.all(np.abs(outf[:m] - tone.ref_bfsk_demod_cf(x, mark, space)) <= tone.bfsk_bound(x, mark, space))
