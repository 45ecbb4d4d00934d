"""CPU tier for the waterfall bank (csdr_b200/csrc/spectrum.cu, csdrb_spectrum_bank_cf): the shipped kernels and launchers run thread by
thread on the emulated library (tests/host_shim) and must give the bytes of the composition of the existing per-block calls
(tests/spectrum/spectrum.py) for every FFT size the bank serves, overlapped, back-to-back and gapped framing, several averages, padded strides,
one and several rows, both output forms; any cut of the stream and any scratch size give the bytes of one call; a row's bytes do not depend on
the other rows; the power stays within a derived float64 bound; NaN/Inf stay in their own lines; the line count is fft_cc's; every refusal.
tests/test_gpu_spectrum.py runs the same bodies on the H100 at full size."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "spectrum"))
import emul_build  # noqa: E402
import spectrum as S  # noqa: E402


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    return S.EmulDev(C.CDLL(str(lib)))


@pytest.fixture(scope="module")
def full_size():
    return False


SIZES = (2, 4, 16, 32, 256, 1024, 4096, 16384)


def _everies(N):
    return sorted({1, max(N // 3, 1), max(N - 1, 1), N, N + 1, 3 * N})


def signal(rng, rows, T):
    return ((rng.standard_normal((rows, T)) + 1j * rng.standard_normal((rows, T))) * 0.3).astype(np.complex64)


def _frames_for(N, A, full_size):
    if N >= 4096 and not full_size:
        return A + 1 if A == 1 else A                                   # the largest sizes with few frames
    return 2 * A + 1


CASES = [(N, E, (1, 3, 7)[(i + j) % 3], (1, 5)[(i + 2 * j) % 2], (i + j) % 2 == 0, 3 * ((i * 5 + j) % 3))
         for i, N in enumerate(SIZES) for j, E in enumerate(_everies(N))]


@pytest.mark.parametrize("N,E,A,rows,compress,pad", CASES)
def test_bank_equals_the_composition(dev, full_size, N, E, A, rows, compress, pad):
    rng = np.random.default_rng(N * 31 + E)
    rows = 64 if full_size and rows > 1 and N <= 4096 else rows
    p = S.Params(N, E, A, int(compress), -70.0)
    T = S.stream_for(N, E, _frames_for(N, A, full_size)) + int(rng.integers(0, E))
    x = signal(rng, rows, T)
    w = S.window(dev.L, N)
    want = S.composition(dev, x, p, w)
    got = S.bank(dev, x, p, w, pad=pad, out_pad=4 * (pad % 2))
    assert got.shape == want.shape and got.shape[1] >= 1
    assert np.array_equal(got, want)


@pytest.mark.parametrize("N,add_db", [(16, 0.0), (256, -70.0), (1024, 3.5)])
def test_one_average_is_logpower_cf(dev, N, add_db):
    """A = 1, E = N: every line is logpower_cf of one frame's spectrum, halves swapped"""
    rng = np.random.default_rng(N)
    x = signal(rng, 1, 5 * N)
    p = S.Params(N, N, 1, 0, add_db)
    w = S.window(dev.L, N)
    got = S.bank(dev, x, p, w)[0].view(np.float32)
    d_fr = dev.put(x[0]); d_w = dev.alloc(8 * 5 * N); d_s = dev.alloc(8 * 5 * N); d_p = dev.alloc(4 * 5 * N); d_win = dev.put(w)
    assert dev.L.csdrb_apply_window_rows_c(dev.ptr(d_fr), dev.ptr(d_w), dev.ptr(d_win), N, 5, dev.stream) >= 0
    assert dev.L.csdrb_fft_c2c_batch(dev.ptr(d_w), N, dev.ptr(d_s), N, N, 5, 0, dev.stream) >= 0
    assert dev.L.csdrb_logpower_cf(dev.ptr(d_s), dev.ptr(d_p), 5 * N, add_db, dev.stream) >= 0
    want = dev.get(d_p, np.float32).reshape(5, N)
    want = np.concatenate([want[:, N // 2:], want[:, :N // 2]], axis=1)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("N,E,A,compress", [(64, 20, 3, 1), (64, 64, 2, 0), (32, 50, 4, 1), (256, 85, 7, 0)])
def test_any_cut_and_any_scratch_give_one_call(dev, N, E, A, compress):
    rng = np.random.default_rng(E * 7 + A)
    rows = 3
    p = S.Params(N, E, A, compress, -20.0)
    T = S.stream_for(N, E, 4 * A + 2) + 5
    x = signal(rng, rows, T)
    w = S.window(dev.L, N)
    one = S.bank(dev, x, p, w)
    # random cuts, with empty calls, single samples, calls shorter than N and cuts inside a line
    cuts = sorted(set(int(c) for c in rng.integers(0, T, 9)) | {0, 1, 2, N // 2, N // 2 + 1, E * A + 1})
    cuts = [c for c in cuts if 0 <= c <= T] + [cuts[3]]                  # a repeated cut: a call with n = 0
    assert np.array_equal(S.bank(dev, x, p, w, cuts=cuts), one)
    assert np.array_equal(S.bank(dev, x, p, w, scratch="min"), one)
    assert np.array_equal(S.bank(dev, x, p, w, cuts=cuts[::2], scratch="min", pad=5), one)


def test_rows_are_independent(dev):
    rng = np.random.default_rng(3)
    N, E, A = 128, 100, 3
    p = S.Params(N, E, A, 1, -50.0)
    T = S.stream_for(N, E, 3 * A)
    x = signal(rng, 4, T)
    w = S.window(dev.L, N)
    all4 = S.bank(dev, x, p, w)
    for r in range(4):
        assert np.array_equal(S.bank(dev, x[r:r + 1], p, w)[0], all4[r])
    y = x.copy(); y[0] *= 1000; y[2] = np.nan
    other = S.bank(dev, y, p, w)
    assert np.array_equal(other[1], all4[1]) and np.array_equal(other[3], all4[3])


@pytest.mark.parametrize("N,A", [(64, 1), (256, 3), (1024, 2)])
def test_power_within_the_float64_bound(dev, N, A):
    rng = np.random.default_rng(N + A)
    E = N // 2
    p = S.Params(N, E, A, 0, -10.0)
    x = signal(rng, 1, S.stream_for(N, E, 3 * A))
    x[0, 5:9] *= 1e3                                                     # a strong component next to the noise floor
    w = S.window(dev.L, N, "BLACKMAN")
    lines = S.bank(dev, x, p, w)[0].view(np.float32)
    assert S.check_power_bound(lines, x[0], p, w) > lines.size // 2


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_nonfinite_input_stays_in_its_lines(dev, bad):
    N, E, A = 64, 24, 2
    rng = np.random.default_rng(11)
    p = S.Params(N, E, A, 0, 0.0)
    T = S.stream_for(N, E, 12 * A)
    x = signal(rng, 2, T)
    w = S.window(dev.L, N)
    clean = S.bank(dev, x, p, w)
    pos = 300
    y = x.copy(); y[0, pos] = complex(bad, 0.0) if bad == bad else complex(0.0, bad)
    dirty = S.bank(dev, y, p, w)
    assert np.array_equal(dirty[1], clean[1])
    frames = [k for k in range(S.frames_at(N, E, T)) if S.frame_start(N, E, k) <= pos < S.frame_start(N, E, k) + N]
    hit = {k // A for k in frames}
    vals = dirty[0].view(np.float32)
    for j in range(clean.shape[1]):
        if j in hit:
            assert not np.isfinite(vals[j]).any(), j
        else:
            assert np.array_equal(dirty[0, j], clean[0, j]), j


def test_line_count_is_fft_ccs(dev):
    L = dev.L
    for N in (2, 4, 8):
        for E in range(1, 3 * N + 2):
            for A in (1, 2, 3):
                for consumed in range(0, 3 * N + 1):
                    st = S.State(consumed, S.frames_bruteforce(N, E, consumed))
                    p = S.Params(N, E, A, 0, 0.0)
                    for n in range(0, 2 * N + 3):
                        want = S.frames_bruteforce(N, E, consumed + n) // A - S.frames_bruteforce(N, E, consumed) // A
                        assert L.csdrb_spectrum_bank_lines(C.byref(p), C.byref(st), n) == want, (N, E, A, consumed, n)


def test_refusals(dev):
    L = dev.L
    N = 64
    x = dev.alloc(8 * 4 * N); w = dev.put(S.window(L, N)); h = dev.alloc(8 * 4 * N); a = dev.alloc(4 * 4 * N); o = dev.alloc(4 * 4 * N * 4)
    p = S.Params(N, N, 1, 0, 0.0)
    sb = L.csdrb_spectrum_bank_scratch_bytes(4, 4 * N, C.byref(p)); s = dev.alloc(sb)
    P = dev.ptr

    def call(xp=None, rows=1, n=2 * N, wp=None, params=None, hp=None, ap=None, st=None, op=None, ostride=4 * N * 4, sp=None, sbytes=None):
        st = st or S.State(0, 0)
        return L.csdrb_spectrum_bank_cf(P(x) if xp is None else xp, 2 * N, rows, n, P(w) if wp is None else wp, C.byref(params or p),
                                        P(h) if hp is None else hp, P(a) if ap is None else ap, C.byref(st), P(o) if op is None else op, ostride,
                                        P(s) if sp is None else sp, sb if sbytes is None else sbytes, dev.stream)
    assert call() == 2
    for kw in (dict(rows=0), dict(n=-1), dict(params=S.Params(N, 0, 1, 0, 0.0)), dict(params=S.Params(N, N, 0, 0, 0.0)), dict(xp=0), dict(wp=0),
               dict(hp=0), dict(ap=0), dict(op=0), dict(sp=0), dict(xp=P(x) + 4), dict(hp=P(h) + 4), dict(ap=P(a) + 2), dict(wp=P(w) + 1),
               dict(op=P(o) + 2), dict(ostride=4 * N * 4 + 2), dict(sp=P(s) + 8), dict(sbytes=4 * N - 1),
               dict(st=S.State(5, 7)), dict(st=S.State(-1, 0))):
        assert call(**kw) == -1, (kw, L.csdrb_last_error())
    for n_bad in (0, 1, 3, 48, 100, 32768, 65536):
        assert call(params=S.Params(n_bad, 1, 1, 0, 0.0)) == -2, n_bad
        assert L.csdrb_spectrum_bank_lines(C.byref(S.Params(n_bad, 1, 1, 0, 0.0)), C.byref(S.State(0, 0)), 10) == -2
        assert L.csdrb_spectrum_bank_scratch_bytes(1, 10, C.byref(S.Params(n_bad, 1, 1, 0, 0.0))) == 0
    assert L.csdrb_spectrum_bank_lines(C.byref(p), C.byref(S.State(0, 0)), -1) == -1
    # ADPCM lines are bytes: any output alignment and stride will do
    pc = S.Params(N, N, 1, 1, 0.0)
    sbc = L.csdrb_spectrum_bank_scratch_bytes(1, 2 * N, C.byref(pc)); sc = dev.alloc(sbc)
    assert L.csdrb_spectrum_bank_cf(P(x), 2 * N, 1, 2 * N, P(w), C.byref(pc), P(h), P(a), C.byref(S.State(0, 0)), P(o) + 1, 75, P(sc), sbc, dev.stream) == 2
