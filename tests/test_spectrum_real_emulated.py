"""CPU tier for the real-input FFT and waterfall (csdr_b200/csrc/fft_real.cuh, spectrum.cu): csdrb_fft_r2c_batch against numpy's float64 rfft
within the bound derived in tests/spectrum/spectrum_real.py, for every single-CTA size and one four-step size; make_fft_r2c + fft_execute against
the batch call, bit for bit; csdrb_spectrum_bank_f against the composition apply_precalculated_window_f -> csdrb_fft_r2c_batch ->
csdrb_accumulate_power_cf -> csdrb_log_ff [-> ADPCM], bit for bit, over sizes, framings (E < 2N, E = 2N, E > 2N), rows and both output forms; any
cut and any scratch give one call's bytes; rows are independent; the line count is fft_fc's; NaN/Inf stay in their lines; every refusal.  The
shipped kernels run thread by thread on the emulated library (tests/host_shim).  tests/test_gpu_spectrum_real.py runs the same bodies on the H100."""
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
import spectrum_real as R  # noqa: E402


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    d = S.EmulDev(C.CDLL(str(lib)))
    R.setup(d.L)
    return d


@pytest.fixture(scope="module")
def full_size():
    return False


def noise(rng, *shape):
    return (rng.standard_normal(shape) * 0.3).astype(np.float32)


# ---- the transform ------------------------------------------------------------------------------------------------------------------------
def check_r2c_bound(dev, n, batch, in_pad=0, out_pad=0, in_offset=0):
    rng = np.random.default_rng(n + batch)
    x = noise(rng, batch, n)
    x[:, 3] += 40.0                                                      # a strong sample next to the noise
    got = R.r2c(dev, x, in_pad, out_pad, in_offset)
    want = np.fft.rfft(x.astype(np.float64), axis=1)
    assert got.shape == want.shape
    bound = R.rfft_bound(x)
    err = np.abs(got.astype(np.complex128) - want)
    assert np.all(err <= bound), float((err / bound).max())
    assert np.all(got[:, 0].imag == 0) and np.all(got[:, -1].imag == 0)
    return got


@pytest.mark.parametrize("n", [1 << k for k in range(2, 16)])
def test_r2c_within_the_bound(dev, n):
    """every single-CTA size, 4..32768 real points, a row at an odd float offset and padded strides"""
    check_r2c_bound(dev, n, 3 if n <= 4096 else 1, in_pad=3, out_pad=1, in_offset=1)


def test_r2c_four_step_size(dev, full_size):
    """2^16 real points: the four-step transform of 32768 packed points, then the split kernel in place"""
    for lg in ((16, 17, 18, 19, 20, 21) if full_size else (16,)):
        check_r2c_bound(dev, 1 << lg, 2 if full_size else 1, in_pad=1 if full_size else 0, out_pad=2 if full_size else 0, in_offset=1)


def test_r2c_impulse_and_cosine(dev):
    n = 256
    x = np.zeros((2, n), np.float32); x[0, 0] = 1.0
    x[1] = np.cos(2 * np.pi * 5 * np.arange(n) / n).astype(np.float32)
    got = R.r2c(dev, x)
    assert np.array_equal(got[0], np.ones(n // 2 + 1, np.complex64))
    assert abs(got[1, 5] - n / 2) < 1e-3 and np.abs(np.delete(got[1], 5)).max() < 1e-3


def test_dropin_plan_equals_the_batch_call(dev):
    L = dev.L
    rng = np.random.default_rng(5)
    for n in (4, 64, 2048, 32768, 65536):
        x = noise(rng, n)
        y = np.full(n // 2 + 8, 7 + 7j, np.complex64)                   # bins past n/2 must stay untouched
        pl = L.make_fft_r2c(n, x.ctypes.data, y.ctypes.data, 0)
        assert pl
        L.fft_execute(pl); L.fft_destroy(pl)
        want = R.r2c(dev, x[None])[0]
        assert np.array_equal(y[:n // 2 + 1].view(np.uint64), want.view(np.uint64)), n
        assert np.all(y[n // 2 + 1:] == 7 + 7j)
    for bad in (0, 1, 2, 6, 100, 1 << 22):
        assert not L.make_fft_r2c(bad, x.ctypes.data, y.ctypes.data, 0), bad


def test_window_f_is_the_float_product(dev):
    rng = np.random.default_rng(2)
    x = noise(rng, 1000); w = rng.random(1000).astype(np.float32); o = np.empty_like(x)
    dev.L.apply_precalculated_window_f(x.ctypes.data, o.ctypes.data, x.size, w.ctypes.data)
    assert np.array_equal(o, x * w)


def test_r2c_refusals(dev):
    L = dev.L
    x = dev.alloc(4 * 4096); y = dev.alloc(8 * 4096)
    P = dev.ptr
    assert L.csdrb_fft_r2c_batch(P(x), 64, P(y), 33, 64, 2, None) == 0
    assert L.csdrb_fft_r2c_batch(P(x), 64, P(y), 33, 64, 0, None) == 0
    for n in (0, 1, 2, 3, 6, 100, 1 << 22):
        assert L.csdrb_fft_r2c_batch(P(x), 64, P(y), 33, n, 1, None) == -1, n
    assert L.csdrb_fft_r2c_batch(0, 64, P(y), 33, 64, 1, None) == -1
    assert L.csdrb_fft_r2c_batch(P(x), 64, 0, 33, 64, 1, None) == -1
    assert L.csdrb_fft_r2c_batch(P(x), 63, P(y), 33, 64, 2, None) == -1                 # rows overlap
    assert L.csdrb_fft_r2c_batch(P(x), 64, P(y), 32, 64, 2, None) == -1


# ---- the bank -----------------------------------------------------------------------------------------------------------------------------
SIZES = (2, 4, 16, 32, 256, 1024, 4096, 16384)


def _everies(N):
    L = 2 * N
    return sorted({1, max(L // 3, 1), L - 1, L, L + 1, 3 * N})


def _frames_for(N, A, full_size):
    if N >= 4096 and not full_size:
        return A + 1 if A == 1 else A
    return 2 * A + 1


CASES = [(N, E, (1, 3, 7)[(i + j) % 3], (1, 5)[(i + 2 * j) % 2], (i + j) % 2 == 0, 3 * ((i * 5 + j) % 3))
         for i, N in enumerate(SIZES) for j, E in enumerate(_everies(N))
         if not (N >= 4096 and E < N // 2)]                             # the largest sizes with a handful of frames only


@pytest.mark.parametrize("N,E,A,rows,compress,pad", CASES)
def test_bank_equals_the_composition(dev, full_size, N, E, A, rows, compress, pad):
    rng = np.random.default_rng(N * 31 + E)
    rows = 64 if full_size and rows > 1 and N <= 4096 else rows
    p = S.Params(N, E, A, int(compress), -70.0)
    T = R.stream_for(N, E, _frames_for(N, A, full_size)) + int(rng.integers(0, E))
    x = noise(rng, rows, T)
    w = S.window(dev.L, 2 * N)
    want = R.composition(dev, x, p, w)
    got = R.bank(dev, x, p, w, pad=pad, out_pad=4 * (pad % 2), offset=1 + pad % 2)
    assert got.shape == want.shape and got.shape[1] >= 1
    assert np.array_equal(got, want)


@pytest.mark.parametrize("N,E,A,compress", [(64, 20, 3, 1), (64, 128, 2, 0), (32, 150, 4, 1), (256, 85, 7, 0)])
def test_any_cut_and_any_scratch_give_one_call(dev, N, E, A, compress):
    rng = np.random.default_rng(E * 7 + A)
    p = S.Params(N, E, A, compress, -20.0)
    T = R.stream_for(N, E, 4 * A + 2) + 5
    x = noise(rng, 3, T)
    w = S.window(dev.L, 2 * N)
    one = R.bank(dev, x, p, w)
    cuts = sorted(set(int(c) for c in rng.integers(0, T, 9)) | {0, 1, 2, N, N + 1, E * A + 1})
    cuts = [c for c in cuts if 0 <= c <= T] + [cuts[3]]                  # a repeated cut: a call with n = 0
    assert np.array_equal(R.bank(dev, x, p, w, cuts=cuts), one)
    assert np.array_equal(R.bank(dev, x, p, w, scratch="min"), one)
    assert np.array_equal(R.bank(dev, x, p, w, cuts=cuts[::2], scratch="min", pad=5, offset=0), one)


def test_rows_are_independent(dev):
    rng = np.random.default_rng(3)
    N, E, A = 128, 300, 3
    p = S.Params(N, E, A, 1, -50.0)
    x = noise(rng, 4, R.stream_for(N, E, 3 * A))
    w = S.window(dev.L, 2 * N)
    all4 = R.bank(dev, x, p, w)
    for r in range(4):
        assert np.array_equal(R.bank(dev, x[r:r + 1], p, w)[0], all4[r])
    y = x.copy(); y[0] *= 1000; y[2] = np.nan
    other = R.bank(dev, y, p, w)
    assert np.array_equal(other[1], all4[1]) and np.array_equal(other[3], all4[3])


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
def test_nonfinite_input_stays_in_its_lines(dev, bad):
    N, E, A = 32, 24, 2
    rng = np.random.default_rng(11)
    p = S.Params(N, E, A, 0, 0.0)
    T = R.stream_for(N, E, 12 * A)
    x = noise(rng, 2, T)
    w = S.window(dev.L, 2 * N)
    clean = R.bank(dev, x, p, w)
    pos = 300
    y = x.copy(); y[0, pos] = bad
    dirty = R.bank(dev, y, p, w)
    assert np.array_equal(dirty[1], clean[1])
    frames = [k for k in range(R.frames_at(N, E, T)) if R.frame_start(N, E, k) <= pos < R.frame_start(N, E, k) + 2 * N]
    hit = {k // A for k in frames}
    assert hit
    vals = dirty[0].view(np.float32)
    for j in range(clean.shape[1]):
        if j in hit:
            assert not np.isfinite(vals[j]).all(), j
        else:
            assert np.array_equal(dirty[0, j], clean[0, j]), j


def test_line_count_is_fft_fcs(dev):
    L = dev.L
    for N in (2, 4):
        for E in range(1, 6 * N + 2):
            for A in (1, 2, 3):
                for consumed in range(0, 6 * N + 1):
                    st = S.State(consumed, R.frames_bruteforce(N, E, consumed))
                    p = S.Params(N, E, A, 0, 0.0)
                    for n in range(0, 4 * N + 3):
                        want = R.frames_bruteforce(N, E, consumed + n) // A - R.frames_bruteforce(N, E, consumed) // A
                        assert L.csdrb_spectrum_bank_lines_f(C.byref(p), C.byref(st), n) == want, (N, E, A, consumed, n)


def test_the_gapped_framing_is_the_references(dev):
    """N = 4, E = 20 on a ramp, BOXCAR: the reference's frames start at 0, 32, 64, ... (2E - 2N apart); bin 0 is the frame's sum"""
    N, E = 4, 20
    x = np.arange(200, dtype=np.float32)[None]
    p = S.Params(N, E, 1, 0, 0.0)
    db = R.bank(dev, x, p, np.ones(2 * N, np.float32))[0].view(np.float32)
    starts = [R.frame_start(N, E, k) for k in range(db.shape[0])]
    assert starts[:3] == [0, 32, 64]
    want = [10 * np.log10(float(sum(range(s, s + 2 * N))) ** 2) for s in starts]
    assert np.allclose(db[:, 0], want, atol=1e-4)


def test_refusals(dev):
    L = dev.L
    N = 64
    x = dev.alloc(4 * 8 * N); w = dev.put(S.window(L, 2 * N)); h = dev.alloc(4 * 8 * N); a = dev.alloc(4 * 4 * N); o = dev.alloc(4 * 4 * N * 4)
    p = S.Params(N, 2 * N, 1, 0, 0.0)
    sb = L.csdrb_spectrum_bank_scratch_bytes_f(4, 8 * N, C.byref(p)); s = dev.alloc(sb)
    P = dev.ptr

    def call(xp=None, rows=1, n=4 * N, wp=None, params=None, hp=None, ap=None, st=None, op=None, ostride=4 * N * 4, sp=None, sbytes=None):
        st = st or S.State(0, 0)
        return L.csdrb_spectrum_bank_f(P(x) if xp is None else xp, 4 * N, rows, n, P(w) if wp is None else wp, C.byref(params or p),
                                       P(h) if hp is None else hp, P(a) if ap is None else ap, C.byref(st), P(o) if op is None else op, ostride,
                                       P(s) if sp is None else sp, sb if sbytes is None else sbytes, dev.stream)
    assert call() == 2
    assert call(xp=P(x) + 4, hp=P(h) + 4) == 2                          # real samples need 4-byte alignment only
    for kw in (dict(rows=0), dict(rows=65536), dict(n=-1), dict(params=S.Params(N, 0, 1, 0, 0.0)), dict(params=S.Params(N, N, 0, 0, 0.0)),
               dict(xp=0), dict(wp=0), dict(hp=0), dict(ap=0), dict(op=0), dict(sp=0), dict(xp=P(x) + 2), dict(hp=P(h) + 2), dict(ap=P(a) + 2),
               dict(wp=P(w) + 1), dict(op=P(o) + 2), dict(ostride=4 * N * 4 + 2), dict(sp=P(s) + 8), dict(sbytes=4 * N - 1),
               dict(st=S.State(5, 7)), dict(st=S.State(-1, 0))):
        assert call(**kw) == -1, (kw, L.csdrb_last_error())
    for n_bad in (0, 1, 3, 48, 100, 32768, 65536):
        assert call(params=S.Params(n_bad, 1, 1, 0, 0.0)) == -2, n_bad
        assert L.csdrb_spectrum_bank_lines_f(C.byref(S.Params(n_bad, 1, 1, 0, 0.0)), C.byref(S.State(0, 0)), 10) == -2
        assert L.csdrb_spectrum_bank_scratch_bytes_f(1, 10, C.byref(S.Params(n_bad, 1, 1, 0, 0.0))) == 0
    assert L.csdrb_spectrum_bank_lines_f(C.byref(p), C.byref(S.State(0, 0)), -1) == -1
    pc = S.Params(N, 2 * N, 1, 1, 0.0)
    sbc = L.csdrb_spectrum_bank_scratch_bytes_f(1, 4 * N, C.byref(pc)); sc = dev.alloc(sbc)
    assert L.csdrb_spectrum_bank_f(P(x), 4 * N, 1, 4 * N, P(w), C.byref(pc), P(h), P(a), C.byref(S.State(0, 0)), P(o) + 1, 75, P(sc), sbc, dev.stream) == 2
