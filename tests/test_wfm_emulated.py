"""CPU tier for the WFM audio bank (csdr_b200/csrc/audio.cu, csdrb_wfm_audio_bank_f_s16): the shipped kernel and launcher run thread by thread
on the emulated library (tests/host_shim) and must give, bit for bit, the oracle's `fractional_decimator_ff R 12 | deemphasis_wfm_ff 48000 TAU |
convert_f_s16` in the CLI's B-sample calls (tests/wfm/wfm.py) for several rates, buffer sizes, channel counts and padded strides; any cut of a
row into calls gives the bytes of one call; rows are independent; a NaN stays in its row and its carry restarts exactly where the reference's
de-emphasis calls start, while +-Inf is carried; the host-only output count agrees with the bank; every refusal, the -2 ones against a
brute-force float replay of the reference's call loop.  tests/test_gpu_wfm.py runs the same bodies on the H100."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "wfm"))
import emul_build  # noqa: E402
import wfm as W  # noqa: E402


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    return W.emul_dev(C.CDLL(str(lib)))


@pytest.fixture(scope="module")
def full_size():
    return False


RATES = (1.25, 5.0, 5.2083333, 5.3333333, 16.0)
BUFSIZES = (1024, 64, 19)                                           # 19: the smallest B whose every call consumes a sample
CHANNELS = (1, 31, 33, 130)
CASES = [(r, b, CHANNELS[(i + j) % 4], 3 * ((i + 2 * j) % 2)) for i, r in enumerate(RATES) for j, b in enumerate(BUFSIZES)]
TAU = 50e-6


def _length(b, full_size):
    return (40 if full_size else 4) * b + 37


@pytest.mark.parametrize("rate,bufsize,rows,pad", CASES)
def test_bank_equals_the_checker(dev, oracle, full_size, rate, bufsize, rows, pad):
    rng = np.random.default_rng(int(rate * 1000) + bufsize)
    x = W.signal(rng, rows, _length(bufsize, full_size))
    p = W.Params(rate, bufsize, TAU, 48000)
    got, s, _ = W.bank(dev, x, p, pad=pad)
    want = np.stack([W.checker(oracle, x[c], rate, bufsize, TAU) for c in range(rows)])
    assert got.shape == want.shape and got.shape[1] > 0
    assert np.array_equal(got, want)
    m, consumed, where = W.replay(rate, bufsize, x.shape[1])
    assert (s.audio, np.float32(s.where)) == (m, np.float32(where))
    assert 5.0 < s.where <= 6.0


@pytest.mark.parametrize("rate,bufsize", [(5.0, 1024), (5.2083333, 64), (16.0, 19), (1.25, 64)])
def test_any_cut_gives_one_call(dev, full_size, rate, bufsize):
    rng = np.random.default_rng(3)
    T = _length(bufsize, full_size) + 5 * bufsize
    x = W.signal(rng, 5, T)
    p = W.Params(rate, bufsize, 75e-6, 48000)
    one, s1, l1 = W.bank(dev, x, p)
    k = bufsize
    for cuts in ([0, 0, 1, bufsize - 1], [k, 2 * k, 3 * k], [k - 1, k, k + 1, 4 * k - 1],
                 sorted(set(rng.integers(1, T, 7).tolist())), list(range(0, T, max(T // 23, 1)))):
        got, s, last = W.bank(dev, x, p, cuts=cuts, pad=1)
        assert np.array_equal(got, one), cuts
        assert (s.where, s.audio) == (s1.where, s1.audio) and np.array_equal(last.view(np.uint32), l1.view(np.uint32))


def test_rows_are_independent(dev):
    rng = np.random.default_rng(5)
    x = W.signal(rng, 33, 3 * 1024 + 500)
    p = W.Params(5.0, 1024, TAU, 48000)
    together, _, _ = W.bank(dev, x, p)
    for c in (0, 17, 31, 32):
        alone, _, _ = W.bank(dev, x[c:c + 1], p)
        assert np.array_equal(together[c], alone[0])


def _next_multiple(k, b):
    return -(-k // b) * b


@pytest.mark.parametrize("bufsize", [64, 1024])
def test_nan_stays_in_its_row_and_restarts_where_the_reference_does(dev, oracle, bufsize):
    rng = np.random.default_rng(7)
    rows, rate = 34, 5.0
    x = W.signal(rng, rows, 12 * bufsize + 100, hot=False)
    clean, _, _ = W.bank(dev, x, W.Params(rate, bufsize, TAU, 48000))
    y = x.copy()
    hit = (3, 32)
    for c, s0 in zip(hit, (2 * bufsize + 77, 3 * bufsize + bufsize // 3)):
        y[c, s0] = np.nan
    got, _, _ = W.bank(dev, y, W.Params(rate, bufsize, TAU, 48000))
    for c in range(rows):
        if c not in hit:
            assert np.array_equal(got[c], clean[c]), c
            continue
        want = W.checker(oracle, y[c], rate, bufsize, TAU)
        assert np.array_equal(got[c], want)
        dec = oracle.fractional_decimator_ff(y[c], rate, 12, None, bufsize)
        bad = np.flatnonzero(np.isnan(dec))
        assert bad.size > 0
        reset = _next_multiple(int(bad[-1]) + 1, bufsize)               # the first de-emphasis call after the last NaN output
        assert reset < got.shape[1]
        assert np.all(got[c, bad[0]:reset] == 0)                         # NaN carried to the reset: INT_MIN & 0xffff = 0
        assert np.count_nonzero(got[c, reset:reset + 8]) >= 6             # audio again from the reset on
        assert np.array_equal(got[c, :bad[0]], clean[c, :bad[0]])
    # the same stream in calls that start mid-period: the carry is reset by the audio index counted from stream start, not at a call's start
    for cuts in (list(range(bufsize // 3 + 5, y.shape[1], bufsize // 3 + 5)), sorted(set(rng.integers(1, y.shape[1], 40).tolist()))):
        starts = []
        cut, _, _ = W.bank(dev, y, W.Params(rate, bufsize, TAU, 48000), cuts=cuts, pad=1, starts=starts)
        assert np.array_equal(cut, got), cuts
        dec = oracle.fractional_decimator_ff(y[hit[0]], rate, 12, None, bufsize)
        bad = np.flatnonzero(np.isnan(dec))
        assert any(bad[0] < a < _next_multiple(int(bad[-1]) + 1, bufsize) and a % bufsize for a in starts)    # a call inside the NaN run


def test_infinite_carry_is_kept_and_a_nan_carry_restarts(dev, oracle):
    rng = np.random.default_rng(8)
    x = W.signal(rng, 4, 2 * 1024 + 300, hot=False)
    last = np.array([np.inf, -np.inf, np.nan, 0.25], np.float32)
    got, _, carry = W.bank(dev, x, W.Params(5.0, 1024, TAU, 48000), last=last)
    for c in range(4):
        assert np.array_equal(got[c], W.checker(oracle, x[c], 5.0, 1024, TAU, last=float(last[c]))), c
    assert np.all(got[0] == 0) and np.all(got[1] == 0)                 # +-Inf stays in the recursion: INT_MIN & 0xffff = 0
    assert carry[0] == np.inf and carry[1] == -np.inf and np.isfinite(carry[2:]).all()
    assert np.count_nonzero(got[2]) > 0.9 * got.shape[1]


def test_outputs_agrees_with_the_bank(dev):
    rng = np.random.default_rng(9)
    x = W.signal(rng, 2, 4000, hot=False)
    for rate, bufsize in ((5.0, 1024), (16.0, 64), (1.25, 19), (5.3333333, 100)):
        p = W.Params(rate, bufsize, TAU, 48000)
        s = W.State(0.0, 0)
        d_last = dev.put(np.zeros(2, np.float32))
        at = 0
        for n in (0, bufsize - 1, bufsize, 3 * bufsize + 5, 700):
            n = min(n, x.shape[1] - at)
            before = (s.where, s.audio)
            m, consumed = W.outputs(dev, p, s, n)
            want = W.replay(rate, bufsize, n, None if before == (0.0, 0) else before[0])
            assert (m, consumed) == want[:2]
            d_in, d_out = dev.put(np.ascontiguousarray(x[:, at:at + max(n, 1)])), dev.alloc(2 * 2 * max(m, 1))   # a real buffer also for n = 0
            got_c = C.c_int(-1)
            got = dev.L.csdrb_wfm_audio_bank_f_s16(dev.ptr(d_in), n, 2, n, C.byref(p), C.byref(s), dev.ptr(d_last), dev.ptr(d_out), max(m, 1),
                                                   C.byref(got_c), dev.stream)
            assert (got, got_c.value) == (m, consumed)
            assert s.audio == before[1] + m
            if consumed == 0:
                assert (s.where, s.audio) == before
            at += consumed


def _call(dev, p, s, rows=2, n=2048, d_in=None, in_stride=None, d_last=None, d_out=None, out_stride=4096, consumed=True):
    ins = dev.alloc(4 * rows * n + 8)
    last = dev.alloc(4 * rows + 8)
    outs = dev.alloc(2 * rows * out_stride + 8)
    c = C.c_int(0)
    return dev.L.csdrb_wfm_audio_bank_f_s16(dev.ptr(ins) if d_in is None else d_in(ins), n if in_stride is None else in_stride, rows, n,
                                            C.byref(p), C.byref(s), dev.ptr(last) if d_last is None else d_last(last),
                                            dev.ptr(outs) if d_out is None else d_out(outs), out_stride, C.byref(c) if consumed else None, dev.stream)


def test_refusals(dev):
    good = W.Params(5.0, 1024, TAU, 48000)
    s0 = W.State(0.0, 0)
    assert _call(dev, good, W.State(0.0, 0)) > 0
    # -1: bad arguments
    assert _call(dev, good, W.State(0.0, 0), rows=0) == -1
    assert _call(dev, good, W.State(0.0, 0), n=-1, in_stride=0) == -1
    for p in (W.Params(1.0, 1024, TAU, 48000), W.Params(0.5, 1024, TAU, 48000), W.Params(float("nan"), 1024, TAU, 48000),
              W.Params(float("inf"), 1024, TAU, 48000),
              W.Params(5.0, 1024, 0.0, 48000), W.Params(5.0, 1024, -TAU, 48000), W.Params(5.0, 1024, float("nan"), 48000),
              W.Params(5.0, 1024, TAU, 0), W.Params(5.0, 1024, TAU, -48000)):
        assert _call(dev, p, W.State(0.0, 0)) == -1
        assert W.outputs(dev, p, s0, 2048)[0] == -1
    for st in (W.State(4.9, 10), W.State(0.0, 5), W.State(6.5, 1000), W.State(5.5, -1), W.State(float("nan"), 3)):
        assert _call(dev, good, st) == -1
        assert W.outputs(dev, good, st, 2048)[0] == -1
    assert _call(dev, good, W.State(5.0, 77)) > 0 and _call(dev, good, W.State(6.0, 77)) > 0
    assert _call(dev, good, W.State(0.0, 0), d_in=lambda b: None) == -1
    assert _call(dev, good, W.State(0.0, 0), d_last=lambda b: None) == -1
    assert _call(dev, good, W.State(0.0, 0), d_out=lambda b: None) == -1
    assert _call(dev, good, W.State(0.0, 0), consumed=False) == -1
    assert _call(dev, good, W.State(0.0, 0), d_in=lambda b: dev.ptr(b) + 2) == -1
    assert _call(dev, good, W.State(0.0, 0), d_last=lambda b: dev.ptr(b) + 1) == -1
    assert _call(dev, good, W.State(0.0, 0), d_out=lambda b: dev.ptr(b) + 1) == -1
    assert _call(dev, good, W.State(0.0, 0), in_stride=2047) == -1
    assert _call(dev, good, W.State(0.0, 0), out_stride=10) == -1
    # -2: geometries the CLI cannot run
    for b in (0, 5, 12):
        p = W.Params(5.0, b, TAU, 48000)
        assert _call(dev, p, W.State(0.0, 0)) == -2 and W.outputs(dev, p, s0, 2048)[0] == -2
    assert W.replay(5.0, 18, 18) is not None and W.replay(5.0, 18, 36) is None    # B = 18: the second call would consume nothing
    assert W.outputs(dev, W.Params(5.0, 18, TAU, 48000), s0, 18)[0] > 0
    assert W.outputs(dev, W.Params(5.0, 18, TAU, 48000), s0, 36)[0] == -2
    # a call that would consume more than B: the first such call of the brute-force replay is where the bank starts refusing
    for rate in (40.0, 25.0):
        n = 1024
        while (r := W.replay(rate, 1024, n)) is not None:
            n = r[1] + 1024                                              # exactly one call more
            assert n < 1024 * 400
        n_ok = n - 1                                                     # the longest input whose calls all run
        assert W.replay(rate, 1024, n_ok) is not None
        p = W.Params(rate, 1024, TAU, 48000)
        assert W.outputs(dev, p, s0, n_ok)[0] == W.replay(rate, 1024, n_ok)[0]
        st = W.State(0.0, 0)
        assert _call(dev, p, st, rows=1, n=n_ok + 1, out_stride=n_ok) == -2
        assert (st.where, st.audio) == (0.0, 0)                          # a refused call leaves the state as it was
    for rate in (16.0, 5.0, 1.25):
        assert W.replay(rate, 1024, 300 * 1024) is not None
    # rates far beyond B: the first call overruns, however large the rate (no int overflow in the replay)
    for rate in (1025.0, 1e6, 3e9, 1e30, 3.4028235e38):
        p = W.Params(rate, 1024, TAU, 48000)
        assert W.replay(rate, 1024, 2048) is None
        st = W.State(0.0, 0)
        assert _call(dev, p, st) == -2 and W.outputs(dev, p, s0, 2048)[0] == -2
        assert (st.where, st.audio) == (0.0, 0)
        assert W.outputs(dev, p, s0, 1023) == (0, 0)                        # no call runs
