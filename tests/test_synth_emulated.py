"""CPU tier of the synthesis bank (csdr_b200/csrc/synth.cu): the whole emulated library (tests/host_shim/emul_build.build_full_once) runs the
shipped kernels and the C ABI thread by thread.  csdrb_synth_bank_cc must equal the numpy restatement of tests/synth/synth.py bit for bit, samples
and carried phases, and lie within its float64 bound of the compiled reference composition.  Covered: I in {1, 2, 3, 5, 50, 256}; T from 1 (no
term) through the register window (h <= 8) to the general path, with taps in shared memory and beyond 8192; C in {1, 2, 3, 31, 32, 33, 100, 257}
(ragged warps, more than one CTA of channels, trees that are not powers of two); rates 0, +-0.5, +-1e-4 and |r| > 1; chunk in {1, 7, 1024} with
offsets inside a chunk; n below one group; random block cuts through the streaming object; NaN/Inf locality; every refusal of the ABI."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "synth"))
sys.path.insert(0, str(ROOT))
import emul_build  # noqa: E402
import synth  # noqa: E402
from oracle.pyoracle import Oracle, Ref  # noqa: E402

needs_ref = pytest.mark.skipif(not synth.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built")
RATES = [0.0, 0.5, -0.5, 1e-4, -1e-4, 1.3, -2.7, 0.085, -0.31, 0.2]

# (channels, I, T, n, chunk, offset): h = ceil((T-1)/I) picks the path
CASES = [
    (1, 1, 1, 40, 7, 3),              # h = 0: no term at all, general path
    (2, 1, 5, 60, 1024, 0),           # I = 1, h = 4
    (3, 2, 17, 50, 7, 6),             # h = 8, the widest register window
    (31, 3, 40, 30, 1024, 1000),      # h = 13: general path, taps in shared memory
    (32, 5, 41, 30, 1, 0),            # chunk 1: every output reseeds
    (33, 50, 401, 12, 1024, 17),      # the flagship geometry, a ragged second warp
    (100, 256, 2049, 11, 1024, 500),  # I = 256, four warps of one CTA
    (257, 2, 2, 40, 7, 2),            # h = 1, two CTAs of channels: the upper tree levels in the second pass
    (5, 50, 9001, 190, 1024, 5),      # T > 8192: taps through the read-only cache
    (4, 5, 3, 20, 7, 0),              # T < I: phases with no term and phases with one
    (3, 256, 300, 6, 1024, 1023),     # h = 2, the last offset of a chunk
    (2, 3, 40, 10, 7, 0),             # n below one group (h = 13): nothing
    (3, 50, 401, 8, 1024, 0),         # n = h: nothing
]


def P(a):
    return a.ctypes.data


def same_bits(a, b):
    fa, fb = np.asarray(a).view(np.float32), np.asarray(b).view(np.float32)
    na, nb = np.isnan(fa), np.isnan(fb)
    return fa.shape == fb.shape and np.array_equal(na, nb) and np.array_equal(fa[~na].view(np.uint32), fb[~nb].view(np.uint32))


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _ = emul_build.build_full_once(tmp_path_factory)
    L = C.CDLL(str(lib))
    vp, lg, it, sz = C.c_void_p, C.c_long, C.c_int, C.c_size_t
    L.csdrb_synth_bank_scratch_bytes.argtypes = [it, it, it, it, it, it]; L.csdrb_synth_bank_scratch_bytes.restype = sz
    L.csdrb_synth_bank_cc.argtypes = [vp, lg, it, it, it, vp, it, vp, vp, it, it, vp, vp, sz, vp]
    L.csdrb_synth_bank_create.argtypes = [it, vp, it, vp, it, it]; L.csdrb_synth_bank_create.restype = vp
    L.csdrb_synth_bank_destroy.argtypes = [vp]
    L.csdrb_synth_bank_process.argtypes = [vp, vp, lg, it, vp, vp]
    L.csdrb_kernel_launches.restype = C.c_long
    L.csdrb_last_error.restype = C.c_char_p
    return L


@pytest.fixture(scope="module")
def ora():
    return Oracle()


def inputs(rng, ch, n, stride=None):
    stride = n if stride is None else stride
    x = np.full((ch, max(stride, 1)), np.nan, np.complex64)
    x[:, :n] = (rng.uniform(-1, 1, (ch, n)) + 1j * rng.uniform(-1, 1, (ch, n))).astype(np.complex64)
    return x


def rates_of(ch):
    return np.array([RATES[c % len(RATES)] for c in range(ch)], np.float32)


def run(L, x, n, rates, I, taps, phases, chunk, offset, stride=None, scratch_bytes=None, expect=None):
    """one csdrb_synth_bank_cc call on host buffers: (rc, y, phases after, output buffer with its sentinel tail)"""
    ch = x.shape[0]
    stride = x.shape[1] if stride is None else stride
    ora = Oracle()
    prm = np.array([ora.shift_addition_init(float(r)) for r in rates], np.float32)
    ph = np.array(phases, np.float32).copy()
    taps = np.ascontiguousarray(taps, np.float32)
    N = synth.nout_of(n, I, taps.size) if I >= 1 and n >= 0 and taps.size >= 1 else 0
    out = np.full(N + 8, 7.0 + 7.0j, np.complex64)
    sb = int(L.csdrb_synth_bank_scratch_bytes(ch, n, I, taps.size, chunk, offset)) if scratch_bytes is None else scratch_bytes
    scratch = np.zeros(max(sb, 16) + 256, np.uint8)
    sp = P(scratch) + (-P(scratch)) % 256
    rc = L.csdrb_synth_bank_cc(P(x), stride, ch, n, I, P(taps), taps.size, P(prm), P(ph), chunk, offset, P(out), sp, sb, None)
    if expect is not None:
        assert rc == expect, (rc, L.csdrb_last_error())
    return rc, out[:max(rc, 0)].copy(), ph, out


@pytest.mark.parametrize("case", CASES, ids=[f"C{c}-I{i}-T{t}-n{n}-chunk{k}-off{o}" for c, i, t, n, k, o in CASES])
def test_bank_equals_restatement(L, ora, case):
    ch, I, T, n, chunk, offset = case
    rng = np.random.default_rng(ch * 1000 + T)
    x = inputs(rng, ch, n, stride=n + 3)                                     # an odd stride: rows are not adjacent
    taps = rng.uniform(-1, 1, T).astype(np.float32)
    rates = rates_of(ch)
    ph0 = rng.uniform(-3.2, 3.2, ch).astype(np.float32)
    N = synth.nout_of(n, I, T)
    rc, y, ph, out = run(L, x, n, rates, I, taps, ph0, chunk, offset, expect=N)
    want, want_ph = synth.restate(ora, x[:, :n], rates, I, taps, ph0, chunk, offset)
    assert same_bits(y, want), f"{case}: first difference at output {int(np.flatnonzero(~np.isclose(y, want, rtol=0, atol=0))[0])}"
    assert same_bits(ph, want_ph), case
    assert np.all(out[N:] == np.complex64(7 + 7j)), "a store past the outputs"


def test_one_channel_is_the_channel(L, ora):
    """C = 1: y = Y0 exactly, the composition of fir_interpolate_cc and shift_addition_cc without a sum"""
    rng = np.random.default_rng(3)
    x = inputs(rng, 1, 300)
    taps = rng.uniform(-1, 1, 81).astype(np.float32)
    _, y, _, _ = run(L, x, 300, [0.085], 5, taps, [0.0], 1024, 0)
    _, _, Y = synth.restate(ora, x, [0.085], 5, taps, None, 1024, 0, per_channel=True)
    assert same_bits(y, Y[0])


def test_three_channels_sum_as_pairs_then_the_third(L, ora):
    rng = np.random.default_rng(4)
    x = inputs(rng, 3, 40)
    taps = rng.uniform(-1, 1, 17).astype(np.float32)
    _, y, _, _ = run(L, x, 40, [0.1, -0.2, 0.3], 2, taps, np.zeros(3), 7, 0)
    _, _, Y = synth.restate(ora, x, [0.1, -0.2, 0.3], 2, taps, None, 7, 0, per_channel=True)
    assert same_bits(y, (Y[0] + Y[1]) + Y[2])


@needs_ref
@pytest.mark.parametrize("case", [CASES[2], CASES[5], CASES[7], CASES[8]], ids=["h8", "flagship", "two-ctas", "long-taps"])
def test_bank_within_bound_of_reference(L, case):
    ch, I, T, n, chunk, offset = case
    rng = np.random.default_rng(11 + ch)
    x = inputs(rng, ch, n)
    taps = synth.tx.ref_lowpass(T, 0.5 / I)
    rates = rates_of(ch)
    ph0 = rng.uniform(-3.1, 3.1, ch).astype(np.float32)
    _, y, _, _ = run(L, x, n, rates, I, taps, ph0, chunk, offset)
    want, Y = synth.ref_compose(Ref(), x, rates, I, taps, ph0, chunk, offset)
    b = synth.bound(x, rates, I, taps, Y, chunk)
    err = np.abs(y.astype(np.complex128) - want)
    assert np.all(err <= b), f"{case}: output {int(np.argmax(err / b))} errs by {err.max():.3e}"


@pytest.mark.parametrize("chunk", [7, 1024])
def test_streaming_cuts_equal_one_call(L, chunk):
    """random block cuts through csdrb_synth_bank_process: each call consumes G inputs, the caller presents the other n - G again"""
    rng = np.random.default_rng(chunk)
    ch, I, T, total = 5, 3, 40, 400
    x = inputs(rng, ch, total)
    taps = rng.uniform(-1, 1, T).astype(np.float32)
    rates = rates_of(ch)
    _, whole, ph_whole, _ = run(L, x, total, rates, I, taps, np.zeros(ch), chunk, 0)
    bank = L.csdrb_synth_bank_create(ch, P(rates), I, P(taps), T, chunk)
    assert bank, L.csdrb_last_error()
    got, pos = [], 0
    try:
        while pos < total:
            n = min(total - pos, int(rng.integers(1, 60)))
            blk = np.ascontiguousarray(x[:, pos:pos + n])
            out = np.zeros(max(n * I, 1), np.complex64)
            rc = L.csdrb_synth_bank_process(bank, P(blk), n, n, P(out), None)
            assert rc >= 0 and rc % I == 0, L.csdrb_last_error()
            got.append(out[:rc])
            pos += rc // I
            if pos + synth.h_of(I, T) >= total:
                break
    finally:
        L.csdrb_synth_bank_destroy(bank)
    assert same_bits(np.concatenate(got), whole)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf], ids=["nan", "inf", "-inf"])
def test_nonfinite_input_stays_local(L, ora, bad):
    """a NaN or Inf in channel c at input k makes non-finite exactly the outputs the restatement makes non-finite; every other output keeps
    the clean run's bits"""
    rng = np.random.default_rng(21)
    ch, I, T, n = 33, 5, 41, 40
    x = inputs(rng, ch, n)
    taps = rng.uniform(-1, 1, T).astype(np.float32)
    rates = rates_of(ch)
    _, clean, _, _ = run(L, x, n, rates, I, taps, np.zeros(ch), 7, 3)
    x[17, 20] = bad
    _, dirty, ph, _ = run(L, x, n, rates, I, taps, np.zeros(ch), 7, 3)
    want, want_ph = synth.restate(ora, x, rates, I, taps, None, 7, 3)
    assert same_bits(dirty, want) and same_bits(ph, want_ph)
    hit = ~np.isfinite(want)
    assert hit.any() and hit.sum() < hit.size // 2
    assert same_bits(dirty[~hit], clean[~hit])


def test_refusals_launch_nothing(L):
    rng = np.random.default_rng(5)
    x = inputs(rng, 2, 40)
    taps = rng.uniform(-1, 1, 17).astype(np.float32)
    ok = dict(n=40, rates=[0.1, 0.2], I=2, taps=taps, phases=[0.5, -0.5], chunk=7, offset=0)
    bad = [dict(I=0), dict(taps=taps[:0]), dict(n=-1), dict(chunk=0), dict(offset=-1), dict(offset=7), dict(stride=39),
           dict(scratch_bytes=16)]
    for b in bad:
        a = dict(ok, **b)
        stride = a.pop("stride", None)
        sb = a.pop("scratch_bytes", None)
        before = L.csdrb_kernel_launches()
        rc, _, ph, out = run(L, x, a["n"], a["rates"], a["I"], a["taps"], a["phases"], a["chunk"], a["offset"], stride=stride, scratch_bytes=sb)
        assert rc == -1 and L.csdrb_last_error(), b
        assert L.csdrb_kernel_launches() == before, b
        assert np.array_equal(ph, np.float32([0.5, -0.5])) and np.all(out == np.complex64(7 + 7j)), b
    # no channel, more outputs than an int counts, a null pointer
    prm = np.zeros((1, 3), np.float32); ph = np.zeros(1, np.float32); s = np.zeros(64, np.uint8); o = np.zeros(4, np.complex64)
    assert L.csdrb_synth_bank_cc(P(x), 40, 0, 40, 2, P(taps), 17, P(prm), P(ph), 7, 0, P(o), P(s), 64, None) == -1
    assert L.csdrb_synth_bank_cc(P(x), 1 << 30, 1, 1 << 30, 4, P(taps), 17, P(prm), P(ph), 7, 0, P(o), P(s), 64, None) == -1
    assert b"2^31" in L.csdrb_last_error()
    assert L.csdrb_synth_bank_cc(None, 40, 1, 40, 2, P(taps), 17, P(prm), P(ph), 7, 0, P(o), P(s), 64, None) == -1
    rates = np.zeros(2, np.float32)
    for args in [(0, P(rates), 2, P(taps), 17, 1024), (2, P(rates), 0, P(taps), 17, 1024), (2, P(rates), 2, P(taps), 0, 1024),
                 (2, P(rates), 2, P(taps), 17, 0), (2, None, 2, P(taps), 17, 1024)]:
        assert not L.csdrb_synth_bank_create(*args), args
    assert L.csdrb_synth_bank_process(None, P(x), 40, 40, P(o), None) == -1
