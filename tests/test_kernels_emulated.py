"""CPU tier: the SHIPPED CUDA sources executed thread by thread on the host.

tests/host_shim/cuda_emul.h turns every CUDA thread of a CTA into a fiber and __syncthreads() / __syncwarp() / bar.sync / mbarrier
waits into real barriers between fibers; tests/host_shim/emul_build.py compiles each csdr_b200/csrc/*.cu file with g++ after two textual
rewrites (`k<<<...>>>(...)` and `extern __shared__`), so kernels AND launchers run with their real index arithmetic, shared-memory
traffic, barrier structure, alignment requirements (128-bit stores and bulk copies are checked) and IEEE single-precision rounding -- in a
container without a GPU.  Every test is repeated under three fiber scheduling orders so that a missing barrier produces a wrong result
in at least one of them.  Test infrastructure only: nothing in the product can reach it, and the product still fails loudly without a
GPU (tests/test_abi.py).  It complements the -m gpu parity tests, it does not replace them.
"""
import ctypes as C
import os
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
os.environ.setdefault("CSDRB_SHIFT_SLICE_MIN", "3000")      # the K2 launcher cuts its chain into slices from 2 x 3000 chunk-channels on (product default: 2 x 768 x 64)
import emul_build  # noqa: E402

from oracle.pyoracle import rel_rms  # noqa: E402

GOLD = np.load(Path(__file__).parent / "golden" / "hotpath_golden.npz")
ORDERS = ["alternate", "reverse", "random"]
_built = {}


def _lib(tmp_path_factory, cu, order, host_c=()):
    """build once per .cu file, load one private copy per scheduling order (the order is read when a copy initialises)"""
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    if cu not in _built:
        out = tmp_path_factory.mktemp("emul_" + Path(cu).stem)
        lib, names = emul_build.build_file(out, cu, host_c=host_c)
        _built[cu] = (Path(lib._name), names, lib)
    so, names, proto_lib = _built[cu]
    copy = so.with_name(f"{so.stem}_{order}.so")
    if not copy.exists():
        shutil.copy(so, copy)
    os.environ["CUDA_EMUL_ORDER"] = order
    lib = C.CDLL(str(copy))
    for n in names:
        f = getattr(lib, "emul_" + n); g = getattr(proto_lib, "emul_" + n)
        f.argtypes, f.restype = g.argtypes, g.restype
    lib.emul_last_error.restype = C.c_char_p; lib.emul_barriers.restype = C.c_long
    return lib


def _fixture(cu, host_c=()):
    @pytest.fixture(scope="module", params=ORDERS)
    def fx(request, tmp_path_factory):
        return _lib(tmp_path_factory, cu, request.param, host_c)
    return fx


elementwise = _fixture("elementwise.cu")
shift = _fixture("shift.cu")
audio = _fixture("audio.cu", ("csdr_b200/host/firdes.c",))
ddc = _fixture("ddc_bank.cu")
fir = _fixture("fir_decimate.cu")
fft = _fixture("fft.cu")


def P(a):
    return a.ctypes.data


# ---- write guards: every array made by Z()/ZL() sits between two canary regions that are checked when the test ends -------------------
_GUARD = 512
_guarded = []


def Z(shape, dtype=np.float64):
    """np.zeros with canaries before and after (and 16-byte alignment): an out-of-bounds write of a kernel trips the check below"""
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    raw = np.full(n + 2 * _GUARD + 32, 0xA5, np.uint8)
    off = _GUARD + ((-(raw.ctypes.data + _GUARD)) % 16)
    raw[off:off + n] = 0
    _guarded.append((raw, off, n))
    return raw[off:off + n].view(dtype).reshape(shape)


def ZL(a):
    return Z(a.shape, a.dtype)


@pytest.fixture(autouse=True)
def _check_guards():
    _guarded.clear()
    yield
    for raw, off, n in _guarded:
        assert np.all(raw[:off] == 0xA5) and np.all(raw[off + n:] == 0xA5), "a kernel wrote outside one of its buffers"
    _guarded.clear()


def _cplx(rng, *shape, amp=1.0):
    return ((rng.uniform(-1, 1, shape) + 1j * rng.uniform(-1, 1, shape)) * amp).astype(np.complex64)


def _aligned(shape, dtype):
    """16-byte aligned array (cudaMalloc gives 256; the kernels' 128-bit paths need 16)"""
    n = int(np.prod(shape)); item = np.dtype(dtype).itemsize
    raw = np.zeros(n * item + 32, np.uint8)
    off = (-raw.ctypes.data) % 16
    return raw[off:off + n * item].view(dtype).reshape(shape)


# ------------------------------------------------------------------------------------------------------------------ K1 / K4 / tail / spectrum
def test_k1_conversions_bit_exact(elementwise, oracle):
    codes = np.arange(256, dtype=np.uint8)
    rng = np.random.default_rng(0)
    for n in (256, 1, 15, 16, 17, 4099, 20_000):
        src = (codes if n == 256 else rng.integers(0, 256, n, dtype=np.uint8))
        u8 = _aligned(n, np.uint8); u8[:] = src; out = _aligned(n, np.float32)
        assert elementwise.emul_launch_convert_u8_f(P(u8), P(out), n) >= 0
        assert np.array_equal(out, oracle.convert_u8_f(u8)), n
        s16 = _aligned(n, np.int16); s16[:] = rng.integers(-32768, 32768, n); out = _aligned(n, np.float32)
        assert elementwise.emul_launch_convert_s16_f(P(s16), P(out), n) >= 0
        assert np.array_equal(out, oracle.convert_s16_f(s16)), n
        f = _aligned(n, np.float32); f[:] = rng.standard_normal(n) * 0.7
        if n > 16:
            f[:8] = [1.0, -1.0, 1.5, -1.5, 3.0, np.nan, np.inf, -np.inf]  # full scale, wrap-around, NaN, infinities
        out = _aligned(n, np.int16)
        assert elementwise.emul_launch_convert_f_s16(P(f), P(out), n) >= 0
        assert np.array_equal(out, oracle.convert_f_s16(f)), n
    assert np.array_equal(oracle.convert_u8_f(codes), GOLD["u8_table"]) if "u8_table" in GOLD.files else True


def test_k4_fmdemod_bank_and_audio_tail(elementwise, oracle):
    rng = np.random.default_rng(1)
    ch, n = 3, 10_001
    x = _cplx(rng, ch, n + 1)[:, :n]                                       # odd length inside an even stride
    stride = x.strides[0] // 8
    last = _cplx(rng, ch); last_out = Z(ch, np.complex64)
    out = Z((ch, n + 3), np.float32)
    assert elementwise.emul_launch_fmdemod_quadri_bank(P(x), stride, P(out), out.shape[1], ch, n, P(last), P(last_out)) >= 0
    for c in range(ch):
        want, wl = oracle.fmdemod_quadri_cf(np.ascontiguousarray(x[c]), complex(last[c]))
        assert np.abs(out[c, :n] - want).max() <= 2e-7 and last_out[c] == np.complex64(wl)
    f = _aligned(20_003, np.float32); f[:] = rng.uniform(-2, 2, f.size); f[7] = np.nan; f[9] = np.inf; f[11] = -np.inf
    out = _aligned(f.size, np.float32)
    assert elementwise.emul_launch_limit_ff(P(f), P(out), f.size, 0.7) >= 0
    assert np.array_equal(out, oracle.limit_ff(f, 0.7))                    # NaN -> +max like the reference build


def test_spectrum_side_path(elementwise, oracle):
    rng = np.random.default_rng(2)
    size, rows = 1000, 5
    x = _cplx(rng, rows * size); w = oracle.precalculate_window(size, "BLACKMAN"); out = ZL(x)
    assert elementwise.emul_launch_apply_window_rows(P(x), P(out), P(w), size, rows) >= 0
    want = np.concatenate([oracle.apply_precalculated_window_c(x[r * size:(r + 1) * size], w) for r in range(rows)])
    assert np.array_equal(out, want)
    p = Z(x.size, np.float32)
    assert elementwise.emul_launch_power(P(x), None, P(p), x.size, -70.0, 0) >= 0
    assert np.abs(p - oracle.logpower_cf(x, -70.0)).max() <= 2e-5


def test_ima_adpcm_rows_bit_exact(elementwise, oracle):
    """8(f) rank 4: the audio / waterfall ADPCM encoder, one thread per row, integer arithmetic -> identical bytes and states"""
    rng = np.random.default_rng(4)
    rows, n = 37, 2050
    x = (rng.standard_normal((rows, n)) * rng.choice([10, 300, 5000, 40000], (rows, 1))).clip(-32768, 32767).astype(np.int16)
    st = np.stack([rng.integers(0, 89, rows), rng.integers(-32768, 32768, rows)], 1).astype(np.int32); st0 = st.copy()
    out = Z((rows, n // 2), np.uint8)
    assert elementwise.emul_launch_adpcm_encode_rows(P(x), n, P(out), n // 2, rows, n, P(st)) >= 0
    for r in range(rows):
        want, (wi, wp) = oracle.encode_ima_adpcm_i16_u8(x[r], int(st0[r, 0]), int(st0[r, 1]))
        assert np.array_equal(out[r], want) and (st[r, 0], st[r, 1]) == (wi, wp), r
    for fft_size in (16, 511, 512, 2048):
        db = rng.uniform(-130, 10, (rows, fft_size)).astype(np.float32); db[0, :3] = [np.nan, 400.0, -400.0]      # beyond +-327.67 dB the short wraps, like the reference
        out = Z((rows, (fft_size + 10) // 2), np.uint8)
        assert elementwise.emul_launch_compress_fft_adpcm_rows(P(db), fft_size, P(out), out.shape[1], rows, fft_size) >= 0
        assert np.array_equal(out, oracle.compress_fft_adpcm_f_u8(db, fft_size)), fft_size


# ------------------------------------------------------------------------------------------------------------------ K2 and shift variants
@pytest.mark.parametrize("n,chunk", [(16384 + 777, 1024), (5000, 1000), (4096, 4096), (3000, 0), (1001, 37), (120 * 1024 + 5, 1024), (9000, 64), (9003, 8), (2 * 4_001 + 1, 2)])   # from the sixth on: > 96 chunks, the chain runs on its wrap table (phase_table.cuh); the last two: 1 126 / 4 002 chunks x 6 channels = two / three chain slices on the side stream (CSDRB_SHIFT_SLICE_MIN below)
def test_k2_shift_bank_replays_reference_chain(shift, oracle, n, chunk):
    rng = np.random.default_rng(n)
    rates = np.array([-0.41, -0.085, 0.0, 0.2, 0.4999, 1e-4], np.float32)
    ch = rates.size
    x = _cplx(rng, n)
    params = np.array([oracle.shift_addition_init(float(r)) for r in rates], np.float32)
    ph0 = rng.uniform(-3, 3, ch).astype(np.float32); ph = ph0.copy()
    out = Z((ch, n), np.complex64)
    sb = shift.emul_shift_bank_scratch_bytes(ch, n, chunk); scratch = Z(sb + 16, np.uint8)
    assert shift.emul_launch_shift_addition_bank(P(x), 0, P(out), n, ch, n, P(params), P(ph), chunk, P(scratch), sb) >= 0, shift.emul_last_error()
    for c, r in enumerate(rates):
        want, wph = oracle.shift_addition_cc(x, float(r), float(ph0[c]), chunk or None)
        assert np.float32(wph) == ph[c], (c, wph, ph[c])                  # carried phase: bit-exact (exact wrap fast-forward included)
        assert np.array_equal(out[c].view(np.uint32), want.view(np.uint32)), c      # the host's libm seeds both: the same bits (tests/shift_ref.py)
    # shift_addfast: same decomposition, one recursion step per four samples, n % 4 tails untouched
    steps = np.stack([oracle.shift_addfast_init(float(r)) for r in rates]); ph = ph0.copy(); out[:] = 0
    assert shift.emul_launch_shift_addfast_bank(P(x), 0, P(out), n, ch, n, P(steps), P(ph), chunk, P(scratch), sb) >= 0
    for c, r in enumerate(rates):
        want, wph = oracle.shift_addfast_cc(x, float(r), float(ph0[c]), chunk or None)
        assert np.float32(wph) == ph[c] and np.array_equal(out[c].view(np.uint32), want.view(np.uint32)), c


def test_k2_decimating_and_unroll(shift, oracle):
    rng = np.random.default_rng(5)
    n, dec = 10_007, 7
    rates = np.array([0.1, -0.3, 0.05], np.float32); ch = rates.size
    xs = _cplx(rng, ch, n)
    params = np.array([oracle.shift_addition_init(float(np.float32(r) * dec)) for r in rates], np.float32)      # decimating_shift_addition_init
    remain = np.array([0, 3, 6], np.int32); ph = np.array([0.0, 1.0, -2.0], np.float32); outsz = Z(ch, np.int32)
    r0, p0 = remain.copy(), ph.copy()
    out = Z((ch, n // dec + 2), np.complex64)
    assert shift.emul_launch_decimating_shift_bank(P(xs), n, P(out), out.shape[1], ch, n, P(params), dec, P(remain), P(ph), P(outsz)) >= 0
    for c, r in enumerate(rates):
        want, (wr, wp) = oracle.decimating_shift_addition_cc(xs[c], float(r), dec, int(r0[c]), float(p0[c]))
        assert outsz[c] == want.size and remain[c] == wr and ph[c] == np.float32(wp)
        assert np.array_equal(out[c, :want.size].view(np.uint32), want.view(np.uint32))
    # shift_unroll: table of 1024 steps per channel, one reference call per 1024 samples
    size = 1024; n = 5000
    x = _cplx(rng, n)
    tabs = [np.empty(size, np.float32) for _ in range(2 * ch)]
    for c, r in enumerate(rates):
        oracle.L.oracle_shift_unroll_init(float(r), size, tabs[2 * c].ctypes.data_as(C.POINTER(C.c_float)), tabs[2 * c + 1].ctypes.data_as(C.POINTER(C.c_float)))
    dsin = np.stack(tabs[0::2]); dcos = np.stack(tabs[1::2])
    params = np.array([oracle.shift_addition_init(float(r)) for r in rates], np.float32)
    ph = Z(ch, np.float32); out = Z((ch, n), np.complex64)
    sb = shift.emul_shift_bank_scratch_bytes(ch, n, size); scratch = Z(sb + 16, np.uint8)
    assert shift.emul_launch_shift_unroll_bank(P(x), 0, P(out), n, ch, n, P(params), P(dsin), P(dcos), size, size, P(ph), P(scratch), sb) >= 0
    for c, r in enumerate(rates):
        want, wph = oracle.shift_unroll_cc(x, float(r), 0.0, size)
        assert np.float32(wph) == ph[c] and np.array_equal(out[c].view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("n", [1, 255, 256, 257, 10_001, 40_000])
def test_shift_math_bank(shift, oracle, n):
    """one rounded phase addition per sample: the per-channel chain thread drops a seed every 256 samples, the lanes re-walk their segment"""
    rng = np.random.default_rng(n)
    rates = np.array([-0.5, -0.31, -0.085, 0.0, 1e-4, 0.2, 0.4999, 0.5], np.float32); ch = rates.size
    x = _cplx(rng, n)
    ph0 = np.array([0.0, 3.0, -7.5, 100.0, 6.2831855, 1.0, 2.0, -0.0], np.float32); ph = ph0.copy()   # starts outside [0, 2*PI] take the reference's loops
    out = Z((ch, n), np.complex64)
    sb = shift.emul_shift_math_scratch_bytes(ch, n); scratch = Z(sb + 16, np.uint8)
    assert shift.emul_launch_shift_math_bank(P(x), 0, P(out), n, ch, n, P(rates), P(ph), P(scratch), sb) >= 0, shift.emul_last_error()
    for c, r in enumerate(rates):
        want, wph = oracle.shift_math_cc(x, float(r), float(ph0[c]))
        assert np.float32(wph).view(np.uint32) == ph[c].view(np.uint32), (c, wph, ph[c])    # the carried phase, bit for bit
        assert np.array_equal(out[c].view(np.uint32), want.view(np.uint32)), c


@pytest.mark.parametrize("n,size", [(257, 65536), (10_001, 65536), (20_000, 1024), (5_000, 100)])
def test_shift_table_bank_bit_exact(shift, oracle, n, size):
    """the table-lookup mixer: same phase chain as shift_math_cc, index arithmetic of the reference BUILD (reciprocal multiplies) -> identical samples"""
    rng = np.random.default_rng(n + size)
    rates = np.array([-0.5, -0.31, -0.085, 0.0, 1e-4, 0.2, 0.4999, 0.5], np.float32); ch = rates.size
    x = _cplx(rng, n); table = oracle.shift_table_init(size)
    ph0 = np.array([0.0, 3.0, 1.5707964, 6.2831855, 0.5, 1.0, 2.0, 4.7], np.float32); ph = ph0.copy()
    out = Z((ch, n), np.complex64)
    sb = shift.emul_shift_math_scratch_bytes(ch, n); scratch = Z(sb + 16, np.uint8)
    assert shift.emul_launch_shift_table_bank(P(x), 0, P(out), n, ch, n, P(rates), P(ph), P(table), size, P(scratch), sb) >= 0, shift.emul_last_error()
    for c, r in enumerate(rates):
        want, wph, _bad = oracle.shift_table_cc(x, float(r), table, float(ph0[c]))
        assert np.float32(wph).view(np.uint32) == ph[c].view(np.uint32), c
        assert np.array_equal(out[c], want), (c, int(np.sum(out[c] != want)))


# ------------------------------------------------------------------------------------------------------------------ K5 / K6 / audio tail
@pytest.mark.parametrize("rate,points,n", [(5.0, 12, 20_000), (1.25, 12, 9_000), (2.5, 4, 5_001), (7.123, 16, 30_000)])
def test_k5_fractional_decimator_bit_exact(audio, oracle, rate, points, n):
    rng = np.random.default_rng(int(rate * 100))
    ch = 3
    x = rng.uniform(-1, 1, (ch, n)).astype(np.float32)
    cap = int(n / rate) + 8
    out = Z((ch, cap), np.float32)
    state = Z((ch, 3), np.int32); state[:, 0] = np.array([points // 2 - 1], np.float32).view(np.int32)[0]       # where = -xifirst at init
    sb = audio.emul_fracdec_scratch_bytes(ch, n, rate); scratch = Z(sb + 16, np.uint8)
    assert audio.emul_launch_fractional_decimator_bank(P(x), n, P(out), cap, ch, n, rate, points, None, 0, P(state), P(scratch), sb) >= 0, audio.emul_last_error()
    for c in range(ch):
        want = oracle.fractional_decimator_ff(x[c], rate, points)
        assert state[c, 2] == want.size                                   # the float position chain picked the same indices ...
        assert np.array_equal(out[c, :want.size], want)                   # ... and the Lagrange evaluation is the same rounding sequence


def test_k6_fastagc_and_deemphasis_bit_exact(audio, oracle):
    rng = np.random.default_rng(7)
    ch, block, nblocks = 4, 1024, 9
    env = np.repeat(rng.uniform(0.001, 1.0, nblocks).astype(np.float32), block)
    x = np.stack([rng.uniform(-1, 1, env.size).astype(np.float32) * env * s for s in (1.0, 0.01, 0.0, 30.0)])
    out = ZL(x); state = Z((ch, 3), np.float32); hist = Z((ch, 2, block), np.float32)
    sb = audio.emul_fastagc_scratch_bytes(ch, nblocks); scratch = Z(sb + 16, np.uint8)
    assert audio.emul_launch_fastagc_bank(P(x), x.shape[1], P(out), out.shape[1], ch, block, nblocks, 0.8, P(state), P(hist), P(scratch), sb) >= 0
    for c in range(ch):
        assert np.array_equal(out[c], oracle.fastagc_ff(x[c], block, 0.8), equal_nan=True), c
    xb = rng.uniform(-1, 1, (37, 5_001)).astype(np.float32); last = np.linspace(-0.5, 0.5, 37).astype(np.float32); last[3] = np.nan
    l0 = last.copy(); yb = ZL(xb)
    assert audio.emul_launch_deemphasis_wfm_bank(P(xb), xb.shape[1], P(yb), yb.shape[1], 37, xb.shape[1], 75e-6, 240000, P(last)) >= 0
    for c in range(37):
        want, wl = oracle.deemphasis_wfm_ff(xb[c], 75e-6, 240000, float(l0[c]))
        assert np.array_equal(yb[c], want) and np.float32(wl) == last[c]


@pytest.mark.parametrize("block", [1024, 1000, 77, 2048])
def test_k6_fused_run_kernel_and_s16_output(audio, oracle, block):
    """blocks <= 1024 take the one-pass kernel (a CTA walks runs of 16 blocks, peaks rolling, two blocks in registers): 37 blocks = three runs, streamed in
    two calls; with the s16 epilogue the result is convert_f_s16(fastagc_ff(x)) bit for bit.  2048 has no fused kernel (the float bank falls back)."""
    rng = np.random.default_rng(block)
    ch, nb = 3, 37
    x = (rng.uniform(-1, 1, (ch, nb * block)) * np.array([[1.0], [0.02], [3.0]])).astype(np.float32)
    x[1, 3 * block:5 * block] = 0.0
    cut = 20 * block
    state = Z((ch, 3), np.float32); hist = Z((ch, 2, block), np.float32)
    sb = audio.emul_fastagc_scratch_bytes(ch, nb); scratch = Z(sb + 16, np.uint8)
    outf = Z((ch, nb * block), np.float32); s16 = Z((ch, nb * block), np.int16)
    st2 = Z((ch, 3), np.float32); h2 = Z((ch, 2, block), np.float32)
    for lo, hi in ((0, cut), (cut, nb * block)):
        xs = np.ascontiguousarray(x[:, lo:hi]); n = (hi - lo) // block
        of = Z((ch, hi - lo), np.float32); os_ = Z((ch, hi - lo), np.int16)
        assert audio.emul_launch_fastagc_bank(P(xs), xs.shape[1], P(of), of.shape[1], ch, block, n, 0.8, P(state), P(hist), P(scratch), sb) >= 0
        rc = audio.emul_launch_fastagc_bank_s16(P(xs), xs.shape[1], P(os_), os_.shape[1], ch, block, n, 0.8, P(st2), P(h2), P(scratch), sb)
        assert rc == (-2 if block > 1024 else 2)
        outf[:, lo:hi] = of; s16[:, lo:hi] = os_
    for c in range(ch):
        want = oracle.fastagc_ff(x[c], block, 0.8)
        assert np.array_equal(outf[c], want), c
        if block <= 1024:
            assert np.array_equal(s16[c], oracle.convert_f_s16(want)), c


@pytest.mark.parametrize("rate", [48000, 44100, 11025, 8000])
def test_nfm_deemphasis_fir_and_fused_limiter(audio, oracle, rate):
    taps = GOLD[f"nfm_taps_{rate}"]; T = taps.size
    rng = np.random.default_rng(rate)
    for n in (T + 1, T + 1024, T + 1025, 5000):
        ch = 2
        x = rng.uniform(-2.5, 2.5, (ch, n)).astype(np.float32); x[0, min(17, n - 1)] = np.nan
        out = np.full((ch, n), np.nan, np.float32)
        rc = audio.emul_launch_deemphasis_nfm_bank(P(x), n, P(out), n, ch, n, rate, 1.0)
        assert rc == n - T
        for c in range(ch):
            want = oracle.deemphasis_nfm_ff(oracle.limit_ff(x[c], 1.0), taps)
            assert np.abs(out[c, :rc] - want).max() <= 1e-6 * np.abs(taps).sum(), (n, c)
    y = Z(GOLD["nfm_in"].size, np.float32); xin = np.ascontiguousarray(GOLD["nfm_in"])
    rc = audio.emul_launch_deemphasis_nfm_bank(P(xin), xin.size, P(y), y.size, 1, xin.size, rate, 0.0)
    assert rel_rms(y[:rc], GOLD[f"nfm_out_{rate}"]) < 1e-5                # the compiled reference's output
    assert audio.emul_launch_deemphasis_nfm_bank(P(xin), xin.size, P(y), y.size, 1, xin.size, 22050, 0.0) == 0


# ------------------------------------------------------------------------------------------------------------------ K3: the headline kernel
@pytest.mark.parametrize("D,T,n,variant", [(10, 199, 9_999, -1), (10, 199, 30_011, 0), (10, 199, 30_011, 3), (10, 199, 4_000, 7), (10, 79, 20_000, -1),
                                           (50, 801, 70_000, -1), (7, 79, 5_001, -1), (10, 199, 199, -1), (10, 199, 208, -1), (10, 199, 150, -1)])
def test_k3_fir_decimate_bank(fir, oracle, D, T, n, variant):
    """bulk-copy tile loads on an mbarrier, polyphase register tiling, FMA pairs, pair reduction through named barriers, streaming stores --
    executed on the host against the oracle; n == T, n < T and ragged ends included."""
    rng = np.random.default_rng(D * 1000 + T + n)
    ch = 3
    stride = n + (n & 1)
    x = _aligned((ch, stride), np.complex64); x[:, :n] = _cplx(rng, ch, n); x[:, n:] = np.nan     # whatever follows a row must never be used
    taps = oracle.firdes_lowpass_f(T, 0.5 / D)
    n_out = (n - T) // D + 1 if n >= T else 0
    ostride = max(n_out + (n_out & 1), 2)
    out = _aligned((ch, ostride), np.complex64); out[:] = np.nan
    fp = taps.ctypes.data_as(C.c_void_p)
    rc = fir.emul_launch_fir_decimate_bank(P(x), stride, P(out), ostride, ch, n, D, fp, fp, 0, T, variant)          # "device" taps for the generic path: the same host array
    assert rc == n_out, fir.emul_last_error()
    for c in range(ch):
        want = oracle.fir_decimate_cc(np.ascontiguousarray(x[c, :n]), D, taps)
        assert want.size == n_out
        if n_out:
            assert rel_rms(out[c, :n_out], want) < 2e-6, (c, rel_rms(out[c, :n_out], want))


@pytest.mark.parametrize("D,T,n", [(10, 199, 40_007), (10, 79, 16_384 + 5), (50, 801, 30_011), (10, 199, 8321), (10, 199, 205)])
def test_k3_u8_front_end_equals_convert_then_filter(fir, oracle, D, T, n):
    """convert_u8_f | fir_decimate_cc in one kernel (csdr-fm:41): the samples the FIR sees are convert_u8_f's bit for bit, so the result must equal the cf32
    bank's on the converted stream EXACTLY (same kernel, same summation order), and the oracle's within the usual bar"""
    rng = np.random.default_rng(n)
    ch = 3
    stride = (n + 7) & ~7
    u8 = _aligned((ch, stride, 2), np.uint8); u8[:] = rng.integers(0, 256, u8.shape, dtype=np.uint8); u8[:, n:] = 0x5A      # row padding must not matter
    if n >= 256:
        u8[0, :256, 0] = np.arange(256); u8[0, :256, 1] = np.arange(255, -1, -1)                                               # every code on both components
    taps = oracle.firdes_lowpass_f(T, 0.5 / D)
    n_out = (n - T) // D + 1
    ostride = n_out + (n_out & 1)
    out = _aligned((ch, ostride), np.complex64); out[:] = np.nan
    fp = taps.ctypes.data_as(C.c_void_p)
    rc = fir.emul_launch_fir_decimate_bank_u8(P(u8), stride, P(out), ostride, ch, n, D, fp, T)
    assert rc == n_out, fir.emul_last_error()
    f = np.stack([oracle.convert_u8_f(np.ascontiguousarray(u8[c, :n]).reshape(-1)).view(np.complex64) for c in range(ch)])
    fs = n + (n & 1); xf = _aligned((ch, fs), np.complex64); xf[:] = 0; xf[:, :n] = f
    ref = _aligned((ch, ostride), np.complex64)
    assert fir.emul_launch_fir_decimate_bank(P(xf), fs, P(ref), ostride, ch, n, D, fp, fp, 0, T, -1) == n_out
    assert np.array_equal(out[:, :n_out], ref[:, :n_out])
    for c in range(ch):
        e = rel_rms(out[c, :n_out], oracle.fir_decimate_cc(np.ascontiguousarray(f[c]), D, taps))
        assert e < (2e-6 if n_out > 8 else 1e-5), (c, e)                     # a single, strongly cancelling output gets the contract's bar
    # a row stride that is not a multiple of 8 samples has no fused path: the launcher says so (-2) and the C ABI falls back to two launches
    assert fir.emul_launch_fir_decimate_bank_u8(P(u8), stride + 2, P(out), ostride, 1, n, D, fp, T) == -2


# ------------------------------------------------------------------------------------------------------------------ fused DDC bank (config 4)
@pytest.mark.parametrize("D,bw,demod", [(50, 0.005, 1), (10, 0.0201, 1), (10, 0.05, 0), (50, 0.005, 0)])
def test_fused_ddc_bank_matches_the_unfused_chain(ddc, oracle, D, bw, demod):
    T = oracle.firdes_filter_len(bw)
    taps = oracle.firdes_lowpass_f(T, 0.5 / D)
    n = 20_000 + 14
    rng = np.random.default_rng(D)
    t = np.arange(n)
    rates = np.array([-0.41, -0.27, -0.13, 0.01, 0.15, 0.29, 0.43], np.float32); ch = rates.size
    wide = sum(0.3 * np.exp(1j * (2 * np.pi * (-float(r)) * t + np.cumsum(0.05 * np.sin(2 * np.pi * t / (2000.0 + 100 * k))))) for k, r in enumerate(rates))
    x = _aligned(n, np.complex64); x[:] = (wide + 0.01 * (rng.normal(size=n) + 1j * rng.normal(size=n))).astype(np.complex64)
    params = np.array([oracle.shift_addition_init(float(r)) for r in rates], np.float32)
    ph = Z(ch, np.float32)
    n_out = (n - T) // D + 1
    stride = n_out + (n_out & 1)
    out = Z((ch, stride), np.float32 if demod else np.complex64)
    last_out = Z(ch, np.complex64); launches = C.c_int(0)
    sb = ddc.emul_ddc_bank_scratch_bytes(ch, n, 1024, 0); scratch = Z(sb + 64, np.uint8)
    fp = taps.ctypes.data_as(C.c_void_p)
    rc = ddc.emul_launch_ddc_bank(P(x), n, ch, P(params), P(ph), 1024, 0, D, fp, T, demod, P(out), stride, None, P(last_out) if demod else None, P(scratch), sb,
                                  C.addressof(launches))
    assert rc == n_out, ddc.emul_last_error()
    for c, r in enumerate(rates):
        sh, _ = oracle.shift_addition_cc(x, float(r), 0.0, 1024)
        base = oracle.fir_decimate_cc(sh, D, taps)
        want = oracle.fmdemod_quadri_cf(base)[0] if demod else base
        assert rel_rms(out[c, :n_out], want) < (1e-5 if demod else 2e-6), (c, rel_rms(out[c, :n_out], want))


# ------------------------------------------------------------------------------------------------------------------ K7 / K9 / K8
def test_k7_fft_every_size_both_directions(fft):
    rng = np.random.default_rng(0)
    for n in (2, 4, 8, 16, 32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384):
        x = _aligned((2, n), np.complex64); x[:] = _cplx(rng, 2, n); y = _aligned((2, n), np.complex64)
        for inv in (0, 1):
            b0 = fft.emul_barriers()
            assert fft.emul_launch_fft_c2c_batch(P(x), n, P(y), n, n, 2, inv) >= 0, fft.emul_last_error()
            if n == 4096:
                assert (fft.emul_barriers() - b0) // 2 == 4                # radix-16 passes from 32 points on: three passes at 4096 (four barriers per row)
            want = np.fft.ifft(x.astype(np.complex128), axis=1) * n if inv else np.fft.fft(x.astype(np.complex128), axis=1)
            assert rel_rms(y, want) < 1e-6, (n, inv)                      # same bar as tests/test_gpu_parity2.py::test_fft_all_sizes_vs_float64_dft
        buf = _cplx(rng, n + 3); out = Z(n + 3, np.complex64)
        off = 1 if (buf.ctypes.data % 16) == 0 else 0                     # a row that is only 8-byte aligned
        fft.emul_launch_fft_c2c_batch(P(buf[off:]), n, P(out[off:]), n, n, 1, 0)
        assert rel_rms(out[off:off + n], np.fft.fft(buf[off:off + n].astype(np.complex128))) < 1e-6
    assert fft.emul_barriers() > 100                                       # the barriers were real


def test_k7_apply_fir_fft_every_size(fft):
    """apply_fir_fft_cc's one-block kernel runs the radix-8 block_fft passes at every size: forward FFT, product with taps_fft, inverse FFT, /N, + the
    previous overlap, against float64"""
    rng = np.random.default_rng(16)
    for n in (2, 4, 8, 16, 32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384):
        ov = n // 4
        x = _cplx(rng, n); H = _cplx(rng, n); last = _cplx(rng, max(ov, 1)); out = Z(n, np.complex64)
        assert fft.emul_launch_apply_fir_fft(P(x), P(H), P(last), ov, P(out), n) >= 0, fft.emul_last_error()
        want = np.fft.ifft(np.fft.fft(x.astype(np.complex128)) * H.astype(np.complex128)); want[:ov] += last[:ov]
        assert rel_rms(out, want) < 1e-6, n


def _overlap_add(x, H, N, isz):
    nb = x.size // isz; out = Z(nb * isz + N - isz, np.complex128)
    for b in range(nb):
        blk = Z(N, np.complex128); blk[:isz] = x[b * isz:(b + 1) * isz]
        out[b * isz:b * isz + N] += np.fft.ifft(np.fft.fft(blk) * H)
    return out[:nb * isz], out[nb * isz:]


@pytest.mark.parametrize("N,isz,nb,bpc", [(4096, 2098, 5, 2), (4096, 2098, 3, 0), (512, 300, 7, 3), (64, 40, 9, 4), (256, 178, 6, 6), (1024, 224, 12, 5),
                                          (2048, 1500, 4, 2), (16, 9, 11, 3), (128, 128, 3, 2), (32, 1, 70, 16), (8192, 7000, 3, 2), (8, 5, 9, 4), (4, 3, 7, 2)])
def test_k9_overlap_add_bank(fft, N, isz, nb, bpc):
    """bandpass_fir_fft_cc block loop: CTA runs of `bpc` blocks (lead-in recomputation), overlap > input_size, no overlap, streaming tails."""
    rng = np.random.default_rng(N + isz)
    ch = 2
    x = _cplx(rng, ch, nb * isz); H = _cplx(rng, ch, N)
    y = ZL(x); tail = Z((ch, N), np.complex64)
    assert fft.emul_launch_olafir_bank(P(x), x.shape[1], P(y), y.shape[1], ch, N, isz, nb, P(H), N, P(tail), bpc) >= 0, fft.emul_last_error()
    for c in range(ch):
        want, wt = _overlap_add(x[c].astype(np.complex128), H[c].astype(np.complex128), N, isz)
        assert rel_rms(y[c], want) < 2e-6
        if N > isz:
            assert rel_rms(tail[c, :N - isz], wt) < 2e-6
    h = nb // 2                                                            # two calls carrying the tail == one call
    xa = np.ascontiguousarray(x[:, :h * isz]); xb = np.ascontiguousarray(x[:, h * isz:]); ya = ZL(xa); yb = ZL(xb)
    t = Z((ch, N), np.complex64)
    fft.emul_launch_olafir_bank(P(xa), xa.shape[1], P(ya), ya.shape[1], ch, N, isz, h, P(H), N, P(t), bpc)
    fft.emul_launch_olafir_bank(P(xb), xb.shape[1], P(yb), yb.shape[1], ch, N, isz, nb - h, P(H), N, P(t), bpc)
    assert rel_rms(np.concatenate([ya, yb], 1), y) < 1e-6
    if N > isz:
        assert rel_rms(t[:, :N - isz], tail[:, :N - isz]) < 1e-6


def test_k9_golden_and_dropin_kernel(fft, oracle):
    """the golden bandpass stream of the compiled reference through the bank kernel, and apply_fir_fft_cc's one-block kernel"""
    T = oracle.firdes_filter_len(0.05); N = 256; isz = N - T + 1
    taps = Z(N, np.complex64); taps[:T] = oracle.firdes_bandpass_c(T, -0.1, 0.2)
    H = oracle.dft(taps)
    x = np.ascontiguousarray(GOLD["bp_in"]); nb = x.size // isz
    y = Z(nb * isz, np.complex64); tail = Z((1, N), np.complex64)
    assert fft.emul_launch_olafir_bank(P(x), x.size, P(y), y.size, 1, N, isz, nb, P(H), N, P(tail), 4) >= 0
    assert rel_rms(y, GOLD["bp_out"][:y.size]) < 5e-6                      # same bar as the GPU test
    rng = np.random.default_rng(3)
    blk = Z(N, np.complex64); blk[:isz] = _cplx(rng, isz); last = _cplx(rng, T - 1); out = Z(N, np.complex64)
    assert fft.emul_launch_apply_fir_fft(P(blk), P(H), P(last), T - 1, P(out), N) >= 0
    want = np.fft.ifft(np.fft.fft(blk.astype(np.complex128)) * H.astype(np.complex128)); want[:T - 1] += last
    assert rel_rms(out, want) < 2e-6


@pytest.mark.parametrize("nb,runs,shifts", [(3, 5, [0.123, -0.31, 0.02]), (100, 4, [0.123, -0.31, 0.02, 0.4, -0.05, 0.33])])
def test_k8_fastddc_inverse_plan_equals_the_stateless_bank(fft, oracle, nb, runs, shifts):
    """csdrb_fastddc_inv_plan_* (state inside, next run prepared ahead) against launch_fastddc_inv_bank run for run, bit for bit: a retune of channel 1
    after the second run and a set_state round trip; the never-retuned channels' last outputs also against the oracle.  The second case has 100 blocks per
    run (the state chain runs on its wrap tables, four channels per warp with a ragged last warp; the plan builds the tables once, the bank call every time)."""
    from oracle.pyoracle import _CF, _p, WINDOWS
    bw, dec = 0.05, 8
    chan_dt = np.dtype([("offsetbin", np.int32), ("sindelta", np.float32), ("cosdelta", np.float32), ("rate", np.float32)])

    def design(shift):
        g, _ = oracle.fastddc_init(bw, dec, shift)
        tf = np.empty(g.fft_size, np.complex64)
        oracle.L.oracle_fastddc_make_taps_fft(C.byref(g), shift, dec, WINDOWS["HAMMING"], _p(tf, _CF))
        row = np.zeros(1, chan_dt)
        row["offsetbin"] = g.offsetbin; row["sindelta"] = g.dsadata.sindelta; row["cosdelta"] = g.dsadata.cosdelta; row["rate"] = g.dsadata.rate
        return g, tf, row
    gs, tfs, rows = zip(*[design(s) for s in shifts])
    g = gs[0]
    nch = len(shifts)
    taps = Z((nch, g.fft_size), np.complex64); taps[:] = np.stack(tfs)
    chan = Z(nch, chan_dt); chan[:] = np.concatenate(rows)
    rng = np.random.default_rng(5)
    x = _cplx(rng, runs * nb * g.input_size, amp=0.5)
    spectra = np.stack(oracle.fastddc_fwd(x, g)).astype(np.complex64)
    width = nb * (g.post_input_size // g.post_decimation + 1) + 2
    plan = C.c_void_p()
    # a geometry the fold path does not cover is refused with a message (the stateless call handles it)
    assert fft.emul_fastddc_inv_plan_create(C.addressof(plan), P(chan), nch, nb, 256, 32, 8, 4, 28, 1) < 0 and b"not covered" in fft.emul_last_error() and not plan.value
    assert fft.emul_fastddc_inv_plan_create(C.addressof(plan), P(chan), nch, nb, g.fft_size, g.fft_inv_size, g.pre_decimation, g.scrap, g.post_input_size, g.post_decimation) == 0, fft.emul_last_error()
    remain = Z(nch, np.int32); phase = Z(nch, np.float32)
    sb = fft.emul_fastddc_inv_scratch_bytes(nch, nb); scratch = Z(sb + 16, np.uint8)
    try:
        for r in range(runs):
            sp = Z((nb, g.fft_size), np.complex64); sp[:] = spectra[r * nb:(r + 1) * nb]
            if r == 2:                                                                            # retune channel 1: both paths from this run on
                g1, tf1, row1 = design(0.27)
                taps[1] = tf1; chan[1] = row1[0]
                one = Z(1, chan_dt); one[:] = row1
                assert fft.emul_fastddc_inv_plan_set_channel(plan, 1, P(one)) == 0
            if r == runs - 2:                                                                     # state out and back in: drops the look-ahead, changes nothing
                hr = Z(nch, np.int32); hp = Z(nch, np.float32)
                assert fft.emul_fastddc_inv_plan_get_state(plan, P(hr), P(hp)) == 0
                assert np.array_equal(hr, remain) and np.array_equal(hp.view(np.uint32), phase.view(np.uint32))
                assert fft.emul_fastddc_inv_plan_set_state(plan, P(hr), P(hp)) == 0
            want = Z((nch, width), np.complex64); wt = Z(nch, np.int32)
            assert fft.emul_launch_fastddc_inv_bank(P(sp), nb, P(taps), P(chan), nch, g.fft_size, g.fft_inv_size, g.pre_decimation, g.scrap, g.post_input_size, g.post_decimation,
                                                    P(remain), P(phase), P(want), width, P(wt), P(scratch), sb) == 4, fft.emul_last_error()
            got = Z((nch, width), np.complex64); gt = Z(nch, np.int32)
            assert fft.emul_fastddc_inv_plan_run(plan, P(sp), P(taps), P(got), width, P(gt)) == nb, fft.emul_last_error()
            assert np.array_equal(gt, wt)
            for c in range(nch):
                assert np.array_equal(got[c, :gt[c]].view(np.uint32), want[c, :wt[c]].view(np.uint32)), (r, c)
        hr = Z(nch, np.int32); hp = Z(nch, np.float32)
        assert fft.emul_fastddc_inv_plan_get_state(plan, P(hr), P(hp)) == 0
        assert np.array_equal(hr, remain) and np.array_equal(hp.view(np.uint32), phase.view(np.uint32))
    finally:
        fft.emul_fastddc_inv_plan_destroy(plan)
    # the channels that were never retuned: their stream over all runs is the oracle's
    for c in [c for c in range(nch) if c != 1]:
        ref = oracle.fastddc_inv(list(spectra), bw, dec, shifts[c])
        assert rel_rms(got[c, :gt[c]], ref[-gt[c]:]) < 5e-6, c


@pytest.mark.parametrize("bw,dec,shift", [(0.05, 8, 0.123), (0.05, 3, -0.2), (0.01, 6, 0.25), (0.05, 4, 0.2), (0.02, 4, 0.05), (0.05, 16, -0.3), (0.05, 32, 0.4),
                                          (0.05, 64, -0.1)])
def test_k8_fastddc_forward_and_inverse(fft, oracle, bw, dec, shift):
    """a12/a13 against the oracle (and, for the first geometry, the golden spectra / channel output of the compiled reference);
    decimation 3 has pre_decimation 1 and takes the one-CTA-per-(block, channel) kernel, 6 has fft_inv_size 2048 and takes it too, decimation 64
    (fft_inv_size 32) the tiled one, the others the fold path."""
    from oracle.pyoracle import _CF, _p, WINDOWS
    g, _ = oracle.fastddc_init(bw, dec, shift)
    rng = np.random.default_rng(dec)
    if (bw, dec) == (0.05, 8):
        x = np.ascontiguousarray(GOLD["ddc_in"])
    else:
        n = 5 * g.input_size; t = np.arange(n)
        x = ((np.exp(2j * np.pi * (-shift + 0.002) * t) * 0.5).astype(np.complex64) + _cplx(rng, n, amp=0.05)).astype(np.complex64)
    nb = x.size // g.input_size
    sp = Z((nb, g.fft_size), np.complex64); carry = Z(max(g.overlap_length, 1), np.complex64)
    assert fft.emul_launch_fastddc_fwd(P(x), P(sp), P(carry), g.fft_size, g.input_size, nb) >= 0
    want_sp = np.stack(oracle.fastddc_fwd(x, g))
    assert rel_rms(sp, want_sp) < 1e-6
    assert np.array_equal(carry[:g.overlap_length], x[nb * g.input_size - g.overlap_length:nb * g.input_size])
    tf = np.empty(g.fft_size, np.complex64)
    oracle.L.oracle_fastddc_make_taps_fft(C.byref(g), shift, dec, WINDOWS["HAMMING"], _p(tf, _CF))
    chan = Z(1, np.dtype([("offsetbin", np.int32), ("sindelta", np.float32), ("cosdelta", np.float32), ("rate", np.float32)]))
    chan["offsetbin"] = g.offsetbin; chan["sindelta"] = g.dsadata.sindelta; chan["cosdelta"] = g.dsadata.cosdelta; chan["rate"] = g.dsadata.rate
    remain = Z(1, np.int32); phase = Z(1, np.float32); total = Z(1, np.int32)
    out = Z((1, nb * (g.post_input_size // g.post_decimation + 1) + 2), np.complex64)
    sb = fft.emul_fastddc_inv_scratch_bytes(1, nb); scratch = Z(sb + 16, np.uint8)
    rc = fft.emul_launch_fastddc_inv_bank(P(want_sp), nb, P(tf), P(chan), 1, g.fft_size, g.fft_inv_size, g.pre_decimation, g.scrap, g.post_input_size, g.post_decimation,
                                          P(remain), P(phase), P(out), out.shape[1], P(total), P(scratch), sb)
    assert rc >= 0, fft.emul_last_error()
    want = oracle.fastddc_inv(list(want_sp), bw, dec, shift)
    assert total[0] == want.size and rel_rms(out[0, :want.size], want) < 5e-6
    if (bw, dec) == (0.05, 8):
        assert rel_rms(sp, GOLD["ddc_fwd_out"]) < 1e-6 and rel_rms(out[0, :total[0]], GOLD["ddc_inv_out"]) < 5e-6


@pytest.mark.parametrize("N", [4, 8, 16, 32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384])
def test_k8_fastddc_forward_every_size(fft, N):
    """the forward step at every size (radix-8 passes below 32 points, radix-16 from 32 on): overlap-save blocks of the carried overlap followed by
    the stream, against float64, and the overlap carried out"""
    isz = N - max(1, N // 8)
    rng = np.random.default_rng(N)
    nb, ov = 5, N - isz
    x = _cplx(rng, nb * isz); sp = Z((nb, N), np.complex64); carry = _cplx(rng, ov)
    stream = np.concatenate([carry, x]).astype(np.complex128)
    assert fft.emul_launch_fastddc_fwd(P(x), P(sp), P(carry), N, isz, nb) >= 0, fft.emul_last_error()
    assert rel_rms(sp, np.stack([np.fft.fft(stream[b * isz:b * isz + N]) for b in range(nb)])) < 1e-6
    assert np.array_equal(carry, x[nb * isz - ov:])
