"""CPU tier for the four-step FFT above 16384 points (csdr_b200/csrc/fft_large.cuh) and every layer it lifts: csdrb_fft_c2c_large_batch, the
make_fft_c2c plans, csdrb_fastddc_fwd_cc, the apply_fir_fft_cc drop-in and the CLI commands on top.  The shipped kernels run thread by thread on
the emulated library (tests/host_shim); tests/test_gpu_fft_large.py runs the same bodies (the check_* functions) on the H100 at every size.

The per-output bound.  Every path from input n to output k goes through log2(N) radix-2-equivalent levels.  A radix-16 pass is four of them: four
rounded additions (u = 2^-24 each), one twiddle product (a table entry that is a product of up to four correctly rounded values, <= 8u, times a
product that rounds to 2u) and the constants of the 16-point butterfly (3u): 17u per four levels, under 5u per level.  The twiddle between the two
steps is one more product of two correctly rounded table values (<= 3u) and its application (2u), with the rounding of the store: 7u.  To first
order |X^_k - X_k| <= (5 log2 N + 7) u sum_n |x_n|, and sum_n |x_n| <= sqrt(N) ||x||_2.  On a sparse input the bound is a few 1e-6 of one sample,
so one wrong inter-step twiddle cannot hide the way it can in an RMS over N outputs."""
import ctypes as C
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "spectrum"))
import emul_build  # noqa: E402
import spectrum as S  # noqa: E402
from oracle.pyoracle import Oracle, rel_rms, _CF, _p, WINDOWS  # noqa: E402

U = 2.0 ** -24
CHUNK_BYTES = 16 << 20                                                  # the intermediate's bound: a batch above CHUNK_BYTES / (8 N) takes a second chunk


def setup(dev):
    import csdr_b200
    L = dev.L
    vp, lg, it, sz = C.c_void_p, C.c_long, C.c_int, C.c_size_t
    L.csdrb_fft_c2c_large_batch.argtypes = [vp, lg, vp, lg, it, it, it, vp]
    L.csdrb_fastddc_fwd_cc.argtypes = [vp, vp, vp, it, it, it, vp]
    L.csdrb_fastddc_inv_bank_scratch_bytes.argtypes = [it, it]; L.csdrb_fastddc_inv_bank_scratch_bytes.restype = sz
    L.csdrb_fastddc_inv_bank_cc.argtypes = [vp, it, vp, vp, it, C.POINTER(csdr_b200.FastDDC), vp, vp, vp, lg, vp, vp, sz, vp]
    L.fastddc_init.argtypes = [C.POINTER(csdr_b200.FastDDC), C.c_float, it, C.c_float]
    L.make_fft_c2c.argtypes = [it, vp, vp, it, it]; L.make_fft_c2c.restype = vp
    L.fft_execute.argtypes = [vp]; L.fft_destroy.argtypes = [vp]
    L.apply_fir_fft_cc.argtypes = [vp, vp, vp, vp, it]
    return dev


@pytest.fixture(scope="module")
def built(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    return emul_build.build_full_once(tmp_path_factory)


@pytest.fixture(scope="module")
def dev(built):
    return setup(S.EmulDev(C.CDLL(str(built[0]))))


@pytest.fixture(scope="module")
def cli(built):
    return str(built[1])


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


def noise(rng, *shape):
    return ((rng.standard_normal(shape) + 1j * rng.standard_normal(shape)) * 0.3).astype(np.complex64)


def fft_large(dev, x, inverse=False, in_pad=0, out_pad=0, expect=None):
    """csdrb_fft_c2c_large_batch on x [batch, N]: the whole padded output array [batch, N + out_pad], pre-filled with a marker"""
    batch, N = x.shape
    xs = np.zeros((batch, N + in_pad), np.complex64); xs[:, :N] = x
    d_x = dev.put(xs)
    d_y = dev.put(np.full((batch, N + out_pad), -7.25 + 3.5j, np.complex64))
    rc = dev.L.csdrb_fft_c2c_large_batch(dev.ptr(d_x), N + in_pad, dev.ptr(d_y), N + out_pad, N, batch, 1 if inverse else 0, dev.stream)
    assert rc == (0 if expect is None else expect), (rc, dev.L.csdrb_last_error())
    assert np.array_equal(dev.get(d_x, np.complex64).view(np.uint32), xs.reshape(-1).view(np.uint32))      # the input is not touched
    return dev.get(d_y, np.complex64).reshape(batch, N + out_pad)


# ---- the transform ---------------------------------------------------------------------------------------------------------------------------
def check_against_numpy(dev, lg, batch):
    N = 1 << lg
    rng = np.random.default_rng(lg * 100 + batch)
    x = noise(rng, batch, N)
    for inverse in (False, True):
        y = fft_large(dev, x, inverse)
        want = np.fft.ifft(x.astype(np.complex128), axis=1) * N if inverse else np.fft.fft(x.astype(np.complex128), axis=1)
        assert rel_rms(y, want) < 1e-6
        bound = (5 * lg + 7) * U * np.abs(x.astype(np.complex128)).sum(axis=1, keepdims=True)
        assert np.all(np.abs(y - want) <= bound), float((np.abs(y - want) / bound).max())


def check_sparse_input_bound(dev, lg):
    """a handful of samples at assorted positions: every output within (5 log2 N + 7) u of their summed magnitudes"""
    N = 1 << lg
    rng = np.random.default_rng(lg)
    x = np.zeros((1, N), np.complex64)
    pos = np.unique(np.concatenate([rng.integers(0, N, 6), [1, N - 1, 1023, 1025]]))
    x[0, pos] = noise(rng, pos.size) * 3
    for inverse in (False, True):
        y = fft_large(dev, x, inverse)[0]
        want = np.fft.ifft(x[0].astype(np.complex128)) * N if inverse else np.fft.fft(x[0].astype(np.complex128))
        bound = (5 * lg + 7) * U * np.abs(x[0].astype(np.complex128)).sum()
        assert np.abs(y - want).max() <= bound, (np.abs(y - want).max(), bound)


def check_impulses_and_tones(dev, lg, n1, n2):
    N = 1 << lg
    ps = sorted({0, 1, n2 - 1, n2, n2 + 1, n1 - 1, n1 + 1, 5 * n2 + 3, N // 2 + 1, N - n2 - 1, N - 1})
    x = np.zeros((len(ps), N), np.complex64)
    for r, p in enumerate(ps):
        x[r, p] = 1.0
    k = np.arange(N, dtype=np.float64)
    for inverse in (False, True):
        y = fft_large(dev, x, inverse).astype(np.complex128)
        for r, p in enumerate(ps):
            want = np.exp((2j if inverse else -2j) * np.pi * ((k * p) % N) / N)
            assert np.abs(np.abs(y[r]) - 1).max() < 1e-6 and np.abs(y[r] - want).max() < 1e-6, (p, inverse)
    # a tone on bin q lands in bin q (forward) and nowhere else
    qs = [1, n1, n1 + 1, N - 1]
    t = np.stack([np.exp(2j * np.pi * ((k * q) % N) / N) for q in qs]).astype(np.complex64)
    y = fft_large(dev, t)
    for r, q in enumerate(qs):
        assert abs(y[r, q] - N) < 1e-5 * N
        rest = np.delete(y[r], q)
        assert np.abs(rest).max() < 2e-5 * N                            # the float32 rounding of the tone's own samples, spread over the bins


def check_round_trip_batch_and_strides(dev, lg):
    N = 1 << lg
    rng = np.random.default_rng(lg + 50)
    x = noise(rng, 3, N)
    y = fft_large(dev, x, False, in_pad=6, out_pad=10)
    assert np.all(y[:, N:] == np.complex64(-7.25 + 3.5j))              # nothing written between the rows
    back = fft_large(dev, np.ascontiguousarray(y[:, :N]), True)[:, :N] / N
    assert np.abs(back - x).max() < 2e-6
    for b in range(3):                                                   # a row of a batched call is the single call, bit for bit
        one = fft_large(dev, x[b:b + 1])[0]
        assert np.array_equal(one.view(np.uint32), y[b, :N].view(np.uint32))
    for bad in (np.nan, np.inf):                                         # a poisoned row stays in its row
        z = x.copy(); z[1, N // 3] = bad
        d = fft_large(dev, z)
        assert np.array_equal(d[0].view(np.uint32), y[0, :N].view(np.uint32)) and np.array_equal(d[2].view(np.uint32), y[2, :N].view(np.uint32))
        assert not np.isfinite(d[1]).all()


def check_second_chunk(dev, lg):
    N = 1 << lg
    batch = CHUNK_BYTES // (8 * N) + 1
    rng = np.random.default_rng(lg + 7)
    x = noise(rng, batch, N)
    y = fft_large(dev, x)
    assert rel_rms(y, np.fft.fft(x.astype(np.complex128), axis=1)) < 1e-6
    last = fft_large(dev, x[-1:])[0]
    assert np.array_equal(last.view(np.uint32), y[-1].view(np.uint32))


def check_refusals(dev):
    L = dev.L
    buf = dev.alloc(8 * 64)
    before = L.csdrb_kernel_launches()
    for n in (0, 2, 1024, 1 << 14, (1 << 15) + 1, 3 << 15, 48000, 1 << 21, -(1 << 15)):
        assert L.csdrb_fft_c2c_large_batch(dev.ptr(buf), n, dev.ptr(buf), n, n, 1, 0, dev.stream) == -1, n
        assert b"32768..1048576" in L.csdrb_last_error(), L.csdrb_last_error()
    assert L.csdrb_fft_c2c_large_batch(None, 1 << 15, dev.ptr(buf), 1 << 15, 1 << 15, 1, 0, dev.stream) == -1
    assert L.csdrb_fft_c2c_large_batch(dev.ptr(buf), 1 << 15, dev.ptr(buf), 1 << 15, 1 << 15, 0, 0, dev.stream) == 0
    assert L.csdrb_kernel_launches() == before                          # nothing was launched
    assert L.csdrb_fft_c2c_batch(dev.ptr(buf), 1 << 15, dev.ptr(buf), 1 << 15, 1 << 15, 1, 0, dev.stream) == -1      # the small call keeps its range
    assert not L.make_fft_c2c(1 << 21, None, None, 1, 0) and not L.make_fft_c2c(3 << 14, None, None, 1, 0)


def check_plan(dev, lg):
    """make_fft_c2c / fft_execute on host buffers, both directions"""
    N = 1 << lg
    rng = np.random.default_rng(lg + 3)
    x = noise(rng, N); y = np.zeros(N, np.complex64)
    for forward in (1, 0):
        pl = dev.L.make_fft_c2c(N, x.ctypes.data, y.ctypes.data, forward, 0)
        assert pl
        dev.L.fft_execute(pl); dev.L.fft_destroy(pl)
        want = np.fft.fft(x.astype(np.complex128)) if forward else np.fft.ifft(x.astype(np.complex128)) * N
        assert rel_rms(y, want) < 1e-6


# ---- fastddc at a long filter ---------------------------------------------------------------------------------------------------------------
def check_fastddc(dev, oracle, bw, dec, nblocks, shifts=(0.1, -0.3137, 0.0021)):
    import csdr_b200
    L = dev.L
    g = csdr_b200.FastDDC()
    assert L.fastddc_init(C.byref(g), bw, dec, 0.0) == 0
    N, isz, ov = g.fft_size, g.input_size, g.overlap_length
    assert N > 16384 and 64 <= g.fft_inv_size <= 1024                     # a four-step forward transform in front of the fold path
    rng = np.random.default_rng(dec)
    x = noise(rng, nblocks * isz)

    def forward(cuts):
        d_ov = dev.put(np.zeros(ov, np.complex64)); parts = []
        for a, b in zip([0] + cuts, cuts + [nblocks]):
            d_x = dev.put(x[a * isz:b * isz]); d_sp = dev.alloc(8 * N * (b - a))
            assert L.csdrb_fastddc_fwd_cc(dev.ptr(d_x), dev.ptr(d_sp), dev.ptr(d_ov), N, isz, b - a, dev.stream) >= 0, L.csdrb_last_error()
            parts.append(dev.get(d_sp, np.complex64).reshape(b - a, N))
        return np.concatenate(parts), dev.get(d_ov, np.complex64)

    sp, carry = forward([])
    padded = np.concatenate([np.zeros(ov, np.complex64), x]).astype(np.complex128)
    want = np.stack([np.fft.fft(padded[b * isz:b * isz + N]) for b in range(nblocks)])
    assert rel_rms(sp, want) < 1e-6
    assert np.array_equal(carry, padded[-ov:].astype(np.complex64))
    sp2, carry2 = forward([1])                                           # the stream cut into two calls (the first shorter than the overlap)
    assert np.array_equal(sp2.view(np.uint32), sp.view(np.uint32)) and np.array_equal(carry2, carry)

    # forward + inverse bank against the oracle's restatement of fastddc_inv_cc on the float64 spectra
    chn = len(shifts)
    gs = []
    for s in shifts:
        gk = csdr_b200.FastDDC(); assert L.fastddc_init(C.byref(gk), bw, dec, s) == 0; gs.append(gk)
    tf = np.empty((chn, N), np.complex64)
    for k, s in enumerate(shifts):
        og, _ = oracle.fastddc_init(bw, dec, s)
        oracle.L.oracle_fastddc_make_taps_fft(C.byref(og), s, dec, WINDOWS["HAMMING"], _p(tf[k], _CF))
    chan = np.zeros(chn, np.dtype([("offsetbin", np.int32), ("sindelta", np.float32), ("cosdelta", np.float32), ("rate", np.float32)]))
    for k, gk in enumerate(gs):
        chan[k] = (gk.offsetbin, gk.dsadata.sindelta, gk.dsadata.cosdelta, gk.dsadata.rate)
    ostride = nblocks * (g.post_input_size // g.post_decimation + 1) + 2
    d_sp = dev.put(sp); d_tf = dev.put(tf); d_chan = dev.put(chan.view(np.uint8))
    d_rem = dev.put(np.zeros(chn, np.int32)); d_ph = dev.put(np.zeros(chn, np.float32)); d_tot = dev.put(np.zeros(chn, np.int32))
    d_out = dev.alloc(8 * chn * ostride)
    sb = L.csdrb_fastddc_inv_bank_scratch_bytes(chn, nblocks); d_scr = dev.alloc(sb + 16)
    rc = L.csdrb_fastddc_inv_bank_cc(dev.ptr(d_sp), nblocks, dev.ptr(d_tf), dev.ptr(d_chan), chn, C.byref(g), dev.ptr(d_rem), dev.ptr(d_ph), dev.ptr(d_out),
                                     ostride, dev.ptr(d_tot), dev.ptr(d_scr), sb, dev.stream)
    assert rc >= 0, L.csdrb_last_error()
    out = dev.get(d_out, np.complex64).reshape(chn, ostride); total = dev.get(d_tot, np.int32)
    for k, s in enumerate(shifts):
        w = oracle.fastddc_inv(list(want.astype(np.complex64)), bw, dec, s)
        assert total[k] == w.size and w.size > 0
        assert rel_rms(out[k, :w.size], w) < 5e-6, (s, rel_rms(out[k, :w.size], w))


def check_fastddc_fwd_short_calls(dev):
    """calls shorter than the overlap (the carried overlap shifts instead of being replaced) equal one call"""
    L, N, isz, nblocks = dev.L, 1 << 15, 1000, 3
    ov = N - isz
    rng = np.random.default_rng(21)
    x = noise(rng, nblocks * isz); first = noise(rng, ov)
    outs = []
    for cuts in ([], [1, 2]):
        d_ov = dev.put(first); parts = []
        for a, b in zip([0] + cuts, cuts + [nblocks]):
            d_x = dev.put(x[a * isz:b * isz]); d_sp = dev.alloc(8 * N * (b - a))
            assert L.csdrb_fastddc_fwd_cc(dev.ptr(d_x), dev.ptr(d_sp), dev.ptr(d_ov), N, isz, b - a, dev.stream) >= 0, L.csdrb_last_error()
            parts.append(dev.get(d_sp, np.complex64).reshape(b - a, N))
        outs.append((np.concatenate(parts), dev.get(d_ov, np.complex64)))
    stream = np.concatenate([first, x])
    assert np.array_equal(outs[0][1], stream[-ov:]) and np.array_equal(outs[1][1], stream[-ov:])
    assert np.array_equal(outs[0][0].view(np.uint32), outs[1][0].view(np.uint32))
    want = np.stack([np.fft.fft(stream[b * isz:b * isz + N].astype(np.complex128)) for b in range(nblocks)])
    assert rel_rms(outs[0][0], want) < 1e-6
    for bad in (1 << 21, 3 << 14):
        assert L.csdrb_fastddc_fwd_cc(dev.ptr(dev.alloc(64)), dev.ptr(dev.alloc(64)), dev.ptr(dev.alloc(64)), bad, 8, 1, dev.stream) == -1
        assert b"1048576" in L.csdrb_last_error()


# ---- apply_fir_fft_cc above 16384 points ----------------------------------------------------------------------------------------------------
def check_apply_fir_fft(dev, lg):
    N = 1 << lg
    L = dev.L
    rng = np.random.default_rng(lg + 11)
    T = N // 2 + 1; isz = N - T + 1; ov = T - 1
    taps = np.zeros(N, np.complex64); taps[:T] = noise(rng, T) / np.sqrt(T)
    H = np.fft.fft(taps.astype(np.complex128)).astype(np.complex64)
    x = noise(rng, 2 * isz)
    inb = np.zeros(N, np.complex64); spec = np.zeros(N, np.complex64); prod = np.zeros(N, np.complex64)
    res = [np.zeros(N, np.complex64), np.zeros(N, np.complex64)]
    fwd = L.make_fft_c2c(N, inb.ctypes.data, spec.ctypes.data, 1, 1)
    inv = [L.make_fft_c2c(N, prod.ctypes.data, res[k].ctypes.data, 0, 1) for k in range(2)]
    got = []
    for b in range(2):                                                   # the block loop of bandpass_fir_fft_cc: the second block adds the first one's tail
        inb[:isz] = x[b * isz:(b + 1) * isz]
        tail = np.ascontiguousarray(res[1 - b][isz:])
        L.apply_fir_fft_cc(fwd, inv[b], H.ctypes.data, tail.ctypes.data, ov)
        got.append(res[b][:isz].copy())
    for p in [fwd] + inv:
        L.fft_destroy(p)
    full = np.zeros(2 * isz + ov, np.complex128)
    for b in range(2):
        blk = np.zeros(N, np.complex128); blk[:isz] = x[b * isz:(b + 1) * isz]
        full[b * isz:b * isz + N] += np.fft.ifft(np.fft.fft(blk) * H.astype(np.complex128))
    assert rel_rms(np.concatenate(got), full[:2 * isz]) < 2e-6


# ---- the CLI -----------------------------------------------------------------------------------------------------------------------------------
def run_graph(cli, stages, data, timeout=900):
    cmd = " | ".join(f"{cli} {s}" for s in stages)
    r = subprocess.run(["bash", "-c", cmd], input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=timeout)
    assert r.returncode == 0, (cmd, r.stderr[-2000:])
    return r.stdout


WATERFALL = ["fft_cc 32768 32768 HAMMING", "logaveragepower_cf -70 32768 2", "fft_exchange_sides_ff 32768"]


def check_cli_waterfall(dev, cli, ref=None):
    """the 32768-bin waterfall pipe gives the bytes of the library composition (and, against the reference CLI, its values)"""
    N, A, lines = 32768, 2, 2
    L = dev.L
    rng = np.random.default_rng(5)
    x = noise(rng, lines * A * N)
    got = np.frombuffer(run_graph(cli, WATERFALL, x.tobytes()), np.float32)
    assert got.size >= lines * N
    w = S.window(L, N)
    d_fr = dev.put(x); d_w = dev.alloc(x.nbytes); d_s = dev.alloc(x.nbytes); d_win = dev.put(w)
    assert L.csdrb_apply_window_rows_c(dev.ptr(d_fr), dev.ptr(d_w), dev.ptr(d_win), N, lines * A, dev.stream) >= 0
    assert L.csdrb_fft_c2c_large_batch(dev.ptr(d_w), N, dev.ptr(d_s), N, N, lines * A, 0, dev.stream) >= 0
    add = np.float32(np.float64(np.float32(-70.0)) - 10.0 * np.log10(float(A)))
    db = dev.alloc(4 * N * lines)
    for j in range(lines):
        acc = dev.alloc(4 * N)
        for f in range(A):
            assert L.csdrb_accumulate_power_cf(dev.ptr(d_s) + 8 * N * (j * A + f), dev.ptr(acc), N, dev.stream) >= 0
        assert L.csdrb_log_ff(dev.ptr(acc), dev.ptr(db) + 4 * N * j, N, float(add), dev.stream) >= 0
    want = dev.get(db, np.float32).reshape(lines, N)
    want = np.concatenate([want[:, N // 2:], want[:, :N // 2]], axis=1).reshape(-1)
    assert np.array_equal(got[:lines * N].view(np.uint32), want.view(np.uint32))
    if ref:
        theirs = np.frombuffer(run_graph(ref, WATERFALL, x.tobytes()), np.float32)
        pa, pb = 10.0 ** (got[:lines * N].astype(np.float64) / 10), 10.0 ** (theirs[:lines * N].astype(np.float64) / 10)
        assert theirs.size == got.size and np.all(np.abs(pa - pb) <= 1e-5 * pb.mean() + 1e-4 * pb)         # as powers: a near-empty bin has no stable dB value


def check_cli_filters(cli, oracle, ref=None):
    rng = np.random.default_rng(9)
    # bandpass_fir_fft_cc with 20001 taps: 32768-point blocks
    T = oracle.firdes_filter_len(0.0002); N = 32768; isz = N - T + 1
    assert 16384 < T < N - 200
    x = noise(rng, 2 * isz)
    got = np.frombuffer(run_graph(cli, ["bandpass_fir_fft_cc -0.05 0.05 0.0002"], x.tobytes()), np.complex64)
    want = oracle.bandpass_fir_fft_cc(x, -0.05, 0.05, 0.0002)
    assert got.size >= want.size == 2 * isz and rel_rms(got[:want.size], want) < 2e-6
    if ref:
        theirs = np.frombuffer(run_graph(ref, ["bandpass_fir_fft_cc -0.05 0.05 0.0002"], x.tobytes()), np.complex64)
        assert theirs.size == got.size and rel_rms(got[:want.size], theirs[:want.size]) < 2e-6
    # fastddc with 8193 taps: 65536-point forward blocks
    g, _ = oracle.fastddc_init(0.0005, 256, 0.1)
    x = noise(rng, 3 * g.input_size)
    stages = ["fastddc_fwd_cc 256 0.0005", "fastddc_inv_cc 0.1 256 0.0005"]
    got = np.frombuffer(run_graph(cli, stages, x.tobytes()), np.complex64)
    want = oracle.fastddc_inv(oracle.fastddc_fwd(x, g), 0.0005, 256, 0.1)
    assert got.size >= want.size > 0 and rel_rms(got[:want.size], want) < 5e-6
    if ref:
        theirs = np.frombuffer(run_graph(ref, stages, x.tobytes()), np.complex64)
        assert theirs.size == got.size and rel_rms(got[:want.size], theirs[:want.size]) < 5e-6
    # a geometry beyond 2^20 points still fails, and says why
    r = subprocess.run(["bash", "-c", f"{cli} fastddc_fwd_cc 256 0.00001"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=120)
    assert r.returncode != 0 and b"1048576" in r.stderr


FACTORS = {15: (256, 128), 16: (256, 256), 17: (512, 256), 18: (512, 512), 19: (1024, 512), 20: (1024, 1024)}


@pytest.mark.parametrize("lg,batch", [(15, 1), (15, 3), (16, 2), (17, 1), (20, 1)])
def test_forward_and_inverse_against_numpy(dev, lg, batch):
    check_against_numpy(dev, lg, batch)


@pytest.mark.parametrize("lg", [15, 16, 17])
def test_sparse_input_within_the_per_output_bound(dev, lg):
    check_sparse_input_bound(dev, lg)


@pytest.mark.parametrize("lg", [15, 17])
def test_impulses_and_tones(dev, lg):
    check_impulses_and_tones(dev, lg, *FACTORS[lg])


@pytest.mark.parametrize("lg", [15, 16])
def test_round_trip_batch_rows_strides_and_nonfinite_rows(dev, lg):
    check_round_trip_batch_and_strides(dev, lg)


def test_a_batch_beyond_one_scratch_chunk(dev):
    check_second_chunk(dev, 15)


def test_refusals(dev):
    check_refusals(dev)


@pytest.mark.parametrize("lg", [15, 16])
def test_plans_above_16384(dev, lg):
    check_plan(dev, lg)


@pytest.mark.parametrize("bw,dec,nblocks", [(0.0005, 256, 3), (0.00025, 256, 2)])
def test_fastddc_with_a_long_filter(dev, oracle, bw, dec, nblocks):
    check_fastddc(dev, oracle, bw, dec, nblocks)


def test_fastddc_forward_calls_shorter_than_the_overlap(dev):
    check_fastddc_fwd_short_calls(dev)


@pytest.mark.parametrize("lg", [15, 16])
def test_apply_fir_fft_above_16384(dev, lg):
    check_apply_fir_fft(dev, lg)


def test_cli_waterfall_at_32768_bins(dev, cli):
    check_cli_waterfall(dev, cli)


def test_cli_long_filters(cli, oracle):
    check_cli_filters(cli, oracle)
