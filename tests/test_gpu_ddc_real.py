"""GPU tests (-m gpu) of the real-input banks: csdrb_shift_addition_bank_fc and the shift_addition_fc drop-in against the reference bit for bit, the
real-input fused DDC bank (csdrb_ddc_bank_f, csdrb_ddc_bank_process_f) against the complex bank fed the same samples as x + 0j, and the
`csdr shift_addition_fc` command.  The same bodies run in the CPU tier on the emulated library (tests/test_ddc_real_emulated.py).

The real bank computes sh = P x with one rounding per component where the complex bank computes fma(P, x.i, Q x.q); for x.q = 0 the two are the
same value up to the sign of a zero, so outputs are compared as float values (+0 == -0, NaN where NaN) and the carried phases bit for bit."""
import ctypes as C
import os
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tests" / "spectrum"))
sys.path.insert(0, str(ROOT / "tests" / "real"))
import real as R  # noqa: E402
import spectrum as S  # noqa: E402
from bitcmp import assert_bits_equal, bits  # noqa: E402
from ddc_generic_ref import BUCKETS, bucket_edges  # noqa: E402
from ddc_ref import n_out_of, rates_for  # noqa: E402

OURS_CLI = ROOT / "csdr_b200" / "csdr"
LIB = ROOT / "csdr_b200" / "libcsdr_b200.so"
REF_CLI = ROOT / "oracle" / "_ref" / "csdr_ref"


def setup(dev):
    L = dev.L
    vp, lg, it, sz = C.c_void_p, C.c_long, C.c_int, C.c_size_t
    L.csdrb_last_error.restype = C.c_char_p
    L.csdrb_kernel_launches.restype = C.c_long
    L.csdrb_shift_addition_bank_scratch_bytes.argtypes = [it, it, it]; L.csdrb_shift_addition_bank_scratch_bytes.restype = sz
    L.csdrb_shift_addition_bank_fc.argtypes = [vp, lg, vp, lg, it, it, vp, vp, it, vp, sz, vp]
    L.csdrb_ddc_bank_scratch_bytes.argtypes = [it, it, it, it]; L.csdrb_ddc_bank_scratch_bytes.restype = sz
    for f in (L.csdrb_ddc_bank, L.csdrb_ddc_bank_f):
        f.argtypes = [vp, it, it, vp, vp, it, it, it, vp, it, it, vp, lg, vp, vp, vp, sz, vp]
    L.csdrb_ddc_bank_create.argtypes = [it, vp, it, vp, it, it, it]; L.csdrb_ddc_bank_create.restype = vp
    L.csdrb_ddc_bank_destroy.argtypes = [vp]
    L.csdrb_ddc_bank_set_rate.argtypes = [vp, it, C.c_float]
    L.csdrb_ddc_bank_process.argtypes = [vp, vp, it, vp, lg, vp]
    L.csdrb_ddc_bank_process_f.argtypes = [vp, vp, it, vp, lg, vp]
    L.csdrb_stream_synchronize.argtypes = [vp]
    L.shift_addition_fc.argtypes = [vp, vp, it, R._Shift, C.c_float]; L.shift_addition_fc.restype = C.c_float
    return dev


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from csdr_b200.build import build
    build()
    return setup(S.CudaDev())


def params_of(rates):
    """shift_addition_data_t per channel, [C, 3] float32"""
    return np.array([[d.sindelta, d.cosdelta, d.rate] for d in (R.shift_init(float(r)) for r in rates)], np.float32)


def assert_values_equal(a, b, what):
    """equal as float values: +0 and -0 alike, NaN at the same places"""
    a = np.ascontiguousarray(a).view(np.float32); b = np.ascontiguousarray(b).view(np.float32)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    if not same.all():
        k = int(np.flatnonzero(~same.reshape(-1))[0])
        raise AssertionError(f"{what}: first difference at flat index {k}: {a.reshape(-1)[k]!r} vs {b.reshape(-1)[k]!r} ({int((~same).sum())} values)")


# ---- shift_addition_fc ------------------------------------------------------------------------------------------------------------------------
def shift_bank_fc(dev, x_rows, rates, phases, chunk, shared):
    """csdrb_shift_addition_bank_fc on x_rows ([N] shared or [C, N]): (y [C, N] complex64, phases [C] float32)"""
    ch = rates.size
    n = x_rows.shape[-1]
    d_x = dev.put(np.ascontiguousarray(x_rows, np.float32))
    d_y = dev.alloc(8 * ch * n)
    d_p = dev.put(params_of(rates)); d_ph = dev.put(np.asarray(phases, np.float32))
    sb = dev.L.csdrb_shift_addition_bank_scratch_bytes(ch, n, chunk); d_s = dev.alloc(sb + 16)
    rc = dev.L.csdrb_shift_addition_bank_fc(dev.ptr(d_x), 0 if shared else n, dev.ptr(d_y), n, ch, n, dev.ptr(d_p), dev.ptr(d_ph), chunk,
                                            dev.ptr(d_s), sb, dev.stream)
    assert rc >= 0, dev.L.csdrb_last_error()
    dev.sync()
    return dev.get(d_y, np.complex64).reshape(ch, n), dev.get(d_ph, np.float32)


SHIFT_CASES = [(1024, True, 5000), (1024, False, 3 * 1024), (77, True, 2000), (1, False, 300), (1000, False, 4097), (4099, True, 9000), (0, True, 777)]


@pytest.mark.parametrize("chunk,shared,n", SHIFT_CASES)
def test_shift_bank_fc_is_the_reference_bit_for_bit(dev, chunk, shared, n):
    """rates 0, +-0.5 and random, chunks of 1024 and odd sizes, one shared row and one row per channel.  The bank gives the C restatement of the
    source bit for bit (each call seeded with cos/sin in double, like the shift_addition_cc bank and the fused banks), the drop-in gives the
    restatement of the reference BUILD (seeded with sincosf) bit for bit, and both match the compiled reference, where it is built: the drop-in
    bit for bit, the bank in every returned phase and within a few ulp per sample (a seed that sincosf rounds the other way)"""
    rng = np.random.default_rng(chunk * 7 + n)
    rates = np.concatenate([np.array([0.0, 0.5, -0.5, 0.25, -0.4999], np.float32), rng.uniform(-0.5, 0.5, 4).astype(np.float32)])
    ch = rates.size
    phases = rng.uniform(-3.1, 3.1, ch).astype(np.float32)
    x = rng.uniform(-1, 1, n if shared else (ch, n)).astype(np.float32)
    y, ph = shift_bank_fc(dev, x, rates, phases, chunk, shared)
    call = chunk if chunk > 0 else None
    for c in range(ch):
        row = x if shared else x[c]
        want, wph = R.shift_addition_fc(row, rates[c], phases[c], call)
        assert_bits_equal(y[c], want, f"channel {c} rate {rates[c]}")
        assert bits(ph[c]) == bits(wph), (c, float(ph[c]), float(wph))
        if R.have_ref():
            rwant, rph = R.shift_addition_fc(row, rates[c], phases[c], call, ref=True)
            assert_bits_equal(R.shift_addition_fc(row, rates[c], phases[c], call, build_seed=True)[0], rwant, f"build restatement, channel {c}")
            assert bits(rph) == bits(wph)
            err = np.abs(y[c] - rwant).max()
            assert err <= 1e-6 * max(1.0, float(np.abs(row).max())), (c, float(err))
    # the drop-in, one call per chunk on host buffers
    for c in (0, 2, ch - 1):
        row = np.ascontiguousarray(x if shared else x[c])
        out = np.empty(n, np.complex64)
        d = R.shift_init(rates[c]); p = float(phases[c]); step = call or n
        for s in range(0, n, step):
            m = min(step, n - s)
            p = dev.L.shift_addition_fc(row[s:].ctypes.data, out[s:].ctypes.data, m, d, p)
        want, wph = R.shift_addition_fc(row, rates[c], phases[c], call, build_seed=True)
        assert_bits_equal(out, want, f"drop-in, channel {c}")
        assert bits(np.float32(p)) == bits(wph) == bits(ph[c])
        if R.have_ref():
            assert_bits_equal(out, R.shift_addition_fc(row, rates[c], phases[c], call, ref=True)[0], f"drop-in against the reference, channel {c}")


# ---- the real-input fused bank --------------------------------------------------------------------------------------------------------------
def ddc_call(dev, real, x, rates, ph0, chunk, offset, D, taps, demod, last=None, misalign=0):
    """one csdrb_ddc_bank(_f) call -> (rc, out [C, n_out] or None, phases, last_out).  Real x sits 8 bytes past a 16-byte boundary (an even sample
    offset, what csdr-bankd hands the bank) unless misalign says otherwise: `misalign` floats further."""
    ch, n, T = rates.size, x.size, taps.size
    if real:
        lead = 2 + misalign
        buf = np.zeros(lead + n + 4, np.float32); buf[lead:lead + n] = x
        d_x = dev.put(buf); xp = dev.ptr(d_x) + 4 * lead
    else:
        d_x = dev.put(np.ascontiguousarray(x, np.complex64)); xp = dev.ptr(d_x)
    n_out = n_out_of(n, D, T)
    stride = n_out + 3
    d_out = dev.alloc(8 * ch * stride + 16)
    d_p = dev.put(params_of(rates)); d_ph = dev.put(np.asarray(ph0, np.float32))
    d_li = dev.put(np.asarray(last, np.complex64)) if last is not None else None
    d_lo = dev.alloc(8 * ch) if demod else None
    sb = dev.L.csdrb_ddc_bank_scratch_bytes(ch, n, chunk, offset); d_s = dev.alloc(sb + 64)
    fn = dev.L.csdrb_ddc_bank_f if real else dev.L.csdrb_ddc_bank
    rc = fn(xp, n, ch, dev.ptr(d_p), dev.ptr(d_ph), chunk, offset, D, taps.ctypes.data, T, demod, dev.ptr(d_out), stride,
            dev.ptr(d_li) if d_li is not None else None, dev.ptr(d_lo) if d_lo is not None else None, dev.ptr(d_s), sb, dev.stream)
    dev.sync()
    if rc < 0:
        return rc, None, dev.get(d_ph, np.float32), None
    dt = np.float32 if demod else np.complex64
    out = dev.get(d_out, dt)[:ch * stride].reshape(ch, stride)[:, :n_out]
    return rc, out, dev.get(d_ph, np.float32), (dev.get(d_lo, np.complex64) if demod else None)


def geometry_cases(emulated):
    """bucket edges of the generic kernel at the decimations of tests/test_ddc_generic_emulated.py, and the D = 50 / 10 geometries the complex bank
    runs on its own kernels (the real bank runs the generic one there)"""
    ds = [2, 6, 12, 40, 126] if emulated else [2, 4, 6, 12, 40, 48, 52, 126, 200, 400]
    out = [(D, T) for D in ds for T in bucket_edges(D)]
    out += [(50, 49), (50, 50), (50, 801), (50, 850), (10, 79), (10, 81), (10, 200)]
    return out


CHUNKS = [(1024, 0), (1024, 1023), (13, 12), (97, 5), (0, 0)]


def check_real_equals_complex(dev, D, T, i, outputs):
    rng = np.random.default_rng(1000 * D + T)
    ch = [1, 33, 65, 31, 64][i % 5]
    chunk, offset = CHUNKS[i % len(CHUNKS)]
    n = T + (outputs - 1) * D + (i % D)
    x = rng.uniform(-1, 1, n).astype(np.float32)
    rates = rates_for(ch, rng)
    ph0 = rng.uniform(-3.1, 3.1, ch).astype(np.float32)
    last = (rng.uniform(-1, 1, ch) + 1j * rng.uniform(-1, 1, ch)).astype(np.complex64)
    taps = rng.uniform(-1, 1, T).astype(np.float32)
    xc = x.astype(np.complex64)
    for demod in (0, 1):
        li = last if demod else None
        rc_r, o_r, p_r, l_r = ddc_call(dev, True, x, rates, ph0, chunk, offset, D, taps, demod, li)
        rc_c, o_c, p_c, l_c = ddc_call(dev, False, xc, rates, ph0, chunk, offset, D, taps, demod, li)
        assert rc_r == rc_c == n_out_of(n, D, T), (rc_r, rc_c, dev.L.csdrb_last_error())
        what = f"D={D} T={T} ch={ch} chunk {chunk}+{offset} demod={demod}"
        assert_values_equal(o_r, o_c, what)
        assert_bits_equal(p_r, p_c, what + ": carried phase")
        if demod:
            assert_values_equal(l_r, l_c, what + ": last_out")


@pytest.mark.parametrize("i,D,T", [(i, D, T) for i, (D, T) in enumerate(geometry_cases(False))])
def test_real_bank_equals_complex_bank_on_x_plus_0j(dev, i, D, T):
    check_real_equals_complex(dev, D, T, i, outputs=300)


def check_nonfinite(dev, D, T):
    """NaN and +-Inf real samples: with demod off exactly the outputs whose window [oD, oD + T) holds one are non-finite, every other output equals the
    clean run; the complex bank on x + 0j agrees value for value, demod included"""
    rng = np.random.default_rng(D + T)
    ch, chunk, offset = 33, 97, 12
    n = T + 60 * D + 7
    x = rng.uniform(-1, 1, n).astype(np.float32)
    rates = rates_for(ch, rng); ph0 = rng.uniform(-3, 3, ch).astype(np.float32)
    taps = rng.uniform(-1, 1, T).astype(np.float32)
    M = -(-T // D)
    M = next(b for b in BUCKETS if M <= b)
    pos = sorted({p for p in (5 * D + T, 5 * D + D * M - 1, 40 * D + T // 2 + 1, 0, n - 1) if 0 <= p < n})
    xp = x.copy()
    for k, p in enumerate(pos):
        xp[p] = [np.nan, np.inf, -np.inf][k % 3]
    n_out = n_out_of(n, D, T)
    o = np.arange(n_out)
    hit = np.zeros(n_out, bool)
    for p in pos:
        hit |= (o * D <= p) & (p < o * D + T)
    _, clean, _, _ = ddc_call(dev, True, x, rates, ph0, chunk, offset, D, taps, 0)
    _, dirty, _, _ = ddc_call(dev, True, xp, rates, ph0, chunk, offset, D, taps, 0)
    fin = np.isfinite(dirty.real) & np.isfinite(dirty.imag)
    for c in range(ch):
        assert np.array_equal(~fin[c], hit), (c, np.flatnonzero(~fin[c])[:10], np.flatnonzero(hit)[:10])
    assert_values_equal(dirty[:, ~hit], clean[:, ~hit], "away from the poisoned samples")
    for demod in (0, 1):
        _, a, pa, la = ddc_call(dev, True, xp, rates, ph0, chunk, offset, D, taps, demod)
        _, b, pb, lb = ddc_call(dev, False, xp.astype(np.complex64), rates, ph0, chunk, offset, D, taps, demod)
        assert_values_equal(a, b, f"demod={demod}: real against complex on x + 0j")
        assert_bits_equal(pa, pb, "carried phase")


NONFINITE = [(2, 7), (12, 97), (50, 801), (10, 79), (126, 2395), (400, 8000)]


@pytest.mark.parametrize("D,T", NONFINITE)
def test_real_bank_nonfinite_stays_in_its_windows(dev, D, T):
    check_nonfinite(dev, D, T)


REFUSED = [(7, 79), (40, 961), (446, 16 * 446 + 1), (1002, 1002 * 7 + 1)]


def check_refusals(dev):
    """odd D and geometries beyond the limits: -2, no launch, the phase untouched; an odd-sample (4-byte) offset: -1 and a message"""
    for D, T in REFUSED:
        n = T + 8 * D
        x = np.ones(n, np.float32)
        before = dev.L.csdrb_kernel_launches()
        rc, _, ph, _ = ddc_call(dev, True, x, np.array([0.1], np.float32), np.array([0.625], np.float32), 1024, 0, D, np.ones(T, np.float32), 0)
        msg = dev.L.csdrb_last_error()
        assert rc == -2 and b"no fused kernel" in msg, (D, T, rc, msg)
        assert dev.L.csdrb_kernel_launches() == before and ph[0] == np.float32(0.625)
    D, T = 50, 801
    x = np.ones(T + 20 * D, np.float32)
    for mis in (1, 3):
        before = dev.L.csdrb_kernel_launches()
        rc, _, ph, _ = ddc_call(dev, True, x, np.array([0.1], np.float32), np.array([0.625], np.float32), 1024, 0, D, np.ones(T, np.float32), 1,
                                misalign=mis)
        msg = dev.L.csdrb_last_error()
        assert rc == -1 and b"8-byte aligned" in msg, (rc, msg)
        assert dev.L.csdrb_kernel_launches() == before and ph[0] == np.float32(0.625)
    # the even offsets are served: 8 bytes past a 16-byte boundary (the default of ddc_call) and on it
    for mis in (0, 2):
        rc, _, _, _ = ddc_call(dev, True, x, np.array([0.1], np.float32), np.array([0.0], np.float32), 1024, 0, D, np.ones(T, np.float32), 1,
                               misalign=mis)
        assert rc == n_out_of(x.size, D, T), dev.L.csdrb_last_error()


def test_real_bank_refusals(dev):
    check_refusals(dev)


# ---- the streaming object on real blocks --------------------------------------------------------------------------------------------------
def stream_run(dev, real, x, rates, D, taps, demod, consumed_per_block, retune):
    """csdrb_ddc_bank_create + process(_f) over x in blocks that each consume `consumed_per_block` samples (the tail re-presented);
    retune = (sample, channel, rate): set_rate before the block that starts at that sample.  Returns the concatenated outputs [C, total]."""
    L = dev.L
    ch, T = rates.size, taps.size
    bank = L.csdrb_ddc_bank_create(ch, rates.ctypes.data, D, taps.ctypes.data, T, demod, 1024)
    assert bank, L.csdrb_last_error()
    n_out = consumed_per_block // D
    N = T + (n_out - 1) * D
    outs = []
    start = 0
    try:
        while start + N <= x.size:
            if retune is not None and start == retune[0]:
                assert L.csdrb_ddc_bank_set_rate(bank, retune[1], retune[2]) == 0
            blk = x[start:start + N]
            if real:
                buf = np.zeros(N + 6, np.float32); buf[2:2 + N] = blk
                d_x = dev.put(buf); xp = dev.ptr(d_x) + 8
            else:
                d_x = dev.put(blk.astype(np.complex64)); xp = dev.ptr(d_x)
            d_o = dev.alloc(8 * ch * n_out + 16)
            fn = L.csdrb_ddc_bank_process_f if real else L.csdrb_ddc_bank_process
            rc = fn(bank, xp, N, dev.ptr(d_o), n_out, dev.stream)
            assert rc == n_out, (rc, L.csdrb_last_error())
            dev.sync()
            outs.append(dev.get(d_o, np.float32 if demod else np.complex64)[:ch * n_out].reshape(ch, n_out))
            start += rc * D
    finally:
        L.csdrb_ddc_bank_destroy(bank)
    return np.concatenate(outs, axis=1)


def check_stream(dev, D, T, blocks_a, blocks_b):
    """real blocks with a set_rate mid-stream: the same outputs whether the stream is cut into blocks of blocks_a or blocks_b outputs (the retune
    falls on a block start of both), the complex object's on x + 0j value for value, and before the retune the one-shot csdrb_ddc_bank_f's"""
    rng = np.random.default_rng(D * 31 + T)
    ch = 37
    rates = rates_for(ch, rng)
    taps = rng.uniform(-1, 1, T).astype(np.float32)
    lcm = blocks_a * blocks_b // np.gcd(blocks_a, blocks_b)
    total_out = 3 * lcm
    x = rng.uniform(-1, 1, T + total_out * D + D).astype(np.float32)
    retune = (lcm * D, 5, -0.123)
    for demod in (1, 0):
        a = stream_run(dev, True, x, rates, D, taps, demod, blocks_a * D, retune)
        b = stream_run(dev, True, x, rates, D, taps, demod, blocks_b * D, retune)
        c = stream_run(dev, False, x, rates, D, taps, demod, blocks_a * D, retune)
        m = min(a.shape[1], b.shape[1])
        assert m >= 2 * lcm
        assert_bits_equal(a[:, :m], b[:, :m], f"demod={demod}: block split")
        assert_values_equal(a, c, f"demod={demod}: real object against the complex object on x + 0j")
        n1 = T + (lcm - 1) * D
        rc, one, _, _ = ddc_call(dev, True, x[:n1], rates, np.zeros(ch, np.float32), 1024, 0, D, taps, demod)
        assert rc == lcm
        assert_bits_equal(a[:, :lcm], one, "before the retune: the one-shot call")
        plain = stream_run(dev, True, x, rates, D, taps, demod, blocks_a * D, None)
        assert_bits_equal(a[:, :lcm], plain[:, :lcm], "before the retune: the stream without it")
        assert not np.array_equal(a[5, lcm:], plain[5, lcm:]), "the retune took effect"


@pytest.mark.parametrize("D,T,ba,bb", [(50, 801, 40, 60), (10, 199, 45, 30), (12, 97, 20, 50)])
def test_bank_object_on_real_blocks(dev, D, T, ba, bb):
    check_stream(dev, D, T, ba, bb)


# ---- the CLI ----------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def cli():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from csdr_b200.build import build
    build()
    return str(OURS_CLI)


def _run(cmd, data, env=None, pass_fds=()):
    e = dict(os.environ); e.update(env or {})
    r = subprocess.run(cmd, input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=e, timeout=300, pass_fds=pass_fds)
    assert r.returncode == 0, r.stderr[-1000:]
    return r


def test_cli_shift_addition_fc(cli):
    """`csdr shift_addition_fc R` on a stream that is not a whole number of its 16384-sample buffers: the model of the reference CLI (1024-sample
    calls, the stale tail of a short last buffer) bit for bit, its `reinitialized to` line, and the reference CLI's bytes where it is built"""
    rng = np.random.default_rng(5)
    x = rng.uniform(-1, 1, 3 * 16384 + 5000).astype(np.float32)
    for rate in (0.0, -0.5, 0.1234):
        r = _run([cli, "shift_addition_fc", str(rate)], x.tobytes())
        got = np.frombuffer(r.stdout, np.complex64)
        assert_bits_equal(got, R.cli_stream(x, rate), f"rate {rate}")
        assert f"reinitialized to {rate:g}".encode() in r.stderr
        if REF_CLI.exists():
            assert r.stdout == _run([str(REF_CLI), "shift_addition_fc", str(rate)], x.tobytes()).stdout


def test_cli_shift_addition_fc_fd_tuning(cli):
    """--fd: the rate waiting on the descriptor at start-up is the rate, as on the command line (the reference CLI's bytes too, where built)"""
    rng = np.random.default_rng(6)
    x = rng.uniform(-1, 1, 40_000).astype(np.float32).tobytes()
    plain = _run([cli, "shift_addition_fc", "-0.085"], x).stdout
    clis = [cli] + ([str(REF_CLI)] if REF_CLI.exists() else [])
    for c in clis:
        r, w = os.pipe()
        os.write(w, b"-0.085\n")
        try:
            got = _run([c, "shift_addition_fc", "--fd", str(r)], x, pass_fds=(r,)).stdout
        finally:
            os.close(r); os.close(w)
        assert got == plain, c


def test_reference_binary_runs_shift_addition_fc_on_our_library(cli):
    """LD_PRELOAD: the reference's csdr computes shift_addition_fc with our library (it reports kernel launches) and writes the same bytes"""
    if not REF_CLI.exists():
        pytest.skip("oracle/_ref/csdr_ref not built")
    lib = os.environ.get("CSDRB_TEST_PRELOAD_LIB", str(LIB))
    x = np.random.default_rng(7).uniform(-1, 1, 2 * 16384 + 333).astype(np.float32).tobytes()
    plain = _run([str(REF_CLI), "shift_addition_fc", "0.21"], x).stdout
    r = _run([str(REF_CLI), "shift_addition_fc", "0.21"], x, env={"LD_PRELOAD": lib, "CSDRB_TRACE": "1"})
    assert r.stdout == plain
    assert b"libcsdr_b200: " in r.stderr and b"kernel launches" in r.stderr, r.stderr[-500:]


# ---- the Python API (GPU only) ---------------------------------------------------------------------------------------------------------------
def test_python_api_on_real_tensors(dev):
    import csdr_b200
    from oracle.pyoracle import Oracle
    ora = Oracle()
    rng = np.random.default_rng(8)
    D, bw = 50, 0.005
    T = ora.firdes_filter_len(bw); taps = csdr_b200.firdes_lowpass_f(T, 0.5 / D)
    rates = np.array([-0.41, 0.03, 0.27], np.float32)
    x = rng.uniform(-1, 1, T + 400 * D).astype(np.float32)
    xt = torch.from_numpy(x).cuda()
    y, ph = csdr_b200.shift_addition_bank_fc(xt, rates, chunk=1024)
    for c, r in enumerate(rates):
        want, wph = R.shift_addition_fc(x, r, 0.0, 1024)
        assert_bits_equal(y[c].cpu().numpy(), want, f"shift_addition_bank_fc channel {c}")
    a, pa, la = csdr_b200.ddc_bank(xt, rates, D, taps, demod=True)
    b, pb, lb = csdr_b200.ddc_bank(xt.to(torch.complex64), rates, D, taps, demod=True)
    assert_values_equal(a.cpu().numpy(), b.cpu().numpy(), "ddc_bank on float32 against complex64")
    bank = csdr_b200.DdcBank(rates, D, taps, demod=True)
    got = bank.process(xt).cpu().numpy(); bank.close()
    assert_bits_equal(got, a.cpu().numpy(), "DdcBank.process on float32 against ddc_bank")
