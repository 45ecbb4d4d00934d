"""CPU tier: the fused DDC bank at every served decimation (csrc/ddc_bank.cu, ddc_bank_generic_kernel) executed on the host under tests/host_shim.

Every geometry of tests/ddc_generic_ref.py runs through the same contract as the D = 50 / 10 kernels (tests/ddc_ref.py): every output within the
error bound of the float64 reference, the carried phases, the discriminator and last_out bit for bit, one channel per lane = two, a channel subset
and a two-block split = the full call, and NaN / +-Inf only in the outputs whose window holds them.  Each case runs under one of the three fiber
orders in turn, so the matrix covers all three at the cost of one.  CSDRB_DDC_CPL is read once per launcher instantiation, so one channel per lane
needs its own loaded copy of the library (as in tests/test_ddc_bank_emulated.py); the emulator's barrier count (one per CTA) shows the grid.
Refusals (odd D, M above the top bucket, D * MP above the tap capacity) are checked on the whole emulated library's C ABI.
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
sys.path.insert(0, str(ROOT / "tests"))
import ddc_ref  # noqa: E402
import emul_build  # noqa: E402
from ddc_generic_ref import BUCKETS, NONFINITE, case_id, cases, expected_ctas, kernel_for, nonfinite_positions  # noqa: E402
from ddc_ref import assert_bits_equal, check_against_reference, check_nonfinite, make_inputs, n_out_of, nco  # noqa: E402

ORDERS = ["alternate", "reverse", "random"]
SENTINEL = np.uint32(0x7FC0DEAD)                                     # a NaN the kernel never produces: padding must keep it
_built = {}
_libs = {}

# small blocks: the emulator walks every wideband sample of every lane; long filters get fewer outputs
CASES = cases(outputs=40, max_wide=16_000, chain_budget=4000,
              extra=[dict(D=40, T=641, channels=65, chunk=1024, offset=0, n=641 + 60 * 40, seed=7, firdes=True),
                     dict(D=1000, T=7001, channels=33, chunk=1024, offset=512, n=7001 + 4 * 1000 + 5, seed=8, firdes=True)])   # D * MP = 8000


@pytest.fixture(scope="module")
def emul(tmp_path_factory, oracle):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, names = emul_build.build_file(tmp_path_factory.mktemp("emul_ddc_generic"), "ddc_bank.cu")
    _built.update(so=Path(lib._name), names=names, proto=lib, oracle=oracle)
    return _built


def _load(order, cpl):
    """a private copy of the emulated library with its fiber order and its channels per lane fixed: each generic launcher reads CSDRB_DDC_CPL at
    its first call, so every bucket is called once while the variable is set"""
    if (order, cpl) in _libs:
        return _libs[(order, cpl)]
    so = _built["so"]
    copy = so.with_name(f"{so.stem}_gen_{order}_cpl{cpl}.so")
    shutil.copy(so, copy)
    saved = {k: os.environ.get(k) for k in ("CUDA_EMUL_ORDER", "CSDRB_DDC_CPL")}
    os.environ["CUDA_EMUL_ORDER"] = order
    if cpl == 1:
        os.environ["CSDRB_DDC_CPL"] = "1"
    else:
        os.environ.pop("CSDRB_DDC_CPL", None)
    try:
        lib = C.CDLL(str(copy))
        for n in _built["names"]:
            f = getattr(lib, "emul_" + n); g = getattr(_built["proto"], "emul_" + n)
            f.argtypes, f.restype = g.argtypes, g.restype
        lib.emul_last_error.restype = C.c_char_p; lib.emul_barriers.restype = C.c_long
        lib.cpl = cpl
        for b in BUCKETS:
            T = (b - 1) * 4 + 1
            _run(lib, np.ones(T, np.complex64), np.zeros(1, np.float32), np.zeros(1, np.float32), 1024, 0, 4, np.ones(T, np.float32), 0, None)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    _libs[(order, cpl)] = lib
    return lib


# ---- write guards: an out-of-bounds write of a kernel trips the canaries -------------------------------------------------------------------
_GUARD = 512
_guarded = []


def Z(shape, dtype):
    n = int(np.prod(shape)) * np.dtype(dtype).itemsize
    raw = np.full(n + 2 * _GUARD + 32, 0xA5, np.uint8)
    off = _GUARD + ((-(raw.ctypes.data + _GUARD)) % 16)
    raw[off:off + n] = 0
    _guarded.append((raw, off, n))
    return raw[off:off + n].view(dtype).reshape(shape)


@pytest.fixture(autouse=True)
def _check_guards():
    _guarded.clear()
    yield
    for raw, off, n in _guarded:
        assert np.all(raw[:off] == 0xA5) and np.all(raw[off + n:] == 0xA5), "a kernel wrote outside one of its buffers"
    _guarded.clear()


def P(a):
    return a.ctypes.data


def _prepass(lib, x, rates, ph0, chunk, offset, D, T):
    ch, n = rates.size, x.size
    xa = Z(n, np.complex64); xa[:] = x
    params = Z((ch, 3), np.float32); params[:] = [_built["oracle"].shift_addition_init(float(r)) for r in rates]
    ph = Z(ch, np.float32); ph[:] = ph0
    sb = lib.emul_ddc_bank_scratch_bytes(ch, n, chunk, offset); scratch = Z(sb + 64, np.uint8)
    assert lib.emul_launch_ddc_prepass(n, ch, P(params), P(ph), chunk, offset, D, T, P(scratch), sb, None) > 0, lib.emul_last_error()
    return xa, params, scratch, ph.copy()


def _main(lib, pre, chunk, offset, D, taps, demod, last_in):
    """the main kernel on a pre-pass -> (out [C, n_out], last_out or None); spare row, columns and last_out entry hold SENTINEL and must come back
    untouched, and the emulator's barrier count must be the grid launch_ddc_main computes for this copy's channels per lane"""
    xa, params, scratch, _ = pre
    ch, n, T = params.shape[0], xa.size, taps.size
    n_out = n_out_of(n, D, T)
    stride = n_out + 3
    out = Z((ch + 1, stride), np.float32 if demod else np.complex64); out.view(np.uint32)[:] = SENTINEL
    last_out = Z(ch + 1, np.complex64); last_out.view(np.uint32)[:] = SENTINEL
    li = None
    if last_in is not None:
        li = Z(ch, np.complex64); li[:] = last_in
    b0 = lib.emul_barriers()
    rc = lib.emul_launch_ddc_main(P(xa), n, ch, P(params), chunk, offset, D, taps.ctypes.data_as(C.c_void_p), T, demod, P(out), stride,
                                  P(li) if li is not None else None, P(last_out) if demod else None, P(scratch))
    assert rc == n_out, lib.emul_last_error()
    assert lib.emul_barriers() - b0 == expected_ctas(ch, n_out, D, T, lib.cpl), "not the grid of the expected kernel and channels per lane"
    words = out.view(np.uint32)
    assert np.all(words[:, n_out if demod else 2 * n_out:] == SENTINEL) and np.all(words[ch] == SENTINEL), "a store beyond n_out or channels"
    assert np.all(last_out.view(np.uint32)[2 * ch if demod else 0:] == SENTINEL), "a last_out store beyond channels, or without demod"
    return out[:ch, :n_out].copy(), (last_out[:ch].copy() if demod else None)


def _run(lib, x, rates, ph0, chunk, offset, D, taps, demod, last_in):
    pre = _prepass(lib, x, rates, ph0, chunk, offset, D, taps.size)
    out, lo = _main(lib, pre, chunk, offset, D, taps, demod, last_in)
    return out, pre[3], lo


def test_geometry_matrix_reaches_every_bucket():
    """the matrix runs every bucket of the generic kernel, its smallest and largest T, and nothing that the D = 50 / 10 kernels serve"""
    kinds = {kernel_for(c["D"], c["T"]) for c in CASES}
    assert kinds == {("generic", b) for b in BUCKETS}
    for b in BUCKETS:
        ds = [c["D"] for c in CASES if kernel_for(c["D"], c["T"]) == ("generic", b)]
        assert len(set(ds)) >= 3, (b, ds)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_generic_ddc_bank_contract(emul, oracle, case):
    """one geometry, both DEMOD kernels and both channels-per-lane copies: reference bound and bit-exact invariants (tests/ddc_ref.py),
    CPL=1 == CPL=2, a channel subset == the full bank, two blocks == one"""
    order = ORDERS[CASES.index(case) % len(ORDERS)]
    cpl2, cpl1 = _load(order, 2), _load(order, 1)
    D, T, chunk, offset = case["D"], case["T"], case["chunk"], case["offset"]
    firdes = oracle.firdes_lowpass_f(T, 0.5 / D) if case.get("firdes") else None
    x, rates, ph0, last, taps = make_inputs(case, firdes)
    ch = rates.size
    pre = _prepass(cpl2, x, rates, ph0, chunk, offset, D, T)
    ph_b = pre[3]
    base, _ = _main(cpl2, pre, chunk, offset, D, taps, 0, None)
    dem, lo = _main(cpl2, pre, chunk, offset, D, taps, 1, last)
    check_against_reference(oracle, case, x, rates, ph0, last, taps, base, ph_b, dem, ph_b, lo)

    for demod, want in ((0, (base, None)), (1, (dem, lo))):
        got = _main(cpl1, pre, chunk, offset, D, taps, demod, last if demod else None)
        for g, w, what in zip(got, want, ("output", "last_out")):
            if w is not None:
                assert_bits_equal(g, w, f"CPL=1 against CPL=2, demod={demod}: {what}")

    sub = np.unique([0, ch // 2, ch - 1])
    got, ph_s, _ = _run(cpl2, x, rates[sub], ph0[sub], chunk, offset, D, taps, 0, None)
    assert_bits_equal(got, base[sub], "channel subset against the full bank")
    assert_bits_equal(ph_s, ph_b[sub], "channel subset: carried phase")

    n_out = base.shape[1]
    if chunk > 0 and n_out >= 2:                                     # chunk = 0 means "one chunk per call": a split changes the NCO by definition
        n1 = T + (n_out // 2) * D - 1
        o1, p1, l1 = _run(cpl1, x[:n1], rates, ph0, chunk, offset, D, taps, 1, last)
        consumed = o1.shape[1] * D
        o2, p2, l2 = _run(cpl2, x[consumed:], rates, p1, chunk, (offset + consumed) % chunk, D, taps, 1, l1)
        assert_bits_equal(np.concatenate([o1, o2], 1), dem, "two blocks with the tail re-presented against one")
        assert_bits_equal(p2, ph_b, "two blocks: carried phase")
        assert_bits_equal(l2, lo, "two blocks: last_out")


@pytest.mark.parametrize("D,T", [(2, 48), (12, 97), (126, 2395)])
def test_generic_unit_tap_is_the_reference_nco(emul, oracle, D, T):
    """x = 1 and a single unit tap at k: output o is the reference phasor at sample oD + k, bit for bit, in both copies"""
    chunk, offset = 13, 12
    rng = np.random.default_rng(D)
    ch = 33
    rates = np.linspace(-0.4999, 0.4999, ch).astype(np.float32)
    ph0 = rng.uniform(-3, 3, ch).astype(np.float32)
    n = T + 30 * D + 3
    x = np.ones(n, np.complex64)
    refs = [nco(oracle, r, ph0[c], chunk, offset, n) for c, r in enumerate(rates)]
    libs = (_load("alternate", 2), _load("alternate", 1))
    pre = _prepass(libs[0], x, rates, ph0, chunk, offset, D, T)
    for k in sorted({0, 1, D - 1, T // 2, T - 1}):
        taps = np.zeros(T, np.float32); taps[k] = 1.0
        for lib in libs:
            out, _ = _main(lib, pre, chunk, offset, D, taps, 0, None)
            for c in range(ch):
                assert_bits_equal(out[c], refs[c][k::D][:out.shape[1]], f"D={D} T={T} k={k} CPL={lib.cpl} channel {c}")


@pytest.mark.parametrize("D,T", NONFINITE)
def test_generic_nonfinite_stays_in_its_windows(emul, monkeypatch, D, T):
    """NaN / +-Inf wideband samples, one at the last zero-padded tap of the bucket's M, reach exactly the outputs whose window holds them
    (ddc_ref.check_nonfinite with this bucket's positions), both DEMOD kernels and both channels-per-lane copies, which give the same bits"""
    monkeypatch.setattr(ddc_ref, "nonfinite_positions", nonfinite_positions)
    chunk, offset = [(1024, 0), (97, 12)][NONFINITE.index((D, T)) % 2]
    case = dict(D=D, T=T, channels=33, chunk=chunk, offset=offset, n=T + 60 * D + 7, seed=D + T + chunk)
    outs = []
    for lib in (_load("reverse", 2), _load("reverse", 1)):
        got = {}

        def run(x, rates, ph0, last, taps, demod):
            out, _, lo = _run(lib, x, rates, ph0, chunk, offset, D, taps, demod, last if demod else None)
            got[(x.tobytes(), demod)] = (out, lo)
            return out, lo
        check_nonfinite(run, case)
        outs.append(got)
    for k in outs[0]:
        for a, b in zip(outs[0][k], outs[1][k]):
            if a is not None:
                assert_bits_equal(b, a, "CPL=1 against CPL=2")


# ---- refusals, on the whole emulated library's C ABI ------------------------------------------------------------------------------------
REFUSED = [(7, 79), (40, 961), (10, 241), (2, 49), (446, 16 * 446 + 1), (402, 8000), (1002, 1002 * 7 + 1)]   # odd D, M > 24, D * MP > 8000
SERVED = [(2, 48), (40, 641), (444, 16 * 444 + 1), (400, 8000), (1000, 7001), (2000, 8000), (10, 240)]


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    L = C.CDLL(str(lib))
    L.csdrb_last_error.restype = C.c_char_p
    vp = C.c_void_p
    L.csdrb_ddc_bank_scratch_bytes.restype = C.c_size_t; L.csdrb_ddc_bank_scratch_bytes.argtypes = [C.c_int] * 4
    L.csdrb_ddc_bank.argtypes = [vp, C.c_int, C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, vp, C.c_int, C.c_int, vp, C.c_long, vp, vp, vp, C.c_size_t, vp]
    L.csdrb_ddc_bank_create.restype = vp
    L.csdrb_ddc_bank_create.argtypes = [C.c_int, vp, C.c_int, vp, C.c_int, C.c_int, C.c_int]
    L.csdrb_ddc_bank_destroy.argtypes = [vp]
    return L


def test_served_set_is_the_geometry_rule():
    """the rule the tests assume: even D, M <= 24, D * MP <= 8000; the two lists below sit on both sides of each limit"""
    assert all(kernel_for(D, T) for D, T in SERVED) and not any(kernel_for(D, T) for D, T in REFUSED)


@pytest.mark.parametrize("D,T", REFUSED)
def test_unserved_geometry_is_refused_and_launches_nothing(L, D, T):
    """csdrb_ddc_bank answers -2 with a message naming the served set, launches no kernel and leaves the carried phase alone;
    csdrb_ddc_bank_create refuses the same geometry"""
    n = T + 8 * D
    raw = np.zeros(2 * n + 8, np.float32); off = (-raw.ctypes.data // 4) % 4
    x = raw[off:off + 2 * n]
    params = np.zeros(3, np.float32); phase = np.array([0.625], np.float32)
    taps = np.ones(T, np.float32)
    out = np.zeros(64, np.complex64)
    sb = L.csdrb_ddc_bank_scratch_bytes(1, n, 1024, 0); scratch = np.zeros(sb + 64, np.uint8)
    before = L.csdrb_kernel_launches()
    rc = L.csdrb_ddc_bank(x.ctypes.data, n, 1, params.ctypes.data, phase.ctypes.data, 1024, 0, D, taps.ctypes.data, T, 0, out.ctypes.data, 32,
                          None, None, scratch.ctypes.data, sb, None)
    msg = L.csdrb_last_error()
    assert rc == -2 and b"no fused kernel" in msg and b"even decimation" in msg and b"8000" in msg, (rc, msg)
    assert L.csdrb_kernel_launches() == before and phase[0] == np.float32(0.625)
    rates = np.array([0.1], np.float32)
    assert not L.csdrb_ddc_bank_create(1, rates.ctypes.data, D, taps.ctypes.data, T, 1, 1024)


@pytest.mark.parametrize("D,T", SERVED)
def test_served_geometry_creates_a_bank(L, D, T):
    rates = np.array([0.1, -0.2], np.float32); taps = np.ones(T, np.float32) / T
    bank = L.csdrb_ddc_bank_create(2, rates.ctypes.data, D, taps.ctypes.data, T, 1, 1024)
    assert bank, L.csdrb_last_error()
    L.csdrb_ddc_bank_destroy(bank)
