"""CPU tier for the BPSK31 kernels (csdr_b200/csrc/psk31.cu): the shipped kernels and launchers run thread by thread under
tests/host_shim/cuda_emul.h and must equal the checker tests/psk31/psk31_oracle.c bit for bit -- outputs, per-channel counts and carried
state -- for channel counts that are not multiples of 32, row strides, any subset of channels, and streams cut into calls of random sizes,
which must equal one long call.  Every test runs under two fiber scheduling orders."""
import ctypes as C
import os
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "psk31"))
import emul_build  # noqa: E402
import psk31  # noqa: E402

_built = {}


@pytest.fixture(scope="module", params=["alternate", "random"])
def K(request, tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    if "psk31" not in _built:
        lib, names = emul_build.build_file(tmp_path_factory.mktemp("emul_psk31"), "psk31.cu")
        _built["psk31"] = (Path(lib._name), names, lib)
    so, names, proto = _built["psk31"]
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
    return a.ctypes.data if a is not None else None


def bits_of(a):
    return np.ascontiguousarray(a).view(np.uint8)


def signal(rng, n, specials=True):
    x = (0.3 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))).astype(np.complex64)
    if specials and n > 40:
        f = x.view(np.float32)
        for v in (0.0, np.nan, np.inf, -np.inf):
            f[rng.integers(0, f.size, 3)] = v
        x[rng.integers(0, n, 3)] = 0
    return x


class TrParams(C.Structure):
    _fields_ = [("algorithm", C.c_int), ("decimation", C.c_int), ("use_q", C.c_int), ("loop_gain", C.c_float), ("max_error", C.c_float)]


# ---- simple_agc_cc ------------------------------------------------------------------------------------------------------------------
def run_agc(K, X, gains, rate=0.001, reference=0.5, max_gain=65535.0, stride=None):
    ch, n = X.shape
    stride = stride or n
    xin = np.zeros((ch, stride), np.complex64); xin[:, :n] = X
    out = np.zeros((ch, stride), np.complex64)
    g = np.array(gains, np.float32)
    assert K.emul_launch_simple_agc_bank(P(xin), stride, P(out), stride, ch, n, rate, reference, max_gain, P(g)) >= 0, K.emul_last_error()
    return out[:, :n], g


@pytest.mark.parametrize("ch,n", [(1, 1), (3, 31), (33, 100), (40, 257)])
def test_simple_agc_bank_equals_checker(K, ch, n):
    rng = np.random.default_rng(ch * 1000 + n)
    X = np.stack([signal(rng, n) for _ in range(ch)])
    g0 = rng.uniform(0.5, 3.0, ch).astype(np.float32)
    y, g = run_agc(K, X, g0, stride=n + 3)
    for c in range(ch):
        yc, gc = psk31.simple_agc_cc(X[c], 0.001, 0.5, 65535.0, float(g0[c]))
        assert np.array_equal(bits_of(y[c]), bits_of(yc)), c
        assert np.float32(gc).tobytes() == g[c].tobytes()


def test_simple_agc_bank_splits_and_subsets(K):
    rng = np.random.default_rng(5)
    ch, n = 35, 300
    X = np.stack([signal(rng, n) for _ in range(ch)])
    whole, gw = run_agc(K, X, np.ones(ch), rate=0.01)
    g = np.ones(ch, np.float32); parts = []; pos = 0
    for size in (1, 40, 17, 200, 42):
        y, g = run_agc(K, X[:, pos:pos + size], g, rate=0.01); parts.append(y); pos += size
    assert np.array_equal(bits_of(np.concatenate(parts, 1)), bits_of(whole)) and np.array_equal(g, gw)
    sub = [34, 3, 17]
    ys, gs = run_agc(K, X[sub], np.ones(len(sub)), rate=0.01)
    assert np.array_equal(bits_of(ys), bits_of(whole[sub])) and np.array_equal(gs, gw[sub])


# ---- timing_recovery_cc -------------------------------------------------------------------------------------------------------------
def run_tr(K, rows, starts, sizes, alg, dec, use_q, loop_gain=0.5, max_error=2.0, co=None):
    ch = len(sizes)
    stride = max(r.size for r in rows) + 5
    xin = np.zeros((ch, stride), np.complex64)
    for c, r in enumerate(rows):
        xin[c, :r.size] = r
    max_size = max(sizes)
    cap = int(K.emul_timing_recovery_max_outputs(dec, max_size, loop_gain, max_error))
    out = np.zeros((ch, cap), np.complex64); err = np.zeros((ch, cap), np.float32); idx = np.zeros((ch, cap), np.int32)
    st = np.zeros((ch, 3), np.int32)
    if co is not None:
        st[:, 0] = co
    p = TrParams(alg, dec, int(use_q), loop_gain, max_error)
    s0 = np.array(starts, np.int32); sz = np.array(sizes, np.int32)
    rc = K.emul_launch_timing_recovery_bank(P(xin), stride, P(s0), P(sz), P(out), cap, P(err), P(idx), ch, C.addressof(p), P(st), max_size)
    assert rc >= 0, K.emul_last_error()
    return out, err, idx, st


@pytest.mark.parametrize("alg", [psk31.GARDNER, psk31.EARLYLATE])
@pytest.mark.parametrize("use_q", [0, 1])
@pytest.mark.parametrize("dec", [8, 12, 256])
@pytest.mark.parametrize("gain,max_error", [(0.5, 2.0), (1.0, 2.0)])
def test_timing_recovery_bank_equals_checker(K, alg, use_q, dec, gain, max_error):
    rng = np.random.default_rng(dec * 10 + alg * 2 + use_q)
    ch = 5
    rows = [signal(rng, int(rng.integers(3 * dec, 40 * dec))) for _ in range(ch)]
    starts = [int(rng.integers(0, 3)) for _ in range(ch)]
    sizes = [r.size - s for r, s in zip(rows, starts)]
    co0 = rng.integers(-dec // 4, dec // 4, ch).astype(np.int32)
    out, err, idx, st = run_tr(K, rows, starts, sizes, alg, dec, use_q, gain, max_error, co=co0)
    for c in range(ch):
        y, e, ix, s = psk31.timing_recovery_cc(rows[c][starts[c]:], alg, dec, use_q, gain, max_error, int(co0[c]))
        m = s[2]
        assert tuple(st[c]) == s
        assert np.array_equal(bits_of(out[c, :m]), bits_of(y)) and np.array_equal(bits_of(err[c, :m]), bits_of(e)) and np.array_equal(idx[c, :m], ix)


def test_timing_recovery_bank_splits(K):
    """a stream cut into calls that re-present the unconsumed input gives the symbols of one call over the whole stream"""
    rng = np.random.default_rng(11)
    dec = 16
    x = psk31.modulate(psk31.ref_varicode_encode(b"split") if psk31.have_ref() else rng.integers(0, 2, 60), dec, rng, freq=0.002)
    y1, e1, i1, s1 = psk31.timing_recovery_cc(x, psk31.GARDNER, dec)
    pos, co, ys, ixs = 0, 0, [], []
    while x.size - pos > 3 * dec // 2:
        size = min(int(rng.integers(2 * dec, 9 * dec)), x.size - pos)
        out, err, idx, st = run_tr(K, [x[pos:pos + size]], [0], [size], psk31.GARDNER, dec, 1, co=co)
        m = st[0, 2]
        ys.append(out[0, :m]); ixs.append(idx[0, :m] + pos)
        co = int(st[0, 0]); pos += int(st[0, 1])
    assert np.array_equal(bits_of(np.concatenate(ys)), bits_of(y1)) and np.array_equal(np.concatenate(ixs), i1)


def test_timing_recovery_refusals(K):
    x = np.zeros(100, np.complex64)
    for alg, dec, gain, err, want in [(2, 8, 0.5, 2.0, -1), (0, 6, 0.5, 2.0, -1), (0, 4, 0.5, 2.0, -1), (0, 8, 1.5, 2.0, -2), (0, 8, -2.0, 1.5, -2), (0, 8, float("nan"), 1.0, -2)]:
        p = TrParams(alg, dec, 1, gain, err)
        st = np.zeros(3, np.int32); z = np.zeros(1, np.int32); n = np.array([100], np.int32); out = np.zeros(100, np.complex64)
        assert K.emul_launch_timing_recovery_bank(P(x), 100, P(z), P(n), P(out), 100, None, None, 1, C.addressof(p), P(st), 100) == want


# ---- dbpsk_decoder_c_u8 -------------------------------------------------------------------------------------------------------------
def test_dbpsk_bank_equals_checker(K):
    rng = np.random.default_rng(3)
    ch, n = 6, 700
    X = np.stack([signal(rng, n) for _ in range(ch)])
    lengths = np.array([n, 0, 1, 513, 699, 2], np.int32)
    last = (rng.standard_normal(ch) + 1j * rng.standard_normal(ch)).astype(np.complex64)
    out = np.zeros((ch, n), np.uint8); last_out = np.zeros(ch, np.complex64)
    assert K.emul_launch_dbpsk_bank(P(X), n, P(out), n, ch, n, P(lengths), P(last), P(last_out)) >= 0
    for c in range(ch):
        b, l = psk31.dbpsk_decoder_c_u8(X[c, :lengths[c]], complex(last[c]))
        assert np.array_equal(out[c, :lengths[c]], b) and np.complex64(l).tobytes() == last_out[c].tobytes()


# ---- varicode -----------------------------------------------------------------------------------------------------------------------
def run_vc(K, rows, hist):
    ch = len(rows); n = max(max(r.size for r in rows), 1)
    xin = np.zeros((ch, n), np.uint8)
    for c, r in enumerate(rows):
        xin[c, :r.size] = r
    lengths = np.array([r.size for r in rows], np.int32)
    out = np.zeros((ch, n), np.uint8); cnt = np.zeros(ch, np.int32); h = np.array(hist, np.uint64)
    assert K.emul_launch_varicode_bank(P(xin), n, P(out), n, ch, n, P(lengths), P(h), P(cnt)) >= 0
    return [out[c, :cnt[c]].tobytes() for c in range(ch)], h


def test_varicode_bank_equals_checker_and_splits(K):
    rng = np.random.default_rng(9)
    text = bytes(range(128)) + b"Hello PSK31 world"
    if psk31.have_ref():
        enc = psk31.ref_varicode_encode(text)
    else:
        enc = np.concatenate([np.r_[[(c >> (b - 1 - k)) & 1 for k in range(b)], [0, 0]] for c, b in (psk31.varicode_table()[t] for t in text)]).astype(np.uint8)
    rows = [enc, rng.integers(0, 2, 900).astype(np.uint8), (rng.integers(0, 2, 300) * rng.integers(1, 256, 300)).astype(np.uint8), np.zeros(0, np.uint8)]
    hist = [0, int(rng.integers(0, 2 ** 63)), 5, 7]
    got, h = run_vc(K, rows, hist)
    for c in range(len(rows)):
        want, wh = psk31.varicode_decode(rows[c], hist[c])
        assert got[c] == want and int(h[c]) == wh
    assert got[0] == text[1:]                                           # NUL decodes to nothing
    # random splits of row 1 and a channel subset
    pos, hh, acc = 0, np.uint64(hist[1]), b""
    while pos < rows[1].size:
        k = int(rng.integers(1, 90))
        g, hv = run_vc(K, [rows[1][pos:pos + k]], [int(hh)]); acc += g[0]; hh = hv[0]; pos += k
    assert acc == got[1] and int(hh) == int(h[1])
