"""CPU tier for the demodulator banks (csdr_b200/csrc/demod.cu, the dcblock recursion of audio.cu, K4's novect form) through the C ABI of the whole
emulated library: every bank bit for bit against the restatements of tests/demod/demod.py and the compiled reference (the emulated atan bank calls
the host's atan2, the reference's libm, so it is exact here) -- lengths 1..9 and a long row, odd strides, several calls equal to one long call,
+-0 in I and Q, subnormals, +-Inf, NaN in I, Q and both, den = 0 for novect, alpha = 0 / a = 0 and explicit values, dcblock in place; the refusals;
the libcsdr drop-ins with their by-value struct returns."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "demod"))
import emul_build  # noqa: E402
import demod as M  # noqa: E402

needs_ref = pytest.mark.skipif(not M.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built")
LENGTHS = list(range(1, 10)) + [31, 1000, 4099]
F = np.float32


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    return M.bind(C.CDLL(str(lib)))


def P(a):
    return a.ctypes.data if a is not None else None


def rows_in(x, stride, dtype):
    """x [C, n] into rows of `stride` elements whose unused tail holds a sentinel"""
    buf = np.full((x.shape[0], stride), 7, dtype)
    buf[:, :x.shape[1]] = x
    return buf


def bank(L, name, x, stride_in, stride_out, carry=None, arg=(0.0, 0.0)):
    """one bank call on host rows; returns (outputs [C, n], carry out)"""
    ch, n = x.shape
    if name == "novect":
        stride_out += stride_out & 1                                   # K4 writes pairs: an even output stride
    out = np.full((ch, stride_out), 7, F)
    if name == "dcblock":
        xin = rows_in(x, stride_in, F)
        st = np.zeros((ch, 2), F) if carry is None else carry.copy()
        assert L.csdrb_dcblock_bank_ff(P(xin), stride_in, P(out), stride_out, ch, n, arg[0], P(st), None) == 0, L.csdrb_last_error()
        carry_out = st
    else:
        xin = rows_in(x, stride_in, np.complex64)
        if name == "atan":
            lo = np.full(ch, 9, F)
            assert L.csdrb_fmdemod_atan_bank_cf(P(xin), stride_in, P(out), stride_out, ch, n, P(carry), P(lo), None) == 0, L.csdrb_last_error()
            carry_out = lo
        elif name == "novect":
            lo = np.zeros(ch, np.complex64)
            assert L.csdrb_fmdemod_quadri_novect_bank_cf(P(xin), stride_in, P(out), stride_out, ch, n, P(carry), P(lo), None) == 0, L.csdrb_last_error()
            carry_out = lo
        else:
            assert L.csdrb_amdemod_estimator_bank_cf(P(xin), stride_in, P(out), stride_out, ch, n, arg[0], arg[1], None) == 0, L.csdrb_last_error()
            carry_out = None
    assert np.all(out[:, n:] == 7), name
    return out[:, :n].copy(), carry_out


def restate(name, row, carry=None, arg=(0.0, 0.0)):
    if name == "atan":
        return M.fmdemod_atan_cf(row, 0.0 if carry is None else carry)
    if name == "novect":
        return M.fmdemod_quadri_novect_cf(row, 0j if carry is None else carry)
    if name == "estimator":
        return M.amdemod_estimator_cf(row, *arg), None
    y, st = M.dcblock_rows(row[None], arg[0], None if carry is None else carry[None])
    return y[0], st[0]


def reference(name, row, carry=None, arg=(0.0, 0.0)):
    if name == "atan":
        return M.ref_atan(row, 0.0 if carry is None else carry)
    if name == "novect":
        return M.ref_novect(row, 0j if carry is None else carry)
    if name == "estimator":
        return M.ref_estimator(row, *arg), None
    y, st = M.ref_dcblock(row, arg[0], (0.0, 0.0) if carry is None else tuple(carry))
    return y, np.array(st, F)


ARGS = {"atan": [(0.0, 0.0)], "novect": [(0.0, 0.0)], "estimator": [(0.0, 0.0), (0.0, 5.0), (1.0, 0.5), (-0.3, 2.0)],
        "dcblock": [(0.0, 0.0), (0.9, 0.0), (1.0, 0.0), (-0.5, 0.0)]}
NAMES = list(ARGS)


def inputs(name, rng, ch, n):
    """random rows with the special values, the edge row in row 0 and an 8-bit receiver's repeating samples in the last row"""
    if name == "dcblock":
        return M.real_rows(rng, ch, n)
    x = M.complex_rows(rng, ch, n)
    x[0, :min(n, M.edge_row().size)] = M.edge_row()[:n]
    x[-1] = M.quantised_rows(rng, 1, n)[0]
    return x


@pytest.mark.parametrize("name", NAMES)
def test_bank_equals_restatement_and_reference(L, name):
    rng = np.random.default_rng(len(name))
    for arg in ARGS[name]:
        for n in LENGTHS:
            x = inputs(name, rng, 3, n)
            for si, so in ((n, n), (n + 1, n + 3), (n + 5 | 1, n + 2)):
                got, carry = bank(L, name, x, si, so, arg=arg)
                for c in range(3):
                    want, wcarry = restate(name, x[c], arg=arg)
                    assert M.same_bits(got[c], want), (name, arg, n, si, c, np.flatnonzero(got[c] != want)[:5])
                    if M.have_ref():
                        rwant, rcarry = reference(name, x[c], arg=arg)
                        assert M.same_bits(got[c], rwant), (name, arg, n, si, c, np.flatnonzero(got[c] != rwant)[:5])
                    if name in ("atan", "dcblock"):
                        assert M.same_bits(carry[c], wcarry), (name, n, c)
                    elif name == "novect":
                        assert carry[c] == np.complex64(x[c, -1]) or np.isnan(x[c, -1]), (n, c)


@pytest.mark.parametrize("name", ["atan", "novect", "dcblock"])
def test_calls_in_pieces_equal_one_call(L, name):
    """the carried state makes any cut of the stream give the bits of one long call"""
    rng = np.random.default_rng(11)
    x = inputs(name, rng, 4, 3000)
    whole, _ = bank(L, name, x, 3001, 3000)
    pieces, carry, at = [], None, 0
    for cut in (1, 2, 7, 100, 1024, 1866):
        got, carry = bank(L, name, x[:, at:at + cut], cut | 1, cut, carry=carry)
        pieces.append(got)
        at += cut
    assert at == 3000
    assert M.same_bits(np.concatenate(pieces, axis=1), whole), name


def test_carried_phase_starts_the_row(L):
    """atan's last_phase_in: a row's first output is taken against it, NULL is 0"""
    x = np.exp(1j * np.array([[0.5, 1.0, -2.0], [3.0, -3.0, 0.1]])).astype(np.complex64)
    last = np.array([0.25, -3.1], F)
    got, carry = bank(L, "atan", x, 3, 3, carry=last)
    for c in range(2):
        want, wc = M.fmdemod_atan_cf(x[c], last[c])
        assert M.same_bits(got[c], want) and M.same_bits(carry[c], wc)
        if M.have_ref():
            assert M.same_bits(got[c], M.ref_atan(x[c], last[c])[0])


def test_novect_divides_where_quadri_gives_zero(L):
    """den = I*I + Q*Q rounding to 0 (zeros and tiny samples): novect's NaN / +-Inf, quadri's 0; equal bits everywhere else"""
    x = np.array([[0, 1e-23 + 1e-23j, -2e-23 + 1e-30j, 1 + 1j, 0, 0.5 - 0.5j, 1e-30j, 3e-39, 0.25j, 0]], np.complex64)
    nov, _ = bank(L, "novect", x, 10, 10)
    quad = np.full((1, 10), 7, F)
    assert L.csdrb_fmdemod_quadri_bank_cf(P(x), 10, P(quad), 10, 1, 10, None, None, None) == 0
    i, q = x.real.astype(F), x.imag.astype(F)
    den0 = ((i * i).astype(F) + (q * q).astype(F)).astype(F) == 0
    assert den0.sum() >= 5
    assert np.all(~np.isfinite(nov[den0])) and np.all(quad[den0] == 0)
    assert M.same_bits(nov[~den0], quad[0, :][~den0[0]])
    assert M.same_bits(nov[0], M.fmdemod_quadri_novect_cf(x[0])[0])
    if M.have_ref():
        assert M.same_bits(nov[0], M.ref_novect(x[0])[0])


def test_novect_on_repeated_samples_in_every_quadrant(L):
    """equal consecutive samples make the numerator a zero; its sign is the build's (I*(Q-Qp) + Q*(Ip-I)), which K4's form does not give
    where I < 0"""
    rng = np.random.default_rng(8)
    x = M.quantised_rows(rng, 4, 20001)
    i = x.real
    rep = np.zeros(x.shape, bool); rep[:, 1:] = x[:, 1:] == x[:, :-1]
    assert np.sum(rep & (i < 0)) > 1000 and np.sum(rep & (i > 0)) > 1000
    nov, _ = bank(L, "novect", x, 20001, 20002)
    for c in range(4):
        assert M.same_bits(nov[c], M.fmdemod_quadri_novect_cf(x[c])[0]), c
        if M.have_ref():
            assert M.same_bits(nov[c], M.ref_novect(x[c])[0]), c
    neg = nov[rep & (i < 0)]
    assert np.any(np.signbit(neg[neg == 0])), "the build's form gives -0 where a repeated sample has I < 0"


def test_dcblock_in_place_equals_separate_buffers(L):
    rng = np.random.default_rng(5)
    for n, stride in ((9, 9), (1000, 1003), (64, 64)):
        x = M.real_rows(rng, 5, n)
        sep, st_sep = bank(L, "dcblock", x, stride, stride + 2, arg=(0.9, 0.0))
        buf = rows_in(x, stride, F)
        st = np.zeros((5, 2), F)
        assert L.csdrb_dcblock_bank_ff(P(buf), stride, P(buf), stride, 5, n, 0.9, P(st), None) == 0, L.csdrb_last_error()
        assert M.same_bits(buf[:, :n], sep) and M.same_bits(st, st_sep), n


def test_refusals(L):
    d_cf = np.zeros(64, np.complex64); d_f = np.zeros(512, F); d_state = np.zeros(16, F)
    assert M.refusals(L, P(d_cf), P(d_f), P(d_state)) == []
    for f, args in ((L.csdrb_fmdemod_atan_bank_cf, (P(d_cf), 0, P(d_f), 0, 0, 0, None, None, None)),
                    (L.csdrb_amdemod_estimator_bank_cf, (P(d_cf), 8, P(d_f), 8, 1, 0, 0.0, 0.0, None)),
                    (L.csdrb_dcblock_bank_ff, (P(d_f), 8, P(d_f), 8, 0, 8, 0.0, P(d_state), None))):
        assert f(*args) == 0                                           # nothing to do is not an error


def test_dropins(L):
    """Part A: the libcsdr signatures with their by-value struct returns, call after call"""
    rng = np.random.default_rng(2)
    x = M.complex_rows(rng, 1, 700)[0]
    x[:M.edge_row().size] = M.edge_row()
    r = M.real_rows(rng, 1, 700)[0]
    y = np.empty(700, F)
    phase, last, dcp = 0.0, M.CF(0.0, 0.0), M.DcBlock(0.0, 0.0)
    want_ph, want_last, want_dc = 0.0, 0j, None
    for a, b in ((0, 300), (300, 301), (301, 700)):
        phase = L.fmdemod_atan_cf(P(x[a:]), P(y), b - a, phase)
        w, want_ph = M.fmdemod_atan_cf(x[a:b], want_ph)
        assert M.same_bits(y[:b - a], w) and M.same_bits(F(phase), want_ph)
        last = L.fmdemod_quadri_novect_cf(P(x[a:]), P(y), b - a, last)
        w, want_last = M.fmdemod_quadri_novect_cf(x[a:b], want_last)
        assert M.same_bits(y[:b - a], w) and (last.i, last.q) == (x[b - 1].real, x[b - 1].imag) or np.isnan(x[b - 1])
        L.amdemod_estimator_cf(P(x[a:]), P(y), b - a, 0.0, 0.0)
        assert M.same_bits(y[:b - a], M.amdemod_estimator_cf(x[a:b]))
        dcp = L.dcblock_ff(P(r[a:]), P(y), b - a, 0.0, dcp)
        w, want_dc = M.dcblock_rows(r[None, a:b], 0.0, want_dc)
        assert M.same_bits(y[:b - a], w[0]) and M.same_bits(np.array([dcp.last_input, dcp.last_output], F), want_dc[0])
    # a zero-length call returns its carry unchanged
    assert L.fmdemod_atan_cf(P(x), P(y), 0, 1.5) == F(1.5)
    keep = L.dcblock_ff(P(r), P(y), 0, 0.0, M.DcBlock(0.5, -0.25))
    assert (keep.last_input, keep.last_output) == (0.5, -0.25)
    # dcblock_ff in place
    buf = r.copy(); sep = np.empty_like(r)
    s1 = L.dcblock_ff(P(r), P(sep), 700, 0.5, M.DcBlock(0.0, 0.0))
    s2 = L.dcblock_ff(P(buf), P(buf), 700, 0.5, M.DcBlock(0.0, 0.0))
    assert M.same_bits(buf, sep) and M.same_bits([s1.last_input, s1.last_output], [s2.last_input, s2.last_output])
