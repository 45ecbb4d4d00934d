"""CPU tier for the amplitude modulator banks (csdr_b200/csrc/modulate.cu) through the C ABI of the whole emulated library: gain_ff, dsb_fc and
add_dcoffset_cc bit for bit against the restatements of tests/modulate/modulate.py and the compiled reference (its scalar and SSE paths, lengths
1..9 and longer), fixed_amplitude_cc bit for bit against its restatement and, with the build, within the float64 bound derived there; +-0,
subnormals, +-Inf and NaN, odd strides, several rows and in-place calls; the refusals; the libcsdr drop-ins."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "modulate"))
import emul_build  # noqa: E402
import modulate as M  # noqa: E402

needs_ref = pytest.mark.skipif(not M.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built")


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    return M.bind(C.CDLL(str(lib)))


def run(L, name, x, n, arg, in_stride=None, out_stride=None, inplace=False):
    """one bank call on host rows: x [C, n]; returns the [C, n] outputs (sentinels behind them must stay)"""
    tin, tout, _ = M.BANKS[name]
    ch = x.shape[0]
    in_stride = in_stride or max(n, 1)
    out_stride = in_stride if inplace else (out_stride or max(n, 1))
    xin = np.full((ch, in_stride), 7, tin); xin[:, :n] = x[:, :n]
    out = xin if inplace else np.full((ch, out_stride), 7, tout)
    assert M.call(L, name, xin.ctypes.data, in_stride, out.ctypes.data, out_stride, ch, n, arg) == n, L.csdrb_last_error()
    assert np.all(out[:, n:] == 7)
    return out[:, :n].copy()


@pytest.mark.parametrize("name", list(M.BANKS))
def test_banks_equal_restatement(L, name):
    rng = np.random.default_rng(len(name))
    for arg in M.ARGS[name]:
        for n in list(range(0, 10)) + [31, 64, 257, 1000]:
            x = M.rows_for(name, rng, 3, n)
            for in_stride, out_stride in ((None, None), (n + 1, n + 3), (n + 5 | 1, n + 2)):
                got = run(L, name, x, n, arg, in_stride, out_stride)
                for c in range(3):
                    assert M.same_bits(got[c], M.restate(name, x[c], arg)), (name, arg, n, in_stride, c)


@pytest.mark.parametrize("name", ["gain", "add_dcoffset", "fixed_amplitude"])
def test_in_place_equals_out_of_place(L, name):
    rng = np.random.default_rng(3)
    for n, stride in ((9, 9), (1000, 1003), (64, 64)):
        x = M.rows_for(name, rng, 4, n)
        arg = M.ARGS[name][-1]
        assert M.same_bits(run(L, name, x, n, arg, stride, inplace=True), run(L, name, x, n, arg, stride, stride + 2)), (name, n)


@needs_ref
@pytest.mark.parametrize("name", ["gain", "dsb", "add_dcoffset"])
def test_bit_for_bit_with_the_build(L, name):
    """the build's scalar path (lengths below 4) and SSE path (from 4 on) over +-0, subnormals, +-Inf, NaN and uniform samples"""
    rng = np.random.default_rng(5)
    for arg in M.ARGS[name]:
        for n in list(range(1, 10)) + [100, 4099]:
            x = M.rows_for(name, rng, 2, n)
            got = run(L, name, x, n, arg, n + 1, n + 3)
            for c in range(2):
                assert M.same_bits(got[c], M.ref_call(name, x[c], arg)), (name, arg, n, c)


@needs_ref
def test_fixed_amplitude_within_bound_of_the_build(L):
    rng = np.random.default_rng(6)
    worst = 0.0
    for A in (1.0, 2.0, 0.3, 1e5):
        for n in list(range(1, 10)) + [2000]:
            x = M.magnitude_rows(rng, 2, n)
            x[0, :min(n, 2)] = [0j, complex(0, -0.0)][:min(n, 2)]
            got = run(L, "fixed_amplitude", x, n, A)
            for c in range(2):
                worst = max(worst, M.fixed_amplitude_ok(got[c], x[c], A, M.ref_call("fixed_amplitude", x[c], A)))
                assert M.same_bits(got[c], M.fixed_amplitude_cc(x[c], A))
    assert worst > 0


def test_fixed_amplitude_specials_follow_the_restatement(L):
    x = np.array([[complex(np.inf, 0.5), complex(np.nan, 1), complex(np.nan, np.nan), 0j, complex(-0.0, -0.0), complex(1e-30, 0),
                   complex(3, 0), complex(0, -4), complex(2e19, 2e19)]], np.complex64)
    got = run(L, "fixed_amplitude", x, x.shape[1], 2.0)
    want = M.fixed_amplitude_cc(x[0], 2.0)
    assert M.same_bits(got[0], want)
    assert np.all(got[0, 3:6] == 0) and got[0, 6] == 2 and got[0, 7] == -2j and np.all(got[0, 8] == 0)


def test_nonfinite_stays_in_its_sample(L):
    rng = np.random.default_rng(7)
    for name in M.BANKS:
        x = M.rows_for(name, rng, 2, 300)
        clean = x.copy(); clean[np.isnan(clean) | np.isinf(clean)] = 0.5
        bad = clean.copy(); bad[1, 100] = np.nan; bad[1, 200] = np.inf
        a, b = run(L, name, clean, 300, 2.0), run(L, name, bad, 300, 2.0)
        keep = np.ones(300, bool); keep[[100, 200]] = False
        assert M.same_bits(a[0], b[0]) and M.same_bits(a[1][keep], b[1][keep]), name


def test_refusals_launch_nothing(L):
    h_in = np.zeros(64, np.complex64); h_out = np.full(64, 7, np.complex64)
    before = L.csdrb_kernel_launches()
    assert M.refusals(L, h_in.ctypes.data, h_out.ctypes.data) == []
    assert L.csdrb_kernel_launches() == before and np.all(h_out == 7)


@needs_ref
def test_dropins_against_the_build(L):
    rng = np.random.default_rng(8)
    for n in (1, 5, 4096):
        x = M.real_rows(rng, 1, n)[0]
        out = np.zeros(n, np.float32)
        L.gain_ff(x.ctypes.data, out.ctypes.data, n, -1.5)
        assert M.same_bits(out, M.ref_call("gain", x, -1.5))
        L.gain_ff(x.ctypes.data, x.ctypes.data, n, -1.5)                          # input == output
        assert M.same_bits(x, out)
        z = M.complex_rows(rng, 1, n)[0]
        outc = np.zeros(n, np.complex64)
        L.add_dcoffset_cc(z.ctypes.data, outc.ctypes.data, n)
        assert M.same_bits(outc, M.ref_call("add_dcoffset", z))
        m = M.magnitude_rows(rng, 1, n)[0]
        L.fixed_amplitude_cc(m.ctypes.data, outc.ctypes.data, n, 1.5)
        assert M.same_bits(outc, M.fixed_amplitude_cc(m, 1.5))
        M.fixed_amplitude_ok(outc, m, 1.5, M.ref_call("fixed_amplitude", m, 1.5))
