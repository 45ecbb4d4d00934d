"""CPU tier: the rational_resampler_ff bank (csdr_b200/csrc/resample.cu) -- its host-side state function and the shipped kernel and launcher
executed under tests/host_shim/cuda_emul.h -- against the compiled reference (exact integer state and output count, outputs within 1e-5), the
strict restatement tests/resampler/resampler_oracle.c (bit for bit) and a float64 sum (per-output rounding bound)."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "resampler"))
import emul_build  # noqa: E402
import resampler as R  # noqa: E402

from oracle.pyoracle import rel_rms  # noqa: E402

INT_MAX = 2**31 - 1


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, names = emul_build.build_file(tmp_path_factory.mktemp("emul_resample"), "resample.cu")
    assert {"rational_resampler_state", "launch_rational_resampler_bank"} <= set(names)
    return lib


@pytest.fixture(scope="module")
def ro():
    return R.Oracle()


@pytest.fixture(scope="module")
def rref():
    if not R.have_ref():
        pytest.skip("oracle/_ref/libcsdr_ref.so not built (needs the reference sources at build time)")
    return R.Ref()


def state(L, n, I, D, T, ltd):
    st = (C.c_int * 3)()
    n_out = L.emul_rational_resampler_state(n, I, D, T, ltd, C.cast(st, C.c_void_p))
    assert n_out == st[1]
    return tuple(st)


def bank(L, x, I, D, taps, ltd=0, in_stride=None, out_stride=None, channels=None):
    """run the emulated launcher on the rows of x ([C, n] float32); returns (rc, out array incl. the sentinel-filled slack, state)"""
    x = np.ascontiguousarray(np.atleast_2d(x), np.float32)
    ch = x.shape[0] if channels is None else channels
    n = x.shape[1]
    in_stride = in_stride or n
    xin = np.full((max(ch, 1), in_stride), np.float32(-7.0)); xin[:x.shape[0], :n] = x
    cap = max(n * I // D, 1)
    out_stride = out_stride or cap + 5
    out = np.full((max(ch, 1), out_stride), np.float32(1234.5))
    taps = np.ascontiguousarray(taps, np.float32)
    st = (C.c_int * 3)()
    rc = L.emul_launch_rational_resampler_bank(xin.ctypes.data, in_stride, out.ctypes.data, out_stride, ch, n, I, D, taps.ctypes.data, taps.size, ltd,
                                               C.cast(st, C.c_void_p))
    return rc, out, tuple(st)


def signal(n, seed=0):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    return (0.7 * np.sin(2 * np.pi * 0.017 * t) + 0.2 * rng.standard_normal(n)).astype(np.float32)


def test_state_equals_the_reference_loop_over_a_sweep(L, ro, rref):
    """I, D <= 24, several T and n, every last_taps_delay: host state == compiled reference == strict oracle"""
    zeros = np.zeros(200, np.float32)
    checked = 0
    for I in range(1, 25):
        for D in range(1, 25):
            for T in (1, 7, 24, 79):
                taps = np.ones(T, np.float32)
                for n in (0, 1, 5, 23, 60, 200):
                    for ltd in range(I):
                        got = state(L, n, I, D, T, ltd)
                        _, so = ro.rational_resampler_ff(zeros[:n], I, D, taps, ltd)
                        assert got == so, (n, I, D, T, ltd, got, so)
                        if n * I // D == 0:
                            assert got == (0, 0, ltd)                 # the reference leaves these fields uninitialised
                            continue
                        _, sr = rref.rational_resampler_ff(zeros[:n], I, D, taps, ltd)
                        assert got == sr, (n, I, D, T, ltd, got, sr)
                        checked += 1
    assert checked > 100_000


GEOMS = [(3, 4, 79), (3, 2, 79), (5, 2, 201), (1, 3, 79), (4, 1, 79), (24, 25, 201), (1, 100, 79), (7, 3, 1001)]


@pytest.mark.parametrize("I,D,T", GEOMS)
def test_bank_bit_exact_vs_oracle_bound_vs_float64_and_near_reference(L, ro, rref, oracle, I, D, T):
    n = 1500 if I * 1500 // D <= 6000 else 700
    taps = R.lowpass(oracle, T, I, D)
    rows = np.stack([signal(n, s) for s in range(3)])
    for ltd in sorted({0, I - 1, I // 2}):
        rc, out, st = bank(L, rows, I, D, taps, ltd, in_stride=n + 9, out_stride=n * I // D + 3)
        want_y, want_st = ro.rational_resampler_ff(rows[0], I, D, taps, ltd)
        assert rc == want_st[1] and st == want_st, (rc, st, want_st)
        assert np.all(out[:, rc:] == np.float32(1234.5))                      # nothing written past the outputs
        s = (np.arange(rc, dtype=np.int64) * D + I - 1 - ltd) // I
        d = (ltd + s * I - np.arange(rc, dtype=np.int64) * D) % I
        terms = (T - d) // I
        for c in range(3):
            yo, _ = ro.rational_resampler_ff(rows[c], I, D, taps, ltd)
            assert np.array_equal(out[c, :rc], yo), (c, ltd)
            # float64 sum of the same terms; bound (terms + 2) ulps-of-1 times I * sum|x h|
            y64 = np.zeros(rc); mag = np.zeros(rc)
            for i in range(int(terms.max(initial=0))):
                live = i < terms
                idx_h = np.where(live, d + i * I, 0); idx_x = np.where(live, s + i, 0)
                p = np.where(live, rows[c][idx_x].astype(np.float64) * taps[idx_h].astype(np.float64), 0.0)
                y64 += p; mag += np.abs(p)
            err = np.abs(out[c, :rc].astype(np.float64) - I * y64)
            assert np.all(err <= (terms + 2) * 2.0**-24 * I * mag + 1e-30), (c, float(err.max()))
            if ltd == 0:
                yr, sr = rref.rational_resampler_ff(rows[c], I, D, taps)
                assert sr == st and rel_rms(out[c, :rc], yr) <= 1e-5


def test_tile_edges_and_many_tiles(L, ro, oracle):
    """4/1 on 3000 samples: 11999 outputs over 12 tiles of 1024; ragged last tile; taps > one tile's outputs (T = 4001)"""
    for I, D, T, n in ((4, 1, 79, 3000), (1, 1, 4001, 5000), (2, 3, 8001, 9000)):
        taps = R.lowpass(oracle, T, I, D)
        x = signal(n, 5)
        rc, out, st = bank(L, x, I, D, taps)
        yo, so = ro.rational_resampler_ff(x, I, D, taps)
        assert rc == so[1] > 0 and st == so and np.array_equal(out[0, :rc], yo), (I, D, T)


def test_nan_and_inf_stay_in_the_outputs_they_touch(L, ro, oracle):
    I, D, T, n = 3, 4, 79, 900
    taps = R.lowpass(oracle, T, I, D)
    x = signal(n, 3)
    x[300] = np.nan; x[611] = np.inf
    rc, out, st = bank(L, x, I, D, taps)
    yo, _ = ro.rational_resampler_ff(x, I, D, taps)
    assert np.array_equal(out[0, :rc], yo, equal_nan=True)
    s = (np.arange(rc) * D + I - 1) // I
    d = (s * I - np.arange(rc) * D) % I
    terms = (T - d) // I
    touched = ((s <= 300) & (300 < s + terms)) | ((s <= 611) & (611 < s + terms))
    assert np.array_equal(~np.isfinite(out[0, :rc]), touched)


def test_fewer_taps_than_interpolation_gives_zeros(L, oracle):
    taps = R.lowpass(oracle, 79, 147, 160)
    rc, out, st = bank(L, signal(2048), 147, 160, taps)
    assert rc == st[1] == 1881 and np.all(out[0, :rc] == 0)


def test_output_cap_repeats_the_last_output_in_the_next_call(L, ro, oracle):
    """rational_resampler_ff(..., 1, 100) with 79 taps on 4096 samples ends on the cap at (3900, 40, 0); the next call (CLI framing) starts
    from output 39's pair and computes it again"""
    taps = R.lowpass(oracle, 79, 1, 100)
    x = signal(8192, 8)
    rc, out, st = bank(L, x[:4096], 1, 100, taps)
    assert (rc, st) == (40, (3900, 40, 0))
    rc2, out2, st2 = bank(L, x[3900:3900 + 4096], 1, 100, taps, st[2])
    assert rc2 == 40 and out2[0, 0] == out[0, 39]


def test_refusals(L):
    taps = np.ones(16385, np.float32)
    st = (C.c_int * 3)()
    sp = C.cast(st, C.c_void_p)
    f = L.emul_launch_rational_resampler_bank
    assert f(None, 0, None, 0, 1, 1000, 3, 4, taps.ctypes.data, 16385, 0, sp) == -2 and b"taps" in L.emul_last_error()
    assert f(None, 0, None, 0, 1, 100000, 3, 4, taps.ctypes.data, 16384, 0, sp) == -1 and b"null" in L.emul_last_error()   # served, null rows
    assert f(None, 0, None, 0, 1, INT_MAX // 3 + 1, 3, 4, taps.ctypes.data, 79, 0, sp) == -2 and b"INT_MAX" in L.emul_last_error()
    assert f(None, 0, None, 0, 0, INT_MAX // 3, 3, 4, taps.ctypes.data, 79, 0, sp) == st[1] > 0        # zero rows: state only, no launch
    assert f(None, 0, None, 0, 1, 1000, 3, 4, taps.ctypes.data, 79, 3, sp) == -1 and b"last_taps_delay" in L.emul_last_error()
    assert f(None, 0, None, 0, 1, 1000, 0, 4, taps.ctypes.data, 79, 0, sp) == -1
    assert f(None, 0, None, 0, 1, 1000, 3, 0, taps.ctypes.data, 79, 0, sp) == -1
    assert f(None, 0, None, 0, 1, 1000, 3, 4, None, 79, 0, sp) == -1
    # the longest filter served at bandwidth 0.0005 (8001 taps) with one interpolation
    assert f(None, 0, None, 0, 0, 100000, 1, 1, taps.ctypes.data, 8001, 0, sp) == st[1] > 0


# ---- the whole library under emulation: the drop-in, the host design function and the `csdr` command (bodies of tests/test_gpu_resampler.py)
import test_gpu_resampler as gr  # noqa: E402


@pytest.fixture(scope="module")
def gpu(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    import csdr_b200
    lib, _ = emul_build.build_full_once(tmp_path_factory)
    saved = csdr_b200.LIB_PATH, csdr_b200._lib
    csdr_b200.LIB_PATH, csdr_b200._lib = lib, None
    csdr_b200.lib()
    yield csdr_b200
    csdr_b200.LIB_PATH, csdr_b200._lib = saved


@pytest.fixture(scope="module")
def clis(tmp_path_factory):
    import test_gpu_cli as g
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    if not g.REF.exists():
        pytest.skip("oracle/_ref/csdr_ref not built (needs the reference sources at build time)")
    _lib, cli = emul_build.build_full_once(tmp_path_factory)
    return str(cli), str(g.REF)


test_lowpass_design_matches_the_oracle = gr.test_lowpass_design_matches_the_oracle
test_rational_resampler_dropin_golden_and_oracle = gr.test_rational_resampler_dropin_golden_and_oracle
test_rational_resampler_command = gr.test_rational_resampler_command
