"""CPU tier of the BPSK31 transmit banks (csdr_b200/csrc/psk31_tx.cu): the checks of tests/psk31_tx/psk31_tx.py on the emulated library
(tests/host_shim/emul_build.build_full_once, the C ABI and the drop-ins included) under the three fiber orders, against the compiled reference
(oracle/_ref/libcsdr_ref.so) and the numpy restatements.  The full-size cases (1024 channels, every rate table up to I = 8192) run in
tests/test_gpu_psk31_tx.py."""
import os
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "psk31_tx"))
import emul_build  # noqa: E402
import psk31_tx as T  # noqa: E402

pytestmark = pytest.mark.skipif(not T.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built (needs the reference sources at build time)")
ORDERS = ["alternate", "reverse", "random"]


@pytest.fixture(scope="module", params=ORDERS)
def drv(request, tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    import csdr_b200
    lib, _ = emul_build.build_full_once(tmp_path_factory)
    copy = Path(lib).with_name(f"libcsdr_b200_emul_psk31tx_{request.param}.so")
    if not copy.exists():
        shutil.copy(lib, copy)
    saved_env = os.environ.get("CUDA_EMUL_ORDER")
    saved = csdr_b200.LIB_PATH, csdr_b200._lib
    os.environ["CUDA_EMUL_ORDER"] = request.param
    csdr_b200.LIB_PATH, csdr_b200._lib = copy, None
    try:
        yield T.EmulDriver(csdr_b200)
    finally:
        csdr_b200.LIB_PATH, csdr_b200._lib = saved
        if saved_env is None:
            os.environ.pop("CUDA_EMUL_ORDER", None)
        else:
            os.environ["CUDA_EMUL_ORDER"] = saved_env


# ---- varicode encoder ---------------------------------------------------------------------------------------------------------------
def test_encoder_every_byte_value(drv):
    T.check_encoder(drv, np.arange(256, dtype=np.uint8)[None, :])
    T.check_encoder(drv, np.arange(256, dtype=np.uint8).reshape(4, 64))


def test_encoder_readme_example(drv):
    bits, ip, os_ = T.encoder_bank(drv, np.frombuffer(b"aaa", np.uint8)[None, :])
    assert bits[0, :os_[0]].tolist() == [1, 0, 1, 1, 0, 0] * 3 and ip[0] == 3


def test_encoder_cut_at_every_position(drv):
    text = np.frombuffer(b"Hi \x85 CQ\x00z~", np.uint8)
    for m in range(-2, 12 * text.size + 3):
        T.check_encoder(drv, text[None, :], output_max_size=m)


def test_encoder_lengths_and_long_rows(drv):
    rng = np.random.default_rng(1)
    text = T.text_rows(rng, 5, 3000)                  # rows of several scan chunks (1024 bytes each)
    T.check_encoder(drv, text, lengths=[0, 3000, 1024, 1025, 7])
    T.check_encoder(drv, text[:2], output_max_size=9000)


def test_encoder_output_decodes_to_the_text(drv):
    import psk31
    rng = np.random.default_rng(2)
    text = T.text_rows(rng, 3, 400)
    bits, ip, os_ = T.encoder_bank(drv, text)
    for c in range(3):
        got, _ = psk31.varicode_decode(np.concatenate([bits[c, :os_[c]], np.zeros(4, np.uint8)]))
        want = bytes(b for b in text[c].tobytes() if 0 < b < 0x80)
        assert got == want, c


# ---- differential codec -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("encode", [1, 0])
def test_codec_against_reference(drv, encode):
    rng = np.random.default_rng(3 + encode)
    for n in (1, 31, 33, 2047, 2049, 5000):
        x = rng.integers(0, 4, (3, n)).astype(np.uint8)
        x[:, rng.integers(0, n, 3)] = 200
        T.check_codec(drv, x, encode, np.array([0, 1, 7], np.uint8))
    x = rng.integers(0, 3, (4, 700)).astype(np.uint8)
    T.check_codec(drv, x, encode, np.array([0, 1, 2, 255], np.uint8), lengths=[0, 700, 33, 699])


@pytest.mark.parametrize("encode", [1, 0])
def test_codec_split_equals_one_call(drv, encode):
    rng = np.random.default_rng(5)
    x = rng.integers(0, 2, (2, 3001)).astype(np.uint8)
    whole, st_whole = T.codec_bank(drv, x, encode, np.zeros(2, np.uint8))
    st, parts, pos = np.zeros(2, np.uint8), [], 0
    for size in (1, 31, 0, 2048, 921):
        out, st = T.codec_bank(drv, np.ascontiguousarray(x[:, pos:pos + size]), encode, st)
        parts.append(out); pos += size
    assert np.array_equal(np.concatenate(parts, 1), whole) and np.array_equal(st, st_whole)


# ---- PSK modulator ------------------------------------------------------------------------------------------------------------------
def test_modulator_every_n_psk_and_byte(drv):
    T.check_modulator_grid(drv)


def test_modulator_rows_and_lengths(drv):
    rng = np.random.default_rng(6)
    x = rng.integers(0, 2, (3, 9000)).astype(np.uint8)
    got = T.modulator_bank(drv, x, 2, lengths=[9000, 0, 8193])
    want = T.ref_psk_modulate(x[0], 2)
    assert np.array_equal(got[0].view(np.uint32), want.view(np.uint32))
    assert np.all(got[1] == 0) and np.all(got[2, 8193:] == 0)
    assert np.array_equal(got[2, :8193].view(np.uint32), T.ref_psk_modulate(x[2, :8193], 2).view(np.uint32))


# ---- sine interpolator --------------------------------------------------------------------------------------------------------------
def test_interpolator_rate_tables(drv):
    T.check_rates(drv, list(range(1, 80)) + [255, 256, 257, 1000, 2047, 2048, 2049, 4096, 8191, 8192, 8193, 9001])


@pytest.mark.parametrize("I", [1, 2, 3, 7, 256, 1000])
def test_interpolator_against_reference(drv, I):
    rng = np.random.default_rng(I)
    n = max(3, 3000 // I)
    x = (rng.standard_normal((3, n)) + 1j * rng.standard_normal((3, n))).astype(np.complex64)
    T.check_interp(drv, x, I, np.array([0, 1 - 1j, 0.5j], np.complex64))
    T.check_interp(drv, x, I, np.array([2 + 2j, 0, 1], np.complex64), lengths=[0, n, n - 1])


def test_interpolator_large_I_path(drv):
    rng = np.random.default_rng(9)
    x = (rng.standard_normal((2, 3)) + 1j * rng.standard_normal((2, 3))).astype(np.complex64)
    T.check_interp(drv, x, 9001, np.array([1j, -1], np.complex64))


def test_interpolator_nan_inf_stay_local(drv):
    rng = np.random.default_rng(10)
    x = (rng.standard_normal((2, 200)) + 1j * rng.standard_normal((2, 200))).astype(np.complex64)
    x = T.with_specials(x, rng)
    out, _ = T.check_interp(drv, x, 7, np.array([np.inf, 0], np.complex64))
    bad = ~np.isfinite(x.view(np.float32).reshape(2, 200, 2)).all(2)
    o = ~np.isfinite(out[:, :1400].view(np.float32).reshape(2, 200, 7, 2)).all(3)
    prev = np.concatenate([np.array([[True], [False]]), bad[:, :-1]], 1)
    assert np.all(~o | bad[:, :, None] | prev[:, :, None])               # an output is non-finite only next to a non-finite input


def test_interpolator_last_carried_across_splits(drv):
    rng = np.random.default_rng(11)
    x = (rng.standard_normal((2, 300)) + 1j * rng.standard_normal((2, 300))).astype(np.complex64)
    whole, last_whole = T.interp_bank(drv, x, 5, np.zeros(2, np.complex64))
    last, parts, pos = np.zeros(2, np.complex64), [], 0
    for size in (1, 0, 137, 162):
        out, last = T.interp_bank(drv, np.ascontiguousarray(x[:, pos:pos + size]), 5, last)
        parts.append(out[:, :size * 5]); pos += size
    assert np.array_equal(np.concatenate(parts, 1).view(np.uint32), whole[:, :1500].view(np.uint32))
    assert np.array_equal(last.view(np.uint32), last_whole.view(np.uint32))


# ---- refusals and drop-ins ----------------------------------------------------------------------------------------------------------
def test_refusals(drv):
    T.refusals(drv)


def test_dropins_equal_the_reference(drv):
    import ctypes as C
    L = drv.L
    rng = np.random.default_rng(12)
    text = T.text_rows(rng, 1, 500)[0]
    out = np.zeros(6000, np.uint8); ip, os_ = C.c_int(), C.c_int()
    L.psk31_varicode_encoder_u8_u8(text.ctypes.data, out.ctypes.data, text.size, 6000, C.byref(ip), C.byref(os_))
    rb, rip, ros = T.ref_varicode_encode(text, 6000)
    assert (ip.value, os_.value) == (rip, ros) and np.array_equal(out[:ros], rb)
    x = rng.integers(0, 3, 777).astype(np.uint8)
    for enc in (0, 1):
        y = np.zeros(777, np.uint8)
        s = L.differential_codec(x.ctypes.data, y.ctypes.data, 777, enc, 5)
        ry, rs = T.ref_differential_codec(x, enc, 5)
        assert np.array_equal(y, ry) and s == rs
    sym = rng.integers(0, 2, 300).astype(np.uint8); z = np.zeros(300, np.complex64)
    L.psk_modulator_u8_c(sym.ctypes.data, z.ctypes.data, 300, 2)
    assert np.array_equal(z.view(np.uint32), T.ref_psk_modulate(sym, 2).view(np.uint32))
    zi = np.zeros(300 * 16, np.complex64)
    import csdr_b200
    r = L.psk31_interpolate_sine_cc(z.ctypes.data, zi.ctypes.data, 300, 16, csdr_b200._CF(0.5, -0.5))
    want, wl = T.ref_interpolate_sine(z, 16, 0.5 - 0.5j)
    assert np.array_equal(zi.view(np.uint32), want.view(np.uint32)) and complex(r.i, r.q) == complex(wl)
