"""CPU tier for the RTTY kernels (csdr_b200/csrc/rtty.cu): the shipped kernels and launchers run thread by thread under
tests/host_shim/cuda_emul.h and must equal the checker tests/rtty/rtty_oracle.c bit for bit -- characters, counts, start positions and the
stuck flag -- for channel counts that are not multiples of 4 warps, ragged starts, many calls per row, every spb / databits / stopbits / ratio
the oracle tests cover, and streams cut into blocks of any size, which must give the text of one pass.  Every test runs under two fiber
scheduling orders.  The drop-in serial_line_decoder_f_u8 runs on the whole emulated library against the compiled reference."""
import ctypes as C
import os
import shutil
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "rtty"))
import emul_build  # noqa: E402
import rtty  # noqa: E402

_built = {}
TEXT = b"RYRY CQ DE TEST 599 73, 14.080 (K1ABC/P) 'OK?' $1 #2\r\n"


@pytest.fixture(scope="module", params=["alternate", "random"])
def K(request, tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    if "rtty" not in _built:
        lib, names = emul_build.build_file(tmp_path_factory.mktemp("emul_rtty"), "rtty.cu")
        _built["rtty"] = (Path(lib._name), names, lib)
    so, names, proto = _built["rtty"]
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


class Params(C.Structure):
    _fields_ = [("samples_per_bits", C.c_float), ("databits", C.c_int), ("stopbits", C.c_float), ("bit_sampling_width_ratio", C.c_float)]


def run_sld(K, rows, starts, end, spb, databits, stopbits, ratio, bufsize, stride=None):
    ch = len(rows)
    stride = stride or max(end, 1) + 3
    xin = np.zeros((ch, stride), np.float32)
    for c, r in enumerate(rows):
        xin[c, :r.size] = r
    cap = rtty.max_outputs(end, spb, databits, stopbits)
    out = np.zeros((ch, cap), np.uint8); cnt = np.zeros(ch, np.int32); stuck = np.full(ch, 7, np.int32)
    st = np.array(starts, np.int32)
    p = Params(spb, databits, stopbits, ratio)
    rc = K.emul_launch_serial_line_bank(P(xin), stride, end, P(st), P(out), cap, P(cnt), P(stuck), ch, C.addressof(p), bufsize)
    assert rc >= 0, K.emul_last_error()
    return [out[c, :cnt[c]].tobytes() for c in range(ch)], st, stuck


def signal_rows(rng, ch, n, spb):
    """RTTY discriminator rows with noise, plus rows of the adversarial kinds of tests/test_oracle_rtty.py"""
    rows = []
    for c in range(ch):
        kind = c % 4
        if kind == 0:
            z = rtty.modulate(TEXT[:12 + c % 7], spb, rng, noise=0.01, lead_bits=float(rng.uniform(1, 9)))
            r = rtty.discriminator(z)
        elif kind == 1:
            r = (rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 30, n)).astype(np.float32)
        elif kind == 2:
            r = rng.choice(np.array([0.0, -0.0, 1e-45, -1e-45, 1.0, -1.0, np.nan, np.inf, -np.inf], np.float32), n)
        else:
            bits = rng.random(int(n / spb) + 2) < 0.5
            r = (np.repeat(np.where(bits, 1.0, -1.0), int(np.ceil(spb)))[:n] + 0.8 * rng.standard_normal(n)).astype(np.float32)
        r = np.resize(r, n).astype(np.float32)
        rows.append(r)
    return rows


@pytest.mark.parametrize("spb,databits,stopbits,ratio", [(5.0, 5, 1.5, 0.4), (44.0, 5, 1.5, 0.4), (44.0, 7, 1.0, 0.0), (176.02, 8, 2.0, 1.0),
                                                         (8.0, 8, 1.0, 0.93), (5.0, 1, 1.0, 0.4)])
def test_serial_line_bank_equals_checker(K, spb, databits, stopbits, ratio):
    """ragged starts, several calls per row (bufsize well below the row), the stuck flag where a call consumes nothing"""
    rng = np.random.default_rng(int(spb * 10) + databits)
    ch = 9
    span = int(np.float32(spb) * (np.float32(1 + databits) + np.float32(stopbits)))
    n = max(8 * span, 600)
    rows = signal_rows(rng, ch, n, spb)
    starts = [int(rng.integers(0, n // 3)) for _ in range(ch)]
    for bufsize in (span + 3, 2 * span + 17, n // 2, n):
        got, st, stuck = run_sld(K, rows, starts, n, spb, databits, stopbits, ratio, bufsize)
        for c in range(ch):
            want, pos, stk = rtty.serial_stream(rows[c], spb, databits, stopbits, ratio, bufsize, starts[c], n)
            assert got[c] == want and st[c] == pos and stuck[c] == int(stk), (bufsize, c)


def test_serial_line_bank_stuck_flag(K):
    """a character that starts at the second sample and does not fit: the call consumes nothing, the row stops with stuck = 1"""
    x = np.ones(64, np.float32); x[1:] = -1.0
    got, st, stuck = run_sld(K, [x, np.ones(64, np.float32)], [0, 0], 64, 44.0, 5, 1.5, 0.4, 64)
    want = rtty.serial_stream(x, 44.0, 5, 1.5, 0.4, 64)
    assert want == (b"", 0, True)
    assert got == [b"", b""] and list(st) == [0, 64] and list(stuck) == [1, 0]


def test_serial_line_bank_blocks_equal_one_pass(K):
    """the daemon's use: a stream arrives in blocks of any size; the rows keep [start, end) and the text equals one pass over the stream"""
    rng = np.random.default_rng(21)
    spb, bufsize = 20.0, 400
    zs = [rtty.modulate(TEXT, spb, rng, noise=0.01, lead_bits=float(3 + k), tail_bits=bufsize / spb + 3) for k in range(3)]
    n = min(z.size for z in zs)
    D = np.stack([rtty.discriminator(z)[:n] for z in zs])
    whole = [rtty.serial_stream(D[c], spb, 5, 1.5, 0.4, bufsize)[0] for c in range(3)]
    assert all(TEXT in rtty.baudot_decode(w)[0] for w in whole)
    acc = [b""] * 3; start = np.zeros(3, np.int32); end = 0
    while end < n:
        end = min(n, end + int(rng.integers(1, 900)))
        got, start, stuck = run_sld(K, list(D[:, :end]), start, end, spb, 5, 1.5, 0.4, bufsize)
        assert not stuck.any()
        acc = [a + g for a, g in zip(acc, got)]
    assert acc == whole


def test_serial_line_refusals(K):
    x = np.zeros(100, np.float32)
    for spb, nb, sb, r, bs in [(5.0, 0, 1.0, 0.4, 100), (5.0, 9, 1.0, 0.4, 100), (0.5, 5, 1.0, 0.4, 100), (5.0, 5, 0.5, 0.4, 100),
                               (5.0, 5, 1.5, 1.5, 100), (5.0, 5, 1.5, -0.1, 100), (float("nan"), 5, 1.5, 0.4, 100), (5.0, 5, 1.5, 0.4, 0)]:
        p = Params(spb, nb, sb, r)
        st = np.zeros(1, np.int32); cnt = np.zeros(1, np.int32); stuck = np.zeros(1, np.int32); out = np.zeros(100, np.uint8)
        assert K.emul_launch_serial_line_bank(P(x), 100, 100, P(st), P(out), 100, P(cnt), P(stuck), 1, C.addressof(p), bs) == -1
    p = Params(5.0, 5, 1.5, 0.4)
    assert K.emul_launch_serial_line_bank(P(x), 100, 100, P(st), P(out), 2, P(cnt), P(stuck), 1, C.addressof(p), 100) == -1     # room


# ---- baudot -------------------------------------------------------------------------------------------------------------------------
def run_bd(K, rows, modes):
    ch = len(rows); n = max(max(r.size for r in rows), 1)
    xin = np.zeros((ch, n + 5), np.uint8)
    for c, r in enumerate(rows):
        xin[c, :r.size] = r
    lengths = np.array([r.size for r in rows], np.int32)
    out = np.zeros((ch, n), np.uint8); cnt = np.zeros(ch, np.int32); m = np.array(modes, np.uint8)
    assert K.emul_launch_baudot_bank(P(xin), n + 5, P(out), n, ch, n, P(lengths), P(m), P(cnt)) >= 0
    return [out[c, :cnt[c]].tobytes() for c in range(ch)], m


def test_baudot_bank_equals_checker_and_carries_the_mode(K):
    rng = np.random.default_rng(9)
    enc = np.array(rtty.ita2_encode(TEXT), np.uint8)
    rows = [enc, rng.integers(0, 256, 700).astype(np.uint8), rng.choice(np.array([27, 31, 0, 1, 16, 4, 33, 255], np.uint8), 300),
            rng.integers(0, 32, 77).astype(np.uint8), np.zeros(0, np.uint8), np.array([27, 27, 31, 31, 27], np.uint8)]
    modes = [0, 1, 0, 1, 1, 0]
    got, m = run_bd(K, rows, modes)
    for c in range(len(rows)):
        want, wm = rtty.baudot_decode(rows[c], modes[c])
        assert got[c] == want and m[c] == wm, c
    assert got[0] == TEXT
    # a row cut into pieces: the FIGS/LTRS mode carries over
    pos, mode, acc = 0, 0, b""
    while pos < enc.size:
        k = int(rng.integers(1, 9))
        g, mv = run_bd(K, [enc[pos:pos + k]], [mode]); acc += g[0]; mode = int(mv[0]); pos += k
    assert acc == TEXT


# ---- the drop-in on the whole emulated library --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    L = C.CDLL(str(lib))
    L.serial_line_decoder_f_u8.argtypes = [C.POINTER(rtty._Serial), C.c_void_p, C.c_void_p, C.c_int]
    return L


@pytest.mark.skipif(not rtty.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built")
def test_dropin_equals_reference(full):
    rng = np.random.default_rng(5)
    for spb, nb, sb, ratio in ((44.0, 5, 1.5, 0.4), (5.0, 8, 1.0, 0.25), (176.02, 7, 2.0, 1.0)):
        d = rtty.discriminator(rtty.modulate(TEXT[:20], spb, rng, noise=0.01))
        for n in (0, 1, 2, 50, int(4 * spb), d.size):
            x = np.ascontiguousarray(d[:n]); out = np.zeros(max(n, 1), np.uint8)
            s = rtty._Serial(spb, nb, sb, 0, 0, ratio)
            full.serial_line_decoder_f_u8(C.byref(s), x.ctypes.data if n else out.ctypes.data, out.ctypes.data, n)
            assert (out[:s.output_size].tobytes(), s.input_used) == rtty.ref_serial_line_decoder(x, spb, nb, sb, ratio), (spb, n)
