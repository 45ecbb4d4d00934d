"""The checker side of the BPSK31 transmit banks (csdr_b200/csrc/psk31_tx.cu): numpy restatements of psk31_varicode_encoder_u8_u8,
differential_codec, psk_modulator_u8_c and psk31_interpolate_sine_cc, bindings to the compiled reference (oracle/_ref/libcsdr_ref.so), the case
matrix, and checks that talk to the C ABI through a driver (dev(array) -> buffer, ptr(buffer), host(buffer) -> array, `L`, `stream`), so the
same bodies run on the emulated library and on the GPU.  TEST INFRASTRUCTURE.

The modulator's bound.  Entry b of the constellation is the float of the double cos/sin of the build's float phase p = fl(fl(b) * inc).  The
correctly rounded float of cos(p) and sin(p) is the restatement; where the double value lies within AMBIG_ULPS double ulps of a float rounding
midpoint, a double cos/sin that is not correctly rounded (the device's, within 2 double ulps) may round to either neighbour, and either is
accepted.  The reference build itself is within 2 float ulps of the restatement (its sincosf and libmvec paths), never in sign: that is the
bound against the build.
"""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
sys.path.insert(0, str(ROOT / "tests" / "psk31"))
sys.path.insert(0, str(ROOT / "tests"))
import psk31  # noqa: E402
from bitcmp import assert_bits_equal  # noqa: E402

REF_SO = ROOT / "oracle" / "_ref" / "libcsdr_ref.so"
AMBIG_ULPS = 4
_ref = None


class _CF(C.Structure):
    _fields_ = [("i", C.c_float), ("q", C.c_float)]


# ---- restatements -------------------------------------------------------------------------------------------------------------------
def _table():
    t = psk31.varicode_table()
    pad = np.zeros((256, 12), np.uint8)
    cnt = np.zeros(256, np.int64)
    for a, (code, bits) in enumerate(t):
        pad[a, :bits] = [(code >> (bits - 1 - k)) & 1 for k in range(bits)]
        cnt[a] = bits + 2
    return pad, cnt


_TAB = None


def varicode_encode(text, output_max_size=None):
    """-> (bits, input_processed, output_size) of one psk31_varicode_encoder_u8_u8 call"""
    global _TAB
    if _TAB is None:
        _TAB = _table()
    pad, cnt = _TAB
    t = np.frombuffer(bytes(text), np.uint8) if not isinstance(text, np.ndarray) else text.astype(np.uint8)
    c = cnt[t]
    incl = np.cumsum(c)
    m = 12 * t.size + 12 if output_max_size is None else output_max_size
    over = np.flatnonzero((incl > m) & (c > 0) | ((c == 0) & (incl - c > max(m, 0))))
    k = int(over[0]) if over.size else t.size
    bits = pad[t[:k]][np.arange(12)[None, :] < c[:k, None]]
    return bits.astype(np.uint8), k, int(bits.size)


def differential_codec(x, encode, state=0):
    """-> (out, state) of one differential_codec call"""
    x = np.asarray(x, np.uint8)
    if x.size == 0:
        return x.copy(), state
    if encode:
        z = np.cumsum(x == 0)
        out = np.where(z == 0, state, np.where(z & 1, int(state == 0), int(state != 0))).astype(np.uint8)
        return out, int(out[-1])
    prev = np.concatenate([[state], x[:-1]]).astype(np.uint8)
    return (x == prev).astype(np.uint8), int(x[-1])


def psk_phase(b, n_psk):
    inc = np.float32((2 * np.pi) / n_psk)
    return (np.asarray(b, np.uint8).astype(np.float32) * inc).astype(np.float32)


def _round_with_ambiguity(d):
    """float32 of float64 values and, per value, whether it lies within AMBIG_ULPS double ulps of a float rounding midpoint"""
    f = d.astype(np.float32)
    lo = np.where(f.astype(np.float64) <= d, f, np.nextafter(f, np.float32(-np.inf)))
    hi = np.nextafter(lo, np.float32(np.inf))
    mid = (lo.astype(np.float64) + hi.astype(np.float64)) / 2
    amb = np.abs(d - mid) <= AMBIG_ULPS * np.spacing(np.abs(d))
    return f, amb, lo, hi


def psk_modulate(b, n_psk):
    """-> (want complex64, ambiguous [N, 2] bool, low, high candidates as float32 [N, 2])"""
    ph = psk_phase(b, n_psk).astype(np.float64)
    d = np.stack([np.cos(ph), np.sin(ph)], 1)
    f, amb, lo, hi = _round_with_ambiguity(d)
    return f.view(np.complex64).reshape(-1), amb, lo, hi


def interpolate_sine(x, rates, last=0j):
    """psk31_interpolate_sine_cc with the given rate table (float32 [I]): every product and the sum rounded to float"""
    x = np.asarray(x, np.complex64)
    r = np.asarray(rates, np.float32)
    omr = (np.float32(1) - r).astype(np.float32)
    prev = np.concatenate([np.array([last], np.complex64), x[:-1]])
    out = np.empty((x.size, r.size, 2), np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        for k, comp in enumerate(("real", "imag")):
            v = getattr(x, comp).astype(np.float32)[:, None]
            p = getattr(prev, comp).astype(np.float32)[:, None]
            out[:, :, k] = ((v * r[None, :]).astype(np.float32) + (p * omr[None, :]).astype(np.float32)).astype(np.float32)
    return out.view(np.complex64).reshape(-1), (x[-1] if x.size else np.complex64(last))


# ---- the compiled reference ---------------------------------------------------------------------------------------------------------
def have_ref() -> bool:
    return REF_SO.exists()


def ref():
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_SO))
        vp, it = C.c_void_p, C.c_int
        L.psk31_varicode_encoder_u8_u8.argtypes = [vp, vp, it, it, C.POINTER(it), C.POINTER(it)]
        L.differential_codec.argtypes = [vp, vp, it, it, C.c_ubyte]; L.differential_codec.restype = C.c_ubyte
        L.psk_modulator_u8_c.argtypes = [vp, vp, it, it]
        L.psk31_interpolate_sine_cc.argtypes = [vp, vp, it, it, _CF]; L.psk31_interpolate_sine_cc.restype = _CF
        _ref = L
    return _ref


def ref_varicode_encode(text, output_max_size):
    t = np.ascontiguousarray(np.frombuffer(bytes(text), np.uint8) if not isinstance(text, np.ndarray) else text, np.uint8)
    out = np.zeros(max(output_max_size, 0) + 16, np.uint8)
    ip, os_ = C.c_int(0), C.c_int(0)
    ref().psk31_varicode_encoder_u8_u8(t.ctypes.data, out.ctypes.data, t.size, output_max_size, C.byref(ip), C.byref(os_))
    return out[:os_.value].copy(), ip.value, os_.value


def ref_differential_codec(x, encode, state=0):
    x = np.ascontiguousarray(x, np.uint8); out = np.zeros(max(x.size, 1), np.uint8)
    s = ref().differential_codec(x.ctypes.data, out.ctypes.data, x.size, int(encode), state)
    return out[:x.size], int(s)


def ref_psk_modulate(b, n_psk):
    b = np.ascontiguousarray(b, np.uint8); out = np.zeros(max(b.size, 1), np.complex64)
    ref().psk_modulator_u8_c(b.ctypes.data, out.ctypes.data, b.size, n_psk)
    return out[:b.size]


def ref_interpolate_sine(x, I, last=0j):
    x = np.ascontiguousarray(x, np.complex64); out = np.zeros(max(x.size * I, 1), np.complex64)
    r = ref().psk31_interpolate_sine_cc(x.ctypes.data, out.ctypes.data, x.size, I, _CF(np.float32(last.real), np.float32(last.imag)))
    return out[:x.size * I], np.complex64(complex(r.i, r.q))


def ref_rates(I):
    """the build's rate table: an input of 1+0j after last = 0 gives exactly r[j]"""
    return ref_interpolate_sine(np.array([1 + 0j], np.complex64), I)[0].real.astype(np.float32)


# ---- drivers ------------------------------------------------------------------------------------------------------------------------
class EmulDriver:
    """'device' buffers are 256-byte aligned host copies (cudaMalloc's alignment)"""
    stream = None

    def __init__(self, pkg):
        self.pkg, self.L = pkg, pkg.lib()

    def dev(self, a):
        a = np.ascontiguousarray(a)
        raw = np.empty(a.nbytes + 256, np.uint8)
        off = (-raw.ctypes.data) % 256
        d = raw[off:off + a.nbytes].view(a.dtype).reshape(a.shape)
        d[...] = a
        return d

    def ptr(self, d):
        return d.ctypes.data if d is not None else None

    def host(self, d):
        return d.copy()


class GpuDriver:
    def __init__(self, pkg):
        import torch
        self.torch, self.pkg, self.L = torch, pkg, pkg.lib()

    @property
    def stream(self):
        return self.pkg._stream()

    def dev(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def ptr(self, t):
        return t.data_ptr() if t is not None else None

    def host(self, t):
        self.torch.cuda.synchronize()
        return t.cpu().numpy()


def launches(drv):
    return int(drv.L.csdrb_kernel_launches())


# ---- bank calls ---------------------------------------------------------------------------------------------------------------------
def encoder_bank(drv, text, lengths=None, output_max_size=None):
    """text [C, N] uint8 -> (bits [C, M], input_processed [C], output_size [C])"""
    ch, n = text.shape
    m = 12 * n if output_max_size is None else output_max_size
    d_in, d_out = drv.dev(text), drv.dev(np.full((ch, max(m, 1)), 0xEE, np.uint8))
    d_ip, d_os = drv.dev(np.full(ch, -7, np.int32)), drv.dev(np.full(ch, -7, np.int32))
    d_len = drv.dev(np.asarray(lengths, np.int32)) if lengths is not None else None
    rc = drv.L.csdrb_psk31_varicode_encoder_bank_u8_u8(drv.ptr(d_in), n, drv.ptr(d_out), max(m, 1), ch, n, drv.ptr(d_len), m, drv.ptr(d_ip),
                                                       drv.ptr(d_os), drv.stream)
    assert rc >= 0, drv.L.csdrb_last_error()
    return drv.host(d_out), drv.host(d_ip), drv.host(d_os)


def codec_bank(drv, x, encode, state, lengths=None):
    ch, n = x.shape
    d_in, d_out = drv.dev(x), drv.dev(np.full((ch, max(n, 1)), 0xEE, np.uint8))
    d_st = drv.dev(np.asarray(state, np.uint8))
    d_len = drv.dev(np.asarray(lengths, np.int32)) if lengths is not None else None
    rc = drv.L.csdrb_differential_codec_bank_u8_u8(drv.ptr(d_in), n, drv.ptr(d_out), max(n, 1), ch, n, drv.ptr(d_len), int(encode), drv.ptr(d_st),
                                                   drv.stream)
    assert rc >= 0, drv.L.csdrb_last_error()
    return drv.host(d_out)[:, :n], drv.host(d_st)


def modulator_bank(drv, x, n_psk, lengths=None):
    ch, n = x.shape
    d_in, d_out = drv.dev(x), drv.dev(np.zeros((ch, max(n, 1)), np.complex64))
    d_len = drv.dev(np.asarray(lengths, np.int32)) if lengths is not None else None
    rc = drv.L.csdrb_psk_modulator_bank_u8_c(drv.ptr(d_in), n, drv.ptr(d_out), max(n, 1), ch, n, drv.ptr(d_len), n_psk, drv.stream)
    assert rc >= 0, drv.L.csdrb_last_error()
    return drv.host(d_out)[:, :n]


def interp_bank(drv, x, I, last, lengths=None):
    ch, n = x.shape
    d_in, d_out = drv.dev(x), drv.dev(np.full((ch, max(n * I, 1)), np.complex64(complex(7, 7))))
    d_last = drv.dev(np.asarray(last, np.complex64))
    d_len = drv.dev(np.asarray(lengths, np.int32)) if lengths is not None else None
    rc = drv.L.csdrb_psk31_interpolate_sine_bank_cc(drv.ptr(d_in), n, drv.ptr(d_out), max(n * I, 1), ch, n, drv.ptr(d_len), I, drv.ptr(d_last),
                                                    drv.stream)
    assert rc >= 0, drv.L.csdrb_last_error()
    return drv.host(d_out), drv.host(d_last)


# ---- checks -------------------------------------------------------------------------------------------------------------------------
def same_complex(got, want, what):
    """bit equality where both are numbers, NaN where either is NaN"""
    g, w = np.asarray(got, np.complex64).view(np.float32), np.asarray(want, np.complex64).view(np.float32)
    ng, nw = np.isnan(g), np.isnan(w)
    assert np.array_equal(ng, nw), (what, int(np.flatnonzero(ng != nw)[0]))
    assert_bits_equal(np.where(ng, 0, g).astype(np.float32), np.where(nw, 0, w).astype(np.float32), what)


def check_encoder(drv, text, lengths=None, output_max_size=None):
    """every row against the compiled reference (bits, input_processed, output_size) and the restatement; nothing past output_size written"""
    bits, ip, os_ = encoder_bank(drv, text, lengths, output_max_size)
    ch, n = text.shape
    m = 12 * n if output_max_size is None else output_max_size
    for c in range(ch):
        L = n if lengths is None else max(0, min(int(lengths[c]), n))
        rb, rip, ros = ref_varicode_encode(text[c, :L], m)
        assert (int(ip[c]), int(os_[c])) == (rip, ros), (c, L, m, int(ip[c]), int(os_[c]), rip, ros)
        assert np.array_equal(bits[c, :ros], rb), c
        assert np.all(bits[c, ros:] == 0xEE), c
        wb, wip, wos = varicode_encode(text[c, :L], m)
        assert (wip, wos) == (rip, ros) and np.array_equal(wb, rb), c
    return bits, ip, os_


def check_codec(drv, x, encode, state, lengths=None):
    out, st = codec_bank(drv, x, encode, state, lengths)
    ch, n = x.shape
    for c in range(ch):
        L = n if lengths is None else max(0, min(int(lengths[c]), n))
        ro, rs = ref_differential_codec(x[c, :L], encode, int(state[c]))
        assert np.array_equal(out[c, :L], ro), (c, encode)
        assert np.all(out[c, L:] == 0xEE), c
        assert int(st[c]) == rs, (c, encode, int(st[c]), rs)
        wo, ws = differential_codec(x[c, :L], encode, int(state[c]))
        assert np.array_equal(wo, ro) and ws == rs, c
    return out, st


def check_modulator_grid(drv, n_psks=range(1, 257)):
    """n_psk x every byte: each component the correctly rounded float (either neighbour where ambiguous), within 2 ulp of both reference paths
    (1-sample calls: its scalar sincosf; one 256-sample call: its libmvec body), bit-equal to both for n_psk 2, 4, 8 with bytes below n_psk.
    Returns the number of ambiguous components met."""
    b = np.arange(256, dtype=np.uint8)
    ambiguous = 0
    for n_psk in n_psks:
        got = modulator_bank(drv, b[None, :], n_psk)[0]
        want, amb, lo, hi = psk_modulate(b, n_psk)
        g, w = got.view(np.float32).reshape(-1, 2), want.view(np.float32).reshape(-1, 2)
        ok = (g.view(np.uint32) == w.view(np.uint32)) | (amb & ((g == lo) | (g == hi)))
        assert ok.all(), (n_psk, np.argwhere(~ok)[:4].tolist())
        ambiguous += int(amb.sum())
        vec = ref_psk_modulate(b, n_psk).view(np.float32).reshape(-1, 2)
        sca = np.array([ref_psk_modulate(b[k:k + 1], n_psk)[0] for k in range(256)], np.complex64).view(np.float32).reshape(-1, 2)
        for r in (vec, sca):
            assert np.array_equal(np.signbit(g), np.signbit(r)), n_psk
            ulps = np.abs(g.view(np.int32).astype(np.int64) - r.view(np.int32).astype(np.int64))
            assert np.all(ulps <= 2), (n_psk, int(ulps.max()))
            if n_psk in (2, 4, 8):
                assert np.array_equal(g[:n_psk].view(np.uint32), r[:n_psk].view(np.uint32)), n_psk
    return ambiguous


def check_rates(drv, Is):
    """the bank's rate table (an input of 1+0j after last = 0) equals the build's for every I"""
    for I in Is:
        got, _ = interp_bank(drv, np.array([[1 + 0j]], np.complex64), I, np.zeros(1, np.complex64))
        assert_bits_equal(got[0, :I].real.astype(np.float32), ref_rates(I), f"rates I={I}")


def check_interp(drv, x, I, last, lengths=None):
    out, new_last = interp_bank(drv, x, I, last, lengths)
    ch, n = x.shape
    rates = ref_rates(I)
    for c in range(ch):
        L = n if lengths is None else max(0, min(int(lengths[c]), n))
        ro, rl = ref_interpolate_sine(x[c, :L], I, complex(last[c]))
        same_complex(out[c, :L * I], ro, (I, c))
        wo, _ = interpolate_sine(x[c, :L], rates, complex(last[c]))
        same_complex(wo, ro, ("restatement", I, c))
        assert np.all(out[c, L * I:] == np.complex64(complex(7, 7))), c
        want_last = rl if L else np.complex64(last[c])
        same_complex(new_last[c:c + 1], np.array([want_last], np.complex64), ("last", I, c))
    return out, new_last


def with_specials(x, rng, k=3):
    f = x.reshape(-1).view(np.float32)
    for v in (np.nan, np.inf, -np.inf):
        f[rng.integers(0, f.size, k)] = v
    return x


def refusals(drv):
    """every refusal returns -1, launches nothing and leaves the _io arrays alone"""
    L = drv.L
    u8 = drv.dev(np.zeros((2, 64), np.uint8)); cf = drv.dev(np.zeros((2, 64), np.complex64)); big = drv.dev(np.zeros((2, 64 * 8), np.complex64))
    ints = drv.dev(np.full(2, 5, np.int32)); st = drv.dev(np.full(2, 3, np.uint8)); last = drv.dev(np.full(2, 1 + 2j, np.complex64))
    p = drv.ptr
    before = launches(drv)
    calls = [
        lambda: L.csdrb_psk31_varicode_encoder_bank_u8_u8(p(u8), 64, p(u8), 63, 2, 64, None, 64, p(ints), p(ints), drv.stream),
        lambda: L.csdrb_psk31_varicode_encoder_bank_u8_u8(p(u8), 63, p(u8), 64, 2, 64, None, 64, p(ints), p(ints), drv.stream),
        lambda: L.csdrb_differential_codec_bank_u8_u8(p(u8), 64, p(u8), 63, 2, 64, None, 1, p(st), drv.stream),
        lambda: L.csdrb_differential_codec_bank_u8_u8(p(u8), 63, p(u8), 64, 2, 64, None, 0, p(st), drv.stream),
        lambda: L.csdrb_psk_modulator_bank_u8_c(p(u8), 64, p(cf), 64, 2, 64, None, 0, drv.stream),
        lambda: L.csdrb_psk_modulator_bank_u8_c(p(u8), 64, p(cf), 64, 2, 64, None, 257, drv.stream),
        lambda: L.csdrb_psk_modulator_bank_u8_c(p(u8), 64, p(cf), 63, 2, 64, None, 2, drv.stream),
        lambda: L.csdrb_psk31_interpolate_sine_bank_cc(p(cf), 64, p(big), 64 * 8 - 1, 2, 64, None, 8, p(last), drv.stream),
        lambda: L.csdrb_psk31_interpolate_sine_bank_cc(p(cf), 64, p(big), 64 * 8, 2, 64, None, 0, p(last), drv.stream),
        lambda: L.csdrb_psk31_interpolate_sine_bank_cc(p(cf), 64, p(big), 64 * 8, 2, 64, None, -3, p(last), drv.stream),
        lambda: L.csdrb_psk31_interpolate_sine_bank_cc(p(cf), 64, p(big), 1 << 62, 3, 64, None, 8, p(last), drv.stream),
        lambda: L.csdrb_psk31_interpolate_sine_bank_cc(p(cf), 63, p(big), 64 * 8, 2, 64, None, 8, p(last), drv.stream),
    ]
    for k, f in enumerate(calls):
        assert f() == -1, k
        assert L.csdrb_last_error(), k
    assert launches(drv) == before
    assert np.all(drv.host(ints) == 5) and np.all(drv.host(st) == 3) and np.all(drv.host(last) == np.complex64(1 + 2j))


def text_rows(rng, ch, n, ascii_only=False):
    t = rng.integers(32, 127, (ch, n)).astype(np.uint8)
    if not ascii_only:
        t[rng.random((ch, n)) < 0.05] = 0
        t[rng.random((ch, n)) < 0.05] = 0x80 + rng.integers(0, 128)
        t[rng.random((ch, n)) < 0.05] = rng.integers(1, 32)
    return t
