"""The checker side of the sample-format conversions convert_s8_f, convert_f_s8, convert_f_u8, convert_s24_f and convert_f_s24
(csdr_b200/csrc/elementwise.cu): numpy restatements of what the reference's -O3 -ffast-math x86 build computes, bindings to the compiled
reference (oracle/_ref/libcsdr_ref.so), the test vectors, and the C ABI calls both tiers make through a `Dev` (the emulated library, whose
device memory is host memory, or the real library on a CUDA device).  TEST INFRASTRUCTURE.

The build's arithmetic, pinned here and checked against the build itself:
  s8 -> f32   (float)b * 0x3c010204 (the float reciprocal of 127), not a division
  f32 -> s8   cvttss2si(x * 127.0f), low byte
  f32 -> u8   cvttsd2si((double)(x * 255.0f) * 0.5 + 128.0), low byte
  f32 -> s24  cvttss2si(x * 8388607.0f), low three bytes; bigendian = 0 writes the most significant byte first, 1 the least
  s24 -> f32  (float)(bytes as the top of an int32) * 0x30000001 (the float reciprocal of 2147483392); the same byte orders
cvttss2si / cvttsd2si give INT_MIN (low bytes zero) for NaN, +-Inf and anything outside the int32 range."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
REF_SO = ROOT / "oracle" / "_ref" / "libcsdr_ref.so"
F = np.float32
S8_RECIP = np.array([0x3C010204], np.uint32).view(F)[0]
S24_RECIP = np.array([0x30000001], np.uint32).view(F)[0]
INT_MIN = -(2 ** 31)
# name: (input item bytes, output item bytes, takes bigendian)
KINDS = {"s8_f": (1, 4, False), "f_s8": (4, 1, False), "f_u8": (4, 1, False), "s24_f": (3, 4, True), "f_s24": (4, 3, True)}
_ref = None


# ---- restatements ------------------------------------------------------------------------------------------------------------------------
def x86_trunc(v):
    """cvttss2si / cvttsd2si on a float32 or float64 array -> int64 values of the int32 result"""
    v = np.asarray(v)
    lo = -2147483648.0 if v.dtype == F else -2147483649.0
    with np.errstate(invalid="ignore"):
        bad = ~((v < 2147483648.0) & ((v >= lo) if v.dtype == F else (v > lo)))
        out = np.where(bad, 0, np.trunc(np.where(bad, 0, v))).astype(np.int64)
    out[bad] = INT_MIN
    return out


def s8_f(b):
    with np.errstate(all="ignore"):
        return (np.asarray(b, np.int8).astype(F) * S8_RECIP).astype(F)


def f_s8(x):
    with np.errstate(all="ignore"):
        return (x86_trunc((np.asarray(x, F) * F(127)).astype(F)) & 0xFF).astype(np.uint8).view(np.int8)


def f_u8(x):
    with np.errstate(all="ignore"):
        p = (np.asarray(x, F) * F(255)).astype(F)
        return (x86_trunc(p.astype(np.float64) * 0.5 + 128.0) & 0xFF).astype(np.uint8)


def f_s24(x, bigendian=0):
    with np.errstate(all="ignore"):
        t = x86_trunc((np.asarray(x, F) * F(8388607)).astype(F))
    b = np.stack([(t >> 16) & 0xFF, (t >> 8) & 0xFF, t & 0xFF], axis=-1).astype(np.uint8)
    return (b[..., ::-1] if bigendian else b).reshape(-1).copy()


def s24_f(b, bigendian=0):
    b = np.asarray(b, np.uint8).reshape(-1, 3).astype(np.uint32)
    if bigendian:
        b = b[:, ::-1]
    w = ((b[:, 0] << 24) | (b[:, 1] << 16) | (b[:, 2] << 8)).astype(np.uint32).view(np.int32)
    return (w.astype(F) * S24_RECIP).astype(F)


def restate(kind, x, bigendian=0):
    return {"s8_f": lambda: s8_f(x), "f_s8": lambda: f_s8(x), "f_u8": lambda: f_u8(x), "s24_f": lambda: s24_f(x, bigendian),
            "f_s24": lambda: f_s24(x, bigendian)}[kind]()


def same(a, b):
    """the same bytes (float outputs: NaN never arises, every conversion gives finite values)"""
    a, b = np.asarray(a), np.asarray(b)
    return a.nbytes == b.nbytes and a.tobytes() == b.tobytes()


# ---- test vectors ----------------------------------------------------------------------------------------------------------------------------
SCALES = {"f_s8": 127.0, "f_u8": 127.5, "f_s24": 8388607.0}      # x * scale (+ 128 for u8) is the value truncated


def straddle(xs):
    """each float32 value and its two neighbours on either side"""
    xs = np.asarray(xs, F)
    out = [xs]
    for d in (np.inf, -np.inf):
        a = np.nextafter(xs, F(d)); out += [a, np.nextafter(a, F(d))]
    return np.concatenate(out)


def float_specials(kind):
    """+-0, subnormals, +-1 and just beyond, the wrap region, |s| just below and at 2^31, +-Inf and NaN"""
    s = SCALES[kind]
    big = [2.0 ** 31 / s, -(2.0 ** 31) / s, 2.0 ** 32 / s, -(2.0 ** 32) / s, 3e38, -3e38] if kind != "f_u8" else \
          [(2.0 ** 31 - 128) / s, (-(2.0 ** 31) - 129) / s, (-(2.0 ** 31) - 128) / s, 3e38, -3e38]
    base = [0.0, -0.0, 1e-45, -1e-45, 1e-39, -1.1e-38, 1e-30, -1e-30, 1.0, -1.0, 1.01, -1.01, 1.02, -1.02, 2.0, -2.0, 0.5, -0.5, 7.5, -300.0]
    x = straddle(np.array(base + big, np.float64).astype(F))
    return np.concatenate([x, np.array([np.inf, -np.inf, np.nan, -np.nan], F)])


def float_boundaries(kind, ks):
    """inputs straddling the truncation boundaries of the integer results ks (where the scaled value crosses an integer)"""
    ks = np.asarray(ks, np.float64)
    x = (ks - 128.0) / 127.5 if kind == "f_u8" else ks / SCALES[kind]
    return straddle(x.astype(F))


def float_inputs(kind, rng, full=False):
    """every boundary of the in-range codes and the wrap region (s24: a subset, or all of them with full=True), specials, uniform values"""
    if kind == "f_s24":
        ks = np.arange(-(2 ** 23) - 2, 2 ** 23 + 3) if full else np.concatenate([np.arange(-300, 301), rng.integers(-(2 ** 23), 2 ** 23, 20000),
                                                                                  np.arange(2 ** 23 - 300, 2 ** 23 + 300), -np.arange(2 ** 23 - 300, 2 ** 23 + 300)])
    else:
        ks = np.arange(-600, 601)
    uni = rng.uniform(-1.5, 1.5, 4096).astype(F)
    return np.concatenate([float_specials(kind), float_boundaries(kind, ks), uni])


def byte_inputs(kind, rng, full=False):
    """s8: all 256 codes.  s24: all 2^24 codes (full) or the edges of the range, every top-byte value and random codes"""
    if kind == "s8_f":
        return np.arange(-128, 128, dtype=np.int16).astype(np.int8).view(np.uint8)
    if full:
        codes = np.arange(2 ** 24, dtype=np.uint32)
    else:
        codes = np.concatenate([np.arange(0, 4096), np.arange(2 ** 24 - 4096, 2 ** 24), np.arange(2 ** 23 - 4096, 2 ** 23 + 4096),
                                np.arange(256) << 16, (np.arange(256) << 16) | 0xFFFF, rng.integers(0, 2 ** 24, 30000)]).astype(np.uint32)
    return np.stack([codes & 0xFF, (codes >> 8) & 0xFF, codes >> 16], axis=-1).astype(np.uint8).reshape(-1)


def inputs(kind, rng, full=False):
    return byte_inputs(kind, rng, full) if kind in ("s8_f", "s24_f") else float_inputs(kind, rng, full)


# ---- the compiled reference ------------------------------------------------------------------------------------------------------------------
def have_ref() -> bool:
    return REF_SO.exists()


def ref():
    global _ref
    if _ref is None:
        L = C.CDLL(str(REF_SO))
        vp, it = C.c_void_p, C.c_int
        for name in ("convert_s8_f", "convert_f_s8", "convert_f_u8"):
            getattr(L, name).argtypes = [vp, vp, it]
        L.convert_s24_f.argtypes = [vp, vp, it, it]
        L.convert_f_s24.argtypes = [vp, vp, it, it]
        _ref = L
    return _ref


def ref_call(kind, x, bigendian=0):
    """the reference library on the whole array x (its input items)"""
    i, o, _ = KINDS[kind]
    x = np.ascontiguousarray(x)
    n = x.nbytes // i
    out = np.zeros(n * o, np.uint8)
    f = getattr(ref(), "convert_" + kind)
    if KINDS[kind][2]:
        f(x.ctypes.data, out.ctypes.data, n, bigendian)
    else:
        f(x.ctypes.data, out.ctypes.data, n)
    return out.view(F) if o == 4 else out.view(np.int8) if kind == "f_s8" else out


# ---- the C ABI through a Dev -------------------------------------------------------------------------------------------------------------------
def bind(L):
    vp, lg, it = C.c_void_p, C.c_long, C.c_int
    for name in ("csdrb_convert_s8_f", "csdrb_convert_f_s8", "csdrb_convert_f_u8"):
        getattr(L, name).argtypes = [vp, vp, lg, vp]
    L.csdrb_convert_s24_f.argtypes = [vp, vp, lg, it, vp]
    L.csdrb_convert_f_s24.argtypes = [vp, vp, lg, it, vp]
    for name in ("convert_s8_f", "convert_f_s8", "convert_f_u8"):
        getattr(L, name).argtypes = [vp, vp, it]
    L.convert_s24_f.argtypes = [vp, vp, it, it]
    L.convert_f_s24.argtypes = [vp, vp, it, it]
    L.csdrb_kernel_launches.restype = C.c_long
    L.csdrb_last_error.restype = C.c_char_p
    return L


def abi(L, kind, d_in, d_out, n, bigendian=0, stream=None):
    f = getattr(L, "csdrb_convert_" + kind)
    return f(d_in, d_out, n, bigendian, stream) if KINDS[kind][2] else f(d_in, d_out, n, stream)


class EmulDev:
    """the emulated library: device memory is host memory"""
    def __init__(self, L):
        self.L = bind(L); self.stream = None

    def buffer(self, data: bytes, nbytes):
        raw = np.zeros(nbytes + 128, np.uint8)
        off = (-raw.ctypes.data) % 64
        b = raw[off:off + nbytes]
        b[:len(data)] = np.frombuffer(data, np.uint8)
        return b

    def ptr(self, buf):
        return buf.ctypes.data

    def read(self, buf):
        return np.array(buf)


class CudaDev:
    """the real library on the current CUDA device, torch tensors as buffers"""
    def __init__(self):
        import torch
        import csdr_b200
        self.torch = torch
        csdr_b200.lib()
        self.L = bind(C.CDLL(str(csdr_b200.LIB_PATH)))                     # a handle of its own: the package's keeps its own argtypes
        self.stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def buffer(self, data: bytes, nbytes):
        t = self.torch.zeros(max(nbytes, 1), dtype=self.torch.uint8, device="cuda")
        if data:
            t[:len(data)] = self.torch.frombuffer(bytearray(data), dtype=self.torch.uint8).cuda()
        return t

    def ptr(self, buf):
        return buf.data_ptr()

    def read(self, buf):
        self.torch.cuda.synchronize()
        return buf.cpu().numpy()


SENTINEL = 0xA5


def run(dev, kind, x, bigendian=0, in_off=0, out_off=0):
    """one C ABI call on x (its input items) with the input at byte offset in_off and the output at out_off of their buffers; returns the
    output bytes and checks that nothing around them was written"""
    i, o, _ = KINDS[kind]
    raw = np.ascontiguousarray(x).view(np.uint8).reshape(-1)
    n = raw.size // i
    b_in = dev.buffer(bytes(in_off) + raw.tobytes(), in_off + raw.size + 16)
    out_bytes = out_off + n * o + 16
    b_out = dev.buffer(bytes([SENTINEL]) * out_bytes, out_bytes)
    rc = abi(dev.L, kind, dev.ptr(b_in) + in_off, dev.ptr(b_out) + out_off, n, bigendian, dev.stream)
    assert rc == 0, (kind, rc, dev.L.csdrb_last_error())
    got = dev.read(b_out)
    assert np.all(got[:out_off] == SENTINEL) and np.all(got[out_off + n * o:] == SENTINEL), (kind, n, in_off, out_off)
    return got[out_off:out_off + n * o].copy()


def as_output(kind, raw):
    o = KINDS[kind][1]
    return raw.view(F) if o == 4 else raw.view(np.int8) if kind == "f_s8" else raw


def check_against(dev, kind, x, bigendian=0, with_ref=True):
    """the kernel on the whole x equals the restatement, and (with the build) the build equals the restatement"""
    want = restate(kind, x, bigendian)
    assert same(as_output(kind, run(dev, kind, x, bigendian)), want), (kind, bigendian)
    if with_ref:
        assert same(ref_call(kind, x, bigendian), want), (kind, bigendian, "the build differs from the restatement")


def offsets_for(kind):
    """(input, output) byte offsets: 16-byte aligned, and off the group alignment -- any byte for byte buffers, whole floats for floats"""
    i, o, _ = KINDS[kind]
    odd = lambda size, k: k if size != 4 else 4 * k                             # noqa: E731
    return ((0, 0), (odd(i, 1), 0), (0, odd(o, 3)), (odd(i, 5), odd(o, 7)), (4, 12))


def check_lengths_and_offsets(dev, kind, x, bigendian=0, with_ref=True, lengths=range(1, 41)):
    """lengths 1..40 (the build's vector body and scalar epilogue) at aligned and unaligned buffer offsets"""
    item = KINDS[kind][0]
    values = np.ascontiguousarray(x).view(np.uint8).reshape(-1)
    for n in lengths:
        part = values[:n * item]
        src = part.view(F) if item == 4 else part
        want = ref_call(kind, src, bigendian) if with_ref else restate(kind, src, bigendian)
        assert same(want, restate(kind, src, bigendian)), (kind, n)
        for in_off, out_off in offsets_for(kind):
            assert same(as_output(kind, run(dev, kind, src, bigendian, in_off, out_off)), want), (kind, n, in_off, out_off, bigendian)


def refusals(dev):
    """null pointers, a float buffer off its 4-byte alignment and n < 0 give -1 and launch nothing; n = 0 gives 0 and launches nothing"""
    L = dev.L
    b_in, b_out = dev.buffer(b"", 256), dev.buffer(bytes([SENTINEL]) * 256, 256)
    pi, po = dev.ptr(b_in), dev.ptr(b_out)
    before = L.csdrb_kernel_launches()
    bad = []
    for kind in KINDS:
        misaligned_float = (pi + 2, po, 8) if KINDS[kind][0] == 4 else (pi, po + 2, 8)      # a float buffer off its 4-byte alignment
        for args, want in (((None, po, 8), -1), ((pi, None, 8), -1), ((None, None, 0), -1), ((pi, po, -1), -1), ((pi, po, 0), 0),
                           (misaligned_float, -1)):
            for be in ((0, 1) if KINDS[kind][2] else (0,)):
                if abi(L, kind, *args, be, dev.stream) != want:
                    bad.append((kind, args, be))
    if L.csdrb_kernel_launches() != before:
        bad.append(("launched", L.csdrb_kernel_launches() - before))
    if not np.all(dev.read(b_out) == SENTINEL):
        bad.append("output written")
    return bad
