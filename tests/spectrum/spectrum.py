"""Checker for the waterfall bank csdrb_spectrum_bank_cf (csdr_b200/csrc/spectrum.cu).  TEST INFRASTRUCTURE.

The bank's contract is `fft_cc N E W | logaveragepower_cf X N A | fft_exchange_sides_ff N [| compress_fft_adpcm_f_u8 N]` on every row, and its
claim is byte identity with the composition of the existing per-block calls on the same stream:
    csdrb_apply_window_rows_c -> csdrb_fft_c2c_batch -> csdrb_accumulate_power_cf (A frames) -> csdrb_log_ff -> halves swapped
    [-> csdrb_compress_fft_adpcm_rows_f_u8]
with the frames cut out of the stream here, on the host, by fft_cc's framing.  Both sides run through a `Dev`: the emulated library
(tests/host_shim, numpy buffers as device memory) or the real one on a GPU (torch CUDA tensors), so the CPU and GPU tiers run the same bodies.

The float64 bound (power_bound).  For a windowed frame y (float32 values, exact) the N-point FFT is a tree of log2(N) radix-2-equivalent
levels.  On a path from input i to bin k every level costs at most one rounded complex addition (|rel err| <= u per component) and a twiddle
multiply whose table entry is within 2 ulp and whose product rounds twice (<= 4u per level), so |X^_k - X_k| <= e_k = (5 log2 N + 1) u sum|y_i|
(u = 2^-24, first-order).  The power p = x^2 + y^2 then has |p^ - p| <= 2|X| e + e^2 + 3u p^ (two products and a sum rounded), and a sum of A
powers in frame order adds A u sum(p) more.  The dB value 10 log10(p) + c is rounded after the double log10: 4.343 |dp|/p plus 2 ulp of the
result."""
from __future__ import annotations

import ctypes as C
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent.parent
sys.path.insert(0, str(ROOT))
U = 2.0 ** -24


class Params(C.Structure):
    _fields_ = [("fft_size", C.c_int), ("every", C.c_int), ("averages", C.c_int), ("compress", C.c_int), ("add_db", C.c_float)]


class State(C.Structure):
    _fields_ = [("consumed", C.c_longlong), ("frames", C.c_longlong)]


def setup(L):
    vp, lg, it, sz = C.c_void_p, C.c_long, C.c_int, C.c_size_t
    L.csdrb_last_error.restype = C.c_char_p
    L.csdrb_spectrum_bank_lines.argtypes = [C.POINTER(Params), C.POINTER(State), lg]; L.csdrb_spectrum_bank_lines.restype = lg
    L.csdrb_spectrum_bank_scratch_bytes.argtypes = [it, lg, C.POINTER(Params)]; L.csdrb_spectrum_bank_scratch_bytes.restype = sz
    L.csdrb_spectrum_bank_cf.argtypes = [vp, lg, it, lg, vp, C.POINTER(Params), vp, vp, C.POINTER(State), vp, lg, vp, sz, vp]
    L.csdrb_apply_window_rows_c.argtypes = [vp, vp, vp, it, lg, vp]
    L.csdrb_fft_c2c_batch.argtypes = [vp, lg, vp, lg, it, it, it, vp]
    L.csdrb_accumulate_power_cf.argtypes = [vp, vp, lg, vp]
    L.csdrb_log_ff.argtypes = [vp, vp, lg, C.c_float, vp]
    L.csdrb_logpower_cf.argtypes = [vp, vp, lg, C.c_float, vp]
    L.csdrb_compress_fft_adpcm_rows_f_u8.argtypes = [vp, lg, vp, lg, it, it, vp]
    L.precalculate_window.argtypes = [it, it]; L.precalculate_window.restype = C.POINTER(C.c_float)
    return L


WINDOWS = {"BOXCAR": 0, "BLACKMAN": 1, "HAMMING": 2}


def window(L, n, name="HAMMING"):
    return np.ctypeslib.as_array(L.precalculate_window(n, WINDOWS[name]), shape=(n,)).copy()


class EmulDev:
    """the emulated library: device memory is host memory"""
    def __init__(self, L):
        self.L = setup(L); self.stream = None

    def alloc(self, nbytes):
        raw = np.zeros(nbytes + 64, np.uint8)
        off = (-raw.ctypes.data) % 64
        return raw[off:off + nbytes]

    def put(self, a):
        b = self.alloc(a.nbytes); b[:] = np.ascontiguousarray(a).view(np.uint8).reshape(-1); return b

    def get(self, buf, dtype):
        return np.array(buf).view(dtype)

    def ptr(self, buf):
        return buf.ctypes.data

    def sync(self):
        pass


class CudaDev:
    """the real library on the current CUDA device, torch tensors as buffers"""
    def __init__(self):
        import torch
        import csdr_b200
        self.torch = torch
        csdr_b200.lib()
        self.L = setup(C.CDLL(str(csdr_b200.LIB_PATH)))                # a handle of its own: the package's keeps its own argtypes
        self.stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def alloc(self, nbytes):
        return self.torch.zeros(max(nbytes, 1), dtype=self.torch.uint8, device="cuda")

    def put(self, a):
        return self.torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()

    def get(self, buf, dtype):
        self.torch.cuda.synchronize()
        return buf.cpu().numpy().view(dtype)

    def ptr(self, buf):
        return buf.data_ptr()

    def sync(self):
        self.torch.cuda.synchronize()


# ---- framing ------------------------------------------------------------------------------------------------------------------------------
def frames_at(N, E, total):
    return total // E if E <= N else ((total - N) // E + 1 if total >= N else 0)


def frames_bruteforce(N, E, total):
    """fft_cc's loop (host/csdr_cli.c cmd_fft_cc) counting the frames whose samples all arrived"""
    if E > N:
        k, pos = 0, 0
        while pos + N <= total:
            k += 1; pos += E
        return k
    k, have = 0, 0
    while have + E <= total:
        have += E; k += 1
    return k


def frame_start(N, E, k):
    return (k + 1) * E - N if E <= N else k * E


def stream_for(N, E, frames):
    """samples that complete exactly `frames` frames"""
    return frames * E if E <= N else (frames - 1) * E + N


def cut_frames(x, N, E, nframes):
    """[nframes, N] frames of one row, zeros before the stream"""
    out = np.zeros((nframes, N), np.complex64)
    for k in range(nframes):
        s = frame_start(N, E, k)
        lo = max(s, 0)
        out[k, lo - s:] = x[lo:s + N]
    return out


def line_bytes(p):
    return (p.fft_size + 10) // 2 if p.compress else 4 * p.fft_size


# ---- the two sides ------------------------------------------------------------------------------------------------------------------------
def composition(dev, x, p, win):
    """the existing per-block calls on the whole stream: [rows, lines, line_bytes] uint8"""
    L, N, A = dev.L, p.fft_size, p.averages
    rows, T = x.shape
    nf = frames_at(N, p.every, T)
    nl = nf // A
    add = np.float32(np.float64(np.float32(p.add_db)) - 10.0 * np.log10(float(A)))
    out = []
    w = dev.put(win)
    for r in range(rows):
        fr = cut_frames(x[r], N, p.every, nl * A)
        if nl == 0:
            out.append(np.zeros((0, line_bytes(p)), np.uint8)); continue
        d_fr = dev.put(fr); d_w = dev.alloc(fr.nbytes); d_s = dev.alloc(fr.nbytes)
        assert L.csdrb_apply_window_rows_c(dev.ptr(d_fr), dev.ptr(d_w), dev.ptr(w), N, nl * A, dev.stream) >= 0
        assert L.csdrb_fft_c2c_batch(dev.ptr(d_w), N, dev.ptr(d_s), N, N, nl * A, 0, dev.stream) >= 0, L.csdrb_last_error()
        db = dev.alloc(4 * N * nl)
        for j in range(nl):
            acc = dev.alloc(4 * N)
            for f in range(A):
                assert L.csdrb_accumulate_power_cf(dev.ptr(d_s) + 8 * N * (j * A + f), dev.ptr(acc), N, dev.stream) >= 0
            assert L.csdrb_log_ff(dev.ptr(acc), dev.ptr(db) + 4 * N * j, N, float(add), dev.stream) >= 0
        lines = dev.get(db, np.float32).reshape(nl, N)
        lines = np.concatenate([lines[:, N // 2:], lines[:, :N // 2]], axis=1)          # fft_exchange_sides_ff
        if p.compress:
            d_l = dev.put(np.ascontiguousarray(lines)); d_b = dev.alloc(nl * line_bytes(p))
            assert L.csdrb_compress_fft_adpcm_rows_f_u8(dev.ptr(d_l), N, dev.ptr(d_b), line_bytes(p), nl, N, dev.stream) >= 0
            out.append(dev.get(d_b, np.uint8).reshape(nl, line_bytes(p)))
        else:
            out.append(np.ascontiguousarray(lines).view(np.uint8))
    return np.stack(out)


def bank(dev, x, p, win, cuts=None, scratch="full", pad=0, out_pad=0):
    """the bank over the stream cut at `cuts` (sample positions, default one call): [rows, lines, line_bytes] uint8, and the launches' rc list"""
    L, N = dev.L, p.fft_size
    rows, T = x.shape
    stride = T + pad
    xs = np.zeros((rows, stride), np.complex64); xs[:, :T] = x
    d_x = dev.put(xs); d_w = dev.put(win)
    hist = dev.alloc(8 * rows * N); acc = dev.alloc(4 * rows * N)
    st = State(0, 0)
    lb = line_bytes(p)
    total = L.csdrb_spectrum_bank_lines(C.byref(p), C.byref(st), T)
    got = [bytearray() for _ in range(rows)]
    bounds = [0] + sorted(cuts or []) + [T]
    for a, b in zip(bounds[:-1], bounds[1:]):
        n = b - a
        nl = L.csdrb_spectrum_bank_lines(C.byref(p), C.byref(st), n)
        ostride = nl * lb + out_pad
        d_o = dev.alloc(max(rows * ostride, 4))
        sb = L.csdrb_spectrum_bank_scratch_bytes(rows, n, C.byref(p)) if scratch == "full" else L.csdrb_spectrum_bank_scratch_bytes(rows, 1, C.byref(p))
        d_s = dev.alloc(sb)
        rc = L.csdrb_spectrum_bank_cf(dev.ptr(d_x) + 8 * a, stride, rows, n, dev.ptr(d_w), C.byref(p), dev.ptr(hist), dev.ptr(acc), C.byref(st),
                                      dev.ptr(d_o), ostride, dev.ptr(d_s), sb, dev.stream)
        assert rc == nl, (rc, nl, L.csdrb_last_error())
        o = dev.get(d_o, np.uint8)
        for r in range(rows):
            got[r] += o[r * ostride:r * ostride + nl * lb].tobytes()
    assert st.consumed == T and st.frames == frames_at(N, p.every, T)
    return np.stack([np.frombuffer(bytes(g), np.uint8).reshape(total, lb) for g in got])


# ---- the float64 bound -----------------------------------------------------------------------------------------------------------------
def check_power_bound(db_lines, x, p, win):
    """dB lines (float output) of one row against numpy's float64 DFT of the windowed float32 frames, within the bound derived above"""
    N, A = p.fft_size, p.averages
    nl = db_lines.shape[0]
    fr = cut_frames(x, N, p.every, nl * A)
    y = (fr.real.astype(np.float32) * win).astype(np.float64) + 1j * (fr.imag.astype(np.float32) * win).astype(np.float64)
    X = np.fft.fft(y, axis=1)
    P = np.abs(X) ** 2
    e = (5 * np.log2(N) + 1) * U * np.abs(y).sum(axis=1, keepdims=True) * np.sqrt(2)
    dP = 2 * np.abs(X) * e + e ** 2 + 3 * U * P
    add = np.float64(np.float32(np.float64(np.float32(p.add_db)) - 10.0 * np.log10(float(A))))
    checked = 0
    for j in range(nl):
        s = P[j * A:(j + 1) * A].sum(axis=0)
        ds = dP[j * A:(j + 1) * A].sum(axis=0) + A * U * s
        want = 10 * np.log10(np.maximum(s, 1e-300)) + add
        got = db_lines[j].astype(np.float64)
        got = np.concatenate([got[N // 2:], got[:N // 2]])                              # back to bin order
        ok = ds < 0.5 * s
        tol = 4.343 * ds / np.maximum(s - ds, 1e-300) + 2 * np.abs(want) * 2.0 ** -23 + 1e-12
        assert np.all(np.abs(got - want)[ok] <= tol[ok]), (j, np.max((np.abs(got - want) - tol)[ok]))
        checked += int(ok.sum())
    return checked
