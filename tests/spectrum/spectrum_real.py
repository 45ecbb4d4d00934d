"""Checker for the real-input FFT and waterfall bank (csdrb_fft_r2c_batch, csdrb_spectrum_bank_f; csdr_b200/csrc/fft_real.cuh, spectrum.cu).
TEST INFRASTRUCTURE, the real-input twin of spectrum.py (whose Params, State and Devs it uses).

The bank's contract is `fft_fc N E W | logaveragepower_cf X N A [| compress_fft_adpcm_f_u8 N]` on every row, and its claim is byte identity with
    apply_precalculated_window_f -> csdrb_fft_r2c_batch (2N points) -> csdrb_accumulate_power_cf (bins 0..N-1, A frames) -> csdrb_log_ff
    [-> csdrb_compress_fft_adpcm_rows_f_u8]
with the frames cut out of the stream here by fft_fc's framing: frame k is [(k+1)E - 2N, (k+1)E) for E <= 2N and starts at k(2E - 2N) for E > 2N
(the reference skips E - 2N complex samples after each frame).

The float64 bound of the r2c transform (rfft_bound).  The packed M = N/2-point c2c of z[n] = x[2n] + i x[2n+1] is within
e_Z = (5 log2 M + 7) u sum|z| of the exact DFT (tests/test_fft_large_emulated.py: the four-step transform, whose bound also covers the single-CTA
passes of spectrum.py's 5 log2 M + 1), and sum|z| <= sum|x|.  The split X[k] = (Z[k] + conj Z[M-k])/2 - i W^k (Z[k] - conj Z[M-k])/2 takes two
such errors through each half (<= e_Z each), rounds the halves once (u |Z| each), multiplies by a table entry within u of W^k (a product rounded
twice and an FMA: 3u |Z|) and rounds the final sum (u |X| <= 2u sum|x|).  |Z| <= sum|x|, so to first order
    |X^_k - X_k| <= (2 (5 log2 M + 7) + 8) u sum|x| = (10 log2 N + 12) u sum|x|,
N the real points, sum over the (windowed) inputs of the transform."""
from __future__ import annotations

import ctypes as C

import numpy as np

import spectrum as S

U = 2.0 ** -24


def setup(L):
    S.setup(L)
    vp, lg, it, sz = C.c_void_p, C.c_long, C.c_int, C.c_size_t
    L.csdrb_fft_r2c_batch.argtypes = [vp, lg, vp, lg, it, it, vp]
    L.csdrb_spectrum_bank_lines_f.argtypes = [C.POINTER(S.Params), C.POINTER(S.State), lg]; L.csdrb_spectrum_bank_lines_f.restype = lg
    L.csdrb_spectrum_bank_scratch_bytes_f.argtypes = [it, lg, C.POINTER(S.Params)]; L.csdrb_spectrum_bank_scratch_bytes_f.restype = sz
    L.csdrb_spectrum_bank_f.argtypes = [vp, lg, it, lg, vp, C.POINTER(S.Params), vp, vp, C.POINTER(S.State), vp, lg, vp, sz, vp]
    L.apply_precalculated_window_f.argtypes = [vp, vp, it, vp]
    L.make_fft_r2c.argtypes = [it, vp, vp, it]; L.make_fft_r2c.restype = vp
    L.fft_execute.argtypes = [vp]; L.fft_destroy.argtypes = [vp]
    return L


def rfft_bound(x):
    """per-bin bound of the r2c transform of the float32 rows x [B, n] (derived above)"""
    n = x.shape[-1]
    return (10 * np.log2(n) + 12) * U * np.abs(x.astype(np.float64)).sum(axis=-1, keepdims=True)


def r2c(dev, x, in_pad=0, out_pad=0, in_offset=0):
    """csdrb_fft_r2c_batch of the float32 rows x [B, n]: [B, n/2 + 1] complex64 (rows at in_stride n + in_pad floats, starting in_offset floats in)"""
    B, n = x.shape
    ist, ost = n + in_pad, n // 2 + 1 + out_pad
    xs = np.zeros(B * ist + in_offset, np.float32)
    for b in range(B):
        xs[in_offset + b * ist:in_offset + b * ist + n] = x[b]
    d_x = dev.put(xs); d_y = dev.alloc(8 * B * ost)
    rc = dev.L.csdrb_fft_r2c_batch(dev.ptr(d_x) + 4 * in_offset, ist, dev.ptr(d_y), ost, n, B, dev.stream)
    assert rc == 0, (rc, dev.L.csdrb_last_error())
    return dev.get(d_y, np.complex64).reshape(B, ost)[:, :n // 2 + 1]


# ---- framing ------------------------------------------------------------------------------------------------------------------------------
def frames_at(N, E, total):
    L = 2 * N
    return total // E if E <= L else ((total - L) // (2 * E - L) + 1 if total >= L else 0)


def frame_start(N, E, k):
    return (k + 1) * E - 2 * N if E <= 2 * N else k * (2 * E - 2 * N)


def frames_bruteforce(N, E, total):
    """fft_fc's loop (csdr.c:3459-3497) counting the frames whose samples all arrived: the E > 2N branch reads 2N floats, then skips E - 2N
    complex samples, i.e. 2(E - 2N) floats"""
    L = 2 * N
    if E > L:
        k, pos = 0, 0
        while pos + L <= total:
            k += 1; pos += L + 2 * (E - L)
        return k
    k, have = 0, 0
    while have + E <= total:
        have += E; k += 1
    return k


def stream_for(N, E, frames):
    """samples that complete exactly `frames` frames"""
    return frames * E if E <= 2 * N else (frames - 1) * (2 * E - 2 * N) + 2 * N


def cut_frames(x, N, E, nframes):
    """[nframes, 2N] frames of one real row, zeros before the stream"""
    L = 2 * N
    out = np.zeros((nframes, L), np.float32)
    for k in range(nframes):
        s = frame_start(N, E, k)
        lo = max(s, 0)
        out[k, lo - s:] = x[lo:s + L]
    return out


# ---- the two sides ------------------------------------------------------------------------------------------------------------------------
def window_frames(dev, fr, win):
    """apply_precalculated_window_f (the library's host function) on every frame"""
    out = np.empty_like(fr)
    for k in range(fr.shape[0]):
        a = np.ascontiguousarray(fr[k]); o = np.empty_like(a)
        dev.L.apply_precalculated_window_f(a.ctypes.data, o.ctypes.data, a.size, win.ctypes.data)
        out[k] = o
    return out


def composition(dev, x, p, win):
    """the existing per-block calls on the whole stream: [rows, lines, line_bytes] uint8"""
    L, N, A = dev.L, p.fft_size, p.averages
    rows, T = x.shape
    nf = frames_at(N, p.every, T)
    nl = nf // A
    add = np.float32(np.float64(np.float32(p.add_db)) - 10.0 * np.log10(float(A)))
    lb = S.line_bytes(p)
    win = np.ascontiguousarray(win, np.float32)
    out = []
    for r in range(rows):
        if nl == 0:
            out.append(np.zeros((0, lb), np.uint8)); continue
        fr = window_frames(dev, cut_frames(x[r], N, p.every, nl * A), win)
        d_fr = dev.put(fr); d_s = dev.alloc(8 * (N + 1) * nl * A)
        assert L.csdrb_fft_r2c_batch(dev.ptr(d_fr), 2 * N, dev.ptr(d_s), N + 1, 2 * N, nl * A, dev.stream) >= 0, L.csdrb_last_error()
        db = dev.alloc(4 * N * nl)
        for j in range(nl):
            acc = dev.alloc(4 * N)
            for f in range(A):
                assert L.csdrb_accumulate_power_cf(dev.ptr(d_s) + 8 * (N + 1) * (j * A + f), dev.ptr(acc), N, dev.stream) >= 0
            assert L.csdrb_log_ff(dev.ptr(acc), dev.ptr(db) + 4 * N * j, N, float(add), dev.stream) >= 0
        lines = dev.get(db, np.float32).reshape(nl, N)
        if p.compress:
            d_l = dev.put(np.ascontiguousarray(lines)); d_b = dev.alloc(nl * lb)
            assert L.csdrb_compress_fft_adpcm_rows_f_u8(dev.ptr(d_l), N, dev.ptr(d_b), lb, nl, N, dev.stream) >= 0
            out.append(dev.get(d_b, np.uint8).reshape(nl, lb))
        else:
            out.append(np.ascontiguousarray(lines).view(np.uint8))
    return np.stack(out)


def bank(dev, x, p, win, cuts=None, scratch="full", pad=0, out_pad=0, offset=1):
    """the real bank over the stream cut at `cuts` (default one call): [rows, lines, line_bytes] uint8.  The rows start `offset` floats into their
    buffer (an odd offset: no frame load may assume 8-byte alignment)."""
    L, N = dev.L, p.fft_size
    rows, T = x.shape
    stride = T + pad
    xs = np.zeros(rows * stride + offset, np.float32)
    for r in range(rows):
        xs[offset + r * stride:offset + r * stride + T] = x[r]
    d_x = dev.put(xs); d_w = dev.put(np.ascontiguousarray(win, np.float32))
    hist = dev.alloc(4 * rows * 2 * N); acc = dev.alloc(4 * rows * N)
    st = S.State(0, 0)
    lb = S.line_bytes(p)
    total = L.csdrb_spectrum_bank_lines_f(C.byref(p), C.byref(st), T)
    got = [bytearray() for _ in range(rows)]
    bounds = [0] + sorted(cuts or []) + [T]
    for a, b in zip(bounds[:-1], bounds[1:]):
        n = b - a
        nl = L.csdrb_spectrum_bank_lines_f(C.byref(p), C.byref(st), n)
        ostride = nl * lb + out_pad
        d_o = dev.alloc(max(rows * ostride, 4))
        sb = L.csdrb_spectrum_bank_scratch_bytes_f(rows, n if scratch == "full" else 1, C.byref(p))
        d_s = dev.alloc(sb)
        rc = L.csdrb_spectrum_bank_f(dev.ptr(d_x) + 4 * (offset + a), stride, rows, n, dev.ptr(d_w), C.byref(p), dev.ptr(hist), dev.ptr(acc), C.byref(st),
                                     dev.ptr(d_o), ostride, dev.ptr(d_s), sb, dev.stream)
        assert rc == nl, (rc, nl, L.csdrb_last_error())
        o = dev.get(d_o, np.uint8)
        for r in range(rows):
            got[r] += o[r * ostride:r * ostride + nl * lb].tobytes()
    assert st.consumed == T and st.frames == frames_at(N, p.every, T)
    return np.stack([np.frombuffer(bytes(g), np.uint8).reshape(total, lb) for g in got])
