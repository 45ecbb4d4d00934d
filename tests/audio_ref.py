"""References, error bounds, case matrix and checks of the FM chain's audio-rate kernels, shared by tests/test_audio_tail_emulated.py (CPU tier,
the emulated library) and tests/test_gpu_audio_tail.py (-m gpu):

    fmdemod_quadri_bank_kernel (csrc/elementwise.cu)        fmdemod_quadri_cf
    fracdec_segments_kernel + fracdec_interp_seg_kernel<12|0>,
    fracdec_positions_kernel + fracdec_interp_kernel (audio.cu)  fractional_decimator_ff
    fastagc_fused_kernel<S16>, fastagc_peaks/apply<S16>/carry   fastagc_ff [| convert_f_s16]
    nfm_deemph_bank_kernel<LIMIT> (fir_valid bank)              [limit_ff |] deemphasis_nfm_ff
    deemphasis_wfm_bank_kernel                                  deemphasis_wfm_ff

Each kernel is held to (1) bits: equal to a restatement of its documented operation order (numpy float32 for fmdemod and the Lagrange sum, the
strict C oracle for fracdec, fastagc and deemphasis_wfm), or, where the order is free (the FIR), to exact invariants; (2) a per-output bound
against the float64 operation on the exact float32 inputs; (3) windows and refusals: a NaN or Inf reaches only the outputs the reference says,
nothing is written outside the outputs, and every refusal returns its code without a launch.  u = 2^-24; gamma_k = k u / (1 - k u); every
bound below carries a factor (1 + 1e-3) for the second-order terms and the float64 reference's own rounding (<= 2^-50 relative).

fmdemod.  dq = fl(Q - Q'), di = fl(I - I') err by u relative; the products I dq, Q di by one more u each, the difference once more.  With
S = |I DQ| + |Q DI| (exact differences) the numerator errs by <= 3u S (cancellation in num is bounded by its terms, not by |num|).  The
denominator I^2 + Q^2 (positive terms) errs by <= 2u relative, K num / den runs in double and rounds once to float (u).  So
    |y - R| <= 3u (1 + 1e-3) (K S / DEN + |R|),       R = K (I DQ - Q DI) / (I^2 + Q^2) in float64.

fracdec.  Output o is the Lagrange polynomial through m points at xw = fl(where_o - low), where_o being the float chain's position (so the
reference is evaluated at the kernel's own positions).  Each weight coef_i / den_i has m - 1 rounded subtractions and m - 2 products in coef,
m - 2 products in den (integer products above 2^24 round) and a division: <= (3m - 4) u relative; times the point (+u), summed in a chain of
m adds (gamma_m); a prefilter point is a chain of T products and adds (gamma_T of sum |x h|).  So
    |y - R| <= (4m - 3 + T) u (1 + 1e-3) sum_i |L_i(xw)| A_i,   A_i = |x_(low+i)|, or sum_t |x_(low+i+t) h_t| with a prefilter.

fastagc.  target = fl(ref / peak) and the carried gain err by u relative, r = fl(i / block) by u, fl(target r) by u, the double ramp rounds
once to float, the product with the sample once more.  With G = LG (1 - r) + TG r from float64 gains LG, TG (capped at 50):
    |y - x G| <= u (1 + 1e-3) |x| (LG + 3 TG r + 2 G).

fir_valid.  One chain of T fused multiply-adds per output (t ascending), whatever the tile: |y - sum h x| <= gamma_T sum |h x|.

deemphasis_wfm.  y_k = fl(fl(a x_k) + fl(k y_(k-1))) with the float coefficients a, k: the local error is <= 2u (|a x_k| + k |y_(k-1)|) and
earlier errors decay by k, so E_k = k E_(k-1) + 2u (1 + 1e-3) (|a x_k| + k (|Y_(k-1)| + E_(k-1))) bounds |y_k - Y_k| for the float64
recursion Y with the same coefficients.

The checks talk to the C ABI through a driver with dev(array) -> buffer, ptr(buffer), host(buffer) -> array, `L` (argtypes set by
csdr_b200.lib()) and `stream`, so the same bodies run on the GPU and on the emulated library.
"""
import ctypes as C
import math

import numpy as np

from bitcmp import SENTINEL, U, assert_bits_equal, bits  # noqa: F401

F32 = np.float32
MARGIN = 1 + 1e-3
FMDEMOD_K = 0.340447550238101026565118445432744920253753662109375
NFM_MAX_TAPS = 208                                                   # kNfmMaxTaps
FD_MAX_SEGS = 96
AGC_RUN = 16
STATE_DT = np.dtype([("where", "<f4"), ("input_processed", "<i4"), ("output_size", "<i4")])
SEG_DT = np.dtype([("k0", "<i4"), ("M", "<u4"), ("q", "<u4"), ("E", "<i4"), ("cnt", "<i4")])        # FdSeg: the segment table in the scratch


def launches(drv):
    return int(drv.L.csdrb_kernel_launches())


def same(a, b, what):
    """bit equality where both are numbers, NaN where either is NaN (the NaN payload is the platform's)"""
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    na, nb = np.isnan(a), np.isnan(b)
    if not np.array_equal(na, nb):
        i = np.flatnonzero((na != nb).reshape(-1))
        raise AssertionError(f"{what}: NaN at different outputs, first at {i[0]} ({i.size} outputs)")
    assert_bits_equal(np.where(na, 0, a).astype(a.dtype), np.where(nb, 0, b).astype(b.dtype), what)


def within(got, want, bnd, what):
    """every finite output within its bound; returns the worst err/bound ratio"""
    err = np.abs(got.astype(np.float64) - want)
    ok = err <= bnd
    if not np.all(ok):
        i = np.argwhere(~ok)[0]
        raise AssertionError(f"{what}: output {tuple(i)} errs by {err[tuple(i)]:.3e}, bound {bnd[tuple(i)]:.3e} ({np.count_nonzero(~ok)} outside)")
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.where(bnd > 0, err / np.where(bnd > 0, bnd, 1), 0.0)
    return float(r.max()) if r.size else 0.0


def rows_in(a, stride, col0=0, fill=np.nan):
    """rows of a [ch, n] placed at column col0 of rows of `stride` elements whose other entries hold `fill`"""
    ch, n = a.shape
    buf = np.full((ch, stride), fill, a.dtype)
    buf[:, col0:col0 + n] = a
    return buf


def sentinel_rows(rows, stride, dtype):
    w = {np.dtype(np.float32): np.uint32, np.dtype(np.int16): np.uint16}[np.dtype(dtype)]
    fill = SENTINEL if w is np.uint32 else np.uint16(0xDEAD)
    return np.full((rows, stride), fill, w).view(dtype)


def untouched(buf, mask, what):
    """entries of buf outside `mask` (True = an output) still hold the sentinel"""
    w = buf.view(np.uint32 if buf.dtype.itemsize == 4 else np.uint16)
    s = SENTINEL if buf.dtype.itemsize == 4 else np.uint16(0xDEAD)
    assert np.all(w[~mask] == s), f"{what}: a store outside the outputs"


# =============================================================================================================================== fmdemod
FM_LAYOUTS = ["pad", "view", "oddstride"]


def fm_layout(n, layout):
    """(row stride, first column) in complex samples: "pad" = 16-byte rows (vector path), "view" = rows one sample in (every row 8-byte aligned:
    scalar path), "oddstride" = an odd stride (rows alternate between the two paths)"""
    return {"pad": (n + (n & 1) + 2, 0), "view": (n + (n & 1) + 4, 1), "oddstride": (n + 1 + (n & 1), 0)}[layout]


def fm_path(addr, n):
    """launch_fmdemod_quadri_bank / the kernel's choice for a row at byte address addr: (path, odd tail by one thread, grid-stride loop)"""
    gx = min(64, max(1, (n // 2 + 255) // 256))
    if addr % 16 == 0:
        return "vector", n % 2 == 1, n // 2 > gx * 256
    return "scalar", False, n > gx * 256


def fmdemod_np(x, last):
    """the kernel's order in numpy float32 (no contraction) with the double K*num/den tail: x [ch, n] complex64, last [ch] complex64"""
    prev = np.concatenate([last[:, None], x[:, :-1]], axis=1)
    I, Q, pI, pQ = x.real, x.imag, prev.real, prev.imag
    with np.errstate(all="ignore"):
        dq, di = Q - pQ, I - pI
        num = I * dq - Q * di
        den = I * I + Q * Q
        y = (FMDEMOD_K * num.astype(np.float64) / den.astype(np.float64)).astype(F32)
    return np.where(den != 0, y, F32(0))


def fmdemod64(x, last):
    """(float64 discriminator on the exact inputs, per-output bound)"""
    prev = np.concatenate([last[:, None], x[:, :-1]], axis=1).astype(np.complex128)
    X = x.astype(np.complex128)
    I, Q, pI, pQ = X.real, X.imag, prev.real, prev.imag
    DQ, DI = Q - pQ, I - pI
    den = I * I + Q * Q
    with np.errstate(all="ignore"):
        R = np.where(den > 0, FMDEMOD_K * (I * DQ - Q * DI) / np.where(den > 0, den, 1), 0.0)
        S = np.where(den > 0, FMDEMOD_K * (np.abs(I * DQ) + np.abs(Q * DI)) / np.where(den > 0, den, 1), 0.0)
    return R, 3 * U * MARGIN * (S + np.abs(R))


def fm_bank(drv, x, last, layout="pad", expect_paths=None):
    """csdrb_fmdemod_quadri_bank_cf on x [ch, n] -> (y [ch, n], carried sample [ch]); outputs land in [ch + 1, n + 4] sentinel rows"""
    ch, n = x.shape
    stride, col0 = fm_layout(n, layout)
    xb = rows_in(x, stride, col0, np.complex64(complex(np.nan, np.nan)))
    ostride = n + (n & 1) + 4
    ob = sentinel_rows(ch + 1, ostride, np.float32)
    dx, do, dl = drv.dev(xb), drv.dev(ob), drv.dev(np.ascontiguousarray(last, np.complex64))
    dlo = drv.dev(sentinel_rows(1, 2 * (ch + 1), np.float32).view(np.complex64)[0])
    base = drv.ptr(dx) + 8 * col0
    if expect_paths is not None:
        expect_paths.update(fm_path(base + 8 * stride * c, n) for c in range(ch))
    rc = drv.L.csdrb_fmdemod_quadri_bank_cf(base, stride, drv.ptr(do), ostride, ch, n, drv.ptr(dl), drv.ptr(dlo), drv.stream)
    assert rc == 0, drv.L.csdrb_last_error()
    got, lo = drv.host(do), drv.host(dlo)
    mask = np.zeros(got.shape, bool); mask[:ch, :n] = True
    untouched(got, mask, f"fmdemod {layout} n={n}")
    assert np.all(lo.view(np.uint32)[2 * ch:] == SENTINEL), "carry stored past the last channel"
    return np.ascontiguousarray(got[:ch, :n]), lo[:ch]


FM_N = [1, 2, 3, 511, 512, 513, 4097]
FM_BIG = 40_001                                                       # > 32768: the 64-CTA grid loops


def fm_inputs(ch, n, seed):
    rng = np.random.default_rng(seed)
    x = (rng.uniform(-1, 1, (ch, n)) + 1j * rng.uniform(-1, 1, (ch, n))).astype(np.complex64)
    last = (rng.uniform(-1, 1, ch) + 1j * rng.uniform(-1, 1, ch)).astype(np.complex64)
    if n >= 8:
        x[0, 3] = 0                                                   # den == 0: the output is 0
        x[0, 5] = x[0, 4]                                             # a repeated sample: num == 0
        x[-1, n // 2] = np.complex64(1e-30 + 1e-30j)                   # den underflows to 0 in float: the output is 0
    return x, last


def check_fmdemod(drv, ch, n, layout, seed=0, paths=None):
    """bits of the numpy restatement, the float64 bound, the carried sample, and the same bits streamed in three calls"""
    x, last = fm_inputs(ch, n, seed)
    y, lo = fm_bank(drv, x, last, layout, paths)
    same(y, fmdemod_np(x, last), f"fmdemod ch={ch} n={n} {layout}: restatement")
    assert_bits_equal(lo, x[:, -1], "carried sample")
    R, B = fmdemod64(x, last)
    normal = (x.real * x.real + x.imag * x.imag) >= F32(2.0 ** -126)   # the bound's relative steps need a normal denominator; den == 0 -> 0 above
    worst = within(y[normal], R[normal], B[normal], f"fmdemod ch={ch} n={n} {layout}: float64 bound")
    if n >= 3:
        cuts = sorted({1, n // 2 | 1, n - 1})
        parts, carry = [], last
        for a, b in zip([0] + cuts, cuts + [n]):
            if b > a:
                yy, carry = fm_bank(drv, np.ascontiguousarray(x[:, a:b]), carry, layout)
                parts.append(yy)
        assert_bits_equal(np.concatenate(parts, axis=1), y, f"fmdemod n={n} {layout}: cut into calls")
    return worst


def check_fmdemod_nonfinite(drv, n, layout, seed=0):
    """NaN, +Inf, -Inf in I or Q at sample p make outputs p and p + 1 non-finite (p + 1 reads it as the previous sample) and change nothing else"""
    ch = 3
    x, last = fm_inputs(ch, n, seed)
    clean, _ = fm_bank(drv, x, last, layout)
    pos = sorted({0, 1, n // 2, n // 2 + 1, n - 2, n - 1})
    bad = np.array([np.nan, np.inf, -np.inf], np.float32)
    xp = x.copy()
    for c in range(ch):
        for i, p in enumerate(pos):
            v = bad[(c + i) % 3]
            xp[c, p] = complex(v, 0.5) if i % 2 else complex(0.25, v)
    got, _ = fm_bank(drv, xp, last, layout)
    same(got, fmdemod_np(xp, last), f"fmdemod n={n} {layout} non-finite: restatement")
    hit = np.zeros(n, bool)
    for p in pos:
        hit[p] = True
        if p + 1 < n:
            hit[p + 1] = True
    for c in range(ch):
        assert np.array_equal(~np.isfinite(got[c]), hit), (c, np.flatnonzero(~np.isfinite(got[c]))[:10], np.flatnonzero(hit)[:10])
        assert_bits_equal(got[c][~hit], clean[c][~hit], f"fmdemod channel {c}: outputs away from the poisoned samples")


def check_fmdemod_refusals(drv):
    x, last = fm_inputs(2, 64, 1)
    dx, dl = drv.dev(x), drv.dev(last)
    ob = sentinel_rows(3, 68, np.float32)
    do = drv.dev(ob)
    n0 = launches(drv)
    L = drv.L
    assert L.csdrb_fmdemod_quadri_bank_cf(drv.ptr(dx), 64, drv.ptr(do) + 4, 68, 2, 64, None, None, drv.stream) == -1      # output 4-byte aligned
    assert L.csdrb_fmdemod_quadri_bank_cf(drv.ptr(dx), 64, drv.ptr(do), 67, 2, 64, None, None, drv.stream) == -1          # odd output stride
    assert L.csdrb_fmdemod_quadri_bank_cf(drv.ptr(dx), 64, drv.ptr(do), 68, 2, 64, drv.ptr(dl), drv.ptr(dl), drv.stream) == -1   # carry aliased
    assert L.csdrb_fmdemod_quadri_bank_cf(None, 64, drv.ptr(do), 68, 2, 64, None, None, drv.stream) == -1
    assert L.csdrb_fmdemod_quadri_bank_cf(drv.ptr(dx), 64, drv.ptr(do), 68, 65536, 64, None, None, drv.stream) == -1
    assert L.csdrb_fmdemod_quadri_bank_cf(drv.ptr(dx), 64, drv.ptr(do), 68, 2, 0, None, None, drv.stream) == 0              # nothing to do
    assert L.csdrb_fmdemod_quadri_bank_cf(drv.ptr(dx), 64, drv.ptr(do), 68, 0, 64, None, None, drv.stream) == 0
    assert launches(drv) == n0
    untouched(drv.host(do), np.zeros((3, 68), bool), "refused fmdemod")


# =============================================================================================================================== fracdec
def _fb(v):
    return int(np.float32(v).view(np.uint32))


def _bf(b):
    return np.uint32(b).view(np.float32)


def fracdec_cap(n, rate):
    return int(n / float(np.float32(rate))) + 8


def fracdec_walk(where, n, rate, points, taps_length=0):
    """host restatement of fracdec_segments_kernel for one channel: dict with the segments [(k0, cnt, branch, end)], the position of every output
    (float32), output_size, the state it leaves and the number of table entries it used"""
    m = points & ~1
    xifirst = 1 - m // 2
    cap = fracdec_cap(n, rate)
    L = n - m - taps_length - 1
    rate = np.float32(rate)
    rb = _fb(rate)
    er = ((rb >> 23) & 0xFF) - 127
    R = (rb & 0x7FFFFF) | 0x800000
    where = np.float32(where)
    k, segs, pos = 0, [], []
    while math.ceil(float(where)) <= L and k < cap:
        cnt, q, branch, end = 1, 0, "single", "-"
        wb = _fb(where)
        E = ((wb >> 23) & 0xFF) - 127
        M = (wb & 0x7FFFFF) | 0x800000
        if where > 0 and 0 <= E <= 22 and len(segs) < FD_MAX_SEGS - 2:
            d = E - er
            cq, regular = 0, False
            if d <= 0:
                if d >= -6:
                    q = R << (-d); cq = q; regular = True; branch = "d<=0"
                else:
                    branch = "d<-6"
            elif d < 24:
                frac, I, half = R & ((1 << d) - 1), R >> d, 1 << (d - 1)
                cq = I + (1 if frac else 0)
                if frac != half:
                    q = I + (1 if frac > half else 0); regular = True; branch = "d>0"
                elif M & 1 == 0:
                    q = I + (I & 1); regular = True; branch = "tie-even"
                else:
                    branch = "tie-odd"
            if regular and q > 0:
                room = (1 << 24) - 1 - cq - M
                jreg = room // q if room >= 0 else -1
                lim = (L << (23 - E)) - M
                jlim = lim // q if lim >= 0 else 0
                j, end = (jreg, "binade") if jreg < jlim else (jlim, "jlim")
                j = max(j, 0)
                if j + 1 > cap - k:
                    j, end = cap - k - 1, "cap"
                cnt = j + 1
        if cnt > 1:
            mant = (M + np.arange(cnt, dtype=np.int64) * q) & 0x7FFFFF
            pos.append((((E + 127) << 23) | mant).astype(np.uint32).view(np.float32))
            last = pos[-1][-1]
        else:
            pos.append(np.array([where], np.float32))
            last = where
        segs.append((k, cnt, branch, end, (k, M, q, E, cnt) if cnt > 1 else (k, wb, 0, -1000, 1)))
        k += cnt
        where = np.float32(last + rate)
    processed = math.ceil(float(where)) - 1 + xifirst
    return dict(segs=segs, pos=np.concatenate(pos) if pos else np.zeros(0, np.float32), output_size=k, cap=cap,
                state=(float(np.float32(where - np.float32(processed))), processed, k))


def fracdec_chain(where, n, rate, points, taps_length=0, cap=None):
    """the reference's own float chain (libcsdr.c:765): positions and the state; `cap` stops storing like fracdec_positions_kernel"""
    m = points & ~1
    xifirst = 1 - m // 2
    where, rate = np.float32(where), np.float32(rate)
    pos = []
    while math.ceil(float(where)) + m + taps_length < n:
        pos.append(where)
        where = np.float32(where + rate)
    processed = math.ceil(float(where)) - 1 + xifirst
    k = len(pos) if cap is None else min(len(pos), cap)
    return np.array(pos[:k], np.float32), (float(np.float32(where - np.float32(processed))), processed, k)


def fracdec_path(n, points, taps):
    """launch_fractional_decimator_bank's kernels and the interpolation loop the case runs"""
    m = points & ~1
    if n >= 1 << 22:
        return ("fracdec_positions_kernel", "fracdec_interp_kernel")
    if taps is None and m == 12:
        return ("fracdec_segments_kernel", "fracdec_interp_seg_kernel<12>")
    return ("fracdec_segments_kernel", "fracdec_interp_seg_kernel<0>", "loop" if (taps is not None or m > 16) else "unrolled16")


def _lagrange_rows(x, pos, m, taps):
    """(low index, xw, the m points) of every output; x one row (float32) whose valid memory may start before index 0 (offset handled by the caller)"""
    low = np.ceil(pos.astype(np.float64)).astype(np.int64) - 1
    xw = (pos - low.astype(np.float32)).astype(np.float32)
    return low, xw


def lagrange_np(xrow, base, pos, points, taps=None):
    """the kernel's (and the reference's) order in numpy float32: xrow is the buffer, base the index of sample 0 in it"""
    m = points & ~1
    xifirst = 1 - m // 2
    low, xw = _lagrange_rows(xrow, pos, m, taps)
    idx = base + low
    acc = np.zeros(pos.size, np.float32)
    with np.errstate(all="ignore"):
        return _lagrange_sum(xrow, idx, xw, acc, m, xifirst, taps)


def _lagrange_sum(xrow, idx, xw, acc, m, xifirst, taps):
    for i in range(m):
        if taps is None:
            pt = xrow[idx + i]
        else:
            pt = np.zeros(xw.size, np.float32)
            for t in range(taps.size):
                pt = (pt + xrow[idx + i + t] * taps[t]).astype(np.float32)
        coef, den = np.ones(xw.size, np.float32), F32(1)
        for j in range(m):
            if j != i:
                coef = coef * (xw - F32(xifirst + j))
                den = F32(den * F32(i - j))
        acc = acc + (coef / den) * pt
    return acc


def lagrange64(xrow, base, pos, points, taps=None):
    """(float64 Lagrange sum at the chain's positions on the exact inputs, per-output bound)"""
    m = points & ~1
    xifirst = 1 - m // 2
    low, xw = _lagrange_rows(xrow, pos, m, taps)
    idx = base + low
    xw = xw.astype(np.float64)
    x64 = xrow.astype(np.float64)
    R = np.zeros(pos.size); S = np.zeros(pos.size)
    T = 0 if taps is None else taps.size
    for i in range(m):
        if taps is None:
            P = x64[idx + i]; A = np.abs(P)
        else:
            P = sum(x64[idx + i + t] * float(taps[t]) for t in range(T))
            A = sum(np.abs(x64[idx + i + t] * float(taps[t])) for t in range(T))
        Li = np.ones(pos.size)
        for j in range(m):
            if j != i:
                Li *= (xw - (xifirst + j)) / (i - j)
        R += Li * P; S += np.abs(Li) * A
    return R, (4 * m - 3 + T) * U * MARGIN * S


# case: rate, points, where per channel (None = the reference's start, -xifirst), n, taps length, calls of block B (None = one call), note
FD_CASES = [
    dict(rate=5.0, points=12, where=[None, 5.5, 5.0078125], n=3001, T=0, B=None, note="default 12 points, d <= 0 and d > 0, binade crossings"),
    dict(rate=1.25, points=12, where=[None, 5.25], n=2001, T=0, B=400, note="CLI calls of 400, carried state"),
    dict(rate=float(np.float32(1.25 + 12 * 2 ** -23)), points=12, where=[8.0, 8.0 + 2 ** -20, None], n=1201, T=0, B=None,
         note="tie in [8, 16) (rate/ulp(where) = I + 1/2 with I odd): M even and M odd"),
    dict(rate=float(np.float32(1.25 + 12 * 2 ** -23)), points=4, where=[8.0 + 2 ** -20, None], n=801, T=0, B=300, note="tie, 4 points, streamed"),
    dict(rate=200.0, points=4, where=[None, 1.5], n=3001, T=0, B=None, note="d < -6: where 1.0, rate >= 128"),
    dict(rate=130.5, points=2, where=[0.75, 0.5], n=1301, T=0, B=None, note="2 points from a carried where, d < -6"),
    dict(rate=2.5, points=16, where=[None, 7.3], n=1501, T=0, B=500, note="16 points: the unrolled generic form"),
    dict(rate=7.123, points=18, where=[None], n=1201, T=0, B=None, note="18 points: the loop"),
    dict(rate=3.3, points=32, where=[None, 15.7], n=901, T=0, B=None, note="32 points"),
    dict(rate=3.3, points=64, where=[None, 31.7], n=901, T=0, B=None, note="64 points: 63! overflows float, every output is NaN as in the reference"),
    dict(rate=4.0, points=12, where=[None, 5.9], n=1201, T=7, B=None, note="prefilter taps: the loop"),
    dict(rate=1.7, points=2, where=[0.9], n=501, T=3, B=200, note="2 points, prefilter, streamed"),
    dict(rate=1.5, points=4, where=[-60.0], n=401, T=0, B=None, note="a where below the row: the cap end", pre=70),
]


def fd_id(c):
    return f"r{c['rate']:.6g}-m{c['points']}-n{c['n']}-T{c['T']}-B{c['B']}"


def fd_walks(c, n=None):
    """the segment walks of every channel and call of a case (from the reference's chain of states)"""
    m = c["points"] & ~1
    out = []
    for w in c["where"]:
        where = float(m // 2 - 1) if w is None else w
        if c["B"] is None:
            out.append(fracdec_walk(where, n or c["n"], c["rate"], m, c["T"]))
            continue
        pos, need = 0, c["B"]
        while pos + need <= (n or c["n"]):
            wk = fracdec_walk(where, c["B"], c["rate"], m, c["T"])
            out.append(wk)
            pos += need
            where, need = wk["state"][0], wk["state"][1]
    return out


def fd_inputs(c, ch, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (ch, c["n"])).astype(np.float32)
    taps = rng.uniform(-1, 1, c["T"]).astype(np.float32) if c["T"] else None
    return x, taps


def fd_bank(drv, x, rate, points, taps, where, pre=0, in_pad=5):
    """one csdrb_fractional_decimator_bank_ff call on x [ch, n] (rows `pre` samples into rows padded with finite samples) from the device state
    `where` -> (outputs per channel, state rows, input rows, segment tables per channel); the output rows start as sentinels and must keep them
    past output_size"""
    ch, n = x.shape
    stride = pre + n + in_pad
    xb = np.full((ch, stride), F32(0.375), np.float32); xb[:, pre:pre + n] = x
    cap = fracdec_cap(n, rate)
    ob = sentinel_rows(ch + 1, cap + 3, np.float32)
    st = np.zeros(ch, STATE_DT); st["where"] = where; st["input_processed"] = -7; st["output_size"] = -7
    sb = drv.L.csdrb_fractional_decimator_bank_scratch_bytes(ch, n, rate)
    dx, do, ds, dsc = drv.dev(xb), drv.dev(ob), drv.dev(st), drv.dev(np.zeros(sb, np.uint8))
    dt = drv.dev(taps) if taps is not None else None
    rc = drv.L.csdrb_fractional_decimator_bank_ff(drv.ptr(dx) + 4 * pre, stride, drv.ptr(do), cap + 3, ch, n, rate, points,
                                                  drv.ptr(dt) if dt is not None else None, taps.size if taps is not None else 0,
                                                  drv.ptr(ds), drv.ptr(dsc), sb, drv.stream)
    assert rc >= 0, drv.L.csdrb_last_error()
    got, st, sc = drv.host(do), drv.host(ds), drv.host(dsc)
    mask = np.zeros(got.shape, bool)
    for c in range(ch):
        mask[c, :st["output_size"][c]] = True
    untouched(got, mask, f"fracdec n={n} rate={rate}: beyond output_size")
    tables = None
    if n < 1 << 22:
        seg = sc[:ch * FD_MAX_SEGS * SEG_DT.itemsize].view(SEG_DT).reshape(ch, FD_MAX_SEGS)
        ns = sc[ch * FD_MAX_SEGS * SEG_DT.itemsize:][:4 * ch].view("<i4")
        tables = [[tuple(int(v) for v in seg[c, i].tolist()) for i in range(min(int(ns[c]), FD_MAX_SEGS))] for c in range(ch)]
    return [got[c, :st["output_size"][c]].copy() for c in range(ch)], st, xb, tables


def check_fracdec(drv, oracle, c, seed=0, ch_rep=1, detail_rows=None):
    """bits and states against the oracle (one call, or the CLI's calls of B samples with the unconsumed rest carried), the host restatement of
    the segment walk and of the float chain, the numpy Lagrange sum, and the float64 bound -> the worst err/bound"""
    m = c["points"] & ~1
    wheres = [float(m // 2 - 1) if w is None else w for w in c["where"]] * ch_rep
    ch = len(wheres)
    x, taps = fd_inputs(c, ch, seed)
    rate = float(np.float32(c["rate"]))
    worst = 0.0
    if c["B"] is None:
        outs, st, xb, tables = fd_bank(drv, x, rate, c["points"], taps, wheres, pre=c.get("pre", 0))
        pre = c.get("pre", 0)
        for k in range(ch):
            if detail_rows is not None and k not in detail_rows:
                same(outs[k], oracle.fractional_decimator_ff(x[k], rate, c["points"], taps, where=wheres[k]), f"{fd_id(c)} channel {k}: oracle")
                continue
            wk = fracdec_walk(wheres[k], c["n"], rate, m, c["T"])
            pos, state = fracdec_chain(wheres[k], c["n"], rate, m, c["T"], cap=wk["cap"])
            assert_bits_equal(wk["pos"], pos, f"{fd_id(c)} channel {k}: segment walk against the float chain")
            assert tables[k] == [sg[4] for sg in wk["segs"]], f"{fd_id(c)} channel {k}: the kernel's segment table against the host walk"
            assert int(st["output_size"][k]) == pos.size == wk["output_size"]
            restated = lagrange_np(xb[k], pre, pos, m, taps)
            same(outs[k], restated, f"{fd_id(c)} channel {k}: numpy Lagrange restatement")
            R, B = lagrange64(xb[k], pre, pos, m, taps)
            fin = np.isfinite(restated)                               # weights overflow float from about 34 points on (the reference's too)
            assert fin.all() or m > 32
            worst = max(worst, within(outs[k][fin], R[fin], B[fin], f"{fd_id(c)} channel {k}: float64 bound"))
            if pre == 0:
                states = []
                want = oracle.fractional_decimator_ff(x[k], rate, c["points"], taps, where=wheres[k], states=states)
                same(outs[k], want, f"{fd_id(c)} channel {k}: oracle")
                assert (np.float32(st["where"][k]), int(st["input_processed"][k]), int(st["output_size"][k])) == \
                       (np.float32(states[0][0]), states[0][1], states[0][2]) == (np.float32(wk["state"][0]), wk["state"][1], wk["state"][2])
            else:                                                     # the cap end: outputs stop at cap, every one at its chain position
                assert wk["segs"][-1][3] == "cap" and int(st["output_size"][k]) == wk["cap"]
        return worst
    # the CLI's framing: B-sample calls, the unconsumed rest moved to the front, the device state carried
    B = c["B"]
    st = np.zeros(ch, STATE_DT); st["where"] = wheres
    ds = drv.dev(st)
    bufs = np.zeros((ch, B), np.float32)
    pos = np.zeros(ch, np.int64); proc = np.zeros(ch, np.int64)
    got = [[] for _ in range(ch)]; states = [[] for _ in range(ch)]
    before = np.float32(wheres)
    sb = drv.L.csdrb_fractional_decimator_bank_scratch_bytes(ch, B, rate)
    dsc = drv.dev(np.zeros(sb, np.uint8)); dt = drv.dev(taps) if taps is not None else None
    cap = fracdec_cap(B, rate)
    while True:
        need = np.where(proc == 0, B, proc)
        if np.any(pos + need > c["n"]):
            break
        for k in range(ch):
            keep = B - need[k]
            bufs[k, :keep] = bufs[k, need[k]:].copy()
            bufs[k, keep:] = x[k, pos[k]:pos[k] + need[k]]
        pos += need
        ob = sentinel_rows(ch, cap + 2, np.float32)
        dx, do = drv.dev(bufs), drv.dev(ob)
        rc = drv.L.csdrb_fractional_decimator_bank_ff(drv.ptr(dx), B, drv.ptr(do), cap + 2, ch, B, rate, c["points"],
                                                      drv.ptr(dt) if dt is not None else None, c["T"], drv.ptr(ds), drv.ptr(dsc), sb, drv.stream)
        assert rc >= 0, drv.L.csdrb_last_error()
        o, s = drv.host(do), drv.host(ds)
        mask = np.zeros(o.shape, bool)
        for k in range(ch):
            mask[k, :s["output_size"][k]] = True
            got[k].append(o[k, :s["output_size"][k]].copy())
            states[k].append((np.float32(s["where"][k]), int(s["input_processed"][k]), int(s["output_size"][k])))
            wk = fracdec_walk(before[k], B, rate, m, c["T"])
            assert (np.float32(wk["state"][0]), wk["state"][1], wk["state"][2]) == states[k][-1], f"{fd_id(c)} channel {k}: walk state"
            R, Bd = lagrange64(bufs[k], 0, wk["pos"], m, taps)
            worst = max(worst, within(got[k][-1], R, Bd, f"{fd_id(c)} channel {k} call {len(got[k])}: float64 bound"))
        untouched(o, mask, f"{fd_id(c)}: beyond output_size")
        proc = s["input_processed"].astype(np.int64)
        before = s["where"].copy()
    assert got[0], "the case made no call"
    for k in range(ch):
        want_states = []
        want = oracle.fractional_decimator_ff(x[k, :pos[k]], rate, c["points"], taps, block=B, where=wheres[k], states=want_states)
        assert [(np.float32(w), a, b) for w, a, b in want_states] == states[k], f"{fd_id(c)} channel {k}: states after every call"
        same(np.concatenate(got[k]), want, f"{fd_id(c)} channel {k}: streamed against the oracle")
    return worst


def check_fracdec_big(drv, oracle, c, seed=0, bound_outputs=50_000):
    """rows of 2^22 samples and more (the sequential fallback): outputs and state against the oracle, the segment walk's positions and state
    (the closed form agrees with the chain the fallback replays), and the float64 bound on the first outputs"""
    assert c["n"] >= 1 << 22 and c["B"] is None
    m = c["points"] & ~1
    wheres = [float(m // 2 - 1) if w is None else w for w in c["where"]]
    x, taps = fd_inputs(c, len(wheres), seed)
    rate = float(np.float32(c["rate"]))
    outs, st, xb, _ = fd_bank(drv, x, rate, c["points"], taps, wheres)
    worst = 0.0
    for k, w in enumerate(wheres):
        states = []
        same(outs[k], oracle.fractional_decimator_ff(x[k], rate, c["points"], taps, where=w, states=states), f"{fd_id(c)} channel {k}: oracle")
        wk = fracdec_walk(w, c["n"], rate, m, c["T"])
        got = (np.float32(st["where"][k]), int(st["input_processed"][k]), int(st["output_size"][k]))
        assert got == (np.float32(states[0][0]), states[0][1], states[0][2]) == (np.float32(wk["state"][0]), wk["state"][1], wk["state"][2]), got
        pos = wk["pos"][:bound_outputs]
        R, B = lagrange64(xb[k], 0, pos, m, taps)
        worst = max(worst, within(outs[k][:pos.size], R, B, f"{fd_id(c)} channel {k}: float64 bound"))
    return worst


def fd_segment_sweep(n=(1 << 22) - 1):
    """the most table entries any walk takes: the matrix and a sweep of rates and point counts at n = 2^22 - 1, from the start and from the far
    ends of the carried range (m/2 - 1, m/2]"""
    worst, at = 0, None
    rates = np.unique(np.concatenate([np.geomspace(1.0001, 2000.0, 60).astype(np.float32),
                                      np.float32([1.25 + 4 * 2 ** -23, 1.5, 2.0, 3.0, 4.0, 5.0, 7.123, 10.0, 128.0, 130.5, 1e5])]))
    for rate in rates:
        for m in (2, 4, 12, 16, 64):
            for w in (float(m // 2 - 1), float(np.nextafter(np.float32(m // 2 - 1), np.float32(m))), float(m // 2)):
                if w <= 0:
                    continue
                s = len(fracdec_walk(w, n, float(rate), m)["segs"])
                if s > worst:
                    worst, at = s, (float(rate), m, w)
    for c in FD_CASES:
        for wk in fd_walks(c):
            if len(wk["segs"]) > worst:
                worst, at = len(wk["segs"]), fd_id(c)
    return worst, at


def check_fracdec_refusals(drv):
    x = np.zeros((2, 200), np.float32)
    st = np.zeros(2, STATE_DT); st["where"] = 5.0
    dx, ds = drv.dev(x), drv.dev(st)
    ob = sentinel_rows(2, 200, np.float32); do = drv.dev(ob)
    sb = drv.L.csdrb_fractional_decimator_bank_scratch_bytes(2, 200, 2.0)
    dsc = drv.dev(np.zeros(sb, np.uint8))
    L, n0 = drv.L, launches(drv)

    def call(rate=2.0, points=12, scratch=sb, ch=2, n=200, inp=True, state=True):
        return L.csdrb_fractional_decimator_bank_ff(drv.ptr(dx) if inp else None, 200, drv.ptr(do), 200, ch, n, rate, points, None, 0,
                                                    drv.ptr(ds) if state else None, drv.ptr(dsc), scratch, drv.stream)
    assert call(rate=1.0) == -1 and call(rate=0.5) == -1 and call(rate=float("nan")) == -1
    assert call(points=1) == -1 and call(points=66) == -1 and call(points=0) == -1
    assert call(scratch=sb - 1) == -1 and call(inp=False) == -1 and call(state=False) == -1 and call(ch=65536) == -1
    assert call(ch=0) == 0 and call(n=0) == 0
    assert launches(drv) == n0
    untouched(drv.host(do), np.zeros((2, 200), bool), "refused fracdec")
    s = drv.host(ds)
    assert np.all(s["where"] == 5.0) and np.all(s["output_size"] == 0), "a refused call changed the state"


# =============================================================================================================================== fastagc
AGC_BLOCKS = [1, 2, 255, 256, 257, 1000, 1023, 1024, 1025, 4096]
AGC_CUTS = {"1": [1], "2": [2], "3": [3], "16": [16], "17": [17], "33": [33], "1-block calls": [1] * 5, "16+1+2": [16, 1, 2], "17+16": [17, 16]}


def agc_path(block, nblocks, s16=False):
    """the launches of launch_fastagc_bank / _s16 for one call"""
    main = (f"fastagc_fused_kernel<{'true' if s16 else 'false'}>",) if block <= 1024 else \
        ("fastagc_peaks_kernel", f"fastagc_apply_kernel<{'true' if s16 else 'false'}>")
    return main + ("fastagc_carry_kernel", "carry: shift history" if nblocks == 1 else "carry: copy two blocks",
                   f"runs: {(nblocks + AGC_RUN - 1) // AGC_RUN}" if block <= 1024 else "one CTA per block")


def agc_inputs(ch, block, nb, seed):
    rng = np.random.default_rng(seed)
    env = rng.uniform(0.001, 1.0, (ch, nb)).astype(np.float32)
    x = (rng.uniform(-1, 1, (ch, nb * block)) * np.repeat(env, block, axis=1) * np.float32(30.0) ** rng.uniform(-1, 1, (ch, 1))).astype(np.float32)
    if nb >= 4:
        x[0, block:3 * block] = 0                                     # zero blocks: gain capped at 50
    return x


def agc64(x, block, reference):
    """(float64 fastagc of the exact inputs, per-output bound) over the whole stream from the start state"""
    ch, n = x.shape
    nb = n // block
    pk = np.abs(x[:, :nb * block].astype(np.float64)).reshape(ch, nb, block).max(axis=2)
    pk = np.concatenate([np.zeros((ch, 2)), pk], axis=1)
    t = np.maximum(np.maximum(pk[:, 2:], pk[:, 1:-1]), pk[:, :-2])
    with np.errstate(divide="ignore"):
        TG = np.minimum(reference / t, 50.0)
    LG = np.concatenate([np.zeros((ch, 1)), TG[:, :-1]], axis=1)
    r = np.arange(block) / block
    G = LG[:, :, None] * (1 - r) + TG[:, :, None] * r
    lv = np.concatenate([np.zeros((ch, 2 * block)), x.astype(np.float64)], axis=1)[:, :nb * block].reshape(ch, nb, block)
    Y = lv * G
    Bd = U * MARGIN * np.abs(lv) * (LG[:, :, None] + 3 * TG[:, :, None] * r + 2 * G)
    return Y.reshape(ch, -1), Bd.reshape(ch, -1)


def agc_bank(drv, x, block, cuts, reference=0.8, s16=False, in_pad=3, out_pad=5, paths=None):
    """csdrb_fastagc_bank_ff / _f_s16 over x [ch, sum(cuts) * block] in calls of cuts[i] blocks, state and history carried on the device; rows
    strided (in_pad, out_pad extra samples) and the output's padding and spare row must keep their sentinels"""
    ch = x.shape[0]
    st = drv.dev(np.zeros((ch, 3), np.float32)); hist = drv.dev(np.zeros((ch, 2, block), np.float32))
    outs, at = [], 0
    dt = np.int16 if s16 else np.float32
    for nb in cuts:
        n = nb * block
        xb = rows_in(x[:, at:at + n], n + in_pad, 0, F32(np.nan)); at += n
        ob = sentinel_rows(ch + 1, n + out_pad, dt)
        sb = drv.L.csdrb_fastagc_bank_scratch_bytes(ch, nb)
        dx, do, dsc = drv.dev(xb), drv.dev(ob), drv.dev(np.zeros(sb, np.uint8))
        f = drv.L.csdrb_fastagc_bank_f_s16 if s16 else drv.L.csdrb_fastagc_bank_ff
        n0 = launches(drv)
        rc = f(drv.ptr(dx), n + in_pad, drv.ptr(do), n + out_pad, ch, block, nb, reference, drv.ptr(st), drv.ptr(hist), drv.ptr(dsc), sb, drv.stream)
        want = agc_path(block, nb, s16)
        assert rc == 0 and launches(drv) - n0 == (2 if block <= 1024 else 3), (rc, launches(drv) - n0, drv.L.csdrb_last_error())
        if paths is not None:
            paths.update(want)
        o = drv.host(do)
        mask = np.zeros(o.shape, bool); mask[:ch, :n] = True
        untouched(o, mask, f"fastagc block={block} call of {nb}")
        outs.append(o[:ch, :n])
    return np.concatenate(outs, axis=1), drv.host(st)


def check_fastagc(drv, oracle, ch, block, cuts, seed=0, s16=True, paths=None, bound_rows=None):
    """float and s16 bits of the oracle over the stream cut into calls, the carried state, and the float64 bound"""
    nb = sum(cuts)
    x = agc_inputs(ch, block, nb, seed)
    y, st = agc_bank(drv, x, block, cuts, paths=paths)
    want = np.stack([oracle.fastagc_ff(x[c], block, 0.8) for c in range(ch)])
    same(y, want, f"fastagc block={block} cuts={cuts}: oracle")
    if s16:
        ys, st2 = agc_bank(drv, x, block, cuts, s16=True, paths=paths)
        assert_bits_equal(ys, np.stack([oracle.convert_f_s16(want[c]) for c in range(ch)]), f"fastagc s16 block={block} cuts={cuts}")
        assert_bits_equal(st2, st, "s16 carried state")
    rows = range(ch) if bound_rows is None else bound_rows
    Y, Bd = agc64(x[list(rows)], block, 0.8)
    worst = within(y[list(rows)], Y, Bd, f"fastagc block={block}: float64 bound")
    # the carried state: peaks of the last two blocks and the last target
    pk = np.abs(x).reshape(ch, nb, block).max(axis=2)
    assert_bits_equal(st[:, 0], pk[:, -2] if nb >= 2 else np.zeros(ch, np.float32), "peak_1")
    assert_bits_equal(st[:, 1], pk[:, -1], "peak_2")
    return worst


def check_fastagc_nonfinite(drv, oracle, block, cuts, seed=0):
    """NaN and +-Inf samples: the outputs equal the oracle's and differ from the clean run exactly where the oracle's do"""
    ch, nb = 3, sum(cuts)
    x = agc_inputs(ch, block, nb, seed)
    xp = x.copy()
    for c, v in enumerate((np.nan, np.inf, -np.inf)):
        xp[c, (block * nb) // 3] = v
        xp[c, block * nb - 1] = v if c == 0 else F32(0.5)
    clean, _ = agc_bank(drv, x, block, cuts)
    got, _ = agc_bank(drv, xp, block, cuts)
    for c in range(ch):
        want = oracle.fastagc_ff(xp[c], block, 0.8)
        same(got[c], want, f"fastagc block={block} poisoned channel {c}")
        wclean = oracle.fastagc_ff(x[c], block, 0.8)
        moved = bits(want) != bits(wclean)
        assert np.array_equal(bits(got[c]) != bits(clean[c]), moved), f"channel {c}: changed outputs differ from the reference's"


def check_fastagc_refusals(drv):
    ch, block, nb = 2, 64, 3
    x = np.zeros((ch, nb * block), np.float32)
    dx = drv.dev(x); do = drv.dev(sentinel_rows(ch, nb * block, np.float32))
    st0 = np.full((ch, 3), 0.25, np.float32)
    st, hist = drv.dev(st0), drv.dev(np.zeros((ch, 2, block), np.float32))
    sb = drv.L.csdrb_fastagc_bank_scratch_bytes(ch, nb); dsc = drv.dev(np.zeros(sb, np.uint8))
    L, n0 = drv.L, launches(drv)
    for f in (L.csdrb_fastagc_bank_ff, L.csdrb_fastagc_bank_f_s16):
        assert f(drv.ptr(dx), nb * block, drv.ptr(do), nb * block, ch, 0, nb, 0.8, drv.ptr(st), drv.ptr(hist), drv.ptr(dsc), sb, drv.stream) == -1
        assert f(drv.ptr(dx), nb * block, drv.ptr(do), nb * block, ch, block, nb, 0.8, drv.ptr(st), drv.ptr(hist), drv.ptr(dsc), sb - 1, drv.stream) == -1
        assert f(drv.ptr(dx), nb * block, drv.ptr(do), nb * block, ch, block, nb, 0.8, None, drv.ptr(hist), drv.ptr(dsc), sb, drv.stream) == -1
        assert f(drv.ptr(dx), nb * block, drv.ptr(do), nb * block, 65536, block, nb, 0.8, drv.ptr(st), drv.ptr(hist), drv.ptr(dsc), sb, drv.stream) == -1
        assert f(drv.ptr(dx), nb * block, drv.ptr(do), nb * block, ch, block, 0, 0.8, drv.ptr(st), drv.ptr(hist), drv.ptr(dsc), sb, drv.stream) == 0
    assert L.csdrb_fastagc_bank_ff(drv.ptr(dx), nb * block, drv.ptr(dx), nb * block, ch, block, nb, 0.8, drv.ptr(st), drv.ptr(hist), drv.ptr(dsc), sb,
                                   drv.stream) == -1                                     # in place
    assert launches(drv) == n0
    untouched(drv.host(do), np.zeros((ch, nb * block), bool), "refused fastagc")
    assert_bits_equal(drv.host(st), st0, "state after refused calls")


# =============================================================================================================================== fir_valid
FV_T = [1, 2, 201, 208]
FV_OUT = [1, 255, 256, 257, 767, 769, 1023, 1024, 1025, 2049]


def fv_bank(drv, x, taps, limit=0.0, in_pad=3, out_pad=4, col0=0):
    """csdrb_fir_valid_bank_ff on x [ch, n] -> y [ch, n - T]; rows strided, the outputs' padding and spare row keep their sentinels"""
    ch, n = x.shape
    T = taps.size
    n_out = max(n - T, 0)
    xb = rows_in(x, col0 + n + in_pad, col0, F32(np.nan))
    ob = sentinel_rows(ch + 1, n_out + out_pad, np.float32)
    dx, do = drv.dev(xb), drv.dev(ob)
    rc = drv.L.csdrb_fir_valid_bank_ff(drv.ptr(dx) + 4 * col0, xb.shape[1], drv.ptr(do), ob.shape[1], ch, n,
                                       np.ascontiguousarray(taps, np.float32).ctypes.data_as(C.POINTER(C.c_float)), T, limit, drv.stream)
    assert rc == n_out, (rc, n_out, drv.L.csdrb_last_error())
    o = drv.host(do)
    mask = np.zeros(o.shape, bool); mask[:ch, :n_out] = True
    untouched(o, mask, f"fir_valid T={T} n={n}")
    return np.ascontiguousarray(o[:ch, :n_out])


def fv64(x, taps):
    """(float64 valid FIR of the exact inputs -- n - T outputs, like the reference loop -- and the gamma_T bound)"""
    T = taps.size
    n_out = x.shape[1] - T
    h = taps.astype(np.float64)
    g = T * U / (1 - T * U) * MARGIN
    Y, Bd = np.zeros((x.shape[0], n_out)), np.zeros((x.shape[0], n_out))
    for c in range(x.shape[0]):                                       # one row at a time: the window view is T times the row
        w = np.lib.stride_tricks.sliding_window_view(x[c].astype(np.float64), T)[:n_out]
        Y[c], Bd[c] = w @ h, g * (np.abs(w) @ np.abs(h))
    return Y, Bd


def fv_path(T, n, limit):
    """launch_fir_valid_bank's kernel and its tiles: which of the four accumulators (outputs 0, 256, 512, 768 of a 1024-output tile) the last
    tile stores"""
    n_out = n - T
    live = (n_out - 1) % 1024 + 1
    return (f"nfm_deemph_bank_kernel<{'true' if limit > 0 else 'false'}>", f"tiles: {(n_out + 1023) // 1024}",
            "last tile accumulators: " + "".join(str(a) for a in range(4) if live > 256 * a))


def fv_inputs(ch, n, T, seed):
    rng = np.random.default_rng(seed)
    return rng.uniform(-2.5, 2.5, (ch, n)).astype(np.float32), rng.uniform(-1, 1, T).astype(np.float32)


def check_fir_valid(drv, oracle, ch, T, n_out, limit=0.0, seed=0, paths=None):
    """bound, oracle agreement within it, and the exact invariants: tile offset, row stride, channel subset, split calls, unit tap, 2^k taps,
    and (limit > 0) the fused limiter equals limit_ff then the FIR"""
    n = n_out + T
    x, h = fv_inputs(ch, n, T, seed)
    if paths is not None:
        paths.update(fv_path(T, n, limit))
    y = fv_bank(drv, x, h, limit)
    xl = np.stack([oracle.limit_ff(r, limit) for r in x]) if limit > 0 else x
    Y, Bd = fv64(xl, h)
    worst = within(y, Y, Bd, f"fir_valid T={T} n_out={n_out}: float64 bound")
    if limit > 0:
        assert_bits_equal(fv_bank(drv, xl, h), y, "fused limiter against limit_ff then the FIR")
    assert_bits_equal(fv_bank(drv, x, h, limit, in_pad=0, out_pad=0, col0=1), y, "tight rows, one sample in")
    rng = np.random.default_rng(seed + 1)
    sub = rng.permutation(ch)[:2]
    assert_bits_equal(fv_bank(drv, x[sub], h, limit), y[sub], "permuted channel subset")
    for s in (1, 255, 256, 257, 511, 768, 1023):
        if s < n_out:
            assert_bits_equal(fv_bank(drv, np.ascontiguousarray(x[:, s:]), h, limit), y[:, s:], f"started {s} outputs later (tile offset)")
    if n_out > 2:
        a = n_out // 3 + 1
        parts = [fv_bank(drv, np.ascontiguousarray(x[:, :a + T]), h, limit), fv_bank(drv, np.ascontiguousarray(x[:, a:]), h, limit)]
        assert_bits_equal(np.concatenate(parts, axis=1), y, "split into two calls")
    for k in sorted({0, T // 2, T - 1}):
        e = np.zeros(T, np.float32); e[k] = 1
        assert_bits_equal(fv_bank(drv, x, e, limit), np.ascontiguousarray(xl[:, k:k + n_out]), f"unit tap at {k}")
    assert_bits_equal(fv_bank(drv, x, (h * F32(2.0 ** -5)).astype(np.float32), limit), (y * F32(2.0 ** -5)).astype(np.float32), "taps scaled by 2^-5")
    return worst


def check_fir_valid_nonfinite(drv, T, n_out, limit=0.0, seed=0):
    """a NaN or +-Inf at sample p makes outputs p - T + 1 .. p non-finite and changes nothing else; with the limiter NaN clamps to +max,
    +-Inf to +-max, and the outputs are the clamped stream's"""
    ch = 3
    n = n_out + T
    x, h = fv_inputs(ch, n, T, seed)
    pos = sorted({0, T - 1, T + 255, min(T + 1024, n - 1), n - 1})
    xp = x.copy()
    bad = np.array([np.nan, np.inf, -np.inf], np.float32)
    for c in range(ch):
        for i, p in enumerate(pos):
            xp[c, p] = bad[(c + i) % 3]
    clean, got = fv_bank(drv, x, h, limit), fv_bank(drv, xp, h, limit)
    if limit > 0:
        xl = np.clip(np.where(np.isnan(xp), F32(limit), xp), -F32(limit), F32(limit)).astype(np.float32)
        assert_bits_equal(got, fv_bank(drv, xl, h), "limited non-finite samples")
        assert np.all(np.isfinite(got))
        return
    o = np.arange(n_out)
    hit = np.zeros(n_out, bool)
    for p in pos:
        hit |= (o <= p) & (p < o + T)
    for c in range(ch):
        assert np.array_equal(~np.isfinite(got[c]), hit), (c, np.flatnonzero(~np.isfinite(got[c]))[:10], np.flatnonzero(hit)[:10])
        assert_bits_equal(got[c][~hit], clean[c][~hit], f"fir_valid channel {c}: outputs away from the poisoned samples")


def check_fir_valid_refusals(drv):
    x = np.zeros((2, 300), np.float32)
    dx = drv.dev(x); do = drv.dev(sentinel_rows(2, 300, np.float32))
    L, n0 = drv.L, launches(drv)
    h = np.ones(NFM_MAX_TAPS + 1, np.float32)
    hp = h.ctypes.data_as(C.POINTER(C.c_float))
    f = L.csdrb_fir_valid_bank_ff
    assert f(drv.ptr(dx), 300, drv.ptr(do), 300, 2, 300, hp, NFM_MAX_TAPS + 1, 0.0, drv.stream) == -1
    assert f(drv.ptr(dx), 300, drv.ptr(do), 300, 2, 300, hp, 0, 0.0, drv.stream) == -1
    assert f(drv.ptr(dx), 300, drv.ptr(do), 300, 2, 300, None, 3, 0.0, drv.stream) == -1
    assert f(None, 300, drv.ptr(do), 300, 2, 300, hp, 3, 0.0, drv.stream) == -1
    assert f(drv.ptr(dx), 300, drv.ptr(do), 300, 65536, 300, hp, 3, 0.0, drv.stream) == -1
    assert f(drv.ptr(dx), 300, drv.ptr(do), 300, 2, 3, hp, 3, 0.0, drv.stream) == 0          # n == T: no output
    assert f(drv.ptr(dx), 300, drv.ptr(do), 300, 0, 300, hp, 3, 0.0, drv.stream) == 0
    assert L.csdrb_deemphasis_nfm_bank_ff(drv.ptr(dx), 300, drv.ptr(do), 300, 2, 300, 22050, 0.0, drv.stream) == 0   # no table for the rate
    assert launches(drv) == n0
    untouched(drv.host(do), np.zeros((2, 300), bool), "refused fir_valid")


# =============================================================================================================================== deemphasis_wfm
WFM_ROWS = [1, 31, 32, 33, 127, 128, 129]
WFM_N = [1, 31, 32, 33, 100]
TAU, SR = 75e-6, 48000


def wfm_path(ch):
    warps = (ch + 31) // 32
    return ("deemphasis_wfm_bank_kernel", f"CTAs: {(ch + 127) // 128}", f"warps: {warps}", f"rows of the last warp: {ch - 32 * (warps - 1)}")


def wfm_coefs(tau=TAU, sr=SR):
    dt = np.float32(1.0 / sr)
    alpha = np.float32(dt / np.float32(np.float32(tau) + dt))
    return alpha, np.float32(1 - alpha)


def wfm64(x, last, tau=TAU, sr=SR):
    """(float64 recursion with the kernel's float coefficients on the exact inputs, running bound); last must be finite"""
    a, k = (float(v) for v in wfm_coefs(tau, sr))
    ch, n = x.shape
    Y = np.zeros((ch, n)); Bd = np.zeros((ch, n))
    y, e = last.astype(np.float64), np.zeros(ch)
    for i in range(n):
        e = k * e + 2 * U * MARGIN * (np.abs(a * x[:, i].astype(np.float64)) + k * (np.abs(y) + e))
        y = a * x[:, i] + k * y
        Y[:, i], Bd[:, i] = y, e
    return Y, Bd


def wfm_bank(drv, x, last, in_pad=3, out_pad=2, tau=TAU, sr=SR):
    ch, n = x.shape
    xb = rows_in(x, n + in_pad, 0, F32(np.nan))
    ob = sentinel_rows(ch + 1, n + out_pad, np.float32)
    lb = np.full(ch + 1, np.float32(np.nan), np.float32); lb[:ch] = last
    lb = lb.view(np.uint32); lb[ch] = SENTINEL; lb = lb.view(np.float32)
    dx, do, dl = drv.dev(xb), drv.dev(ob), drv.dev(lb)
    rc = drv.L.csdrb_deemphasis_wfm_bank_ff(drv.ptr(dx), n + in_pad, drv.ptr(do), n + out_pad, ch, n, tau, sr, drv.ptr(dl), drv.stream)
    assert rc >= 0, drv.L.csdrb_last_error()
    o, l = drv.host(do), drv.host(dl)
    mask = np.zeros(o.shape, bool); mask[:ch, :n] = True
    untouched(o, mask, f"deemphasis_wfm ch={ch} n={n}")
    assert l.view(np.uint32)[ch] == SENTINEL, "carry stored past the last channel"
    return np.ascontiguousarray(o[:ch, :n]), l[:ch]


def wfm_inputs(ch, n, seed):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-1, 1, (ch, n)).astype(np.float32)
    last = rng.uniform(-1, 1, ch).astype(np.float32)
    special = np.array([np.nan, np.inf, -np.inf, 0.0], np.float32)
    at = np.arange(0, ch, 7) if ch >= 28 else np.arange(min(ch, 4))
    last[at] = special[np.arange(at.size) % 4]                       # carried NaN (restarts from 0), +-Inf (kept), 0
    return x, last


def check_wfm(drv, oracle, ch, n, seed=0, cuts=None, paths=None):
    """bits and carry of the oracle (a NaN carry restarts from 0 at every call, Inf is kept), the float64 bound on rows with a finite carry,
    and the stream cut into equal calls"""
    x, last = wfm_inputs(ch, n, seed)
    if paths is not None:
        paths.update(wfm_path(ch))
    y, lo = wfm_bank(drv, x, last)
    for c in range(ch):
        want, wl = oracle.deemphasis_wfm_ff(x[c], TAU, SR, float(last[c]))
        same(y[c], want, f"deemphasis_wfm ch={ch} n={n} channel {c}")
        same(lo[c:c + 1], np.float32([wl]), f"deemphasis_wfm channel {c}: carry")
    l0 = np.where(np.isnan(last), 0, last)
    ok = np.isfinite(l0)
    Y, Bd = wfm64(x[ok], l0[ok])
    worst = within(y[ok], Y, Bd, f"deemphasis_wfm ch={ch} n={n}: float64 bound") if ok.any() else 0.0
    if cuts:
        parts, carry = [], last
        for a in range(0, n, cuts):
            yy, carry = wfm_bank(drv, np.ascontiguousarray(x[:, a:a + cuts]), carry)
            parts.append(yy)
        for c in range(ch):
            want, _ = oracle.deemphasis_wfm_ff(x[c], TAU, SR, float(last[c]), block=cuts)
            same(np.concatenate(parts, axis=1)[c], want, f"deemphasis_wfm channel {c} in calls of {cuts}")
    return worst


def check_wfm_refusals(drv):
    x = np.zeros((2, 40), np.float32)
    dx, do = drv.dev(x), drv.dev(sentinel_rows(2, 40, np.float32))
    l0 = np.float32([0.5, -0.5]); dl = drv.dev(l0)
    L, n0 = drv.L, launches(drv)
    f = L.csdrb_deemphasis_wfm_bank_ff
    assert f(drv.ptr(dx), 40, drv.ptr(do), 40, 2, 40, TAU, 0, drv.ptr(dl), drv.stream) == -1
    assert f(drv.ptr(dx), 40, drv.ptr(do), 40, 2, 40, TAU, -48000, drv.ptr(dl), drv.stream) == -1
    assert f(drv.ptr(dx), 40, drv.ptr(do), 40, 2, 40, TAU, SR, None, drv.stream) == -1
    assert f(None, 40, drv.ptr(do), 40, 2, 40, TAU, SR, drv.ptr(dl), drv.stream) == -1
    assert f(drv.ptr(dx), 40, drv.ptr(do), 40, 2, 0, TAU, SR, drv.ptr(dl), drv.stream) == 0
    assert f(drv.ptr(dx), 40, drv.ptr(do), 40, 0, 40, TAU, SR, drv.ptr(dl), drv.stream) == 0
    assert launches(drv) == n0
    untouched(drv.host(do), np.zeros((2, 40), bool), "refused deemphasis_wfm")
    assert_bits_equal(drv.host(dl), l0, "carry after refused calls")


# =============================================================================================================================== coverage
FD_BRANCHES = {"d<=0", "d<-6", "d>0", "tie-even", "tie-odd", "single"}
FD_ENDS = {"binade", "jlim", "cap"}


def fd_coverage(cases):
    """segment branches and segment ends the cases' walks take, and the kernels they launch"""
    br, ends, kern = set(), set(), set()
    for c in cases:
        kern.add(fracdec_path(c["n"] if c["B"] is None else c["B"], c["points"], None if not c["T"] else True))
        for wk in fd_walks(c):
            for _, cnt, b, e, _ in wk["segs"]:
                br.add(b)
                if cnt > 1 or e == "cap":
                    ends.add(e)
    return br, ends, kern
