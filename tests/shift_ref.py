"""Restatements, error bounds, case matrix and checks of the NCO shift banks, shared by tests/test_shift_emulated.py (CPU tier, the emulated
library) and tests/test_gpu_shift.py (-m gpu):

    shift_phase_chain_kernel + shift_bank_kernel<float2>     csdrb_shift_addition_bank_cc, shift_addition_cc
    shift_phase_chain_kernel + shift_bank_kernel<float>      csdrb_shift_addition_bank_fc, shift_addition_fc (seeded by the host's sincosf)
    addfast_phase_chain_kernel + shift_addfast_bank_kernel   csdrb_shift_addfast_bank_cc, shift_addfast_cc
    shift_math_chain_kernel + shift_math_bank_kernel         csdrb_shift_math_bank_cc, shift_math_cc
    shift_math_chain_kernel + shift_table_bank_kernel        csdrb_shift_table_bank_cc, shift_table_cc
    shift_phase_chain_kernel + shift_unroll_bank_kernel      csdrb_shift_unroll_bank_cc, shift_unroll_cc
    dshift_kernel                                            csdrb_decimating_shift_addition_bank_cc, decimating_shift_addition_cc

Every check holds a call to four things.

(1) The phase chains, bit for bit: the start phase of every chunk (the scratch's first [C][nchunks] floats), every 256-sample segment phase
of shift_math / shift_table ([C][nseg]), the carried phase_io and the decimating state {remain, phase, output_size}, against the oracle's
float chains (oracle_shift_chain, oracle_shift_math_phases, oracle_decimating_shift_addition_cc).  No cos is involved: exact on any device.

(2) The samples, bit for bit: a numpy float32 restatement of each mixer (separately rounded products and sums, the kernels' operand order)
from the seeds.  A seed is (float)cos((double)ph), (float)sin((double)ph).  The device evaluates cos/sin in CUDA's double libm (2 ulp), the
restatement in the host's (glibc's, within an ulp); when the double value lies within AMBIG_ULPS = 4 double ulps of a float rounding midpoint
the two may round the component to different neighbours, and the recursion carries that through the chunk.  Such a seed is *ambiguous*
(about 2^-26 of all components): its chunk (sample for shift_math, call for unroll/decimating) must equal the restatement for one of the
candidate roundings of its components, bit for bit.  Every other chunk must equal the restatement for the host's rounding.  The emulated
library calls the host's libm, so there the host's rounding is the only one that can match.

(3) A float64 per-sample bound.  u = 2^-24.  A rotation rotate_rn(p, v) rounds two products and a sum per component:
    |fl(fl(ab) -+ fl(cd)) - (ab -+ cd)| <= 2u (|ab| + |cd|) (1 + u),   and |ab| + |cd| <= |p| |v| (Cauchy-Schwarz),
so its complex error is at most 2 sqrt2 u |p| |v| (1 + u).  The model is the exact product of the kernels' float inputs: the float seed s,
the float step d of shift_addition_init, the float table entries.
  * shift_addition (recursion p_(j+1) = rot(p_j, d)): e_(j+1) = e_j d + delta_j, |delta_j| <= 2 sqrt2 u |p_j| |d| (1 + u), so with
    G_j = 1 + 4 (j + 2) u >= max |p_i|, |d|^i (i <= j) to first order,
        |y_j - x_j s d^j| <= 2 sqrt2 u (j + 1) G_j |x_j|                               (cc: the sample's own rotation is the "+ 1")
        |y_j - x_j s d^j| <= (2 sqrt2 j + 1) u G_j |x_j|                               (fc: one rounded product per component)
  * shift_addfast: the phasor advances by d_4 once per group g = j // 4, then the group phasor rot(p_g, d_q) (q = j % 4 + 1) and the
    sample's rotation add one rotation each: model x_j s d_4^g d_q, bound 2 sqrt2 u (g + 2) G_j |x_j|.
  * shift_math: y = rot(s_j, x_j), model x_j s_j, bound 2 sqrt2 u |x_j| G_0.  shift_table: the same with the table entry t_j.
  * shift_unroll: p = rot(s, t_j), y = rot(p, x_j): model x_j s t_j, bound 4 sqrt2 u G_1 |x_j|.
  * decimating: the recursion over produced outputs m: model x_pos s d^m, the shift_addition bound at j = m.
A chunk whose seed is ambiguous adds sqrt2 u G_j |x_j| (one float ulp of each seed component, both below 1 in magnitude).  Every bound
carries MARGIN = 1 + 1e-3 for second-order terms and the float64 model's own rounding.  The inputs carry unit impulses at every chunk
start and end, where j is 0 and largest, so the bound is met where it is tightest.

(4) Invariants, windows and refusals: a bank's channel equals the one-channel bank; in_stride 0 equals per-row copies; tight, padded and odd
output strides give the same bits and never touch the padding or rows outside the call; a permuted channel subset taken by pointer offset
gives the same bits; a stream cut into calls at chunk multiples (any cut for shift_math / shift_table) gives the same bits, and so do the
wrap-table chain and the direct chain, the sliced and the unsliced launches; NaN or Inf at sample i changes output i only, never the phase;
every refusal returns -1 without a launch and leaves phase_io alone.

The checks talk to the C ABI through a driver with dev(array) -> buffer, ptr(buffer), host(buffer) -> array, `L` (argtypes set by
csdr_b200.lib()), `stream` and `pkg` (the csdr_b200 module, for the drop-ins), so the same bodies run on the GPU and on the emulated library.
"""
import ctypes as C
import ctypes.util
import itertools
import math
import os

import numpy as np

from bitcmp import SENTINEL, U, assert_bits_equal

F32 = np.float32
PI = F32(math.pi)                                                    # the reference's PI as a float
MARGIN = 1 + 1e-3
SQ2 = math.sqrt(2.0)
AMBIG_ULPS = 4
MATH_SEG = 256
WRAP_TABLE_MIN_STEPS = 96                                            # kWrapTableMinSteps: more chunks than this -> the wrap-table chain
MAX_SLICES = 3
PRODUCT_SLICE_MIN = 768 * 64
KINDS = ("cc", "fc", "addfast", "math", "table", "unroll")
BLOCK = 1 << 21                                                      # samples per block of channels in the host restatement


# ================================================================================================================ case matrix
RATES = [0.0, 1e-7, -1e-7, 0.085, -0.085, 0.25, -0.25, 0.4999, -0.4999, 0.5, -0.5, 0.75, -1.3]     # |rate| > 0.5: the init takes any rate
PHASES = [PI, -PI, np.nextafter(PI, F32(0)), np.nextafter(PI, F32(4)), np.nextafter(-PI, F32(0)), np.nextafter(-PI, F32(-4)), 100.0, -7.5,
          6.2831855, 0.0, 1.0, -2.0, 3.0]


def rates_phases(ch, shift=0):
    r = [RATES[(i + shift) % len(RATES)] for i in range(ch)]
    p = [PHASES[(i + 3 * shift) % len(PHASES)] for i in range(ch)]
    return np.array(r, F32), np.array(p, F32)


# (kind, channels, n, chunk, table size, input layout, output layout)
BANK_CASES = [
    ("cc", 13, 1, 0, None, "tight", "tight"), ("cc", 13, 1, 5, None, "pad", "odd"), ("cc", 13, 7, 0, None, "shared", "pad"),
    ("cc", 13, 200, 1, None, "tight", "odd"), ("cc", 13, 203, 2, None, "pad", "tight"), ("cc", 13, 301, 3, None, "tight", "pad"),
    ("cc", 13, 402, 4, None, "shared", "tight"), ("cc", 13, 503, 5, None, "tight", "tight"),
    ("cc", 13, 32 * 33 + 5, 31, None, "tight", "odd"), ("cc", 13, 32 * 32, 32, None, "pad", "pad"), ("cc", 13, 33 * 33, 33, None, "tight", "tight"),
    ("cc", 4, 8 * 127, 8, None, "tight", "tight"), ("cc", 4, 8 * 128, 8, None, "tight", "odd"), ("cc", 4, 8 * 128 + 3, 8, None, "pad", "tight"),
    ("cc", 4, 16 * 96, 16, None, "tight", "tight"), ("cc", 4, 16 * 97, 16, None, "tight", "pad"),
    ("cc", 3, 3 * 1023 + 7, 1023, None, "tight", "tight"), ("cc", 3, 2048, 1024, None, "tight", "odd"), ("cc", 3, 2 * 1025, 1025, None, "pad", "tight"),
    ("cc", 6, 9003, 8, None, "tight", "tight"), ("cc", 6, 2 * 4001, 2, None, "tight", "odd"), ("cc", 60, 1000, 10, None, "pad", "tight"),
    ("fc", 13, 1, 0, None, "tight", "tight"), ("fc", 13, 1000, 7, None, "pad", "odd"), ("fc", 4, 16 * 97 + 1, 16, None, "shared", "tight"),
    ("fc", 6, 9003, 8, None, "tight", "pad"), ("fc", 6, 2 * 4001, 2, None, "tight", "tight"),
    ("addfast", 13, 1, 0, None, "tight", "tight"), ("addfast", 13, 3, 0, None, "tight", "tight"), ("addfast", 13, 1001, 0, None, "pad", "odd"),
    ("addfast", 13, 1000, 5, None, "tight", "tight"), ("addfast", 13, 997, 4, None, "shared", "pad"), ("addfast", 13, 300, 3, None, "tight", "tight"),
    ("addfast", 4, 33 * 97 + 2, 33, None, "tight", "odd"), ("addfast", 3, 3000, 1024, None, "tight", "tight"),
    ("math", 13, 1, 0, None, "tight", "tight"), ("math", 13, 255, 0, None, "pad", "odd"), ("math", 13, 256, 0, None, "tight", "tight"),
    ("math", 13, 257, 0, None, "shared", "pad"), ("math", 13, 4001, 0, None, "tight", "tight"), ("math", 3, 128 * 256 + 5, 0, None, "tight", "odd"),
    ("table", 13, 1, 0, 2, "tight", "tight"), ("table", 13, 257, 0, 100, "pad", "odd"), ("table", 13, 3000, 0, 1024, "tight", "tight"),
    ("table", 13, 2001, 0, 65536, "shared", "pad"),
    ("unroll", 13, 1, 0, 1, "tight", "tight"), ("unroll", 13, 100, 0, 5, "pad", "odd"), ("unroll", 13, 1000, 0, 32, "tight", "tight"),
    ("unroll", 13, 3000, 0, 1024, "shared", "pad"), ("unroll", 13, 50, 0, 1024, "tight", "tight"), ("unroll", 4, 4 * 97 + 1, 0, 4, "tight", "odd"),
]
# (kind, channels, n, chunk, table size): the exact invariants
INV_CASES = [("cc", 4, 16 * 97 + 3, 16, None), ("cc", 6, 9003, 8, None), ("cc", 3, 2 * 1025 + 1, 1024, None), ("fc", 6, 9003, 8, None),
             ("fc", 3, 1000, 0, None), ("addfast", 4, 7 * 100 + 2, 7, None), ("addfast", 3, 2049, 1024, None), ("math", 4, 3 * 256 + 17, 0, None),
             ("table", 4, 1001, 0, 1024), ("unroll", 4, 5 * 99 + 2, 0, 5), ("unroll", 3, 2000, 0, 1024)]
NONFINITE_CASES = [("cc", 1000, 64, None), ("fc", 1000, 64, None), ("addfast", 1002, 66, None), ("math", 600, 0, None), ("table", 600, 0, 1024),
                   ("unroll", 700, 0, 256)]
# (decimation, call sizes): remain >= n for the first call of the last two
DEC_CASES = [(1, [100, 7]), (3, [1000, 1, 2, 999]), (7, [10_007, 3]), (64, [5, 100, 5000]), (2, [0, 9, 4])]

DROPIN_CASES = [(3000, 1024, -0.085, -7.5), (777, 100, 0.31, 3.1415927), (5, 5, 0.5, 0.0)]     # (n, samples per call, rate, phase)


def case_id(c):
    return "-".join(str(v) for v in c if v is not None)


def launches(drv):
    return int(drv.L.csdrb_kernel_launches())


# ================================================================================================================ launcher restatement
def slice_min():
    """CSDRB_SHIFT_SLICE_MIN as launch_shift_bank reads it (atol; 0 or garbage -> 1), else the product default"""
    v = os.environ.get("CSDRB_SHIFT_SLICE_MIN")
    if v is None:
        return PRODUCT_SLICE_MIN
    try:
        v = int(v.strip().split()[0])
    except (ValueError, IndexError):
        v = 0
    return v if v > 0 else 1


def eff_chunk(n, chunk):
    return n if chunk <= 0 or chunk > n else chunk


def shift_path(channels, n, chunk, kind="cc"):
    """the launcher's choice for a call: chunk, nchunks, wrap-table chain or direct, side stream or not, the chain slices it launches (whole
    CTAs of 128 chunks each: a side-stream chain of at most 128 chunks is one slice), the kernel launches it counts"""
    if kind in ("math", "table"):
        nseg = -(-n // MATH_SEG)
        return dict(chunk=MATH_SEG, nchunks=nseg, table=False, side=False, slices=1, launches=2)
    chunk = eff_chunk(n, chunk)
    nchunks = -(-n // chunk)
    table = nchunks > WRAP_TABLE_MIN_STEPS
    slices, side = 1, False
    if kind in ("cc", "fc"):
        want = min(MAX_SLICES, nchunks * channels // slice_min())
        if want >= 2:
            side = True
            per = -(-(-(-nchunks // want)) // 128) * 128               # whole CTAs of 128 chunks per slice
            slices = sum(1 for i in range(want) if i * per < nchunks)
    return dict(chunk=chunk, nchunks=nchunks, table=table, side=side, slices=slices, launches=2 * slices)


# ================================================================================================================ parameters
def inc1(rate):
    """fl(fl(2 rate) PI): the per-sample increment of every shift chain"""
    return F32(F32(2) * F32(rate)) * PI


def make_params(oracle, kind, rates, tsize=None):
    """the per-channel parameter rows each entry point takes, and (for unroll) its tables"""
    rates = np.asarray(rates, F32)
    if kind in ("math", "table"):
        return rates.copy(), None
    if kind == "addfast":
        return np.stack([oracle.shift_addfast_init(float(r)) for r in rates]).astype(F32), None
    prm = np.array([oracle.shift_addition_init(float(r)) for r in rates], F32)
    if kind != "unroll":
        return prm, None
    tabs = np.empty((2, rates.size, tsize), F32)
    fp = C.POINTER(C.c_float)
    for c, r in enumerate(rates):
        oracle.L.oracle_shift_unroll_init(float(r), tsize, tabs[0, c].ctypes.data_as(fp), tabs[1, c].ctypes.data_as(fp))
    return prm, tabs                                                 # tabs[0] = dsin, tabs[1] = dcos


def table_of(oracle, tsize):
    return oracle.shift_table_init(tsize)


# ================================================================================================================ inputs
def make_input(kind, ch, n, seg, seed, shared=False):
    """uniform noise with unit impulses at every segment's first and last sample (where the bound is tightest); one row if shared"""
    rng = np.random.default_rng(seed)
    rows = 1 if shared else ch
    if kind == "fc":
        x = rng.uniform(-1, 1, (rows, n)).astype(F32)
        imp = F32(1)
    else:
        x = (rng.uniform(-1, 1, (rows, n)) + 1j * rng.uniform(-1, 1, (rows, n))).astype(np.complex64)
        imp = np.complex64(1)
    if n:
        starts = np.arange(0, n, max(seg, 1))
        x[:, starts] = imp
        x[:, np.minimum(starts + seg - 1, n - 1)] = -imp
    return np.repeat(x, ch, axis=0) if shared else x


# ================================================================================================================ one call through the C ABI
def _sentinel(rows, cols, dtype):
    w = np.full((rows, cols * (2 if dtype == np.complex64 else 1)), SENTINEL, np.uint32)
    return w.view(F32).view(dtype) if dtype == np.complex64 else w.view(F32)


def out_stride_of(n, layout):
    return {"tight": max(n, 1), "pad": n + 4, "odd": n + (1 if n % 2 == 0 else 2)}[layout]


def written_mask(kind, n, chunk, ch, rows, stride):
    """which output entries a call writes: every sample, but for addfast only whole groups of four of each call"""
    m = np.zeros((rows, stride), bool)
    if kind == "addfast":
        chunk = eff_chunk(n, chunk)
        w = np.zeros(n, bool)
        for s in range(0, n, chunk):
            w[s:s + ((min(chunk, n - s)) & ~3)] = True
        m[:ch, :n] = w
    else:
        m[:ch, :n] = True
    return m


def call_bank(drv, kind, x, prm, ph0, n, chunk=0, aux=None, in_layout="tight", out_layout="tight", c0=0, ch=None, scratch_bytes=None,
              expect_rc=None):
    """csdrb_<kind>_bank on channels c0 .. c0 + ch - 1 of the host arrays x [C, n] (or one row for in_layout "shared"), prm [C, ...], ph0 [C],
    each taken by pointer offset.  Returns dict(y [ch, n], phase [ch], scratch (bytes), rc, launched, full output buffer, its mask)."""
    C_all = prm.shape[0]
    ch = C_all - c0 if ch is None else ch
    cplx = kind != "fc"
    itemsize = 8 if cplx else 4
    if in_layout == "shared":
        xb, in_stride = np.ascontiguousarray(x[:1]), 0
    elif in_layout == "pad":
        in_stride = n + 3
        xb = np.full((C_all, in_stride), np.nan, x.dtype)
        xb[:, :n] = x
    else:
        in_stride, xb = n, np.ascontiguousarray(x)
    ostride = out_stride_of(n, out_layout)
    ob = _sentinel(C_all + 1, ostride, np.complex64)
    dx, do, dp, dph = drv.dev(xb), drv.dev(ob), drv.dev(np.ascontiguousarray(prm)), drv.dev(np.ascontiguousarray(ph0, F32))
    L = drv.L
    if kind in ("math", "table"):
        sb = int(L.csdrb_shift_math_bank_scratch_bytes(ch, n))
    else:
        sb = int(L.csdrb_shift_addition_bank_scratch_bytes(ch, n, aux[1].shape[-1] if kind == "unroll" else chunk))
    sb = sb if scratch_bytes is None else scratch_bytes
    ds = drv.dev(np.full(max(sb, 4) + 64, 0xA5, np.uint8))
    px = drv.ptr(dx) + (0 if in_stride == 0 else c0 * in_stride * itemsize)
    po = drv.ptr(do) + c0 * ostride * 8
    pp = drv.ptr(dp) + c0 * prm.strides[0] if prm.ndim > 1 else drv.ptr(dp) + c0 * 4
    pph = drv.ptr(dph) + 4 * c0
    n0 = launches(drv)
    if kind in ("cc", "fc"):
        fn = L.csdrb_shift_addition_bank_cc if kind == "cc" else L.csdrb_shift_addition_bank_fc
        rc = fn(px, in_stride, po, ostride, ch, n, pp, pph, chunk, drv.ptr(ds), sb, drv.stream)
    elif kind == "addfast":
        rc = L.csdrb_shift_addfast_bank_cc(px, in_stride, po, ostride, ch, n, pp, pph, chunk, drv.ptr(ds), sb, drv.stream)
    elif kind == "math":
        rc = L.csdrb_shift_math_bank_cc(px, in_stride, po, ostride, ch, n, pp, pph, drv.ptr(ds), sb, drv.stream)
    elif kind == "table":
        dt = drv.dev(aux)
        rc = L.csdrb_shift_table_bank_cc(px, in_stride, po, ostride, ch, n, pp, pph, drv.ptr(dt), aux.size, drv.ptr(ds), sb, drv.stream)
    else:
        tabs = np.ascontiguousarray(aux[1])
        dtb = drv.dev(tabs)
        tstride = tabs.shape[-1]
        rc = L.csdrb_shift_unroll_bank_cc(px, in_stride, po, ostride, ch, n, pp, drv.ptr(dtb) + 4 * c0 * tstride,
                                          drv.ptr(dtb) + 4 * (tabs.shape[1] + c0) * tstride, tstride, tstride, pph, drv.ptr(ds), sb, drv.stream)
    launched = launches(drv) - n0
    if expect_rc is None:
        assert rc >= 0, drv.L.csdrb_last_error()
    else:
        assert rc == expect_rc, (rc, expect_rc, drv.L.csdrb_last_error())
    got = drv.host(do).reshape(C_all + 1, ostride)
    ph = drv.host(dph)
    scratch = drv.host(ds)
    # rows c0 .. c0 + ch - 1 are the call's; everything else, and the unwritten samples of its rows, keep the sentinel
    mask = np.zeros(got.shape, bool)
    if launched > 0:
        mask[c0:c0 + ch] = written_mask(kind, n, chunk, ch, ch, ostride)
    w = got.view(np.uint32).reshape(C_all + 1, ostride, 2)
    bad = ~np.all(w == SENTINEL, axis=-1) & ~mask
    assert not bad.any(), f"{kind}: a store outside the outputs at {tuple(np.argwhere(bad)[0])}"
    return dict(y=np.ascontiguousarray(got[c0:c0 + ch, :n]), phase=ph[c0:c0 + ch], phase_all=ph, scratch=scratch, rc=rc, launched=launched,
                mask=mask[c0:c0 + ch, :n])


# ================================================================================================================ restatements
def _rot(pc, ps, xr, xi):
    """rotate_rn((pc, ps), (xr, xi)) in float32: two rounded products, a rounded difference / sum per component"""
    return pc * xr - ps * xi, ps * xr + pc * xi


def _planes(Y):
    return Y.view(F32).reshape(Y.shape + (2,))


def mix_addition(X, seed, d, fc=False):
    """the shift_bank_kernel recursion over the last axis of X [..., L]; seed [..., 2] (cos, sin); d [..., 2] (cosd, sind), broadcastable"""
    pc, ps = seed[..., 0].astype(F32), seed[..., 1].astype(F32)
    dc, ds = d[..., 0].astype(F32), d[..., 1].astype(F32)
    Y = np.empty(X.shape, np.complex64)
    P = _planes(Y)
    with np.errstate(all="ignore"):
        for j in range(X.shape[-1]):
            if fc:
                xr = X[..., j]
                P[..., j, 0], P[..., j, 1] = pc * xr, ps * xr
            else:
                P[..., j, 0], P[..., j, 1] = _rot(pc, ps, X[..., j].real, X[..., j].imag)
            pc, ps = _rot(pc, ps, dc, ds)
    return Y


def mix_addfast(X, seed, dq):
    """shift_addfast_bank_kernel: groups of four; dq [..., 4, 2] = (dcos, dsin) of 1..4 increments; X's last axis a multiple of 4"""
    pc, ps = seed[..., 0].astype(F32), seed[..., 1].astype(F32)
    Y = np.empty(X.shape, np.complex64)
    P = _planes(Y)
    with np.errstate(all="ignore"):
        for g in range(X.shape[-1] // 4):
            gs = [_rot(pc, ps, dq[..., q, 0], dq[..., q, 1]) for q in range(4)]
            for q in range(4):
                j = 4 * g + q
                P[..., j, 0], P[..., j, 1] = _rot(gs[q][0], gs[q][1], X[..., j].real, X[..., j].imag)
            pc, ps = gs[3]
    return Y


def mix_each(X, seeds):
    """one rotation per sample by its own phasor (shift_math: the seed; shift_table: the table pair)"""
    Y = np.empty(X.shape, np.complex64)
    P = _planes(Y)
    with np.errstate(all="ignore"):
        P[..., 0], P[..., 1] = _rot(seeds[..., 0], seeds[..., 1], X.real, X.imag)
    return Y


def mix_unroll(X, seed, tc, ts):
    """shift_unroll_bank_kernel: p = rot(seed, (dcos[j], dsin[j])), y = rot(p, x); X [..., L], seed [..., 2], tc/ts [..., L]"""
    with np.errstate(all="ignore"):
        pc, ps = _rot(seed[..., 0:1], seed[..., 1:2], tc, ts)
    return mix_each(X, np.stack([pc, ps], -1))


def _eq(a, b):
    """bit equality per complex sample where both are numbers; NaN matches NaN (the payload is the platform's)"""
    A, B = _planes(np.ascontiguousarray(a)), _planes(np.ascontiguousarray(b))
    return np.all((A.view(np.uint32) == B.view(np.uint32)) | (np.isnan(A) & np.isnan(B)), axis=-1)


def _candidates(seed, alt):
    """every seed the device may have used: each ambiguous component rounded either way"""
    out = []
    for cc, ss in itertools.product({float(seed[0]), float(alt[0])}, {float(seed[1]), float(alt[1])}):
        out.append(np.array([cc, ss], F32))
    return out


def within(got, model, bnd, what):
    err = np.abs(got.astype(np.complex128) - model)
    ok = err <= bnd
    if not np.all(ok):
        i = tuple(np.argwhere(~ok)[0])
        raise AssertionError(f"{what}: sample {i} errs by {err[i]:.3e}, bound {bnd[i]:.3e} ({np.count_nonzero(~ok)} outside)")
    return float((err / np.where(bnd > 0, bnd, 1)).max()) if err.size else 0.0


def _chunked(a, nchunks, seg, fill=0):
    """[ch, n] -> [ch, nchunks, seg], the short last chunk padded"""
    ch, n = a.shape
    b = np.full((ch, nchunks * seg), fill, a.dtype)
    b[:, :n] = a
    return b.reshape(ch, nchunks, seg)


# ================================================================================================================ the main check
def expected_chain(oracle, kind, rates, ph0, n, chunk, tsize=None):
    """(per-chunk / per-segment start phases [ch, nchunks], per-sample phases for math/table or None, carried phase [ch]) from the oracle"""
    ch = len(rates)
    if kind in ("math", "table"):
        per = np.empty((ch, n), F32)
        end = np.empty(ch, F32)
        for c in range(ch):
            per[c], end[c] = oracle.shift_math_phases(float(rates[c]), float(ph0[c]), n)
        return np.ascontiguousarray(per[:, ::MATH_SEG]), per, end
    seg = eff_chunk(n, tsize if kind == "unroll" else chunk)
    nchunks = -(-n // seg)
    starts = np.empty((ch, nchunks), F32)
    end = np.empty(ch, F32)
    for c in range(ch):
        inc = oracle.shift_addfast_init(float(rates[c]))[8] if kind == "addfast" else inc1(rates[c])
        starts[c], end[c] = oracle.shift_chain(float(inc), float(ph0[c]), n, seg)
    return starts, None, end


def check_samples(oracle, kind, x, y, prm, aux, rates, ph0, n, chunk, phases=None, tsize=None, what=""):
    """(2) and (3) on y [ch, n] (finite or not): returns (ambiguous seeds met, worst err/bound).  phases: from expected_chain."""
    with np.errstate(invalid="ignore", over="ignore"):
        return _check_samples(oracle, kind, x, y, prm, aux, rates, ph0, n, chunk, phases, tsize, what)


def _check_samples(oracle, kind, x, y, prm, aux, rates, ph0, n, chunk, phases, tsize, what):
    ch = x.shape[0]
    starts, per, _ = phases
    amb_total, worst = 0, 0.0
    if kind in ("math", "table"):
        step = max(1, BLOCK // max(n, 1))
        for a in range(0, ch, step):
            b = min(ch, a + step)
            X, Y = x[a:b], y[a:b]
            if kind == "math":
                seeds, alt, k = oracle.seed_phasors(per[a:b], AMBIG_ULPS)
            else:
                seeds = alt = np.stack([_table_pairs(oracle, aux, rates[c], ph0[c], n) for c in range(a, b)]).astype(F32)
                k = 0
            if kind == "math":
                want = mix_each(X, seeds)
            else:                                                        # no cos in shift_table: the oracle's bits (the pairs above lose the sign of a zero)
                want = np.stack([oracle.shift_table_cc(X[c], float(rates[a + c]), aux, float(ph0[a + c]))[0] for c in range(b - a)])
            eq = _eq(Y, want)
            amb = np.any(seeds != alt, axis=-1)
            bad = ~eq & ~amb
            if bad.any():
                i = tuple(np.argwhere(bad)[0])
                raise AssertionError(f"{what}: sample {(i[0] + a, i[1])} differs from the restatement ({np.count_nonzero(bad)} samples)")
            for i in np.argwhere(amb & ~eq):
                cands = [mix_each(X[tuple(i)][None], s[None])[0] for s in _candidates(seeds[tuple(i)], alt[tuple(i)])]
                assert any(_eq(Y[tuple(i)][None], c[None])[0] for c in cands), f"{what}: sample {(i[0] + a, i[1])} matches no rounding of its seed"
            amb_total += int(np.count_nonzero(amb))
            fin = np.isfinite(X) & np.isfinite(Y)
            model = X.astype(np.complex128) * (seeds[..., 0].astype(np.float64) + 1j * seeds[..., 1].astype(np.float64))
            mag = np.abs(X.astype(np.complex128)) * np.abs(seeds[..., 0].astype(np.float64) + 1j * seeds[..., 1])
            bnd = (2 * SQ2 * U * (1 + U) * mag + amb * SQ2 * U * np.abs(X)) * (1 + 8 * U) * MARGIN
            worst = max(worst, within(Y[fin], model[fin], bnd[fin], what + ": float64 bound"))
        return amb_total, worst
    # chunked kinds: one seed per chunk
    seg = eff_chunk(n, tsize if kind == "unroll" else chunk)
    nchunks = starts.shape[1]
    step = max(1, BLOCK // max(nchunks * seg, 1))
    for a in range(0, ch, step):
        b = min(ch, a + step)
        fill = F32(0) if kind == "fc" else np.complex64(0)
        X = _chunked(x[a:b], nchunks, seg, fill)
        Y = _chunked(y[a:b], nchunks, seg, np.complex64(0))
        seeds, alt, k = oracle.seed_phasors(starts[a:b], AMBIG_ULPS)
        lens = np.minimum(seg, n - np.arange(nchunks) * seg)
        valid = np.arange(seg)[None, :] < lens[:, None]                       # [nchunks, seg]
        if kind == "addfast":
            valid &= np.arange(seg)[None, :] < (lens[:, None] & ~3)

        def restate(Xs, S, c_idx):
            if kind in ("cc", "fc"):
                d = np.stack([prm[c_idx, 1], prm[c_idx, 0]], -1)[..., None, :]  # (cosd, sind), one per channel
                return mix_addition(Xs, S, d, fc=kind == "fc")
            if kind == "addfast":
                dq = np.stack([prm[c_idx, 4:8], prm[c_idx, 0:4]], -1)[..., None, :, :]
                L4 = Xs.shape[-1] & ~3
                out = np.zeros(Xs.shape, np.complex64)
                out[..., :L4] = mix_addfast(Xs[..., :L4], S, dq)
                return out
            ts, tc = aux[1][0][c_idx][..., None, :seg], aux[1][1][c_idx][..., None, :seg]
            return mix_unroll(Xs, S, tc, ts)

        cidx = np.arange(a, b)
        want = restate(X, seeds, cidx)
        eq = _eq(Y, want) | ~valid
        chunk_ok = eq.all(-1)
        amb = np.any(seeds != alt, axis=-1)
        bad = ~chunk_ok & ~amb
        if bad.any():
            c, kk = np.argwhere(bad)[0]
            j = int(np.flatnonzero(~eq[c, kk])[0])
            raise AssertionError(f"{what}: channel {c + a} chunk {kk} sample {j} differs from the restatement ({np.count_nonzero(bad)} chunks)")
        for c, kk in np.argwhere(amb & ~chunk_ok):
            ok = False
            for s in _candidates(seeds[c, kk], alt[c, kk]):
                w1 = restate(X[c, kk][None, None], s[None, None], np.array([c + a]))[0, 0]
                ok = ok or bool(np.all(_eq(Y[c, kk], w1) | ~valid[kk]))
            assert ok, f"{what}: channel {c + a} chunk {kk} matches no rounding of its ambiguous seed"
        amb_total += int(np.count_nonzero(amb))
        # float64 model and bound
        S = seeds[..., 0].astype(np.float64) + 1j * seeds[..., 1].astype(np.float64)        # [blk, nchunks]
        Xd = X.astype(np.complex128)
        j = np.arange(seg)
        if kind in ("cc", "fc"):
            d = prm[a:b, 1].astype(np.float64) + 1j * prm[a:b, 0].astype(np.float64)
            Dp = d[:, None] ** j[None, :]                                       # exact enough: |rounding| ~ j 2^-53
            model = Xd * S[..., None] * Dp[:, None, :]
            G = 1 + 4 * (j + 2) * U
            coef = (2 * SQ2 * (j + 1)) if kind == "cc" else (2 * SQ2 * j + 1)
        elif kind == "addfast":
            d4 = prm[a:b, 7].astype(np.float64) + 1j * prm[a:b, 3].astype(np.float64)
            dq = prm[a:b, 4:8].astype(np.float64) + 1j * prm[a:b, 0:4].astype(np.float64)
            g = j // 4
            model = Xd * S[..., None] * (d4[:, None] ** g[None, :] * dq[:, j % 4])[:, None, :]
            G = 1 + 4 * (g + 3) * U
            coef = 2 * SQ2 * (g + 2)
        else:
            T = aux[1][1][a:b, :seg].astype(np.float64) + 1j * aux[1][0][a:b, :seg].astype(np.float64)
            model = Xd * S[..., None] * T[:, None, :]
            G = 1 + 8 * U
            coef = 4 * SQ2 * np.ones(seg)
        absx = np.abs(Xd)
        bnd = (coef * G * U * absx + amb[..., None] * SQ2 * U * G * absx) * MARGIN
        fin = valid[None] & np.isfinite(X) & np.isfinite(Y)
        worst = max(worst, within(Y[fin], model[fin], bnd[fin], what + ": float64 bound"))
    return amb_total, worst


def _table_pairs(oracle, table, rate, ph0, n):
    """the (cos, sin) table pair shift_table_cc applies to each sample: its output for x = 1"""
    ones = np.ones(n, np.complex64)
    y, _, _ = oracle.shift_table_cc(ones, float(rate), table, float(ph0))
    return np.stack([y.real, y.imag], -1)


def check_bank(drv, oracle, kind, rates, ph0, n, chunk=0, tsize=None, in_layout="tight", out_layout="tight", seed=0, x=None):
    """one call of a bank: path and launch count, phase chains (1), samples (2), bound (3), padding.  Returns (ambiguous seeds, worst ratio)."""
    rates = np.asarray(rates, F32)
    ph0 = np.asarray(ph0, F32)
    ch = rates.size
    prm, tabs = make_params(oracle, kind, rates, tsize)
    aux = table_of(oracle, tsize) if kind == "table" else (None, tabs)
    seg = MATH_SEG if kind in ("math", "table") else eff_chunk(n, tsize if kind == "unroll" else chunk)
    if x is None:
        x = make_input(kind, ch, n, seg, seed, shared=in_layout == "shared")
    path = shift_path(ch, n, tsize if kind == "unroll" else chunk, kind)
    r = call_bank(drv, kind, x, prm, ph0, n, chunk, aux, in_layout, out_layout, expect_rc=0)
    assert r["launched"] == path["launches"], (r["launched"], path)
    what = f"{kind} ch={ch} n={n} chunk={chunk} {in_layout}/{out_layout}"
    phases = expected_chain(oracle, kind, rates, ph0, n, chunk, tsize)
    starts = phases[0]
    got_starts = r["scratch"][:starts.size * 4].view(F32).reshape(starts.shape)
    assert_bits_equal(got_starts, starts, what + ": chunk / segment start phases")
    assert_bits_equal(r["phase"], phases[2], what + ": carried phase")
    if kind == "cc" and ch <= 8 and n <= 1 << 16:
        for c in range(ch):                                              # the restatement is the oracle's operation (both seed with the host's libm)
            want, _ = oracle.shift_addition_cc(x[c], float(rates[c]), float(ph0[c]), seg)
            mine = mix_addition(_chunked(x[c:c + 1], starts.shape[1], seg, np.complex64(0)), oracle.seed_phasors(starts[c:c + 1])[0],
                                np.array([prm[c, 1], prm[c, 0]], F32))
            assert_bits_equal(mine.reshape(-1)[:n], want, what + ": restatement = oracle")
    amb, worst = check_samples(oracle, kind, x, r["y"], prm, aux, rates, ph0, n, chunk, phases, tsize, what)
    return amb, worst


# ================================================================================================================ invariants
def check_invariants(drv, oracle, kind, rates, ph0, n, chunk=0, tsize=None, seed=0, cuts=None):
    """exact invariants of one bank: channel = one-channel bank (whatever either's slicing), in_stride 0 = copies, output strides, a permuted
    subset by pointer offset, a stream cut into calls (chunk multiples; any cut for math/table), the table chain = the direct chain.
    Returns the set of paths the calls took."""
    rates = np.asarray(rates, F32)
    ph0 = np.asarray(ph0, F32)
    ch = rates.size
    prm, tabs = make_params(oracle, kind, rates, tsize)
    aux = table_of(oracle, tsize) if kind == "table" else (None, tabs)
    ck = tsize if kind == "unroll" else chunk
    seg = MATH_SEG if kind in ("math", "table") else eff_chunk(n, ck)
    x = make_input(kind, ch, n, seg, seed)
    paths = {("bank",) + tuple(sorted(shift_path(ch, n, ck, kind).items()))}
    base = call_bank(drv, kind, x, prm, ph0, n, chunk, aux)
    what = f"{kind} ch={ch} n={n} chunk={chunk}"
    # one channel at a time
    for c in range(ch):
        one = call_bank(drv, kind, x, prm, ph0, n, chunk, aux, c0=c, ch=1)
        assert_bits_equal(one["y"][0], base["y"][c], f"{what}: channel {c} alone")
        assert_bits_equal(one["phase"], base["phase"][c:c + 1], f"{what}: channel {c} alone, phase")
        paths.add(("one",) + tuple(sorted(shift_path(1, n, ck, kind).items())))
    # output strides
    for lay in ("pad", "odd"):
        r = call_bank(drv, kind, x, prm, ph0, n, chunk, aux, out_layout=lay)
        assert_bits_equal(r["y"], base["y"], f"{what}: out stride {lay}")
    r = call_bank(drv, kind, x, prm, ph0, n, chunk, aux, in_layout="pad")
    assert_bits_equal(r["y"], base["y"], f"{what}: padded input rows")
    # in_stride 0 = per-row copies of one row
    xs = np.repeat(x[:1], ch, axis=0)
    a = call_bank(drv, kind, xs, prm, ph0, n, chunk, aux, in_layout="shared")
    b = call_bank(drv, kind, xs, prm, ph0, n, chunk, aux)
    assert_bits_equal(a["y"], b["y"], f"{what}: in_stride 0")
    # a permuted subset by pointer offset
    if ch > 1:
        perm = np.random.default_rng(seed + 1).permutation(ch)
        auxp = aux if kind != "unroll" else (None, np.ascontiguousarray(tabs[:, perm]))
        r = call_bank(drv, kind, x[perm], prm[perm], ph0[perm], n, chunk, auxp, c0=1)
        assert_bits_equal(r["y"], base["y"][perm[1:]], f"{what}: permuted subset")
        assert_bits_equal(r["phase"], base["phase"][perm[1:]], f"{what}: permuted subset, phase")
    # a stream cut into calls with the phase carried
    bounds = _cuts(kind, n, seg, cuts)
    ph = ph0.copy()
    parts = []
    for s, e in zip(bounds[:-1], bounds[1:]):
        xp = np.ascontiguousarray(x[:, s:e])
        r = call_bank(drv, kind, xp, prm, ph, e - s, chunk, aux)
        parts.append(r["y"])
        ph = r["phase"].copy()
        paths.add(("cut",) + tuple(sorted(shift_path(ch, e - s, ck, kind).items())))
    assert_bits_equal(np.concatenate(parts, axis=1), base["y"], f"{what}: cut at {bounds}")
    assert_bits_equal(ph, base["phase"], f"{what}: cut, carried phase")
    return paths


def _cuts(kind, n, seg, cuts):
    """call boundaries: at most 96 chunks per call (the direct chain) for the chunked kinds, uneven cuts for math/table"""
    if kind in ("math", "table"):
        pts = sorted({0, n} | {c for c in (cuts or (1, n // 3 + 7, n - 1)) if 0 < c < n})
        return pts
    step = seg * (cuts or WRAP_TABLE_MIN_STEPS)
    return list(range(0, n, step)) + [n]


# ================================================================================================================ non-finite input
def check_nonfinite(drv, oracle, kind, n, chunk=0, tsize=None, seed=0):
    """NaN, +Inf, -Inf at sample i change output i only (both components as the restatement says), never the carried phase"""
    rates = np.array([0.0, 0.125, -0.3], F32)
    ph0 = np.array([0.0, 1.0, -2.5], F32)                               # rate 0 from phase 0: the seed (1, 0), a zero component for fc's Inf
    ch = rates.size
    prm, tabs = make_params(oracle, kind, rates, tsize)
    aux = table_of(oracle, tsize) if kind == "table" else (None, tabs)
    seg = MATH_SEG if kind in ("math", "table") else eff_chunk(n, tsize if kind == "unroll" else chunk)
    x = make_input(kind, ch, n, seg, seed)
    clean = call_bank(drv, kind, x, prm, ph0, n, chunk, aux)
    pos = sorted({0, 1, seg - 1, seg, n // 2, n - 1} & set(range(n)))
    if kind == "addfast":
        pos = [p for p in pos if clean["mask"][0, p]]
    bad = np.array([np.nan, np.inf, -np.inf], F32)
    xp = x.copy()
    for c in range(ch):
        for i, p in enumerate(pos):
            v = bad[(c + i) % 3]
            if kind == "fc":
                xp[c, p] = v
            else:
                xp[c, p] = complex(v, 0.5) if i % 2 else complex(0.25, v)
    r = call_bank(drv, kind, xp, prm, ph0, n, chunk, aux)
    assert_bits_equal(r["phase"], clean["phase"], f"{kind} non-finite: carried phase")
    hit = np.zeros(n, bool)
    hit[pos] = True
    for c in range(ch):
        assert_bits_equal(r["y"][c][~hit], clean["y"][c][~hit], f"{kind} non-finite: channel {c} away from the poisoned samples")
        assert not np.isfinite(r["y"][c][hit]).all(), (kind, c)
    phases = expected_chain(oracle, kind, rates, ph0, n, chunk, tsize)
    check_samples(oracle, kind, xp, r["y"], prm, aux, rates, ph0, n, chunk, phases, tsize, f"{kind} non-finite")
    if kind == "fc":                                                    # channel 0 keeps the phasor (1, 0): Inf x 0 = NaN, so +-Inf -> (+-Inf, NaN)
        for i, p in enumerate(pos):
            if np.isinf(xp[0, p]):
                assert r["y"][0, p].real == xp[0, p] and np.isnan(r["y"][0, p].imag), (p, r["y"][0, p])


# ================================================================================================================ decimating
def check_decimating(drv, oracle, rates, ph0, remain0, dec, sizes, seed=0):
    """a stream cut into calls of `sizes`: the state {remain, phase, output_size} after every call bit for bit, the outputs of each call
    bit for bit (one seed per call) and within the recursion's bound; rows past output_size untouched"""
    rates = np.asarray(rates, F32)
    ch = rates.size
    prm = np.empty((ch, 3), F32)
    d = [oracle.L.oracle_decimating_shift_addition_init(float(r), dec) for r in rates]
    for c in range(ch):
        prm[c] = (d[c].sindelta, d[c].cosdelta, d[c].rate)
    rng = np.random.default_rng(seed)
    total = sum(sizes)
    x = (rng.uniform(-1, 1, (ch, total)) + 1j * rng.uniform(-1, 1, (ch, total))).astype(np.complex64)
    remain = np.asarray(remain0, np.int32).copy()
    ph = np.asarray(ph0, F32).copy()
    L = drv.L
    s0, amb_total, worst = 0, 0, 0.0
    from oracle.pyoracle import _DShiftStatus, _CF, _p
    for n in sizes:
        xc = np.ascontiguousarray(x[:, s0:s0 + n]) if n else np.zeros((ch, 1), np.complex64)
        ostride = n // dec + 3
        dx, do = drv.dev(xc), drv.dev(_sentinel(ch + 1, ostride, np.complex64))
        dp, drm, dph = drv.dev(prm), drv.dev(remain), drv.dev(ph)
        dsz = drv.dev(np.full(ch + 1, -7, np.int32))
        n0 = launches(drv)
        rc = L.csdrb_decimating_shift_addition_bank_cc(drv.ptr(dx), xc.shape[1], drv.ptr(do), ostride, ch, n, drv.ptr(dp), dec, drv.ptr(drm),
                                                       drv.ptr(dph), drv.ptr(dsz), drv.stream)
        assert rc == 0 and launches(drv) - n0 == 1, (rc, L.csdrb_last_error())
        got, g_rm, g_ph, g_sz = drv.host(do).reshape(ch + 1, ostride), drv.host(drm), drv.host(dph), drv.host(dsz)
        assert g_sz[ch] == -7, "output_size stored past the last channel"
        for c in range(ch):
            want = np.empty(n // dec + 2, np.complex64)
            st = oracle.L.oracle_decimating_shift_addition_cc(_p(xc[c], _CF), _p(want, _CF), n, d[c], dec, _DShiftStatus(int(remain[c]), float(ph[c]), 0))
            what = f"decimating dec={dec} call of {n}, channel {c}"
            assert (int(g_rm[c]), int(g_sz[c])) == (st.decimation_remain, st.output_size), (what, g_rm[c], g_sz[c], st.decimation_remain, st.output_size)
            assert_bits_equal(g_ph[c:c + 1], np.array([st.starting_phase], F32), what + ": phase")
            m = st.output_size
            w = got[c].view(np.uint32).reshape(ostride, 2)
            assert np.all(w[m:] == SENTINEL), what + ": a store past output_size"
            pos = int(remain[c]) + dec * np.arange(m)
            Xs = xc[c, pos] if m else np.zeros(0, np.complex64)
            seeds, alt, k = oracle.seed_phasors(ph[c:c + 1], AMBIG_ULPS)
            dd = np.array([prm[c, 1], prm[c, 0]], F32)
            cands = [seeds[0]] + ([s for s in _candidates(seeds[0], alt[0])] if k else [])
            ok = any(np.all(_eq(got[c, :m], mix_addition(Xs[None], s[None], dd)[0])) for s in cands)
            assert ok, what + ": outputs differ from the restatement"
            amb_total += k
            j = np.arange(m)
            S = seeds[0, 0].astype(np.float64) + 1j * seeds[0, 1].astype(np.float64)
            model = Xs.astype(np.complex128) * S * (dd[0].astype(np.float64) + 1j * dd[1].astype(np.float64)) ** j
            G = 1 + 4 * (j + 2) * U
            bnd = (2 * SQ2 * (j + 1) + (SQ2 if k else 0)) * G * U * np.abs(Xs.astype(np.complex128)) * MARGIN
            worst = max(worst, within(got[c, :m], model, bnd, what + ": float64 bound"))
        remain, ph = g_rm.copy(), g_ph.copy()
        s0 += n
    return amb_total, worst


# ================================================================================================================ refusals
def check_refusals(drv, oracle):
    """every refusal returns -1 without a launch and leaves phase_io and the output alone; nothing to do returns 0 without a launch"""
    L = drv.L
    n, ch = 64, 2
    x = make_input("cc", ch, n, 16, 1)
    xf = make_input("fc", ch, n, 16, 1)
    dx, dxf = drv.dev(x), drv.dev(xf)
    do = drv.dev(_sentinel(ch, n, np.complex64))
    prm = drv.dev(np.array([oracle.shift_addition_init(0.1)] * ch, F32))
    pf = drv.dev(np.stack([oracle.shift_addfast_init(0.1)] * ch))
    rates = drv.dev(np.array([0.1, -0.2], F32))
    ph_host = np.array([0.5, 4.0], F32)                                  # 4.0 > pi: a launch would wrap it
    ph = drv.dev(ph_host)
    table = drv.dev(oracle.shift_table_init(1024))
    tabs = drv.dev(np.ones((2, ch, 16), F32))
    rem = drv.dev(np.zeros(ch, np.int32))
    sb_add = int(L.csdrb_shift_addition_bank_scratch_bytes(ch, n, 16))
    sb_math = int(L.csdrb_shift_math_bank_scratch_bytes(ch, n))
    sc = drv.dev(np.zeros(max(sb_add, sb_math) + 64, np.uint8))
    P = drv.ptr
    S = drv.stream
    n0 = launches(drv)

    calls = []
    for fn, xin in ((L.csdrb_shift_addition_bank_cc, dx), (L.csdrb_shift_addition_bank_fc, dxf)):
        calls += [
            (-1, lambda fn=fn, xin=xin: fn(P(xin), n, P(do), n, ch, n, P(prm), P(ph), 16, P(sc), sb_add - 1, S)),         # scratch one byte short
            (-1, lambda fn=fn, xin=xin: fn(P(xin), n, P(do), n, ch, n, P(prm), P(ph), 16, None, sb_add, S)),
            (-1, lambda fn=fn: fn(None, n, P(do), n, ch, n, P(prm), P(ph), 16, P(sc), sb_add, S)),
            (-1, lambda fn=fn, xin=xin: fn(P(xin), n, None, n, ch, n, P(prm), P(ph), 16, P(sc), sb_add, S)),
            (-1, lambda fn=fn, xin=xin: fn(P(xin), n, P(do), n, ch, n, None, P(ph), 16, P(sc), sb_add, S)),
            (-1, lambda fn=fn, xin=xin: fn(P(xin), n, P(do), n, ch, n, P(prm), None, 16, P(sc), sb_add, S)),
            (-1, lambda fn=fn, xin=xin: fn(P(xin), 0, P(do), n, 65536, n, P(prm), P(ph), 16, P(sc), sb_add, S)),
            (0, lambda fn=fn, xin=xin: fn(P(xin), n, P(do), n, 0, n, P(prm), P(ph), 16, P(sc), sb_add, S)),
            (0, lambda fn=fn, xin=xin: fn(P(xin), n, P(do), n, ch, 0, P(prm), P(ph), 16, P(sc), sb_add, S)),
        ]
    fa = L.csdrb_shift_addfast_bank_cc
    calls += [
        (-1, lambda: fa(P(dx), n, P(do), n, ch, n, P(pf), P(ph), 16, P(sc), sb_add - 1, S)),
        (-1, lambda: fa(P(dx), n, P(do), n, ch, n, P(pf), P(ph), 16, None, sb_add, S)),
        (-1, lambda: fa(None, n, P(do), n, ch, n, P(pf), P(ph), 16, P(sc), sb_add, S)),
        (-1, lambda: fa(P(dx), n, P(do), n, ch, n, None, P(ph), 16, P(sc), sb_add, S)),
        (-1, lambda: fa(P(dx), n, P(do), n, ch, n, P(pf), None, 16, P(sc), sb_add, S)),
        (-1, lambda: fa(P(dx), 0, P(do), n, 65536, n, P(pf), P(ph), 16, P(sc), sb_add, S)),
        (0, lambda: fa(P(dx), n, P(do), n, 0, n, P(pf), P(ph), 16, P(sc), sb_add, S)),
        (0, lambda: fa(P(dx), n, P(do), n, ch, 0, P(pf), P(ph), 16, P(sc), sb_add, S)),
    ]
    fm, ft = L.csdrb_shift_math_bank_cc, L.csdrb_shift_table_bank_cc
    calls += [
        (-1, lambda: fm(P(dx), n, P(do), n, ch, n, P(rates), P(ph), P(sc), sb_math - 17, S)),    # scratch_bytes adds 16 bytes of slack
        (-1, lambda: fm(P(dx), n, P(do), n, ch, n, P(rates), P(ph), None, sb_math, S)),
        (-1, lambda: fm(None, n, P(do), n, ch, n, P(rates), P(ph), P(sc), sb_math, S)),
        (-1, lambda: fm(P(dx), n, None, n, ch, n, P(rates), P(ph), P(sc), sb_math, S)),
        (-1, lambda: fm(P(dx), n, P(do), n, ch, n, None, P(ph), P(sc), sb_math, S)),
        (-1, lambda: fm(P(dx), n, P(do), n, ch, n, P(rates), None, P(sc), sb_math, S)),
        (-1, lambda: fm(P(dx), 0, P(do), n, 65536, n, P(rates), P(ph), P(sc), sb_math, S)),
        (0, lambda: fm(P(dx), n, P(do), n, 0, n, P(rates), P(ph), P(sc), sb_math, S)),
        (0, lambda: fm(P(dx), n, P(do), n, ch, 0, P(rates), P(ph), P(sc), sb_math, S)),
        (-1, lambda: ft(P(dx), n, P(do), n, ch, n, P(rates), P(ph), P(table), 1024, P(sc), sb_math - 17, S)),
        (-1, lambda: ft(P(dx), n, P(do), n, ch, n, P(rates), P(ph), P(table), 1024, None, sb_math, S)),
        (-1, lambda: ft(P(dx), n, P(do), n, ch, n, P(rates), P(ph), None, 1024, P(sc), sb_math, S)),
        (-1, lambda: ft(P(dx), n, P(do), n, ch, n, P(rates), P(ph), P(table), 1, P(sc), sb_math, S)),   # table size < 2
        (-1, lambda: ft(P(dx), n, P(do), n, ch, n, P(rates), P(ph), P(table), 0, P(sc), sb_math, S)),
        (-1, lambda: ft(None, n, P(do), n, ch, n, P(rates), P(ph), P(table), 1024, P(sc), sb_math, S)),
        (-1, lambda: ft(P(dx), 0, P(do), n, 65536, n, P(rates), P(ph), P(table), 1024, P(sc), sb_math, S)),
        (0, lambda: ft(P(dx), n, P(do), n, 0, n, P(rates), P(ph), P(table), 1024, P(sc), sb_math, S)),
        (0, lambda: ft(P(dx), n, P(do), n, ch, 0, P(rates), P(ph), P(table), 1024, P(sc), sb_math, S)),
    ]
    fu = L.csdrb_shift_unroll_bank_cc
    sb_u = int(L.csdrb_shift_addition_bank_scratch_bytes(ch, n, 16))
    ts_ = P(tabs)
    tc_ = P(tabs) + 4 * ch * 16
    calls += [
        (-1, lambda: fu(P(dx), n, P(do), n, ch, n, P(prm), ts_, tc_, 16, 16, P(ph), P(sc), ch * 4 * 4 - 1, S)),   # [C][4 chunks] floats, one byte short
        (-1, lambda: fu(P(dx), n, P(do), n, ch, n, P(prm), ts_, tc_, 16, 16, P(ph), None, sb_u, S)),
        (-1, lambda: fu(P(dx), n, P(do), n, ch, n, P(prm), ts_, tc_, 16, 0, P(ph), P(sc), sb_u, S)),              # table size <= 0
        (-1, lambda: fu(P(dx), n, P(do), n, ch, n, P(prm), ts_, tc_, 16, -3, P(ph), P(sc), sb_u, S)),
        (-1, lambda: fu(None, n, P(do), n, ch, n, P(prm), ts_, tc_, 16, 16, P(ph), P(sc), sb_u, S)),
        (-1, lambda: fu(P(dx), n, P(do), n, ch, n, None, ts_, tc_, 16, 16, P(ph), P(sc), sb_u, S)),
        (-1, lambda: fu(P(dx), n, P(do), n, ch, n, P(prm), None, tc_, 16, 16, P(ph), P(sc), sb_u, S)),
        (-1, lambda: fu(P(dx), n, P(do), n, ch, n, P(prm), ts_, None, 16, 16, P(ph), P(sc), sb_u, S)),
        (-1, lambda: fu(P(dx), n, P(do), n, ch, n, P(prm), ts_, tc_, 16, 16, None, P(sc), sb_u, S)),
        (-1, lambda: fu(P(dx), 0, P(do), n, 65536, n, P(prm), ts_, tc_, 16, 16, P(ph), P(sc), sb_u, S)),
        (0, lambda: fu(P(dx), n, P(do), n, 0, n, P(prm), ts_, tc_, 16, 16, P(ph), P(sc), sb_u, S)),
        (0, lambda: fu(P(dx), n, P(do), n, ch, 0, P(prm), ts_, tc_, 16, 16, P(ph), P(sc), sb_u, S)),
    ]
    fd = L.csdrb_decimating_shift_addition_bank_cc
    calls += [
        (-1, lambda: fd(P(dx), n, P(do), n, ch, n, P(prm), 0, P(rem), P(ph), None, S)),                          # decimation <= 0
        (-1, lambda: fd(P(dx), n, P(do), n, ch, n, P(prm), -2, P(rem), P(ph), None, S)),
        (-1, lambda: fd(None, n, P(do), n, ch, n, P(prm), 3, P(rem), P(ph), None, S)),
        (-1, lambda: fd(P(dx), n, None, n, ch, n, P(prm), 3, P(rem), P(ph), None, S)),
        (-1, lambda: fd(P(dx), n, P(do), n, ch, n, None, 3, P(rem), P(ph), None, S)),
        (-1, lambda: fd(P(dx), n, P(do), n, ch, n, P(prm), 3, None, P(ph), None, S)),
        (-1, lambda: fd(P(dx), n, P(do), n, ch, n, P(prm), 3, P(rem), None, None, S)),
        (0, lambda: fd(P(dx), n, P(do), n, 0, n, P(prm), 3, P(rem), P(ph), None, S)),
    ]
    for i, (want, f) in enumerate(calls):
        rc = f()
        assert rc == want, (i, rc, want, L.csdrb_last_error())
        assert launches(drv) == n0, f"call {i} launched a kernel"
    assert_bits_equal(drv.host(ph), ph_host, "phase_io after the refusals")
    w = drv.host(do).view(np.uint32)
    assert np.all(w == SENTINEL), "a refused call wrote its output"
    assert np.all(drv.host(rem) == 0)
    return len(calls)


# ================================================================================================================ drop-ins
def _libm_sincosf(ph):
    libm = C.CDLL(ctypes.util.find_library("m"))
    s, c = C.c_float(), C.c_float()
    libm.sincosf.argtypes = [C.c_float, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    libm.sincosf(float(ph), C.byref(s), C.byref(c))
    return np.array([c.value, s.value], F32)


def check_dropins(drv, oracle, n, call, rate, phase, seed=0):
    """the libcsdr drop-ins, one call per `call` samples: bits of the bank restatement (shift_addition_fc from the host's sincosf seed, as the
    reference build seeds it) and of the oracle's carried phase"""
    lc = drv.pkg.libcsdr
    rng = np.random.default_rng(seed)
    x = (rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)).astype(np.complex64)
    xr = rng.uniform(-1, 1, n).astype(F32)
    amb = 0
    r = np.array([rate], F32)
    p = np.array([phase], F32)
    for kind, fn in (("cc", lambda: lc.shift_addition_cc(x, rate, phase, call)), ("math", lambda: lc.shift_math_cc(x, rate, phase, call)),
                     ("addfast", lambda: lc.shift_addfast_cc(x, rate, phase, call))):
        y, ph = fn()
        prm, _ = make_params(oracle, kind, r)
        phases = expected_chain(oracle, kind, r, p, n, call)
        assert_bits_equal(np.array([ph], F32), phases[2], f"drop-in {kind}: phase")
        if kind == "addfast":                                           # the drop-in leaves each call's n % 4 tail as it was (the wrapper: 0)
            m = written_mask("addfast", n, call, 1, 1, n)[0]
            assert np.all(y[~m] == 0), "drop-in addfast wrote a tail"
        a, _ = check_samples(oracle, kind, x[None], y[None], prm, None, r, p, n, call, phases, None, f"drop-in {kind}")
        amb += a
    # shift_unroll_cc: one call per table of `call` entries
    prm, tabs = make_params(oracle, "unroll", r, call)
    y, ph = lc.shift_unroll_cc(x, rate, phase, call)
    phases = expected_chain(oracle, "unroll", r, p, n, 0, call)
    assert_bits_equal(np.array([ph], F32), phases[2], "drop-in unroll: phase")
    a, _ = check_samples(oracle, "unroll", x[None], y[None], prm, (None, tabs), r, p, n, 0, phases, call, "drop-in unroll")
    amb += a
    # shift_table_cc: the oracle's bits
    table = oracle.shift_table_init(4096)
    y, ph = lc.shift_table_cc(x, rate, table, phase, call)
    want, wph, _ = oracle.shift_table_cc(x, rate, table, phase, call)
    assert_bits_equal(y, want, "drop-in table")
    assert_bits_equal(np.array([ph], F32), np.array([wph], F32), "drop-in table: phase")
    # shift_addition_fc: every call seeded with the host's sincosf of its start phase
    y, ph = lc.shift_addition_fc(xr, rate, phase, call)
    prm, _ = make_params(oracle, "fc", r)
    starts, _, end = expected_chain(oracle, "fc", r, p, n, call)
    assert_bits_equal(np.array([ph], F32), end, "drop-in fc: phase")
    seeds = np.stack([_libm_sincosf(s) for s in starts[0]])[None]
    nch = starts.shape[1]
    want = mix_addition(_chunked(xr[None], nch, call, F32(0)), seeds, np.array([prm[0, 1], prm[0, 0]], F32)).reshape(-1)[:n]
    assert_bits_equal(y, want, "drop-in fc: samples")
    # decimating_shift_addition_cc: state and samples of each call
    dec = 5
    st = (0, phase)
    d = oracle.L.oracle_decimating_shift_addition_init(rate, dec)
    dd = np.array([d.cosdelta, d.sindelta], F32)
    for s0 in range(0, n, call):
        xc = x[s0:s0 + call]
        y, st2 = lc.decimating_shift_addition_cc(xc, rate, dec, st[0], st[1])
        want, st_w = oracle.decimating_shift_addition_cc(xc, rate, dec, st[0], st[1])
        assert (st2[0], np.float32(st2[1]).view(np.uint32)) == (st_w[0], np.float32(st_w[1]).view(np.uint32)), (st2, st_w)
        seeds, alt, k = oracle.seed_phasors(np.array([st[1]], F32), AMBIG_ULPS)
        pos = st[0] + dec * np.arange(y.size)
        cands = [seeds[0]] + (_candidates(seeds[0], alt[0]) if k else [])
        assert any(np.all(_eq(y, mix_addition(xc[pos][None], s[None], dd)[0])) for s in cands), "drop-in decimating: samples"
        amb += k
        st = st2
    return amb
