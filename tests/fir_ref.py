"""Reference, error bound, case matrix and checks of the FIR bank contract (csrc/fir_decimate.cu), shared by tests/test_fir_bank_emulated.py
(CPU tier, the emulated library) and tests/test_gpu_fir_bank.py (-m gpu).

The bank computes, per channel c and output o, the reference fir_decimate_cc
    y_c[o] = sum_{k < T} h[k] * x_c[oD + k]          (I and Q separately)
so every output depends only on its own window [oD, oD + T) of its own row.  The checks hold the kernels to
    * bound():  every output within a per-output error bound of fir64(), the float64 FIR of the exact float32 values;
    * bits:     results that do not depend on the tiling (for one summation order), the tile boundaries, the channel set, row padding, output stride,
                I/Q swap, sign or a power-of-two scale, the u8 front end, the host pipeline or the libcsdr drop-in;
    * windows:  a NaN or +-Inf sample makes exactly the outputs whose window holds it non-finite, as in the reference, and no other output changes.

The checks talk to the library's C ABI through a driver with dev(array) -> buffer, ptr(buffer), host(buffer) -> array, `L` (the ctypes library,
argtypes set by csdr_b200.lib()) and `stream`, so the same code runs on the GPU and on the emulated library.
"""
import ctypes as C

import numpy as np

from bitcmp import SENTINEL, U, assert_bits_equal, bits  # noqa: F401

# (D, M, R, NPAIR, MINB, U8) of every compiled fir_bank_fast_kernel instantiation: D*M padded taps, R outputs per thread, NPAIR warp pairs per CTA
KERNELS = [(10, 8, 15, 2, 3, False), (10, 20, 13, 2, 3, False), (10, 20, 15, 2, 2, False), (10, 20, 15, 4, 1, False), (10, 20, 9, 4, 2, False),
           (10, 20, 13, 1, 5, False), (10, 20, 9, 2, 4, False), (10, 20, 11, 2, 3, False), (10, 20, 17, 2, 2, False), (50, 18, 3, 2, 2, False),
           (10, 8, 15, 2, 3, True), (10, 20, 13, 2, 3, True), (50, 18, 3, 2, 2, True)]
CF32_KERNELS = [k for k in KERNELS if not k[5]]
U8_KERNELS = [k for k in KERNELS if k[5]]
GENERIC = "fir_bank_generic_kernel"
U8_ROWS = "u8_rows_to_cf32_kernel"
VARIANT_TILING = {1: (10, 20, 15, 2, 2), 2: (10, 20, 15, 4, 1), 3: (10, 20, 9, 4, 2), 4: (10, 20, 13, 1, 5), 5: (10, 20, 9, 2, 4),
                  6: (10, 20, 11, 2, 3), 7: (10, 20, 17, 2, 2)}                  # launch_fir_decimate_bank's switch; 0 and -1 take the default
VARIANTS = [-1, 0, 1, 2, 3, 4, 5, 6, 7]


def out_pair(k):
    return 32 * k[2]


def out_tile(k):
    return k[3] * 32 * k[2]


def kernel_name(k):
    return GENERIC if k == GENERIC else f"fir_bank_fast_kernel<{k[0]}, {k[1]}, {k[2]}, {k[3]}, {k[4]}, {'true' if k[5] else 'false'}>"


def kernel_for(D, T, variant=-1, aligned=True, u8=False):
    """the instantiation the launchers pick: a KERNELS entry or GENERIC.  cf32 (launch_fir_decimate_bank): `aligned` = the first row on a 16-byte
    boundary and an even row stride.  u8 (launch_fir_decimate_bank_u8): `aligned` = 16-byte rows (stride % 8 == 0); without a fused tiling the C ABI
    converts (u8_rows_to_cf32_kernel) into an aligned temporary and runs the cf32 bank with variant -1 -- kernel_for(D, T) then names that."""
    if u8:
        if aligned and D == 10 and T <= 200:
            return (10, 8, 15, 2, 3, True) if T <= 80 else (10, 20, 13, 2, 3, True)
        if aligned and D == 50 and T <= 900:
            return (50, 18, 3, 2, 2, True)
        return kernel_for(D, T)
    if aligned and D == 10 and T <= 80 and variant < 0:
        return (10, 8, 15, 2, 3, False)
    if aligned and D == 10 and T <= 200:
        return VARIANT_TILING.get(variant, (10, 20, 13, 2, 3)) + (False,)
    if aligned and D == 50 and T <= 900:
        return (50, 18, 3, 2, 2, False)
    return GENERIC


def n_out_of(n, D, T):
    return (n - T) // D + 1 if n >= T else 0


def _windows(a, T, D, n_out):
    return np.lib.stride_tricks.sliding_window_view(a, T, axis=-1)[..., ::D, :][..., :n_out, :]


def fir64(x, taps, D):
    """float64 fir_decimate_cc of the exact float32 values, x [..., n] complex64 -> [..., n_out] complex128"""
    T = taps.size
    n_out = n_out_of(x.shape[-1], D, T)
    return _windows(x.astype(np.complex128), T, D, n_out) @ taps.astype(np.float64)


def bound(x, taps, D):
    """per-output, per-component bound of |kernel - fir64| as a complex array (real part: the I bound, imaginary part: the Q bound).

    Fast path: the tap range is split in two halves (warps of a pair); each half is a serial chain of fused multiply-adds acc = fl(acc + h_k x_k)
    over at most T live taps.  The padded taps k >= T have h_k = 0 and add nothing: fma(x, 0, acc) = acc for a finite x, and an output with a
    non-finite sample under a padded tap is summed again without the padding.  A chain of n FMAs errs by at most gamma_n sum |h_k x_k| with
    gamma_n = nu / (1 - nu), and the two halves meet in one rounded add, so
        |y - y64| <= ((1 + u) gamma_T + u) sum_k |h_k| |x_k|  <=  (T + 2) u (1 + 1e-3) sum_k |h_k| |x_k|        (T <= 900, u = 2^-24)
    per component.  The generic path is one chain of T FMAs (gamma_T), inside the same bound.  fir64 adds ~T 2^-53 relative, far inside the
    1e-3 margin.  This is the contract of CUDA-core FP32 kernels; a kernel with other arithmetic (split-TF32 ...) must argue its own bound here."""
    T = taps.size
    n_out = n_out_of(x.shape[-1], D, T)
    h = np.abs(taps.astype(np.float64))
    k = (T + 2) * U * (1 + 1e-3)
    return k * (_windows(np.abs(x.real).astype(np.float64), T, D, n_out) @ h) + 1j * k * (_windows(np.abs(x.imag).astype(np.float64), T, D, n_out) @ h)


def assert_within_bound(got, x, taps, D, what):
    """every output of got [ch, n_out] within bound() of fir64(); returns the worst err/bound ratio"""
    worst = 0.0
    for c in range(got.shape[0]):                                    # one row at a time: the window views are T/D times the row's size
        worst = max(worst, _row_within_bound(got[c], x[c], taps, D, f"{what}, channel {c}"))
    return worst


def _row_within_bound(got, x, taps, D, what):
    want, bnd = fir64(x, taps, D), bound(x, taps, D)
    g = got.astype(np.complex128)
    worst = 0.0
    for part in (np.real, np.imag):
        err, b = np.abs(part(g) - part(want)), part(bnd)
        ok = err <= b
        if not np.all(ok):
            i = tuple(np.argwhere(~ok)[0])
            raise AssertionError(f"{what}: output {i} errs by {err[i]:.3e}, bound {b[i]:.3e} ({np.count_nonzero(~ok)} outputs outside)")
        with np.errstate(invalid="ignore", divide="ignore"):
            r = np.where(b > 0, err / np.where(b > 0, b, 1), 0.0)
        worst = max(worst, float(r.max()) if r.size else 0.0)
    return worst


# ---- case matrix ------------------------------------------------------------------------------------------------------------------------------
T_FAST = {10: [1, 9, 10, 11, 79, 80, 81, 150, 199, 200], 50: [1, 49, 50, 51, 801, 850, 899, 900]}
CHANNELS = [1, 3, 64, 257]
SIZES = ["T", "T+D-1", "T+D", "tile", "tile-1", "tile+1", "pair-1", "pair+1", "odd"]
GENERIC_CASES = [(10, 201, "pad"), (50, 901, "pad"), (1, 17, "pad"), (3, 40, "pad"), (7, 79, "pad"), (11, 120, "pad"), (64, 300, "pad"),
                 (10, 199, "view"), (10, 199, "oddstride")]


def input_size(kind, D, T, k, tiles=2):
    """wideband row length for a size kind; k = the tiling (or GENERIC: pair and tile sizes of the default tiling stand in)"""
    kk = k if k != GENERIC else (10, 20, 13, 2, 3, False)
    n_of = lambda n_out, extra=0: T + (n_out - 1) * D + extra
    return {"T": T, "T+D-1": T + D - 1, "T+D": T + D,
            "tile": n_of(tiles * out_tile(kk)), "tile-1": n_of(tiles * out_tile(kk) - 1, D - 1), "tile+1": n_of(tiles * out_tile(kk) + 1),
            "pair-1": n_of(out_pair(kk) - 1, D // 2), "pair+1": n_of(out_pair(kk) + 1, 1),
            "odd": n_of(out_tile(kk) + 7) | 1}[kind]


def cases(max_work=None, tiles=2):
    """the matrix: D = 10 with every T of T_FAST and every variant, D = 50 with every T, the generic geometries.  Channel counts, size kinds and
    variants are walked with strides prime to their list lengths, so each entry of each list appears.  `max_work` caps channels x samples of a
    case (the CPU emulation): the channel count is lowered to the largest entry of CHANNELS that fits."""
    out, i = [], 0

    def add(D, T, variant, layout, seed):
        nonlocal i
        kind = SIZES[(4 * i) % len(SIZES)]
        aligned = layout == "pad"
        k = kernel_for(D, T, variant, aligned)
        n = input_size(kind, D, T, k, tiles)
        ch = CHANNELS[(3 * i) % len(CHANNELS)]
        if max_work:
            ch = max([1] + [c for c in CHANNELS if c * n <= max_work and c <= ch])
        out.append(dict(D=D, T=T, variant=variant, layout=layout, kind=kind, n=n, channels=ch, seed=seed))
        i += 1

    for T in T_FAST[10]:
        for rep in range(2):
            add(10, T, VARIANTS[(5 * i) % len(VARIANTS)], "pad", 10_000 + 10 * T + rep)
    for T in T_FAST[50]:
        for rep in range(2):
            add(50, T, -1, "pad", 50_000 + 10 * T + rep)
    for D, T, layout in GENERIC_CASES:
        add(D, T, -1, layout, 90_000 + 100 * D + T)
    return out


def case_id(c):
    return f"D{c['D']}-T{c['T']}-v{c['variant']}-{c['layout']}-{c['kind']}-n{c['n']}-ch{c['channels']}"


def make_inputs(case, taps=None):
    """x [channels, n] complex64 uniform in the unit square, and taps: uniform(-1, 1) (asymmetric: a reversed tap order shows), or the given ones"""
    rng = np.random.default_rng(case["seed"])
    ch, n, T = case["channels"], case["n"], case["T"]
    x = (rng.uniform(-1, 1, (ch, n)) + 1j * rng.uniform(-1, 1, (ch, n))).astype(np.complex64)
    h = rng.uniform(-1, 1, T).astype(np.float32) if taps is None else np.ascontiguousarray(taps, np.float32)
    return x, h


# ---- calls through the C ABI ------------------------------------------------------------------------------------------------------------------
def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def layout_rows(x, layout):
    """x [ch, n] -> (buffer [ch, stride] complex64 whose padding holds NaN, first column): "pad" = 16-byte aligned rows (even stride),
    "tight" = stride n, "view" = rows starting one sample in (8-byte aligned), "oddstride" = an odd row stride"""
    ch, n = x.shape
    stride, col0 = {"pad": (n + (n & 1) + 2, 0), "tight": (n, 0), "view": (n + 1 + (n & 1) + 2, 1), "oddstride": (n + 1 + (n & 1), 0)}[layout]
    buf = np.full((ch, stride), np.complex64(complex(np.nan, np.nan)), np.complex64)
    buf[:, col0:col0 + n] = x
    return buf, col0


def bank(drv, x, D, taps, variant=-1, layout="pad", ostride=None):
    """csdrb_fir_decimate_bank_cc on x [ch, n] laid out by layout_rows into an output [ch + 1, ostride] that starts as SENTINEL -> y [ch, n_out].
    The output's padding columns and spare row must come back untouched."""
    ch, n = x.shape
    T = taps.size
    n_out = n_out_of(n, D, T)
    ostride = n_out + 3 if ostride is None else ostride
    xb, col0 = layout_rows(x, layout)
    ob = np.full((ch + 1, 2 * ostride), SENTINEL, np.uint32).view(np.complex64)
    dx, do = drv.dev(xb), drv.dev(ob)
    rc = drv.L.csdrb_fir_decimate_bank_cc(drv.ptr(dx) + 8 * col0, xb.shape[1], drv.ptr(do), ostride, ch, n, D, _fp(taps), T, variant, drv.stream)
    assert rc == n_out, (rc, n_out, drv.L.csdrb_last_error())
    got = drv.host(do)
    w = got.view(np.uint32)
    assert np.all(w[:, 2 * n_out:] == SENTINEL) and np.all(w[ch] == SENTINEL), "a store beyond n_out or the last channel"
    return np.ascontiguousarray(got[:ch, :n_out])


def bank_u8(drv, u8, n, D, taps, stride):
    """csdrb_fir_decimate_bank_u8_cc on u8 [ch, n, 2] placed in rows of `stride` samples (padding 0x5A) -> y [ch, n_out]"""
    ch = u8.shape[0]
    T = taps.size
    n_out = n_out_of(n, D, T)
    ub = np.full((ch, stride, 2), 0x5A, np.uint8)
    ub[:, :n] = u8
    ob = np.full((ch + 1, 2 * (n_out + 3)), SENTINEL, np.uint32).view(np.complex64)
    du, do = drv.dev(ub), drv.dev(ob)
    rc = drv.L.csdrb_fir_decimate_bank_u8_cc(drv.ptr(du), stride, drv.ptr(do), n_out + 3, ch, n, D, _fp(taps), T, drv.stream)
    assert rc == n_out, (rc, n_out, drv.L.csdrb_last_error())
    got = drv.host(do)
    w = got.view(np.uint32)
    assert np.all(w[:, 2 * n_out:] == SENTINEL) and np.all(w[ch] == SENTINEL), "a u8 store beyond n_out or the last channel"
    return np.ascontiguousarray(got[:ch, :n_out])


# ---- the checks -------------------------------------------------------------------------------------------------------------------------------
def check_case(drv, case, taps=None, invariants=True):
    """one case: the bound at every output, then (invariants) the bit-exact ones that hold for every kernel -> the worst err/bound ratio"""
    D, T, variant, layout = case["D"], case["T"], case["variant"], case["layout"]
    x, h = make_inputs(case, taps)
    ch, n = x.shape
    k = kernel_for(D, T, variant, layout == "pad")
    y = bank(drv, x, D, h, variant, layout)
    worst = assert_within_bound(y, x, h, D, case_id(case))
    if not invariants or y.shape[1] == 0:
        return worst
    n_out = y.shape[1]
    # row padding and output stride: tight rows (when they keep the tiling) and a tight output stride n_out (odd n_out: every other row on an
    # 8-byte boundary, the scalar store path)
    if kernel_for(D, T, variant, n % 2 == 0) == k and layout == "pad":
        assert_bits_equal(bank(drv, x, D, h, variant, "tight", ostride=n_out), y, "tight rows, output stride n_out")
    else:
        assert_bits_equal(bank(drv, x, D, h, variant, layout, ostride=n_out), y, "output stride n_out")
    # channels: a permuted subset and one channel alone
    rng = np.random.default_rng(case["seed"] + 1)
    sub = rng.permutation(ch)[:3]
    assert_bits_equal(bank(drv, x[sub], D, h, variant, layout), y[sub], "permuted channel subset")
    c = ch - 1
    assert_bits_equal(bank(drv, x[c:c + 1], D, h, variant, layout), y[c:c + 1], "one channel alone")
    # position: starting j outputs later moves every tile boundary; the outputs are the same
    shifts = (1, out_pair(k) - 1, out_tile(k) + 1) if k != GENERIC else (1, 37)
    for j in shifts:
        if j < n_out:
            assert_bits_equal(bank(drv, np.ascontiguousarray(x[:, j * D:]), D, h, variant, layout), y[:, j:], f"stream started {j} outputs later")
    # symmetry: I <-> Q, sign, a power-of-two scale are exact on both sides
    swapped = (x.imag + 1j * x.real).astype(np.complex64)
    assert_bits_equal(bank(drv, swapped, D, h, variant, layout), (y.imag + 1j * y.real).astype(np.complex64), "I and Q swapped")
    assert_bits_equal(bank(drv, -x, D, h, variant, layout), -y, "negated input")
    assert_bits_equal(bank(drv, (x * np.float32(2.0 ** -7)).astype(np.complex64), D, h, variant, layout), (y * np.float32(2.0 ** -7)).astype(np.complex64),
                      "input scaled by 2^-7")
    return worst


def check_tilings(drv, D, T, n, ch=3, seed=0):
    """D = 10: every variant gives the bits of the default tiling.  The present kernels sum each output in one order (per half: phase pairs,
    sub-taps, the pair's two phases; halves of M*D/2 taps meet in one add), whatever the outputs per thread or warp pairs per CTA -- so for
    80 < T <= 200 all of -1 and 0-7 agree, and for T <= 80 variants 0-7 (M = 20) agree while -1 runs M = 8, whose halves split the taps
    elsewhere: that one is held to the bound only.  A kernel with another summation order would have to drop this check, not the bound."""
    x, h = make_inputs(dict(seed=seed, channels=ch, n=n, T=T))
    ref = bank(drv, x, D, h, 0)
    for v in VARIANTS:
        y = bank(drv, x, D, h, v)
        if T > 80 or v >= 0:
            assert_bits_equal(y, ref, f"T={T}: variant {v} against variant 0")
        else:
            assert_within_bound(y, x, h, D, f"T={T} variant -1 (M = 8)")


def nonfinite_positions(D, T, k, n):
    """samples to poison: around tile and pair boundaries, just past a window and at the last padded tap of a window (the samples that only
    padded taps meet), and the last sample of the row"""
    kk = k if k != GENERIC else (10, 20, 13, 2, 3, False)
    M = kk[1] if k != GENERIC else 1
    o = 20
    pos = {o * D + T, o * D + max(D * M, T + 1) - 1, out_tile(kk) * D, out_tile(kk) * D - 1, out_pair(kk) * D + 1, n - 1, 3}
    return sorted(p for p in pos if 0 <= p < n)


def check_nonfinite(drv, D, T, variant, n, ch=3, seed=0):
    """NaN, +Inf and -Inf (channel c gets the c-th of the three) at nonfinite_positions(): exactly the outputs whose window [oD, oD + T) holds one
    are non-finite, every other output has the clean run's bits"""
    k = kernel_for(D, T, variant)
    x, h = make_inputs(dict(seed=seed, channels=ch, n=n, T=T))
    clean = bank(drv, x, D, h, variant)
    n_out = clean.shape[1]
    pos = nonfinite_positions(D, T, k, n)
    bad = np.array([np.nan, np.inf, -np.inf], np.float32)
    xp = x.copy()
    for c in range(ch):
        for i, p in enumerate(pos):
            v = bad[(c + i) % 3]
            xp[c, p] = complex(v, 0.5) if i % 2 == 0 else complex(0.25, v)          # the I or the Q component
    got = bank(drv, xp, D, h, variant)
    o = np.arange(n_out)
    hit = np.zeros(n_out, bool)
    for p in pos:
        hit |= (o * D <= p) & (p < o * D + T)
    for c in range(ch):
        fin = np.isfinite(got[c].real) & np.isfinite(got[c].imag)
        assert np.array_equal(~fin, hit), (f"{kernel_name(k)} D={D} T={T} channel {c}: non-finite outputs {np.flatnonzero(~fin)[:12]}, "
                                           f"expected {np.flatnonzero(hit)[:12]}")
        assert_bits_equal(got[c][~hit], clean[c][~hit], f"{kernel_name(k)} D={D} T={T} channel {c}: outputs away from the poisoned samples")


NONFINITE = [(10, 79, -1), (10, 1, -1), (10, 81, 0), (10, 199, 0), (10, 200, -1)] + [(10, 81, v) for v in range(1, 8)] + \
            [(10, 150, v) for v in (3, 7)] + [(50, 801, -1), (50, 51, -1), (50, 900, -1), (7, 79, -1), (10, 201, -1)]


def nonfinite_n(D, T, variant):
    k = kernel_for(D, T, variant)
    kk = k if k != GENERIC else (10, 20, 13, 2, 3, False)
    return T + (out_tile(kk) + 40) * D + 5


def u8_inputs(ch, n, seed):
    rng = np.random.default_rng(seed)
    u8 = rng.integers(0, 256, (ch, n, 2), dtype=np.uint8)
    if n >= 256:
        u8[0, :256, 0] = np.arange(256); u8[0, :256, 1] = np.arange(255, -1, -1)   # every code on both components
    return u8


def convert_u8(u8):
    """convert_u8_f of libcsdr: (float)((double)(float)b / (255 / 2.0) - 1.0) per byte, as complex64 rows"""
    f = ((u8.astype(np.float32).astype(np.float64) / (255 / 2.0)) - 1.0).astype(np.float32)
    return np.ascontiguousarray(f).view(np.complex64)[..., 0]


def check_u8(drv, D, T, n, ch=3, seed=0):
    """the fused u8 call gives the cf32 call's bits on convert_u8_f's output (same tiling, same order), at a 16-byte row stride and, through the
    two-launch fallback, at a stride that is not a multiple of 8 samples"""
    u8 = u8_inputs(ch, n, seed)
    h = np.random.default_rng(seed + 1).uniform(-1, 1, T).astype(np.float32)
    ref = bank(drv, convert_u8(u8), D, h)
    assert_within_bound(ref, convert_u8(u8), h, D, f"u8 D={D} T={T}")
    assert_bits_equal(bank_u8(drv, u8, n, D, h, (n + 7) & ~7), ref, f"fused u8 D={D} T={T} n={n}")
    assert_bits_equal(bank_u8(drv, u8, n, D, h, ((n + 7) & ~7) + 2), ref, f"two-launch u8 D={D} T={T} n={n}")
