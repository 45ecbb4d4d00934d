"""CPU tier for the single-CTA FFT family (csdr_b200/csrc/fft.cuh, fft16.cuh, fft_kernels.cuh): the batched c2c transform at 2..16384 points,
the overlap-add bank, the apply_fir_fft_cc kernel, the fastddc forward step and the three fastddc inverse paths, each against a float64 model
with a per-output bound derived below, and against exact invariants.  The check_* bodies run through the C ABI (tests/spectrum/spectrum.py's
EmulDev here, on the emulated full library; CudaDev in tests/test_gpu_fft_bound.py, on the H100 at every size and at bank sizes the emulator
cannot afford).

The per-output bound, to first order in u = 2^-24 (round to nearest: a rounded real z has |fl(z) - z| <= u|z|).
An N-point transform is a sequence of passes; a pass maps every input leg v_r of a butterfly to its outputs through a twiddle product and
a small DFT.  Every later operation is a unit-modulus map, so an error made at one pass reaches an output unchanged in size, and the values
that feed one output at one pass partition the input: |X^_k - X_k| <= eps(N) * sum_n |x_n|, eps(N) = sum over passes of the worst cost of a
leg through its butterfly.  The costs, in units of u:
  - complex addition, rounded per component: u |a + b| <= u (|a| + |b|).  dft2: 1; dft4 (two addition levels, * -i exact): 2.
  - dft8: two dft4 levels (2), then h * (o.x +- o.y): the sum, the product and the rounded constant h each give u per component, and the
    pair ((o.x + o.y), (o.y - o.x)) has norm sqrt(2) |o|, so 3 h sqrt(2) |o| = 3 |o|; then one addition (1): 6.
  - mul_w16 (dft16's inner twiddles, constants C1, S1, H rounded once): the constant (1), the rounded product inside the fmaf (1), the fmaf
    (1): 3.  dft16 = dft4 + mul_w16 + dft4: 7.
  - cmul_w / cmul of unit-modulus operands: the rounded product inside the fmaf (norm <= u |a|) and the fmaf (u |a|): 2.
  - twiddle tables: w1, w2, w4 (and w8) rounded once from double: 1.  Radix 8: w3, w5, w6 = one cmul of two table values: 2 + 1 + 1 = 4;
    w7 = (w1 w2) w4: 2 + 4 + 1 = 7; applied: 2, so the worst leg of a twiddled radix-8 pass costs 9 + dft8 6 = 15 (5 per level).
    Radix 16: eleven derived twiddles, the worst w15 = ((w1 w2) w4) w8: 2 + 7 + 1 = 10; applied: 2, so 12 + dft16 7 = 19 (4.75 per level).
  - The first pass has no twiddles: dft2 1, dft4 2, dft8 6, dft16 7.
So with L = log2 N:  radix-8 form (first radix 2, 4 or 8, then radix 8)   eps = 1 + 15 p, 2 + 15 p or 6 + 15 (p - 1)  <= (5 L - 4) u;
                     radix-16 form (first radix 2, 4, 8 or 16, then 16)   eps = 1 + 19 p, 2 + 19 p, 6 + 19 p, 7 + 19 (p - 1)  <= (4.75 L - 3.75) u.
eps_fft() adds up the passes exactly.  (The four-step kernel's docstring puts a radix-16 pass at 17u; with w15 at 10u and dft16 at 7u it is
19u, inside its 5u per level.)

Overlap-add block and apply_fir_fft: y = IFFT(FFT(x_blk) H) / N.  The forward error is eps_f ||x_blk||_1 per bin, |X_k| <= ||x_blk||_1; the
product of libcsdr.c:827-828 (two separate products and a rounded sum per component) costs (1 + sqrt 2) u |X||H| <= 3u; the inverse adds
eps_i sum_k |P_k|; /N is exact.  Per output: (eps_f + eps_i + 3u) ||x_blk||_1 mean_k |H_k| for every block that reaches it, and each
overlap-add addition u times the sum of the magnitudes it adds.  The model is the same block-wise computation on the float32 H promoted to
float64 (for an impulse: the taps shifted to the impulse).

fastddc inverse, per output of a block: the fold F_r = sum_p Xs[r + pM] H[r + pM] of the float32 spectrum and taps in float64, /pre, the
float64 IFFT_M / M, the kept samples scrap + remain + k * post_decimation, times the phasor the kernel replays -- taken from the oracle's
decimating_shift_addition_cc on an all-ones input (exact: c * 1 - s * 0), block by block with the carried (remain, phase).  Bound:
  - the fold, a sequential sum per component: separate products (tiled and generic kernels) round every term P + 2 times at most, the fold
    kernel's FFMA pairs chain 2P fused terms per component, so gamma_{P+2} or gamma_{2P} (gamma_n = n u / (1 - n u)) times
    sqrt(2) sum_p |Xs| |H| (the per-component sums |xr hr| + |xi hi|, |xr hi| + |xi hr| have norm <= sqrt 2 |x||h|); for P > 2 the fused form
    is the larger one.  Every residue reaches every output through the IFFT: (1/M) sum_r of it.
  - the IFFT: eps_fft(M, radix 8) sum_r |F_r| / M.
  - the rotation (rotate_rn: two products and a sum per component): 3u |y|.
pre_decimation and M are powers of two, so /pre and /M are exact.

A bound is never fitted to observed errors: every helper asserts the kernel stays below it and records the worst error/bound ratio per path
(printed by the coverage test).  rel_rms is asserted as well, so a regression of the old aggregate bars still names itself."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "spectrum"))
import emul_build  # noqa: E402
import spectrum as S  # noqa: E402
import test_fft_large_emulated as LE  # noqa: E402
from oracle.pyoracle import Oracle, rel_rms  # noqa: E402

U = 2.0 ** -24
SM_COUNT = 132                                                          # kSmCount in csrc/common.cuh: the dispatch rules below use it
DFT = {2: 1, 4: 2, 8: 6, 16: 7}                                         # untwiddled butterflies, in u
PASS8, PASS16 = 9 + 6, 12 + 7                                           # twiddled passes: worst leg's twiddle + butterfly
CHAN_DT = np.dtype([("offsetbin", np.int32), ("sindelta", np.float32), ("cosdelta", np.float32), ("rate", np.float32)])


# ---- the bound helpers (also used by tests/fuzz/fuzz_emulated_fft.py) -------------------------------------------------------------------------
def eps_fft(n, form):
    """first-order per-output error of an n-point transform, in units of sum |x| (see the module docstring); form "r8" or "r16" """
    lg = n.bit_length() - 1
    if form == "r8":
        p, q = divmod(lg, 3)
        u = DFT[8] + (p - 1) * PASS8 if q == 0 else DFT[1 << q] + p * PASS8
    else:
        p, q = divmod(lg, 4)
        u = DFT[16] + (p - 1) * PASS16 if q == 0 else DFT[1 << q] + p * PASS16
    return u * U


def gamma(n):
    return n * U / (1 - n * U)


def c2c_form(n):
    """launch_fft_c2c_batch / launch_fastddc_fwd: radix-16 passes from 32 points on"""
    return "r16" if n >= 32 else "r8"


def ola_form(n):
    """launch_olafir_bank: radix-16 passes at 256 and 4096 points (olafir_bank_fused16_kernel), radix 8 elsewhere"""
    return "r16" if n in (256, 4096) else "r8"


def first_radix8(n):
    lg = n.bit_length() - 1
    return {1: 2, 2: 4, 0: 8}[lg % 3]


def c2c_bound(x, form):
    """[batch, N] -> per-output bound of the transform of every row"""
    n = x.shape[-1]
    return np.broadcast_to(eps_fft(n, form) * np.abs(x.astype(np.complex128)).sum(axis=-1, keepdims=True), x.shape)


def block_conv_bound(x_blk, H, form):
    """overlap-add block / apply_fir_fft before any tail addition: the bound of every output of y = IFFT(FFT(x_blk) H) / N"""
    n = H.shape[-1]
    return (2 * eps_fft(n, form) + 3 * U) * np.abs(x_blk.astype(np.complex128)).sum() * np.abs(H.astype(np.complex128)).mean()


def ola_model(x, H, N, isz, form, tail=None):
    """float64 overlap-add of one channel's stream x with the float32 H (after the carried `tail` of a previous call, if given), and the
    per-output bound: (model, bound) over nblocks * isz outputs"""
    nb = x.size // isz
    Hd = H.astype(np.complex128)
    full = np.zeros(nb * isz + N, np.complex128); mag = np.zeros(nb * isz + N); cnt = np.zeros(nb * isz + N); bnd = np.zeros(nb * isz + N)
    if tail is not None:
        full[:N - isz] = tail[:N - isz]; mag[:N - isz] = np.abs(tail[:N - isz]); cnt[:N - isz] = 1
    for b in range(nb):
        blk = np.zeros(N, np.complex128); blk[:isz] = x[b * isz:(b + 1) * isz]
        yb = np.fft.ifft(np.fft.fft(blk) * Hd)
        sl = slice(b * isz, b * isz + N)
        full[sl] += yb; mag[sl] += np.abs(yb); cnt[sl] += 1
        bnd[sl] += block_conv_bound(blk, H, form)
    bnd += np.maximum(cnt - 1, 0) * U * mag
    return full[:nb * isz], bnd[:nb * isz]


def phasor_chain(oracle, g, chan, nblocks, remain, phase):
    """the post-shift phasors every block replays and the (remain, phase) it starts from: the oracle's decimating_shift_addition_cc on all-ones
    input of post_input_size samples per block, state carried from block to block.  Returns ([(remain, phasors)] per block, remain, phase)."""
    d = oracle.L.oracle_decimating_shift_addition_init(g.post_shift, g.post_decimation)
    assert (np.float32(d.sindelta), np.float32(d.cosdelta), np.float32(d.rate)) == (chan["sindelta"], chan["cosdelta"], chan["rate"])
    ones = np.ones(g.post_input_size, np.complex64)
    blocks = []
    for _ in range(nblocks):
        ph, (r2, p2) = oracle.decimating_shift_addition_cc(ones, g.post_shift, g.post_decimation, remain, phase)
        blocks.append((remain, ph.astype(np.complex128)))
        remain, phase = r2, p2
    return blocks, remain, phase


def fastddc_inv_model(oracle, sp, taps, chan, g, path, remain=0, phase=0.0):
    """float64 model of one channel of the inverse bank over the blocks sp [nb, N] (module docstring): (outputs, bounds, per-block counts,
    carried remain, carried phase)"""
    N, M = sp.shape[1], g.fft_inv_size
    P, half = N // M, N // 2
    assert P == g.pre_decimation
    gam = gamma(2 * P) if path == "fold" else gamma(P + 2)
    H = taps.astype(np.complex128)
    off = int(chan["offsetbin"])
    chain, remain, phase = phasor_chain(oracle, g, chan, sp.shape[0], remain, phase)
    ys, bs, counts = [], [], []
    for b0 in range(0, sp.shape[0], 256):
        Xs = sp[b0:b0 + 256].astype(np.complex128)
        Xs = np.concatenate([Xs[:, half:], Xs[:, :half]], axis=1)                   # the first half swap (fastddc.c:123)
        F = (Xs * H).reshape(-1, P, M).sum(axis=1) / P
        Fabs = (np.abs(Xs) * np.abs(H)).reshape(-1, P, M).sum(axis=1) / P
        t = np.fft.ifft(np.roll(F, -off, axis=1), axis=1)                          # inv_input[(r - offsetbin) mod M] = F[r]; IFFT / M
        common = (gam * np.sqrt(2) * Fabs.sum(axis=1) + eps_fft(M, "r8") * np.abs(F).sum(axis=1)) / M
        for j in range(t.shape[0]):
            r0, ph = chain[b0 + j]
            v = t[j, g.scrap + r0 + g.post_decimation * np.arange(ph.size)]
            y = v * ph
            ys.append(y); bs.append(np.abs(ph) * common[j] + 3 * U * np.abs(y)); counts.append(ph.size)
    return np.concatenate(ys), np.concatenate(bs), counts, remain, phase


# ---- recording: the worst error/bound ratio per path, and which paths ran -------------------------------------------------------------------------
def note(dev, path, ratio=None):
    if not hasattr(dev, "worst"):
        dev.worst = {}
    if ratio is not None or path not in dev.worst:
        dev.worst[path] = max(dev.worst.get(path, 0.0), ratio or 0.0)


def within(dev, path, got, want, bound):
    """every output within its bound (outputs whose bound is 0 must be exact); records the worst ratio for `path`"""
    got = np.asarray(got).astype(np.complex128)
    assert got.shape == want.shape == np.shape(bound), (got.shape, want.shape, np.shape(bound))
    assert np.isfinite(got).all(), path
    err = np.abs(got - want)
    ratio = float(np.max(np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err > 0, np.inf, 0)))) if err.size else 0.0
    note(dev, path, ratio)
    bad = np.argwhere(err > bound)
    assert bad.size == 0, f"{path}: {len(bad)} outputs beyond the per-output bound, worst error/bound {ratio:.3g}, first at {bad[:4].tolist()}"
    return ratio


def launches(dev):
    return dev.L.csdrb_kernel_launches()


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def setup(dev):
    LE.setup(dev)
    L = dev.L
    vp, lg, it = C.c_void_p, C.c_long, C.c_int
    L.csdrb_kernel_launches.restype = C.c_long
    L.csdrb_bandpass_fir_fft_bank_cc.argtypes = [vp, lg, vp, lg, it, it, it, it, vp, lg, vp, vp]
    return dev


def noise(rng, *shape):
    return ((rng.standard_normal(shape) + 1j * rng.standard_normal(shape)) * 0.5).astype(np.complex64)


# ---- c2c ----------------------------------------------------------------------------------------------------------------------------------------
def c2c(dev, x, inverse=False, misalign=False):
    """csdrb_fft_c2c_batch on the rows of x [batch, N]; misalign: both rows start 8 bytes past a 16-byte boundary (the scalar FftRowIn/Out path)"""
    batch, N = x.shape
    k = 1 if misalign else 0
    xs = np.zeros(batch * N + k, np.complex64); xs[k:] = x.reshape(-1)
    d_x = dev.put(xs); d_y = dev.alloc(8 * (batch * N + k))
    before = launches(dev)
    rc = dev.L.csdrb_fft_c2c_batch(dev.ptr(d_x) + 8 * k, N, dev.ptr(d_y) + 8 * k, N, N, batch, 1 if inverse else 0, dev.stream)
    assert rc == 0 and launches(dev) - before == 1, (rc, dev.L.csdrb_last_error())
    note(dev, f"c2c {c2c_form(N)}")
    return dev.get(d_y, np.complex64)[k:].reshape(batch, N)


def exact_dft_rows(N, cols, inverse):
    k = np.arange(N)
    return np.exp((2j if inverse else -2j) * np.pi * ((np.asarray(cols)[:, None] * k[None, :]) % N) / N)


def impulse_columns(N, rng, full_up_to, subset):
    if N <= full_up_to:
        return np.arange(N)
    cols = set(range(0, N, max(1, N // subset))) | set(rng.choice(N, subset, replace=False).tolist()) | set(range(16)) | {N // 2 - 1, N // 2, N - 1}
    cols = np.array(sorted(cols))
    assert set((cols % 16).tolist()) == set(range(16))
    return cols


def check_c2c_impulse_matrix(dev, N, full_up_to=256, subset=48, chunk=512):
    """impulses at every input position (or a strided + random subset, all residues mod 16): the computed DFT matrix column by column, every entry
    within eps(N) of the exact w^(kp) -- every twiddle-table entry of every pass is on some path"""
    rng = np.random.default_rng(N)
    cols = impulse_columns(N, rng, full_up_to, subset)
    form = c2c_form(N)
    for a in range(0, cols.size, chunk):
        cc = cols[a:a + chunk]
        x = np.zeros((cc.size, N), np.complex64); x[np.arange(cc.size), cc] = 1
        for inverse in (False, True):
            y = c2c(dev, x, inverse)
            within(dev, f"c2c {form} impulses", y, exact_dft_rows(N, cc, inverse), c2c_bound(x, form))


def boundary_positions(N, form):
    """each pass's index boundaries: 0, 1, N/R0 - 1, N/R0, NS +- 1 for every sub-transform size NS, N - 1"""
    lg = N.bit_length() - 1
    if form == "r8":
        r0, step = first_radix8(N), 8
    else:
        r0, step = {1: 2, 2: 4, 3: 8, 0: 16}[lg % 4], 16
    pos = {0, 1, N // r0 - 1, N // r0, N - 1}
    ns = r0
    while ns < N:
        pos |= {ns - 1, ns, ns + 1}
        ns *= step
    return sorted(p for p in pos if 0 <= p < N)


def check_c2c_sparse_and_tones(dev, N):
    """<= 16 nonzeros on the passes' index boundaries, and tones on bins 1, N/16 + 1, N - 1: every output within eps(N) sum|x|"""
    rng = np.random.default_rng(N + 1)
    form = c2c_form(N)
    pos = boundary_positions(N, form)
    rows = []
    for a in range(0, len(pos), 16):
        r = np.zeros(N, np.complex64); r[pos[a:a + 16]] = noise(rng, len(pos[a:a + 16])) * 3; rows.append(r)
    n = np.arange(N)
    for q in sorted({1, N // 16 + 1, N - 1}):
        rows.append(np.exp(2j * np.pi * ((q * n) % N) / N).astype(np.complex64))
    x = np.stack(rows)
    for inverse in (False, True):
        y = c2c(dev, x, inverse)
        xd = x.astype(np.complex128)
        want = np.fft.ifft(xd, axis=1) * N if inverse else np.fft.fft(xd, axis=1)
        within(dev, f"c2c {form} sparse", y, want, c2c_bound(x, form))


def check_c2c_invariants(dev, N, batch=3):
    """dense rows: bound and rel_rms; a row of a batch == the single call; 8-byte == 16-byte aligned rows; inverse(x) == conj(forward(conj x));
    a NaN or Inf stays in its row and makes every output of it non-finite"""
    rng = np.random.default_rng(N + 2)
    form = c2c_form(N)
    x = noise(rng, batch, N)
    y = c2c(dev, x)
    want = np.fft.fft(x.astype(np.complex128), axis=1)
    within(dev, f"c2c {form} noise", y, want, c2c_bound(x, form))
    assert rel_rms(y, want) < 1e-6
    for b in range(batch):
        assert np.array_equal(bits(c2c(dev, x[b:b + 1])[0]), bits(y[b])), b
    assert np.array_equal(bits(c2c(dev, x, misalign=True)), bits(y))
    yi = c2c(dev, x, inverse=True)
    assert np.array_equal(bits(c2c(dev, np.conj(x), misalign=True, inverse=True)), bits(np.conj(y)))
    assert np.array_equal(bits(yi), bits(np.conj(c2c(dev, np.conj(x))))), "inverse(x) != conj(forward(conj(x)))"
    for bad in (np.nan, np.inf):
        z = x.copy(); z[1, (N * 5) // 7] = bad
        for inverse, clean in ((False, y), (True, yi)):
            d = c2c(dev, z, inverse)
            assert np.array_equal(bits(d[0]), bits(clean[0])) and np.array_equal(bits(d[2:]), bits(clean[2:]))
            assert not np.isfinite(d[1]).any(), (bad, inverse)


# ---- the overlap-add bank -----------------------------------------------------------------------------------------------------------------------
def auto_blocks_per_cta(channels, nblocks):
    """launch_olafir_bank's choice when the caller passes 0 (csdrb_bandpass_fir_fft_bank_cc)"""
    want = (SM_COUNT * 8 + channels - 1) // channels
    bpc = (nblocks + want - 1) // want
    return bpc if bpc >= 16 else min(nblocks, 16)


def ola_path(N):
    if N in (4, 8):
        return "ola staged"
    if N in (256, 4096):
        return "ola fused16"
    r0 = first_radix8(N)
    return f"ola fused R0={r0}" + (" hand-over" if r0 == 8 else "")


def ola_bank(dev, x, H, N, isz, taps_stride=None, cuts=(), tail=None):
    """csdrb_bandpass_fir_fft_bank_cc over the stream x [C, nb * isz], cut into calls at block indices `cuts`: (output, carried tail)"""
    L = dev.L
    ch, T = x.shape
    nb = T // isz
    taps_stride = N if taps_stride is None else taps_stride
    d_H = dev.put(H); d_tail = dev.put(np.zeros((ch, N), np.complex64) if tail is None else tail)
    outs = []
    for a, b in zip([0] + list(cuts), list(cuts) + [nb]):
        n = (b - a) * isz
        d_x = dev.put(np.ascontiguousarray(x[:, a * isz:b * isz])); d_y = dev.alloc(8 * max(ch * n, 1))
        before = launches(dev)
        rc = L.csdrb_bandpass_fir_fft_bank_cc(dev.ptr(d_x), n, dev.ptr(d_y), n, ch, N, isz, b - a, dev.ptr(d_H), taps_stride, dev.ptr(d_tail), dev.stream)
        assert rc == 0 and launches(dev) - before == (1 if b > a else 0), (rc, L.csdrb_last_error())
        outs.append(dev.get(d_y, np.complex64)[:ch * n].reshape(ch, n))
    note(dev, ola_path(N))
    return np.concatenate(outs, axis=1), dev.get(d_tail, np.complex64).reshape(ch, N)


def ola_impulses(N, isz, nb, rng):
    """one impulse in every block at a varying offset, plus impulses on block boundaries and the 16-block CTA-run boundaries"""
    x = np.zeros(nb * isz, np.complex64)
    for b in range(nb):
        x[b * isz + (b * 7) % isz] = noise(rng, 1)[0] * 2
    for p in [isz - 1, isz, 15 * isz - 1, 16 * isz, 16 * isz + isz // 2, 32 * isz - 1, 32 * isz, nb * isz - 1]:
        if p < x.size:
            x[p] += 1
    return x


def check_ola(dev, N, isz, nb):
    """two channels, impulses in one and dense noise in the other, per-output bound against the block-wise float64 model; the carried tail"""
    rng = np.random.default_rng(N * 7 + isz)
    x = np.stack([ola_impulses(N, isz, nb, rng), noise(rng, nb * isz)])
    H = noise(rng, 2, N)
    y, tail = ola_bank(dev, x, H, N, isz)
    form = ola_form(N)
    for c in range(2):
        want, bound = ola_model(x[c], H[c], N, isz, form)
        within(dev, ola_path(N) + (" impulses" if c == 0 else " noise"), y[c], want, bound)
        assert rel_rms(y[c], want) < 2e-6
    return x, H, y, tail


def check_ola_invariants(dev, N, isz, nb):
    """the output does not depend on how the stream is cut into calls (calls of one block, of many); taps_stride 0 == per-channel copies of one
    taps row; channel c of a 3-channel call == a one-channel call.  Compared with == (a zero lead-in tail may give -0 for +0)."""
    rng = np.random.default_rng(N + isz + 5)
    x = noise(rng, 3, nb * isz)
    H = noise(rng, 3, N)
    y, tail = ola_bank(dev, x, H, N, isz)
    for cuts in ([1], [nb // 2, nb // 2 + 1], list(range(1, nb, 5))):
        y2, tail2 = ola_bank(dev, x, H, N, isz, cuts=cuts)
        assert np.array_equal(y2, y) and np.array_equal(tail2[:, :N - isz], tail[:, :N - isz]), cuts
    for c in range(3):
        y1, _ = ola_bank(dev, x[c:c + 1], H[c:c + 1], N, isz)
        assert np.array_equal(y1[0], y[c]), c
    ys, _ = ola_bank(dev, x, H[:1], N, isz, taps_stride=0)
    yc, _ = ola_bank(dev, x, np.repeat(H[:1], 3, axis=0), N, isz)
    assert np.array_equal(ys, yc)


def check_ola_nonfinite(dev, N, isz, nb):
    """a NaN/Inf sample in block b of channel c damages exactly stream positions [b*isz, b*isz + N) of channel c; a bad tap, channel c only"""
    rng = np.random.default_rng(N + isz + 9)
    x = noise(rng, 3, nb * isz); H = noise(rng, 3, N)
    clean, _ = ola_bank(dev, x, H, N, isz)
    T = nb * isz
    for bad in (np.nan, np.inf):
        for b in sorted({0, nb // 2, 16 % nb, nb - 1}):
            z = x.copy(); z[1, b * isz + (isz - 1) // 2] = bad
            y, _ = ola_bank(dev, z, H, N, isz)
            win = np.zeros(T, bool); win[b * isz:min(T, b * isz + N)] = True
            assert np.array_equal(bits(y[[0, 2]]), bits(clean[[0, 2]]))
            assert np.array_equal(bits(y[1, ~win]), bits(clean[1, ~win])), (bad, b)
            assert not np.isfinite(y[1, win]).any(), (bad, b)
        Hb = H.copy(); Hb[2, N // 3] = bad
        y, _ = ola_bank(dev, x, Hb, N, isz)
        assert np.array_equal(bits(y[:2]), bits(clean[:2])) and not np.isfinite(y[2]).any()


def sweep_bins(N, full_up_to, subset, rng):
    return impulse_columns(N, rng, full_up_to, subset) if N >= 16 else np.arange(N)


def check_ola_bin_sweep(dev, N, isz, full_up_to=256, subset=24, chunk=1024):
    """one block per channel, channel c's taps_fft a single bin k_c and its input one impulse: y = X_k H_k w^(-ki) / N, every output of the block
    (the emitted input_size and the carried tail) within the bound (mean |H| = |H_k| / N: as tight as the c2c bound).  Sweeping k runs every
    forward and inverse twiddle of the fused and staged kernels -- the radix-8 tables above 16 points are reached by no c2c call."""
    rng = np.random.default_rng(N + 3 * isz)
    bins = sweep_bins(N, full_up_to, subset, rng)
    form = ola_form(N)
    for a in range(0, bins.size, chunk):
        kk = bins[a:a + chunk]
        ch = kk.size
        H = np.zeros((ch, N), np.complex64); H[np.arange(ch), kk] = noise(rng, ch) * 2
        x = np.zeros((ch, isz), np.complex64); x[np.arange(ch), (np.arange(ch) * 7 + a) % isz] = 1
        y, tail = ola_bank(dev, x, H, N, isz)
        blk = np.zeros((ch, N), np.complex128); blk[:, :isz] = x
        want = np.fft.ifft(np.fft.fft(blk, axis=1) * H.astype(np.complex128), axis=1)
        bound = (2 * eps_fft(N, form) + 3 * U) * np.abs(H.astype(np.complex128)).mean(axis=1, keepdims=True) * np.ones((1, N))
        within(dev, ola_path(N) + " bin sweep", np.concatenate([y, tail[:, :N - isz]], axis=1), want, bound)


# ---- apply_fir_fft_cc ---------------------------------------------------------------------------------------------------------------------------
def apply_fir_fft(dev, x, H, last, ov):
    L = dev.L
    N = x.size
    x = np.ascontiguousarray(x); res = np.zeros(N, np.complex64); spec = np.zeros(N, np.complex64)
    fwd = L.make_fft_c2c(N, x.ctypes.data, spec.ctypes.data, 1, 1)
    inv = L.make_fft_c2c(N, spec.ctypes.data, res.ctypes.data, 0, 1)
    before = launches(dev)
    L.apply_fir_fft_cc(fwd, inv, np.ascontiguousarray(H).ctypes.data, last.ctypes.data, ov)
    assert launches(dev) - before == 1
    L.fft_destroy(fwd); L.fft_destroy(inv)
    return res


def check_apply_fir_fft_bin_sweep(dev, N, full_up_to=64, subset=12):
    """taps_fft a single bin k, input one impulse: every output within the (tight) bound, k swept as in check_ola_bin_sweep"""
    rng = np.random.default_rng(N + 23)
    for k in sweep_bins(N, full_up_to, subset, rng):
        H = np.zeros(N, np.complex64); H[k] = noise(rng, 1)[0] * 2
        x = np.zeros(N, np.complex64); x[(k * 5) % N] = 1
        res = apply_fir_fft(dev, x, H, np.zeros(1, np.complex64), 0)
        want = np.fft.ifft(np.fft.fft(x.astype(np.complex128)) * H.astype(np.complex128))
        within(dev, "apply_fir_fft bin sweep", res, want, np.full(N, block_conv_bound(x, H, "r8")))


def check_apply_fir_fft(dev, N):
    """the one-block kernel (radix-8 passes at every size): sparse block + the previous overlap, per-output bound"""
    rng = np.random.default_rng(N + 17)
    ov = N // 4
    H = noise(rng, N)
    for case in range(2):
        x = np.zeros(N, np.complex64)
        pos = boundary_positions(N, "r8")[:16] if case == 0 else rng.choice(N, min(N, 5), replace=False)
        x[pos] = noise(rng, len(pos)) * 2
        last = noise(rng, max(ov, 1))
        res = apply_fir_fft(dev, x, H, last, ov)
        want = np.fft.ifft(np.fft.fft(x.astype(np.complex128)) * H.astype(np.complex128))
        bound = np.full(N, block_conv_bound(x, H, "r8"))
        want[:ov] += last[:ov]
        bound[:ov] += U * np.abs(want[:ov])
        within(dev, "apply_fir_fft", res, want, bound)
    note(dev, "apply_fir_fft")


# ---- fastddc forward ----------------------------------------------------------------------------------------------------------------------------
def fastddc_fwd(dev, x, carry, N, isz, cuts=()):
    L = dev.L
    nb = x.size // isz
    ov = N - isz
    d_ov = dev.put(carry.astype(np.complex64) if ov else np.zeros(1, np.complex64))
    parts = []
    for a, b in zip([0] + list(cuts), list(cuts) + [nb]):
        d_x = dev.put(x[a * isz:b * isz]); d_sp = dev.alloc(8 * N * (b - a))
        before = launches(dev)
        assert L.csdrb_fastddc_fwd_cc(dev.ptr(d_x), dev.ptr(d_sp), dev.ptr(d_ov), N, isz, b - a, dev.stream) == 0, L.csdrb_last_error()
        assert launches(dev) - before == (2 if ov else 1)
        parts.append(dev.get(d_sp, np.complex64).reshape(b - a, N))
    note(dev, f"fastddc fwd {c2c_form(N)}")
    return np.concatenate(parts), dev.get(d_ov, np.complex64)[:ov]


def check_fastddc_fwd(dev, N, isz, nb):
    """the spectra of block b == csdrb_fft_c2c_batch on the explicit window, bit for bit; any cut into calls (calls shorter than the overlap
    included) changes nothing; a NaN/Inf sample damages exactly the blocks whose window holds it, and the carried overlap where it holds it"""
    rng = np.random.default_rng(N + isz)
    ov = N - isz
    x = noise(rng, nb * isz); carry = noise(rng, ov)
    stream = np.concatenate([carry, x])
    sp, c_out = fastddc_fwd(dev, x, carry, N, isz)
    win = np.stack([stream[b * isz:b * isz + N] for b in range(nb)])
    assert np.array_equal(bits(sp), bits(c2c(dev, win)))
    within(dev, f"fastddc fwd {c2c_form(N)}", sp, np.fft.fft(win.astype(np.complex128), axis=1), c2c_bound(win, c2c_form(N)))
    assert np.array_equal(bits(c_out), bits(stream[stream.size - ov:]))
    for cuts in ([1], list(range(1, nb))):
        sp2, c2 = fastddc_fwd(dev, x, carry, N, isz, cuts)
        assert np.array_equal(bits(sp2), bits(sp)) and np.array_equal(bits(c2), bits(c_out)), cuts
    for bad in (np.nan, np.inf):
        t = x.size - 1 - (isz // 3)
        z = x.copy(); z[t] = bad
        sp2, c2 = fastddc_fwd(dev, z, carry, N, isz)
        hit = np.array([b * isz <= ov + t < b * isz + N for b in range(nb)])
        assert hit.any() and np.array_equal(bits(sp2[~hit]), bits(sp[~hit])) and not np.isfinite(sp2[hit]).any()
        chit = np.arange(ov) == (ov + t) - (stream.size - ov)
        assert np.array_equal(bits(c2[~chit]), bits(c_out[~chit])) and not np.isfinite(c2[chit]).any()


# ---- fastddc inverse ----------------------------------------------------------------------------------------------------------------------------
# (bw, decimation, hand-set fft_inv_size or None): every row of the dispatch table of launch_fastddc_inv_bank.  fastddc_init never gives
# fft_inv_size below 16 when pre_decimation >= 2, so M = 8 (tiled) and M = 4 (generic) use the 1024-point geometry of (0.05, 8) with the
# frequency-domain decimation raised by hand.
INV_GEOMS = {
    "tiled M=8": (0.05, 8, 8), "tiled M=16": (0.1, 128, None), "tiled M=32": (0.05, 64, None),
    "fold M=64": (0.05, 32, None), "fold M=128 P=2": (0.2, 4, None), "fold M=256": (0.05, 8, None),
    "fold M=1024 post 3": (0.01, 12, None), "fold M=1024 post 5": (0.02, 10, None),
    "generic M=4": (0.05, 8, 4), "generic M=1024 P=1": (0.05, 3, None), "generic M=2048": (0.01, 6, None), "generic M=4096": (0.01, 2, None),
}
INV_SHIFTS = (-0.5, -0.2, -0.013, 0.0, 0.2, 0.4999)                     # offsetbin near +N/2, positive, zero, negative, near -N/2


def inv_geometry(dev, bw, dec, shift, hand_m=None):
    import csdr_b200
    g = csdr_b200.FastDDC()
    assert dev.L.fastddc_init(C.byref(g), bw, dec, shift) == 0
    if hand_m:
        g.fft_inv_size = hand_m; g.pre_decimation = g.fft_size // hand_m
        g.scrap = 1; g.post_input_size = hand_m - 1
    return g


def inv_channels(dev, name, shifts=INV_SHIFTS):
    bw, dec, hand = INV_GEOMS[name]
    gs = [inv_geometry(dev, bw, dec, s, hand) for s in shifts]
    chan = np.zeros(len(gs), CHAN_DT)
    for k, gk in enumerate(gs):
        chan[k] = (gk.offsetbin, gk.dsadata.sindelta, gk.dsadata.cosdelta, gk.dsadata.rate)
    return gs, chan


def inv_path(g, nblocks, channels):
    """launch_fastddc_inv_bank's dispatch (fastddc_inv_fold_ok, then the tiled kernel's tile rule, then the generic kernel)"""
    N, M = g.fft_size, g.fft_inv_size
    P = N // M
    if 64 <= M <= 1024 and P >= 2 and P % 2 == 0:
        return "fold"
    if 8 <= M <= 32 and P % 2 == 0:
        return "tiled 2x2" if -(-nblocks // 4) * -(-channels // 4) < 2 * SM_COUNT else "tiled 4x4"
    return "generic"


def inv_row_tags(g, path):
    """the rows of the path table a call exercises"""
    M, P = g.fft_inv_size, g.fft_size // g.fft_inv_size
    if path == "generic":
        return {"generic M<=4" if M <= 4 else ("generic P=1" if P == 1 else "generic M>=2048")}
    if path == "fold":
        return {"fold"} | ({"fold non-steady"} if g.post_input_size % g.post_decimation else set())
    return {path}


def run_inv(dev, g, sp, taps, chan, remain=None, phase=None):
    """csdrb_fastddc_inv_bank_cc: (out [C, stride], totals, remain, phase, path)"""
    L = dev.L
    nb, chn = sp.shape[0], chan.size
    ostride = nb * (g.post_input_size // g.post_decimation + 1) + 2
    d_sp = dev.put(sp); d_tf = dev.put(taps); d_chan = dev.put(chan.view(np.uint8))
    d_rem = dev.put(np.zeros(chn, np.int32) if remain is None else remain); d_ph = dev.put(np.zeros(chn, np.float32) if phase is None else phase)
    d_tot = dev.put(np.zeros(chn, np.int32)); d_out = dev.alloc(8 * chn * ostride)
    sb = L.csdrb_fastddc_inv_bank_scratch_bytes(chn, nb); d_scr = dev.alloc(sb + 16)
    before = launches(dev)
    rc = L.csdrb_fastddc_inv_bank_cc(dev.ptr(d_sp), nb, dev.ptr(d_tf), dev.ptr(d_chan), chn, C.byref(g), dev.ptr(d_rem), dev.ptr(d_ph), dev.ptr(d_out),
                                     ostride, dev.ptr(d_tot), dev.ptr(d_scr), sb, dev.stream)
    assert rc == 0, L.csdrb_last_error()
    path = inv_path(g, nb, chn)
    assert launches(dev) - before == (4 if path == "fold" else 2), (path, launches(dev) - before)         # fold: chain, phasors, fold, IFFT rows
    for tag in inv_row_tags(g, path):
        note(dev, "inv " + tag)
    return (dev.get(d_out, np.complex64).reshape(chn, ostride), dev.get(d_tot, np.int32), dev.get(d_rem, np.int32), dev.get(d_ph, np.float32), path)


def inv_bins(N, M, full):
    """single-bin blocks: every bin, or every residue mod M once (alias index varying) plus the half-swap edges"""
    if full:
        return np.arange(N)
    P = N // M
    res = range(M) if M <= 256 else sorted(set(range(0, M, M // 64)) | {1, M // 2 - 1, M // 2, M // 2 + 1, M - 1})
    return np.array(sorted({r + M * ((r * 7 + 3) % P) for r in res} | {0, N // 2 - 1, N // 2, N // 2 + 1, N - 1}))


def check_inv_bound(dev, oracle, name, full=False, shifts=INV_SHIFTS, expect=None):
    """single-bin spectra (each alias into its residue), then a few sparse multi-bin blocks, through every channel; per-output bound against
    the float64 model, output counts and the carried (remain, phase) against the oracle's chain"""
    gs, chan = inv_channels(dev, name, shifts)
    g = gs[0]
    N, M = g.fft_size, g.fft_inv_size
    rng = np.random.default_rng(N + M)
    bins = inv_bins(N, M, full)
    nb = bins.size + 4
    sp = np.zeros((nb, N), np.complex64)
    sp[np.arange(bins.size), bins] = noise(rng, bins.size) * 2
    for b in range(bins.size, nb):
        sp[b, rng.choice(N, 8, replace=False)] = noise(rng, 8)
    taps = noise(rng, len(gs), N)
    out, total, rem, ph, path = run_inv(dev, g, sp, taps, chan)
    if expect:
        assert path.startswith(expect), (name, path)                      # the tiled kernel's tile depends on the bank's size
    for c in range(len(gs)):
        want, bound, counts, r_end, p_end = fastddc_inv_model(oracle, sp, taps[c], chan[c], gs[c], path)
        assert total[c] == want.size == sum(counts), (c, total[c], want.size)
        within(dev, f"inv {path} M={M}", out[c, :want.size], want, bound)
        assert rel_rms(out[c, :want.size], want) < 5e-6
        assert rem[c] == r_end and bits(ph[c:c + 1])[0] == bits(np.array([p_end], np.float32))[0], (c, rem[c], r_end, ph[c], p_end)
    return gs, chan, sp, taps, out, total


def check_inv_channel_equals_one_channel(dev, name, nb, chn):
    """channel c of a bank == the one-channel bank on the same spectra, bit for bit (the tile shadowing of ragged edges must not matter)"""
    shifts = [INV_SHIFTS[c % len(INV_SHIFTS)] * (1 - 0.01 * c) for c in range(chn)]
    gs, chan = inv_channels(dev, name, shifts)
    g = gs[0]
    rng = np.random.default_rng(nb * 31 + chn)
    sp = noise(rng, nb, g.fft_size); taps = noise(rng, chn, g.fft_size)
    out, total, rem, ph, path = run_inv(dev, g, sp, taps, chan)
    for c in sorted({0, 1, chn // 2, chn - 2, chn - 1}):
        o1, t1, r1, p1, _ = run_inv(dev, g, sp, taps[c:c + 1], chan[c:c + 1])
        assert t1[0] == total[c] and r1[0] == rem[c] and bits(p1)[0] == bits(ph[c:c + 1])[0]
        assert np.array_equal(bits(o1[0, :t1[0]]), bits(out[c, :total[c]])), (name, c)
    return path


def check_inv_block_calls(dev, name, nb=200, chn=2):
    """one nb-block call == nb one-block calls carrying (remain, phase): outputs, totals, carried state.  More than 96 blocks: the state chain of
    the long call runs on its wrap tables, the one-block calls step by step."""
    gs, chan = inv_channels(dev, name, INV_SHIFTS[1:1 + chn])
    g = gs[0]
    rng = np.random.default_rng(nb + chn)
    sp = noise(rng, nb, g.fft_size); taps = noise(rng, chn, g.fft_size)
    out, total, rem, ph, _ = run_inv(dev, g, sp, taps, chan)
    r = np.zeros(chn, np.int32); p = np.zeros(chn, np.float32); got = [[] for _ in range(chn)]
    for b in range(nb):
        o, t, r, p, _ = run_inv(dev, g, sp[b:b + 1], taps, chan, r, p)
        for c in range(chn):
            got[c].append(o[c, :t[c]])
    assert np.array_equal(r, rem) and np.array_equal(bits(p), bits(ph))
    for c in range(chn):
        one = np.concatenate(got[c])
        assert one.size == total[c] and np.array_equal(bits(one), bits(out[c, :total[c]])), c


def check_inv_nonfinite(dev, oracle, name, nb, chn, bad_block, bad_chan):
    """a NaN/Inf bin in block b damages exactly block b's outputs of every channel (at its offset, its count); a bad taps row only its channel"""
    shifts = [INV_SHIFTS[c % len(INV_SHIFTS)] * (1 - 0.01 * c) for c in range(chn)]
    gs, chan = inv_channels(dev, name, shifts)
    g = gs[0]
    rng = np.random.default_rng(nb * 3 + chn)
    sp = noise(rng, nb, g.fft_size); taps = noise(rng, chn, g.fft_size)
    clean, total, _, _, path = run_inv(dev, g, sp, taps, chan)
    for bad in (np.nan, np.inf):
        z = sp.copy(); z[bad_block, g.fft_size // 3] = bad
        out, t2, _, _, _ = run_inv(dev, g, z, taps, chan)
        assert np.array_equal(t2, total)
        for c in range(chn):
            counts = [blk[1].size for blk in phasor_chain(oracle, gs[c], chan[c], nb, 0, 0.0)[0]]
            lo = sum(counts[:bad_block]); hi = lo + counts[bad_block]
            assert hi > lo and not np.isfinite(out[c, lo:hi]).any(), (bad, c)
            keep = np.r_[0:lo, hi:total[c]]
            assert np.array_equal(bits(out[c, keep]), bits(clean[c, keep])), (bad, c)
        tb = taps.copy(); tb[bad_chan, g.fft_size // 5] = bad
        out, _, _, _, _ = run_inv(dev, g, sp, tb, chan)
        for c in range(chn):
            if c == bad_chan:
                assert not np.isfinite(out[c, :total[c]]).any()
            else:
                assert np.array_equal(bits(out[c, :total[c]]), bits(clean[c, :total[c]])), c
    return path


# ---- the CPU tier -------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _ = emul_build.build_full_once(tmp_path_factory)
    return setup(S.EmulDev(C.CDLL(str(lib))))


@pytest.fixture(scope="module")
def oracle():
    return Oracle()


SIZES = [1 << k for k in range(1, 15)]


@pytest.mark.parametrize("N", SIZES)
def test_c2c_impulse_matrix(dev, N):
    check_c2c_impulse_matrix(dev, N, full_up_to=256, subset=24)


@pytest.mark.parametrize("N", SIZES)
def test_c2c_sparse_boundaries_and_tones(dev, N):
    check_c2c_sparse_and_tones(dev, N)


@pytest.mark.parametrize("N", SIZES)
def test_c2c_rows_alignment_conjugate_symmetry_and_nonfinite_rows(dev, N):
    check_c2c_invariants(dev, N)


# (N, input_size, nblocks): staged 4/8 points, fused R0 = 2/4/8 (hand-over at 64 and 512), fused16 at 256/4096, overlap > input_size, overlap 0,
# input_size 1; 33+ blocks so that the automatic 16-block CTA runs give three runs with lead-in recomputation
OLA_CPU = [(4, 3, 35), (8, 8, 33), (16, 1, 40), (32, 20, 35), (64, 20, 35), (128, 128, 33), (256, 100, 35), (512, 300, 34), (2048, 1500, 33),
           (4096, 2098, 33)]


@pytest.mark.parametrize("N,isz,nb", OLA_CPU)
def test_overlap_add_bank_bound(dev, N, isz, nb):
    assert nb >= 33 and auto_blocks_per_cta(2, nb) == 16                  # three CTA runs per channel
    check_ola(dev, N, isz, nb)


@pytest.mark.parametrize("N,isz,nb", [(8, 5, 19), (64, 20, 21), (256, 100, 18), (512, 512, 17)])
def test_overlap_add_bank_cuts_channels_and_shared_taps(dev, N, isz, nb):
    check_ola_invariants(dev, N, isz, nb)


@pytest.mark.parametrize("N,isz,nb", [(8, 3, 20), (64, 20, 20), (4096, 2098, 18)])
def test_overlap_add_bank_nonfinite_windows(dev, N, isz, nb):
    check_ola_nonfinite(dev, N, isz, nb)


@pytest.mark.parametrize("N,isz", [(4, 3), (8, 8), (16, 1), (32, 20), (64, 20), (128, 100), (256, 100), (512, 300), (1024, 1000), (2048, 1500),
                                   (4096, 2098), (8192, 7000)])
def test_overlap_add_single_bin_sweep(dev, N, isz):
    check_ola_bin_sweep(dev, N, isz)


@pytest.mark.parametrize("N", SIZES)
def test_apply_fir_fft_bound(dev, N):
    check_apply_fir_fft(dev, N)
    check_apply_fir_fft_bin_sweep(dev, N)


@pytest.mark.parametrize("N,isz,nb", [(8, 3, 6), (16, 12, 5), (64, 20, 6), (4096, 3000, 4)])
def test_fastddc_forward_is_the_c2c_of_its_window(dev, N, isz, nb):
    check_fastddc_fwd(dev, N, isz, nb)


@pytest.mark.parametrize("name", list(INV_GEOMS))
def test_fastddc_inverse_bound(dev, oracle, name):
    check_inv_bound(dev, oracle, name, full=False, expect=name.split(" M=")[0])


@pytest.mark.parametrize("name,nb,chn,expect", [("tiled M=16", 70, 67, "tiled 4x4"), ("tiled M=32", 7, 5, "tiled 2x2"), ("fold M=64", 21, 18, "fold"),
                                                ("generic M=1024 P=1", 3, 3, "generic")])
def test_fastddc_inverse_channel_equals_one_channel_bank(dev, name, nb, chn, expect):
    assert check_inv_channel_equals_one_channel(dev, name, nb, chn) == expect


@pytest.mark.parametrize("name", ["fold M=64", "tiled M=16"])
def test_fastddc_inverse_long_call_equals_one_block_calls(dev, name):
    check_inv_block_calls(dev, name)


@pytest.mark.parametrize("name,nb,chn,bad_block,bad_chan", [("fold M=64", 21, 18, 5, 17), ("tiled M=32", 7, 5, 6, 4), ("generic M=1024 P=1", 3, 2, 1, 0)])
def test_fastddc_inverse_nonfinite_windows(dev, oracle, name, nb, chn, bad_block, bad_chan):
    check_inv_nonfinite(dev, oracle, name, nb, chn, bad_block, bad_chan)


# every blocks_per_cta through the launcher itself (csdrb_bandpass_fir_fft_bank_cc always picks its own)
def test_overlap_add_every_blocks_per_cta(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    import test_kernels_emulated as K
    fft = K._lib(tmp_path_factory, "fft.cu", "alternate")
    P = lambda a: a.ctypes.data  # noqa: E731
    for N, isz, nb in [(4, 3, 7), (16, 1, 9), (64, 20, 8), (256, 100, 6), (512, 300, 5), (4096, 2098, 4)]:
        rng = np.random.default_rng(N)
        x = np.stack([ola_impulses(N, isz, nb, rng), noise(rng, nb * isz)]); H = noise(rng, 2, N)
        ref = None
        for bpc in range(1, nb + 1):
            y = np.zeros_like(x); tail = np.zeros((2, N), np.complex64)
            assert fft.emul_launch_olafir_bank(P(x), x.shape[1], P(y), y.shape[1], 2, N, isz, nb, P(H), N, P(tail), bpc) == 1, fft.emul_last_error()
            if ref is None:
                ref = (y, tail)
                for c in range(2):
                    want, bound = ola_model(x[c], H[c], N, isz, ola_form(N))
                    assert np.all(np.abs(y[c] - want) <= bound), (N, bpc, c)
            assert np.array_equal(y, ref[0]) and np.array_equal(tail[:, :N - isz], ref[1][:, :N - isz]), (N, bpc)


OLA_ROWS = {"ola staged", "ola fused R0=2", "ola fused R0=4", "ola fused R0=8 hand-over", "ola fused16"}
INV_ROWS = {"inv generic M<=4", "inv generic P=1", "inv generic M>=2048", "inv tiled 2x2", "inv tiled 4x4", "inv fold", "inv fold non-steady"}
ALL_ROWS = {"c2c r8", "c2c r16", "apply_fir_fft", "fastddc fwd r8", "fastddc fwd r16"} | OLA_ROWS | INV_ROWS

def check_coverage(dev):
    worst = getattr(dev, "worst", {})
    for k in sorted(worst):
        if worst[k]:
            print(f"worst error/bound  {k:40s} {worst[k]:.3f}")
    missing = ALL_ROWS - set(worst)
    assert not missing, f"path table rows never exercised: {sorted(missing)}"


def test_every_path_row_was_exercised(dev):
    """runs last in this file: every row of the path table was hit (and the worst error/bound ratio per path, printed with -s)"""
    check_coverage(dev)
