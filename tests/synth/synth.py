"""The checker side of the synthesis bank (csdr_b200/csrc/synth.cu), composed from the existing restatements.  TEST INFRASTRUCTURE.

  restate()      numpy, bit for bit: fir_interpolate_cc in the kernel's order (tests/tx/tx.py), shift_addition_cc's recursion (tests/shift_ref.py)
                 with the chunks counted on the absolute stream (output 0 `offset` samples into chunk 0; start phases from the oracle's float chain,
                 seeds (float)cos/sin in double), and the pairwise tree over the channel index in float32.
  ref_compose()  the same composition with the compiled reference's fir_interpolate_cc and shift_addition_cc (oracle/_ref), summed in float64.
  bound()        per output, how far the two may lie apart: the float64 interpolator bound of tests/tx/tx.py carried through the rotation, the
                 rotations' own rounding, and the tree's gamma(ceil(log2 C)) * sum_c |Y_c|.
"""
from __future__ import annotations

import math
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent / "tx"))
import shift_ref  # noqa: E402
import tx  # noqa: E402

F32 = np.float32
U = 2.0 ** -24
SQ2 = math.sqrt(2.0)
MARGIN = 1 + 1e-3


def h_of(I, T):
    return (T - 1 + I - 1) // I


def nout_of(n, I, T):
    return tx.groups(n, I, T) * I


def chunk_starts(oracle, rate, ph0, nout, chunk, offset):
    """start phase of every absolute chunk the call touches (one more than those holding an output), and the phase at the start of the chunk
    that contains output nout"""
    K = -(-(offset + nout) // chunk) + 1
    starts, _ = oracle.shift_chain(float(shift_ref.inc1(rate)), float(ph0), K * chunk, chunk)
    return starts, F32(starts[(offset + nout) // chunk]) if nout else F32(ph0)


def shifted(oracle, W, rate, ph0, chunk, offset):
    """shift_addition_cc of one interpolated row W, chunks on the absolute stream: (Y, carried phase)"""
    N = W.size
    starts, end = chunk_starts(oracle, rate, ph0, N, chunk, offset)
    if N == 0:
        return np.zeros(0, np.complex64), end
    seeds, _, _ = oracle.seed_phasors(starts)
    K = -(-(offset + N) // chunk)
    X = np.zeros(K * chunk, np.complex64)
    X[offset:offset + N] = W
    prm = np.array(oracle.shift_addition_init(float(rate)), F32)
    d = np.array([prm[1], prm[0]], F32)                                  # (cosd, sind)
    Y = shift_ref.mix_addition(X.reshape(K, chunk), seeds[:K], d[None, :])
    return Y.reshape(-1)[offset:offset + N], end


def tree_sum(Y):
    """the pairwise tree over the channel index (axis 0), float32 per component; a node with one present child is that child"""
    Y = np.array(Y, np.complex64, copy=True)
    C = Y.shape[0]
    s = 1
    with np.errstate(all="ignore"):
        while s < C:
            for b in range(0, C - s, 2 * s):
                Y[b] = Y[b] + Y[b + s]
            s *= 2
    return Y[0] if C else np.zeros(Y.shape[1:], np.complex64)


def restate(oracle, x, rates, I, taps, phases=None, chunk=1024, offset=0, per_channel=False):
    """(y, carried phases) of the synthesis bank on x [C, n]; per_channel: also the rows Y_c before the sum"""
    x = np.asarray(x, np.complex64)
    C, n = x.shape
    ph = np.zeros(C, F32) if phases is None else np.asarray(phases, F32)
    Ys, ends = [], np.empty(C, F32)
    for c in range(C):
        W = tx.fir_interpolate_cc(x[c], I, taps)
        Y, ends[c] = shifted(oracle, W, float(rates[c]), ph[c], chunk, offset)
        Ys.append(Y)
    Y = np.stack(Ys) if C else np.zeros((0, 0), np.complex64)
    y = tree_sum(Y)
    return (y, ends, Y) if per_channel else (y, ends)


# ---- the compiled reference --------------------------------------------------------------------------------------------------------------
def have_ref() -> bool:
    return tx.have_ref()


def ref_compose(refo, x, rates, I, taps, phases=None, chunk=1024, offset=0):
    """the reference's fir_interpolate_cc, then its shift_addition_cc once per absolute chunk, summed over the channels in float64; also the
    rows |Y_c| for the bound"""
    x = np.asarray(x, np.complex64)
    C, n = x.shape
    ph = np.zeros(C, F32) if phases is None else np.asarray(phases, F32)
    total, rows = None, []
    for c in range(C):
        W = tx.ref_fir_interpolate_cc(x[c], I, taps)
        N = W.size
        K = -(-(offset + N) // chunk)
        X = np.zeros(K * chunk, np.complex64)
        X[offset:offset + N] = W
        Y, _ = refo.shift_addition_cc(X, float(rates[c]), float(ph[c]), chunk)
        Y = Y[offset:offset + N].astype(np.complex128)
        rows.append(Y)
        total = Y if total is None else total + Y
    return total, np.stack(rows)


def bound(x, rates, I, taps, Y, chunk):
    """per output, the distance allowed between the kernel's y and the float64 sum of the reference composition.  Per channel: the two
    interpolations lie within tx.interp_bound (bi, bq) of each other, a rotation by a phasor |p| <= G moves that by at most G |dW|, each side's
    rotation of W rounds within 2 sqrt2 u G |W| (1 + u), and a seed of either side may sit one float ulp off (sqrt2 u G |W|), G = 1 + 4 (chunk + 2) u
    the recursion's growth over a chunk.  The tree adds gamma(ceil(log2 C)) * sum_c (|Re Y_c| + |Im Y_c|) per component."""
    x = np.asarray(x, np.complex64)
    C = x.shape[0]
    G = 1 + 4 * (chunk + 2) * U
    tot = None
    absY = np.zeros(Y.shape[1]) if C else None
    for c in range(C):
        bi, bq = tx.interp_bound(x[c], I, taps)
        dW = np.hypot(bi, bq)
        W = np.abs(tx.fir_interpolate_cc(x[c], I, taps).astype(np.complex128))
        b = G * dW + (2 * 2 * SQ2 * U * (1 + U) + SQ2 * U) * G * (W + dW)
        tot = b if tot is None else tot + b
        absY += np.abs(Y[c].real) + np.abs(Y[c].imag) + 2 * b
    L = math.ceil(math.log2(C)) if C > 1 else 0
    gam = L * U / (1 - L * U)
    return (tot + SQ2 * gam * absY) * MARGIN
