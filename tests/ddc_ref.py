"""Reference helpers and the shared case matrix of the fused DDC bank tests (tests/test_ddc_bank_emulated.py, tests/test_gpu_ddc_bank.py).

The fused bank computes, per channel c and output o,
    y_c[o] = sum_k h[k] * x[oD + k] * p_c[oD + k]
where p_c is the reference NCO: shift_addition_cc's float recursion, re-seeded from the float phase chain at every chunk boundary.  Every output
depends only on its own samples and phasors, so the result must not depend on how the work is cut: channels per lane (CPL), segments, channel
sets, channel count or block split.  The helpers give
    * nco():        the phasor sequence, bit for bit (the oracle's shift_addition_cc run on ones),
    * baseband64(): the FIR of x*p in float64 from the exact float32 values,
    * bound():      a per-output, per-component error bound of the kernel's float32 arithmetic against baseband64().
"""
import numpy as np

from bitcmp import U, assert_bits_equal, bits  # noqa: F401  (re-exported for the DDC bank test modules)

KERNELS = [(50, 17), (10, 8), (10, 20)]                              # the compiled (D, M) instantiations of ddc_bank_fused2_kernel
T_VALUES = {50: [1, 49, 50, 751, 800, 801, 850], 10: [1, 9, 10, 79, 80, 81, 199, 200]}
CHANNELS = [1, 31, 32, 33, 63, 64, 65, 97, 129]
# (chunk, offset): chunk boundaries at the block start and one sample in, chunks shorter than the 10-sample unrolled group, one sample per chunk,
# chunk = 0 (the whole block is one chunk) and a chunk longer than the block
CHUNKS = [(1024, 0), (1024, 1023), (1000, 999), (13, 12), (7, 3), (1, 0), (0, 0), (1 << 20, 12345)]
SIZES = ["T", "T+D-1", "T+D", "ragged", "ragged2", "large"]


def kernel_for(D, T):
    """the (D, M) instantiation launch_ddc_main picks"""
    if D == 50:
        return (50, 17)
    return (10, 8) if T <= 80 else (10, 20)


def input_size(kind, D, T, large):
    """wideband block length for a size kind; `large` = number of outputs of the large block"""
    return {"T": T, "T+D-1": T + D - 1, "T+D": T + D,
            "ragged": T + 3 * D + 7,                                 # never a multiple of 10: the unrolled groups end inside a period
            "ragged2": T + 5 * D + 3,
            "large": T + (large - 1) * D + D - 3}[kind]


def cases(large=120, extra=(), chain_budget=None):
    """two cases per T of every kernel, each run with both DEMOD values: all channel counts, (chunk, offset) pairs and size kinds appear.
    `chain_budget` caps channels x chunks of a case (the serial phase chain is what the CPU emulation spends its time on with short chunks):
    the block is shortened towards T, then the channel count lowered to the largest entry of CHANNELS that fits.
    The three lists are walked with strides prime to their lengths, so every entry of each appears and the combinations differ from T to T."""
    out = []
    i = 0
    for D in (50, 10):
        for T in T_VALUES[D]:
            for rep in range(2):
                ch = CHANNELS[(7 * i) % len(CHANNELS)]
                chunk, offset = CHUNKS[(3 * i) % len(CHUNKS)]
                kind = SIZES[(5 * i) % len(SIZES)]
                n = input_size(kind, D, T, large)
                if chunk == 1:
                    n = min(n, T + 20 * D)                           # one chunk per sample: keep the serial phase chain short
                if chain_budget and 0 < chunk < n:
                    nch = lambda n: (offset + n) // chunk + 1
                    n = max(T, min(n, (chain_budget // ch) * chunk - offset))
                    ch = max([1] + [c for c in CHANNELS if c * nch(n) <= chain_budget and c <= ch])
                out.append(dict(D=D, T=T, channels=ch, chunk=chunk, offset=offset, n=n, seed=1000 * D + 10 * T + rep))
                i += 1
    out.extend(extra)
    return out


def case_id(c):
    return f"D{c['D']}-T{c['T']}-ch{c['channels']}-chunk{c['chunk']}+{c['offset']}-n{c['n']}"


def rates_for(channels, rng):
    """rates from -0.4999 to 0.4999 with the edges, 0, 1e-4 and +-0.25 among them"""
    special = np.array([-0.4999, 0.4999, 0.0, 1e-4, 0.25, -0.25], np.float32)
    r = rng.uniform(-0.4999, 0.4999, channels).astype(np.float32)
    r[:min(channels, special.size)] = special[:channels]
    return rng.permutation(r)


def make_inputs(case, firdes=None):
    """wideband block, rates, starting phases, last_in and taps of a case.  Taps: uniform(-1, 1) so that every tap (the last one included) matters;
    `firdes` = the product's lowpass taps of that length instead."""
    rng = np.random.default_rng(case["seed"])
    n, ch, T = case["n"], case["channels"], case["T"]
    x = (rng.uniform(-1, 1, n) + 1j * rng.uniform(-1, 1, n)).astype(np.complex64)
    rates = rates_for(ch, rng)
    ph0 = rng.uniform(-3.1, 3.1, ch).astype(np.float32)
    last = (rng.uniform(-1, 1, ch) + 1j * rng.uniform(-1, 1, ch)).astype(np.complex64)
    taps = firdes if firdes is not None else rng.uniform(-1, 1, T).astype(np.float32)
    return x, rates, ph0, last, np.ascontiguousarray(taps, np.float32)


def n_out_of(n, D, T):
    return (n - T) // D + 1 if n >= T else 0


def nco(oracle, rate, phase0, chunk, offset, n):
    """the reference phasors (cos, sin) of n samples of a block that starts `offset` samples into its chunk, chunk 0 starting at phase0: the oracle's
    shift_addition_cc on ones, called once per chunk like the CLI (the rotation of 1 + 0j is the phasor itself, exactly)"""
    ones = np.ones(offset + n, np.complex64)
    y, _ = oracle.shift_addition_cc(ones, float(rate), float(phase0), chunk if chunk > 0 else None)
    return y[offset:]


def carried_phase(oracle, rate, phase0, chunk, offset, n, D, T):
    """the phase at the start of the chunk that holds the next block's first sample (offset + n_out*D samples in), as the bank returns it"""
    if chunk <= 0:
        chunk = n
    nxt = (offset + n_out_of(n, D, T) * D) // chunk
    if nxt == 0:
        return np.float32(phase0)
    _, ph = oracle.shift_addition_cc(np.ones(nxt * chunk, np.complex64), float(rate), float(phase0), chunk)
    return np.float32(ph)


def _windows(a, T, D, n_out):
    return np.lib.stride_tricks.sliding_window_view(a, T)[::D][:n_out]


def baseband64(x, p, taps, D):
    """float64 fir_decimate of the shifted stream x*p, from the exact float32 values of x and p: y[o] = sum_k h[k] x[oD+k] p[oD+k]"""
    T = taps.size
    n_out = n_out_of(x.size, D, T)
    s = x.astype(np.complex128) * p.astype(np.complex128)
    return _windows(s, T, D, n_out) @ taps.astype(np.float64)


def bound(x, p, taps, D):
    """per-output, per-component bound of |kernel - baseband64| (same value for the I and the Q component).

    The kernel forms each shifted sample with one rounded product and one fused multiply-add,
        sh.i = fl(p.i*x.i + fl(-p.q*x.q)),   sh.q = fl(p.q*x.i + fl(p.i*x.q)),
    so |sh - x*p| <= 2u(1+u) m_k a_k per component, with a_k = |x.i| + |x.q|, m_k = max(|p.i|, |p.q|) and u = 2^-24; note |(x*p)_k| <= m_k a_k.
    Each output then is a serial chain of T fused multiply-adds acc = fl(acc + h_k sh_k) in sample order (taps beyond T are zero and add
    nothing), whose error is at most gamma_T sum_k |h_k sh_k| with gamma_T = Tu / (1 - Tu).  Together
        |y - y64| <= (gamma_T (1 + 2u(1+u)) + 2u(1+u)) sum_k |h_k| m_k a_k  <=  (T + 2) u (1 + 1e-3) sum_k |h_k| m_k a_k
    for T <= 850.  The float64 reference adds ~T 2^-53 relative, far inside the 1e-3 margin."""
    T = taps.size
    n_out = n_out_of(x.size, D, T)
    a = (np.abs(x.real) + np.abs(x.imag)).astype(np.float64) * np.maximum(np.abs(p.real), np.abs(p.imag)).astype(np.float64)
    return (T + 2) * U * (1 + 1e-3) * (_windows(a, T, D, n_out) @ np.abs(taps.astype(np.float64)))


def check_against_reference(oracle, case, x, rates, ph0, last, taps, base, phase, demod, demod_phase, last_out):
    """every assertion that needs only the oracle: the baseband (demod = 0 run) within bound() of the float64 reference at every output, the carried
    phases bit for bit, and the demod run = fmdemod_quadri_cf on the bank's own baseband, bit for bit, last_out included"""
    D, T, chunk, offset = case["D"], case["T"], case["chunk"], case["offset"]
    n_out = n_out_of(x.size, D, T)
    assert base.shape == (rates.size, n_out) and demod.shape == (rates.size, n_out)
    for c, r in enumerate(rates):
        p = nco(oracle, r, ph0[c], chunk, offset, x.size)
        want = baseband64(x, p, taps, D)
        bnd = bound(x, p, taps, D)
        got = base[c].astype(np.complex128)
        err = np.maximum(np.abs(got.real - want.real), np.abs(got.imag - want.imag))
        worst = int(np.argmax(err / bnd))
        assert np.all(err <= bnd), (c, float(r), "output", worst, float(err[worst]), float(bnd[worst]))
        wph = carried_phase(oracle, r, ph0[c], chunk, offset, x.size, D, T)
        assert bits(np.float32(phase[c])) == bits(wph), (c, float(r), float(phase[c]), float(wph))
        assert bits(np.float32(demod_phase[c])) == bits(wph), c
        wd, wl = oracle.fmdemod_quadri_cf(base[c], complex(last[c]))
        assert_bits_equal(demod[c], wd, f"demod of channel {c}")
        assert_bits_equal(np.complex64(last_out[c]), np.complex64(wl), f"last_out of channel {c}")


NONFINITE = [(50, 801), (50, 51), (10, 79), (10, 9), (10, 199), (10, 81)]     # every (D, M) kernel, a full and a nearly empty last tap block


def nonfinite_positions(D, T, n):
    """wideband samples to poison: just past output 5's window, at its last zero-padded tap (D*M - 1), a sample in mid-window of a later output,
    the first and the last sample of the block"""
    M = kernel_for(D, T)[1]
    pos = {5 * D + T, 5 * D + D * M - 1, 40 * D + T // 2 + 1, 0, n - 1}
    return sorted(p for p in pos if 0 <= p < n)


def check_nonfinite(run, case):
    """NaN, +Inf and -Inf in the wideband block (in turn, on the I or the Q component): with demod off exactly the outputs whose window
    [oD, oD + T) holds one are non-finite and every other output keeps the clean run's bits; with demod on every output whose own or previous
    baseband sample is clean keeps its bits, last_out included.  run(x, rates, ph0, last, taps, demod) -> (out, last_out or None)."""
    D, T = case["D"], case["T"]
    x, rates, ph0, last, taps = make_inputs(case)
    n = x.size
    pos = nonfinite_positions(D, T, n)
    xp = x.copy()
    bad = [np.nan, np.inf, -np.inf]
    for i, p in enumerate(pos):
        xp[p] = complex(bad[i % 3], 0.5) if i % 2 == 0 else complex(-0.25, bad[i % 3])
    n_out = n_out_of(n, D, T)
    o = np.arange(n_out)
    hit = np.zeros(n_out, bool)
    for p in pos:
        hit |= (o * D <= p) & (p < o * D + T)
    what = f"D={D} T={T} chunk {case['chunk']}+{case['offset']}"
    base0, _ = run(x, rates, ph0, last, taps, 0)
    base1, _ = run(xp, rates, ph0, last, taps, 0)
    for c in range(rates.size):
        fin = np.isfinite(base1[c].real) & np.isfinite(base1[c].imag)
        assert np.array_equal(~fin, hit), f"{what} channel {c}: non-finite outputs {np.flatnonzero(~fin)[:12]}, expected {np.flatnonzero(hit)[:12]}"
    assert_bits_equal(base1[:, ~hit], base0[:, ~hit], f"{what}: baseband away from the poisoned samples")
    dem0, lo0 = run(x, rates, ph0, last, taps, 1)
    dem1, lo1 = run(xp, rates, ph0, last, taps, 1)
    near = hit | np.concatenate([[False], hit[:-1]])
    assert_bits_equal(dem1[:, ~near], dem0[:, ~near], f"{what}: discriminator away from the poisoned samples")
    if not hit[-1]:
        assert_bits_equal(lo1, lo0, f"{what}: last_out")
