"""The case matrix of the fused DDC bank at every served decimation (tests/test_ddc_generic_emulated.py, tests/test_gpu_ddc_generic.py).

Decimation 50 up to 850 taps and 10 up to 200 taps keep their own kernels, ddc_bank_fused2_kernel<D, M, CPL, DEMOD>; every other geometry the bank
serves runs ddc_bank_generic_kernel<M, CPL, DEMOD>, with D a kernel argument and M the smallest bucket >= ceil(T/D).  The contract is the one of
tests/ddc_ref.py, unchanged.  kernel_for() and nonfinite_positions() here know the generic buckets; the rest comes from ddc_ref.
"""
from ddc_ref import CHANNELS, CHUNKS, n_out_of

BUCKETS = [4, 8, 12, 17, 20, 24]                                     # kDdcBuckets (csrc/ddc_bank.cu)
CAPACITY = 8000                                                      # kDdcTapCapacity: D * MP taps of a generic geometry
D_VALUES = [2, 4, 6, 12, 40, 48, 52, 126, 200, 400]


def mp(m):
    return (m + 1) & ~1


def bucket_of(D, T):
    """the generic bucket of (D, T), or None when the bank refuses the geometry"""
    if D <= 0 or D % 2 or T <= 0:
        return None
    m = -(-T // D)
    for b in BUCKETS:
        if m <= b:
            return b if D * mp(b) <= CAPACITY else None
    return None


def kernel_for(D, T):
    """the kernel launch_ddc_main picks: ("fused2", D, M) or ("generic", M_bucket)"""
    if D == 50 and T <= 850:
        return ("fused2", 50, 17)
    if D == 10 and T <= 80:
        return ("fused2", 10, 8)
    if D == 10 and T <= 200:
        return ("fused2", 10, 20)
    b = bucket_of(D, T)
    return None if b is None else ("generic", b)


def bucket_edges(D):
    """T at the edges of every bucket that D can use: 1, D-1, D, D+1, then (M_b - 1) D + 1 (the first T of M = M_b) and M_b D (the last of the bucket)"""
    ts = {1, D - 1, D, D + 1}
    for b in BUCKETS:
        ts |= {(b - 1) * D + 1, b * D}
    return sorted(t for t in ts if t >= 1 and kernel_for(D, t) and kernel_for(D, t)[0] == "generic")


def cases(outputs, extra=(), chain_budget=None, max_wide=None):
    """one case per (D, T) of bucket_edges plus D = 10 beyond 200 taps.  `outputs` = outputs of a block (fewer for long filters when `max_wide`
    caps the block's samples); channel counts, (chunk, offset) pairs and block remainders rotate through the lists of tests/ddc_ref.py.
    `chain_budget` caps channels x chunks (the serial phase chain the CPU emulation spends its time on with short chunks), as ddc_ref.cases does."""
    geoms = [(D, T) for D in D_VALUES for T in bucket_edges(D)] + [(10, 201), (10, 240)]
    out = []
    for i, (D, T) in enumerate(geoms):
        ch = CHANNELS[(7 * i) % len(CHANNELS)]
        chunk, offset = CHUNKS[(3 * i) % len(CHUNKS)]
        k = outputs
        if max_wide:
            k = max(3, min(k, (max_wide - T) // D))
        n = T + (k - 1) * D + (i % D if D > 1 else 0)                # a remainder of 0 .. D-1 samples that no output uses
        if chain_budget and 0 < chunk < n:
            nch = lambda n: (offset + n) // chunk + 1
            n = max(T, min(n, (chain_budget // ch) * chunk - offset))
            ch = max([1] + [c for c in CHANNELS if c * nch(n) <= chain_budget and c <= ch])
        out.append(dict(D=D, T=T, channels=ch, chunk=chunk, offset=offset, n=n, seed=100_000 * D + T))
    out.extend(extra)
    return out


# one geometry per bucket (two for 17), among them the largest D * MP served (400 x 20 = 8000) and decimation 10 beyond its own kernels
NONFINITE = [(2, 7), (6, 37), (12, 97), (48, 769), (52, 833), (126, 2395), (400, 8000), (10, 231)]


def nonfinite_positions(D, T, n):
    """wideband samples to poison: just past output 5's window, at the last zero-padded tap of the bucket's M (5D + D*M_b - 1), a sample in
    mid-window of a later output, the first and the last sample of the block"""
    M = kernel_for(D, T)[-1]
    pos = {5 * D + T, 5 * D + D * M - 1, 40 * D + T // 2 + 1, 0, n - 1}
    return sorted(p for p in pos if 0 <= p < n)


def expected_ctas(channels, n_out, D, T, cpl, sm_count=132):
    """the grid launch_ddc_main computes: segments sized to fill sm_count x (resident warps per SM) warps, at least 2M outputs each, one warp per
    (segment, channel set); 12 resident warps for the D = 50 / 10 kernels, four per CTA of the bucket's __launch_bounds__ for the generic one"""
    k = kernel_for(D, T)
    M = k[-1]
    if k[0] == "fused2":
        warps = 12
    elif cpl == 1:
        warps = 4 * (6 if M <= 8 else 5 if M <= 12 else 4 if M <= 20 else 3)
    else:
        warps = 4 * (5 if M <= 4 else 4 if M <= 8 else 3 if M <= 17 else 2)
    wps = -(-channels // (32 * cpl))
    want = -(-sm_count * warps // wps)
    seg = max(-(-n_out // want), 2 * M)
    return (-(-n_out // seg) * wps + 3) // 4


def n_out(case):
    return n_out_of(case["n"], case["D"], case["T"])


def case_id(c):
    return f"D{c['D']}-T{c['T']}-ch{c['channels']}-chunk{c['chunk']}+{c['offset']}-n{c['n']}"


