"""CPU tier: the RTTY checker (tests/rtty/rtty_oracle.c) pinned to the compiled reference (oracle/_ref/libcsdr_ref.so) bit for bit --
serial_line_decoder_f_u8's characters and input_used over random, noisy and adversarial inputs, window sums at +-0 and tiny values, NaN and
+-Inf inside windows, characters cut by the end of a call, every parameter the CLI accepts in range; rtty_baudot_decoder_lookup over all
256 inputs in both modes -- and the reference's own CLI pipe decoding the seeded text, which shows that its RTTY chain is complete."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "rtty"))
import rtty  # noqa: E402

pytestmark = pytest.mark.skipif(not rtty.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built (needs the reference sources at build time)")

TEXT = b"RYRYRY CQ CQ DE TEST TEST 599 73, 14.080 MHZ (K1ABC/P) 'OK?' = 100 + -5 $1 #2 @3 *4 :5\r\n"


def same(x, spb, databits, stopbits, ratio):
    got = rtty.serial_line_decoder(x, spb, databits, stopbits, ratio)
    want = rtty.ref_serial_line_decoder(x, spb, databits, stopbits, ratio)
    assert got == want, (spb, databits, stopbits, ratio, got, want)
    return got


def heavy(rng, n):
    """random signs over 80 decades: any other summation order changes some window's sign"""
    return (rng.standard_normal(n) * 10.0 ** rng.uniform(-30, 30, n)).astype(np.float32)


def levels(rng, n, spb, p0=0.5):
    """a noisy square wave with bit-long runs of +-1, edges where the runs change"""
    bits = rng.random(int(n / spb) + 2) < p0
    lev = np.repeat(np.where(bits, 1.0, -1.0), int(np.ceil(spb)))[:n]
    return (lev + 0.8 * rng.standard_normal(n)).astype(np.float32)


@pytest.mark.parametrize("spb", [5.0, 44.0, 176.02])
@pytest.mark.parametrize("databits,stopbits", [(5, 1.5), (7, 1.0), (8, 2.0), (5, 1.0), (1, 1.0)])
def test_serial_line_decoder_bit_exact(spb, databits, stopbits):
    rng = np.random.default_rng(int(spb * 100) + databits * 10 + int(stopbits * 2))
    for ratio in (0.4, 0.0, 1.0, 0.37, 0.93):
        for n in (0, 1, 2, 3, 17, int(spb * 9), 3000, 16384):
            for x in (heavy(rng, n), levels(rng, n, spb), rng.standard_normal(n).astype(np.float32)):
                same(x, spb, databits, stopbits, ratio)


def test_window_sums_at_zero_and_tiny_values():
    """windows whose sum is +-0, a denormal or cancels exactly: the sign decides the bit (> 0) and the stop test (< 0)"""
    rng = np.random.default_rng(2)
    tiny = np.array([0.0, -0.0, 1e-45, -1e-45, 1.4e-45, -3e-38, 3e-38, 1.0, -1.0, 1e30, -1e30], np.float32)
    for spb in (5.0, 8.0, 44.0):
        for _ in range(200):
            n = int(rng.integers(40, 400))
            x = rng.choice(tiny, n).astype(np.float32)
            x[rng.integers(1, n, 8)] = -1.0                                   # edges
            for databits, stopbits in ((5, 1.5), (8, 1.0), (7, 2.0)):
                same(x, spb, databits, stopbits, 0.4)


def test_nan_and_inf_inside_windows():
    rng = np.random.default_rng(3)
    for spb in (5.0, 44.0):
        for _ in range(60):
            x = levels(rng, 4000, spb)
            for v in (np.nan, np.inf, -np.inf):
                x[rng.integers(0, x.size, 6)] = v
            for databits, stopbits, ratio in ((5, 1.5, 0.4), (8, 1.0, 1.0), (7, 2.0, 0.0)):
                same(x, spb, databits, stopbits, ratio)
    # a NaN before a negative sample is an edge in the build (comiss), not in the source
    x = np.array([1, 1, np.nan, -1, -1, -1, -1, -1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1], np.float32)
    assert same(x, 2.0, 5, 1.0, 0.4) == rtty.ref_serial_line_decoder(x, 2.0, 5, 1.0, 0.4)


def test_characters_cut_by_the_end_of_a_call():
    """an RTTY signal decoded in calls of every size from one character to many: the 'does not fit' and 'faulty stop bit' returns and
    what they consume, at every cut"""
    rng = np.random.default_rng(4)
    for spb in (5.0, 44.0, 176.02):
        d = rtty.discriminator(rtty.modulate(TEXT[:30], spb, rng, noise=0.1))
        pos = 0
        while pos < d.size:
            n = int(rng.integers(1, int(12 * spb)))
            _, used = same(d[pos:pos + n], spb, 5, 1.5, 0.4)
            pos += max(used, 1)


def test_baudot_lookup_all_inputs():
    for mode in (0, 1):
        for c in range(256):
            assert rtty.baudot_lookup(c, mode) == rtty.ref_baudot_lookup(c, mode), (c, mode)


def test_checker_chain_decodes_seeded_text():
    rng = np.random.default_rng(31)
    for spb, noise in ((44.0, 0.01), (176.02, 0.003), (5.0, 0.01)):
        z = rtty.modulate(TEXT, spb, rng, freq=0.001, noise=noise, tail_bits=16384 / spb + 2)
        assert TEXT in rtty.chain(z, spb), spb


def test_reference_pipe_decodes_seeded_text():
    """fmdemod_quadri_cf | serial_line_decoder_f_u8 44 5 1.5 | rtty_baudot2ascii_u8_u8 of the unmodified reference CLI"""
    if not rtty.REF_CLI.exists():
        pytest.skip("oracle/_ref/csdr_ref not built")
    rng = np.random.default_rng(45)
    z = rtty.modulate(TEXT, 44.0, rng, freq=0.002, noise=0.01, tail_bits=16384 / 44 + 2)
    cli = str(rtty.REF_CLI)
    r = subprocess.run(["bash", "-c", f"{cli} fmdemod_quadri_cf | {cli} serial_line_decoder_f_u8 44 5 1.5 | {cli} rtty_baudot2ascii_u8_u8"],
                       input=z.tobytes(), stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=120)
    assert r.returncode == 0, r.stderr
    assert TEXT in r.stdout, r.stdout
