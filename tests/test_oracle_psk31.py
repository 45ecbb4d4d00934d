"""CPU tier: the BPSK31 checker (tests/psk31/psk31_oracle.c) pinned to the compiled reference (oracle/_ref/libcsdr_ref.so).
timing_recovery_cc, dbpsk_decoder_c_u8 and the varicode decoder are bit-exact; simple_agc_cc differs only through the reference build's
rsqrtss seed (DESIGN.md section 7), so its gains are held to a relative bound."""
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "psk31"))
import psk31  # noqa: E402

pytestmark = pytest.mark.skipif(not psk31.have_ref(), reason="oracle/_ref/libcsdr_ref.so not built (needs the reference sources at build time)")


def bits_of(a):
    return np.ascontiguousarray(a).view(np.uint8)


def with_specials(x, rng):
    f = x.view(np.float32)
    for v in (0.0, np.nan, np.inf, -np.inf):
        f[rng.integers(0, f.size, 4)] = v
    x[rng.integers(0, x.size, 4)] = 0
    return x


@pytest.mark.parametrize("sps", [8, 12, 256, 1024])
def test_simple_agc_within_bound(sps):
    rng = np.random.default_rng(sps)
    x = psk31.modulate(rng.integers(0, 2, 40), sps, rng, freq=0.1 / sps)
    x = with_specials(x, rng)
    for rate, ref_, mg in [(0.001, 0.5, 65535.0), (0.05, 1.0, 3.0)]:
        y, g = psk31.simple_agc_cc(x, rate, ref_, mg)
        yr, gr = psk31.ref_simple_agc_cc(x, rate, ref_, mg)
        fin = np.isfinite(yr.view(np.float32)).reshape(-1, 2).all(1)
        assert np.array_equal(np.isfinite(y.view(np.float32)), np.isfinite(yr.view(np.float32)))
        assert np.max(np.abs(y[fin] - yr[fin]) / np.maximum(np.abs(yr[fin]), 1e-30)) < 2e-5
        assert abs(g - gr) <= 2e-5 * abs(gr)


@pytest.mark.parametrize("sps", [8, 12, 256, 1024])
@pytest.mark.parametrize("alg", [psk31.GARDNER, psk31.EARLYLATE])
@pytest.mark.parametrize("use_q", [False, True])
def test_timing_recovery_bit_exact(sps, alg, use_q):
    rng = np.random.default_rng(sps * 4 + alg * 2 + use_q)
    x = psk31.modulate(rng.integers(0, 2, 60), sps, rng, freq=0.1 / sps)
    for xs in (x, with_specials(x.copy(), rng)):
        for co in (0, sps // 8, -sps // 4 + 1):
            for gain, me in [(0.5, 2.0), (0.25, 1.0), (1.0, 1.0), (1.0, 2.0), (-0.5, 4.0)]:
                got = psk31.timing_recovery_cc(xs, alg, sps, use_q, gain, me, co)
                want = psk31.ref_timing_recovery_cc(xs, alg, sps, use_q, gain, me, co)
                assert got[3] == want[3]
                for a, b in zip(got[:3], want[:3]):
                    assert np.array_equal(bits_of(a), bits_of(b))


def test_timing_recovery_split_invariance():
    """the CLI re-presents the unconsumed input; any split of the stream gives the symbols of one call over all of it"""
    rng = np.random.default_rng(7)
    sps = 16
    x = psk31.modulate(rng.integers(0, 2, 300), sps, rng, freq=0.003)
    y1, e1, i1, _ = psk31.timing_recovery_cc(x, psk31.GARDNER, sps)
    for trial in range(5):
        calls = list(rng.integers(2 * sps, 20 * sps, 400))
        y2, e2, i2, _ = psk31.timing_stream(x, psk31.GARDNER, sps, calls)
        m = y2.size
        assert m >= y1.size - 2
        assert np.array_equal(bits_of(y2), bits_of(y1[:m])) and np.array_equal(i2, i1[:m]) and np.array_equal(bits_of(e2), bits_of(e1[:m]))


def test_dbpsk_bits_equal_reference():
    rng = np.random.default_rng(3)
    x = (rng.standard_normal(20000) + 1j * rng.standard_normal(20000)).astype(np.complex64)
    x = with_specials(x, rng)
    # phase steps right at +-pi/2 and +-pi
    ang = np.array([np.pi / 2, -np.pi / 2, np.pi, -np.pi, np.pi / 2 + 1e-7], np.float64)
    extra = np.exp(1j * np.cumsum(np.repeat(ang, 20))).astype(np.complex64)
    x = np.concatenate([x, extra])
    for last in (0j, 1 + 1j):
        got, _ = psk31.dbpsk_decoder_c_u8(x, last)
        want = psk31.ref_dbpsk_decoder_c_u8(x, last)
        bad = np.nonzero(got != want)[0]
        prev = np.concatenate([[np.complex64(last)], x[:-1]])
        for i in bad:                                                   # only a phase step within a few ulps of +-pi/2 may decide differently
            d = np.float32(np.arctan2(x[i].imag, x[i].real)) - np.float32(np.arctan2(prev[i].imag, prev[i].real))
            d = (d + np.pi) % (2 * np.pi) - np.pi
            assert abs(abs(d) - np.pi / 2) < 1e-6, (i, d)


def test_varicode_table_and_decoder_equal_reference():
    for a, (code, bits) in enumerate(psk31.varicode_table()):
        enc = psk31.ref_varicode_encode(bytes([a]))
        assert list(enc) == [(code >> (bits - 1 - k)) & 1 for k in range(bits)] + [0, 0], a
    text = bytes(range(128))
    enc = psk31.ref_varicode_encode(text)
    assert psk31.varicode_decode(enc) == psk31.ref_varicode_decode(enc)
    assert psk31.varicode_decode(enc)[0] == text[1:]
    rng = np.random.default_rng(5)
    for k in range(4):
        b = rng.integers(0, 2, 5000).astype(np.uint8) * rng.integers(1, 256, 5000).astype(np.uint8)
        h = int(rng.integers(0, 2 ** 63))
        assert psk31.varicode_decode(b, h) == psk31.ref_varicode_decode(b, h)


def test_chain_decodes_seeded_text():
    rng = np.random.default_rng(31)
    text = b"CQ CQ CQ de TEST TEST pse k"
    x = psk31.modulate(psk31.ref_varicode_encode(text), 256, rng, freq=0.2 / (2 * np.pi * 256), noise=0.03)
    assert text in psk31.chain(x, 256)
