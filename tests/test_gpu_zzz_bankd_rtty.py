"""GPU tests (-m gpu) of csdr-bankd's RTTY tail (--tail rtty --sps F, csdr_b200/host/bankd.c): three RTTY signals at different offsets of one
u8 or f32 wideband stream, two block sizes, two --rtty-bufsize values.  Each sink's text must be exactly the checker's chain (tests/rtty) run on
the DDC bank's own discriminator output for the same stream -- what the daemon itself writes with --tail none -- and must contain the seeded
text; --devices gives the same bytes; the combinations the daemon refuses exit with a message.  tests/test_bankd_rtty_emulated.py runs the same
bodies on the emulated library."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from test_gpu_zzz_bankd import bankd  # noqa: F401  (the fixture)
import test_gpu_zzz_bankd as base

pytestmark = pytest.mark.gpu
sys.path.insert(0, str(Path(__file__).resolve().parent / "rtty"))
import rtty  # noqa: E402

RATES = (-0.3, 0.05, 0.25)
TEXT = b"CQ DE K1ABC/P 599 73"
D, BW, SPB = 10, 0.05, 20.0                                       # 200 wideband samples per bit


def wideband(spb_wide, seed, fmt, text=TEXT, tail_wide=0, dec=D):
    """an idle mark after the text covers what the daemon cannot decode yet: the last --rtty-bufsize baseband samples and the partial last
    block it drops; 2 baseband samples of mark follow each character (rtty.modulate's gap)"""
    rng = np.random.default_rng(seed)
    sigs = [rtty.modulate(text, spb_wide, rng, freq=-r, noise=0.0, amplitude=0.25, lead_bits=float(rng.uniform(2, 6)),
                          tail_bits=tail_wide / spb_wide + 4, gap=2.0 * dec) for r in RATES]
    n = min(s.size for s in sigs)
    z = sum(s[:n].astype(np.complex128) for s in sigs) + 0.01 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    if fmt == "f32":
        return z.astype(np.complex64).tobytes()
    iq = np.empty(2 * n); iq[0::2] = z.real; iq[1::2] = z.imag
    return np.clip(np.floor(iq * 127.5 + 128), 0, 255).astype(np.uint8).tobytes()


def run(bankd, args, data, sinks, timeout=900):
    cmd = [bankd] + args + [f"{r}:{p}" for r, p in zip(RATES, sinks)]
    r = subprocess.run(cmd, input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=timeout)
    assert r.returncode == 0, r.stderr[-2000:]


def decode(bankd, tmp_path, args, data, spb, bufsize, tag):
    """(text per channel from --tail rtty, the checker's decoder on the bank's discriminator output from --tail none)"""
    raw = [tmp_path / f"{tag}_raw{k}.f32" for k in range(len(RATES))]
    txt = [tmp_path / f"{tag}_{k}.txt" for k in range(len(RATES))]
    run(bankd, ["--tail", "none"] + args, data, raw)
    run(bankd, ["--tail", "rtty", "--sps", str(spb), "--rtty-bufsize", str(bufsize)] + args, data, txt)
    want = [rtty.baudot_decode(rtty.serial_stream(np.fromfile(p, np.float32), spb, 5, 1.5, 0.4, bufsize)[0])[0] for p in raw]
    return [p.read_bytes() for p in txt], want


@pytest.mark.parametrize("fmt", ["u8", "f32"])
@pytest.mark.parametrize("block", [16384, 40000])
@pytest.mark.parametrize("bufsize", [256, 1024])
def test_rtty_tail_equals_the_checker_on_the_banks_discriminator(bankd, tmp_path, fmt, block, bufsize):
    data = wideband(SPB * D, 3, fmt, tail_wide=(bufsize + 8) * D + block)
    args = [f"--{fmt}", "--decimation", str(D), "--bw", str(BW), "--block", str(block)]
    got, want = decode(bankd, tmp_path, args, data, SPB, bufsize, f"{fmt}{block}_{bufsize}")
    for g, w in zip(got, want):
        assert g == w
        assert TEXT in g, g


def test_rtty_tail_over_several_devices(bankd, tmp_path):
    """--devices: the slices return discriminator rows and the tail runs on the first device -- the single-device bytes"""
    data = wideband(SPB * D, 4, "u8", tail_wide=300 * D + 16384)
    args = ["--u8", "--decimation", str(D), "--bw", str(BW), "--block", "16384", "--tail", "rtty", "--sps", str(SPB), "--rtty-bufsize", "256"]
    one = [tmp_path / f"one{k}.txt" for k in range(len(RATES))]
    run(bankd, args, data, one)
    assert all(TEXT in p.read_bytes() for p in one)
    for devices in base.MULTI_DEVICES():
        many = [tmp_path / f"m{devices.replace(',', '_')}{k}.txt" for k in range(len(RATES))]
        run(bankd, args + ["--devices", devices], data, many)
        for a, b in zip(one, many):
            assert a.read_bytes() == b.read_bytes(), devices


def test_rtty_refusals(bankd, tmp_path):
    for args in (["--tail", "rtty"], ["--tail", "rtty", "--sps", "0.5"], ["--tail", "rtty", "--sps", "44", "--databits", "9"],
                 ["--tail", "rtty", "--sps", "44", "--databits", "0"], ["--tail", "rtty", "--sps", "44", "--stopbits", "0.5"],
                 ["--tail", "rtty", "--sps", "44", "--rtty-bufsize", "332"], ["--tail", "rtty", "--sps", "44", "--resample", "3:4"],
                 ["--tail", "nfm", "--databits", "5"], ["--tail", "bpsk31", "--sps", "32", "--rtty-bufsize", "1024"]):
        r = subprocess.run([bankd] + args + [f"0.1:{tmp_path / 'x.txt'}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode != 0 and b"csdr-bankd:" in r.stderr, args
    # sps*(1 + 5 + 1.5) + 2 = 332 is refused above; one sample more is served
    r = subprocess.run([bankd, "--tail", "rtty", "--sps", "44", "--rtty-bufsize", "333", f"0.1:{tmp_path / 'y.txt'}"], input=b"",
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
    assert r.returncode == 0, r.stderr


def test_rtty_skimmer_geometry_of_the_help(bankd, tmp_path):
    """the worked example: 2.4 Msps, --decimation 1200 --bw 0.001 (2 kHz baseband, 4001 taps, M = 4), --sps 44 (45.45 Bd), the default
    --rtty-bufsize of 16384"""
    data = wideband(44 * 1200, 5, "u8", b"CQ TEST", tail_wide=(16384 + 300) * 1200 + (1 << 18), dec=1200)
    args = ["--u8", "--decimation", "1200", "--bw", "0.001"]
    got, want = decode(bankd, tmp_path, args, data, 44.0, 16384, "skim")
    for g, w in zip(got, want):
        assert g == w and b"CQ TEST" in g, g
