"""GPU tests (-m gpu) of csdr-bankd's BPSK31 tail (--tail bpsk31 --sps N, csdr_b200/host/bankd.c): three PSK31 signals at different offsets of one
u8 or f32 wideband stream, two block sizes.  Each sink's text must be exactly the checker's chain (tests/psk31) run on the DDC bank's own baseband
for the same stream -- the baseband the daemon itself writes with --tail iq -- and must contain the seeded text; --devices gives the same bytes; the
combinations the daemon refuses exit with a message.  tests/test_bankd_psk31_emulated.py runs the same bodies on the emulated library."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from test_gpu_zzz_bankd import bankd  # noqa: F401  (the fixture)
import test_gpu_zzz_bankd as base

pytestmark = pytest.mark.gpu
sys.path.insert(0, str(Path(__file__).resolve().parent / "psk31"))
import psk31  # noqa: E402

RATES = (-0.3, 0.05, 0.25)
TEXT = b"CQ de TEST k"
D, BW, SPS = 10, 0.05, 32                                          # 320 wideband samples per symbol


def wideband(sps_wide, seed, fmt, text=TEXT, tail=160):
    """idle reversals after the text cover the partial last block the daemon drops"""
    rng = np.random.default_rng(seed)
    bits = psk31.ref_varicode_encode(text)
    sigs = [psk31.modulate(bits, sps_wide, rng, freq=-r + 0.2 / (2 * np.pi * sps_wide), noise=0.0, amplitude=0.25, lead=96, tail=tail) for r in RATES]
    n = min(s.size for s in sigs)
    z = sum(s[:n].astype(np.complex128) for s in sigs) + 0.01 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    if fmt == "f32":
        return z.astype(np.complex64).tobytes()
    iq = np.empty(2 * n); iq[0::2] = z.real; iq[1::2] = z.imag
    return np.clip(np.floor(iq * 127.5 + 128), 0, 255).astype(np.uint8).tobytes()


def run(bankd, args, data, sinks, timeout=600):
    cmd = [bankd] + args + [f"{r}:{p}" for r, p in zip(RATES, sinks)]
    r = subprocess.run(cmd, input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=timeout)
    assert r.returncode == 0, r.stderr[-2000:]


def decode(bankd, tmp_path, args, data, sps, tag):
    """(text per channel from --tail bpsk31, the checker's chain on the bank's baseband from --tail iq)"""
    iq = [tmp_path / f"{tag}_iq{k}.cf32" for k in range(len(RATES))]
    txt = [tmp_path / f"{tag}_{k}.txt" for k in range(len(RATES))]
    run(bankd, ["--tail", "iq"] + args, data, iq)
    run(bankd, ["--tail", "bpsk31", "--sps", str(sps)] + args, data, txt)
    want = [psk31.chain(np.fromfile(p, np.complex64), sps) for p in iq]
    return [p.read_bytes() for p in txt], want


@pytest.mark.parametrize("fmt", ["u8", "f32"])
@pytest.mark.parametrize("block", [16384, 40000])
def test_bpsk31_tail_equals_the_checker_on_the_banks_baseband(bankd, tmp_path, fmt, block):
    data = wideband(SPS * D, 3, fmt)
    args = [f"--{fmt}", "--decimation", str(D), "--bw", str(BW), "--block", str(block)]
    got, want = decode(bankd, tmp_path, args, data, SPS, f"{fmt}{block}")
    for g, w in zip(got, want):
        assert g == w
        assert TEXT in g, g


def test_bpsk31_tail_over_several_devices(bankd, tmp_path):
    """--devices: the slices return baseband and the tail runs on the first device -- the single-device bytes"""
    data = wideband(SPS * D, 4, "u8")
    args = ["--u8", "--decimation", str(D), "--bw", str(BW), "--block", "16384", "--tail", "bpsk31", "--sps", str(SPS)]
    one = [tmp_path / f"one{k}.txt" for k in range(len(RATES))]
    run(bankd, args, data, one)
    assert all(TEXT in p.read_bytes() for p in one)
    for devices in base.MULTI_DEVICES():
        many = [tmp_path / f"m{devices.replace(',', '_')}{k}.txt" for k in range(len(RATES))]
        run(bankd, args + ["--devices", devices], data, many)
        for a, b in zip(one, many):
            assert a.read_bytes() == b.read_bytes(), devices


def test_bpsk31_refusals(bankd, tmp_path):
    for args in (["--tail", "bpsk31"], ["--tail", "bpsk31", "--sps", "30"], ["--tail", "bpsk31", "--sps", "4"],
                 ["--tail", "bpsk31", "--sps", "32", "--resample", "3:4"], ["--tail", "nfm", "--sps", "32"]):
        r = subprocess.run([bankd] + args + [f"0.1:{tmp_path / 'x.txt'}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode != 0 and b"csdr-bankd:" in r.stderr, args


def test_bpsk31_skimmer_geometry_of_the_help(bankd, tmp_path):
    """the worked example: 2.4 Msps, --decimation 300 --bw 0.001 (8 kHz baseband, 4001 taps, M = 14), --sps 256 (31.25 Bd)"""
    data = wideband(256 * 300, 5, "u8", b"CQ TEST", tail=16)
    args = ["--u8", "--decimation", "300", "--bw", "0.001"]
    got, want = decode(bankd, tmp_path, args, data, 256, "skim")
    for g, w in zip(got, want):
        assert g == w and b"CQ TEST" in g, g
