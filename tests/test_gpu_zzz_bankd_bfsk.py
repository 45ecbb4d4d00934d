"""GPU tests (-m gpu) of csdr-bankd's RTTY tail with tone filters (--tail rtty --bfsk SPACING:LENGTH, csdr_b200/host/bankd.c): three RTTY
signals at different offsets of one u8 or f32 wideband stream.  Each sink's text must be exactly what our csdr CLI gives stage by stage,
`bfsk_demod_cf | serial_line_decoder_f_u8 | rtty_baudot2ascii_u8_u8`, on the daemon's own baseband (--tail iq), and the same as the whole pipe
`shift_addition_cc | fir_decimate_cc | bfsk_demod_cf | ...` on the wideband stream; it must contain the sent text.  --devices gives the same
bytes, --bfsk with another tail is refused, and in noise where the discriminator tail garbles the text the tone filters make fewer errors.
tests/test_bankd_bfsk_emulated.py runs the same bodies on the emulated library."""
import os
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
D, BW, SPB, B = 10, 0.05, 20.0, 1024                               # 200 wideband samples per bit; the decoder's calls of B samples
SPACING, L = 0.187, 20                                             # 170 Hz at 45.45 Bd and 20 samples per bit: 0.187 cycles per sample
BFSK = f"{SPACING}:{L}"
CLI = Path(__file__).resolve().parent.parent / "csdr_b200" / "csdr"


def wideband(seed, fmt, text=TEXT, noise=0.01, block=16384):
    """an idle mark after the text covers what the daemon cannot decode yet: the last B baseband samples and the partial last block it drops"""
    rng = np.random.default_rng(seed)
    sigs = [rtty.modulate(text, SPB * D, rng, freq=-r, noise=0.0, amplitude=0.25, lead_bits=float(rng.uniform(2, 6)),
                          tail_bits=((B + 8) * D + block) / (SPB * D) + 4, gap=2.0 * D) for r in RATES]
    n = min(s.size for s in sigs)
    z = sum(s[:n].astype(np.complex128) for s in sigs) + noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    if fmt == "f32":
        return z.astype(np.complex64).tobytes()
    iq = np.empty(2 * n); iq[0::2] = z.real; iq[1::2] = z.imag
    return np.clip(np.floor(iq * 127.5 + 128), 0, 255).astype(np.uint8).tobytes()


def run(bankd, args, data, sinks, timeout=900):
    cmd = [bankd] + args + [f"{r}:{p}" for r, p in zip(RATES, sinks)]
    r = subprocess.run(cmd, input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=timeout)
    assert r.returncode == 0, r.stderr[-2000:]


def pipe(stages, data):
    e = dict(os.environ); e["CSDR_FIXED_BUFSIZE"] = str(B)
    c = str(CLI)
    r = subprocess.run(["bash", "-c", " | ".join(f"{c} {s}" for s in stages)], input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       env=e, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    return r.stdout


DECODE = [f"bfsk_demod_cf {SPACING} {L}", f"serial_line_decoder_f_u8 {SPB} 5 1.5", "rtty_baudot2ascii_u8_u8"]


def bfsk_texts(bankd, tmp_path, args, data, tag):
    txt = [tmp_path / f"{tag}_{k}.txt" for k in range(len(RATES))]
    run(bankd, ["--tail", "rtty", "--sps", str(SPB), "--rtty-bufsize", str(B), "--bfsk", BFSK] + args, data, txt)
    return [p.read_bytes() for p in txt]


@pytest.mark.parametrize("fmt,block", [("u8", 16384), ("f32", 40000)])
def test_bfsk_tail_equals_the_cli_pipe(bankd, tmp_path, fmt, block):
    data = wideband(3, fmt, block=block)
    args = [f"--{fmt}", "--decimation", str(D), "--bw", str(BW), "--block", str(block)]
    got = bfsk_texts(bankd, tmp_path, args, data, f"{fmt}{block}")
    iq = [tmp_path / f"{fmt}{block}_iq{k}.cf" for k in range(len(RATES))]
    run(bankd, ["--tail", "iq"] + args, data, iq)
    for g, p in zip(got, iq):
        assert g == pipe(DECODE, p.read_bytes())
        assert TEXT in g, g
    if fmt == "f32":                                               # the whole chain of the CLI on the wideband stream
        for g, r in zip(got, RATES):
            assert g == pipe([f"shift_addition_cc {r}", f"fir_decimate_cc {D} {BW}"] + DECODE, data), r


def test_bfsk_tail_over_several_devices(bankd, tmp_path):
    data = wideband(4, "u8")
    args = ["--u8", "--decimation", str(D), "--bw", str(BW), "--block", "16384"]
    one = bfsk_texts(bankd, tmp_path, args, data, "one")
    assert all(TEXT in t for t in one)
    for devices in base.MULTI_DEVICES():
        assert bfsk_texts(bankd, tmp_path, args + ["--devices", devices], data, "m" + devices.replace(",", "_")) == one, devices


def test_bfsk_refusals(bankd, tmp_path):
    for args in (["--tail", "nfm", "--bfsk", BFSK], ["--tail", "iq", "--bfsk", BFSK], ["--tail", "rtty", "--sps", "44", "--bfsk", "0.085"],
                 ["--tail", "rtty", "--sps", "44", "--bfsk", "0.085:1"], ["--tail", "rtty", "--sps", "44", "--bfsk", "0.085:4097"],
                 ["--tail", "rtty", "--sps", "44", "--bfsk", "0:44"], ["--tail", "rtty", "--sps", "44", "--bfsk", "1.5:44"]):
        r = subprocess.run([bankd] + args + [f"0.1:{tmp_path / 'x.txt'}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode != 0 and b"csdr-bankd:" in r.stderr and b"--bfsk" in r.stderr, args


def edits(a: bytes, b: bytes) -> int:
    """Levenshtein distance: characters lost, garbled or invented"""
    prev = list(range(len(b) + 1))
    for i, ca in enumerate(a, 1):
        cur = [i]
        for j, cb in enumerate(b, 1):
            cur.append(min(prev[j] + 1, cur[j - 1] + 1, prev[j - 1] + (ca != cb)))
        prev = cur
    return prev[-1]


NOISY = 0.3                                                        # about 3 dB SNR in the 240 Hz a tone filter passes


def test_tone_filters_beat_the_discriminator_in_noise(bankd, tmp_path):
    """the same noisy stream through --tail rtty with and without --bfsk: character errors against the sent text, per channel, for this
    seed (the counts are what the seeded stream gives; the point is that the tone filters' are lower)"""
    text = TEXT + b" " + TEXT
    data = wideband(8, "f32", text=text, noise=NOISY)
    args = ["--f32", "--decimation", str(D), "--bw", str(BW), "--block", "16384", "--tail", "rtty", "--sps", str(SPB), "--rtty-bufsize", str(B)]
    disc = [tmp_path / f"disc{k}.txt" for k in range(len(RATES))]
    tone = [tmp_path / f"tone{k}.txt" for k in range(len(RATES))]
    run(bankd, args, data, disc)
    run(bankd, args + ["--bfsk", BFSK], data, tone)
    e_disc = [edits(p.read_bytes(), text) for p in disc]
    e_tone = [edits(p.read_bytes(), text) for p in tone]
    assert (e_disc, e_tone) == ([15, 15, 33], [10, 6, 3])
    assert sum(e_tone) < sum(e_disc)
