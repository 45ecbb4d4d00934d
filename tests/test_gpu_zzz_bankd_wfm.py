"""GPU tests (-m gpu) of csdr-bankd's WFM tail (--tail wfm [--wfm-rate R] [--tau T], csdr_b200/host/bankd.c): three FM stations, each modulated
by its own tone, in one u8 or f32 wideband stream.  Each sink's s16 audio must be exactly the checker (tests/wfm: fractional_decimator_ff R 12 |
deemphasis_wfm_ff 48000 T | convert_f_s16 in 1024-sample calls) run on the daemon's own discriminator output for the same arguments -- what it
writes with --tail none; --devices gives the same bytes; the combinations the daemon refuses exit with a message; and on the GPU only, the
README's 2.4 Msps receiver is held against the compiled reference's whole CLI pipe per station, each station's audio peaking at its own tone.
tests/test_bankd_wfm_emulated.py runs the same bodies except the last on the emulated library."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from test_gpu_zzz_bankd import bankd  # noqa: F401  (the fixture)
import test_gpu_zzz_bankd as base

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "wfm"))
import wfm as W  # noqa: E402

REF_CLI = ROOT / "oracle" / "_ref" / "csdr_ref"
RATES = (-0.085, 0.0, 0.2)                                          # the --help example's channels
TONES = (1000.0, 2500.0, 4000.0)
FS, D, BW = 2.4e6, 10, 0.05


def wideband(n, seed, fmt, deviation=15e3):
    """three FM stations at -RATES of a 2.4 Msps stream, station k modulated by TONES[k] with `deviation` Hz peak, plus a little noise"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    z = sum(0.25 * np.exp(1j * (2 * np.pi * (-r) * t + deviation / f * np.sin(2 * np.pi * f / FS * t) + rng.uniform(0, 2 * np.pi)))
            for r, f in zip(RATES, TONES))
    z = z + 0.003 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    if fmt == "f32":
        return z.astype(np.complex64).tobytes()
    iq = np.empty(2 * n); iq[0::2] = z.real; iq[1::2] = z.imag
    return np.clip(np.floor(iq * 127.5 + 128), 0, 255).astype(np.uint8).tobytes()


def run(bankd, args, data, sinks, timeout=900):
    cmd = [bankd] + args + [f"{r}:{p}" for r, p in zip(RATES, sinks)]
    r = subprocess.run(cmd, input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=timeout)
    assert r.returncode == 0, r.stderr[-2000:]


def audio(bankd, tmp_path, args, wfm_args, data, tag):
    """(s16 audio per channel from --tail wfm, the daemon's discriminator output per channel from --tail none)"""
    raw = [tmp_path / f"{tag}_raw{k}.f32" for k in range(len(RATES))]
    pcm = [tmp_path / f"{tag}_{k}.s16" for k in range(len(RATES))]
    run(bankd, ["--tail", "none"] + args, data, raw)
    run(bankd, ["--tail", "wfm"] + wfm_args + args, data, pcm)
    return [np.fromfile(p, np.int16) for p in pcm], [np.fromfile(p, np.float32) for p in raw]


@pytest.mark.parametrize("fmt", ["u8", "f32"])
@pytest.mark.parametrize("block", [16384, 40000])
@pytest.mark.parametrize("rate", [5.0, 5.2083333])
def test_wfm_tail_equals_the_checker_on_the_banks_discriminator(bankd, oracle, tmp_path, fmt, block, rate):
    data = wideband(max(4 * block, 110000) + 12345, 3, fmt)
    args = [f"--{fmt}", "--decimation", str(D), "--bw", str(BW), "--block", str(block)]
    tau = 75e-6 if rate != 5.0 else 50e-6
    wfm_args = [] if rate == 5.0 else ["--wfm-rate", str(rate), "--tau", str(tau)]
    got, raw = audio(bankd, tmp_path, args, wfm_args, data, f"{fmt}{block}")
    for g, d in zip(got, raw):
        want = W.checker(oracle, d, rate, 1024, tau)
        assert g.size == want.size and g.size > 2000
        assert np.array_equal(g, want)


def test_wfm_tail_over_several_devices(bankd, tmp_path):
    """--devices: the slices return discriminator rows and the tail runs on the first device -- the single-device bytes"""
    data = wideband(5 * 16384, 4, "u8")
    args = ["--u8", "--decimation", str(D), "--bw", str(BW), "--block", "16384", "--tail", "wfm"]
    one = [tmp_path / f"one{k}.s16" for k in range(len(RATES))]
    run(bankd, args, data, one)
    assert all(p.stat().st_size > 2000 for p in one)
    for devices in base.MULTI_DEVICES():
        many = [tmp_path / f"m{devices.replace(',', '_')}{k}.s16" for k in range(len(RATES))]
        run(bankd, args + ["--devices", devices], data, many)
        for a, b in zip(one, many):
            assert a.read_bytes() == b.read_bytes(), devices


def test_wfm_refusals(bankd, tmp_path):
    for args in (["--tail", "wfm", "--resample", "3:4"], ["--tail", "nfm", "--wfm-rate", "5"], ["--tail", "none", "--tau", "75e-6"],
                 ["--wfm-rate", "5"], ["--tail", "wfm", "--wfm-rate", "1"], ["--tail", "wfm", "--wfm-rate", "0.5"],
                 ["--tail", "wfm", "--wfm-rate", "16.01"], ["--tail", "wfm", "--wfm-rate", "40"], ["--tail", "wfm", "--wfm-rate", "nan"],
                 ["--tail", "wfm", "--tau", "0"], ["--tail", "wfm", "--tau", "-50e-6"]):
        r = subprocess.run([bankd] + args + [f"0.1:{tmp_path / 'x.s16'}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode != 0 and b"csdr-bankd:" in r.stderr, args
    for args in (["--tail", "wfm", "--wfm-rate", "16"], ["--tail", "wfm", "--wfm-rate", "1.01", "--tau", "75e-6"]):
        r = subprocess.run([bankd] + args + [f"0.1:{tmp_path / 'y.s16'}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode == 0, (args, r.stderr)


def test_three_stations_against_the_reference_cli(bankd, oracle, tmp_path):
    """the --help example, --decimation 10 --bw 0.05 --tail wfm at 2.4 Msps, against the compiled reference's whole pipe per station: within
    1 count over the common prefix (the discriminators differ by float rounding between the fused DDC bank and fir_decimate_cc); every
    station's audio peaks at its own tone"""
    if not REF_CLI.exists():
        pytest.skip("oracle/_ref/csdr_ref not built")
    block = 1 << 18
    data = wideband(12 * block, 5, "u8", deviation=10e3)               # 1.3 s
    pcm = [tmp_path / f"st{k}.s16" for k in range(len(RATES))]
    run(bankd, ["--u8", "--decimation", str(D), "--bw", str(BW), "--block", str(block), "--tail", "wfm"], data, pcm)
    for k, (r, tone, p) in enumerate(zip(RATES, TONES, pcm)):
        got = np.fromfile(p, np.int16)
        stages = ["convert_u8_f", f"shift_addition_cc {r}", f"fir_decimate_cc {D} {BW} HAMMING", "fmdemod_quadri_cf", "fractional_decimator_ff 5",
                  "deemphasis_wfm_ff 48000 50e-6", "convert_f_s16"]
        cmd = " | ".join(f"{REF_CLI} {s}" for s in stages)
        res = subprocess.run(["bash", "-c", cmd], input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=900,
                             env={"PATH": "/usr/bin:/bin"})
        assert res.returncode == 0, res.stderr[-2000:]
        want = np.frombuffer(res.stdout, np.int16)
        m = min(got.size, want.size)
        assert m > 0.95 * got.size and got.size > 48000
        diff = np.abs(got[:m].astype(np.int32) - want[:m].astype(np.int32))
        print(f"station {k} at {r}: {np.count_nonzero(diff)} of {m} samples differ from the reference CLI pipe, largest by {diff.max()}")
        assert diff.max() <= 1
        a = got[2048:].astype(np.float64)
        spec = np.abs(np.fft.rfft(a * np.hanning(a.size)))
        freqs = np.fft.rfftfreq(a.size, 1 / 48000.0)
        band = (freqs > 200) & (freqs < 15000)
        assert abs(freqs[band][np.argmax(spec[band])] - tone) < 20, (k, tone)
