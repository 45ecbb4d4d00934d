"""GPU tests (-m gpu) of csdr-bankd --s8, HackRF's signed 8-bit IQ: every sink must hold the bytes of the same daemon run with --f32 on the
stream converted by the reference's convert_s8_f, on the single-GPU path (the bytes converted on the device) and with --devices (converted on
the host), for the nfm, usb, iq and wfm tails, two block sizes and the waterfall; the input flags stay last-flag-wins; and a HackRF-like
10 Msps stream with three NFM stations comes out one station per channel at --decimation 200 --resample 24:25.
The bodies but the last also run on the emulated library (tests/test_bankd_s8_emulated.py)."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent / "formats"))
import formats as M  # noqa: E402
import test_gpu_zzz_bankd as base  # noqa: E402  (stream generator, runner, device lists)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
bankd = base.bankd
N, CHANNELS = 3 * 16384 + 1000, 2
D10 = ["--decimation", "10", "--bw", "0.05"]


def s8_stream(n, seed):
    """HackRF-style s8 IQ of the test stations, and the same stream as cf32 through the reference's convert_s8_f"""
    s8 = (base.wideband_u8(n, seed=seed).astype(np.int16) - 128).astype(np.int8)
    f = M.ref_call("s8_f", s8.view(np.uint8)) if M.have_ref() else M.s8_f(s8)
    return s8.tobytes(), np.asarray(f, np.float32).tobytes()


def sinks_of(bankd, tmp_path, tag, args, data, waterfall=False):
    sinks = [tmp_path / f"{tag}{k}.out" for k in range(CHANNELS)]
    extra = ["--waterfall", str(tmp_path / f"{tag}.wf"), "--fft-size", "1024"] if waterfall else []
    base.run(bankd, args + extra, data, sinks)
    return [p.read_bytes() for p in sinks] + ([(tmp_path / f"{tag}.wf").read_bytes()] if waterfall else [])


@pytest.mark.parametrize("tail", ["nfm", "usb", "iq", "wfm"])
@pytest.mark.parametrize("block", [16384, 20000])
def test_s8_equals_f32_of_the_converted_stream(bankd, tmp_path, tail, block):
    s8, f32 = s8_stream(N, seed=41)
    args = ["--block", str(block), "--tail", tail] + D10
    want = sinks_of(bankd, tmp_path, "f32", args + ["--f32"], f32, waterfall=tail == "nfm")
    assert all(len(w) > 0 for w in want)
    got = sinks_of(bankd, tmp_path, "s8", args + ["--s8"], s8, waterfall=tail == "nfm")
    assert got == want, tail
    multi = sinks_of(bankd, tmp_path, "s8dev", args + ["--s8", "--devices", base.MULTI_DEVICES()[-1]], s8, waterfall=tail == "nfm")
    assert multi == want, (tail, "--devices")


def test_input_flags_stay_last_flag_wins(bankd, tmp_path):
    s8, f32 = s8_stream(N, seed=42)
    args = ["--block", "16384", "--tail", "iq"] + D10
    assert sinks_of(bankd, tmp_path, "a", args + ["--f32", "--s8"], s8) == sinks_of(bankd, tmp_path, "b", args + ["--s8"], s8)
    assert sinks_of(bankd, tmp_path, "c", args + ["--s8", "--f32"], f32) == sinks_of(bankd, tmp_path, "d", args + ["--f32"], f32)
    assert sinks_of(bankd, tmp_path, "e", args + ["--s8", "--u8"], s8) == sinks_of(bankd, tmp_path, "f", args + ["--u8"], s8)


def test_hackrf_10msps_three_nfm_stations(bankd, tmp_path):
    """three NFM stations in a 10 Msps s8 stream, --decimation 200 --resample 24:25 (48 kHz audio): each channel's audio is its own
    station's tone"""
    import subprocess
    fs, n = 10e6, 8_000_000
    rates, tones = (-0.1, 0.05, 0.2), (700.0, 1100.0, 1700.0)
    t = np.arange(n)
    z = sum(0.3 * np.exp(1j * (2 * np.pi * (-r) * t + (2500.0 / f) * np.sin(2 * np.pi * f / fs * t))) for r, f in zip(rates, tones))
    z = z + 0.01 * np.array([1, 1j]) @ np.random.default_rng(43).normal(size=(2, n))
    iq = np.empty(2 * n); iq[0::2] = z.real; iq[1::2] = z.imag
    s8 = np.clip(np.round(iq * 127), -127, 127).astype(np.int8)
    sinks = [tmp_path / f"st{k}.s16" for k in range(3)]
    r = subprocess.run([bankd, "--s8", "--decimation", "200", "--resample", "24:25"] + [f"{q}:{p}" for q, p in zip(rates, sinks)],
                       input=s8.tobytes(), stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    for k, p in enumerate(sinks):
        a = np.frombuffer(p.read_bytes(), np.int16).astype(np.float64)[4800:]
        assert a.size > 20000, a.size
        spec = np.abs(np.fft.rfft(a * np.hanning(a.size)))
        freqs = np.fft.rfftfreq(a.size, 1 / 48000.0)
        band = (freqs > 200) & (freqs < 4000)
        peak = freqs[band][np.argmax(spec[band])]
        assert abs(peak - tones[k]) < 10, (k, peak)
        others = [spec[np.argmin(np.abs(freqs - f))] for j, f in enumerate(tones) if j != k]
        assert max(others) < 0.1 * spec[np.argmin(np.abs(freqs - tones[k]))], k
