"""GPU tests (-m gpu) of csdr-bankd --resample I:D[:BW]: rational_resampler_ff right behind the discriminator, so that wideband rates that give no
48 kHz at any even decimation (rtl_sdr's 2.048 Msps: /32 = 64 kHz, then 3/4) feed the NFM tail at the rate its de-emphasis is designed for.
Per channel the stream must equal the oracle's graph run over the whole stream, with the resampler as ONE call over the whole discriminator
stream.  The bodies also run on the emulated library (tests/test_bankd_resample_emulated.py)."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "resampler"))
sys.path.insert(0, str(ROOT / "tests"))
import resampler as R  # noqa: E402
import test_gpu_zzz_bankd as g  # noqa: E402  (stream generator, runner, device lists)

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
bankd = g.bankd
D, BW, BLOCK = 32, 0.01, 131072                     # 2.048 Msps / 32 = 64 kHz; 0.01 keeps the filter inside the fused bank (401 taps, M = 13)


def used_samples(oracle, n, block):
    T = oracle.firdes_filter_len(BW)
    consumed = ((block - T) // D + 1) * D
    return block + ((n - block) // consumed) * consumed if n >= block else 0


def oracle_channel(oracle, wide, rate, I, Dr, tail, rs_bw=0.05):
    taps = oracle.firdes_lowpass_f(oracle.firdes_filter_len(BW), 0.5 / D)
    sh, _ = oracle.shift_addition_cc(wide, float(np.float32(rate)), 0.0, 1024)
    d = oracle.fmdemod_quadri_cf(oracle.fir_decimate_cc(sh, D, taps))[0]
    r, _ = R.Oracle().rational_resampler_ff(d, I, Dr, R.lowpass(oracle, oracle.firdes_filter_len(rs_bw), I, Dr))
    if tail == "none":
        return r
    return oracle.convert_f_s16(oracle.fastagc_ff(oracle.deemphasis_nfm_ff(oracle.limit_ff(r, 1.0), g.GOLD["nfm_taps_48000"]), 1024, 1.0))


def test_nfm_resampled_to_48k_equals_the_oracle_graph(bankd, oracle, tmp_path):
    n = 5 * BLOCK
    u8 = g.wideband_u8(n, seed=21)
    used = used_samples(oracle, n, BLOCK)
    args = ["--decimation", str(D), "--bw", str(BW), "--resample", "3:4", "--block", str(BLOCK)]
    sinks = [tmp_path / f"ch{k}.s16" for k in range(len(g.RATES))]
    g.run(bankd, args, u8.tobytes(), sinks)
    wide = oracle.convert_u8_f(u8[:2 * used]).view(np.complex64)
    for rate, path in zip(g.RATES, sinks):
        got = np.fromfile(path, np.int16)
        want = oracle_channel(oracle, wide, rate, 3, 4, "nfm")
        assert got.size == want.size and got.size >= 8 * 1024, (rate, got.size, want.size)
        assert np.abs(got.astype(np.int32) - want.astype(np.int32)).max() <= 1, rate
    # --devices: the discriminator rows come back from their devices and are resampled and de-emphasised on the first one, through the same kernels
    devices = g.MULTI_DEVICES()[-1]
    msinks = [tmp_path / f"m{k}.s16" for k in range(len(g.RATES))]
    g.run(bankd, args + ["--devices", devices], u8.tobytes(), msinks)
    for a, b in zip(sinks, msinks):
        assert a.read_bytes() == b.read_bytes(), devices


def test_raw_resampled_discriminator_output(bankd, oracle, tmp_path):
    """--tail none --resample 24:25:0.02 (the 10 Msps / 200 case scaled down): float output within 1e-5 of the oracle, --devices byte-identical"""
    n = 3 * BLOCK
    u8 = g.wideband_u8(n, seed=23)
    used = used_samples(oracle, n, BLOCK)
    args = ["--tail", "none", "--decimation", str(D), "--bw", str(BW), "--resample", "24:25:0.02", "--block", str(BLOCK)]
    sinks = [tmp_path / f"ch{k}.f32" for k in range(len(g.RATES))]
    g.run(bankd, args, u8.tobytes(), sinks)
    wide = oracle.convert_u8_f(u8[:2 * used]).view(np.complex64)
    from oracle.pyoracle import rel_rms
    for rate, path in zip(g.RATES, sinks):
        got = np.fromfile(path, np.float32)
        want = oracle_channel(oracle, wide, rate, 24, 25, "none", 0.02)
        assert got.size == want.size and got.size > 0 and rel_rms(got, want) < 1e-5, (rate, got.size, want.size)
    devices = g.MULTI_DEVICES()[-1]
    msinks = [tmp_path / f"m{k}.f32" for k in range(len(g.RATES))]
    g.run(bankd, args + ["--devices", devices], u8.tobytes(), msinks)
    for a, b in zip(sinks, msinks):
        assert a.read_bytes() == b.read_bytes(), devices


def test_refused_resample_geometries(bankd, tmp_path):
    """a geometry whose resampler calls could end on the output cap (1:100 with 79 taps) and the AM / SSB tails are refused with a message"""
    sink = str(tmp_path / "x")
    for args, words in ((["--resample", "1:100"], b"output cap"), (["--tail", "am", "--resample", "3:4"], b"--tail nfm"),
                        (["--resample", "3"], b"I:D")):
        r = subprocess.run([bankd] + args + [f"0.1:{sink}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=120)
        assert r.returncode != 0 and words in r.stderr, (args, r.stderr[-500:])
    r = subprocess.run([bankd, "--help"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
    assert b"(T/I + 1)*I >= 2*D + I - 1" in r.stderr
