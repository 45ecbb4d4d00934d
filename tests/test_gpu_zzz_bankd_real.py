"""GPU tests (-m gpu) of csdr-bankd on REAL wideband streams (--real-s16, --real-f32) and complex s16 (--s16), csdr_b200/host/bankd.c: per channel
the stream must be the oracle's convert_s16_f | shift_addition_fc r | fir_decimate_cc D bw | <tail> over the whole stream, whatever the block size
(65536 samples at D = 50 leave a tail of 786 samples, so every later block lands 8 bytes off a 16-byte boundary).  Stations sit at +f of a real
stream and are tuned with rate -f/fs.  tests/test_bankd_real_emulated.py runs the same bodies on the emulated library."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parent / "real"))
import real as R  # noqa: E402
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_am_ssb as amg  # noqa: E402
from test_gpu_zzz_bankd import bankd  # noqa: E402,F401  (the fixture)

pytestmark = pytest.mark.gpu
FREQS = (0.045, 0.12, 0.2, 0.31, 0.42)                                # stations, fractions of the sample rate
RATES = tuple(-f for f in FREQS)
D, BW = 50, 0.005


def real_stream(n, seed=3):
    """a real stream: five FM stations at +f (each a cosine, so its mirror sits at -f) and a little noise, as s16"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    x = sum(0.15 * np.cos(2 * np.pi * f * t + np.cumsum(2 * np.pi * 3000.0 / 2.4e6 * np.sin(2 * np.pi * (600.0 + 250 * k) / 2.4e6 * t)))
            for k, f in enumerate(FREQS))
    x = x + 0.002 * rng.normal(size=n)
    return np.clip(np.round(x * 32767), -32768, 32767).astype(np.int16)


def run(bankd, args, data, sinks, expect_ok=True, timeout=300):
    cmd = [bankd] + args + [f"{r}:{p}" for r, p in zip(RATES, sinks)]
    r = subprocess.run(cmd, input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=timeout)
    if expect_ok:
        assert r.returncode == 0, r.stderr[-2000:]
    return r


def used(oracle, n, block):
    """samples of an n-sample stream the daemon processes: blocks of a constant size, each presenting the previous call's unconsumed tail"""
    T = oracle.firdes_filter_len(BW)
    consumed = ((block - T) // D + 1) * D
    return block + ((n - block) // consumed) * consumed if n >= block else 0


def discriminator(oracle, x, rate, taps):
    sh, _ = R.shift_addition_fc(x, float(np.float32(rate)), 0.0, 1024)
    return oracle.fmdemod_quadri_cf(oracle.fir_decimate_cc(sh, D, taps))[0]


def nfm_audio(oracle, x, rate, taps):
    d = discriminator(oracle, x, rate, taps)
    return oracle.convert_f_s16(oracle.fastagc_ff(oracle.deemphasis_nfm_ff(oracle.limit_ff(d, 1.0), base.GOLD["nfm_taps_48000"]), 1024, 1.0))


@pytest.mark.parametrize("block", [131072, 65536])
def test_real_s16_nfm_equals_the_oracle_graph(bankd, oracle, tmp_path, block):
    """--real-s16 --tail nfm, per channel, within one s16 count of convert_s16_f | shift_addition_fc | fir_decimate_cc | fmdemod_quadri_cf | limit_ff |
    deemphasis_nfm_ff 48000 | fastagc_ff | convert_f_s16; 65536-sample blocks leave a tail with keep % 4 == 2, 131072-sample ones keep % 4 == 0"""
    T = oracle.firdes_filter_len(BW)
    assert (block - ((block - T) // D + 1) * D) % 4 == (2 if block == 65536 else 0)
    n = 5 * 131072
    s16 = real_stream(n)
    sinks = [tmp_path / f"ch{k}.s16" for k in range(len(RATES))]
    r = run(bankd, ["--real-s16", "--block", str(block)], s16.tobytes(), sinks)
    assert b"real s16 input" in r.stderr
    u = used(oracle, n, block)
    x = oracle.convert_s16_f(s16[:u])
    taps = oracle.firdes_lowpass_f(T, 0.5 / D)
    for rate, path in zip(RATES, sinks):
        got = np.fromfile(path, np.int16)
        want = nfm_audio(oracle, x, rate, taps)
        assert got.size == want.size and got.size >= 10 * 1024, (rate, got.size, want.size)
        assert np.abs(got.astype(np.int32) - want.astype(np.int32)).max() <= 1, rate
    # the mirror image: +f tunes the station conjugated, so its discriminator output is negated
    if block == 131072:
        pos = [tmp_path / f"p{k}.f32" for k in range(len(RATES))]
        subprocess.run([bankd, "--real-s16", "--tail", "none", "--block", str(block)] + [f"{f}:{p}" for f, p in zip(FREQS, pos)],
                       input=s16.tobytes(), check=True, capture_output=True, timeout=300)
        neg = [tmp_path / f"n{k}.f32" for k in range(len(RATES))]
        run(bankd, ["--real-s16", "--tail", "none", "--block", str(block)], s16.tobytes(), neg)
        for a, b in zip(pos, neg):
            pa, nb = np.fromfile(a, np.float32), np.fromfile(b, np.float32)
            assert pa.size == nb.size and np.corrcoef(pa[100:], nb[100:])[0, 1] < -0.99


def test_real_f32_raw_discriminator(bankd, oracle, tmp_path):
    """--real-f32 --tail none: the raw discriminator output of each channel, rel RMS < 1e-5 against the oracle graph"""
    from oracle.pyoracle import rel_rms
    n, block = 3 * 131072, 131072
    x = oracle.convert_s16_f(real_stream(n, seed=4))
    sinks = [tmp_path / f"ch{k}.f32" for k in range(len(RATES))]
    run(bankd, ["--real-f32", "--tail", "none", "--block", str(block)], x.tobytes(), sinks)
    T = oracle.firdes_filter_len(BW)
    taps = oracle.firdes_lowpass_f(T, 0.5 / D)
    u = used(oracle, n, block)
    for rate, path in zip(RATES, sinks):
        got = np.fromfile(path, np.float32)
        want = discriminator(oracle, x[:u], rate, taps)
        assert got.size == want.size and rel_rms(got, want) < 1e-5, (rate, got.size, want.size)


def test_real_s16_usb(bankd, oracle, tmp_path):
    """--real-s16 --tail usb: the baseband (--tail iq) is the oracle's shift_addition_fc | fir_decimate_cc, and the audio is the SSB tail of
    tests/test_gpu_zzz_bankd_am_ssb.py on that baseband, byte for byte"""
    from oracle.pyoracle import rel_rms
    n, block = 3 * 131072, 65536
    s16 = real_stream(n, seed=5)
    data = s16.tobytes()
    args = ["--real-s16", "--block", str(block)]
    iq = [tmp_path / f"iq{k}.cf32" for k in range(len(RATES))]
    run(bankd, ["--tail", "iq"] + args, data, iq)
    bb = np.stack([np.fromfile(p, np.complex64) for p in iq])
    T = oracle.firdes_filter_len(BW)
    taps = oracle.firdes_lowpass_f(T, 0.5 / D)
    x = oracle.convert_s16_f(s16[:used(oracle, n, block)])
    for k, rate in enumerate(RATES):
        sh, _ = R.shift_addition_fc(x, float(np.float32(rate)), 0.0, 1024)
        want = oracle.fir_decimate_cc(sh, D, taps)
        assert bb[k].size == want.size and rel_rms(bb[k], want) < 1e-5, k
    sinks = [tmp_path / f"usb{k}.s16" for k in range(len(RATES))]
    run(bankd, ["--tail", "usb"] + args, data, sinks)
    want = amg.expected("usb", bb, oracle)
    for k, p in enumerate(sinks):
        got = np.fromfile(p, np.int16)
        assert got.size == want[k].size and got.size >= 4096, (k, got.size, want[k].size)
        assert np.array_equal(got, want[k]), (k, int(np.argmax(got != want[k])))


def test_complex_s16_equals_f32_of_its_conversion(bankd, oracle, tmp_path):
    """--s16 --tail none: the bytes of --f32 on convert_s16_f of the same interleaved stream"""
    rng = np.random.default_rng(6)
    n, block = 3 * 65536, 65536
    iq = np.clip(np.round(base.wideband_u8(n, seed=6).astype(np.float64) * 200 - 25600 + rng.normal(size=2 * n)), -32768, 32767).astype(np.int16)
    a = [tmp_path / f"s{k}.f32" for k in range(len(RATES))]
    b = [tmp_path / f"f{k}.f32" for k in range(len(RATES))]
    run(bankd, ["--s16", "--tail", "none", "--block", str(block)], iq.tobytes(), a)
    run(bankd, ["--f32", "--tail", "none", "--block", str(block)], oracle.convert_s16_f(iq).tobytes(), b)
    for x, y in zip(a, b):
        assert x.stat().st_size > 4 * 1024 and x.read_bytes() == y.read_bytes()


def test_real_input_over_several_devices(bankd, tmp_path):
    """--devices with --real-s16: blocks expanded to x + 0j on the host through the complex multi-GPU bank -- the single-device run's audio"""
    s16 = real_stream(8 * 65536, seed=7).tobytes()
    for devices in base.MULTI_DEVICES():
        a = [tmp_path / f"a{devices.replace(',', '_')}{k}.s16" for k in range(len(RATES))]
        b = [tmp_path / f"b{devices.replace(',', '_')}{k}.s16" for k in range(len(RATES))]
        run(bankd, ["--real-s16", "--block", "65536"], s16, a)
        r = run(bankd, ["--real-s16", "--block", "65536", "--devices", devices], s16, b)
        assert b"real s16 input" in r.stderr
        for x, y in zip(a, b):
            assert x.stat().st_size >= 4 * 2 * 1024 and x.read_bytes() == y.read_bytes(), devices


def test_real_input_refuses_the_waterfall(bankd, tmp_path):
    r = run(bankd, ["--real-s16", "--waterfall", str(tmp_path / "wf.bin")], b"", [tmp_path / f"w{k}.s16" for k in range(len(RATES))], expect_ok=False)
    assert r.returncode != 0 and b"--waterfall needs a complex input" in r.stderr, r.stderr
