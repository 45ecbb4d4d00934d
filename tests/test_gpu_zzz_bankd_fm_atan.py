"""GPU tests (-m gpu) of csdr-bankd --fm-demod atan (csdr_b200/host/bankd.c): the bank gives the complex baseband and fmdemod_atan_cf runs on it.
Per channel --tail none must be the reference's fmdemod_atan_cf over the daemon's own --tail iq output of the same run (under the atan rounding
rule of tests/demod/demod.py); nfm (also behind --resample), wfm and rtty must be their checkers on that discriminator output; --devices gives
the single-device bytes; the combinations the daemon refuses exit with a message.  On the GPU only: loud broadcast FM (75 kHz deviation, 1 kHz
tone, 2.4 Msps, --decimation 10 --bw 0.05) comes out with its harmonics at least 60 dB down with atan and at most 20 dB down without it, and the
wfm tail's s16 is WfmAudioBank's on the atan discriminator, byte for byte.  tests/test_bankd_fm_atan_emulated.py runs the other bodies on the
emulated library."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

from test_gpu_zzz_bankd import bankd  # noqa: F401  (the fixture)
import test_gpu_zzz_bankd as base
import test_gpu_zzz_bankd_rtty as brtty

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "wfm"))
sys.path.insert(0, str(ROOT / "tests" / "demod"))
sys.path.insert(0, str(ROOT / "tests" / "resampler"))
sys.path.insert(0, str(ROOT / "tests" / "rtty"))
import demod as M  # noqa: E402
import resampler as R  # noqa: E402
import rtty  # noqa: E402
import wfm as W  # noqa: E402

RATES = (-0.3, 0.0, 0.3)
FS, D, BW = 2.4e6, 10, 0.05


def wideband(n, seed, fmt, deviation=15e3, tone=(1000.0, 2500.0, 4000.0), noise=0.003):
    """three FM stations at -RATES of a 2.4 Msps stream, station k modulated by tone[k] with `deviation` Hz peak"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    z = sum(0.25 * np.exp(1j * (2 * np.pi * (-r) * t + deviation / f * np.sin(2 * np.pi * f / FS * t) + rng.uniform(0, 2 * np.pi)))
            for r, f in zip(RATES, tone))
    z = z + noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    if fmt == "f32":
        return z.astype(np.complex64).tobytes()
    iq = np.empty(2 * n); iq[0::2] = z.real; iq[1::2] = z.imag
    return np.clip(np.floor(iq * 127.5 + 128), 0, 255).astype(np.uint8).tobytes()


def run(bankd, args, data, sinks, rates=RATES, timeout=900):
    cmd = [bankd] + args + [f"{r}:{p}" for r, p in zip(rates, sinks)]
    r = subprocess.run(cmd, input=data, stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=timeout)
    assert r.returncode == 0, r.stderr[-2000:]


def outputs(bankd, tmp_path, args, data, tag, dtype, rates=RATES):
    sinks = [tmp_path / f"{tag}{k}" for k in range(len(rates))]
    run(bankd, args, data, sinks, rates)
    return [np.fromfile(p, dtype) for p in sinks]


def reference_atan(iq):
    return M.ref_atan(iq)[0] if M.have_ref() else M.fmdemod_atan_cf(iq)[0]


@pytest.mark.parametrize("fmt,block", [("u8", 16384), ("f32", 40000)])
def test_none_is_fmdemod_atan_over_the_iq_tail(bankd, tmp_path, fmt, block):
    data = wideband(4 * block + 12345, 3, fmt)
    args = [f"--{fmt}", "--decimation", str(D), "--bw", str(BW), "--block", str(block)]
    iq = outputs(bankd, tmp_path, args + ["--tail", "iq"], data, "iq", np.complex64)
    disc = outputs(bankd, tmp_path, args + ["--tail", "none", "--fm-demod", "atan"], data, "at", np.float32)
    near = 0
    for x, d in zip(iq, disc):
        assert d.size == x.size and d.size > 4000
        near += M.atan_matches(d, reference_atan(x), x)[0]
    assert near < 10, near


def test_tails_equal_their_checkers_on_the_atan_discriminator(bankd, oracle, tmp_path):
    """nfm (limit_ff | deemphasis_nfm_ff | fastagc_ff | convert_f_s16, also behind --resample 1:5) and wfm (fractional_decimator_ff 5 |
    deemphasis_wfm_ff | convert_f_s16 in 1024-sample calls) on the daemon's own --tail none --fm-demod atan output"""
    block = 16384
    data = wideband(6 * block, 4, "u8")
    args = ["--u8", "--decimation", str(D), "--bw", str(BW), "--block", str(block), "--fm-demod", "atan"]
    disc = outputs(bankd, tmp_path, args + ["--tail", "none"], data, "d", np.float32)
    nfm = outputs(bankd, tmp_path, args + ["--tail", "nfm"], data, "n", np.int16)
    wfm = outputs(bankd, tmp_path, args + ["--tail", "wfm"], data, "w", np.int16)
    rs_none = outputs(bankd, tmp_path, args + ["--tail", "none", "--resample", "1:5"], data, "rn", np.float32)
    rs_nfm = outputs(bankd, tmp_path, args + ["--tail", "nfm", "--resample", "1:5"], data, "rs", np.int16)
    taps48 = base.GOLD["nfm_taps_48000"]
    nfm_chain = lambda d: oracle.convert_f_s16(oracle.fastagc_ff(oracle.deemphasis_nfm_ff(oracle.limit_ff(d, 1.0), taps48), 1024, 1.0))  # noqa: E731
    for d, n, w, rn, rs in zip(disc, nfm, wfm, rs_none, rs_nfm):
        want = nfm_chain(d)
        assert n.size == want.size and n.size >= 4 * 1024
        assert np.abs(n.astype(np.int32) - want.astype(np.int32)).max() <= 1
        ww = W.checker(oracle, d, 5.0, 1024, 50e-6)
        assert w.size == ww.size and w.size > 1000 and np.array_equal(w, ww)
        r, _ = R.Oracle().rational_resampler_ff(d, 1, 5, R.lowpass(oracle, oracle.firdes_filter_len(0.05), 1, 5))
        assert rn.size == r.size and np.abs(rn - r).max() <= 1e-6
        want = nfm_chain(r)
        assert rs.size == want.size and rs.size >= 1024
        assert np.abs(rs.astype(np.int32) - want.astype(np.int32)).max() <= 1


def test_rtty_tail_on_the_atan_discriminator(bankd, tmp_path):
    block, bufsize = 16384, 256
    data = brtty.wideband(brtty.SPB * brtty.D, 3, "u8", tail_wide=(bufsize + 8) * brtty.D + block)
    args = ["--u8", "--decimation", str(brtty.D), "--bw", str(brtty.BW), "--block", str(block), "--fm-demod", "atan"]
    disc = outputs(bankd, tmp_path, args + ["--tail", "none"], data, "rd", np.float32, brtty.RATES)
    sinks = [tmp_path / f"rt{k}.txt" for k in range(len(brtty.RATES))]
    run(bankd, args + ["--tail", "rtty", "--sps", str(brtty.SPB), "--rtty-bufsize", str(bufsize)], data, sinks, brtty.RATES)
    for d, p in zip(disc, sinks):
        want = rtty.baudot_decode(rtty.serial_stream(d, brtty.SPB, 5, 1.5, 0.4, bufsize)[0])[0]
        got = p.read_bytes()
        assert got == want and brtty.TEXT in got, (got, want)


def test_atan_over_several_devices(bankd, tmp_path):
    """--devices: the slices return baseband rows, the atan stage and the tail run on the first device -- the single-device bytes, also for
    --tail none, which atan keeps off the host-fed shortcut"""
    data = wideband(5 * 16384, 5, "u8")
    for tail in ("none", "wfm", "nfm"):
        args = ["--u8", "--decimation", str(D), "--bw", str(BW), "--block", "16384", "--tail", tail, "--fm-demod", "atan"]
        one = [tmp_path / f"one{tail}{k}" for k in range(len(RATES))]
        run(bankd, args, data, one)
        assert all(p.stat().st_size > 2000 for p in one)
        for devices in base.MULTI_DEVICES():
            many = [tmp_path / f"m{tail}{devices.replace(',', '_')}{k}" for k in range(len(RATES))]
            run(bankd, args + ["--devices", devices], data, many)
            for a, b in zip(one, many):
                assert a.read_bytes() == b.read_bytes(), (tail, devices)


def test_fm_demod_refusals(bankd, tmp_path):
    for args in (["--tail", "iq", "--fm-demod", "atan"], ["--tail", "am", "--fm-demod", "atan"], ["--tail", "usb", "--fm-demod", "atan"],
                 ["--tail", "lsb", "--fm-demod", "atan"], ["--tail", "bpsk31", "--sps", "16", "--fm-demod", "atan"],
                 ["--tail", "rtty", "--sps", "20", "--bfsk", "0.085:44", "--fm-demod", "atan"], ["--fm-demod", "atn"], ["--fm-demod", ""]):
        r = subprocess.run([bankd] + args + [f"0.1:{tmp_path / 'x.out'}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode != 0 and b"csdr-bankd:" in r.stderr, args
    for args in (["--fm-demod", "quadri"], ["--tail", "iq", "--fm-demod", "quadri"], ["--tail", "wfm", "--fm-demod", "atan"],
                 ["--tail", "rtty", "--sps", "20", "--fm-demod", "atan"]):
        r = subprocess.run([bankd] + args + [f"0.1:{tmp_path / 'y.out'}"], input=b"", stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=60)
        assert r.returncode == 0, (args, r.stderr)


# ---- GPU only ------------------------------------------------------------------------------------------------------------------------------
def harmonics_db(d, fs_out=FS / D, tone=1000.0, skip=4800, cycles=400):
    """the strongest of the 2nd, 3rd and 5th harmonics relative to the tone, over a whole number of tone periods"""
    per = int(round(fs_out / tone))
    seg = d[skip:skip + cycles * per].astype(np.float64)
    assert seg.size == cycles * per
    spec = np.abs(np.fft.rfft(seg - seg.mean()))
    return 20 * np.log10(max(spec[h * cycles] for h in (2, 3, 5)) / spec[cycles])


def test_loud_broadcast_fm_is_not_distorted(bankd, tmp_path):
    """75 kHz deviation at 2.4 Msps, --decimation 10 --bw 0.05 (the README's WFM example): atan keeps the 2nd, 3rd and 5th harmonics 60 dB
    below a 1 kHz tone (a float64 simulation gives -86 dB); the quadri-correlator's sin() leaves them within 20 dB (simulation: -13.5 dB)"""
    data = wideband(int(FS * 0.5), 6, "f32", deviation=75e3, tone=(1000.0, 1000.0, 1000.0), noise=0.0)
    args = ["--f32", "--decimation", str(D), "--bw", str(BW), "--tail", "none"]
    atan = outputs(bankd, tmp_path, args + ["--fm-demod", "atan"], data, "a", np.float32)
    quadri = outputs(bankd, tmp_path, args, data, "q", np.float32)
    for a, q in zip(atan, quadri):
        ha, hq = harmonics_db(a), harmonics_db(q)
        print(f"harmonics: atan {ha:.1f} dB, quadri {hq:.1f} dB")
        assert ha <= -60, ha
        assert hq >= -20, hq


def test_wfm_tail_is_wfm_audio_bank_on_the_atan_discriminator(bankd, tmp_path):
    import torch
    import csdr_b200
    data = wideband(6 * 16384, 7, "u8", deviation=75e3)
    args = ["--u8", "--decimation", str(D), "--bw", str(BW), "--block", "16384", "--fm-demod", "atan"]
    disc = outputs(bankd, tmp_path, args + ["--tail", "none"], data, "d", np.float32)
    wfm = outputs(bankd, tmp_path, args + ["--tail", "wfm"], data, "w", np.int16)
    bank = csdr_b200.WfmAudioBank(len(RATES))
    want = bank.process(torch.from_numpy(np.stack(disc)).cuda()).cpu().numpy()
    for k, w in enumerate(wfm):
        assert w.size == want.shape[1] and w.size > 1000 and np.array_equal(w, want[k]), k
