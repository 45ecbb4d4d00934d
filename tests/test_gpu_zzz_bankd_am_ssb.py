"""GPU tests (-m gpu) of csdr-bankd's AM and SSB tails (--tail am|usb|lsb, csdr_b200/host/bankd.c): per channel, the s16 audio must be exactly the
oracle's tail (tests/am_ssb) run on the DDC bank's own complex baseband for the same stream -- the baseband the daemon itself writes with
--tail iq.  For usb/lsb the overlap-add bandpass stage is the product's csdrb_bandpass_fir_fft_bank_cc with the same taps (BANDPASS), whose
FFT arithmetic the oracle does not restate bit for bit.  tests/test_bankd_am_ssb_emulated.py runs the same bodies on the emulated library."""
import sys
from pathlib import Path

import numpy as np
import pytest

from test_gpu_zzz_bankd import RATES, bankd, run, wideband_u8  # noqa: F401  (the fixture and the helpers)
import test_gpu_zzz_bankd as base

pytestmark = pytest.mark.gpu
sys.path.insert(0, str(Path(__file__).resolve().parent / "am_ssb"))
import am_ssb  # noqa: E402

SSB_BW = 0.05
SSB_BANDS = {"usb": (0.0, 0.1), "lsb": (-0.1, 0.0)}


def ssb_geometry():
    import csdr_b200
    T = csdr_b200.firdes_filter_len(SSB_BW)
    N = 1 << (T - 1).bit_length()
    if N - T < 200:
        N <<= 1
    return T, N, N - T + 1


def BANDPASS(bb, lo, hi):
    """bandpass_fir_fft_cc lo hi 0.05 over the whole blocks of every row of bb [C, n] complex64, through the product's overlap-add bank"""
    import torch
    import csdr_b200
    T, N, isz = ssb_geometry()
    taps = np.zeros(N, np.complex64); taps[:T] = csdr_b200.firdes_bandpass_c(T, lo, hi)
    tf = csdr_b200.fft_c2c(torch.from_numpy(taps).cuda())
    nb = bb.shape[1] // isz
    y, _ = csdr_b200.bandpass_fir_fft_bank_cc(torch.from_numpy(np.ascontiguousarray(bb[:, :nb * isz])).cuda(), tf, isz)
    return y.cpu().numpy()


def baseband(bankd, tmp_path, args, data):
    sinks = [tmp_path / f"iq{k}.cf32" for k in range(len(RATES))]
    run(bankd, ["--tail", "iq"] + args, data, sinks)
    rows = [np.fromfile(p, np.complex64) for p in sinks]
    assert len({r.size for r in rows}) == 1 and rows[0].size > 4096
    return np.stack(rows)


def expected(tail, bb, oracle, agc_ref=0.2, limit=1.0):
    if tail == "am":
        out = []
        for row in bb:
            env, _ = am_ssb.am_front(row, 1024)
            out.append(am_ssb.agc_tail(env, oracle, 1024, limit, True, reference=agc_ref))
        return out
    filt = base_bandpass()(bb, *SSB_BANDS[tail])
    return [am_ssb.agc_tail(row, oracle, 1024, limit, True, reference=agc_ref) for row in filt]


def base_bandpass():
    return sys.modules[__name__].BANDPASS


@pytest.mark.parametrize("block,fmt", [(131072, "u8"), (100_000, "f32")])
def test_am_ssb_tails_equal_the_oracle_on_the_banks_baseband(bankd, oracle, tmp_path, block, fmt):
    n = 3 * 131072
    u8 = wideband_u8(n, seed=21)
    data = u8.tobytes() if fmt == "u8" else oracle.convert_u8_f(u8).tobytes()
    args = ["--" + fmt, "--block", str(block)]
    bb = baseband(bankd, tmp_path, args, data)
    for tail, extra, ref in (("am", [], 0.2), ("usb", [], 0.2), ("lsb", ["--agc-ref", "0.5", "--limit", "0.8"], 0.5)):
        limit = 0.8 if "--limit" in extra else 1.0
        sinks = [tmp_path / f"{tail}{k}.s16" for k in range(len(RATES))]
        run(bankd, ["--tail", tail] + args + extra, data, sinks)
        want = expected(tail, bb, oracle, ref, limit)
        for k, p in enumerate(sinks):
            got = np.fromfile(p, np.int16)
            assert got.size == want[k].size and got.size >= 4096, (tail, k, got.size, want[k].size)
            assert np.array_equal(got, want[k]), (tail, k, int(np.argmax(got != want[k])))


def test_am_ssb_tails_over_several_devices(bankd, tmp_path):
    """--devices: slices with demod = 0 return baseband, the audio tail runs on the first device -- the single-device bytes"""
    u8 = wideband_u8(4 * 65536, seed=23).tobytes()
    for tail in ("am", "usb"):
        for devices in base.MULTI_DEVICES():
            a = [tmp_path / f"{tail}s{k}.s16" for k in range(len(RATES))]
            b = [tmp_path / f"{tail}m{devices.replace(',', '_')}{k}.s16" for k in range(len(RATES))]
            run(bankd, ["--tail", tail, "--block", "65536"], u8, a)
            run(bankd, ["--tail", tail, "--block", "65536", "--devices", devices], u8, b)
            for x, y in zip(a, b):
                assert x.stat().st_size >= 2 * 1024 and x.read_bytes() == y.read_bytes(), (tail, devices)
