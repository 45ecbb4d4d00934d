"""GPU tests (-m gpu) of csdr-bankd at a decimation other than 10 and 50: --decimation 40 --bw 0.00625 (639 taps, the generic bank kernel's
M = 17 bucket).  Per channel the raw discriminator (--tail none) and the complex baseband (--tail iq) must equal the oracle's
shift_addition_cc | fir_decimate_cc 40 [| fmdemod_quadri_cf] over the whole stream at two block sizes, and --devices must give the single-device bytes.
tests/test_bankd_generic_emulated.py runs the same bodies on the emulated library."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent))
import test_gpu_zzz_bankd as g  # noqa: E402

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
D, BW = 40, 0.00625
N = 3 * 65536                                                         # wideband samples fed to the daemon


def MULTI_DEVICES():
    return g.MULTI_DEVICES()


@pytest.fixture(scope="module")
def bankd():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from csdr_b200.build import build
    build()
    assert g.BANKD.exists()
    return str(g.BANKD)


def stream_used(T, n, block):
    """samples of an n-sample stream the daemon processes (constant presented size: every call after the first takes what the previous one consumed)"""
    consumed = ((block - T) // D + 1) * D
    return block + ((n - block) // consumed) * consumed if n >= block else 0


def oracle_channel(oracle, wide, rate, taps, tail):
    sh, _ = oracle.shift_addition_cc(wide, float(np.float32(rate)), 0.0, 1024)
    bb = oracle.fir_decimate_cc(sh, D, taps)
    return bb if tail == "iq" else oracle.fmdemod_quadri_cf(bb)[0]


@pytest.mark.parametrize("tail", ["none", "iq"])
@pytest.mark.parametrize("block", [65536, 50_000])
def test_decimation_40_equals_the_reference_chain(bankd, oracle, tmp_path, tail, block):
    from oracle.pyoracle import rel_rms
    T = oracle.firdes_filter_len(BW)
    assert T == 639
    wide = oracle.convert_u8_f(g.wideband_u8(N, seed=40)).view(np.complex64)
    sinks = [tmp_path / f"ch{k}.cf" for k in range(len(g.RATES))]
    err = g.run(bankd, ["--tail", tail, "--f32", "--decimation", str(D), "--bw", str(BW), "--block", str(block)], wide.tobytes(), sinks)
    assert "decimation 40, 639 taps" in err
    taps = oracle.firdes_lowpass_f(T, 0.5 / D)
    used = stream_used(T, N, block)
    for rate, path in zip(g.RATES, sinks):
        got = np.fromfile(path, np.complex64 if tail == "iq" else np.float32)
        want = oracle_channel(oracle, wide[:used], rate, taps, tail)
        assert got.size == want.size and got.size >= 3000, (rate, got.size, want.size)
        assert rel_rms(got, want) < (2e-6 if tail == "iq" else 1e-5), (rate, rel_rms(got, want))
    if block == 50_000:                                               # the channels sliced over devices: the same bytes
        for devices in MULTI_DEVICES():
            msinks = [tmp_path / f"m{devices.replace(',', '_')}_{k}.cf" for k in range(len(g.RATES))]
            g.run(bankd, ["--tail", tail, "--f32", "--decimation", str(D), "--bw", str(BW), "--block", str(block), "--devices", devices],
                  wide.tobytes(), msinks)
            for a, b in zip(sinks, msinks):
                assert a.read_bytes() == b.read_bytes(), devices


def test_odd_decimation_is_refused(bankd, tmp_path):
    import subprocess
    r = subprocess.run([bankd, "--decimation", "7", f"0.1:{tmp_path / 'x'}"], input=b"", capture_output=True, timeout=60)
    assert r.returncode != 0 and b"even" in r.stderr
