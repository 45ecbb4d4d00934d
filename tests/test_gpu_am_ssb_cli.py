"""GPU tests (-m gpu) of the AM and SSB graphs of the reference README (README.md:95 and :110) on our csdr CLI, stage for stage: every
stage gets the reference CLI's output of the previous stage, and must give the reference CLI's bytes (amdemod_cf: within the ulp bound
measured in tests/test_oracle_am_ssb.py, the reference build's square root being vendor-dependent).  tests/test_am_ssb_cli_emulated.py
runs the same bodies on the emulated library."""
import numpy as np
import pytest

from test_gpu_cli import clis, run_graph  # noqa: F401  (the fixture: our CLI and the reference CLI)

pytestmark = pytest.mark.gpu
AMDEMOD_ULP = 3


def baseband(n, seed):
    """complex baseband of an AM carrier with a little noise, some silence and a burst, as fir_decimate_cc would hand it on"""
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    env = 0.3 * (1 + 0.7 * np.sin(2 * np.pi * t / 97.0)) * (1 + 0.5 * np.sin(2 * np.pi * t / 7000.0))
    env[n // 3: n // 3 + 2000] *= 1e-3
    env[n // 2: n // 2 + 500] *= 20
    x = env * np.exp(1j * (0.01 * t + 0.3)) + 0.002 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return x.astype(np.complex64)


def stage(cli, name, data):
    return run_graph(cli, [name], data)


def test_am_graph_stage_for_stage(clis):
    """README.md:95 after the DDC: amdemod_cf | fastdcblock_ff | agc_ff | limit_ff | convert_f_s16"""
    ours, ref = clis
    x = baseband(1024 * 24, 1).tobytes()
    r1, o1 = stage(ref, "amdemod_cf", x), stage(ours, "amdemod_cf", x)
    a, b = np.frombuffer(r1, np.int32).astype(np.int64), np.frombuffer(o1, np.int32).astype(np.int64)
    assert a.size == b.size and np.abs(a - b).max() <= AMDEMOD_ULP
    prev = r1
    for s in ("fastdcblock_ff", "agc_ff", "limit_ff", "convert_f_s16"):
        want, got = stage(ref, s, prev), stage(ours, s, prev)
        assert got == want, s
        prev = want


def test_ssb_tail_stage_for_stage(clis):
    """README.md:110 after the bandpass filter: realpart_cf | agc_ff | limit_ff | convert_f_s16, plus non-default agc_ff and fastdcblock_ff
    arguments (a block size that is not a multiple of 4 and hang / attack-wait counts)"""
    ours, ref = clis
    x = baseband(1024 * 24, 2).tobytes()
    prev = x
    for s in ("realpart_cf", "agc_ff 30 0.4 0.05 0.001 500 3 0.99", "limit_ff 0.5", "convert_f_s16"):
        want, got = stage(ref, s, prev), stage(ours, s, prev)
        assert got == want, s
        prev = want
    f = stage(ref, "realpart_cf", x)
    assert stage(ours, "fastdcblock_ff 1027", f) == stage(ref, "fastdcblock_ff 1027", f)
