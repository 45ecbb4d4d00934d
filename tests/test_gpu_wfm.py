"""GPU tests (-m gpu) of the WFM audio bank csdrb_wfm_audio_bank_f_s16: the bodies of tests/test_wfm_emulated.py on the H100 through the real
library (torch CUDA tensors as device buffers) at full size, plus 1024 channels, the Python class csdr_b200.WfmAudioBank, and the compiled
reference CLI pipe `fractional_decimator_ff R | deemphasis_wfm_ff 48000 T | convert_f_s16` on the same discriminator stream."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "wfm"))
import wfm as W  # noqa: E402
import test_wfm_emulated as E  # noqa: E402

REF_CLI = ROOT / "oracle" / "_ref" / "csdr_ref"


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from csdr_b200.build import build
    build()
    return W.cuda_dev()


@pytest.fixture(scope="module")
def full_size():
    return True


test_bank_equals_the_checker = E.test_bank_equals_the_checker
test_any_cut_gives_one_call = E.test_any_cut_gives_one_call
test_rows_are_independent = E.test_rows_are_independent
test_nan_stays_in_its_row_and_restarts_where_the_reference_does = E.test_nan_stays_in_its_row_and_restarts_where_the_reference_does
test_infinite_carry_is_kept_and_a_nan_carry_restarts = E.test_infinite_carry_is_kept_and_a_nan_carry_restarts
test_outputs_agrees_with_the_bank = E.test_outputs_agrees_with_the_bank
test_refusals = E.test_refusals


def test_1024_channels(dev, oracle):
    """1024 channels x 1 s at 240 kHz, rate 5, cut into three calls: the checker's bytes on every row"""
    rng = np.random.default_rng(11)
    x = W.signal(rng, 1024, 240000)
    p = W.Params(5.0, 1024, 50e-6, 48000)
    got, _, _ = W.bank(dev, x, p, cuts=[70001, 150000], pad=2)
    assert got.shape[1] > 47000
    for c in range(1024):
        assert np.array_equal(got[c], W.checker(oracle, x[c], 5.0, 1024, 50e-6)), c


def test_python_class_equals_the_bank(dev):
    import csdr_b200
    rng = np.random.default_rng(12)
    x = W.signal(rng, 6, 30000)
    want, _, _ = W.bank(dev, x, W.Params(5.2083333, 1024, 75e-6, 48000))
    b = csdr_b200.WfmAudioBank(6, rate=5.2083333, tau=75e-6)
    parts = [b.process(torch.from_numpy(x[:, a:c].copy()).cuda()) for a, c in ((0, 500), (500, 500), (500, 12345), (12345, 30000))]
    got = torch.cat(parts, dim=1).cpu().numpy()
    assert np.array_equal(got, want)
    for rate in (1.0, float("inf"), float("nan")):
        with pytest.raises(csdr_b200.CsdrB200Error):
            csdr_b200.WfmAudioBank(2, rate=rate)


@pytest.mark.parametrize("rate,tau", [(5.0, 50e-6), (5.2083333, 75e-6)])
def test_reference_cli_pipe(dev, rate, tau):
    """the compiled reference's own pipe on a discriminator-like stream: equal over the common prefix within 1 count.  At rate 5 no sample
    differs; elsewhere the reference's -ffast-math build rounds the Lagrange weights differently by ulps (DESIGN.md §7), which moves a few
    samples by 1 count.  The count of differing samples is printed."""
    if not REF_CLI.exists():
        pytest.skip("oracle/_ref/csdr_ref not built")
    rng = np.random.default_rng(13)
    x = W.signal(rng, 1, 200000)
    got, _, _ = W.bank(dev, x, W.Params(rate, 1024, tau, 48000))
    cmd = f"{REF_CLI} fractional_decimator_ff {rate} | {REF_CLI} deemphasis_wfm_ff 48000 {tau} | {REF_CLI} convert_f_s16"
    r = subprocess.run(["bash", "-c", cmd], input=x[0].tobytes(), stdout=subprocess.PIPE, stderr=subprocess.PIPE, timeout=300,
                       env={"PATH": "/usr/bin:/bin"})
    assert r.returncode == 0, r.stderr[-2000:]
    want = np.frombuffer(r.stdout, np.int16)
    n = min(got.shape[1], want.size)
    assert n > 0.95 * got.shape[1]
    diff = np.abs(got[0, :n].astype(np.int32) - want[:n].astype(np.int32))
    print(f"wfm bank vs reference CLI pipe, rate {rate}: {np.count_nonzero(diff)} of {n} samples differ, largest by {diff.max()}")
    assert diff.max() <= 1
