"""GPU tests (-m gpu) of the real-input FFT and waterfall bank: the bodies of tests/test_spectrum_real_emulated.py on the H100 through the real
library (torch CUDA tensors as device buffers) at full size -- every four-step size up to 2^21 real points, 64 rows for the bank's size sweep --
plus 1024 rows at 2048 real points and the 16384-bin bank with many frames, against the composition of the existing per-block calls, bit for bit."""
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
sys.path.insert(0, str(Path(__file__).resolve().parent / "spectrum"))
import spectrum as S  # noqa: E402
import spectrum_real as R  # noqa: E402
import test_spectrum_real_emulated as E  # noqa: E402


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from csdr_b200.build import build
    build()
    d = S.CudaDev()
    R.setup(d.L)
    return d


@pytest.fixture(scope="module")
def full_size():
    return True


test_r2c_within_the_bound = E.test_r2c_within_the_bound
test_r2c_four_step_size = E.test_r2c_four_step_size
test_r2c_impulse_and_cosine = E.test_r2c_impulse_and_cosine
test_dropin_plan_equals_the_batch_call = E.test_dropin_plan_equals_the_batch_call
test_window_f_is_the_float_product = E.test_window_f_is_the_float_product
test_r2c_refusals = E.test_r2c_refusals
test_bank_equals_the_composition = E.test_bank_equals_the_composition
test_any_cut_and_any_scratch_give_one_call = E.test_any_cut_and_any_scratch_give_one_call
test_rows_are_independent = E.test_rows_are_independent
test_nonfinite_input_stays_in_its_lines = E.test_nonfinite_input_stays_in_its_lines
test_line_count_is_fft_fcs = E.test_line_count_is_fft_fcs
test_the_gapped_framing_is_the_references = E.test_the_gapped_framing_is_the_references
test_refusals = E.test_refusals


@pytest.mark.parametrize("compress", [0, 1])
def test_1024_rows_at_2048_points(dev, compress):
    """1024 rows of real samples, N = 1024 bins (2048 real points), E = 2N, A = 2, cut into three calls with minimum scratch"""
    rng = np.random.default_rng(40 + compress)
    rows, N, A = 1024, 1024, 2
    p = S.Params(N, 2 * N, A, compress, -70.0)
    x = (rng.standard_normal((rows, 8 * N + 100)) * 0.2).astype(np.float32)
    w = S.window(dev.L, 2 * N)
    want = R.composition(dev, x, p, w)
    assert np.array_equal(R.bank(dev, x, p, w), want)
    assert np.array_equal(R.bank(dev, x, p, w, cuts=[1000, 5000], scratch="min", pad=3), want)


def test_16384_bins_with_many_frames(dev):
    """the largest bank size, overlapped frames (E = N), 12 lines of A = 3"""
    rng = np.random.default_rng(9)
    N, E_, A = 16384, 16384, 3
    p = S.Params(N, E_, A, 1, -70.0)
    x = (rng.standard_normal((1, R.stream_for(N, E_, 36) + 99)) * 0.3).astype(np.float32)
    w = S.window(dev.L, 2 * N, "BLACKMAN")
    want = R.composition(dev, x, p, w)
    assert want.shape[1] == 12
    assert np.array_equal(R.bank(dev, x, p, w, cuts=[50000, 50001, 200000]), want)


def test_python_api(dev):
    import csdr_b200
    rng = np.random.default_rng(77)
    rows, N, E_, A = 8, 1024, 3000, 3
    x = (rng.standard_normal((rows, 40000)) * 0.3).astype(np.float32)
    p = S.Params(N, E_, A, 1, -40.0)
    want = R.bank(dev, x, p, S.window(dev.L, 2 * N))
    b = csdr_b200.SpectrumBank(rows, N, E_, A, -40.0, compress=True, real=True)
    parts = [b.process(torch.from_numpy(x[:, a:c].copy()).cuda()) for a, c in ((0, 7000), (7000, 7001), (7001, 40000))]
    assert np.array_equal(torch.cat(parts, dim=1).cpu().numpy(), want)
    y = torch.from_numpy(x[:2, :4096].copy()).cuda()
    assert np.array_equal(csdr_b200.fft_r2c(y).cpu().numpy(), R.r2c(dev, x[:2, :4096]))
    assert csdr_b200.fft_r2c(y[0]).shape == (2049,)
