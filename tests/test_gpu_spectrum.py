"""GPU tests (-m gpu) of the waterfall bank csdrb_spectrum_bank_cf: the bodies of tests/test_spectrum_emulated.py on the H100 through the real
library (torch CUDA tensors as device buffers) at full size -- every FFT size up to 16384 points with its frames, 64 rows for the size sweep --
plus one wideband-server geometry of 1024 rows, against the composition of the existing per-block calls, bit for bit."""
import sys
from pathlib import Path

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
sys.path.insert(0, str(Path(__file__).resolve().parent / "spectrum"))
import spectrum as S  # noqa: E402
import test_spectrum_emulated as E  # noqa: E402


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from csdr_b200.build import build
    build()
    return S.CudaDev()


@pytest.fixture(scope="module")
def full_size():
    return True


test_bank_equals_the_composition = E.test_bank_equals_the_composition
test_one_average_is_logpower_cf = E.test_one_average_is_logpower_cf
test_any_cut_and_any_scratch_give_one_call = E.test_any_cut_and_any_scratch_give_one_call
test_rows_are_independent = E.test_rows_are_independent
test_power_within_the_float64_bound = E.test_power_within_the_float64_bound
test_nonfinite_input_stays_in_its_lines = E.test_nonfinite_input_stays_in_its_lines
test_line_count_is_fft_ccs = E.test_line_count_is_fft_ccs
test_refusals = E.test_refusals


@pytest.mark.parametrize("compress", [0, 1])
def test_1024_rows_at_2048_points(dev, compress):
    """1024 rows x 2^13 samples, N = 2048, E = N, A = 2, cut into three calls with minimum scratch: the composition's bytes on every row"""
    rng = np.random.default_rng(40 + compress)
    rows, N, A = 1024, 2048, 2
    p = S.Params(N, N, A, compress, -70.0)
    x = ((rng.standard_normal((rows, 4 * N + 100)) + 1j * rng.standard_normal((rows, 4 * N + 100))) * 0.2).astype(np.complex64)
    w = S.window(dev.L, N)
    want = S.composition(dev, x, p, w)
    assert np.array_equal(S.bank(dev, x, p, w), want)
    assert np.array_equal(S.bank(dev, x, p, w, cuts=[1000, 5000], scratch="min", pad=3), want)


def test_python_class_equals_the_bank(dev):
    import csdr_b200
    rng = np.random.default_rng(77)
    rows, N, E_, A = 8, 1024, 300, 3
    x = ((rng.standard_normal((rows, 20000)) + 1j * rng.standard_normal((rows, 20000))) * 0.3).astype(np.complex64)
    p = S.Params(N, E_, A, 1, -40.0)
    want = S.bank(dev, x, p, S.window(dev.L, N))
    b = csdr_b200.SpectrumBank(rows, N, E_, A, -40.0, compress=True)
    parts = [b.process(torch.from_numpy(x[:, a:c].copy()).cuda()) for a, c in ((0, 7000), (7000, 7001), (7001, 20000))]
    got = torch.cat(parts, dim=1).cpu().numpy()
    assert np.array_equal(got, want)
