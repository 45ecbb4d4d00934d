"""GPU tests (-m gpu) of the four-step FFT above 16384 points and the layers on top of it: the bodies of tests/test_fft_large_emulated.py on the
H100 through the real library, at every size 2^15 .. 2^20, batches 1, 3 and one beyond a scratch chunk, and the three CLI pipes also against the
compiled reference CLI where oracle/_ref holds it."""
import sys
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "spectrum"))
import spectrum as S  # noqa: E402
import test_fft_large_emulated as E  # noqa: E402

REF = ROOT / "oracle" / "_ref" / "csdr_ref"
oracle = E.oracle
ALL = sorted(E.FACTORS)


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from csdr_b200.build import build
    build()
    return E.setup(S.CudaDev())


@pytest.fixture(scope="module")
def cli(dev):
    return str(ROOT / "csdr_b200" / "csdr")


@pytest.fixture(scope="module")
def ref():
    return str(REF) if REF.exists() else None


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("lg", ALL)
def test_forward_and_inverse_against_numpy(dev, lg, batch):
    E.check_against_numpy(dev, lg, batch)


@pytest.mark.parametrize("lg", ALL)
def test_sparse_input_within_the_per_output_bound(dev, lg):
    E.check_sparse_input_bound(dev, lg)


@pytest.mark.parametrize("lg", ALL)
def test_impulses_and_tones(dev, lg):
    E.check_impulses_and_tones(dev, lg, *E.FACTORS[lg])


@pytest.mark.parametrize("lg", ALL)
def test_round_trip_batch_rows_strides_and_nonfinite_rows(dev, lg):
    E.check_round_trip_batch_and_strides(dev, lg)


@pytest.mark.parametrize("lg", ALL)
def test_a_batch_beyond_one_scratch_chunk(dev, lg):
    E.check_second_chunk(dev, lg)


def test_refusals(dev):
    E.check_refusals(dev)


@pytest.mark.parametrize("lg", ALL)
def test_plans_above_16384(dev, lg):
    E.check_plan(dev, lg)


@pytest.mark.parametrize("bw,dec,nblocks", [(0.0005, 256, 5), (0.00025, 256, 4), (0.0005, 512, 3)])
def test_fastddc_with_a_long_filter(dev, oracle, bw, dec, nblocks):
    E.check_fastddc(dev, oracle, bw, dec, nblocks)


def test_fastddc_forward_calls_shorter_than_the_overlap(dev):
    E.check_fastddc_fwd_short_calls(dev)


@pytest.mark.parametrize("lg", [15, 16, 20])
def test_apply_fir_fft_above_16384(dev, lg):
    E.check_apply_fir_fft(dev, lg)


def test_cli_waterfall_at_32768_bins(dev, cli, ref):
    E.check_cli_waterfall(dev, cli, ref)


def test_cli_long_filters(cli, oracle, ref):
    E.check_cli_filters(cli, oracle, ref)


def test_python_fft_c2c_takes_the_large_sizes(dev):
    import numpy as np
    import csdr_b200
    x = E.noise(np.random.default_rng(1), 2, 1 << 16)
    y = csdr_b200.fft_c2c(torch.from_numpy(x).cuda()).cpu().numpy()
    assert E.rel_rms(y, np.fft.fft(x.astype(np.complex128), axis=1)) < 1e-6
