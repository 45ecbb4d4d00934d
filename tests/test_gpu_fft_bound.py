"""GPU tests (-m gpu) of the single-CTA FFT family against the per-output bounds and exact invariants of tests/test_fft_bound_emulated.py: the
same check_* bodies on the H100 through the real library, with the full impulse matrix up to 4096 points (2048 columns, every residue mod 16,
at 8192 and 16384), every single-bin sweep, every bin of the fastddc single-bin spectra, and the bank sizes the emulator cannot afford."""
import sys
from pathlib import Path

import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests"))
sys.path.insert(0, str(ROOT / "tests" / "spectrum"))
import spectrum as S  # noqa: E402
import test_fft_bound_emulated as E  # noqa: E402

oracle = E.oracle


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from csdr_b200.build import build
    build()
    return E.setup(S.CudaDev())


@pytest.mark.parametrize("N", E.SIZES)
def test_c2c_impulse_matrix(dev, N):
    E.check_c2c_impulse_matrix(dev, N, full_up_to=4096, subset=2048, chunk=256)


@pytest.mark.parametrize("N", E.SIZES)
def test_c2c_sparse_boundaries_and_tones(dev, N):
    E.check_c2c_sparse_and_tones(dev, N)


@pytest.mark.parametrize("N", E.SIZES)
def test_c2c_rows_alignment_conjugate_symmetry_and_nonfinite_rows(dev, N):
    E.check_c2c_invariants(dev, N, batch=67)


OLA_GPU = E.OLA_CPU + [(1024, 400, 34), (8192, 7000, 33), (8192, 100, 40)]


@pytest.mark.parametrize("N,isz,nb", OLA_GPU)
def test_overlap_add_bank_bound(dev, N, isz, nb):
    assert E.auto_blocks_per_cta(2, nb) == 16
    E.check_ola(dev, N, isz, nb)


@pytest.mark.parametrize("N,isz", [(4, 3), (8, 8), (16, 1), (32, 20), (64, 20), (128, 100), (256, 100), (512, 300), (1024, 1000), (2048, 1500),
                                   (4096, 2098), (8192, 7000)])
def test_overlap_add_single_bin_sweep(dev, N, isz):
    E.check_ola_bin_sweep(dev, N, isz, full_up_to=8192, chunk=512)


@pytest.mark.parametrize("N,isz,nb", [(8, 5, 40), (64, 20, 50), (256, 100, 40), (4096, 2098, 36), (8192, 7000, 34)])
def test_overlap_add_bank_cuts_channels_and_shared_taps(dev, N, isz, nb):
    E.check_ola_invariants(dev, N, isz, nb)


@pytest.mark.parametrize("N,isz,nb", [(8, 3, 40), (64, 20, 40), (4096, 2098, 36), (8192, 7000, 34)])
def test_overlap_add_bank_nonfinite_windows(dev, N, isz, nb):
    E.check_ola_nonfinite(dev, N, isz, nb)


@pytest.mark.parametrize("N", E.SIZES)
def test_apply_fir_fft_bound(dev, N):
    E.check_apply_fir_fft(dev, N)
    E.check_apply_fir_fft_bin_sweep(dev, N, full_up_to=1024, subset=256)


@pytest.mark.parametrize("N,isz,nb", [(8, 3, 40), (16, 12, 30), (64, 20, 40), (4096, 3000, 20), (16384, 9000, 6)])
def test_fastddc_forward_is_the_c2c_of_its_window(dev, N, isz, nb):
    E.check_fastddc_fwd(dev, N, isz, nb)


@pytest.mark.parametrize("name", list(E.INV_GEOMS))
def test_fastddc_inverse_bound(dev, oracle, name):
    E.check_inv_bound(dev, oracle, name, full=True, expect=name.split(" M=")[0])


@pytest.mark.parametrize("name,nb,chn,expect", [("tiled M=16", 70, 67, "tiled 4x4"), ("tiled M=8", 70, 67, "tiled 4x4"), ("tiled M=32", 7, 5, "tiled 2x2"),
                                                ("fold M=64", 37, 35, "fold"), ("fold M=1024 post 3", 21, 19, "fold"),
                                                ("generic M=2048", 5, 4, "generic"), ("generic M=4", 9, 3, "generic")])
def test_fastddc_inverse_channel_equals_one_channel_bank(dev, name, nb, chn, expect):
    assert E.check_inv_channel_equals_one_channel(dev, name, nb, chn) == expect


@pytest.mark.parametrize("name", ["fold M=64", "fold M=1024 post 5", "tiled M=16", "generic M=1024 P=1"])
def test_fastddc_inverse_long_call_equals_one_block_calls(dev, name):
    E.check_inv_block_calls(dev, name, nb=200, chn=3)


@pytest.mark.parametrize("name,nb,chn,bad_block,bad_chan", [("fold M=64", 37, 35, 21, 34), ("fold M=256", 21, 18, 5, 17), ("tiled M=32", 7, 5, 6, 4),
                                                            ("tiled M=16", 70, 67, 69, 66), ("generic M=2048", 3, 2, 1, 0)])
def test_fastddc_inverse_nonfinite_windows(dev, oracle, name, nb, chn, bad_block, bad_chan):
    E.check_inv_nonfinite(dev, oracle, name, nb, chn, bad_block, bad_chan)


def test_every_path_row_was_exercised(dev):
    """runs last in this file: every row of the path table was hit on the GPU (and the worst error/bound ratio per path, printed with -s)"""
    E.check_coverage(dev)
