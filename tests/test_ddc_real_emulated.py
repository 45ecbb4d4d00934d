"""CPU tier: the real-input banks on the emulated library -- the test bodies of tests/test_gpu_ddc_real.py (shift_addition_fc bank, drop-in and CLI
against the reference bit for bit, the real fused DDC bank against the complex one on x + 0j, non-finite windows, refusals, the streaming object on
real blocks) with fewer and shorter cases, since the emulator walks every sample of every lane on the CPU."""
import ctypes as C
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_ddc_real as g  # noqa: E402
import spectrum as S  # noqa: E402  (tests/spectrum, on the path test_gpu_ddc_real sets)


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    return g.setup(S.EmulDev(C.CDLL(str(lib))))


@pytest.fixture(scope="module")
def cli(tmp_path_factory, monkeypatch_module):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, cli = emul_build.build_full_once(tmp_path_factory)
    monkeypatch_module.setenv("CSDRB_TEST_PRELOAD_LIB", str(lib))
    return str(cli)


@pytest.fixture(scope="module")
def monkeypatch_module():
    mp = pytest.MonkeyPatch()
    yield mp
    mp.undo()


@pytest.mark.parametrize("chunk,shared,n", g.SHIFT_CASES[:5])
def test_shift_bank_fc_is_the_reference_bit_for_bit(dev, chunk, shared, n):
    g.test_shift_bank_fc_is_the_reference_bit_for_bit(dev, chunk, shared, n)


@pytest.mark.parametrize("i,D,T", [(i, D, T) for i, (D, T) in enumerate(g.geometry_cases(True))])
def test_real_bank_equals_complex_bank_on_x_plus_0j(dev, i, D, T):
    g.check_real_equals_complex(dev, D, T, i, outputs=12)


@pytest.mark.parametrize("D,T", [(2, 7), (12, 97), (50, 801), (10, 79)])
def test_real_bank_nonfinite_stays_in_its_windows(dev, D, T):
    g.check_nonfinite(dev, D, T)


test_real_bank_refusals = g.test_real_bank_refusals


@pytest.mark.parametrize("D,T,ba,bb", [(50, 801, 4, 6), (12, 97, 2, 5)])
def test_bank_object_on_real_blocks(dev, D, T, ba, bb):
    g.check_stream(dev, D, T, ba, bb)


test_cli_shift_addition_fc = g.test_cli_shift_addition_fc
test_cli_shift_addition_fc_fd_tuning = g.test_cli_shift_addition_fc_fd_tuning
test_reference_binary_runs_shift_addition_fc_on_our_library = g.test_reference_binary_runs_shift_addition_fc_on_our_library
