"""CPU tier: the demodulator commands of our csdr CLI on the emulated library, against the unmodified reference CLI -- the bodies of
tests/test_gpu_demod_cli.py with the emulated build of tests/host_shim/emul_build.py (see tests/test_cli_emulated.py)."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_cli as gc  # noqa: E402
import test_gpu_demod_cli as g  # noqa: E402


@pytest.fixture(scope="module")
def clis(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    if not gc.REF.exists():
        pytest.skip("oracle/_ref/csdr_ref not built (needs the reference sources at build time)")
    lib, cli = emul_build.build_full_once(tmp_path_factory)
    yield str(cli), str(gc.REF)


test_bytes_equal_the_reference_cli = g.test_bytes_equal_the_reference_cli
test_novect_bytes_equal_the_reference_cli = g.test_novect_bytes_equal_the_reference_cli
test_atan_whole_blocks_under_the_rounding_rule = g.test_atan_whole_blocks_under_the_rounding_rule
