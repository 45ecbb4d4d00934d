"""CPU tier: the sample-format commands of our csdr CLI on the emulated library, against the unmodified reference CLI and library -- the bodies
of tests/test_gpu_formats_cli.py with the emulated build of tests/host_shim/emul_build.py (see tests/test_cli_emulated.py)."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_cli as gc  # noqa: E402
import test_gpu_formats_cli as g  # noqa: E402


@pytest.fixture(scope="module")
def clis(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    if not gc.REF.exists():
        pytest.skip("oracle/_ref/csdr_ref not built (needs the reference sources at build time)")
    lib, cli = emul_build.build_full_once(tmp_path_factory)
    saved = gc.LIB
    gc.LIB = lib                                                           # what the LD_PRELOAD test injects into the reference binary
    yield str(cli), str(gc.REF)
    gc.LIB = saved


test_bytes_equal_the_reference_cli = g.test_bytes_equal_the_reference_cli
test_convert_s24_f_is_the_reference_library_in_the_cli_loop = g.test_convert_s24_f_is_the_reference_library_in_the_cli_loop
test_s24_round_trips = g.test_s24_round_trips
test_reference_binary_runs_on_our_library = g.test_reference_binary_runs_on_our_library
