"""CPU tier: the BPSK31 commands of our csdr CLI on the emulated library, against the unmodified reference CLI -- the CLI test bodies of
tests/test_gpu_psk31.py with the emulated build of tests/host_shim/emul_build.py (see tests/test_cli_emulated.py)."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_cli as gc  # noqa: E402
import test_gpu_psk31 as g  # noqa: E402


@pytest.fixture(scope="module")
def clis(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    if not gc.REF.exists():
        pytest.skip("oracle/_ref/csdr_ref not built (needs /root/reference at build time)")
    lib, cli = emul_build.build_full_once(tmp_path_factory)
    yield str(cli), str(gc.REF)


test_psk31_commands_stage_for_stage = g.test_psk31_commands_stage_for_stage
test_psk31_pipe_decodes_seeded_text = g.test_psk31_pipe_decodes_seeded_text
test_psk31_refusals = g.test_psk31_refusals
