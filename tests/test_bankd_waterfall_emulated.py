"""CPU tier: csdr-bankd --waterfall on the emulated library, with two pretend devices for --devices -- the test bodies of
tests/test_gpu_zzz_bankd_waterfall.py except the comparison with the compiled reference CLI, which needs the real library."""
import os
import subprocess
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_waterfall as g  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, cli = emul_build.build_full_once(tmp_path_factory)
    fake = tmp_path_factory.mktemp("fake_nccl_wf") / "libfake_nccl.so"
    subprocess.run(["gcc", "-O1", "-fPIC", "-shared", str(ROOT / "tests" / "host_shim" / "fake_nccl.c"), "-o", str(fake)], check=True)
    os.environ["CUDA_EMUL_DEVICES"] = "2"; os.environ["CSDRB_NCCL_LIB"] = str(fake)
    saved, saved_cli = base.MULTI_DEVICES, g.CLI[0]
    base.MULTI_DEVICES = lambda: ["0", "0,1"]
    g.CLI[0] = cli                                                      # the product CLI on the same emulated library
    yield str(lib.parent / "csdr-bankd_emul")
    base.MULTI_DEVICES, g.CLI[0] = saved, saved_cli
    del os.environ["CUDA_EMUL_DEVICES"], os.environ["CSDRB_NCCL_LIB"]


test_waterfall_equals_the_cli_pipe = g.test_waterfall_equals_the_cli_pipe
test_waterfall_over_several_devices = g.test_waterfall_over_several_devices
test_slow_fifo_gets_whole_lines_only = g.test_slow_fifo_gets_whole_lines_only
test_waterfall_refusals = g.test_waterfall_refusals
