"""CPU tier: csdr-bankd's WFM tail on the emulated library, with two pretend devices for --devices -- the test bodies of
tests/test_gpu_zzz_bankd_wfm.py except the comparison with the compiled reference CLI pipe at 2.4 Msps, which is too large for the emulator."""
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
import test_gpu_zzz_bankd_wfm as g  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    fake = tmp_path_factory.mktemp("fake_nccl_wfm") / "libfake_nccl.so"
    subprocess.run(["gcc", "-O1", "-fPIC", "-shared", str(ROOT / "tests" / "host_shim" / "fake_nccl.c"), "-o", str(fake)], check=True)
    os.environ["CUDA_EMUL_DEVICES"] = "2"; os.environ["CSDRB_NCCL_LIB"] = str(fake)
    saved = base.MULTI_DEVICES
    base.MULTI_DEVICES = lambda: ["0", "0,1"]
    yield str(lib.parent / "csdr-bankd_emul")
    base.MULTI_DEVICES = saved
    del os.environ["CUDA_EMUL_DEVICES"], os.environ["CSDRB_NCCL_LIB"]


test_wfm_tail_equals_the_checker_on_the_banks_discriminator = g.test_wfm_tail_equals_the_checker_on_the_banks_discriminator
test_wfm_tail_over_several_devices = g.test_wfm_tail_over_several_devices
test_wfm_refusals = g.test_wfm_refusals
