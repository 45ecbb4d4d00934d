"""CPU tier: csdr-bankd --decimation 40 (host/bankd.c on the generic bank kernel) linked against the emulated library, against the oracle over the
whole stream, with two pretend devices for --devices.  Same test bodies as tests/test_gpu_zzz_bankd_generic.py."""
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
import test_gpu_zzz_bankd_generic as gen  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    fake = tmp_path_factory.mktemp("fake_nccl_gen") / "libfake_nccl.so"
    subprocess.run(["gcc", "-O1", "-fPIC", "-shared", str(ROOT / "tests" / "host_shim" / "fake_nccl.c"), "-o", str(fake)], check=True)
    os.environ["CUDA_EMUL_DEVICES"] = "2"; os.environ["CSDRB_NCCL_LIB"] = str(fake)
    saved = gen.MULTI_DEVICES
    gen.MULTI_DEVICES = lambda: ["0,1"]
    yield str(lib.parent / "csdr-bankd_emul")
    gen.MULTI_DEVICES = saved
    del os.environ["CUDA_EMUL_DEVICES"], os.environ["CSDRB_NCCL_LIB"]


test_decimation_40_equals_the_reference_chain = gen.test_decimation_40_equals_the_reference_chain
test_odd_decimation_is_refused = gen.test_odd_decimation_is_refused
