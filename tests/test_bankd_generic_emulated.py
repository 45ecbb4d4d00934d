"""CPU tier: csdr-bankd --decimation 40 (host/bankd.c on the generic bank kernel) linked against the emulated library, against the oracle over the
whole stream, with two pretend devices for --devices.  Same test bodies as tests/test_gpu_zzz_bankd_generic.py."""
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
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(gen, "MULTI_DEVICES", lambda: ["0,1"])])


test_decimation_40_equals_the_reference_chain = gen.test_decimation_40_equals_the_reference_chain
test_odd_decimation_is_refused = gen.test_odd_decimation_is_refused
