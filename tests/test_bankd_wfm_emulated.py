"""CPU tier: csdr-bankd's WFM tail on the emulated library, with two pretend devices for --devices -- the test bodies of
tests/test_gpu_zzz_bankd_wfm.py except the comparison with the compiled reference CLI pipe at 2.4 Msps, which is too large for the emulator."""
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
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(base, "MULTI_DEVICES", lambda: ["0", "0,1"])])


test_wfm_tail_equals_the_checker_on_the_banks_discriminator = g.test_wfm_tail_equals_the_checker_on_the_banks_discriminator
test_wfm_tail_over_several_devices = g.test_wfm_tail_over_several_devices
test_wfm_refusals = g.test_wfm_refusals
