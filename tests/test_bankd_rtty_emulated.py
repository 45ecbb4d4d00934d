"""CPU tier: csdr-bankd's RTTY tail on the emulated library, with two pretend devices for --devices -- the test bodies of
tests/test_gpu_zzz_bankd_rtty.py except the 2.4 Msps skimmer geometry, which is too large for the emulator."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_rtty as g  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(base, "MULTI_DEVICES", lambda: ["0", "0,1"])])


test_rtty_tail_equals_the_checker_on_the_banks_discriminator = g.test_rtty_tail_equals_the_checker_on_the_banks_discriminator
test_rtty_tail_over_several_devices = g.test_rtty_tail_over_several_devices
test_rtty_refusals = g.test_rtty_refusals
