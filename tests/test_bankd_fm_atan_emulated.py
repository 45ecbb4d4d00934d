"""CPU tier: csdr-bankd --fm-demod atan on the emulated library, with two pretend devices for --devices -- the test bodies of
tests/test_gpu_zzz_bankd_fm_atan.py except the distortion measurement and the WfmAudioBank comparison, which need the GPU."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_fm_atan as g  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(base, "MULTI_DEVICES", lambda: ["0", "0,1"])])


test_none_is_fmdemod_atan_over_the_iq_tail = g.test_none_is_fmdemod_atan_over_the_iq_tail
test_tails_equal_their_checkers_on_the_atan_discriminator = g.test_tails_equal_their_checkers_on_the_atan_discriminator
test_rtty_tail_on_the_atan_discriminator = g.test_rtty_tail_on_the_atan_discriminator
test_atan_over_several_devices = g.test_atan_over_several_devices
test_fm_demod_refusals = g.test_fm_demod_refusals
