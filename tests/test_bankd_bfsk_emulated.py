"""CPU tier: csdr-bankd's RTTY tail with tone filters on the emulated library, with two pretend devices for --devices -- the test bodies of
tests/test_gpu_zzz_bankd_bfsk.py, the CLI pipes run by the emulated csdr."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_bfsk as g  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    def patches(lib, cli):
        return [(base, "MULTI_DEVICES", lambda: ["0", "0,1"]), (g, "CLI", cli)]
    yield from emul_build.emulated_bankd(tmp_path_factory, patches)


test_bfsk_tail_equals_the_cli_pipe = g.test_bfsk_tail_equals_the_cli_pipe
test_bfsk_tail_over_several_devices = g.test_bfsk_tail_over_several_devices
test_bfsk_refusals = g.test_bfsk_refusals
test_tone_filters_beat_the_discriminator_in_noise = g.test_tone_filters_beat_the_discriminator_in_noise
