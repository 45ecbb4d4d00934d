"""CPU tier: csdr-bankd --s8 on the emulated library, with two pretend devices -- the test bodies of tests/test_gpu_zzz_bankd_s8.py but the
10 Msps end-to-end case."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_s8 as g  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(base, "MULTI_DEVICES", lambda: ["0", "0,1"])])


test_s8_equals_f32_of_the_converted_stream = g.test_s8_equals_f32_of_the_converted_stream
test_input_flags_stay_last_flag_wins = g.test_input_flags_stay_last_flag_wins
