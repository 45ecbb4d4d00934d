"""CPU tier: csdr-bankd --waterfall on the emulated library, with two pretend devices for --devices -- the test bodies of
tests/test_gpu_zzz_bankd_waterfall.py except the comparison with the compiled reference CLI, which needs the real library."""
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
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(base, "MULTI_DEVICES", lambda: ["0", "0,1"]),
                                                                             (g.CLI, 0, cli)])   # the product CLI on the same emulated library


test_waterfall_equals_the_cli_pipe = g.test_waterfall_equals_the_cli_pipe
test_waterfall_over_several_devices = g.test_waterfall_over_several_devices
test_slow_fifo_gets_whole_lines_only = g.test_slow_fifo_gets_whole_lines_only
test_waterfall_refusals = g.test_waterfall_refusals
