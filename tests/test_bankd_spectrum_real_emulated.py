"""CPU tier: `csdr fft_fc` and csdr-bankd --fft-real on the emulated library, with two pretend devices for --devices -- the test bodies of
tests/test_gpu_zzz_bankd_spectrum_real.py except the daemon-against-reference comparison and the full-rate FT8 run.  `csdr fft_fc` is compared with
the compiled reference CLI (oracle/_ref/csdr_ref) where that was built."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_spectrum_real as g  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(base, "MULTI_DEVICES", lambda: ["0", "0,1"]),
                                                                             (g.CLI, 0, cli)])   # the product CLI on the same emulated library


ref_cli = g.ref_cli
test_fft_fc_against_the_reference = g.test_fft_fc_against_the_reference
test_fft_fc_pipe_against_the_reference = g.test_fft_fc_pipe_against_the_reference
test_fft_fc_refusals = g.test_fft_fc_refusals
test_real_waterfall_equals_the_cli_pipe = g.test_real_waterfall_equals_the_cli_pipe
test_real_waterfall_over_several_devices = g.test_real_waterfall_over_several_devices
test_real_waterfall_refusals = g.test_real_waterfall_refusals
