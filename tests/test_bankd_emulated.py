"""CPU tier: csdr-bankd (host/bankd.c) linked against the emulated library -- the daemon's streaming bookkeeping (tails of the wideband
stream, the de-emphasis FIR's carried inputs, AGC block remainders), TCP ingest and TCP sink, checked against the oracle without a GPU.
Same test bodies as tests/test_gpu_zzz_bankd.py."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_zzz_bankd as g  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(g, "MULTI_DEVICES", lambda: ["0", "0,1"])])


test_nfm_bank_equals_the_readme_graph_per_channel = g.test_nfm_bank_equals_the_readme_graph_per_channel
test_raw_discriminator_output_and_f32_input = g.test_raw_discriminator_output_and_f32_input
test_tcp_ingest_and_tcp_sink = g.test_tcp_ingest_and_tcp_sink
