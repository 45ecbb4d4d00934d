"""CPU tier: csdr-bankd's single-GPU and --devices loops on the emulated library, with two pretend devices -- the test bodies of
tests/test_gpu_zzz_bankd_paths.py."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_paths as g  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(base, "MULTI_DEVICES", lambda: ["0", "0,1"])])


test_every_tail_gets_the_same_bytes_on_both_paths = g.test_every_tail_gets_the_same_bytes_on_both_paths
test_real_f32_gets_the_same_bytes_on_both_paths = g.test_real_f32_gets_the_same_bytes_on_both_paths
