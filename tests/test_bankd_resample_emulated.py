"""CPU tier: csdr-bankd --resample on the emulated library (the bodies of tests/test_gpu_zzz_bankd_resample.py), and a brute-force check of
the condition under which the daemon accepts a resampler geometry."""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests" / "resampler"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402
import resampler as R  # noqa: E402

pytest.importorskip("torch")
import test_gpu_zzz_bankd as g  # noqa: E402
import test_gpu_zzz_bankd_resample as gr  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(g, "MULTI_DEVICES", lambda: ["0", "0,1"])])


test_nfm_resampled_to_48k_equals_the_oracle_graph = gr.test_nfm_resampled_to_48k_equals_the_oracle_graph
test_raw_resampled_discriminator_output = gr.test_raw_resampled_discriminator_output
test_refused_resample_geometries = gr.test_refused_resample_geometries


def test_resample_condition_rules_out_the_cap_by_brute_force():
    """The daemon accepts (I, D, T) when (T/I + 1)*I >= 2*D + I - 1.  For every I, D <= 24 and a spread of T around the boundary, the reference loop
    replayed over every call size up to 250 and every last_taps_delay never ends on the output cap inside the condition -- so the carried state
    continues the stream exactly -- while geometries outside it do (the condition is not vacuous)."""
    ro = R.Oracle()
    outside = 0
    for I in range(1, 25):
        for D in range(1, 25):
            for T in sorted({1, I, 2 * D - 1, 2 * D + I - 3, 2 * D + I - 2, 2 * D + I + 5, 79} - {0, -1}):
                endings = ro.cap_endings(I, D, T, 250)
                if (T // I + 1) * I >= 2 * D + I - 1:
                    assert endings == 0, (I, D, T, endings)
                else:
                    outside += endings
    assert outside > 0
