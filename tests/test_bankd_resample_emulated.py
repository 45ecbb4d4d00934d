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
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    lib, _cli = emul_build.build_full_once(tmp_path_factory)
    # --devices 0,1: two pretend devices and a memcpy stand-in for NCCL (tests/host_shim/fake_nccl.c), as in tests/test_bankd_emulated.py
    import os, subprocess
    fake = tmp_path_factory.mktemp("fake_nccl_r") / "libfake_nccl.so"
    subprocess.run(["gcc", "-O1", "-fPIC", "-shared", str(ROOT / "tests" / "host_shim" / "fake_nccl.c"), "-o", str(fake)], check=True)
    os.environ["CUDA_EMUL_DEVICES"] = "2"; os.environ["CSDRB_NCCL_LIB"] = str(fake)
    saved = g.MULTI_DEVICES
    g.MULTI_DEVICES = lambda: ["0", "0,1"]
    yield str(lib.parent / "csdr-bankd_emul")
    g.MULTI_DEVICES = saved
    del os.environ["CUDA_EMUL_DEVICES"], os.environ["CSDRB_NCCL_LIB"]


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
