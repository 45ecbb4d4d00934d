"""CPU tier: csdr-bankd on real (--real-s16, --real-f32) and complex s16 (--s16) streams, linked against the emulated library, with two pretend
devices for --devices -- the test bodies of tests/test_gpu_zzz_bankd_real.py.  The usb bandpass reference is the emulated library's own
csdrb_bandpass_fir_fft_bank_cc (tests/test_bankd_am_ssb_emulated.py)."""
import ctypes as C
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_bankd_am_ssb_emulated as ae  # noqa: E402
import test_gpu_zzz_bankd as base  # noqa: E402
import test_gpu_zzz_bankd_am_ssb as amg  # noqa: E402
import test_gpu_zzz_bankd_real as g  # noqa: E402


@pytest.fixture(scope="module")
def bankd(tmp_path_factory):
    yield from emul_build.emulated_bankd(tmp_path_factory, lambda lib, cli: [(base, "MULTI_DEVICES", lambda: ["0", "0,1"]), (ae._emul, "lib", C.CDLL(str(lib))),
                                                                             (amg, "BANDPASS", ae.emul_bandpass)])


test_real_s16_nfm_equals_the_oracle_graph = g.test_real_s16_nfm_equals_the_oracle_graph
test_real_f32_raw_discriminator = g.test_real_f32_raw_discriminator
test_real_s16_usb = g.test_real_s16_usb
test_complex_s16_equals_f32_of_its_conversion = g.test_complex_s16_equals_f32_of_its_conversion
test_real_input_over_several_devices = g.test_real_input_over_several_devices
test_real_input_refuses_the_waterfall = g.test_real_input_refuses_the_waterfall
