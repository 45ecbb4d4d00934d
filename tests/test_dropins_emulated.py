"""CPU tier: the libcsdr-named host-pointer drop-ins (Part A of include/csdr_b200.h) on the EMULATED library.

The drop-in tests of the GPU modules run here unchanged: the fixtures below point csdr_b200 at the library that
tests/host_shim/emul_build.build_full() compiles from every product translation unit, so each drop-in's own contract (returned
phase, carried state structs, the fractional decimator's `where`, fastagc_ff's buffer rotation, untouched tails, return values
read from host memory) is pinned without a GPU (see tests/test_cli_emulated.py for the same arrangement with the CLI).
"""
import sys
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tests" / "host_shim"))
sys.path.insert(0, str(ROOT / "tests"))
import emul_build  # noqa: E402

pytest.importorskip("torch")
import test_gpu_am_ssb as am  # noqa: E402  (only their test bodies; their fixtures and gpu marks stay behind)
import test_gpu_nfm_tail as nfm  # noqa: E402
import test_gpu_parity as p1  # noqa: E402
import test_gpu_parity2 as p2  # noqa: E402
import test_gpu_shift_variants as sv  # noqa: E402
import test_gpu_zz_adpcm as za  # noqa: E402
import test_gpu_zz_shift_math as zm  # noqa: E402
import test_gpu_zz_shift_table as zt  # noqa: E402


@pytest.fixture(scope="module")
def gpu(tmp_path_factory):
    if not emul_build.available():
        pytest.skip("needs g++ and the CUDA toolkit headers")
    import csdr_b200
    lib, _ = emul_build.build_full_once(tmp_path_factory)
    saved = csdr_b200.LIB_PATH, csdr_b200._lib
    csdr_b200.LIB_PATH, csdr_b200._lib = lib, None
    csdr_b200.lib()
    yield csdr_b200
    csdr_b200.LIB_PATH, csdr_b200._lib = saved


@pytest.fixture(scope="module")
def cb(gpu):
    return gpu


test_convert_u8_f_dropin_bit_exact = p1.test_convert_u8_f_dropin_bit_exact
test_convert_s16_dropin_both_ways_bit_exact = p1.test_convert_s16_dropin_both_ways_bit_exact
test_fir_dropin_edge_geometries = p1.test_fir_dropin_edge_geometries
test_fir_dropin_golden = p1.test_fir_dropin_golden
test_fmdemod_quadri_dropin = p1.test_fmdemod_quadri_dropin

test_shift_dropin_and_golden = p2.test_shift_dropin_and_golden
test_fractional_decimator_positions_are_exact = p2.test_fractional_decimator_positions_are_exact
test_fractional_decimator_dropin_prefilter_and_golden = p2.test_fractional_decimator_dropin_prefilter_and_golden
test_fastagc_dropin = p2.test_fastagc_dropin
test_fft_dropin_all_sizes_vs_float64_dft = p2.test_fft_dropin_all_sizes_vs_float64_dft
test_bandpass_fir_fft_dropin_golden_and_reference = p2.test_bandpass_fir_fft_dropin_golden_and_reference
test_fastddc_dropin_golden = p2.test_fastddc_dropin_golden
test_audio_tail_dropin_limit_and_deemphasis = p2.test_audio_tail_dropin_limit_and_deemphasis
test_spectrum_path_and_shift_unroll_dropins = p2.test_spectrum_path_and_shift_unroll_dropins

test_deemphasis_nfm_dropin_golden_and_oracle = nfm.test_deemphasis_nfm_dropin_golden_and_oracle
test_deemphasis_nfm_dropin_degenerate_calls = nfm.test_deemphasis_nfm_dropin_degenerate_calls
test_shift_addfast_dropin_against_golden_and_oracle = sv.test_shift_addfast_dropin_against_golden_and_oracle
test_shift_math_dropin = zm.test_shift_math_dropin
test_shift_table_dropin_bit_exact = zt.test_shift_table_dropin_bit_exact
test_adpcm_dropin_bit_exact = za.test_adpcm_dropin_bit_exact
test_host_dropins = am.test_host_dropins
