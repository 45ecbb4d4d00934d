"""csdr_b200 -- H100-native csdr block-DSP hot path.

This package is a thin Python mirror of the C ABI in ``include/csdr_b200.h`` (ctypes; no torch types cross
the boundary -- tensors are passed as raw device pointers + the current CUDA stream handle).  PyTorch is
used for device memory, streams and torch.distributed only.  There is no CPU fallback: every compute call
goes to ``libcsdr_b200.so`` and raises if that library or a CUDA device is missing.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

import numpy as np

PKG = Path(__file__).resolve().parent
LIB_PATH = PKG / "libcsdr_b200.so"
WINDOWS = {"BOXCAR": 0, "BLACKMAN": 1, "HAMMING": 2}


class CsdrB200Error(RuntimeError):
    pass


class _CF(C.Structure):
    _fields_ = [("i", C.c_float), ("q", C.c_float)]


class _Shift(C.Structure):
    _fields_ = [("sindelta", C.c_float), ("cosdelta", C.c_float), ("rate", C.c_float)]


class _DShiftStatus(C.Structure):
    _fields_ = [("decimation_remain", C.c_int), ("starting_phase", C.c_float), ("output_size", C.c_int)]


class _FracDec(C.Structure):            # include/csdr_b200.h fractional_decimator_ff_t (= libcsdr.h:151-168)
    _fields_ = [("where", C.c_float), ("input_processed", C.c_int), ("output_size", C.c_int), ("num_poly_points", C.c_int),
                ("poly_precalc_denomiator", C.c_void_p), ("coeffs_buf", C.c_void_p), ("filtered_buf", C.c_void_p),
                ("xifirst", C.c_int), ("xilast", C.c_int), ("rate", C.c_float), ("taps", C.c_void_p), ("taps_length", C.c_int)]


class _Resampler(C.Structure):          # rational_resampler_ff_t (= libcsdr.h:132-137)
    _fields_ = [("input_processed", C.c_int), ("output_size", C.c_int), ("last_taps_delay", C.c_int)]


class _FastAgc(C.Structure):            # fastagc_ff_t (= libcsdr.h:118-128)
    _fields_ = [("buffer_1", C.c_void_p), ("buffer_2", C.c_void_p), ("buffer_input", C.c_void_p), ("peak_1", C.c_float),
                ("peak_2", C.c_float), ("input_size", C.c_int), ("reference", C.c_float), ("last_gain", C.c_float)]


class AgcParams(C.Structure):           # csdrb_agc_params_t; defaults = the agc_ff CLI's (csdr.c:1342-1361) with its 1024-sample calls
    _fields_ = [("reference", C.c_float), ("attack_rate", C.c_float), ("decay_rate", C.c_float), ("max_gain", C.c_float),
                ("hang_time", C.c_int), ("attack_wait_time", C.c_int), ("gain_filter_alpha", C.c_float), ("chunk", C.c_int)]

    def __init__(self, reference=0.2, attack_rate=0.01, decay_rate=0.0001, max_gain=65536.0, hang_time=200, attack_wait_time=0,
                 gain_filter_alpha=0.999, chunk=1024):
        super().__init__(reference, attack_rate, decay_rate, max_gain, hang_time, attack_wait_time, gain_filter_alpha, chunk)


class TimingRecoveryParams(C.Structure):    # csdrb_timing_recovery_params_t; algorithm 0 = GARDNER, 1 = EARLYLATE
    _fields_ = [("algorithm", C.c_int), ("decimation", C.c_int), ("use_q", C.c_int), ("loop_gain", C.c_float), ("max_error", C.c_float)]


class _TimingRecovery(C.Structure):     # timing_recovery_state_t (= libcsdr.h:322-336)
    _fields_ = [("algorithm", C.c_int), ("decimation_rate", C.c_int), ("output_size", C.c_int), ("input_processed", C.c_int),
                ("use_q", C.c_int), ("debug_phase", C.c_int), ("debug_every_nth", C.c_int), ("debug_writefiles_path", C.c_char_p),
                ("last_correction_offset", C.c_int), ("earlylate_ratio", C.c_float), ("loop_gain", C.c_float), ("max_error", C.c_float)]


class SerialLineParams(C.Structure):    # csdrb_serial_line_params_t
    _fields_ = [("samples_per_bits", C.c_float), ("databits", C.c_int), ("stopbits", C.c_float), ("bit_sampling_width_ratio", C.c_float)]


class SpectrumParams(C.Structure):      # csdrb_spectrum_params_t
    _fields_ = [("fft_size", C.c_int), ("every", C.c_int), ("averages", C.c_int), ("compress", C.c_int), ("add_db", C.c_float)]


class SpectrumState(C.Structure):       # csdrb_spectrum_state_t; {0, 0} at stream start
    _fields_ = [("consumed", C.c_longlong), ("frames", C.c_longlong)]


class WfmAudioParams(C.Structure):     # csdrb_wfm_audio_params_t
    _fields_ = [("rate", C.c_float), ("bufsize", C.c_int), ("tau", C.c_float), ("sample_rate", C.c_int)]


class WfmAudioState(C.Structure):      # csdrb_wfm_audio_state_t; zeroed at stream start
    _fields_ = [("where", C.c_float), ("audio", C.c_longlong)]


class _SerialLine(C.Structure):         # serial_line_t (= libcsdr.h:278-286)
    _fields_ = [("samples_per_bits", C.c_float), ("databits", C.c_int), ("stopbits", C.c_float), ("output_size", C.c_int),
                ("input_used", C.c_int), ("bit_sampling_width_ratio", C.c_float)]


class _Unroll(C.Structure):             # shift_unroll_data_t (= libcsdr.h:199-205)
    _fields_ = [("dsin", C.POINTER(C.c_float)), ("dcos", C.POINTER(C.c_float)), ("phase_increment", C.c_float), ("size", C.c_int)]


class _Table(C.Structure):              # shift_table_data_t (= libcsdr.h:180-184)
    _fields_ = [("table", C.POINTER(C.c_float)), ("table_size", C.c_int)]


class _Ima(C.Structure):                # ima_adpcm_state_t (= ima_adpcm.h:35-38)
    _fields_ = [("index", C.c_int), ("previousValue", C.c_int)]


class _AddFast(C.Structure):            # shift_addfast_data_t (= libcsdr.h:189-194)
    _fields_ = [("dsin", C.c_float * 4), ("dcos", C.c_float * 4), ("phase_increment", C.c_float)]


class _Plan(C.Structure):               # struct fft_plan_s (= fft_fftw.h:14-20)
    _fields_ = [("size", C.c_int), ("input", C.c_void_p), ("output", C.c_void_p), ("plan", C.c_void_p)]


class FastDDC(C.Structure):             # fastddc_t (= fastddc.h:5-24)
    _fields_ = [(n, C.c_int) for n in ("pre_decimation", "post_decimation", "taps_length", "taps_min_length", "overlap_length",
                                       "fft_size", "fft_inv_size", "input_size", "post_input_size")] + \
               [("pre_shift", C.c_float), ("startbin", C.c_int), ("v", C.c_int), ("offsetbin", C.c_int), ("post_shift", C.c_float),
                ("output_scrape", C.c_int), ("scrap", C.c_int), ("dsadata", _Shift)]


_lib = None


def build(force: bool = False):
    from .build import build as _b
    return _b(force=force)


def lib() -> C.CDLL:
    """Load libcsdr_b200.so (once).  Fails loudly when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise CsdrB200Error(f"{LIB_PATH} not built: run `python -m csdr_b200.build` (needs nvcc); there is no CPU fallback")
    L = C.CDLL(str(LIB_PATH))
    L.csdrb_last_error.restype = C.c_char_p
    L.csdrb_version.restype = C.c_char_p
    L.csdrb_kernel_launches.restype = C.c_long
    vp, lg, it = C.c_void_p, C.c_long, C.c_int
    L.csdrb_convert_u8_f.argtypes = [vp, vp, lg, vp]
    L.csdrb_convert_s16_f.argtypes = [vp, vp, lg, vp]
    L.csdrb_convert_f_s16.argtypes = [vp, vp, lg, vp]
    for name in ("csdrb_convert_s8_f", "csdrb_convert_f_s8", "csdrb_convert_f_u8"):
        getattr(L, name).argtypes = [vp, vp, lg, vp]
    L.csdrb_convert_s24_f.argtypes = [vp, vp, lg, it, vp]
    L.csdrb_convert_f_s24.argtypes = [vp, vp, lg, it, vp]
    L.csdrb_fir_decimate_bank_cc.argtypes = [vp, lg, vp, lg, it, it, it, C.POINTER(C.c_float), it, it, vp]
    L.csdrb_fmdemod_quadri_bank_cf.argtypes = [vp, lg, vp, lg, it, it, vp, vp, vp]
    L.csdrb_stream_synchronize.argtypes = [vp]
    L.csdrb_fir_decimate_bank_cc_host.argtypes = [vp, lg, vp, lg, it, it, it, C.POINTER(C.c_float), it, it]
    L.csdrb_fir_decimate_bank_u8_cc.argtypes = [vp, lg, vp, lg, it, it, it, C.POINTER(C.c_float), it, vp]
    L.csdrb_fir_decimate_bank_u8_host.argtypes = [vp, lg, vp, lg, it, it, it, C.POINTER(C.c_float), it, it]
    L.csdrb_host_alloc.argtypes = [C.c_size_t]; L.csdrb_host_alloc.restype = vp
    L.csdrb_host_free.argtypes = [vp]
    sz = C.c_size_t
    L.csdrb_shift_addition_bank_scratch_bytes.argtypes = [it, it, it]; L.csdrb_shift_addition_bank_scratch_bytes.restype = sz
    L.csdrb_shift_addition_bank_cc.argtypes = [vp, lg, vp, lg, it, it, vp, vp, it, vp, sz, vp]
    L.csdrb_shift_addition_bank_fc.argtypes = [vp, lg, vp, lg, it, it, vp, vp, it, vp, sz, vp]
    L.csdrb_decimating_shift_addition_bank_cc.argtypes = [vp, lg, vp, lg, it, it, vp, it, vp, vp, vp, vp]
    L.csdrb_fractional_decimator_bank_scratch_bytes.argtypes = [it, it, C.c_float]; L.csdrb_fractional_decimator_bank_scratch_bytes.restype = sz
    L.csdrb_fractional_decimator_bank_ff.argtypes = [vp, lg, vp, lg, it, it, C.c_float, it, vp, it, vp, vp, sz, vp]
    L.csdrb_fastagc_bank_scratch_bytes.argtypes = [it, it]; L.csdrb_fastagc_bank_scratch_bytes.restype = sz
    L.csdrb_fastagc_bank_ff.argtypes = [vp, lg, vp, lg, it, it, it, C.c_float, vp, vp, vp, sz, vp]
    L.csdrb_fastagc_bank_f_s16.argtypes = [vp, lg, vp, lg, it, it, it, C.c_float, vp, vp, vp, sz, vp]
    L.csdrb_amdemod_cf.argtypes = [vp, vp, lg, vp]
    L.csdrb_fastdcblock_bank_ff.argtypes = [vp, lg, it, vp, lg, it, it, it, vp, vp]
    L.csdrb_agc_bank_ff.argtypes = [vp, lg, it, vp, lg, it, it, it, C.POINTER(AgcParams), vp, C.c_float, vp]
    L.amdemod_cf.argtypes = [vp, vp, it]
    L.fastdcblock_ff.argtypes = [vp, vp, it, C.c_float]; L.fastdcblock_ff.restype = C.c_float
    L.agc_ff.argtypes = [vp, vp, it, C.c_float, C.c_float, C.c_float, C.c_float, C.c_short, C.c_short, C.c_float, C.c_float]
    L.agc_ff.restype = C.c_float
    L.csdrb_fft_c2c_batch.argtypes = [vp, lg, vp, lg, it, it, it, vp]
    L.csdrb_fft_c2c_large_batch.argtypes = [vp, lg, vp, lg, it, it, it, vp]
    L.csdrb_fft_r2c_batch.argtypes = [vp, lg, vp, lg, it, it, vp]
    L.csdrb_bandpass_fir_fft_bank_cc.argtypes = [vp, lg, vp, lg, it, it, it, it, vp, lg, vp, vp]
    L.csdrb_ddc_bank_scratch_bytes.argtypes = [it, it, it, it]; L.csdrb_ddc_bank_scratch_bytes.restype = sz
    L.csdrb_ddc_bank.argtypes = [vp, it, it, vp, vp, it, it, it, C.POINTER(C.c_float), it, it, vp, lg, vp, vp, vp, sz, vp]
    L.csdrb_ddc_bank_f.argtypes = [vp, it, it, vp, vp, it, it, it, C.POINTER(C.c_float), it, it, vp, lg, vp, vp, vp, sz, vp]
    L.csdrb_ddc_bank_create.argtypes = [it, C.POINTER(C.c_float), it, C.POINTER(C.c_float), it, it, it]; L.csdrb_ddc_bank_create.restype = vp
    L.csdrb_ddc_bank_destroy.argtypes = [vp]
    L.csdrb_ddc_bank_set_rate.argtypes = [vp, it, C.c_float]
    L.csdrb_ddc_bank_offset.argtypes = [vp]
    L.csdrb_ddc_bank_process.argtypes = [vp, vp, it, vp, lg, vp]
    L.csdrb_ddc_bank_process_f.argtypes = [vp, vp, it, vp, lg, vp]
    L.csdrb_ddc_bank_rechunk.argtypes = [vp]
    L.csdrb_fastddc_inv_plan_create.argtypes = [vp, it, vp, it]; L.csdrb_fastddc_inv_plan_create.restype = vp
    L.csdrb_fastddc_inv_plan_run.argtypes = [vp, vp, vp, vp, lg, vp, vp]
    L.csdrb_fastddc_inv_plan_set_channel.argtypes = [vp, it, vp]
    L.csdrb_fastddc_inv_plan_get_state.argtypes = [vp, vp, vp]
    L.csdrb_fastddc_inv_plan_set_state.argtypes = [vp, vp, vp]
    L.csdrb_fastddc_inv_plan_destroy.argtypes = [vp]
    L.csdrb_multi_bank_create.argtypes = [it, C.POINTER(C.c_int), it, C.POINTER(C.c_float), it, C.POINTER(C.c_float), it, it, it, it]; L.csdrb_multi_bank_create.restype = vp
    L.csdrb_multi_bank_destroy.argtypes = [vp]
    L.csdrb_multi_bank_devices.argtypes = [vp]
    L.csdrb_multi_bank_slice.argtypes = [vp, it, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.csdrb_multi_bank_set_rate.argtypes = [vp, it, C.c_float]
    L.csdrb_multi_bank_submit.argtypes = [vp, vp, it, vp, lg]
    L.csdrb_multi_bank_collect.argtypes = [vp, it]
    L.csdrb_multi_bank_process_host.argtypes = [vp, vp, it, vp, lg]
    L.csdrb_apply_window_rows_c.argtypes = [vp, vp, vp, it, lg, vp]
    L.csdrb_logpower_cf.argtypes = [vp, vp, lg, C.c_float, vp]
    L.csdrb_accumulate_power_cf.argtypes = [vp, vp, lg, vp]
    L.csdrb_log_ff.argtypes = [vp, vp, lg, C.c_float, vp]
    L.csdrb_shift_unroll_bank_cc.argtypes = [vp, lg, vp, lg, it, it, vp, vp, vp, lg, it, vp, vp, sz, vp]
    L.precalculate_window.argtypes = [it, it]; L.precalculate_window.restype = C.POINTER(C.c_float)
    L.apply_precalculated_window_c.argtypes = [vp, vp, it, vp]
    L.apply_window_c.argtypes = [vp, vp, it, it]
    L.logpower_cf.argtypes = [vp, vp, it, C.c_float]
    L.accumulate_power_cf.argtypes = [vp, vp, it]
    L.log_ff.argtypes = [vp, vp, it, C.c_float]
    L.shift_unroll_init.argtypes = [C.c_float, it]; L.shift_unroll_init.restype = _Unroll
    L.shift_unroll_cc.argtypes = [vp, vp, it, C.POINTER(_Unroll), C.c_float]; L.shift_unroll_cc.restype = C.c_float
    L.shift_math_cc.argtypes = [vp, vp, it, C.c_float, C.c_float]; L.shift_math_cc.restype = C.c_float
    L.shift_table_init.argtypes = [it]; L.shift_table_init.restype = _Table
    L.shift_table_deinit.argtypes = [_Table]
    L.shift_table_cc.argtypes = [vp, vp, it, C.c_float, _Table, C.c_float]; L.shift_table_cc.restype = C.c_float
    L.csdrb_shift_table_bank_cc.argtypes = [vp, lg, vp, lg, it, it, vp, vp, vp, it, vp, sz, vp]
    L.encode_ima_adpcm_i16_u8.argtypes = [vp, vp, it, _Ima]; L.encode_ima_adpcm_i16_u8.restype = _Ima
    L.csdrb_encode_ima_adpcm_rows_i16_u8.argtypes = [vp, lg, vp, lg, it, it, vp, vp]
    L.csdrb_compress_fft_adpcm_rows_f_u8.argtypes = [vp, lg, vp, lg, it, it, vp]
    L.csdrb_shift_math_bank_scratch_bytes.argtypes = [it, it]; L.csdrb_shift_math_bank_scratch_bytes.restype = sz
    L.csdrb_shift_math_bank_cc.argtypes = [vp, lg, vp, lg, it, it, vp, vp, vp, sz, vp]
    L.shift_addfast_init.argtypes = [C.c_float]; L.shift_addfast_init.restype = _AddFast
    L.shift_addfast_cc.argtypes = [vp, vp, it, C.POINTER(_AddFast), C.c_float]; L.shift_addfast_cc.restype = C.c_float
    L.csdrb_shift_addfast_bank_cc.argtypes = [vp, lg, vp, lg, it, it, vp, vp, it, vp, sz, vp]
    L.csdrb_limit_ff.argtypes = [vp, vp, lg, C.c_float, vp]
    L.csdrb_deemphasis_wfm_bank_ff.argtypes = [vp, lg, vp, lg, it, it, C.c_float, it, vp, vp]
    L.limit_ff.argtypes = [vp, vp, it, C.c_float]
    L.deemphasis_nfm_ff.argtypes = [vp, vp, it, it]
    L.csdrb_deemphasis_nfm_bank_ff.argtypes = [vp, lg, vp, lg, it, it, it, C.c_float, vp]
    L.csdrb_deemphasis_nfm_taps.argtypes = [it, C.POINTER(it)]; L.csdrb_deemphasis_nfm_taps.restype = C.POINTER(C.c_float)
    L.csdrb_fir_valid_bank_ff.argtypes = [vp, lg, vp, lg, it, it, C.POINTER(C.c_float), it, C.c_float, vp]
    L.deemphasis_wfm_ff.argtypes = [vp, vp, it, C.c_float, it, C.c_float]; L.deemphasis_wfm_ff.restype = C.c_float
    L.csdrb_fastddc_fwd_cc.argtypes = [vp, vp, vp, it, it, it, vp]
    L.csdrb_fastddc_inv_bank_scratch_bytes.argtypes = [it, it]; L.csdrb_fastddc_inv_bank_scratch_bytes.restype = sz
    L.csdrb_fastddc_inv_bank_cc.argtypes = [vp, it, vp, vp, it, C.POINTER(FastDDC), vp, vp, vp, lg, vp, vp, sz, vp]
    L.fastddc_init.argtypes = [C.POINTER(FastDDC), C.c_float, it, C.c_float]
    L.decimating_shift_addition_init.argtypes = [C.c_float, it]; L.decimating_shift_addition_init.restype = _Shift
    L.shift_addition_cc.argtypes = [vp, vp, it, _Shift, C.c_float]; L.shift_addition_cc.restype = C.c_float
    L.shift_addition_fc.argtypes = [vp, vp, it, _Shift, C.c_float]; L.shift_addition_fc.restype = C.c_float
    L.decimating_shift_addition_cc.argtypes = [vp, vp, it, _Shift, it, _DShiftStatus]; L.decimating_shift_addition_cc.restype = _DShiftStatus
    L.fractional_decimator_ff_init.argtypes = [C.c_float, it, vp, it]; L.fractional_decimator_ff_init.restype = _FracDec
    L.fractional_decimator_ff.argtypes = [vp, vp, it, C.POINTER(_FracDec)]
    L.fastagc_ff.argtypes = [C.POINTER(_FastAgc), vp]
    L.rational_resampler_ff.argtypes = [vp, vp, it, it, it, C.POINTER(C.c_float), it, it]; L.rational_resampler_ff.restype = _Resampler
    L.rational_resampler_get_lowpass_f.argtypes = [C.POINTER(C.c_float), it, it, it, it]
    L.csdrb_rational_resampler_bank_ff.argtypes = [vp, lg, vp, lg, it, it, it, it, C.POINTER(C.c_float), it, it, C.POINTER(_Resampler), vp]
    L.make_fft_c2c.argtypes = [it, vp, vp, it, it]; L.make_fft_c2c.restype = C.POINTER(_Plan)
    L.make_fft_r2c.argtypes = [it, vp, vp, it]; L.make_fft_r2c.restype = C.POINTER(_Plan)
    L.apply_precalculated_window_f.argtypes = [vp, vp, it, vp]
    L.fft_execute.argtypes = [C.POINTER(_Plan)]
    L.fft_destroy.argtypes = [C.POINTER(_Plan)]
    L.apply_fir_fft_cc.argtypes = [C.POINTER(_Plan), C.POINTER(_Plan), vp, vp, it]
    L.fastddc_inv_cc.argtypes = [vp, vp, C.POINTER(FastDDC), C.POINTER(_Plan), vp, _DShiftStatus]; L.fastddc_inv_cc.restype = _DShiftStatus
    L.fft_swap_sides.argtypes = [vp, it]
    # host-side design helpers (Part A)
    L.firdes_filter_len.argtypes = [C.c_float]
    L.firdes_lowpass_f.argtypes = [C.POINTER(C.c_float), it, C.c_float, it]
    L.firdes_bandpass_c.argtypes = [C.POINTER(_CF), it, C.c_float, C.c_float, it]
    L.shift_addition_init.argtypes = [C.c_float]; L.shift_addition_init.restype = _Shift
    L.next_pow2.argtypes = [it]
    # Part A compute wrappers on host pointers
    L.convert_u8_f.argtypes = [vp, vp, it]
    L.convert_s16_f.argtypes = [vp, vp, it]
    L.convert_f_s16.argtypes = [vp, vp, it]
    L.convert_s8_f.argtypes = [vp, vp, it]
    L.convert_f_s8.argtypes = [vp, vp, it]
    L.convert_f_u8.argtypes = [vp, vp, it]
    L.convert_s24_f.argtypes = [vp, vp, it, it]
    L.convert_f_s24.argtypes = [vp, vp, it, it]
    L.fir_decimate_cc.argtypes = [vp, vp, it, it, C.POINTER(C.c_float), it]
    L.fmdemod_quadri_cf.argtypes = [vp, vp, it, vp, _CF]; L.fmdemod_quadri_cf.restype = _CF
    L.csdrb_simple_agc_bank_cc.argtypes = [vp, lg, vp, lg, it, it, C.c_float, C.c_float, C.c_float, vp, vp]
    L.csdrb_timing_recovery_bank_cc.argtypes = [vp, lg, vp, vp, it, vp, lg, vp, vp, it, C.POINTER(TimingRecoveryParams), vp, vp]
    L.csdrb_dbpsk_decoder_bank_c_u8.argtypes = [vp, lg, vp, lg, it, it, vp, vp, vp, vp]
    L.csdrb_psk31_varicode_decoder_bank_u8_u8.argtypes = [vp, lg, vp, lg, it, it, vp, vp, vp, vp]
    L.simple_agc_cc.argtypes = [vp, vp, it, C.c_float, C.c_float, C.c_float, vp]
    L.dbpsk_decoder_c_u8.argtypes = [vp, vp, it]
    L.timing_recovery_init.argtypes = [it, it, it, C.c_float, C.c_float, it, C.c_char_p]; L.timing_recovery_init.restype = _TimingRecovery
    L.timing_recovery_cc.argtypes = [vp, vp, it, vp, vp, C.POINTER(_TimingRecovery)]
    L.csdrb_serial_line_decoder_bank_f_u8.argtypes = [vp, lg, it, vp, vp, lg, vp, vp, it, C.POINTER(SerialLineParams), it, vp]
    L.csdrb_rtty_baudot2ascii_bank_u8_u8.argtypes = [vp, lg, vp, lg, it, it, vp, vp, vp, vp]
    L.serial_line_decoder_f_u8.argtypes = [C.POINTER(_SerialLine), vp, vp, it]
    L.firdes_add_peak_c.argtypes = [vp, it, C.c_float, it, it, it]
    L.csdrb_apply_fir_bank_cc.argtypes = [vp, lg, vp, lg, it, it, vp, it, vp]
    L.csdrb_bfsk_demod_bank_cf.argtypes = [vp, lg, vp, lg, it, it, vp, vp, it, vp]
    L.csdrb_fir_interpolate_bank_cc.argtypes = [vp, lg, vp, lg, it, it, it, vp, it, vp]
    L.csdrb_fmmod_bank_fc.argtypes = [vp, lg, vp, lg, it, it, vp, vp]
    L.csdrb_gain_bank_ff.argtypes = [vp, lg, vp, lg, it, it, C.c_float, vp]
    L.csdrb_dsb_bank_fc.argtypes = [vp, lg, vp, lg, it, it, C.c_float, vp]
    L.csdrb_add_dcoffset_bank_cc.argtypes = [vp, lg, vp, lg, it, it, vp]
    L.csdrb_fixed_amplitude_bank_cc.argtypes = [vp, lg, vp, lg, it, it, C.c_float, vp]
    L.gain_ff.argtypes = [vp, vp, it, C.c_float]
    L.add_dcoffset_cc.argtypes = [vp, vp, it]
    L.fixed_amplitude_cc.argtypes = [vp, vp, it, C.c_float]
    L.csdrb_psk31_varicode_encoder_bank_u8_u8.argtypes = [vp, lg, vp, lg, it, it, vp, it, vp, vp, vp]
    L.csdrb_differential_codec_bank_u8_u8.argtypes = [vp, lg, vp, lg, it, it, vp, it, vp, vp]
    L.csdrb_psk_modulator_bank_u8_c.argtypes = [vp, lg, vp, lg, it, it, vp, it, vp]
    L.csdrb_psk31_interpolate_sine_bank_cc.argtypes = [vp, lg, vp, lg, it, it, vp, it, vp, vp]
    L.psk31_varicode_encoder_u8_u8.argtypes = [vp, vp, it, it, C.POINTER(it), C.POINTER(it)]
    L.differential_codec.argtypes = [vp, vp, it, it, C.c_ubyte]; L.differential_codec.restype = C.c_ubyte
    L.psk_modulator_u8_c.argtypes = [vp, vp, it, it]
    L.psk31_interpolate_sine_cc.argtypes = [vp, vp, it, it, _CF]; L.psk31_interpolate_sine_cc.restype = _CF
    L.csdrb_synth_bank_scratch_bytes.argtypes = [it, it, it, it, it, it]; L.csdrb_synth_bank_scratch_bytes.restype = sz
    L.csdrb_synth_bank_cc.argtypes = [vp, lg, it, it, it, vp, it, vp, vp, it, it, vp, vp, sz, vp]
    L.csdrb_synth_bank_create.argtypes = [it, C.POINTER(C.c_float), it, C.POINTER(C.c_float), it, it]; L.csdrb_synth_bank_create.restype = vp
    L.csdrb_synth_bank_destroy.argtypes = [vp]
    L.csdrb_synth_bank_process.argtypes = [vp, vp, lg, it, vp, vp]
    L.csdrb_spectrum_bank_lines.argtypes = [C.POINTER(SpectrumParams), C.POINTER(SpectrumState), lg]; L.csdrb_spectrum_bank_lines.restype = lg
    L.csdrb_spectrum_bank_scratch_bytes.argtypes = [it, lg, C.POINTER(SpectrumParams)]; L.csdrb_spectrum_bank_scratch_bytes.restype = sz
    L.csdrb_spectrum_bank_cf.argtypes = [vp, lg, it, lg, vp, C.POINTER(SpectrumParams), vp, vp, C.POINTER(SpectrumState), vp, lg, vp, sz, vp]
    L.csdrb_spectrum_bank_lines_f.argtypes = [C.POINTER(SpectrumParams), C.POINTER(SpectrumState), lg]; L.csdrb_spectrum_bank_lines_f.restype = lg
    L.csdrb_spectrum_bank_scratch_bytes_f.argtypes = [it, lg, C.POINTER(SpectrumParams)]; L.csdrb_spectrum_bank_scratch_bytes_f.restype = sz
    L.csdrb_spectrum_bank_f.argtypes = [vp, lg, it, lg, vp, C.POINTER(SpectrumParams), vp, vp, C.POINTER(SpectrumState), vp, lg, vp, sz, vp]
    L.csdrb_wfm_audio_bank_outputs.argtypes = [C.POINTER(WfmAudioParams), C.POINTER(WfmAudioState), it, C.POINTER(it)]
    L.csdrb_wfm_audio_bank_f_s16.argtypes = [vp, lg, it, it, C.POINTER(WfmAudioParams), C.POINTER(WfmAudioState), vp, vp, lg, C.POINTER(it), vp]
    _lib = L
    return L


def _check(rc: int, what: str) -> int:
    if rc < 0:
        raise CsdrB200Error(f"{what}: {lib().csdrb_last_error().decode()} (rc={rc})")
    return rc


def _stream():
    import torch
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _fp(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def kernel_launches() -> int:
    return int(lib().csdrb_kernel_launches())


# --------------------------------------------------------------------------------------------------
# host-side design helpers (run on the CPU exactly where the reference runs them)
# --------------------------------------------------------------------------------------------------
def firdes_filter_len(transition_bw: float) -> int:
    return int(lib().firdes_filter_len(transition_bw))


def firdes_lowpass_f(length: int, cutoff_rate: float, window: str = "HAMMING") -> np.ndarray:
    t = np.empty(length, np.float32)
    lib().firdes_lowpass_f(_fp(t), length, cutoff_rate, WINDOWS[window])
    return t


def rational_resampler_get_lowpass_f(length: int, interpolation: int, decimation: int, window: str = "HAMMING") -> np.ndarray:
    """the lowpass rational_resampler_ff's CLI designs (libcsdr.c:665-673): cutoff at half the lower of 1/I and 1/D"""
    t = np.empty(length, np.float32)
    lib().rational_resampler_get_lowpass_f(_fp(t), length, interpolation, decimation, WINDOWS[window])
    return t


def firdes_bandpass_c(length: int, lowcut: float, highcut: float, window: str = "HAMMING") -> np.ndarray:
    t = np.empty(length, np.complex64)
    lib().firdes_bandpass_c(t.ctypes.data_as(C.POINTER(_CF)), length, lowcut, highcut, WINDOWS[window])
    return t


# --------------------------------------------------------------------------------------------------
# device-resident bank API (torch CUDA tensors in, torch CUDA tensors out)
# --------------------------------------------------------------------------------------------------
def _as_cf32_rows(x):
    """Accept [C, N] complex64 or [C, N, 2] float32 CUDA tensors; return (tensor, data_ptr, row stride in samples, C, N)."""
    import torch
    if x.dtype == torch.complex64:
        xr = torch.view_as_real(x)
    elif x.dtype == torch.float32 and x.shape[-1] == 2:
        xr = x
    else:
        raise TypeError("expected complex64 [C,N] or float32 [C,N,2]")
    if xr.dim() == 2:
        xr = xr.unsqueeze(0)
    if not xr.is_cuda:
        raise CsdrB200Error("bank API needs CUDA tensors (no CPU fallback)")
    if xr.stride(2) != 1 or xr.stride(1) != 2:
        raise ValueError("samples must be contiguous within a channel row")
    return xr, xr.data_ptr(), xr.stride(0) // 2, xr.shape[0], xr.shape[1]


def convert_u8_f(x, out=None):
    import torch
    assert x.dtype == torch.uint8 and x.is_cuda and x.is_contiguous()
    out = torch.empty(x.shape, dtype=torch.float32, device=x.device) if out is None else out
    _check(lib().csdrb_convert_u8_f(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "convert_u8_f")
    return out


def convert_s16_f(x, out=None):
    import torch
    assert x.dtype == torch.int16 and x.is_cuda and x.is_contiguous()
    out = torch.empty(x.shape, dtype=torch.float32, device=x.device) if out is None else out
    _check(lib().csdrb_convert_s16_f(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "convert_s16_f")
    return out


def convert_f_s16(x, out=None):
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    out = torch.empty(x.shape, dtype=torch.int16, device=x.device) if out is None else out
    _check(lib().csdrb_convert_f_s16(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "convert_f_s16")
    return out


def convert_s8_f(x, out=None):
    """HackRF-style signed 8-bit values -> float32 of the same shape: (float)b * (1.0f/127.0f), as the reference build computes it."""
    import torch
    assert x.dtype == torch.int8 and x.is_cuda and x.is_contiguous()
    out = torch.empty(x.shape, dtype=torch.float32, device=x.device) if out is None else out
    _check(lib().csdrb_convert_s8_f(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "convert_s8_f")
    return out


def convert_f_s8(x, out=None):
    """float32 -> int8 of the same shape: x*127 truncated, the low byte kept (out of range wraps, NaN/Inf give 0)."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    out = torch.empty(x.shape, dtype=torch.int8, device=x.device) if out is None else out
    _check(lib().csdrb_convert_f_s8(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "convert_f_s8")
    return out


def convert_f_u8(x, out=None):
    """float32 -> uint8 of the same shape: x*255*0.5 + 128 truncated, the low byte kept (out of range wraps, NaN/Inf give 0)."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    out = torch.empty(x.shape, dtype=torch.uint8, device=x.device) if out is None else out
    _check(lib().csdrb_convert_f_u8(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "convert_f_u8")
    return out


def convert_s24_f(x, bigendian=False, out=None):
    """24-bit samples, a uint8 tensor of 3n bytes -> n float32.  ``bigendian`` is the reference's flag: False reads the most significant
    byte first, True the least significant byte first (on x86 the flag does the opposite of its name)."""
    import torch
    assert x.dtype == torch.uint8 and x.is_cuda and x.is_contiguous() and x.numel() % 3 == 0
    n = x.numel() // 3
    out = torch.empty(n, dtype=torch.float32, device=x.device) if out is None else out
    _check(lib().csdrb_convert_s24_f(x.data_ptr(), out.data_ptr(), n, int(bool(bigendian)), _stream()), "convert_s24_f")
    return out


def convert_f_s24(x, bigendian=False, out=None):
    """n float32 -> 3n uint8 bytes of 24-bit samples: x*8388607 truncated, the low three bytes kept, in the order ``bigendian`` gives (as in
    convert_s24_f)."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    out = torch.empty(3 * x.numel(), dtype=torch.uint8, device=x.device) if out is None else out
    _check(lib().csdrb_convert_f_s24(x.data_ptr(), out.data_ptr(), x.numel(), int(bool(bigendian)), _stream()), "convert_f_s24")
    return out


def fir_out_len(input_size: int, decimation: int, taps_length: int) -> int:
    """Outputs of one fir_decimate_cc call (reference libcsdr.c:537-547)."""
    return (input_size - taps_length) // decimation + 1 if input_size >= taps_length else 0


def fir_decimate_bank_cc(x, decimation: int, taps: np.ndarray, out=None, variant: int = -1):
    """C independent cf32 streams [C, N] -> [C, n_out]; all channels share ``taps`` (host float32 array)."""
    import torch
    xr, ptr, stride, ch, n = _as_cf32_rows(x)
    taps = np.ascontiguousarray(taps, np.float32)
    n_out = fir_out_len(n, decimation, taps.size)
    if out is None:
        out = torch.empty((ch, n_out + (n_out & 1)), dtype=torch.complex64, device=xr.device)
    orr, optr, ostride, och, on = _as_cf32_rows(out)
    assert och == ch and on >= n_out
    rc = _check(lib().csdrb_fir_decimate_bank_cc(ptr, stride, optr, ostride, ch, n, decimation, _fp(taps), taps.size, variant, _stream()),
                "fir_decimate_bank_cc")
    assert rc == n_out, (rc, n_out)
    return out[:, :n_out]


class PinnedArray:
    """A page-locked host buffer from csdrb_host_alloc exposed as a numpy array (freed on close/del)."""

    def __init__(self, shape, dtype):
        self.shape = tuple(shape); self.dtype = np.dtype(dtype)
        nbytes = int(np.prod(self.shape)) * self.dtype.itemsize
        self.ptr = lib().csdrb_host_alloc(nbytes)
        if not self.ptr:
            raise CsdrB200Error(f"csdrb_host_alloc({nbytes}): {lib().csdrb_last_error().decode()}")
        buf = (C.c_char * nbytes).from_address(self.ptr)
        self.array = np.frombuffer(buf, dtype=self.dtype).reshape(self.shape)

    def close(self):
        if getattr(self, "ptr", None):
            self.array = None
            lib().csdrb_host_free(self.ptr); self.ptr = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def fir_decimate_bank_cc_host(x: np.ndarray, decimation: int, taps: np.ndarray, out: np.ndarray | None = None, chunk_channels: int = 0):
    """End-to-end call on HOST arrays: x [C, N] complex64 -> out [C, n_out] complex64 (H2D, kernel, D2H inside)."""
    assert x.dtype == np.complex64 and x.ndim == 2 and x.strides[1] == 8
    taps = np.ascontiguousarray(taps, np.float32)
    ch, n = x.shape
    n_out = fir_out_len(n, decimation, taps.size)
    if out is None:
        out = np.empty((ch, n_out), np.complex64)
    assert out.dtype == np.complex64 and out.shape[0] == ch and out.shape[1] >= n_out and out.strides[1] == 8
    rc = _check(lib().csdrb_fir_decimate_bank_cc_host(x.ctypes.data, x.strides[0] // 8, out.ctypes.data, out.strides[0] // 8, ch, n,
                                                      decimation, _fp(taps), taps.size, chunk_channels), "fir_decimate_bank_cc_host")
    assert rc == n_out
    return out[:, :n_out]


def fir_decimate_bank_u8_cc(x, decimation: int, taps: np.ndarray, out=None):
    """convert_u8_f | fir_decimate_cc fused: x [C, N, 2] uint8 CUDA tensor (interleaved I,Q; rows N samples apart or padded) -> [C, n_out] cf32."""
    import torch
    assert x.dtype == torch.uint8 and x.dim() == 3 and x.shape[2] == 2 and x.stride(2) == 1 and x.stride(1) == 2 and x.stride(0) % 2 == 0
    ch, n = x.shape[0], x.shape[1]
    taps = np.ascontiguousarray(taps, np.float32)
    n_out = fir_out_len(n, decimation, taps.size)
    if out is None:
        out = torch.empty((ch, n_out + (n_out & 1)), dtype=torch.complex64, device=x.device)
    orr, optr, ostride, och, on = _as_cf32_rows(out)
    assert och == ch and on >= n_out
    rc = _check(lib().csdrb_fir_decimate_bank_u8_cc(x.data_ptr(), x.stride(0) // 2, optr, ostride, ch, n, decimation, _fp(taps), taps.size, _stream()),
                "fir_decimate_bank_u8_cc")
    assert rc == n_out, (rc, n_out)
    return out[:, :n_out]


def fir_decimate_bank_u8_host(x: np.ndarray, decimation: int, taps: np.ndarray, out: np.ndarray | None = None, chunk_channels: int = 0):
    """End-to-end call on HOST arrays with rtl_sdr-style input: x [C, N, 2] uint8 -> out [C, n_out] complex64 (2 bytes per sample over PCIe)."""
    assert x.dtype == np.uint8 and x.ndim == 3 and x.shape[2] == 2 and x.strides[2] == 1 and x.strides[1] == 2
    taps = np.ascontiguousarray(taps, np.float32)
    ch, n = x.shape[0], x.shape[1]
    n_out = fir_out_len(n, decimation, taps.size)
    if out is None:
        out = np.empty((ch, n_out), np.complex64)
    assert out.dtype == np.complex64 and out.shape[0] == ch and out.shape[1] >= n_out and out.strides[1] == 8
    rc = _check(lib().csdrb_fir_decimate_bank_u8_host(x.ctypes.data, x.strides[0] // 2, out.ctypes.data, out.strides[0] // 8, ch, n,
                                                      decimation, _fp(taps), taps.size, chunk_channels), "fir_decimate_bank_u8_host")
    assert rc == n_out
    return out[:, :n_out]


def fmdemod_quadri_bank_cf(x, last=None, out=None, return_last: bool = False):
    """[C, N] cf32 -> [C, N] f32.  ``last`` is a [C] complex64 CUDA tensor (sample before each block) or None."""
    import torch
    xr, ptr, stride, ch, n = _as_cf32_rows(x)
    if out is None:
        out = torch.empty((ch, n + (n & 1)), dtype=torch.float32, device=xr.device)
    assert out.stride(1) == 1 and out.shape[0] == ch
    last_out = torch.empty(ch, dtype=torch.complex64, device=xr.device) if return_last else None
    _check(lib().csdrb_fmdemod_quadri_bank_cf(ptr, stride, out.data_ptr(), out.stride(0), ch, n,
                                              last.data_ptr() if last is not None else None,
                                              last_out.data_ptr() if last_out is not None else None, _stream()),
           "fmdemod_quadri_bank_cf")
    res = out[:, :n]
    return (res, last_out) if return_last else res


# --------------------------------------------------------------------------------------------------
# libcsdr drop-in calls on HOST arrays (Part A of the C ABI) -- what the reference's callers bind
# --------------------------------------------------------------------------------------------------
class libcsdr:
    """numpy-in / numpy-out front-end over the libcsdr-named host-pointer entry points."""

    @staticmethod
    def convert_u8_f(x):
        x = np.ascontiguousarray(x, np.uint8); y = np.empty(x.size, np.float32)
        lib().convert_u8_f(x.ctypes.data, y.ctypes.data, x.size); return y

    @staticmethod
    def simple_agc_cc(x, rate, reference=1.0, max_gain=65535.0, gain=1.0):
        """-> (y, gain)"""
        x = np.ascontiguousarray(x, np.complex64); y = np.empty_like(x); g = np.array([gain], np.float32)
        lib().simple_agc_cc(x.ctypes.data, y.ctypes.data, x.size, rate, reference, max_gain, g.ctypes.data); return y, float(g[0])

    @staticmethod
    def dbpsk_decoder_c_u8(x):
        """the previous sample of the last call is library state, as in the reference"""
        x = np.ascontiguousarray(x, np.complex64); y = np.empty(x.size, np.uint8)
        lib().dbpsk_decoder_c_u8(x.ctypes.data, y.ctypes.data, x.size); return y

    @staticmethod
    def timing_recovery_cc(x, algorithm, decimation, use_q=True, loop_gain=0.5, max_error=2.0, last_correction_offset=0):
        """-> (symbols, error, indexes, (last_correction_offset, input_processed, output_size))"""
        x = np.ascontiguousarray(x, np.complex64); cap = max(x.size, 1)
        y = np.empty(cap, np.complex64); e = np.empty(cap, np.float32); ix = np.empty(cap, np.int32)
        st = lib().timing_recovery_init(algorithm, decimation, int(use_q), loop_gain, max_error, -1, None)
        st.last_correction_offset = last_correction_offset
        lib().timing_recovery_cc(x.ctypes.data, y.ctypes.data, x.size, e.ctypes.data, ix.ctypes.data, C.byref(st))
        m = st.output_size
        return y[:m].copy(), e[:m].copy(), ix[:m].copy(), (st.last_correction_offset, st.input_processed, m)

    @staticmethod
    def serial_line_decoder_f_u8(x, samples_per_bits, databits=8, stopbits=1.0, bit_sampling_width_ratio=0.4):
        """one call -> (characters as bytes, input_used)"""
        x = np.ascontiguousarray(x, np.float32); y = np.empty(max(x.size, 1), np.uint8)
        s = _SerialLine(samples_per_bits, databits, stopbits, 0, 0, bit_sampling_width_ratio)
        lib().serial_line_decoder_f_u8(C.byref(s), x.ctypes.data, y.ctypes.data, x.size)
        return y[:s.output_size].tobytes(), s.input_used

    @staticmethod
    def convert_s16_f(x):
        x = np.ascontiguousarray(x, np.int16); y = np.empty(x.size, np.float32)
        lib().convert_s16_f(x.ctypes.data, y.ctypes.data, x.size); return y

    @staticmethod
    def convert_f_s16(x):
        x = np.ascontiguousarray(x, np.float32); y = np.empty(x.size, np.int16)
        lib().convert_f_s16(x.ctypes.data, y.ctypes.data, x.size); return y

    @staticmethod
    def convert_s8_f(x):
        x = np.ascontiguousarray(x, np.int8); y = np.empty(x.size, np.float32)
        lib().convert_s8_f(x.ctypes.data, y.ctypes.data, x.size); return y

    @staticmethod
    def convert_f_s8(x):
        x = np.ascontiguousarray(x, np.float32); y = np.empty(x.size, np.int8)
        lib().convert_f_s8(x.ctypes.data, y.ctypes.data, x.size); return y

    @staticmethod
    def convert_f_u8(x):
        x = np.ascontiguousarray(x, np.float32); y = np.empty(x.size, np.uint8)
        lib().convert_f_u8(x.ctypes.data, y.ctypes.data, x.size); return y

    @staticmethod
    def convert_s24_f(x, bigendian=False):
        x = np.ascontiguousarray(x, np.uint8); y = np.empty(x.size // 3, np.float32)
        lib().convert_s24_f(x.ctypes.data, y.ctypes.data, y.size, int(bool(bigendian))); return y

    @staticmethod
    def convert_f_s24(x, bigendian=False):
        x = np.ascontiguousarray(x, np.float32); y = np.empty(3 * x.size, np.uint8)
        lib().convert_f_s24(x.ctypes.data, y.ctypes.data, x.size, int(bool(bigendian))); return y

    @staticmethod
    def fir_decimate_cc(x, decimation, taps):
        x = np.ascontiguousarray(x, np.complex64); taps = np.ascontiguousarray(taps, np.float32)
        y = np.empty(max(x.size // decimation + 1, 1), np.complex64)
        n = lib().fir_decimate_cc(x.ctypes.data, y.ctypes.data, x.size, decimation, _fp(taps), taps.size)
        return y[:n].copy()

    @staticmethod
    def shift_addition_cc(x, rate, phase=0.0, chunk=None):
        x = np.ascontiguousarray(x, np.complex64); y = np.empty_like(x); d = lib().shift_addition_init(rate)
        chunk = chunk or max(x.size, 1)
        for s in range(0, x.size, chunk):
            n = min(chunk, x.size - s)
            phase = lib().shift_addition_cc(x[s:].ctypes.data, y[s:].ctypes.data, n, d, phase)
        return y, float(np.float32(phase))

    @staticmethod
    def shift_addition_fc(x, rate, phase=0.0, chunk=None):
        """real x -> (complex64 y, phase): one shift_addition_fc call per `chunk` samples"""
        x = np.ascontiguousarray(x, np.float32); y = np.empty(x.size, np.complex64); d = lib().shift_addition_init(rate)
        chunk = chunk or max(x.size, 1)
        for s in range(0, x.size, chunk):
            n = min(chunk, x.size - s)
            phase = lib().shift_addition_fc(x[s:].ctypes.data, y[s:].ctypes.data, n, d, phase)
        return y, float(np.float32(phase))

    @staticmethod
    def decimating_shift_addition_cc(x, rate, decimation, remain=0, phase=0.0):
        x = np.ascontiguousarray(x, np.complex64); y = np.empty(x.size // decimation + 2, np.complex64)
        d = lib().decimating_shift_addition_init(rate, decimation)
        st = lib().decimating_shift_addition_cc(x.ctypes.data, y.ctypes.data, x.size, d, decimation, _DShiftStatus(remain, phase, 0))
        return y[:st.output_size].copy(), (st.decimation_remain, st.starting_phase)

    @staticmethod
    def fractional_decimator_ff(x, rate, num_poly_points=12, taps=None, block=None):
        """block=None: one call; else the CLI's block loop with tail re-feeding (csdr.c:1510-1522)."""
        x = np.ascontiguousarray(x, np.float32)
        tp = np.ascontiguousarray(taps, np.float32) if taps is not None else None
        d = lib().fractional_decimator_ff_init(rate, num_poly_points, tp.ctypes.data if tp is not None else None, tp.size if tp is not None else 0)
        if block is None:
            out = np.empty(int(x.size / max(rate, 1.0)) + 16, np.float32)
            lib().fractional_decimator_ff(x.ctypes.data, out.ctypes.data, x.size, C.byref(d))
            return out[:d.output_size].copy()
        buf = np.zeros(block, np.float32); out = np.empty(block, np.float32); outs = []; pos = 0
        while True:
            if d.input_processed == 0:
                need, keep = block, 0
            else:
                need = d.input_processed; keep = block - need
                buf[:keep] = buf[need:].copy()
            if pos + need > x.size:
                break
            buf[keep:] = x[pos:pos + need]; pos += need
            if d.input_processed == 0:
                d.input_processed = block
            lib().fractional_decimator_ff(buf.ctypes.data, out.ctypes.data, block, C.byref(d))
            outs.append(out[:d.output_size].copy())
        return np.concatenate(outs) if outs else np.zeros(0, np.float32)

    @staticmethod
    def rational_resampler_ff(x, interpolation, decimation, taps, block=None, last_taps_delay=0):
        """block=None: one call on all of x, returns (y, (input_processed, output_size, last_taps_delay)).
        Else the CLI's block loop (csdr.c:1448-1461) over the complete reads of x: the first call takes `block` samples, each later one the
        unconsumed tail plus input_processed new samples; returns the concatenated output."""
        x = np.ascontiguousarray(x, np.float32); taps = np.ascontiguousarray(taps, np.float32)
        if block is None:
            y = np.empty(max(x.size * interpolation // decimation, 1), np.float32)
            d = lib().rational_resampler_ff(x.ctypes.data, y.ctypes.data, x.size, interpolation, decimation, _fp(taps), taps.size, last_taps_delay)
            return y[:d.output_size].copy(), (d.input_processed, d.output_size, d.last_taps_delay)
        buf = np.zeros(block, np.float32); out = np.empty(max(block * interpolation // decimation, 1), np.float32)
        d = _Resampler(0, 0, last_taps_delay); pos = 0; outs = []
        while True:
            need = block if d.input_processed == 0 else d.input_processed
            if d.input_processed:
                buf[:block - need] = buf[need:].copy()
            if pos + need > x.size:
                break
            buf[block - need:] = x[pos:pos + need]; pos += need
            d = lib().rational_resampler_ff(buf.ctypes.data, out.ctypes.data, block, interpolation, decimation, _fp(taps), taps.size, d.last_taps_delay)
            outs.append(out[:d.output_size].copy())
        return np.concatenate(outs) if outs else np.zeros(0, np.float32)

    @staticmethod
    def fastagc_ff(x, block=1024, reference=1.0):
        x = np.ascontiguousarray(x, np.float32); nblk = x.size // block
        bufs = [np.zeros(block, np.float32) for _ in range(3)]
        byaddr = {b.ctypes.data: b for b in bufs}
        st = _FastAgc(bufs[0].ctypes.data, bufs[1].ctypes.data, bufs[2].ctypes.data, 0, 0, block, reference, 0)
        y = np.empty(nblk * block, np.float32)
        for b in range(nblk):
            byaddr[st.buffer_input][:] = x[b * block:(b + 1) * block]
            lib().fastagc_ff(C.byref(st), y[b * block:].ctypes.data)
        return y

    @staticmethod
    def amdemod_cf(x):
        x = np.ascontiguousarray(x, np.complex64); y = np.empty(x.size, np.float32)
        lib().amdemod_cf(x.ctypes.data, y.ctypes.data, x.size); return y

    @staticmethod
    def fastdcblock_ff(x, last_dc=0.0):
        """one call on one block: (y, block average)"""
        x = np.ascontiguousarray(x, np.float32); y = np.empty_like(x)
        avg = lib().fastdcblock_ff(x.ctypes.data, y.ctypes.data, x.size, last_dc); return y, float(np.float32(avg))

    @staticmethod
    def agc_ff(x, reference=0.2, attack_rate=0.01, decay_rate=0.0001, max_gain=65536.0, hang_time=200, attack_wait_time=0,
               gain_filter_alpha=0.999, last_gain=1.0):
        """one agc_ff call: (y, last gain)"""
        x = np.ascontiguousarray(x, np.float32); y = np.empty_like(x)
        g = lib().agc_ff(x.ctypes.data, y.ctypes.data, x.size, reference, attack_rate, decay_rate, max_gain, hang_time, attack_wait_time,
                         gain_filter_alpha, last_gain)
        return y, float(np.float32(g))

    @staticmethod
    def deemphasis_wfm_ff(x, tau, sample_rate, last=0.0, block=None):
        x = np.ascontiguousarray(x, np.float32); y = np.empty_like(x); block = block or max(x.size, 1)
        for s0 in range(0, x.size, block):
            n = min(block, x.size - s0)
            last = lib().deemphasis_wfm_ff(x[s0:].ctypes.data, y[s0:].ctypes.data, n, tau, sample_rate, last)
        return y, float(np.float32(last))

    @staticmethod
    def limit_ff(x, max_amplitude=1.0):
        x = np.ascontiguousarray(x, np.float32); y = np.empty_like(x)
        lib().limit_ff(x.ctypes.data, y.ctypes.data, x.size, max_amplitude); return y

    @staticmethod
    def deemphasis_nfm_ff(x, sample_rate):
        x = np.ascontiguousarray(x, np.float32); y = np.zeros_like(x)
        n = lib().deemphasis_nfm_ff(x.ctypes.data, y.ctypes.data, x.size, sample_rate)
        return y[:n].copy()

    @staticmethod
    def precalculate_window(size, window="HAMMING"):
        p = lib().precalculate_window(size, WINDOWS[window]); return np.ctypeslib.as_array(p, shape=(size,)).copy()

    @staticmethod
    def apply_window_c(x, window="HAMMING"):
        x = np.ascontiguousarray(x, np.complex64); y = np.empty_like(x)
        lib().apply_window_c(x.ctypes.data, y.ctypes.data, x.size, WINDOWS[window]); return y

    @staticmethod
    def logpower_cf(x, add_db=0.0):
        x = np.ascontiguousarray(x, np.complex64); y = np.empty(x.size, np.float32)
        lib().logpower_cf(x.ctypes.data, y.ctypes.data, x.size, add_db); return y

    @staticmethod
    def logaveragepower_cf(x, add_db, fft_size, avgnumber):
        x = np.ascontiguousarray(x, np.complex64); out = []
        adj = np.float32(np.float32(add_db) - np.float32(10.0 * np.log10(avgnumber)))
        for b in range(x.size // (fft_size * avgnumber)):
            acc = np.zeros(fft_size, np.float32)
            for n in range(avgnumber):
                seg = x[(b * avgnumber + n) * fft_size:(b * avgnumber + n + 1) * fft_size]
                lib().accumulate_power_cf(seg.ctypes.data, acc.ctypes.data, fft_size)
            y = np.empty(fft_size, np.float32); lib().log_ff(acc.ctypes.data, y.ctypes.data, fft_size, float(adj)); out.append(y)
        return np.concatenate(out) if out else np.zeros(0, np.float32)

    @staticmethod
    def shift_unroll_cc(x, rate, phase=0.0, size=1024):
        x = np.ascontiguousarray(x, np.complex64); y = np.empty_like(x)
        d = lib().shift_unroll_init(rate, size)
        for s0 in range(0, x.size, size):
            n = min(size, x.size - s0)
            phase = lib().shift_unroll_cc(x[s0:].ctypes.data, y[s0:].ctypes.data, n, C.byref(d), phase)
        return y, float(np.float32(phase))

    @staticmethod
    def encode_ima_adpcm_i16_u8(x, index=0, previous=0):
        x = np.ascontiguousarray(x, np.int16); y = np.empty(x.size // 2, np.uint8)
        st = lib().encode_ima_adpcm_i16_u8(x.ctypes.data, y.ctypes.data, x.size, _Ima(index, previous))
        return y, (st.index, st.previousValue)

    @staticmethod
    def shift_table_init(size=65536):
        d = lib().shift_table_init(size); t = np.ctypeslib.as_array(d.table, shape=(size,)).copy(); lib().shift_table_deinit(d); return t

    @staticmethod
    def shift_table_cc(x, rate, table, phase=0.0, chunk=None):
        x = np.ascontiguousarray(x, np.complex64); y = np.empty_like(x); table = np.ascontiguousarray(table, np.float32); chunk = chunk or max(x.size, 1)
        d = _Table(table.ctypes.data_as(C.POINTER(C.c_float)), table.size)
        for s0 in range(0, x.size, chunk):
            n = min(chunk, x.size - s0)
            phase = lib().shift_table_cc(x[s0:].ctypes.data, y[s0:].ctypes.data, n, rate, d, phase)
        return y, float(np.float32(phase))

    @staticmethod
    def shift_math_cc(x, rate, phase=0.0, chunk=None):
        x = np.ascontiguousarray(x, np.complex64); y = np.empty_like(x); chunk = chunk or max(x.size, 1)
        for s0 in range(0, x.size, chunk):
            n = min(chunk, x.size - s0)
            phase = lib().shift_math_cc(x[s0:].ctypes.data, y[s0:].ctypes.data, n, rate, phase)
        return y, float(np.float32(phase))

    @staticmethod
    def shift_addfast_cc(x, rate=None, phase=0.0, chunk=1024, steps=None):
        """calls of <= chunk samples like csdr.c:781-791; `steps` (9 floats: dsin[4], dcos[4], increment) overrides shift_addfast_init(rate);
        samples a call leaves untouched (n % 4) come back as 0"""
        x = np.ascontiguousarray(x, np.complex64); y = np.zeros_like(x); chunk = chunk or max(x.size, 1)
        d = lib().shift_addfast_init(rate) if steps is None else _AddFast((C.c_float * 4)(*steps[0:4]), (C.c_float * 4)(*steps[4:8]), float(steps[8]))
        for s0 in range(0, x.size, chunk):
            n = min(chunk, x.size - s0)
            phase = lib().shift_addfast_cc(x[s0:].ctypes.data, y[s0:].ctypes.data, n, C.byref(d), phase)
        return y, float(np.float32(phase))

    @staticmethod
    def dft(x, forward=True):
        x = np.ascontiguousarray(x, np.complex64).copy(); y = np.empty_like(x)
        pl = lib().make_fft_c2c(x.size, x.ctypes.data, y.ctypes.data, 1 if forward else 0, 0)
        lib().fft_execute(pl); lib().fft_destroy(pl); return y

    @staticmethod
    def rdft(x):
        """make_fft_r2c + fft_execute: x.size real points -> x.size // 2 + 1 bins"""
        x = np.ascontiguousarray(x, np.float32).copy(); y = np.empty(x.size // 2 + 1, np.complex64)
        pl = lib().make_fft_r2c(x.size, x.ctypes.data, y.ctypes.data, 0)
        lib().fft_execute(pl); lib().fft_destroy(pl); return y

    @staticmethod
    def bandpass_fir_fft_cc(x, lo, hi, bw, window="HAMMING"):
        """The CLI block loop of csdr.c:1833-1883 over the libcsdr-named entry points (complete blocks only)."""
        x = np.ascontiguousarray(x, np.complex64)
        T, N, isz, ov = bandpass_geometry(bw)
        taps = np.zeros(N, np.complex64); taps[:T] = firdes_bandpass_c(T, lo, hi, window)
        taps_fft = libcsdr.dft(taps)
        inp = np.zeros(N, np.complex64); spec = np.empty(N, np.complex64); ospec = np.empty(N, np.complex64)
        o = [np.zeros(N, np.complex64), np.zeros(N, np.complex64)]
        pf = lib().make_fft_c2c(N, inp.ctypes.data, spec.ctypes.data, 1, 0)
        pi = [lib().make_fft_c2c(N, ospec.ctypes.data, o[k].ctypes.data, 0, 0) for k in range(2)]
        out = []
        for b in range(x.size // isz):
            inp[:isz] = x[b * isz:(b + 1) * isz]
            cur, prev = (1, 0) if b & 1 else (0, 1)
            tail = o[prev][isz:]
            lib().apply_fir_fft_cc(pf, pi[cur], taps_fft.ctypes.data, tail.ctypes.data, ov)
            out.append(o[cur][:isz].copy())
        lib().fft_destroy(pf); [lib().fft_destroy(p) for p in pi]
        return np.concatenate(out) if out else np.zeros(0, np.complex64)

    @staticmethod
    def fastddc_inv(spectra, bw, decimation, shift, window="HAMMING"):
        """csdr.c:2335-2371 over the libcsdr-named entry points."""
        ddc = fastddc_init(bw, decimation, shift)
        hb = np.float32(0.5 / decimation); sh = np.float32(shift)
        taps = np.zeros(ddc.fft_size, np.complex64)
        taps[:ddc.taps_length] = firdes_bandpass_c(ddc.taps_length, float(-sh - hb), float(-sh + hb), window)
        tf = libcsdr.dft(taps); lib().fft_swap_sides(tf.ctypes.data, ddc.fft_size)
        st = _DShiftStatus(0, 0.0, 0); out = []
        for sp in spectra:
            sp = np.ascontiguousarray(sp, np.complex64).copy(); y = np.empty(ddc.post_input_size, np.complex64)
            st = lib().fastddc_inv_cc(sp.ctypes.data, y.ctypes.data, C.byref(ddc), None, tf.ctypes.data, st)
            out.append(y[:st.output_size].copy())
        return np.concatenate(out) if out else np.zeros(0, np.complex64)

    @staticmethod
    def fmdemod_quadri_cf(x, last=0j):
        x = np.ascontiguousarray(x, np.complex64); y = np.empty(x.size, np.float32)
        r = lib().fmdemod_quadri_cf(x.ctypes.data, y.ctypes.data, x.size, None, _CF(np.float32(last.real), np.float32(last.imag)))
        return y, complex(r.i, r.q)


# --------------------------------------------------------------------------------------------------
# K2 / K5 / K6 / K7 / K8 / K9 bank calls (torch CUDA tensors)
# --------------------------------------------------------------------------------------------------
def shift_addition_init(rate: float):
    d = lib().shift_addition_init(rate)
    return (d.sindelta, d.cosdelta, d.rate)


def fastddc_init(transition_bw: float, decimation: int, shift_rate: float) -> FastDDC:
    d = FastDDC()
    if lib().fastddc_init(C.byref(d), transition_bw, decimation, shift_rate):
        raise CsdrB200Error("fastddc_init: fft_size <= 2")
    return d


def _scratch(nbytes: int, device):
    import torch
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def shift_addition_bank_cc(x, rates, phases=None, chunk: int = 1024, out=None):
    """x: [N] (one shared wideband stream) or [C, N] complex64; rates: C floats.  Returns (y [C,N], new phases [C] tensor)."""
    import torch
    rates = np.atleast_1d(np.asarray(rates, np.float32))
    ch = rates.size
    shared = (x.dim() == 1) if x.dtype == torch.complex64 else (x.dim() == 2)
    xr, ptr, stride, xc, n = _as_cf32_rows(x)
    if shared:
        stride = 0
    else:
        assert xc == ch
    params = np.array([shift_addition_init(float(r)) for r in rates], np.float32)           # host: bit-exact deltas
    d_params = torch.from_numpy(params).to(xr.device)
    d_phase = torch.zeros(ch, dtype=torch.float32, device=xr.device) if phases is None else phases.clone()
    if out is None:
        out = torch.empty((ch, n), dtype=torch.complex64, device=xr.device)
    sb = lib().csdrb_shift_addition_bank_scratch_bytes(ch, n, chunk)
    scratch = _scratch(sb, xr.device)
    _check(lib().csdrb_shift_addition_bank_cc(ptr, stride, out.data_ptr(), out.stride(0), ch, n, d_params.data_ptr(), d_phase.data_ptr(), chunk,
                                              scratch.data_ptr(), scratch.numel(), _stream()), "shift_addition_bank_cc")
    return out, d_phase


def shift_addition_bank_fc(x, rates, phases=None, chunk: int = 1024, out=None):
    """x: [N] (one shared real wideband stream) or [C, N] float32 CUDA tensor; rates: C floats.  Returns (y [C, N] complex64, new phases [C]):
    shift_addition_fc called once per `chunk` samples, bit for bit."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.dim() in (1, 2) and x.stride(-1) == 1
    rates = np.atleast_1d(np.asarray(rates, np.float32))
    ch = rates.size
    n = x.shape[-1]
    if x.dim() == 1:
        stride = 0
    else:
        assert x.shape[0] == ch
        stride = x.stride(0)
    d_params = torch.from_numpy(np.array([shift_addition_init(float(r)) for r in rates], np.float32)).to(x.device)
    d_phase = torch.zeros(ch, dtype=torch.float32, device=x.device) if phases is None else phases.clone()
    if out is None:
        out = torch.empty((ch, n), dtype=torch.complex64, device=x.device)
    scratch = _scratch(lib().csdrb_shift_addition_bank_scratch_bytes(ch, n, chunk), x.device)
    _check(lib().csdrb_shift_addition_bank_fc(x.data_ptr(), stride, out.data_ptr(), out.stride(0), ch, n, d_params.data_ptr(), d_phase.data_ptr(), chunk,
                                              scratch.data_ptr(), scratch.numel(), _stream()), "shift_addition_bank_fc")
    return out, d_phase


def encode_ima_adpcm_rows_i16_u8(x, state=None):
    """x [R, N] int16 -> (bytes [R, N/2] uint8, state [R, 2] int32 = index, previousValue carried per row)"""
    import torch
    assert x.dtype == torch.int16 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    rows, n = x.shape
    out = torch.empty((rows, n // 2), dtype=torch.uint8, device=x.device)
    state = torch.zeros((rows, 2), dtype=torch.int32, device=x.device) if state is None else state
    _check(lib().csdrb_encode_ima_adpcm_rows_i16_u8(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), rows, n, state.data_ptr(), _stream()), "encode_ima_adpcm_rows")
    return out, state


def compress_fft_adpcm_rows_f_u8(db):
    """db [R, fft_size] float32 (dB) -> [R, (fft_size + 10) / 2] uint8: one fresh ADPCM encoder per waterfall line (csdr.c:1745-1767)"""
    import torch
    assert db.dtype == torch.float32 and db.is_cuda and db.dim() == 2 and db.stride(1) == 1
    rows, n = db.shape
    out = torch.empty((rows, (n + 10) // 2), dtype=torch.uint8, device=db.device)
    _check(lib().csdrb_compress_fft_adpcm_rows_f_u8(db.data_ptr(), db.stride(0), out.data_ptr(), out.stride(0), rows, n, _stream()), "compress_fft_adpcm_rows")
    return out


def shift_math_bank_cc(x, rates, phases=None, out=None):
    """x: [N] (one shared wideband stream) or [C, N] complex64; returns (y [C, N], new phases [C])."""
    import torch
    rates = np.atleast_1d(np.asarray(rates, np.float32)); ch = rates.size
    shared = (x.dim() == 1) if x.dtype == torch.complex64 else (x.dim() == 2)
    xr, ptr, stride, xc, n = _as_cf32_rows(x)
    if shared:
        stride = 0
    else:
        assert xc == ch
    d_rates = torch.from_numpy(rates).to(xr.device)
    d_phase = torch.zeros(ch, dtype=torch.float32, device=xr.device) if phases is None else phases.clone()
    if out is None:
        out = torch.empty((ch, n), dtype=torch.complex64, device=xr.device)
    scratch = _scratch(lib().csdrb_shift_math_bank_scratch_bytes(ch, n), xr.device)
    _check(lib().csdrb_shift_math_bank_cc(ptr, stride, out.data_ptr(), out.stride(0), ch, n, d_rates.data_ptr(), d_phase.data_ptr(),
                                          scratch.data_ptr(), scratch.numel(), _stream()), "shift_math_bank_cc")
    return out, d_phase


def shift_table_bank_cc(x, rates, table, phases=None, out=None):
    """x: [N] (one shared wideband stream) or [C, N] complex64; table: quarter-wave sine table (numpy or CUDA tensor); returns (y [C, N], new phases [C])."""
    import torch
    rates = np.atleast_1d(np.asarray(rates, np.float32)); ch = rates.size
    shared = (x.dim() == 1) if x.dtype == torch.complex64 else (x.dim() == 2)
    xr, ptr, stride, xc, n = _as_cf32_rows(x)
    if shared:
        stride = 0
    else:
        assert xc == ch
    d_table = table if isinstance(table, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(table, np.float32)).to(xr.device)
    d_rates = torch.from_numpy(rates).to(xr.device)
    d_phase = torch.zeros(ch, dtype=torch.float32, device=xr.device) if phases is None else phases.clone()
    if out is None:
        out = torch.empty((ch, n), dtype=torch.complex64, device=xr.device)
    scratch = _scratch(lib().csdrb_shift_math_bank_scratch_bytes(ch, n), xr.device)
    _check(lib().csdrb_shift_table_bank_cc(ptr, stride, out.data_ptr(), out.stride(0), ch, n, d_rates.data_ptr(), d_phase.data_ptr(), d_table.data_ptr(),
                                           d_table.numel(), scratch.data_ptr(), scratch.numel(), _stream()), "shift_table_bank_cc")
    return out, d_phase


def shift_addfast_init(rate: float) -> np.ndarray:
    """9 floats: dsin[4], dcos[4], phase_increment (host; shift_addfast_data_t member order)"""
    d = lib().shift_addfast_init(rate)
    return np.array(list(d.dsin) + list(d.dcos) + [d.phase_increment], np.float32)


def shift_addfast_bank_cc(x, rates=None, phases=None, chunk: int = 1024, out=None, steps=None):
    """x: [N] (one shared wideband stream) or [C, N] complex64; one reference call per `chunk` samples.  `steps` [C, 9] overrides the
    per-channel shift_addfast_init(rate).  Samples a call does not touch (its n % 4 tail) are 0.  Returns (y [C, N], new phases [C])."""
    import torch
    params = np.stack([shift_addfast_init(float(r)) for r in np.atleast_1d(np.asarray(rates, np.float32))]) if steps is None \
        else np.ascontiguousarray(steps, np.float32).reshape(-1, 9)
    ch = params.shape[0]
    shared = (x.dim() == 1) if x.dtype == torch.complex64 else (x.dim() == 2)
    xr, ptr, stride, xc, n = _as_cf32_rows(x)
    if shared:
        stride = 0
    else:
        assert xc == ch
    d_params = torch.from_numpy(params).to(xr.device)
    d_phase = torch.zeros(ch, dtype=torch.float32, device=xr.device) if phases is None else phases.clone()
    if out is None:
        out = torch.zeros((ch, n), dtype=torch.complex64, device=xr.device)
    scratch = _scratch(lib().csdrb_shift_addition_bank_scratch_bytes(ch, n, chunk), xr.device)
    _check(lib().csdrb_shift_addfast_bank_cc(ptr, stride, out.data_ptr(), out.stride(0), ch, n, d_params.data_ptr(), d_phase.data_ptr(), chunk,
                                             scratch.data_ptr(), scratch.numel(), _stream()), "shift_addfast_bank_cc")
    return out, d_phase


def fractional_decimator_bank_ff(x, rate: float, num_poly_points: int = 12, taps=None, where=None):
    """x [C, N] float32 -> (y [C, cap] float32, state tensor [C,3] int32-view (where bits, input_processed, output_size))."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    cap = int(n / max(rate, 1.0)) + 8
    out = torch.empty((ch, cap), dtype=torch.float32, device=x.device)
    state = torch.zeros((ch, 3), dtype=torch.int32, device=x.device)
    w0 = np.float32(num_poly_points // 2 - 1 if where is None else 0)            # where = -xifirst at init (libcsdr.c:736)
    if where is None:
        state[:, 0] = int(np.array([w0], np.float32).view(np.int32)[0])
    else:
        state[:, 0] = torch.as_tensor(np.asarray(where, np.float32).view(np.int32), device=x.device)
    d_taps = torch.from_numpy(np.ascontiguousarray(taps, np.float32)).to(x.device) if taps is not None else None
    sb = lib().csdrb_fractional_decimator_bank_scratch_bytes(ch, n, rate)
    scratch = _scratch(sb, x.device)
    _check(lib().csdrb_fractional_decimator_bank_ff(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, rate, num_poly_points,
                                                    d_taps.data_ptr() if d_taps is not None else None, d_taps.numel() if d_taps is not None else 0,
                                                    state.data_ptr(), scratch.data_ptr(), scratch.numel(), _stream()), "fractional_decimator_bank_ff")
    return out, state


def rational_resampler_bank_ff(x, interpolation: int, decimation: int, taps, last_taps_delay: int = 0, out=None):
    """x [C, N] float32 CUDA tensor -> (y [C, n_out], (input_processed, output_size, last_taps_delay)): every row through rational_resampler_ff
    with the shared host ``taps`` and last_taps_delay.  The state is computed on the host; nothing waits for the device."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    taps = np.ascontiguousarray(taps, np.float32)
    ch, n = x.shape
    if out is None:
        out = torch.empty((ch, max(n * interpolation // decimation, 1)), dtype=torch.float32, device=x.device)
    assert out.dtype == torch.float32 and out.shape[0] == ch and out.stride(1) == 1
    st = _Resampler()
    rc = _check(lib().csdrb_rational_resampler_bank_ff(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, interpolation, decimation,
                                                       _fp(taps), taps.size, last_taps_delay, C.byref(st), _stream()), "rational_resampler_bank_ff")
    assert out.shape[1] >= rc
    return out[:, :rc], (st.input_processed, st.output_size, st.last_taps_delay)


def fastagc_bank_ff(x, block: int = 1024, reference: float = 1.0, state=None, hist=None):
    """x [C, nblocks*block] float32 -> y same shape (two blocks of latency); returns (y, state [C,3] f32, hist [C,2,block])."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    nblocks = n // block
    out = torch.empty((ch, nblocks * block), dtype=torch.float32, device=x.device)
    state = torch.zeros((ch, 3), dtype=torch.float32, device=x.device) if state is None else state
    hist = torch.zeros((ch, 2, block), dtype=torch.float32, device=x.device) if hist is None else hist
    scratch = _scratch(lib().csdrb_fastagc_bank_scratch_bytes(ch, nblocks), x.device)
    _check(lib().csdrb_fastagc_bank_ff(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, block, nblocks, reference,
                                       state.data_ptr(), hist.data_ptr(), scratch.data_ptr(), scratch.numel(), _stream()), "fastagc_bank_ff")
    return out, state, hist


def fastagc_bank_f_s16(x, block: int = 1024, reference: float = 1.0, state=None, hist=None):
    """fastagc_ff | convert_f_s16 in one pass: x [C, nblocks*block] float32 -> int16 of the same shape; returns (y, state, hist)."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    nblocks = n // block
    out = torch.empty((ch, nblocks * block), dtype=torch.int16, device=x.device)
    state = torch.zeros((ch, 3), dtype=torch.float32, device=x.device) if state is None else state
    hist = torch.zeros((ch, 2, block), dtype=torch.float32, device=x.device) if hist is None else hist
    scratch = _scratch(lib().csdrb_fastagc_bank_scratch_bytes(ch, nblocks), x.device)
    _check(lib().csdrb_fastagc_bank_f_s16(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, block, nblocks, reference,
                                          state.data_ptr(), hist.data_ptr(), scratch.data_ptr(), scratch.numel(), _stream()), "fastagc_bank_f_s16")
    return out, state, hist


def amdemod_cf(x, out=None):
    """|x| of a complex64 CUDA tensor (amdemod_cf, correctly rounded sqrt(i*i + q*q)) -> float32 of the same shape."""
    import torch
    assert x.dtype == torch.complex64 and x.is_cuda and x.is_contiguous()
    out = torch.empty(x.shape, dtype=torch.float32, device=x.device) if out is None else out
    _check(lib().csdrb_amdemod_cf(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "amdemod_cf")
    return out


def fastdcblock_bank_ff(x, block: int = 1024, last_dc=None):
    """[amdemod_cf |] fastdcblock_ff over the whole blocks of each row: x [C, N] float32 (or complex64: its magnitude is taken first)
    -> (y [C, (N // block) * block] float32, last_dc [C] float32).  The N % block samples left over are the caller's to carry."""
    import torch
    assert x.dtype in (torch.float32, torch.complex64) and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    nblocks = n // block
    out = torch.empty((ch, nblocks * block), dtype=torch.float32, device=x.device)
    last_dc = torch.zeros(ch, dtype=torch.float32, device=x.device) if last_dc is None else last_dc
    _check(lib().csdrb_fastdcblock_bank_ff(x.data_ptr(), x.stride(0), int(x.dtype == torch.complex64), out.data_ptr(), out.stride(0), ch, block,
                                           nblocks, last_dc.data_ptr(), _stream()), "fastdcblock_bank_ff")
    return out, last_dc


def agc_state(channels: int, device="cuda"):
    """csdrb_agc_state_t [C] at stream start (gain 1, offset 0), as a [C, 5] int32 tensor"""
    import torch
    st = torch.zeros((channels, 5), dtype=torch.int32)
    st[:, 0] = int(np.array([1.0], np.float32).view(np.int32)[0])
    return st.to(device)


def agc_bank_ff(x, params: AgcParams | None = None, state=None, limit_max: float = 0.0, s16: bool = False):
    """[realpart_cf |] agc_ff [| limit_ff limit_max] [| convert_f_s16] per row: x [C, N] float32 (or complex64: real part)
    -> (y [C, N] float32 or int16, state).  Cutting a stream into calls of any sizes gives the bits of one call."""
    import torch
    assert x.dtype in (torch.float32, torch.complex64) and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    params = AgcParams() if params is None else params
    state = agc_state(ch, x.device) if state is None else state
    out = torch.empty((ch, n), dtype=torch.int16 if s16 else torch.float32, device=x.device)
    _check(lib().csdrb_agc_bank_ff(x.data_ptr(), x.stride(0), int(x.dtype == torch.complex64), out.data_ptr(), out.stride(0), int(s16), ch, n,
                                   C.byref(params), state.data_ptr(), limit_max, _stream()), "agc_bank_ff")
    return out, state


def simple_agc_bank_cc(x, rate: float = 0.001, reference: float = 1.0, max_gain: float = 65535.0, gain=None):
    """simple_agc_cc per row: x [C, N] complex64 -> (y [C, N], gain [C] float32, carried between calls; 1.0 at stream start)"""
    import torch
    assert x.dtype == torch.complex64 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    gain = torch.ones(ch, dtype=torch.float32, device=x.device) if gain is None else gain
    out = torch.empty((ch, n), dtype=torch.complex64, device=x.device)
    _check(lib().csdrb_simple_agc_bank_cc(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, rate, reference, max_gain, gain.data_ptr(),
                                          _stream()), "simple_agc_bank_cc")
    return out, gain


def timing_recovery_bank_cc(x, algorithm: int, decimation: int, use_q: bool = True, loop_gain: float = 0.5, max_error: float = 2.0,
                            start=None, size=None, state=None, outputs: str = "symbols"):
    """one timing_recovery_cc call per row over x[c, start[c]:start[c] + size[c]] (start 0 and size N by default): returns
    (symbols [C, cap] complex64, error [C, cap] float32 or None, indexes [C, cap] int32 or None, state [C, 3] int32 =
    {last_correction_offset, input_processed, output_size}).  Pass `state` back to continue a stream; its counts are data-dependent."""
    import torch
    assert x.dtype == torch.complex64 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    start = torch.zeros(ch, dtype=torch.int32, device=x.device) if start is None else start
    size = torch.full((ch,), n, dtype=torch.int32, device=x.device) if size is None else size
    state = torch.zeros((ch, 3), dtype=torch.int32, device=x.device) if state is None else state
    # room for every symbol one call can make: n/(decimation/2) + 1 while |loop_gain*max_error| <= 1, n above (a symbol may not advance)
    cap = (n // (decimation // 2) + 1 if abs(loop_gain * max_error) <= 1 else max(n, 1)) if decimation >= 2 else 1
    out = torch.empty((ch, cap), dtype=torch.complex64, device=x.device)
    err = torch.empty((ch, cap), dtype=torch.float32, device=x.device)
    idx = torch.empty((ch, cap), dtype=torch.int32, device=x.device)
    p = TimingRecoveryParams(algorithm, decimation, int(use_q), loop_gain, max_error)
    _check(lib().csdrb_timing_recovery_bank_cc(x.data_ptr(), x.stride(0), start.data_ptr(), size.data_ptr(), n, out.data_ptr(), cap, err.data_ptr(),
                                               idx.data_ptr(), ch, C.byref(p), state.data_ptr(), _stream()), "timing_recovery_bank_cc")
    return out, err, idx, state


def dbpsk_decoder_bank_c_u8(x, lengths=None, last=None):
    """dbpsk_decoder_c_u8 per row: x [C, N] complex64 (row c holds lengths[c] samples) -> (bits [C, N] uint8, last sample [C] complex64)"""
    import torch
    assert x.dtype == torch.complex64 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    last = torch.zeros(ch, dtype=torch.complex64, device=x.device) if last is None else last
    new_last = torch.empty_like(last)
    out = torch.zeros((ch, n), dtype=torch.uint8, device=x.device)
    _check(lib().csdrb_dbpsk_decoder_bank_c_u8(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n,
                                               lengths.data_ptr() if lengths is not None else None, last.data_ptr(), new_last.data_ptr(), _stream()),
           "dbpsk_decoder_bank_c_u8")
    return out, new_last


def psk31_varicode_decoder_bank_u8_u8(bits, lengths=None, hist=None):
    """the varicode decoder per row: bits [C, N] uint8 (row c holds lengths[c] bits) -> (chars [C, N] uint8, count [C] int32, hist [C] int64,
    the decoder's shift register carried between calls)"""
    import torch
    assert bits.dtype == torch.uint8 and bits.is_cuda and bits.dim() == 2 and bits.stride(1) == 1
    ch, n = bits.shape
    hist = torch.zeros(ch, dtype=torch.int64, device=bits.device) if hist is None else hist
    out = torch.zeros((ch, max(n, 1)), dtype=torch.uint8, device=bits.device)
    count = torch.zeros(ch, dtype=torch.int32, device=bits.device)
    _check(lib().csdrb_psk31_varicode_decoder_bank_u8_u8(bits.data_ptr(), bits.stride(0), out.data_ptr(), out.stride(0), ch, n,
                                                         lengths.data_ptr() if lengths is not None else None, hist.data_ptr(), count.data_ptr(),
                                                         _stream()), "psk31_varicode_decoder_bank_u8_u8")
    return out, count, hist


def serial_line_decoder_bank_f_u8(x, samples_per_bits: float, databits: int = 8, stopbits: float = 1.0, bit_sampling_width_ratio: float = 0.4,
                                  bufsize: int | None = None, start=None, end: int | None = None):
    """serial_line_decoder_f_u8 per row, framed like the CLI: while at least bufsize samples of x[c, start[c]:end] remain, one call on exactly
    bufsize of them (bufsize and end default to N: one call per row).  x [C, N] float32 -> (characters [C, cap] uint8, count [C] int32,
    start [C] int32 advanced past what the calls consumed, stuck [C] int32: 1 where a call consumed nothing)"""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    end = n if end is None else end
    bufsize = n if bufsize is None else bufsize
    start = torch.zeros(ch, dtype=torch.int32, device=x.device) if start is None else start
    p = SerialLineParams(samples_per_bits, databits, stopbits, bit_sampling_width_ratio)
    span = np.float32(samples_per_bits) * (np.float32(1 + databits) + np.float32(stopbits))
    cap = end // max(int(span), 1) + 1
    out = torch.zeros((ch, cap), dtype=torch.uint8, device=x.device)
    count = torch.zeros(ch, dtype=torch.int32, device=x.device)
    stuck = torch.zeros(ch, dtype=torch.int32, device=x.device)
    _check(lib().csdrb_serial_line_decoder_bank_f_u8(x.data_ptr(), x.stride(0), end, start.data_ptr(), out.data_ptr(), cap, count.data_ptr(),
                                                     stuck.data_ptr(), ch, C.byref(p), bufsize, _stream()), "serial_line_decoder_bank_f_u8")
    return out, count, start, stuck


def rtty_baudot2ascii_bank_u8_u8(codes, lengths=None, fig_mode=None):
    """rtty_baudot_decoder_lookup per row: codes [C, N] uint8 (row c holds lengths[c] codes) -> (chars [C, N] uint8, count [C] int32,
    fig_mode [C] uint8, the letters/figures mode carried between calls)"""
    import torch
    assert codes.dtype == torch.uint8 and codes.is_cuda and codes.dim() == 2 and codes.stride(1) == 1
    ch, n = codes.shape
    fig_mode = torch.zeros(ch, dtype=torch.uint8, device=codes.device) if fig_mode is None else fig_mode
    out = torch.zeros((ch, max(n, 1)), dtype=torch.uint8, device=codes.device)
    count = torch.zeros(ch, dtype=torch.int32, device=codes.device)
    _check(lib().csdrb_rtty_baudot2ascii_bank_u8_u8(codes.data_ptr(), codes.stride(0), out.data_ptr(), out.stride(0), ch, n,
                                                    lengths.data_ptr() if lengths is not None else None, fig_mode.data_ptr(), count.data_ptr(),
                                                    _stream()), "rtty_baudot2ascii_bank_u8_u8")
    return out, count, fig_mode



def firdes_peak_c(rate: float, length: int, window: str = "HAMMING") -> np.ndarray:
    """firdes_add_peak_c(taps, length, rate, window, 0, 1) (libcsdr.c:2219-2258): a windowed complex tone at -rate cycles per sample, scaled so
    that its magnitudes sum to 1 -- as the reference's build computes it"""
    t = np.zeros(max(length, 1), np.complex64)
    lib().firdes_add_peak_c(t.ctypes.data, length, rate, WINDOWS[window], 0, 1)
    return t[:length]


def _tone_rows(x):
    import torch
    assert x.dtype == torch.complex64 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    return x.shape


def apply_fir_bank_cc(x, taps):
    """apply_fir_cc per row (libcsdr.c:2261-2273), bit for bit with the reference build: x [C, N] complex64 CUDA, taps [L] complex64 (numpy or
    CUDA, 2 <= L <= 4096, shared by all rows) -> [C, N - L + 1] complex64, the valid convolution"""
    import torch
    ch, n = _tone_rows(x)
    t = torch.as_tensor(np.asarray(taps, np.complex64) if not torch.is_tensor(taps) else taps, device=x.device).contiguous()
    out = torch.empty((ch, max(n - t.numel() + 1, 1)), dtype=torch.complex64, device=x.device)
    m = _check(lib().csdrb_apply_fir_bank_cc(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, t.data_ptr(), t.numel(), _stream()),
               "apply_fir_bank_cc")
    return out[:, :m]


def fir_interpolate_bank(x, interpolation: int, taps):
    """fir_interpolate_cc per row (libcsdr.c:579-602): x [C, N] complex64 CUDA, taps [T] float32 (numpy or CUDA, shared by all rows) ->
    [C, I * (N - ceil((T-1)/I))] complex64, one reference call per row (tap 0 unused, as there).  A stream keeps the inputs a call did not
    consume, N minus the outputs / I, in front of its next call."""
    import torch
    ch, n = _tone_rows(x)
    t = torch.as_tensor(np.asarray(taps, np.float32) if not torch.is_tensor(taps) else taps, device=x.device)
    assert not t.is_complex(), "fir_interpolate_bank: real taps"
    t = t.to(torch.float32).contiguous()
    groups = max(n - (t.numel() - 1 + interpolation - 1) // interpolation, 0)
    out = torch.empty((ch, max(groups * interpolation, 1)), dtype=torch.complex64, device=x.device)
    if ch == 0 or groups == 0:
        return out[:, :0]
    m = _check(lib().csdrb_fir_interpolate_bank_cc(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, interpolation, t.data_ptr(),
                                                   t.numel(), _stream()), "fir_interpolate_bank")
    return out[:, :m]


def fmmod_bank(x, phase=None):
    """fmmod_fc per row (libcsdr.c:1180-1192): x [C, N] float32 CUDA -> [C, N] complex64 (cos, sin) of the phase advanced by x*PI per sample.
    phase: a [C] float32 CUDA tensor carried between calls (zeros at stream start), updated in place; None starts from 0."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    if phase is None:
        phase = torch.zeros(ch, dtype=torch.float32, device=x.device)
    assert phase.dtype == torch.float32 and phase.is_cuda and phase.numel() == ch and phase.is_contiguous()
    out = torch.empty((ch, max(n, 1)), dtype=torch.complex64, device=x.device)
    if ch == 0 or n == 0:
        return out[:, :0]
    _check(lib().csdrb_fmmod_bank_fc(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, phase.data_ptr(), _stream()), "fmmod_bank")
    return out[:, :n]


def _mod_rows(x, dtype, what):
    import torch
    assert x.dtype == dtype and x.is_cuda and x.dim() == 2 and x.stride(1) == 1, f"{what}: [C, N] {dtype} CUDA rows"
    return x.shape


def gain_bank(x, gain: float, out=None):
    """gain_ff per row (libcsdr.c:1139): x [C, N] float32 CUDA -> [C, N] float32 gain*x, bit for bit the reference build.  out may be x (in place)."""
    import torch
    ch, n = _mod_rows(x, torch.float32, "gain_bank")
    out = torch.empty((ch, n), dtype=torch.float32, device=x.device) if out is None else out
    _check(lib().csdrb_gain_bank_ff(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, gain, _stream()), "gain_bank")
    return out


def dsb_bank(x, q_value: float = 0.0):
    """the dsb_fc command per row (csdr.c:2084-2102): x [C, N] float32 CUDA -> [C, N] complex64 (x, q_value)"""
    import torch
    ch, n = _mod_rows(x, torch.float32, "dsb_bank")
    out = torch.empty((ch, n), dtype=torch.complex64, device=x.device)
    _check(lib().csdrb_dsb_bank_fc(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, q_value, _stream()), "dsb_bank")
    return out


def add_dcoffset_bank(x, out=None):
    """add_dcoffset_cc per row (libcsdr.c:1174) as the reference build runs it: x [C, N] complex64 CUDA -> [C, N] complex64
    ((i + 1)*0.5, q*0.5) in float, bit for bit.  out may be x (in place)."""
    import torch
    ch, n = _mod_rows(x, torch.complex64, "add_dcoffset_bank")
    out = torch.empty((ch, n), dtype=torch.complex64, device=x.device) if out is None else out
    _check(lib().csdrb_add_dcoffset_bank_cc(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, _stream()), "add_dcoffset_bank")
    return out


def fixed_amplitude_bank(x, new_amplitude: float, out=None):
    """fixed_amplitude_cc per row (libcsdr.c:1194): x [C, N] complex64 CUDA -> [C, N] complex64 x*A/|x| (0 where |x| is not positive), the
    source's sqrt and division correctly rounded (DESIGN.md section 7).  out may be x (in place)."""
    import torch
    ch, n = _mod_rows(x, torch.complex64, "fixed_amplitude_bank")
    out = torch.empty((ch, n), dtype=torch.complex64, device=x.device) if out is None else out
    _check(lib().csdrb_fixed_amplitude_bank_cc(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, new_amplitude, _stream()),
           "fixed_amplitude_bank")
    return out


def _u8_rows(x):
    import torch
    assert x.dtype == torch.uint8 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    return x.shape


def psk31_varicode_encoder_bank_u8_u8(text, lengths=None, output_max_size=None):
    """psk31_varicode_encoder_u8_u8 per row (libcsdr.c:1551-1575): text [C, N] uint8 (row c holds lengths[c] bytes) -> (bits [C, M] uint8, one
    byte 0/1 per bit, input_processed [C] int32, output_size [C] int32).  M = output_max_size, by default 12*N: every character fits (the longest
    code has 10 bits, then two 0 bits).  output_size can be passed on as the next bank's lengths."""
    import torch
    ch, n = _u8_rows(text)
    m = 12 * n if output_max_size is None else output_max_size
    out = torch.zeros((ch, max(m, 1)), dtype=torch.uint8, device=text.device)
    processed = torch.zeros(ch, dtype=torch.int32, device=text.device)
    size = torch.zeros(ch, dtype=torch.int32, device=text.device)
    _check(lib().csdrb_psk31_varicode_encoder_bank_u8_u8(text.data_ptr(), text.stride(0), out.data_ptr(), out.stride(0), ch, n,
                                                         lengths.data_ptr() if lengths is not None else None, m, processed.data_ptr(),
                                                         size.data_ptr(), _stream()), "psk31_varicode_encoder_bank_u8_u8")
    return out[:, :max(m, 0)], processed, size


def differential_codec_bank_u8_u8(x, encode: bool, lengths=None, state=None):
    """differential_codec per row (libcsdr.c:1828-1843): x [C, N] uint8 -> (out [C, N] uint8, state [C] uint8).  state: the codec state
    carried between calls (zeros at stream start), a [C] uint8 CUDA tensor updated in place; None starts from 0."""
    import torch
    ch, n = _u8_rows(x)
    state = torch.zeros(ch, dtype=torch.uint8, device=x.device) if state is None else state
    assert state.dtype == torch.uint8 and state.is_cuda and state.numel() == ch and state.is_contiguous()
    out = torch.zeros((ch, max(n, 1)), dtype=torch.uint8, device=x.device)
    _check(lib().csdrb_differential_codec_bank_u8_u8(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n,
                                                     lengths.data_ptr() if lengths is not None else None, int(bool(encode)), state.data_ptr(),
                                                     _stream()), "differential_codec_bank_u8_u8")
    return out[:, :n], state


def psk_modulator_bank_u8_c(x, n_psk: int, lengths=None):
    """psk_modulator_u8_c per row (libcsdr.c:1772-1782): symbols x [C, N] uint8 -> [C, N] complex64, (cos, sin)(b * 2pi/n_psk), 1 <= n_psk <= 256"""
    import torch
    ch, n = _u8_rows(x)
    out = torch.zeros((ch, max(n, 1)), dtype=torch.complex64, device=x.device)
    _check(lib().csdrb_psk_modulator_bank_u8_c(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n,
                                               lengths.data_ptr() if lengths is not None else None, n_psk, _stream()), "psk_modulator_bank_u8_c")
    return out[:, :n]


def psk31_interpolate_sine_bank_cc(x, interpolation: int, lengths=None, last=None):
    """psk31_interpolate_sine_cc per row (libcsdr.c:1793-1808): x [C, N] complex64 -> ([C, N*interpolation] complex64, last [C] complex64).
    last: the previous input of each row carried between calls (zeros at stream start), a [C] complex64 CUDA tensor updated in place."""
    import torch
    assert x.dtype == torch.complex64 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    last = torch.zeros(ch, dtype=torch.complex64, device=x.device) if last is None else last
    assert last.dtype == torch.complex64 and last.is_cuda and last.numel() == ch and last.is_contiguous()
    m = n * max(interpolation, 0)
    out = torch.zeros((ch, max(m, 1)), dtype=torch.complex64, device=x.device)
    _check(lib().csdrb_psk31_interpolate_sine_bank_cc(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n,
                                                      lengths.data_ptr() if lengths is not None else None, interpolation, last.data_ptr(),
                                                      _stream()), "psk31_interpolate_sine_bank_cc")
    return out[:, :m], last


def _synth_rows(x):
    import torch
    assert x.dtype == torch.complex64 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1, "synthesis bank: [C, n] complex64 CUDA rows"
    return x.shape


def _real_taps(taps, what):
    t = np.asarray(taps)
    if np.iscomplexobj(t):
        raise TypeError(f"{what}: real taps")
    return np.ascontiguousarray(t, np.float32)


def synth_bank(x, rates, interpolation: int, taps, phases=None, chunk: int = 1024, offset: int = 0):
    """Synthesis bank (csdrb_synth_bank_cc): x [C, n] complex64 CUDA baseband rows -> (y [G*I] complex64, phases [C]), y the sum over the
    channels of shift_addition_cc(fir_interpolate_cc(x_c, I, taps), rate_c) in a fixed pairwise tree over the channel index, G = n - ceil((T-1)/I)
    (or 0).  shift_addition_cc runs once per `chunk` wideband samples counted on the absolute stream: output 0 lies `offset` samples into a chunk,
    phases[c] is the phase at the start of that chunk (zeros when None) and the returned one the phase at the start of the chunk holding output G*I."""
    import torch
    ch, n = _synth_rows(x)
    rates = np.atleast_1d(np.asarray(rates, np.float32))
    assert rates.size == ch, "synth_bank: one rate per row"
    t = torch.from_numpy(_real_taps(taps.cpu().numpy() if torch.is_tensor(taps) else taps, "synth_bank")).to(x.device)
    params = torch.from_numpy(np.array([shift_addition_init(float(r)) for r in rates], np.float32)).to(x.device)
    d_phase = torch.zeros(ch, dtype=torch.float32, device=x.device) if phases is None else phases.to(torch.float32).clone()
    groups = max(n - (t.numel() - 1 + interpolation - 1) // interpolation, 0) if interpolation >= 1 else 0
    out = torch.empty(max(groups * interpolation, 1), dtype=torch.complex64, device=x.device)
    scratch = _scratch(lib().csdrb_synth_bank_scratch_bytes(ch, n, interpolation, t.numel(), chunk, offset), x.device)
    m = _check(lib().csdrb_synth_bank_cc(x.data_ptr(), x.stride(0), ch, n, interpolation, t.data_ptr(), t.numel(), params.data_ptr(), d_phase.data_ptr(),
                                         chunk, offset, out.data_ptr(), scratch.data_ptr(), scratch.numel(), _stream()), "synth_bank")
    return out[:m], d_phase


class SynthBank:
    """Streaming synthesis bank (csdrb_synth_bank_*): the rates, taps, phases and the place inside the current NCO chunk live in the object.
    process(x) takes [C, n] complex64 CUDA rows and returns the G*I wideband outputs; it consumes G = n - ceil((T-1)/I) inputs per row, and the
    caller presents the last n - G again at the front of the next block (fir_interpolate_cc's block contract)."""

    def __init__(self, rates, interpolation: int, taps, chunk: int = 1024):
        self.rates = np.ascontiguousarray(np.atleast_1d(rates), np.float32)
        self.taps = _real_taps(taps, "SynthBank")
        self.interpolation, self.channels = interpolation, self.rates.size
        self.h = lib().csdrb_synth_bank_create(self.channels, _fp(self.rates), interpolation, _fp(self.taps), self.taps.size, chunk)
        if not self.h:
            raise CsdrB200Error(f"csdrb_synth_bank_create: {lib().csdrb_last_error().decode()}")

    def process(self, x):
        import torch
        ch, n = _synth_rows(x)
        assert ch == self.channels, "SynthBank.process: one row per channel"
        groups = max(n - (self.taps.size - 1 + self.interpolation - 1) // self.interpolation, 0)
        out = torch.empty(max(groups * self.interpolation, 1), dtype=torch.complex64, device=x.device)
        m = _check(lib().csdrb_synth_bank_process(self.h, x.data_ptr(), x.stride(0), n, out.data_ptr(), _stream()), "synth_bank_process")
        return out[:m]

    def close(self):
        if getattr(self, "h", None):
            lib().csdrb_synth_bank_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def bfsk_demod_bank_cf(x, spacing: float, filter_length: int):
    """bfsk_demod_cf per row (libcsdr.c:2335-2351) with the CLI's taps (csdr.c:3283-3286): Hamming peaks at +spacing/2 (mark) and
    -spacing/2 (space), spacing in cycles per sample.  x [C, N] complex64 CUDA -> [C, N - L + 1] float32, |mark|^2 - |space|^2"""
    import torch
    ch, n = _tone_rows(x)
    mark = torch.from_numpy(firdes_peak_c(spacing / 2, filter_length)).to(x.device)
    space = torch.from_numpy(firdes_peak_c(-spacing / 2, filter_length)).to(x.device)
    out = torch.empty((ch, max(n - filter_length + 1, 1)), dtype=torch.float32, device=x.device)
    m = _check(lib().csdrb_bfsk_demod_bank_cf(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, mark.data_ptr(), space.data_ptr(),
                                              filter_length, _stream()), "bfsk_demod_bank_cf")
    return out[:, :m]


def fft_c2c(x, inverse: bool = False):
    """Batched unnormalised DFT along the last axis of a [B, N] (or [N]) complex64 CUDA tensor; N a power of two from 2 to 2^20
    (csdrb_fft_c2c_batch up to 16384 points, csdrb_fft_c2c_large_batch above)."""
    import torch
    xr, ptr, stride, b, n = _as_cf32_rows(x)
    out = torch.empty((b, n), dtype=torch.complex64, device=xr.device)
    call = lib().csdrb_fft_c2c_batch if n <= 16384 else lib().csdrb_fft_c2c_large_batch
    _check(call(ptr, stride, out.data_ptr(), out.stride(0), n, b, 1 if inverse else 0, _stream()), "fft_c2c")
    return out if x.dim() > 1 or x.dtype != torch.complex64 else out[0]


def _as_f32_rows(x):
    """Accept [C, N] (or [N]) float32 CUDA tensors whose rows are contiguous; return (tensor, data_ptr, row stride in floats, C, N)."""
    import torch
    if x.dtype != torch.float32:
        raise TypeError("expected float32 [C,N]")
    xr = x.unsqueeze(0) if x.dim() == 1 else x
    if not xr.is_cuda:
        raise CsdrB200Error("bank API needs CUDA tensors (no CPU fallback)")
    if xr.dim() != 2 or xr.stride(1) != 1:
        raise ValueError("samples must be contiguous within a row")
    return xr, xr.data_ptr(), xr.stride(0), xr.shape[0], xr.shape[1]


def fft_r2c(x):
    """Forward real-to-complex DFT along the last axis of a [B, N] (or [N]) float32 CUDA tensor: N a power of two from 4 to 2^21 real points,
    N // 2 + 1 complex64 bins per row as FFTW's r2c gives them (csdrb_fft_r2c_batch)."""
    import torch
    xr, ptr, stride, b, n = _as_f32_rows(x)
    out = torch.empty((b, n // 2 + 1), dtype=torch.complex64, device=xr.device)
    _check(lib().csdrb_fft_r2c_batch(ptr, stride, out.data_ptr(), out.stride(0), n, b, _stream()), "fft_r2c")
    return out if x.dim() > 1 else out[0]


def bandpass_geometry(transition_bw: float):
    """(taps_length, fft_size, input_size, overlap) exactly as csdr.c:1833-1838 sizes them."""
    T = firdes_filter_len(transition_bw)
    N = int(lib().next_pow2(T))
    if N - T < 200:
        N <<= 1
    return T, N, N - T + 1, T - 1


def bandpass_taps_fft(low_cut: float, high_cut: float, transition_bw: float, window: str = "HAMMING", device="cuda"):
    import torch
    T, N, _, _ = bandpass_geometry(transition_bw)
    taps = np.zeros(N, np.complex64)
    taps[:T] = firdes_bandpass_c(T, low_cut, high_cut, window)
    return fft_c2c(torch.from_numpy(taps).to(device))


def bandpass_fir_fft_bank_cc(x, taps_fft, input_size: int, tail=None):
    """x [C, nblocks*input_size] complex64 -> y same shape; taps_fft [N] (shared) or [C, N]; tail [C, N] carried state."""
    import torch
    xr, ptr, stride, ch, n = _as_cf32_rows(x)
    N = taps_fft.shape[-1]
    nblocks = n // input_size
    out = torch.empty((ch, nblocks * input_size), dtype=torch.complex64, device=xr.device)
    tail = torch.zeros((ch, N), dtype=torch.complex64, device=xr.device) if tail is None else tail
    tstride = 0 if taps_fft.dim() == 1 else taps_fft.stride(0)
    _check(lib().csdrb_bandpass_fir_fft_bank_cc(ptr, stride, out.data_ptr(), out.stride(0), ch, N, input_size, nblocks, taps_fft.data_ptr(), tstride,
                                                tail.data_ptr(), _stream()), "bandpass_fir_fft_bank_cc")
    return out, tail


def fastddc_fwd_cc(x, ddc: FastDDC, overlap=None):
    """x [nblocks*input_size] complex64 -> spectra [nblocks, fft_size]; overlap [fft_size-input_size] carried state."""
    import torch
    assert x.dtype == torch.complex64 and x.is_cuda and x.dim() == 1
    nblocks = x.numel() // ddc.input_size
    spectra = torch.empty((nblocks, ddc.fft_size), dtype=torch.complex64, device=x.device)
    overlap = torch.zeros(ddc.overlap_length, dtype=torch.complex64, device=x.device) if overlap is None else overlap
    _check(lib().csdrb_fastddc_fwd_cc(x.data_ptr(), spectra.data_ptr(), overlap.data_ptr(), ddc.fft_size, ddc.input_size, nblocks, _stream()), "fastddc_fwd_cc")
    return spectra, overlap


def fastddc_make_taps_fft(ddc: FastDDC, shift_rate: float, decimation: int, window: str = "HAMMING", device="cuda"):
    """csdr.c:2342-2351: bandpass taps at -shift -+ 0.5/decimation, zero pad, forward FFT, swap sides."""
    import torch
    hb = np.float32(0.5 / decimation); sh = np.float32(shift_rate)
    taps = np.zeros(ddc.fft_size, np.complex64)
    taps[:ddc.taps_length] = firdes_bandpass_c(ddc.taps_length, float(-sh - hb), float(-sh + hb), window)
    tf = fft_c2c(torch.from_numpy(taps).to(device))
    return torch.roll(tf, ddc.fft_size // 2)


def fastddc_inv_bank_cc(spectra, shifts, decimation: int, transition_bw: float, window: str = "HAMMING", state=None):
    """All channels (one per entry of ``shifts``) consume the same spectra [nblocks, fft_size].
    Returns (out [C, nblocks*post_input_size/post_decimation + 1], counts [C] int32, state dict)."""
    import torch
    dev = spectra.device
    nblocks = spectra.shape[0]
    ch = len(shifts)
    if state is not None:
        g = state["geometry"]                                         # per-channel host work happens once, at bank creation
    else:
        ddcs = [fastddc_init(transition_bw, decimation, float(s)) for s in shifts]
        g = ddcs[0]
    if state is None:
        taps_fft = torch.stack([fastddc_make_taps_fft(d, float(s), decimation, window, dev) for d, s in zip(ddcs, shifts)]).contiguous()
        chan = np.zeros((ch, 4), np.float32)
        chan.view(np.int32)[:, 0] = [d.offsetbin for d in ddcs]
        chan[:, 1] = [d.dsadata.sindelta for d in ddcs]; chan[:, 2] = [d.dsadata.cosdelta for d in ddcs]; chan[:, 3] = [d.dsadata.rate for d in ddcs]
        state = {"taps_fft": taps_fft, "chan": torch.from_numpy(chan).to(dev), "remain": torch.zeros(ch, dtype=torch.int32, device=dev),
                 "phase": torch.zeros(ch, dtype=torch.float32, device=dev), "geometry": g}
    per_block = g.post_input_size // g.post_decimation + 1
    key = ("buffers", nblocks)
    if key not in state:
        state[key] = (torch.empty((ch, nblocks * per_block + 2), dtype=torch.complex64, device=dev), torch.zeros(ch, dtype=torch.int32, device=dev),
                      _scratch(lib().csdrb_fastddc_inv_bank_scratch_bytes(ch, nblocks), dev))
    out, counts, scratch = state[key]
    _check(lib().csdrb_fastddc_inv_bank_cc(spectra.data_ptr(), nblocks, state["taps_fft"].data_ptr(), state["chan"].data_ptr(), ch, C.byref(g),
                                           state["remain"].data_ptr(), state["phase"].data_ptr(), out.data_ptr(), out.stride(0), counts.data_ptr(),
                                           scratch.data_ptr(), scratch.numel(), _stream()), "fastddc_inv_bank_cc")
    return out, counts, state


def _fastddc_chan_rows(ddcs) -> np.ndarray:
    chan = np.zeros((len(ddcs), 4), np.float32)                          # csdrb_fastddc_chan_t {int offsetbin; float sindelta, cosdelta, rate}
    chan.view(np.int32)[:, 0] = [d.offsetbin for d in ddcs]
    chan[:, 1] = [d.dsadata.sindelta for d in ddcs]; chan[:, 2] = [d.dsadata.cosdelta for d in ddcs]; chan[:, 3] = [d.dsadata.rate for d in ddcs]
    return chan


class FastddcInvPlan:
    """csdrb_fastddc_inv_plan_*: the fastddc inverse bank with the carried post-shift state inside and a fixed number of blocks per run; the state chain and
    the phasors of run k+1 are prepared while run k executes.  Same outputs as fastddc_inv_bank_cc, bit for bit."""

    def __init__(self, shifts, decimation: int, transition_bw: float, nblocks: int, window: str = "HAMMING", device="cuda"):
        import torch
        self.shifts = [float(s) for s in shifts]
        self.decimation, self.transition_bw, self.window, self.nblocks, self.device = decimation, transition_bw, window, nblocks, device
        ddcs = [fastddc_init(transition_bw, decimation, s) for s in self.shifts]
        self.geometry = ddcs[0]
        self.channels = len(ddcs)
        self.taps_fft = torch.stack([fastddc_make_taps_fft(d, s, decimation, window, device) for d, s in zip(ddcs, self.shifts)]).contiguous()
        chan = _fastddc_chan_rows(ddcs)
        self.h = lib().csdrb_fastddc_inv_plan_create(chan.ctypes.data, self.channels, C.addressof(self.geometry), nblocks)
        if not self.h:
            raise CsdrB200Error(f"csdrb_fastddc_inv_plan_create: {lib().csdrb_last_error().decode()}")
        per_block = self.geometry.post_input_size // self.geometry.post_decimation + 1
        self.out = torch.empty((self.channels, nblocks * per_block + 2), dtype=torch.complex64, device=device)
        self.counts = torch.zeros(self.channels, dtype=torch.int32, device=device)

    def run(self, spectra, out=None):
        """spectra [nblocks, fft_size] complex64 (fastddc_fwd_cc) -> (out [C, ...], counts [C] int32 on the device)"""
        assert spectra.shape == (self.nblocks, self.geometry.fft_size) and spectra.is_contiguous()
        out = self.out if out is None else out
        _check(lib().csdrb_fastddc_inv_plan_run(self.h, spectra.data_ptr(), self.taps_fft.data_ptr(), out.data_ptr(), out.stride(0), self.counts.data_ptr(), _stream()),
               "fastddc_inv_plan_run")
        return out, self.counts

    def set_shift(self, channel: int, shift: float):
        """retune one channel from the next run on (csdr.c:2342-2351 redone for that channel)"""
        d = fastddc_init(self.transition_bw, self.decimation, float(shift))
        self.taps_fft[channel].copy_(fastddc_make_taps_fft(d, float(shift), self.decimation, self.window, self.device))
        row = _fastddc_chan_rows([d])
        _check(lib().csdrb_fastddc_inv_plan_set_channel(self.h, channel, row.ctypes.data), "fastddc_inv_plan_set_channel")
        self.shifts[channel] = float(shift)

    def state(self):
        remain = np.zeros(self.channels, np.int32); phase = np.zeros(self.channels, np.float32)
        _check(lib().csdrb_fastddc_inv_plan_get_state(self.h, remain.ctypes.data, phase.ctypes.data), "fastddc_inv_plan_get_state")
        return remain, phase

    def set_state(self, remain, phase):
        remain = np.ascontiguousarray(remain, np.int32); phase = np.ascontiguousarray(phase, np.float32)
        _check(lib().csdrb_fastddc_inv_plan_set_state(self.h, remain.ctypes.data, phase.ctypes.data), "fastddc_inv_plan_set_state")

    def close(self):
        if getattr(self, "h", None):
            lib().csdrb_fastddc_inv_plan_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def ddc_bank(wide, rates, decimation: int, taps: np.ndarray, demod: bool = True, chunk: int = 1024, offset: int = 0,
             phases=None, last=None, out=None):
    """Fused shared-input bank: one wideband block [N] complex64 -> per channel shift | fir_decimate | (fmdemod).  A float32 block is a REAL
    stream (shift_addition_fc in front, csdrb_ddc_bank_f): tune a station at f Hz of a stream sampled at fs with rate -f/fs.
    Any even decimation D whose filter has M = ceil(len(taps) / D) <= 24 and D * MP <= 8000 taps (MP = the smallest of 4, 8, 12, 18, 20, 24 >= M);
    an odd D or a longer filter raises CsdrB200Error.
    Returns (out [C, n_out], new chunk-start phases [C], last baseband samples [C] or None)."""
    import torch
    assert wide.dtype in (torch.complex64, torch.float32) and wide.is_cuda and wide.dim() == 1
    entry = lib().csdrb_ddc_bank_f if wide.dtype == torch.float32 else lib().csdrb_ddc_bank
    rates = np.atleast_1d(np.asarray(rates, np.float32)); ch = rates.size
    taps = np.ascontiguousarray(taps, np.float32)
    n = wide.numel()
    n_out = fir_out_len(n, decimation, taps.size)
    dev = wide.device
    params = torch.from_numpy(np.array([shift_addition_init(float(r)) for r in rates], np.float32)).to(dev)
    d_phase = torch.zeros(ch, dtype=torch.float32, device=dev) if phases is None else phases.clone()
    stride = n_out + (n_out & 1)
    if out is None:
        out = torch.empty((ch, stride), dtype=torch.float32 if demod else torch.complex64, device=dev)
    last_out = torch.empty(ch, dtype=torch.complex64, device=dev) if demod else None
    scratch = _scratch(lib().csdrb_ddc_bank_scratch_bytes(ch, n, chunk, offset), dev)
    rc = _check(entry(wide.data_ptr(), n, ch, params.data_ptr(), d_phase.data_ptr(), chunk, offset, decimation, _fp(taps), taps.size,
                                     1 if demod else 0, out.data_ptr(), out.stride(0), last.data_ptr() if last is not None else None,
                                     last_out.data_ptr() if last_out is not None else None, scratch.data_ptr(), scratch.numel(), _stream()), "ddc_bank")
    assert rc == n_out
    return out[:, :n_out], d_phase, last_out


def limit_ff(x, max_amplitude: float = 1.0, out=None):
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.is_contiguous()
    out = torch.empty_like(x) if out is None else out
    _check(lib().csdrb_limit_ff(x.data_ptr(), out.data_ptr(), x.numel(), max_amplitude, _stream()), "limit_ff")
    return out


def deemphasis_wfm_bank_ff(x, tau: float, sample_rate: int, last=None, out=None):
    """x [C, N] float32 -> (y [C, N], carried last outputs [C])."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    out = torch.empty((ch, n), dtype=torch.float32, device=x.device) if out is None else out
    last = torch.zeros(ch, dtype=torch.float32, device=x.device) if last is None else last.clone()
    _check(lib().csdrb_deemphasis_wfm_bank_ff(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, tau, sample_rate, last.data_ptr(), _stream()),
           "deemphasis_wfm_bank_ff")
    return out, last


def deemphasis_nfm_taps(sample_rate: int):
    """the fixed FIR deemphasis_nfm_ff uses at this rate (host table of the library), or None"""
    n = C.c_int(0)
    p = lib().csdrb_deemphasis_nfm_taps(sample_rate, C.byref(n))
    return np.ctypeslib.as_array(p, shape=(n.value,)).copy() if n.value else None


def deemphasis_nfm_bank_ff(x, sample_rate: int, limit_max: float = 0.0, out=None):
    """x [C, N] float32 -> y [C, N - taps] (empty when the rate has no table); limit_max > 0 clamps the input first (fused limit_ff)."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    ch, n = x.shape
    out = torch.empty((ch, n), dtype=torch.float32, device=x.device) if out is None else out
    rc = _check(lib().csdrb_deemphasis_nfm_bank_ff(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, sample_rate, limit_max, _stream()),
                "deemphasis_nfm_bank_ff")
    return out[:, :rc]


def fir_valid_bank_ff(x, taps, limit_max: float = 0.0, out=None):
    """x [C, N] float32, taps (host, <= 208) -> y [C, N - taps]: the de-emphasis FIR kernel with caller-supplied taps."""
    import torch
    assert x.dtype == torch.float32 and x.is_cuda and x.dim() == 2 and x.stride(1) == 1
    taps = np.ascontiguousarray(taps, np.float32)
    ch, n = x.shape
    out = torch.empty((ch, n), dtype=torch.float32, device=x.device) if out is None else out
    rc = _check(lib().csdrb_fir_valid_bank_ff(x.data_ptr(), x.stride(0), out.data_ptr(), out.stride(0), ch, n, _fp(taps), taps.size, limit_max, _stream()),
                "fir_valid_bank_ff")
    return out[:, :rc]


class DdcBank:
    """Streaming shared-input DDC/NFM bank (csdrb_ddc_bank_*): shift | fir_decimate | [fmdemod] for C channels of one wideband stream,
    one call per block, all per-channel state inside; the phase-chain pre-pass of the next block overlaps the current block.
    Serves the geometries ddc_bank() serves (any even decimation within the tap limits); the constructor raises CsdrB200Error for the others."""

    def __init__(self, rates, decimation: int, taps: np.ndarray, demod: bool = True, chunk: int = 1024):
        self.rates = np.ascontiguousarray(np.atleast_1d(rates), np.float32)
        self.taps = np.ascontiguousarray(taps, np.float32)
        self.decimation, self.demod, self.channels = decimation, demod, self.rates.size
        self.h = lib().csdrb_ddc_bank_create(self.channels, _fp(self.rates), decimation, _fp(self.taps), self.taps.size, 1 if demod else 0, chunk)
        if not self.h:
            raise CsdrB200Error(f"csdrb_ddc_bank_create: {lib().csdrb_last_error().decode()}")

    def process(self, wide, out=None):
        """wide: [N] complex64 CUDA tensor starting where the previous call stopped consuming (n_out*decimation samples in); a float32 tensor is
        a block of a real stream (csdrb_ddc_bank_process_f)."""
        import torch
        assert wide.dtype in (torch.complex64, torch.float32) and wide.is_cuda and wide.dim() == 1
        entry = lib().csdrb_ddc_bank_process_f if wide.dtype == torch.float32 else lib().csdrb_ddc_bank_process
        n_out = fir_out_len(wide.numel(), self.decimation, self.taps.size)
        if out is None:
            out = torch.empty((self.channels, n_out + (n_out & 1)), dtype=torch.float32 if self.demod else torch.complex64, device=wide.device)
        rc = _check(entry(self.h, wide.data_ptr(), wide.numel(), out.data_ptr(), out.stride(0), _stream()), "ddc_bank_process")
        return out[:, :rc]

    def set_rate(self, channel: int, rate: float):
        _check(lib().csdrb_ddc_bank_set_rate(self.h, channel, rate), "ddc_bank_set_rate")

    @property
    def offset(self) -> int:
        return int(lib().csdrb_ddc_bank_offset(self.h))

    def close(self):
        if getattr(self, "h", None):
            lib().csdrb_ddc_bank_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class MultiBank:
    """One process, several GPUs (csdrb_multi_bank_*): the shared-input DDC/NFM bank in contiguous channel slices over `devices`, the wideband block
    broadcast from devices[0] with NCCL.  Host (ideally pinned) numpy buffers in and out; submit()/collect() pipeline two blocks."""

    def __init__(self, devices, rates, decimation: int, taps: np.ndarray, demod: bool = True, chunk: int = 1024, max_block: int = 1 << 21):
        self.rates = np.ascontiguousarray(np.atleast_1d(rates), np.float32)
        self.taps = np.ascontiguousarray(taps, np.float32)
        self.decimation, self.demod, self.channels = decimation, demod, self.rates.size
        devs = (C.c_int * len(devices))(*devices)
        self.h = lib().csdrb_multi_bank_create(len(devices), devs, self.channels, _fp(self.rates), decimation, _fp(self.taps), self.taps.size, 1 if demod else 0,
                                               chunk, max_block)
        if not self.h:
            raise CsdrB200Error(f"csdrb_multi_bank_create: {lib().csdrb_last_error().decode()}")

    def slices(self):
        out = []
        for i in range(lib().csdrb_multi_bank_devices(self.h)):
            d, c0, n = C.c_int(), C.c_int(), C.c_int()
            _check(lib().csdrb_multi_bank_slice(self.h, i, C.byref(d), C.byref(c0), C.byref(n)), "multi_bank_slice")
            out.append((d.value, c0.value, n.value))
        return out

    def submit(self, wide: np.ndarray, out: np.ndarray) -> int:
        assert wide.dtype == np.complex64 and wide.ndim == 1 and out.ndim == 2 and out.shape[0] == self.channels and out.strides[1] == out.itemsize
        assert out.dtype == (np.float32 if self.demod else np.complex64)
        return _check(lib().csdrb_multi_bank_submit(self.h, wide.ctypes.data, wide.size, out.ctypes.data, out.strides[0] // out.itemsize), "multi_bank_submit")

    def collect(self, ticket: int) -> int:
        return _check(lib().csdrb_multi_bank_collect(self.h, ticket), "multi_bank_collect")

    def process(self, wide: np.ndarray, out: np.ndarray) -> int:
        return self.collect(self.submit(wide, out))

    def set_rate(self, channel: int, rate: float):
        _check(lib().csdrb_multi_bank_set_rate(self.h, channel, rate), "multi_bank_set_rate")

    def close(self):
        if getattr(self, "h", None):
            lib().csdrb_multi_bank_destroy(self.h); self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def shift_unroll_bank_cc(x, rates, phases=None, table_size: int = 1024, out=None):
    """shift_unroll_cc for C channels; x [N] (shared wideband input) or [C, N].  Returns (y [C, N], carried phases [C])."""
    import torch
    rates = np.atleast_1d(np.asarray(rates, np.float32)); ch = rates.size
    shared = (x.dim() == 1) if x.dtype == torch.complex64 else (x.dim() == 2)
    xr, ptr, stride, xc, n = _as_cf32_rows(x)
    if shared:
        stride = 0
    dev = xr.device
    params = torch.from_numpy(np.array([shift_addition_init(float(r)) for r in rates], np.float32)).to(dev)
    ds = np.empty((ch, table_size), np.float32); dc = np.empty((ch, table_size), np.float32)
    for c, r in enumerate(rates):
        d = lib().shift_unroll_init(float(r), table_size)
        ds[c] = np.ctypeslib.as_array(d.dsin, shape=(table_size,)); dc[c] = np.ctypeslib.as_array(d.dcos, shape=(table_size,))
    d_ds, d_dc = torch.from_numpy(ds).to(dev), torch.from_numpy(dc).to(dev)
    d_phase = torch.zeros(ch, dtype=torch.float32, device=dev) if phases is None else phases.clone()
    out = torch.empty((ch, n), dtype=torch.complex64, device=dev) if out is None else out
    scratch = _scratch(lib().csdrb_shift_addition_bank_scratch_bytes(ch, n, min(table_size, n)) + 16, dev)
    _check(lib().csdrb_shift_unroll_bank_cc(ptr, stride, out.data_ptr(), out.stride(0), ch, n, params.data_ptr(), d_ds.data_ptr(), d_dc.data_ptr(), table_size,
                                            table_size, d_phase.data_ptr(), scratch.data_ptr(), scratch.numel(), _stream()), "shift_unroll_bank_cc")
    return out, d_phase


class SpectrumBank:
    """The OpenWebRX waterfall chain `fft_cc N E W | logaveragepower_cf ADD_DB N A | fft_exchange_sides_ff N [| compress_fft_adpcm_f_u8 N]` on
    `rows` streams at once (csdrb_spectrum_bank_cf).  Owns the window table, the carried history and partial line, and the host state;
    process(x) takes the next n samples of every row ([rows, n] complex64 CUDA tensor, or [n] for one row) and returns the lines they complete:
    [rows, lines, N] float32 dB, or [rows, lines, (N + 10) // 2] uint8 with compress=True.
    real=True: the chain of a real stream, `fft_fc N E W | logaveragepower_cf ADD_DB N A [| compress_fft_adpcm_f_u8 N]` (csdrb_spectrum_bank_f):
    process(x) takes [rows, n] (or [n]) float32 real samples, `every` counts real samples, a frame is 2N of them and the lines are N bins in
    bin order (DC first)."""

    def __init__(self, rows: int, fft_size: int, every: int, averages: int, add_db: float, window: str = "HAMMING", compress: bool = False,
                 device="cuda", real: bool = False):
        import torch
        self.rows, self.device, self.real = rows, torch.device(device), real
        self.params = SpectrumParams(fft_size, every, averages, 1 if compress else 0, add_db)
        self.state = SpectrumState(0, 0)
        frame = 2 * fft_size if real else fft_size
        self.window = torch.from_numpy(libcsdr.precalculate_window(frame, window)).to(self.device)
        self.hist = torch.zeros((rows, frame), dtype=torch.float32 if real else torch.complex64, device=self.device)
        self.acc = torch.zeros((rows, fft_size), dtype=torch.float32, device=self.device)
        self.line_bytes = (fft_size + 10) // 2 if compress else 4 * fft_size

    def lines(self, n: int) -> int:
        f = lib().csdrb_spectrum_bank_lines_f if self.real else lib().csdrb_spectrum_bank_lines
        return _check(f(C.byref(self.params), C.byref(self.state), n), "spectrum_bank_lines")

    def process(self, x, scratch_bytes: int | None = None):
        import torch
        if self.real:
            xr, ptr, stride, rows, n = _as_f32_rows(x)
        else:
            if x.dtype == torch.complex64 and x.dim() == 1:
                x = x.unsqueeze(0)
            xr, ptr, stride, rows, n = _as_cf32_rows(x)
        if rows != self.rows:
            raise ValueError(f"expected {self.rows} rows, got {rows}")
        N, L = self.params.fft_size, self.lines(n)
        if self.params.compress:
            out = torch.empty((rows, L, self.line_bytes), dtype=torch.uint8, device=self.device)
        else:
            out = torch.empty((rows, L, N), dtype=torch.float32, device=self.device)
        if scratch_bytes is None:
            scratch_bytes = (lib().csdrb_spectrum_bank_scratch_bytes_f if self.real else lib().csdrb_spectrum_bank_scratch_bytes)(rows, n, C.byref(self.params))
        scratch = _scratch(scratch_bytes + 16, self.device)
        bank = lib().csdrb_spectrum_bank_f if self.real else lib().csdrb_spectrum_bank_cf
        got = _check(bank(ptr if n else self.hist.data_ptr(), stride, rows, n, self.window.data_ptr(), C.byref(self.params),
                          self.hist.data_ptr(), self.acc.data_ptr(), C.byref(self.state),
                          out.data_ptr() if out.numel() else self.acc.data_ptr(),
                          out.stride(0) * out.element_size(), scratch.data_ptr(), scratch_bytes, _stream()),
                     "spectrum_bank_f" if self.real else "spectrum_bank_cf")
        assert got == L
        return out


class WfmAudioBank:
    """The WFM audio tail `fractional_decimator_ff rate 12 | deemphasis_wfm_ff sample_rate tau | convert_f_s16` on `channels` streams at once,
    in the CLI's calls of `bufsize` samples (csdrb_wfm_audio_bank_f_s16).  Owns the unconsumed rest of every row, the de-emphasis carry and the
    host state; process(x) takes the next samples of every row ([channels, n] float32 CUDA tensor) and returns the audio they complete as
    [channels, m] int16."""

    def __init__(self, channels: int, rate: float = 5.0, tau: float = 50e-6, sample_rate: int = 48000, bufsize: int = 1024, device="cuda"):
        import torch
        self.channels, self.device = channels, torch.device(device)
        self.params = WfmAudioParams(rate, bufsize, tau, sample_rate)
        self.state = WfmAudioState(0.0, 0)
        self.last = torch.zeros(channels, dtype=torch.float32, device=self.device)
        self.rest = torch.zeros((channels, 0), dtype=torch.float32, device=self.device)
        _check(self.outputs(0)[0], "wfm_audio_bank_outputs")               # refuses bad parameters here rather than at the first call

    def outputs(self, n: int):
        """(s16 samples per row, samples consumed per row) of a call on n samples, from the host state alone"""
        consumed = C.c_int(0)
        m = lib().csdrb_wfm_audio_bank_outputs(C.byref(self.params), C.byref(self.state), n, C.byref(consumed))
        return m, consumed.value

    def process(self, x):
        import torch
        if x.dim() != 2 or x.shape[0] != self.channels or x.dtype != torch.float32 or not x.is_cuda:
            raise ValueError(f"expected a [{self.channels}, n] float32 CUDA tensor")
        x = torch.cat([self.rest, x], dim=1) if self.rest.shape[1] else x.contiguous()
        n = x.shape[1]
        m, _ = self.outputs(n)
        _check(m, "wfm_audio_bank_outputs")
        out = torch.empty((self.channels, m), dtype=torch.int16, device=self.device)
        consumed = C.c_int(0)
        got = _check(lib().csdrb_wfm_audio_bank_f_s16(x.data_ptr() if n else self.last.data_ptr(), max(n, 1), self.channels, n, C.byref(self.params),
                                                      C.byref(self.state), self.last.data_ptr(), out.data_ptr() if m else self.last.data_ptr(),
                                                      max(m, 1), C.byref(consumed), _stream()), "wfm_audio_bank_f_s16")
        assert got == m
        self.rest = x[:, consumed.value:].clone()
        return out


def spectrum_logpower(x, fft_size: int, window: str = "HAMMING", add_db: float = 0.0):
    """fft_cc | logpower_cf for a whole stream on the device: frames of fft_size samples -> [frames, fft_size] dB values."""
    import torch
    assert x.dtype == torch.complex64 and x.is_cuda and x.dim() == 1
    frames = x.numel() // fft_size
    xs = x[:frames * fft_size].contiguous().view(frames, fft_size)
    w = torch.from_numpy(libcsdr.precalculate_window(fft_size, window)).to(x.device)
    xw = torch.empty_like(xs)
    _check(lib().csdrb_apply_window_rows_c(xs.data_ptr(), xw.data_ptr(), w.data_ptr(), fft_size, frames, _stream()), "apply_window_rows_c")
    spec = fft_c2c(xw)
    out = torch.empty((frames, fft_size), dtype=torch.float32, device=x.device)
    _check(lib().csdrb_logpower_cf(spec.data_ptr(), out.data_ptr(), frames * fft_size, add_db, _stream()), "logpower_cf")
    return out
