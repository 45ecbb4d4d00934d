// kernels.h -- internal launcher prototypes (host side of each .cu).  Not part of the public C ABI.
#pragma once
#include <cuda_runtime.h>

namespace csdrb {

// K3 fir_decimate.cu
int launch_fir_decimate_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n_in,
                             int D, const float* h_taps, const float* d_taps, long taps_stride, int T, int variant,
                             cudaStream_t st);
int fir_bank_variant_count();
int launch_u8_rows_to_cf32(const unsigned char* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, cudaStream_t st);
int launch_fir_decimate_bank_u8(const unsigned char* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n_in,
                                int D, const float* h_taps, int T, cudaStream_t st);

// K1/K4 elementwise.cu
int launch_convert_u8_f(const unsigned char* d_in, float* d_out, long n, cudaStream_t st);
int launch_convert_s16_f(const short* d_in, float* d_out, long n, cudaStream_t st);
int launch_convert_f_s16(const float* d_in, short* d_out, long n, cudaStream_t st);
// the other sample formats: byte buffers at any address, float buffers 4-byte aligned; s24 counts values (3 bytes each), bigendian as the reference's flag
int launch_convert_s8_f(const unsigned char* d_in, float* d_out, long n, cudaStream_t st);
int launch_convert_f_s8(const float* d_in, unsigned char* d_out, long n, cudaStream_t st);
int launch_convert_f_u8(const float* d_in, unsigned char* d_out, long n, cudaStream_t st);
int launch_convert_s24_f(const unsigned char* d_in, float* d_out, long n, int bigendian, cudaStream_t st);
int launch_convert_f_s24(const float* d_in, unsigned char* d_out, long n, int bigendian, cudaStream_t st);
int launch_fmdemod_quadri_bank(const float2* d_in, long in_stride, float* d_out, long out_stride, int channels, int n,
                               const float2* d_last_in, float2* d_last_out, cudaStream_t st);

int launch_adpcm_encode_rows(const short* d_in, long in_stride, unsigned char* d_out, long out_stride, int rows, int n, void* d_state_io, cudaStream_t st);
int launch_compress_fft_adpcm_rows(const float* d_in, long in_stride, unsigned char* d_out, long out_stride, int rows, int fft_size, cudaStream_t st);
int launch_limit_ff(const float* d_in, float* d_out, long n, float max_amplitude, cudaStream_t st);
int launch_deemphasis_wfm_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, float tau, int sample_rate,
                               float* d_last_io, cudaStream_t st);
// WFM audio tail `fractional_decimator_ff R 12 | deemphasis_wfm_ff SR TAU | convert_f_s16`, audio.cu.  Parameters and state are the host
// csdrb_wfm_audio_params_t / csdrb_wfm_audio_state_t; both return the s16 samples per row (< 0 refused).
int wfm_audio_outputs(const void* h_params, const void* h_state, int n, int* consumed_out);
int launch_wfm_audio_bank(const float* d_in, long in_stride, int channels, int n, const void* h_params, void* h_state_io, float* d_last_io,
                          short* d_out, long out_stride, int* consumed_out, int* launches, cudaStream_t st);

// deemphasis_nfm_ff: the tap tables live in host/firdes.c (public accessor, see include/csdr_b200.h)
constexpr int kNfmMaxTaps = 208;
extern "C" const float* csdrb_deemphasis_nfm_taps(int sample_rate, int* taps_length);
int launch_fir_valid_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, const float* h_taps, int T,
                          float limit_max, cudaStream_t st);
int launch_deemphasis_nfm_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, int sample_rate,
                               float limit_max, cudaStream_t st);

int launch_apply_window_rows(const float2* d_in, float2* d_out, const float* d_window, int size, long rows, cudaStream_t st);
int launch_power(const float2* d_in_c, const float* d_in_f, float* d_out, long n, float add_db, int mode, cudaStream_t st);
int launch_shift_unroll_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n,
                             const float* d_params, const float* d_dsin, const float* d_dcos, long table_stride, int table_size,
                             float* d_phase_io, void* d_scratch, size_t scratch_bytes, cudaStream_t st);

void shift_unroll_bank_single(const float2* d_in, float2* d_out, int n, const float* d_dsin, const float* d_dcos, const float* d_phase, cudaStream_t st);

// K2 shift.cu
size_t shift_bank_scratch_bytes(int channels, int n, int chunk);
int launch_shift_addition_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n,
                               const float* d_params, float* d_phase_io, int chunk, void* d_scratch, size_t scratch_bytes, cudaStream_t st);
// shift_addition_fc: real rows in (in_stride 0: every channel shifts the same row), complex rows out; the phase chain and scratch of the _cc bank
int launch_shift_addition_bank_fc(const float* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n,
                                  const float* d_params, float* d_phase_io, int chunk, void* d_scratch, size_t scratch_bytes, cudaStream_t st);
// one shift_addition_fc call (n samples, one channel) whose phasor starts at *d_seed instead of (cos, sin) of *d_phase_io evaluated in double
int launch_shift_addition_fc_seeded(const float* d_in, float2* d_out, int n, const float* d_params, float* d_phase_io, const float2* d_seed,
                                    void* d_scratch, size_t scratch_bytes, cudaStream_t st);
int launch_shift_addfast_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n,
                              const float* d_params, float* d_phase_io, int chunk, void* d_scratch, size_t scratch_bytes, cudaStream_t st);
size_t shift_math_scratch_bytes(int channels, int n);
int launch_shift_math_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, const float* d_rates,
                           float* d_phase_io, void* d_scratch, size_t scratch_bytes, cudaStream_t st);
int launch_shift_table_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, const float* d_rates,
                            float* d_phase_io, const float* d_table, int table_size, void* d_scratch, size_t scratch_bytes, cudaStream_t st);
int launch_decimating_shift_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n,
                                 const float* d_params, int decimation, int* d_remain_io, float* d_phase_io, int* d_out_size, cudaStream_t st);

// K5/K6 audio.cu
size_t fracdec_scratch_bytes(int channels, int n, float rate);
int launch_fractional_decimator_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n,
                                     float rate, int num_poly_points, const float* d_taps, int taps_length, void* d_state,
                                     void* d_scratch, size_t scratch_bytes, cudaStream_t st);
size_t fastagc_scratch_bytes(int channels, int nblocks);
int launch_fastagc_bank_s16(const float* d_in, long in_stride, short* d_out, long out_stride, int channels, int block, int nblocks,
                            float reference, void* d_state, float* d_hist, void* d_scratch, size_t scratch_bytes, cudaStream_t st);
int launch_fastagc_bank_s16_any(const float* d_in, long in_stride, short* d_out, long out_stride, int channels, int block, int nblocks,
                                float reference, void* d_state, float* d_hist, void* d_scratch, size_t scratch_bytes, cudaStream_t st);
int launch_fastagc_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int block, int nblocks,
                        float reference, void* d_state, float* d_hist, void* d_scratch, size_t scratch_bytes, cudaStream_t st);

// rational_resampler_ff, resample.cu.  The bank returns outputs per channel and writes the reference's state
// {input_processed, output_size, last_taps_delay} to h_state (host memory) without waiting for the device.
constexpr int kRsMaxTaps = 16384;
int rational_resampler_state(int input_size, int interpolation, int decimation, int taps_length, int last_taps_delay, int* h_state);
int launch_rational_resampler_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int input_size,
                                   int interpolation, int decimation, const float* h_taps, int taps_length, int last_taps_delay,
                                   int* h_state, cudaStream_t st);

// AM / SSB receiver blocks, agc.cu.  AgcParams / AgcState have the layout of csdrb_agc_params_t / csdrb_agc_state_t (include/csdr_b200.h).
struct AgcParams { float reference, attack_rate, decay_rate, max_gain; int hang_time, attack_wait_time; float gain_filter_alpha; int chunk; };
struct AgcState { float gain, last_peak; int hang_counter, attack_wait_counter, offset; };
int launch_amdemod_cf(const float2* d_in, float* d_out, long n, cudaStream_t st);
int launch_fastdcblock_bank(const void* d_in, long in_stride, int cf32, float* d_out, long out_stride, int channels, int block, int nblocks,
                            float* d_last_dc_io, cudaStream_t st);
int launch_agc_bank(const void* d_in, long in_stride, int cf32, void* d_out, long out_stride, int s16, int channels, int n, const void* h_params_v,
                    void* d_state_v, float limit_max, cudaStream_t st);   // AgcParams on the host, AgcState[channels] on the device

// BPSK31 receive chain, psk31.cu.  TrParams / TrState have the layout of csdrb_timing_recovery_params_t / csdrb_timing_recovery_state_t.
struct TrParams { int algorithm, decimation, use_q; float loop_gain, max_error; };
struct TrState { int last_correction_offset, input_processed, output_size; };
int launch_simple_agc_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, float rate, float reference,
                           float max_gain, float* d_gain_io, cudaStream_t st);
int timing_recovery_max_outputs(int decimation, int input_size, float loop_gain, float max_error);   // symbols one call on input_size samples can make
int launch_timing_recovery_bank(const float2* d_in, long in_stride, const int* d_start, const int* d_size, float2* d_out, long out_stride, float* d_err,
                                int* d_idx, int channels, const void* h_params_v, void* d_state_v, int max_size, cudaStream_t st);   // TrParams on the host, TrState[channels] on the device
int launch_dbpsk_bank(const float2* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int n, const int* d_lengths,
                      const float2* d_last_in, float2* d_last_out, cudaStream_t st);
int launch_varicode_bank(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int n, const int* d_lengths,
                         unsigned long long* d_hist_io, int* d_count, cudaStream_t st);

// BPSK31 transmit chain, psk31_tx.cu: one row per channel, d_lengths optional (NULL: n for every row); each returns the launches it made
extern "C" int csdrb_psk31_sine_rates(int interpolation, float* rates);   // host/psk31_rates.c: the build's rate table; -1 without libmvec
int launch_varicode_encoder_bank(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int n,
                                 const int* d_lengths, int output_max_size, int* d_input_processed, int* d_output_size, cudaStream_t st);
int launch_differential_codec_bank(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int n,
                                   const int* d_lengths, int encode, unsigned char* d_state_io, cudaStream_t st);
int launch_psk_modulator_bank(const unsigned char* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, const int* d_lengths,
                              int n_psk, cudaStream_t st);
int launch_psk31_interpolate_sine_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, const int* d_lengths,
                                       int interpolation, float2* d_last_io, cudaStream_t st);

// RTTY receive chain, rtty.cu.  SerialLineParams has the layout of csdrb_serial_line_params_t.
struct SerialLineParams { float samples_per_bits; int databits; float stopbits, bit_sampling_width_ratio; };
int serial_line_max_outputs(float samples_per_bits, int databits, float stopbits, int input_size);   // characters input_size samples can hold at most
int launch_serial_line_bank(const float* d_in, long in_stride, int end, int* d_start_io, unsigned char* d_out, long out_stride, int* d_count,
                            int* d_stuck, int channels, const void* h_params_v, int bufsize, cudaStream_t st);   // SerialLineParams on the host
int launch_baudot_bank(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int n, const int* d_lengths,
                       unsigned char* d_mode_io, int* d_count, cudaStream_t st);

// tone filters, tone.cu: the valid convolution of each row with shared complex taps (2 <= L <= kToneMaxTaps, else -2); n - L + 1 per row
constexpr int kToneMaxTaps = 4096;
int launch_apply_fir_bank_cc(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, const float2* d_taps, int L,
                             cudaStream_t st);
int launch_bfsk_demod_bank_cf(const float2* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, const float2* d_mark,
                              const float2* d_space, int L, cudaStream_t st);

// K7/K8/K9 fft.cu.  row_fft_twiddles: the device table of block_row_fft_io<n> (fft16.cuh), cached per device and size.
int row_fft_twiddles(int n, const float2** out, cudaStream_t st);
int launch_fft_c2c_batch(const float2* d_in, long in_stride, float2* d_out, long out_stride, int n, int batch, int inverse, cudaStream_t st);
int launch_olafir_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int fft_size, int input_size,
                       int nblocks, const float2* d_taps_fft, long taps_stride, float2* d_tail_io, int blocks_per_cta, cudaStream_t st);
int launch_apply_fir_fft(const float2* d_in, const float2* d_taps_fft, const float2* d_last_overlap, int overlap_size, float2* d_out,
                         int fft_size, cudaStream_t st);
int launch_fastddc_fwd(const float2* d_in, float2* d_spectra, float2* d_overlap_io, int fft_size, int input_size, int nblocks, cudaStream_t st);
// four-step transforms above the single-CTA range, fft.cu: the batched c2c call, and the forms launch_fastddc_fwd and launch_apply_fir_fft hand
// their sizes above 16384 to (same contracts)
constexpr int kFftLargeMinN = 1 << 15, kFftLargeMaxN = 1 << 20;
int launch_fft_c2c_large_batch(const float2* d_in, long in_stride, float2* d_out, long out_stride, int n, int batch, int inverse, cudaStream_t st);
int launch_fastddc_fwd_large(const float2* d_in, float2* d_spectra, float2* d_overlap_io, int fft_size, int input_size, int nblocks, cudaStream_t st);
int launch_apply_fir_fft_large(const float2* d_in, const float2* d_taps_fft, const float2* d_last_overlap, int overlap_size, float2* d_out,
                               int fft_size, cudaStream_t st);
// real-to-complex transforms (fft.cu, kernels fft_real.cuh): n real points (power of two, 4..2*kFftLargeMaxN) -> n/2 + 1 bins per row; the split
// table W_n^k, k = 0..n/4, of the n/2-point packed transform (cached per device and size)
int get_rfft_twiddles(int m, const float2** out, cudaStream_t st);
int launch_fft_r2c_batch(const float* d_in, long in_stride, float2* d_out, long out_stride, int n, int batch, cudaStream_t st);
size_t fastddc_inv_scratch_bytes(int channels, int nblocks);
int launch_fastddc_inv_bank(const float2* d_spectra, int nblocks, const float2* d_taps_fft, const void* d_chan, int channels,
                            int fft_size, int fft_inv_size, int pre_decimation, int scrap, int post_input_size, int post_decimation,
                            int* d_remain_io, float* d_phase_io, float2* d_out, long out_stride, int* d_out_total,
                            void* d_scratch, size_t scratch_bytes, cudaStream_t st);

// fastddc inverse bank with look-ahead (fft.cu): a plan owns the post-shift state and prepares the next run's chain + phasors during the current one
int fastddc_inv_plan_create(void** out_plan, const void* h_chan, int channels, int nblocks, int fft_size, int fft_inv_size, int pre_decimation, int scrap,
                            int post_input_size, int post_decimation);
int fastddc_inv_plan_run(void* plan, const float2* d_spectra, const float2* d_taps_fft, float2* d_out, long out_stride, int* d_out_total, cudaStream_t st);
int fastddc_inv_plan_set_channel(void* plan, int c, const void* h_chan_one);
int fastddc_inv_plan_get_state(void* plan, int* h_remain, float* h_phase);
int fastddc_inv_plan_set_state(void* plan, const int* h_remain, const float* h_phase);
void fastddc_inv_plan_destroy(void* plan);

// waterfall spectrum bank, spectrum.cu.  SpectrumParams / SpectrumState have the layout of csdrb_spectrum_params_t / csdrb_spectrum_state_t.
struct SpectrumParams { int fft_size, every, averages, compress; float add_db; };
struct SpectrumState { long long consumed, frames; };
// real = 1: the real-input bank (fft_fc N E W | logaveragepower_cf X N A [| compress_fft_adpcm_f_u8 N]): n, every and the history count real samples.
long long spectrum_frames_at(int fft_size, int every, long long total);        // frames fft_cc completes on the first `total` samples of a stream
long long spectrum_frames_at_f(int fft_size, int every, long long total);      // frames fft_fc completes (fft_size bins, 2*fft_size real points)
long spectrum_lines(const void* h_params_v, const void* h_state_v, long n, int real);   // lines a call on n samples completes; < 0 for bad arguments
size_t spectrum_scratch_bytes(int rows, long n, const void* h_params_v);         // one launch for a whole call; 0 for bad arguments
int launch_spectrum_bank(const float2* d_in, long in_stride, int rows, long n, const float* d_window, const void* h_params_v, float2* d_hist_io,
                         float* d_acc_io, void* h_state_io, void* d_out, long out_stride_bytes, void* d_scratch, size_t scratch_bytes, int* launches,
                         cudaStream_t st);   // SpectrumParams and SpectrumState on the host; returns lines written per row
int launch_spectrum_bank_f(const float* d_in, long in_stride, int rows, long n, const float* d_window, const void* h_params_v, float* d_hist_io,
                           float* d_acc_io, void* h_state_io, void* d_out, long out_stride_bytes, void* d_scratch, size_t scratch_bytes, int* launches,
                           cudaStream_t st);   // the real-input bank: d_window 2N floats, d_hist_io [rows][2N] floats

// transmit banks, interpolate.cu: fir_interpolate_cc rows (returns the outputs per row) and fmmod_fc rows (returns n); -1 for bad arguments
int launch_fir_interpolate_bank_cc(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, int interpolation,
                                   const float* d_taps, int taps_length, cudaStream_t st);
int launch_fmmod_bank_fc(const float* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, float* d_phase_io, cudaStream_t st);
// modulate.cu: gain_ff, dsb_fc, add_dcoffset_cc and fixed_amplitude_cc rows; each returns the launches it made (0 or 1), -1 for bad arguments
int launch_gain_bank_ff(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, float gain, cudaStream_t st);
int launch_dsb_bank_fc(const float* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, float q_value, cudaStream_t st);
int launch_add_dcoffset_bank_cc(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, cudaStream_t st);
int launch_fixed_amplitude_bank_cc(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, float amplitude,
                                   cudaStream_t st);

// synthesis bank, synth.cu: C channels of fir_interpolate_cc | shift_addition_cc summed in a fixed pairwise tree over the channel index into one
// wideband row.  Returns G*I outputs (< 0 refused); *launches gets the kernels it launched
size_t synth_bank_scratch_bytes(int channels, int n, int interpolation, int taps_length, int chunk, int offset);
int launch_synth_bank(const float2* d_in, long in_stride, int channels, int n, int interpolation, const float* d_taps, int taps_length,
                      const float* d_params, float* d_phase_io, int chunk, int offset, float2* d_out, void* d_scratch, size_t scratch_bytes,
                      int* launches, cudaStream_t st);

// fused shared-input DDC bank, ddc_bank.cu
int ddc_bank_geometry(int decimation, int taps_length);               // 0 when the bank serves (decimation, taps_length); else -2 with the error set
size_t ddc_bank_scratch_bytes(int channels, int input_size, int chunk, int offset);
size_t ddc_bank_tables_bytes(int channels);                            // persistent phase-wrap tables of a bank (phase_table.cuh), one per channel
int launch_ddc_rechunk(int channels, const float* d_params, float* d_phase_io, int n, cudaStream_t st);
int launch_ddc_tables(int channels, const float* d_params, int chunk, void* d_tables, cudaStream_t st);
int launch_ddc_prepass(int input_size, int channels, const float* d_params, float* d_phase_io, int chunk, int offset, int decimation,
                       int taps_length, void* d_scratch, size_t scratch_bytes, const void* d_tables, cudaStream_t st);   // d_tables NULL: built per call in d_scratch
// where launch_ddc_prepass left the (cos, sin) seeds of a block's absolute chunks, [channels][*nchunks], in its scratch
const float2* ddc_prepass_seeds(const void* d_scratch, int channels, int input_size, int chunk, int offset, int* nchunks);
int launch_ddc_main(const float2* d_wide, int input_size, int channels, const float* d_params, int chunk, int offset, int decimation,
                    const float* h_taps, int taps_length, int demod, void* d_out, long out_stride, const float2* d_last_in, float2* d_last_out,
                    const void* d_scratch, cudaStream_t st);
int launch_ddc_bank(const float2* d_wide, int input_size, int channels, const float* d_params, float* d_phase_io, int chunk, int offset,
                    int decimation, const float* h_taps, int taps_length, int demod, void* d_out, long out_stride,
                    const float2* d_last_in, float2* d_last_out, void* d_scratch, size_t scratch_bytes, int* launches, cudaStream_t st);
// the same bank on real wideband samples (shift_addition_fc | fir_decimate_cc [| fmdemod_quadri_cf]): d_wide 8-byte aligned, same geometries and contract
int launch_ddc_main_f(const float* d_wide, int input_size, int channels, const float* d_params, int chunk, int offset, int decimation,
                      const float* h_taps, int taps_length, int demod, void* d_out, long out_stride, const float2* d_last_in, float2* d_last_out,
                      const void* d_scratch, cudaStream_t st);
int launch_ddc_bank_f(const float* d_wide, int input_size, int channels, const float* d_params, float* d_phase_io, int chunk, int offset,
                      int decimation, const float* h_taps, int taps_length, int demod, void* d_out, long out_stride,
                      const float2* d_last_in, float2* d_last_out, void* d_scratch, size_t scratch_bytes, int* launches, cudaStream_t st);

}  // namespace csdrb
