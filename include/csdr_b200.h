/*
 * csdr_b200.h -- public C ABI of libcsdr_b200.so (H100 / sm_90a implementation of the csdr block-DSP hot path).
 *
 * Two layers, both plain C (System V x86-64, no C++ or torch types in any signature):
 *
 *   Part A  "libcsdr drop-in": the SAME names, argument meaning and return values as the reference
 *           library for the hot-path functions, taking HOST pointers and behaving synchronously, so
 *           the reference's own callers (csdr.c, test200.c) link against this library unchanged.
 *           Each prototype cites the reference declaration it replaces (file:line in ha7ilm/csdr @6ef2a742).
 *
 *   Part B  "bank API" (csdrb_*): the device-resident many-channel entry points the reference can only
 *           express as one process chain per channel (ddcd_old.h:51-61).  Pointers named d_* are DEVICE
 *           pointers, h_* are host pointers; `stream` is a cudaStream_t passed as void* (NULL = legacy
 *           default stream).  Calls are asynchronous on that stream unless stated otherwise.
 *
 * Error model: Part A keeps the reference's (no error codes); a CUDA failure prints to stderr and
 * aborts the process, which is the closest equivalent of the reference's behaviour on a fatal fault.
 * Part B returns >= 0 on success (usually an output count) and a negative value on failure;
 * csdrb_last_error() returns the message of the calling thread's last failure.
 * There is NO CPU fallback anywhere: without a usable CUDA device every compute entry point fails.
 */
#ifndef CSDR_B200_H
#define CSDR_B200_H
#include <stdio.h>
#ifdef __cplusplus
extern "C" {
#endif

/* =====================================================================================================
 * Part A -- libcsdr drop-in surface
 * =================================================================================================== */

typedef struct complexf_s { float i; float q; } complexf;                        /* libcsdr.h:46 */
typedef enum window_s { WINDOW_BOXCAR, WINDOW_BLACKMAN, WINDOW_HAMMING } window_t; /* libcsdr.h:70-75 */
#define WINDOW_DEFAULT WINDOW_HAMMING                                             /* libcsdr.h:77 */

/* filter design -- stays on the host, in C (libcsdr.h:85-92; libcsdr.c:57-174) */
void  firdes_lowpass_f(float *output, int length, float cutoff_rate, window_t window);
void  firdes_bandpass_c(complexf *output, int length, float lowcut, float highcut, window_t window);
float firdes_wkernel_blackman(float input);
float firdes_wkernel_hamming(float input);
float firdes_wkernel_boxcar(float input);
window_t firdes_get_window_from_string(char *input);
char *firdes_get_string_from_window(window_t window);
int   firdes_filter_len(float transition_bw);
int   log2n(int x);                                                               /* libcsdr.h:209 */
int   next_pow2(int x);                                                           /* libcsdr.h:210 */

/* sample-format conversion (libcsdr.h:220-227; libcsdr.c:2363-2401) */
void convert_u8_f(unsigned char *input, float *output, int input_size);
void convert_s16_f(short *input, float *output, int input_size);
void convert_i16_f(short *input, float *output, int input_size);
void convert_f_s16(float *input, short *output, int input_size);
void convert_f_i16(float *input, short *output, int input_size);
/* the other sample formats (libcsdr.h:221-223, 228-229; libcsdr.c:2368-2437): HackRF's s8 IQ, rtl_tcp-style u8 out, 24-bit sound cards */
void convert_s8_f(signed char *input, float *output, int input_size);
void convert_f_s8(float *input, signed char *output, int input_size);
void convert_f_u8(float *input, unsigned char *output, int input_size);
void convert_f_s24(float *input, unsigned char *output, int input_size, int bigendian);
void convert_s24_f(unsigned char *input, float *output, int input_size, int bigendian);

/* NCO shift by phasor recursion (libcsdr_gpl.h:26-46; libcsdr_gpl.c:27-52, 81-89, 126-160) */
typedef struct shift_addition_data_s { float sindelta; float cosdelta; float rate; } shift_addition_data_t;
shift_addition_data_t shift_addition_init(float rate);
float shift_addition_cc(complexf *input, complexf *output, int input_size, shift_addition_data_t d, float starting_phase);
/* real input (libcsdr_gpl.h; libcsdr_gpl.c:54-77): output[i] = (cos phi * input[i], sin phi * input[i]), the same phasor recursion and returned phase */
float shift_addition_fc(float *input, complexf *output, int input_size, shift_addition_data_t d, float starting_phase);
typedef struct decimating_shift_addition_status_s { int decimation_remain; float starting_phase; int output_size; } decimating_shift_addition_status_t;
shift_addition_data_t decimating_shift_addition_init(float rate, int decimation);
decimating_shift_addition_status_t decimating_shift_addition_cc(complexf *input, complexf *output, int input_size,
        shift_addition_data_t d, int decimation, decimating_shift_addition_status_t s);

/* decimating FIR (libcsdr.h:104; libcsdr.c:528-549): returns the number of outputs written */
int fir_decimate_cc(complexf *input, complexf *output, int input_size, int decimation, float *taps, int taps_length);

/* FM demodulator (libcsdr.h:95; libcsdr.c:1040-1071): `temp` is accepted and ignored */
complexf fmdemod_quadri_cf(complexf *input, float *output, int input_size, float *temp, complexf last_sample);

/* fractional decimator (libcsdr.h:151-170; libcsdr.c:715-793) */
typedef struct fractional_decimator_ff_s {
    float where; int input_processed; int output_size; int num_poly_points;
    float *poly_precalc_denomiator; float *coeffs_buf; float *filtered_buf;
    int xifirst; int xilast; float rate; float *taps; int taps_length;
} fractional_decimator_ff_t;
fractional_decimator_ff_t fractional_decimator_ff_init(float rate, int num_poly_points, float *taps, int taps_length);
void fractional_decimator_ff(float *input, float *output, int input_size, fractional_decimator_ff_t *d);

/* rational resampler (libcsdr.h:132-140; libcsdr.c:607-673).  The returned state is the reference's: when the input runs out, the index pair
 * of the first output not produced; when the output cap input_size*interpolation/decimation ends the call, the pair of the last output
 * produced (the next call computes it again).  With no output at all the reference leaves the fields uninitialised; here they are
 * {0, 0, last_taps_delay}.  At most 16384 taps; input_size*interpolation must not exceed INT_MAX (the reference's int arithmetic). */
typedef struct rational_resampler_ff_s { int input_processed; int output_size; int last_taps_delay; } rational_resampler_ff_t;
rational_resampler_ff_t rational_resampler_ff(float *input, float *output, int input_size, int interpolation, int decimation, float *taps,
                                              int taps_length, int last_taps_delay);
void rational_resampler_get_lowpass_f(float *output, int output_size, int interpolation, int decimation, window_t window);

/* block AGC (libcsdr.h:118-130; libcsdr.c:944-991) */
typedef struct fastagc_ff_s {
    float *buffer_1; float *buffer_2; float *buffer_input;
    float peak_1; float peak_2; int input_size; float reference; float last_gain;
} fastagc_ff_t;
void fastagc_ff(fastagc_ff_t *input, float *output);

/* AM demodulator, DC block and AGC of the AM / SSB graphs (libcsdr.h:98, 116; libcsdr_gpl.h:37; libcsdr.c:861-873, 920-941;
 * libcsdr_gpl.c:163-260) */
void  amdemod_cf(complexf *input, float *output, int input_size);
float fastdcblock_ff(float *input, float *output, int input_size, float last_dc_level);
float agc_ff(float *input, float *output, int input_size, float reference, float attack_rate, float decay_rate, float max_gain,
             short hang_time, short attack_wait_time, float gain_filter_alpha, float last_gain);

/* BPSK31 receive chain (libcsdr.h:314-336, 340-345; libcsdr.c:1960-2072, 2201-2217, 2319-2333), computed as the reference's -O3 -ffast-math build
 * computes it (DESIGN.md section 7).  simple_agc_cc: *current_gain carries the gain between calls (1.0 at stream start).  dbpsk_decoder_c_u8 keeps
 * the reference's static previous sample as library state (zero at process start).  timing_recovery_cc serves GARDNER and EARLYLATE with
 * |loop_gain * max_error| <= 2; the octave debug output (debug_every_nth >= 0) is not part of this build: such a call prints
 * `libcsdr_b200: timing_recovery_cc failed: ...` and aborts, like any other failing drop-in.  psk31_varicode_decoder_push, one bit per call,
 * is not offered here: the bank csdrb_psk31_varicode_decoder_bank_u8_u8 decodes whole streams. */
void simple_agc_cc(complexf *input, complexf *output, int input_size, float rate, float reference, float max_gain, float *current_gain);
void dbpsk_decoder_c_u8(complexf *input, unsigned char *output, int input_size);
typedef enum timing_recovery_algorithm_e { TIMING_RECOVERY_ALGORITHM_GARDNER, TIMING_RECOVERY_ALGORITHM_EARLYLATE } timing_recovery_algorithm_t;
typedef struct timing_recovery_state_s {
    timing_recovery_algorithm_t algorithm; int decimation_rate; int output_size; int input_processed; int use_q; int debug_phase; int debug_every_nth;
    char *debug_writefiles_path; int last_correction_offset; float earlylate_ratio; float loop_gain; float max_error;
} timing_recovery_state_t;
timing_recovery_state_t timing_recovery_init(timing_recovery_algorithm_t algorithm, int decimation_rate, int use_q, float loop_gain, float max_error,
                                             int debug_every_nth, char *debug_writefiles_path);
void timing_recovery_cc(complexf *input, complexf *output, int input_size, float *timing_error, int *sampled_indexes, timing_recovery_state_t *state);

/* RTTY receive chain (libcsdr.h:278-287; libcsdr.c:1662-1729), computed as the reference's -O3 -ffast-math build computes it (DESIGN.md
 * section 7).  serial_line_decoder_f_u8 serves what the CLI accepts -- databits 1..8, samples_per_bits and stopbits >= 1 -- with
 * 0 <= bit_sampling_width_ratio <= 1 and input_size <= 2^22; other values print `libcsdr_b200: serial_line_decoder_f_u8 failed: ...` and
 * abort, like any other failing drop-in.  rtty_baudot_decoder_lookup and _push, one symbol per call, are not offered here: the bank
 * csdrb_rtty_baudot2ascii_bank_u8_u8 decodes whole streams. */
typedef struct serial_line_s {
    float samples_per_bits; int databits; float stopbits; int output_size; int input_used; float bit_sampling_width_ratio;
} serial_line_t;
void serial_line_decoder_f_u8(serial_line_t *s, float *input, unsigned char *output, int input_size);

/* tone filters (libcsdr.c:2219-2273, 2335-2351).  firdes_add_peak_c computes its taps as the reference's -O3 -ffast-math build does (DESIGN.md
 * section 7): sincosf of the float phase, the window at |(float)(middle - i) * (1/(float)middle)|, the sum of magnitudes in double rounded to
 * float after every tap, the taps scaled by 1/sum.  apply_fir_cc is bit-exact with that build; bfsk_demod_cf sums in source order and lies
 * within the bound of tests/test_tone_emulated.py of it.  Both serve 2 <= taps_length <= 4096 and abort with a message outside it; an
 * input_size below taps_length gives 0 outputs, like the reference. */
void firdes_add_peak_c(complexf *output, int length, float rate, window_t window, int add, int normalize);
int  apply_fir_cc(complexf *input, complexf *output, int input_size, complexf *taps, int taps_length);
int  bfsk_demod_cf(complexf *input, float *output, int input_size, complexf *mark_filter, complexf *space_filter, int taps_length);

/* transmit side (libcsdr.c:579-602, 1180-1192).  fir_interpolate_cc sums each output in the source's tap order, every product and sum rounded
 * (within a float64 per-output bound of the reference build) and returns the reference's count, I outputs per group; tap 0 is never used, as in
 * the reference.  fmmod_fc follows the reference build's phase chain bit for bit and returns the last phase; its samples are within one float
 * ulp of the build's sincosf (DESIGN.md section 7). */
int   fir_interpolate_cc(complexf *input, complexf *output, int input_size, int interpolation, float *taps, int taps_length);
float fmmod_fc(float *input, complexf *output, int input_size, float last_phase);
/* the rest of the library's modulators (libcsdr.c:1139, 1174, 1194): gain_ff and add_dcoffset_cc are bit for bit the reference build;
 * fixed_amplitude_cc is the source's sqrt/division form correctly rounded, within a float64 bound of the build (DESIGN.md section 7).
 * input == output is allowed. */
void  gain_ff(float *input, float *output, int input_size, float gain);
void  add_dcoffset_cc(complexf *input, complexf *output, int input_size);
void  fixed_amplitude_cc(complexf *input, complexf *output, int input_size, float new_amplitude);

/* BPSK31 transmit chain (libcsdr.h:343-347; libcsdr.c:1551-1575, 1772-1808, 1828-1843), the reference's own pipe
 * psk31_varicode_encoder_u8_u8 | differential_encoder_u8_u8 | psk_modulator_u8_c 2 | psk31_interpolate_sine_cc <sps>.  The encoder, the
 * differential codec and the interpolator are bit for bit the reference build.  psk_modulator_u8_c is the float of the double cos/sin of the
 * build's float phase: bit for bit the build for n_psk 2, 4 and 8 with symbols below n_psk, within 2 float ulps of it elsewhere (the build's
 * own scalar and vector paths differ by that much, DESIGN.md section 7). */
void          psk31_varicode_encoder_u8_u8(unsigned char *input, unsigned char *output, int input_size, int output_max_size, int *input_processed,
                                           int *output_size);
unsigned char differential_codec(unsigned char *input, unsigned char *output, int input_size, int encode, unsigned char state);
void          psk_modulator_u8_c(unsigned char *input, complexf *output, int input_size, int n_psk);
complexf      psk31_interpolate_sine_cc(complexf *input, complexf *output, int input_size, int interpolation, complexf last_input);

/* audio tail of the WFM graph, SURVEY 8(f) rank 1 (libcsdr.h:100-105; libcsdr.c:1081-1097, 1130-1137) */
float deemphasis_wfm_ff(float *input, float *output, int input_size, float tau, int sample_rate, float last_output);
void  limit_ff(float *input, float *output, int input_size, float max_amplitude);
/* NFM audio tail (libcsdr.h:106; libcsdr.c:1099-1128, tables predefined.h:56-68): fixed FIR chosen by sample rate
 * (48000, 44100, 11025, 8000); returns the number of outputs = input_size - taps_length, 0 for any other rate */
int   deemphasis_nfm_ff(float *input, float *output, int input_size, int sample_rate);

/* waterfall / audio compression, SURVEY 8(f) rank 4 (ima_adpcm.h:35-41; ima_adpcm.c:95-150): IMA ADPCM, two samples per output byte */
typedef struct ImaState { int index; int previousValue; } ima_adpcm_state_t;
ima_adpcm_state_t encode_ima_adpcm_i16_u8(short *input, unsigned char *output, int input_length, ima_adpcm_state_t state);

/* spectrum side path and shift_unroll, SURVEY 8(f) ranks 3-4 (libcsdr.h:142-149, 199-207; libcsdr.c:1245-1276, 1296-1314, 283-320) */
float *precalculate_window(int size, window_t window);                                   /* host table, malloc'ed like the reference's */
void  apply_window_c(complexf *input, complexf *output, int size, window_t window);
void  apply_precalculated_window_c(complexf *input, complexf *output, int size, float *windowt);
void  apply_precalculated_window_f(float *input, float *output, int size, float *windowt);                 /* host loop, libcsdr.c:1278-1282 */
void  logpower_cf(complexf *input, float *output, int size, float add_db);
void  accumulate_power_cf(complexf *input, float *output, int size);
void  log_ff(float *input, float *output, int size, float add_db);
typedef struct shift_unroll_data_s { float *dsin; float *dcos; float phase_increment; int size; } shift_unroll_data_t;
shift_unroll_data_t shift_unroll_init(float rate, int size);
float shift_unroll_cc(complexf *input, complexf *output, int input_size, shift_unroll_data_t *d, float starting_phase);
/* shift_math (libcsdr.h:171; libcsdr.c:186-209): cos/sin of a float phase advanced by one rounded addition per sample, wrapped to [0, 2*PI] */
float shift_math_cc(complexf *input, complexf *output, int input_size, float rate, float starting_phase);
/* shift_table (libcsdr.h:180-186; libcsdr.c:210-260): cos/sin from a quarter-wave table (host memory, made by shift_table_init).  Index
 * arithmetic as the reference's own build executes it; an index the source would read outside the table is clamped. */
typedef struct shift_table_data_s { float *table; int table_size; } shift_table_data_t;
shift_table_data_t shift_table_init(int table_size);
void  shift_table_deinit(shift_table_data_t table_data);
float shift_table_cc(complexf *input, complexf *output, int input_size, float rate, shift_table_data_t table_data, float starting_phase);
/* shift_addfast (libcsdr.h:189-197; libcsdr.c:307-317, 396-433): recursion advanced once per four samples; only input_size/4*4
 * samples of `output` are written, like the reference */
typedef struct shift_addfast_data_s { float dsin[4]; float dcos[4]; float phase_increment; } shift_addfast_data_t;
shift_addfast_data_t shift_addfast_init(float rate);
float shift_addfast_cc(complexf *input, complexf *output, int input_size, shift_addfast_data_t *d, float starting_phase);

/* FFT abstraction (fft_fftw.h:10-27; fft_fftw.c:6-46).  Callers read ->size/->input/->output directly
 * (libcsdr.c:822-835, fastddc.c:112-116), so the first three members keep the reference layout. */
struct fft_plan_s { int size; void *input; void *output; void *plan; };
#define FFT_PLAN_T struct fft_plan_s
FFT_PLAN_T *make_fft_c2c(int size, complexf *input, complexf *output, int forward, int benchmark);
/* fft_fftw.c:16-24: a forward r2c plan of `size` real points (a power of two, 4..2097152); fft_execute writes size/2 + 1 bins to output */
FFT_PLAN_T *make_fft_r2c(int size, float *input, complexf *output, int benchmark);
void  fft_execute(FFT_PLAN_T *plan);
void  fft_destroy(FFT_PLAN_T *plan);
void *csdrb_fft_malloc(size_t bytes);            /* stands in for the fft_malloc macro (fft_fftw.h:11) */
void  csdrb_fft_free(void *p);
#define fft_malloc csdrb_fft_malloc
#define fft_free   csdrb_fft_free

/* overlap-add FFT filter step (libcsdr.h:211; libcsdr.c:814-849) */
void apply_fir_fft_cc(FFT_PLAN_T *plan, FFT_PLAN_T *plan_inverse, complexf *taps_fft, complexf *last_overlap, int overlap_size);

/* fastddc (fastddc.h:5-29; fastddc.c:38-166) */
typedef struct fastddc_s {
    int pre_decimation; int post_decimation; int taps_length; int taps_min_length; int overlap_length;
    int fft_size; int fft_inv_size; int input_size; int post_input_size;
    float pre_shift; int startbin; int v; int offsetbin; float post_shift; int output_scrape; int scrap;
    shift_addition_data_t dsadata;
} fastddc_t;
int  fastddc_init(fastddc_t *ddc, float transition_bw, int decimation, float shift_rate);
decimating_shift_addition_status_t fastddc_inv_cc(complexf *input, complexf *output, fastddc_t *ddc,
        FFT_PLAN_T *plan_inverse, complexf *taps_fft, decimating_shift_addition_status_t shift_stat);
void fastddc_print(fastddc_t *ddc, char *source);
void fft_swap_sides(complexf *io, int fft_size);

/* =====================================================================================================
 * Part B -- device-resident bank API
 * =================================================================================================== */

const char *csdrb_last_error(void);
const char *csdrb_version(void);
int  csdrb_device_count(void);                   /* < 0 when the CUDA runtime cannot be initialised */
int  csdrb_set_device(int device);
int  csdrb_stream_synchronize(void *stream);
long csdrb_kernel_launches(void);                /* kernels this library has launched so far (per process) */

/* Device memory and streams for hosts that do not want the CUDA headers (the csdr-bankd daemon is plain C on top of these).
 * Copies are asynchronous on `stream` (NULL = the default stream); host buffers should come from csdrb_host_alloc(). */
void *csdrb_device_alloc(size_t bytes);          /* zero-filled; NULL on failure (csdrb_last_error) */
void  csdrb_device_free(void *d_ptr);
void *csdrb_stream_create(void);
void  csdrb_stream_destroy(void *stream);
int csdrb_copy_h2d(void *d_dst, const void *h_src, size_t bytes, void *stream);
int csdrb_copy_d2h(void *h_dst, const void *d_src, size_t bytes, void *stream);
int csdrb_copy_d2d(void *d_dst, const void *d_src, size_t bytes, void *stream);
int csdrb_copy2d_d2d(void *d_dst, size_t dst_pitch_bytes, const void *d_src, size_t src_pitch_bytes, size_t width_bytes, size_t rows, void *stream);
int csdrb_copy2d_d2h(void *h_dst, size_t dst_pitch_bytes, const void *d_src, size_t src_pitch_bytes, size_t width_bytes, size_t rows, void *stream);
int csdrb_copy2d_h2d(void *d_dst, size_t dst_pitch_bytes, const void *h_src, size_t src_pitch_bytes, size_t width_bytes, size_t rows, void *stream);

/* K1 conversions on device buffers (16-byte aligned) */
int csdrb_convert_u8_f(const unsigned char *d_in, float *d_out, long n, void *stream);
int csdrb_convert_s16_f(const short *d_in, float *d_out, long n, void *stream);
int csdrb_convert_f_s16(const float *d_in, short *d_out, long n, void *stream);
/* The other sample formats (libcsdr.c:2368-2437), bit for bit the reference's x86 build, on device buffers (bytes at any
 * address, floats 4-byte aligned); n counts values
 * (an s24 value is 3 bytes).  f32 -> s8/u8/s24 truncate toward zero and keep the low bytes of the int32 as x86's cvttss2si/cvttsd2si give it:
 * out of range wraps, NaN and +-Inf store zeros.  `bigendian` is the reference flag passed straight through; on x86 it selects the opposite
 * order of its name: 0 = most significant byte first, 1 = least significant byte first.  Returns 0; -1 for a null pointer, a misaligned float
 * buffer or n < 0, with nothing launched.  n = 0 does nothing. */
int csdrb_convert_s8_f(const signed char *d_in, float *d_out, long n, void *stream);
int csdrb_convert_f_s8(const float *d_in, signed char *d_out, long n, void *stream);
int csdrb_convert_f_u8(const float *d_in, unsigned char *d_out, long n, void *stream);
int csdrb_convert_s24_f(const unsigned char *d_in, float *d_out, long n, int bigendian, void *stream);
int csdrb_convert_f_s24(const float *d_in, unsigned char *d_out, long n, int bigendian, void *stream);

/* K3 fir_decimate_cc bank: channel c reads d_in + c*in_stride (input_size samples) and writes
 * d_out + c*out_stride; all channels share h_taps (HOST pointer, copied into the launch).
 * Returns outputs per channel = input_size >= T ? (input_size - T)/D + 1 : 0  (reference libcsdr.c:537-547).
 * `variant` < 0 lets the library choose the tiling; >= 0 forces one (bench/tuning only). */
int csdrb_fir_decimate_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels,
                               int input_size, int decimation, const float *h_taps, int taps_length, int variant, void *stream);
int csdrb_fir_bank_variants(void);

/* Same operation on HOST buffers (the end-to-end path): streams the bank through the device in chunks of
 * `chunk_channels` channels (<= 0: automatic) on three streams so H2D, kernel and D2H overlap; synchronous.
 * Page-locked host memory (csdrb_host_alloc) is needed for full PCIe rate. */
int csdrb_fir_decimate_bank_cc_host(const complexf *h_in, long in_stride, complexf *h_out, long out_stride, int channels,
                                    int input_size, int decimation, const float *h_taps, int taps_length, int chunk_channels);
/* page-locked host memory placed on the NUMA node of the current device (CSDRB_NO_NUMA=1: wherever the calling thread happens to run) */
void *csdrb_host_alloc(size_t bytes);
void  csdrb_host_free(void *p);

/* convert_u8_f | fir_decimate_cc fused (libcsdr.c:2363-2366 + :528-549; the front of csdr-fm:41): the bank reads rtl_sdr-style interleaved unsigned 8-bit
 * I,Q -- 2 bytes per sample instead of 8 over HBM and PCIe -- and converts on the way into the FIR tile with the reference's own expression, so the
 * result equals convert_u8_f followed by fir_decimate_cc bit for bit in the conversion and like the cf32 bank in the filter.  in_stride counts
 * SAMPLES between rows.  Fused tilings: d=10 T<=200, d=50 T<=900 with in_stride % 8 == 0 and a 16-byte aligned d_in; other geometries convert into a
 * temporary and run the cf32 bank.  The _host form is the end-to-end call (chunked three-stream pipeline, see above). */
int csdrb_fir_decimate_bank_u8_cc(const unsigned char *d_in, long in_stride, complexf *d_out, long out_stride, int channels,
                                  int input_size, int decimation, const float *h_taps, int taps_length, void *stream);
int csdrb_fir_decimate_bank_u8_host(const unsigned char *h_in, long in_stride, complexf *h_out, long out_stride, int channels,
                                    int input_size, int decimation, const float *h_taps, int taps_length, int chunk_channels);

/* K4 fmdemod_quadri_cf bank: d_last_in[c] is the sample preceding channel c's block (NULL = zeros),
 * d_last_out[c] receives its last sample (may be NULL; must not alias d_last_in). */
int csdrb_fmdemod_quadri_bank_cf(const complexf *d_in, long in_stride, float *d_out, long out_stride, int channels,
                                 int input_size, const complexf *d_last_in, complexf *d_last_out, void *stream);

/* K2 shift_addition_cc bank.  in_stride == 0: every channel shifts the SAME wideband input (ddcd use case).
 * d_params[c] = shift_addition_init(rate_c) computed on the host (bit-exact sin/cos deltas); d_phase_io[c] is the
 * starting phase on entry and the phase to continue from on return.  `chunk` is how the reference caller cuts
 * the stream into shift_addition_cc() calls (the CLI uses 1024, csdr.c:911-918; <= 0 means one call).
 * Scratch: csdrb_shift_addition_bank_scratch_bytes() bytes of device memory. */
size_t csdrb_shift_addition_bank_scratch_bytes(int channels, int input_size, int chunk);
int csdrb_shift_addition_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int input_size,
                                 const shift_addition_data_t *d_params, float *d_phase_io, int chunk,
                                 void *d_scratch, size_t scratch_bytes, void *stream);
/* shift_addition_fc bank: real rows in (d_in + c*in_stride floats; in_stride == 0: every channel shifts the SAME real wideband row, e.g. a
 * direct-sampling receiver's stream), complexf rows out; d_params, d_phase_io, chunk and scratch (csdrb_shift_addition_bank_scratch_bytes) as above.
 * Output and returned phase equal the reference's shift_addition_fc called once per chunk, bit for bit. */
int csdrb_shift_addition_bank_fc(const float *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int input_size,
                                 const shift_addition_data_t *d_params, float *d_phase_io, int chunk,
                                 void *d_scratch, size_t scratch_bytes, void *stream);
int csdrb_decimating_shift_addition_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels,
                                            int input_size, const shift_addition_data_t *d_params, int decimation,
                                            int *d_remain_io, float *d_phase_io, int *d_out_size, void *stream);

/* Fused shared-input DDC / NFM bank = shift_addition_cc(rate_c) | fir_decimate_cc(D, taps) [| fmdemod_quadri_cf] for `channels`
 * channels of ONE wideband block (ddcd_old.h:51-57 as one launch).  d_params / d_phase_io / chunk as in the shift bank, except
 * that chunks are counted on the absolute stream: the block starts `offset` samples into a chunk and d_phase_io[c] is the phase at
 * the START of that chunk; on return it is the phase at the start of the chunk containing sample n_out*decimation, where the caller
 * must start the next block (re-presenting the unconsumed tail exactly like fir_decimate_cc's callers do, csdr.c:1172-1174).
 * demod = 0: d_out is complexf [channels][out_stride] baseband; demod = 1: float [channels][out_stride] discriminator output,
 * d_last_in/d_last_out carry the previous baseband sample per channel (NULL = zeros / not wanted).
 * Served geometries: any even decimation D with M = ceil(taps_length / D) <= 24 and D * MP <= 8000, MP being the smallest of 4, 8, 12, 18, 20, 24
 * >= M (e.g. T = 16 D + 1 up to D = 444, D = 1000 up to M = 8, D = 2 up to 48 taps).  D = 50 up to 850 taps and D = 10 up to 200 taps run their own
 * kernels, every other served geometry one kernel with D as an argument; the outputs follow the same contract either way.
 * Returns outputs per channel, -2 for an odd decimation or a geometry beyond those limits (nothing is launched, d_phase_io is left as it was) -- use
 * the unfused bank calls, or the fastddc overlap-save bank (csdrb_fastddc_fwd_cc with fft_size up to 2^20, csdrb_fastddc_inv_bank_cc with
 * fft_inv_size up to 4096) for very large decimations and long filters, then. */
size_t csdrb_ddc_bank_scratch_bytes(int channels, int input_size, int chunk, int offset);
int csdrb_ddc_bank(const complexf *d_wide, int input_size, int channels, const shift_addition_data_t *d_params, float *d_phase_io,
                   int chunk, int offset, int decimation, const float *h_taps, int taps_length, int demod, void *d_out, long out_stride,
                   const complexf *d_last_in, complexf *d_last_out, void *d_scratch, size_t scratch_bytes, void *stream);
/* The same bank on a REAL wideband stream = shift_addition_fc(rate_c) | fir_decimate_cc(D, taps) [| fmdemod_quadri_cf]: same arguments, served
 * geometries, return codes and scratch size; d_wide is 8-byte aligned (any even sample of a 16-byte aligned buffer; otherwise -1 and a message).
 * On x it gives the complex bank's outputs on x + 0j (equal float values: a zero may differ in sign) and the same carried phases, bit for bit.
 * A station at frequency f of a real stream sampled at fs is tuned with rate -f/fs; +f/fs gives its conjugate (sidebands swapped). */
int csdrb_ddc_bank_f(const float *d_wide, int input_size, int channels, const shift_addition_data_t *d_params, float *d_phase_io,
                     int chunk, int offset, int decimation, const float *h_taps, int taps_length, int demod, void *d_out, long out_stride,
                     const complexf *d_last_in, complexf *d_last_out, void *d_scratch, size_t scratch_bytes, void *stream);

/* Streaming bank object over the fused kernel: owns rates, chunk phases, discriminator history and the position inside the current
 * NCO chunk, so a wideband stream is processed with one call per block; internally the serial phase-chain pre-pass of block k+1 runs on
 * a private stream while the caller's stream executes block k.  Contract of process(): it consumes n_out*decimation samples (the return
 * value is n_out); the next block must start there, i.e. the caller re-presents the unconsumed tail exactly like fir_decimate_cc's
 * callers do (csdr.c:1172-1174).  d_out is float [channels][out_stride] when the bank was created with demod = 1, else complexf.
 * create() serves the geometries csdrb_ddc_bank serves and returns NULL for the others (csdrb_last_error() names the served set). */
typedef struct csdrb_ddc_bank_s csdrb_ddc_bank_t;
csdrb_ddc_bank_t *csdrb_ddc_bank_create(int channels, const float *h_rates, int decimation, const float *h_taps, int taps_length, int demod, int chunk);
void csdrb_ddc_bank_destroy(csdrb_ddc_bank_t *bank);
/* retune one channel; effective from the first sample of the next block.  The phase is continuous across the retune: the bank closes the current NCO
 * chunk at that sample for every channel (a shorter shift_addition_cc call, libcsdr_gpl.c:48-50) and starts a fresh chunk there, like the reference CLI
 * re-initialises between two buffers (csdr.c:897-925) */
int  csdrb_ddc_bank_set_rate(csdrb_ddc_bank_t *bank, int channel, float rate);
int  csdrb_ddc_bank_rechunk(csdrb_ddc_bank_t *bank);                               /* close the NCO chunk at the next block's first sample, rates unchanged */
int  csdrb_ddc_bank_offset(const csdrb_ddc_bank_t *bank);                          /* samples of the current NCO chunk already consumed */
int  csdrb_ddc_bank_process(csdrb_ddc_bank_t *bank, const complexf *d_wide, int input_size, void *d_out, long out_stride, void *stream);
/* the same with a block of real samples (csdrb_ddc_bank_f's kernel and alignment); block contract, set_rate, rechunk and offset as above */
int  csdrb_ddc_bank_process_f(csdrb_ddc_bank_t *bank, const float *d_wide, int input_size, void *d_out, long out_stride, void *stream);

/* The same bank sliced over several GPUs of one node, driven from ONE process (what nmux + one process chain per channel do in the reference,
 * nmux.cpp:246-353, ddcd_old.h:51-57): contiguous channel slices per device, the wideband block goes host -> devices[0] once and on to the other
 * devices by ncclBroadcast (NCCL is loaded with dlopen on first use; a one-device bank never needs it).  submit() only enqueues (H2D, broadcast, slice
 * kernels, D2H of the results) and returns a ticket; collect(ticket) waits for that block.  Up to two blocks may be in flight, so a caller that submits
 * block k+1 before collecting block k has the broadcast of k+1 under the kernels of k.  h_wide / h_out of a submitted block belong to the library until
 * its collect returns (page-locked memory from csdrb_host_alloc for full PCIe rate).  h_out is [channels][out_stride] floats (demod = 1) or complexf.
 * Block contract as for csdrb_ddc_bank_process: a block consumes n_out*decimation samples, the caller re-presents the tail.  devices == NULL: 0..ndev-1.
 * create() serves the (decimation, taps_length) geometries csdrb_ddc_bank serves and returns NULL for the others. */
typedef struct csdrb_multi_bank_s csdrb_multi_bank_t;
csdrb_multi_bank_t *csdrb_multi_bank_create(int ndev, const int *devices, int channels, const float *h_rates, int decimation, const float *h_taps,
                                            int taps_length, int demod, int chunk, int max_block);
void csdrb_multi_bank_destroy(csdrb_multi_bank_t *bank);
int  csdrb_multi_bank_devices(const csdrb_multi_bank_t *bank);
int  csdrb_multi_bank_slice(const csdrb_multi_bank_t *bank, int index, int *device, int *first_channel, int *channels);
int  csdrb_multi_bank_set_rate(csdrb_multi_bank_t *bank, int channel, float rate);
int  csdrb_multi_bank_submit(csdrb_multi_bank_t *bank, const complexf *h_wide, int input_size, void *h_out, long out_stride);
int  csdrb_multi_bank_collect(csdrb_multi_bank_t *bank, int ticket);
int  csdrb_multi_bank_process_host(csdrb_multi_bank_t *bank, const complexf *h_wide, int input_size, void *h_out, long out_stride);   /* submit + collect */

/* audio tail banks: hard limiter (elementwise) and the 1-pole de-emphasis IIR (d_last_io[c] = previous output of channel c) */
int csdrb_limit_ff(const float *d_in, float *d_out, long n, float max_amplitude, void *stream);
int csdrb_deemphasis_wfm_bank_ff(const float *d_in, long in_stride, float *d_out, long out_stride, int channels, int input_size,
                                 float tau, int sample_rate, float *d_last_io, void *stream);
/* WFM audio tail: `fractional_decimator_ff rate 12 | deemphasis_wfm_ff sample_rate tau | convert_f_s16` (README.md:66) per row, run the way the CLI
 * runs it with buffer size B = bufsize:
 *   - the decimator runs calls on exactly B samples from the row's start while B samples remain; each call is the reference loop (12 points,
 *     no prefilter), `where` carried and reduced by input_processed after each call (csdr.c:1510-1522, libcsdr.c:751-793);
 *   - the de-emphasis carry is kept, and a NaN carry restarts from 0 where the audio sample index, counted from stream start, is a multiple of B
 *     (libcsdr.c:1092; Inf is kept); alpha and 1 - alpha as csdrb_deemphasis_wfm_bank_ff computes them;
 *   - s16 as csdrb_convert_f_s16.
 * All rows run in lockstep.  Carried state: *state_io on the host (zeroed at stream start; the call advances it) and d_last_io[c] on the device
 * (0 at stream start).  A call reads n samples of each row at d_in + c*in_stride and consumes the same *consumed_out samples of every row; the
 * caller presents the unconsumed rest (fewer than B) again at the start of each row next time.  Row c's audio goes to d_out + c*out_stride.
 * Returns the s16 samples written per row; csdrb_wfm_audio_bank_outputs gives that count and the consumed samples on the host alone.
 * -1 for bad arguments (channels < 1, n < 0, rate <= 1 or not finite, tau <= 0, sample_rate <= 0, strides below n or the output count, a null or misaligned
 * pointer, a state that is not a stream start and has `where` outside [5, 6]), -2 for a call the CLI cannot run: bufsize <= 12, or a call that
 * would consume no sample or more than bufsize samples (the reference would memmove a negative length); the state is then unchanged. */
typedef struct csdrb_wfm_audio_params_s { float rate; int bufsize; float tau; int sample_rate; } csdrb_wfm_audio_params_t;
typedef struct csdrb_wfm_audio_state_s { float where; long long audio; } csdrb_wfm_audio_state_t;
int csdrb_wfm_audio_bank_outputs(const csdrb_wfm_audio_params_t *params, const csdrb_wfm_audio_state_t *state, int n, int *consumed_out);
int csdrb_wfm_audio_bank_f_s16(const float *d_in, long in_stride, int channels, int n, const csdrb_wfm_audio_params_t *params,
                               csdrb_wfm_audio_state_t *state_io, float *d_last_io, short *d_out, long out_stride, int *consumed_out, void *stream);

/* NFM de-emphasis bank: every row through the fixed FIR of `sample_rate`; returns outputs per row (input_size - taps_length),
 * 0 when the rate has no table.  limit_max > 0 fuses the preceding `limit_ff limit_max` of the NFM graph (README.md:87) into the load.
 * csdrb_deemphasis_nfm_taps() exposes the (host) table: NULL / *taps_length = 0 for an unknown rate. */
int csdrb_deemphasis_nfm_bank_ff(const float *d_in, long in_stride, float *d_out, long out_stride, int channels, int input_size,
                                 int sample_rate, float limit_max, void *stream);
const float *csdrb_deemphasis_nfm_taps(int sample_rate, int *taps_length);
/* the same kernel with caller-supplied (host) taps, taps_length <= 208: out[c][i] = sum_t taps[t] * in[c][i+t], i < input_size - taps_length
 * (e.g. a de-emphasis FIR designed for a sample rate the reference has no table for) */
int csdrb_fir_valid_bank_ff(const float *d_in, long in_stride, float *d_out, long out_stride, int channels, int input_size,
                            const float *taps, int taps_length, float limit_max, void *stream);

/* IMA ADPCM on device rows: d_state_io[r] carries row r's encoder state between calls.  csdrb_compress_fft_adpcm_rows_f_u8 is the waterfall line of
 * csdr.c:1745-1767 for many lines at once: each row of fft_size dB values -> (fft_size + 10) / 2 bytes, encoder state fresh per row. */
int csdrb_encode_ima_adpcm_rows_i16_u8(const short *d_in, long in_stride, unsigned char *d_out, long out_stride, int rows, int input_length,
                                       ima_adpcm_state_t *d_state_io, void *stream);
int csdrb_compress_fft_adpcm_rows_f_u8(const float *d_in, long in_stride, unsigned char *d_out, long out_stride, int rows, int fft_size, void *stream);

/* spectrum side path on device buffers: `rows` frames of `size` values share one window table; power modes as the reference's
 * logpower_cf / accumulate_power_cf (d_out is read-modify-write) / log_ff */
int csdrb_apply_window_rows_c(const complexf *d_in, complexf *d_out, const float *d_window, int size, long rows, void *stream);
int csdrb_logpower_cf(const complexf *d_in, float *d_out, long n, float add_db, void *stream);
int csdrb_accumulate_power_cf(const complexf *d_in, float *d_acc, long n, void *stream);
int csdrb_log_ff(const float *d_in, float *d_out, long n, float add_db, void *stream);
/* Waterfall bank: `fft_cc N E W | logaveragepower_cf ADD_DB N A | fft_exchange_sides_ff N [| compress_fft_adpcm_f_u8 N]` (csdr.c:1569-1715,
 * 1745-1767) on `rows` independent streams in lockstep, any cut of a stream into calls giving the bytes of one call.
 *   framing : with s counted from stream start, frame k is [(k+1)E - N, (k+1)E) for E <= N and [kE, kE + N) for E > N; samples before the
 *             stream are 0.  d_window is precalculate_window(N, W) (device, N floats).
 *   line j  : the bin powers of frames jA .. jA+A-1 summed in frame order from 0.0f, 10*log10 + (float)(add_db - 10*log10(A)), halves swapped;
 *             with compress = 1 each line is then (N + 10) / 2 bytes of compress_fft_adpcm_f_u8 (fresh encoder per line), else N floats.
 * The FFT, power, dB and ADPCM arithmetic are those of csdrb_apply_window_rows_c, csdrb_fft_c2c_batch, csdrb_accumulate_power_cf, csdrb_log_ff and
 * csdrb_compress_fft_adpcm_rows_f_u8, so the bank gives their composition's bytes.  The caller owns the carried state: d_hist_io [rows][N]
 * complexf (the last N samples so far) and d_acc_io [rows][N] floats (the partial line), both zero at stream start, and *state_io (host,
 * {0, 0} at stream start), which the call advances.  Row r's input is n samples at d_in + r*in_stride; its line j of the call lands at
 * (char *)d_out + r*out_stride_bytes + j*line_bytes.  csdrb_spectrum_bank_lines gives the lines a call completes (the same for every row);
 * csdrb_spectrum_bank_scratch_bytes the scratch for one launch of the whole call.  Less scratch is served in several launches, down to one
 * frame per row; the bytes do not change.  Returns the lines written per row; -1 for bad arguments (rows < 1, n < 0, every < 1,
 * averages < 1, a state that does not belong to the parameters, a null or misaligned pointer: input and history 8 bytes, accumulator and
 * window 4, float output and its stride 4, scratch 16; scratch below one frame per row), -2 for fft_size other than a power of two in 2..16384. */
typedef struct csdrb_spectrum_params_s { int fft_size, every, averages, compress; float add_db; } csdrb_spectrum_params_t;
typedef struct csdrb_spectrum_state_s { long long consumed, frames; } csdrb_spectrum_state_t;
long csdrb_spectrum_bank_lines(const csdrb_spectrum_params_t *p, const csdrb_spectrum_state_t *s, long n);
size_t csdrb_spectrum_bank_scratch_bytes(int rows, long n, const csdrb_spectrum_params_t *p);
int csdrb_spectrum_bank_cf(const complexf *d_in, long in_stride, int rows, long n, const float *d_window, const csdrb_spectrum_params_t *p,
                           complexf *d_hist_io, float *d_acc_io, csdrb_spectrum_state_t *state_io, void *d_out, long out_stride_bytes,
                           void *d_scratch, size_t scratch_bytes, void *stream);
/* Real-input waterfall bank: `fft_fc N E W | logaveragepower_cf ADD_DB N A [| compress_fft_adpcm_f_u8 N]` (csdr.c:3414-3498) on `rows` real
 * streams, with the parameters and state structs of the complex bank.  fft_size = N is the number of bins (fft_fc's argument, a power of two in
 * 2..16384); a frame is 2N real samples and n, every and the state count real samples.
 *   framing : frame k is [(k+1)E - 2N, (k+1)E) for E <= 2N; for E > 2N fft_fc skips E - 2N complex samples after each frame (its skip counts
 *             floats but reads complexf items), so frame k is [k(2E - 2N), k(2E - 2N) + 2N).  Samples before the stream are 0.  d_window is
 *             precalculate_window(2N, W) (device, 2N floats).
 *   line j  : bins 0..N-1 of frames jA .. jA+A-1 (no half swap, no Nyquist bin), power summed and converted as in the complex bank; N floats or
 *             (N + 10) / 2 ADPCM bytes.
 * Bits: those of apply_precalculated_window_f -> csdrb_fft_r2c_batch -> csdrb_accumulate_power_cf (A frames) -> csdrb_log_ff
 * [-> csdrb_compress_fft_adpcm_rows_f_u8].  d_hist_io is [rows][2N] floats (zero at stream start), d_acc_io [rows][N] floats.  Any cut into
 * calls and any scratch down to one frame per row give the same bytes.  Returns the lines written per row; -1 for bad arguments (as the complex
 * bank; input, history, accumulator, window and float output 4-byte aligned, scratch 16), -2 for an unsupported fft_size. */
long csdrb_spectrum_bank_lines_f(const csdrb_spectrum_params_t *p, const csdrb_spectrum_state_t *s, long n);
size_t csdrb_spectrum_bank_scratch_bytes_f(int rows, long n, const csdrb_spectrum_params_t *p);
int csdrb_spectrum_bank_f(const float *d_in, long in_stride, int rows, long n, const float *d_window, const csdrb_spectrum_params_t *p,
                          float *d_hist_io, float *d_acc_io, csdrb_spectrum_state_t *state_io, void *d_out, long out_stride_bytes,
                          void *d_scratch, size_t scratch_bytes, void *stream);
/* shift_math_cc bank: d_rates[c] is the plain rate argument; d_phase_io[c] the carried float phase.  The phase chain is sequential over the
 * whole block (one thread per channel walks it), the rotation itself runs fully parallel. */
size_t csdrb_shift_math_bank_scratch_bytes(int channels, int input_size);
int csdrb_shift_math_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int input_size,
                             const float *d_rates, float *d_phase_io, void *d_scratch, size_t scratch_bytes, void *stream);
/* shift_table_cc bank: like the shift_math bank plus the quarter-wave table in DEVICE memory (d_table, table_size floats) */
int csdrb_shift_table_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int input_size,
                              const float *d_rates, float *d_phase_io, const float *d_table, int table_size, void *d_scratch, size_t scratch_bytes,
                              void *stream);
/* shift_addfast_cc bank: d_params[c] = shift_addfast_init(rate_c); one reference call per `chunk` samples (csdr.c:781-791 uses 1024);
 * scratch as for the shift_addition bank (csdrb_shift_addition_bank_scratch_bytes) */
int csdrb_shift_addfast_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int input_size,
                                const shift_addfast_data_t *d_params, float *d_phase_io, int chunk, void *d_scratch, size_t scratch_bytes,
                                void *stream);

/* shift_unroll_cc bank: d_params as for the shift_addition bank (shift_addition_init(rate_c): its .rate is the same 2*rate), tables
 * d_dsin/d_dcos [channels][table_stride] from shift_unroll_init(rate_c, table_size); one reference call per table_size samples */
int csdrb_shift_unroll_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int input_size,
                               const shift_addition_data_t *d_params, const float *d_dsin, const float *d_dcos, long table_stride,
                               int table_size, float *d_phase_io, void *d_scratch, size_t scratch_bytes, void *stream);

/* K5 fractional_decimator_ff bank: d_state[c].where carries the reference's `where`; on return input_processed
 * and output_size are filled like fractional_decimator_ff() fills them (libcsdr.c:789-792). */
typedef struct csdrb_fracdec_state_s { float where; int input_processed; int output_size; } csdrb_fracdec_state_t;
size_t csdrb_fractional_decimator_bank_scratch_bytes(int channels, int input_size, float rate);
int csdrb_fractional_decimator_bank_ff(const float *d_in, long in_stride, float *d_out, long out_stride, int channels, int input_size,
                                       float rate, int num_poly_points, const float *d_taps, int taps_length,
                                       csdrb_fracdec_state_t *d_state, void *d_scratch, size_t scratch_bytes, void *stream);

/* rational_resampler_ff bank: every row resampled by interpolation/decimation with the shared h_taps (HOST pointer, copied on the stream) and
 * one shared last_taps_delay, rows in lockstep.  Each output is summed in the reference's order, so a row equals rational_resampler_ff() on
 * it bit for bit against a strict-IEEE build of the reference source.  Returns outputs per row and writes the reference's returned state
 * (see rational_resampler_ff above) to *h_state_out on the host, computed from the sizes alone: the call stays asynchronous.
 * -1 for invalid arguments (interpolation or decimation < 1, no taps, last_taps_delay outside 0..interpolation-1), -2 for more than
 * 16384 taps or input_size*interpolation > INT_MAX. */
int csdrb_rational_resampler_bank_ff(const float *d_in, long in_stride, float *d_out, long out_stride, int channels, int input_size,
                                     int interpolation, int decimation, const float *h_taps, int taps_length, int last_taps_delay,
                                     rational_resampler_ff_t *h_state_out, void *stream);

/* K6 fastagc_ff bank: nblocks consecutive blocks of `block` samples per channel; d_hist is [channels][2][block]
 * (the reference's buffer_1, buffer_2; zero it at stream start), d_state[c] = {peak_1, peak_2, last_gain}. */
typedef struct csdrb_fastagc_state_s { float peak_1, peak_2, last_gain; } csdrb_fastagc_state_t;
size_t csdrb_fastagc_bank_scratch_bytes(int channels, int nblocks);
int csdrb_fastagc_bank_ff(const float *d_in, long in_stride, float *d_out, long out_stride, int channels, int block, int nblocks,
                          float reference, csdrb_fastagc_state_t *d_state, float *d_hist, void *d_scratch, size_t scratch_bytes, void *stream);

/* fastagc_ff | convert_f_s16 in one pass: d_out is short [channels][out_stride]; everything else as above */
int csdrb_fastagc_bank_f_s16(const float *d_in, long in_stride, short *d_out, long out_stride, int channels, int block, int nblocks,
                             float reference, csdrb_fastagc_state_t *d_state, float *d_hist, void *d_scratch, size_t scratch_bytes, void *stream);

/* AM / SSB receiver blocks (README.md:95, :110), computed as the reference's -O3 -ffast-math build computes them (DESIGN.md section 7).
 *
 * amdemod_cf over n samples (libcsdr.c:861-873): sqrt(i*i + q*q) with the correctly rounded square root. */
int csdrb_amdemod_cf(const complexf *d_in, float *d_out, long n, void *stream);

/* fastdcblock_ff bank (libcsdr.c:920-941, CLI loop csdr.c:952-968): nblocks whole blocks of `block` samples per channel (the caller
 * holds any remainder).  cf32_in = 1: d_in is complexf rows and the bank runs amdemod_cf | fastdcblock_ff; 0: d_in is float rows.
 * Strides count elements of the row's own type.  d_last_dc_io[c] is the reference's last_dc_level (0 at stream start).
 * A block is staged whole in one CTA's shared memory: block <= 49152 samples (an error beyond; so for the drop-in fastdcblock_ff and the CLI). */
int csdrb_fastdcblock_bank_ff(const void *d_in, long in_stride, int cf32_in, float *d_out, long out_stride, int channels, int block, int nblocks,
                              float *d_last_dc_io, void *stream);

/* agc_ff bank (libcsdr_gpl.c:163-260, CLI loop csdr.c:1337-1373): [realpart_cf |] agc_ff [| limit_ff] [| convert_f_s16] over n samples per
 * channel.  agc_ff restarts every `chunk` samples counted from stream start (the CLI's the_bufsize), so a stream cut into bank calls of
 * any sizes gives the bits of one long call.  hang_time and attack_wait_time are taken as the reference's `short`.
 * cf32_in = 1: d_in is complexf rows of which only the real part is read (realpart_cf).  limit_max > 0 applies limit_ff limit_max.
 * s16_out = 1: d_out is short rows (convert_f_s16), else float rows.  A stream starts at d_state[c] = {1.0f, 0, 0, 0, 0}. */
typedef struct csdrb_agc_params_s {
    float reference, attack_rate, decay_rate, max_gain;
    int hang_time, attack_wait_time;
    float gain_filter_alpha;
    int chunk;
} csdrb_agc_params_t;
typedef struct csdrb_agc_state_s { float gain, last_peak; int hang_counter, attack_wait_counter, offset; } csdrb_agc_state_t;
int csdrb_agc_bank_ff(const void *d_in, long in_stride, int cf32_in, void *d_out, long out_stride, int s16_out, int channels, int n,
                      const csdrb_agc_params_t *params, csdrb_agc_state_t *d_state, float limit_max, void *stream);

/* BPSK31 receive chain banks (psk31.cu), one row per channel.
 *
 * simple_agc_cc bank: input_size samples per row; d_gain_io[c] is the reference's current_gain (1.0f at stream start).  Each sample's
 * reference/sqrt(i*i + q*q) is correctly rounded where the reference build uses a vendor-dependent rsqrtss approximation; everything else is the
 * build's arithmetic.  Returns input_size. */
int csdrb_simple_agc_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int input_size, float rate,
                             float reference, float max_gain, float *d_gain_io, void *stream);
/* timing_recovery_cc bank: channel c runs one timing_recovery_cc call over the d_size[c] samples at d_in + c*in_stride + d_start[c] (every
 * d_size[c] <= max_size), bit for bit with the reference build.  d_state[c].last_correction_offset carries the loop between calls (0 at stream
 * start); on return d_state[c] = {last_correction_offset, input_processed, output_size} as the reference fills them.  The next call re-presents
 * the input from input_processed on, like the reference CLI (csdr.c:2621-2636); positions are absolute, so any split of a stream into calls gives
 * the same symbols.  d_out (and d_error, d_indexes when not NULL) are rows of out_stride elements, at least max_size/(decimation/2) + 1 when
 * |loop_gain * max_error| <= 1 (every symbol then advances by decimation/2 or more) and max_size above that (a symbol may not advance); the indexes
 * count from the call's first sample.  Serves algorithm 0 (GARDNER) and 1 (EARLYLATE), decimation > 4 and divisible by 4, -1 otherwise;
 * -2 when |loop_gain * max_error| > 2 (a correction can then move a symbol back, and the reference reads before its input).
 * The output counts are data-dependent: read d_state back to use them.  Returns 0. */
typedef struct csdrb_timing_recovery_params_s { int algorithm, decimation, use_q; float loop_gain, max_error; } csdrb_timing_recovery_params_t;
typedef struct csdrb_timing_recovery_state_s { int last_correction_offset, input_processed, output_size; } csdrb_timing_recovery_state_t;
int csdrb_timing_recovery_bank_cc(const complexf *d_in, long in_stride, const int *d_start, const int *d_size, int max_size, complexf *d_out,
                                  long out_stride, float *d_error, int *d_indexes, int channels, const csdrb_timing_recovery_params_t *params,
                                  csdrb_timing_recovery_state_t *d_state, void *stream);
/* dbpsk_decoder_c_u8 bank: row c holds d_lengths[c] <= input_size samples (d_lengths NULL: input_size each); one output bit per sample.
 * d_last_in[c] is the sample before the row (NULL = zeros), d_last_out[c] receives the row's last sample (d_last_in[c] for an empty row;
 * may be NULL; must not alias d_last_in).  Returns input_size. */
int csdrb_dbpsk_decoder_bank_c_u8(const complexf *d_in, long in_stride, unsigned char *d_out, long out_stride, int channels, int input_size,
                                  const int *d_lengths, const complexf *d_last_in, complexf *d_last_out, void *stream);
/* psk31_varicode_decoder bank: row c holds d_lengths[c] <= input_size bits (bytes, non-zero = 1; d_lengths NULL: input_size each) and is pushed
 * through psk31_varicode_decoder_push (libcsdr.c:1536-1549) bit by bit; the non-zero characters go to the row of d_out in order and their count
 * to d_count[c].  d_hist_io[c] is the decoder's shift register (0 at stream start).  out_stride >= input_size.  Returns 0. */
int csdrb_psk31_varicode_decoder_bank_u8_u8(const unsigned char *d_in, long in_stride, unsigned char *d_out, long out_stride, int channels,
                                            int input_size, const int *d_lengths, unsigned long long *d_hist_io, int *d_count, void *stream);

/* BPSK31 transmit chain banks (psk31_tx.cu), one row per channel.  Row c holds d_lengths[c] <= input_size elements (d_lengths NULL: input_size
 * each), so the encoder's d_output_size can feed the next bank's d_lengths directly.  Refusals return -1 with csdrb_last_error() set, launch
 * nothing and leave every _io array unchanged; an empty row leaves its state or last input unchanged.  Returns 0 on success.
 *
 * psk31_varicode_encoder bank: psk31_varicode_encoder_u8_u8 on each row with output_max_size bits of room; the bits (one byte each, 0 or 1) go
 * to row c of d_out, d_input_processed[c] and d_output_size[c] receive the reference's counts.  out_stride >= output_max_size. */
int csdrb_psk31_varicode_encoder_bank_u8_u8(const unsigned char *d_in, long in_stride, unsigned char *d_out, long out_stride, int channels,
                                            int input_size, const int *d_lengths, int output_max_size, int *d_input_processed, int *d_output_size,
                                            void *stream);
/* differential codec bank: differential_codec(row, encode, d_state_io[c]) per row (0 at stream start); d_state_io[c] receives the state the
 * reference returns (in decode mode the last byte itself).  out_stride >= input_size; d_out must not alias d_in. */
int csdrb_differential_codec_bank_u8_u8(const unsigned char *d_in, long in_stride, unsigned char *d_out, long out_stride, int channels,
                                        int input_size, const int *d_lengths, int encode, unsigned char *d_state_io, void *stream);
/* psk_modulator bank: one complexf per symbol byte, n_psk 1..256 (the CLI's range); the constellation contract of psk_modulator_u8_c above. */
int csdrb_psk_modulator_bank_u8_c(const unsigned char *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int input_size,
                                  const int *d_lengths, int n_psk, void *stream);
/* psk31_interpolate_sine bank: psk31_interpolate_sine_cc per row, interpolation >= 1 outputs per input; d_last_io[c] is the reference's
 * last_input (0 at stream start), replaced by the row's last input.  out_stride >= input_size * interpolation. */
int csdrb_psk31_interpolate_sine_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int input_size,
                                         const int *d_lengths, int interpolation, complexf *d_last_io, void *stream);

/* RTTY receive chain banks (rtty.cu), one row per channel.
 *
 * serial_line_decoder_f_u8 bank: channel c's unconsumed discriminator samples are d_in[c*in_stride + d_start_io[c] .. end) (0 <= d_start_io[c]
 * <= end, one end for all rows).  While at least bufsize of them remain, one serial_line_decoder_f_u8 call (libcsdr.c:1662-1729) runs on
 * exactly bufsize samples from d_start_io[c], bit for bit with the reference build, and d_start_io[c] advances by its input_used: the CLI's
 * memmove-and-refill framing (csdr.c:2517-2527), so a row gives the bytes the CLI gives with the same buffer size, and bufsize = n on rows of
 * n samples is exactly one call.  A call that consumes nothing is where the CLI exits with "got stuck": the row stops there and d_stuck[c] = 1
 * (else 0).  The characters (one byte each) go to row c of d_out in order and their count to d_count[c]; out_stride must hold the most a row
 * can give, end / floor(all_bits * samples_per_bits) + 1 with all_bits = 1 + databits + stopbits (float).  Serves databits 1..8,
 * samples_per_bits in [1, 1e6], stopbits in [1, 1000], 0 <= bit_sampling_width_ratio <= 1 (the CLI uses 0.4) and 1 <= bufsize <= 2^22; -1
 * otherwise.  The counts and positions are data-dependent: read them back to use them.  Returns 0. */
typedef struct csdrb_serial_line_params_s { float samples_per_bits; int databits; float stopbits, bit_sampling_width_ratio; } csdrb_serial_line_params_t;
int csdrb_serial_line_decoder_bank_f_u8(const float *d_in, long in_stride, int end, int *d_start_io, unsigned char *d_out, long out_stride, int *d_count,
                                        int *d_stuck, int channels, const csdrb_serial_line_params_t *params, int bufsize, void *stream);
/* rtty_baudot2ascii bank: row c holds d_lengths[c] <= input_size ITA2 codes (d_lengths NULL: input_size each) and goes through
 * rtty_baudot_decoder_lookup (libcsdr.c:1608-1616) code by code; the non-zero characters go to the row of d_out in order and their count to
 * d_count[c].  d_fig_mode_io[c] is the letters (0) / figures (1) mode, carried between calls (0 at stream start).  out_stride >= input_size.
 * Returns 0. */
int csdrb_rtty_baudot2ascii_bank_u8_u8(const unsigned char *d_in, long in_stride, unsigned char *d_out, long out_stride, int channels, int input_size,
                                       const int *d_lengths, unsigned char *d_fig_mode_io, int *d_count, void *stream);

/* tone filter banks (tone.cu), one row per channel, the taps shared by all rows and on the device.  Row c's input is n complexf at
 * d_in + c*in_stride; it gives the n - taps_length + 1 outputs of the valid convolution (the caller carries the last taps_length - 1 inputs
 * between calls) at d_out + c*out_stride.
 *   apply_fir_bank_cc: apply_fir_cc (libcsdr.c:2261-2273), complexf outputs, bit for bit with the reference build.
 *   bfsk_demod_bank_cf: bfsk_demod_cf (libcsdr.c:2335-2351), float outputs |mark|^2 - |space|^2 of the two tap sets, summed in source order.
 * Both return the outputs per row; -1 for a null or misaligned pointer (complexf 8 bytes, float 4), in_stride < n, out_stride < n - taps_length
 * + 1 or n < taps_length; -2 (nothing launched) for taps_length outside 2..4096. */
int csdrb_apply_fir_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int n, const complexf *d_taps,
                            int taps_length, void *stream);
int csdrb_bfsk_demod_bank_cf(const complexf *d_in, long in_stride, float *d_out, long out_stride, int channels, int n, const complexf *d_mark,
                             const complexf *d_space, int taps_length, void *stream);

/* transmit banks (interpolate.cu), one row per channel.
 *   fir_interpolate_bank_cc: row c is one fir_interpolate_cc call on the n complexf at d_in + c*in_stride with the shared device taps
 *     (interpolation I, taps_length T): output i*I + ip = sum over si of x[i+si]*taps[(I-ip) + si*I] for (I-ip) + si*I < T, I and Q summed
 *     separately in tap order without FMA.  Returns the outputs per row, I*(n - ceil((T-1)/I)) or 0, the reference's count; the caller keeps the
 *     inputs not consumed (n minus the returned count / I) for the next call.  -1 for I < 1, T < 1, a null or misaligned pointer (complexf
 *     8 bytes, taps 4), in_stride < n or out_stride below the row's outputs.
 *   fmmod_bank_fc: row c is fmmod_fc on n floats with the phase d_phase_io[c] carried between calls (0 at stream start); complexf out.
 *     Returns n; -1 for a null or misaligned pointer or strides below n. */
int csdrb_fir_interpolate_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int n, int interpolation,
                                  const float *d_taps, int taps_length, void *stream);
int csdrb_fmmod_bank_fc(const float *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int n, float *d_phase_io, void *stream);

/* amplitude modulator banks (modulate.cu), one row per channel, row c of the input at d_in + c*in_stride and of the output at d_out + c*out_stride
 * (strides in elements).  With fmmod_bank_fc and bandpass_fir_fft_bank_cc they make the reference's transmit pipes: AM `gain_ff G | dsb_fc |
 * add_dcoffset_cc`, DSB `gain_ff G | dsb_fc`, USB/LSB `gain_ff G | dsb_fc | bandpass_fir_fft_cc 0 0.1 0.05` (-0.1 0 0.05), FM `gain_ff G | fmmod_fc`.
 *   gain_bank_ff: gain_ff (libcsdr.c:1139), y = gain*x, bit for bit the reference build.
 *   dsb_bank_fc: the dsb_fc command's loop (csdr.c:2084-2102), y = (x, q_value): a real signal as the I of a complex one.
 *   add_dcoffset_bank_cc: add_dcoffset_cc (libcsdr.c:1174) as the -ffast-math build runs it, y = ((i + 1.0f)*0.5f, q*0.5f) in float, bit for bit.
 *   fixed_amplitude_bank_cc: fixed_amplitude_cc (libcsdr.c:1194), the source's expression correctly rounded: s = i*i + q*q, a = sqrt(s),
 *     g = a > 0 ? new_amplitude/a : 0, y = (i*g, q*g).  The build's rsqrtss seed differs between CPUs; both lie within a float64 bound of
 *     new_amplitude*x/|x| (DESIGN.md section 7).
 * Each returns n; -1 (csdrb_last_error() set, nothing launched) for n < 0, channels < 0, a stride below n, a null pointer with work to do, a
 * misaligned one (complexf 8 bytes, float 4) or d_in == d_out with unequal strides (gain, add_dcoffset, fixed_amplitude: in place with equal
 * strides is allowed; dsb_fc is never in place). */
int csdrb_gain_bank_ff(const float *d_in, long in_stride, float *d_out, long out_stride, int channels, int n, float gain, void *stream);
int csdrb_dsb_bank_fc(const float *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int n, float q_value, void *stream);
int csdrb_add_dcoffset_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int n, void *stream);
int csdrb_fixed_amplitude_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int n, float new_amplitude,
                                  void *stream);

/* Synthesis bank (synth.cu): C baseband channels into ONE wideband stream,
 *     y = sum over c of shift_addition_cc(fir_interpolate_cc(x_c, I, taps), rate_c)
 * with the C upshifted intermediates never in memory.  Per channel the contribution is bit for bit csdrb_fir_interpolate_bank_cc followed by
 * csdrb_shift_addition_bank_cc called once per `chunk` samples, the chunks counted on the absolute stream as in csdrb_ddc_bank: output 0 lies
 * `offset` samples into a chunk, d_phase_io[c] is the phase at the start of that chunk and on return the phase at the start of the chunk that
 * contains output G*I.  d_params[c] = shift_addition_init(rate_c) (host), one set of real taps shared by all channels (tap 0 unused, as in
 * fir_interpolate_cc), row c of the input at d_in + c*in_stride, n inputs per row giving G = n - ceil((T-1)/I) groups (or none).  The channels are
 * summed in a fixed pairwise tree over the channel index, I and Q separately, each add rounded: level 0 pairs channels (2k, 2k+1), the next level
 * those sums, and so on; a node with one present child is that child (C = 3: (Y0 + Y1) + Y2; C = 1: Y0 exactly).  The order depends on C alone.
 *   csdrb_synth_bank_cc returns G*I, the outputs written to d_out; -1 (csdrb_last_error() set, nothing launched, d_phase_io untouched) for I < 1,
 *   T < 1, channels < 1, n < 0, chunk < 1, offset outside [0, chunk), in_stride < n, more than 2^31 - 1 outputs, a null or misaligned pointer
 *   or scratch_bytes below csdrb_synth_bank_scratch_bytes() of the same arguments.
 *   The streaming object owns the rates, the device taps, the phases, the offset and the scratch; process() is csdrb_synth_bank_cc on its state.
 *   Block contract of fir_interpolate_cc: a call on n inputs per channel consumes G of them (returns G*I), and the caller presents the last n - G
 *   again at the front of the next block.  create() returns NULL for bad arguments (csdrb_last_error() set). */
size_t csdrb_synth_bank_scratch_bytes(int channels, int input_size, int interpolation, int taps_length, int chunk, int offset);
int csdrb_synth_bank_cc(const complexf *d_in, long in_stride, int channels, int input_size, int interpolation, const float *d_taps, int taps_length,
                        const shift_addition_data_t *d_params, float *d_phase_io, int chunk, int offset, complexf *d_out, void *d_scratch,
                        size_t scratch_bytes, void *stream);
typedef struct csdrb_synth_bank_s csdrb_synth_bank_t;
csdrb_synth_bank_t *csdrb_synth_bank_create(int channels, const float *h_rates, int interpolation, const float *h_taps, int taps_length, int chunk);
void csdrb_synth_bank_destroy(csdrb_synth_bank_t *bank);
int  csdrb_synth_bank_process(csdrb_synth_bank_t *bank, const complexf *d_in, long in_stride, int input_size, complexf *d_out, void *stream);

/* K7 batched unnormalised c2c DFT (power-of-two size 2..16384), sign -1 forward / +1 inverse */
int csdrb_fft_c2c_batch(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int size, int batch, int inverse, void *stream);
/* The same transform for the sizes above one CTA's shared memory: power-of-two size 32768..1048576 (2^15..2^20), two launches per chunk of
 * 2^21/size transforms (four-step algorithm, csrc/fft_large.cuh), the intermediate in stream-ordered scratch of at most 16 MiB; out of place
 * (d_out must not overlap d_in); the call does not wait for the device.  -1 for any other size (nothing is launched). */
int csdrb_fft_c2c_large_batch(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int size, int batch, int inverse, void *stream);
/* Forward real-to-complex DFT (FFTW's r2c, sign -1): `size` real points per row (a power of two, 4..2097152 = 2^21) -> size/2 + 1 bins, the
 * imaginary parts of bins 0 and size/2 exactly 0.  Rows may start at any float (in_stride in floats, out_stride in complexf); with batch > 1 they
 * must not overlap (in_stride >= size, out_stride >= size/2 + 1).  The size/2-point c2c of the packed pairs x[2n] + i x[2n+1] (single CTA up to
 * 32768 real points, above that the four-step transform of csdrb_fft_c2c_large_batch written into d_out) and a split with a per-size table;
 * out of place; the call does not wait for the device.  -1 for a null pointer, another size or overlapping rows (nothing is launched); 0 for
 * batch <= 0. */
int csdrb_fft_r2c_batch(const float *d_in, long in_stride, complexf *d_out, long out_stride, int size, int batch, void *stream);

/* K9 overlap-add FFT filter bank = bandpass_fir_fft_cc block loop (csdr.c:1872-1883) for many channels.
 * d_taps_fft: FFT of the zero-padded taps (taps_stride 0 = shared); d_tail_io [channels][fft_size] carries the
 * previous block's tail between calls (zero at stream start). nblocks blocks of input_size samples per channel. */
int csdrb_bandpass_fir_fft_bank_cc(const complexf *d_in, long in_stride, complexf *d_out, long out_stride, int channels, int fft_size,
                                   int input_size, int nblocks, const complexf *d_taps_fft, long taps_stride, complexf *d_tail_io, void *stream);

/* fastddc forward step (csdr.c:2288-2299): nblocks x input_size new samples -> nblocks x fft_size bins;
 * d_overlap_io [fft_size - input_size] carries the overlap between calls (zero at stream start).  fft_size is a power of two from 4 to
 * 1048576 (2^20); above 16384 the transform is the four-step one of csdrb_fft_c2c_large_batch (stream-ordered scratch, at most 16 MiB), so
 * fastddc_init geometries up to 131073 taps are served. */
int csdrb_fastddc_fwd_cc(const complexf *d_in, complexf *d_spectra, complexf *d_overlap_io, int fft_size, int input_size, int nblocks, void *stream);

/* K8 fastddc_inv_cc bank: every channel c (its own d_taps_fft + c*fft_size, offsetbin and post-shift NCO) consumes the
 * same nblocks spectra.  d_remain_io/d_phase_io carry decimating_shift_addition_status_t between calls;
 * d_out_total[c] receives the samples written for channel c.  `geometry` is a HOST fastddc_t (fastddc_init). */
typedef struct csdrb_fastddc_chan_s { int offsetbin; float sindelta, cosdelta, rate; } csdrb_fastddc_chan_t;
size_t csdrb_fastddc_inv_bank_scratch_bytes(int channels, int nblocks);
int csdrb_fastddc_inv_bank_cc(const complexf *d_spectra, int nblocks, const complexf *d_taps_fft, const csdrb_fastddc_chan_t *d_chan,
                              int channels, const fastddc_t *geometry, int *d_remain_io, float *d_phase_io, complexf *d_out,
                              long out_stride, int *d_out_total, void *d_scratch, size_t scratch_bytes, void *stream);

/* The same bank as a plan object that OWNS the carried post-shift state (decimating_shift_addition_status_t per channel, fastddc.c:151-165 /
 * libcsdr_gpl.c:154-158) and a fixed nblocks: the data-independent half of run k+1 (state chain, post-shift phasors) is computed on a private
 * stream while run k's IFFT step and the caller's next forward FFT execute, so a run is fold + IFFT only.  Outputs are those of
 * csdrb_fastddc_inv_bank_cc bit for bit.  `chan` is a HOST array; geometries outside the fold path (fft_inv_size 64..1024, even
 * pre-decimation) are refused -- use the stateless call for them.  set_channel retunes one channel from the next run on (replace that
 * channel's row of d_taps_fft on your stream as well); get/set_state read and write the state the NEXT run starts from. */
typedef struct csdrb_fastddc_inv_plan csdrb_fastddc_inv_plan_t;
csdrb_fastddc_inv_plan_t *csdrb_fastddc_inv_plan_create(const csdrb_fastddc_chan_t *chan, int channels, const fastddc_t *geometry, int nblocks);
int csdrb_fastddc_inv_plan_run(csdrb_fastddc_inv_plan_t *plan, const complexf *d_spectra, const complexf *d_taps_fft, complexf *d_out, long out_stride,
                               int *d_out_total, void *stream);
int csdrb_fastddc_inv_plan_set_channel(csdrb_fastddc_inv_plan_t *plan, int channel, const csdrb_fastddc_chan_t *chan);
int csdrb_fastddc_inv_plan_get_state(csdrb_fastddc_inv_plan_t *plan, int *remain, float *phase);
int csdrb_fastddc_inv_plan_set_state(csdrb_fastddc_inv_plan_t *plan, const int *remain, const float *phase);
void csdrb_fastddc_inv_plan_destroy(csdrb_fastddc_inv_plan_t *plan);

#ifdef __cplusplus
}
#endif
#endif
