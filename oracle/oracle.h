/*
 * oracle.h -- CPU restatement of the csdr block-DSP hot path.  TEST INFRASTRUCTURE.
 *
 * This is the checker, not the product: only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs may load it.  The shipped path (csdr_b200/csrc) never
 * calls anything declared here and fails loudly when its CUDA library is missing.
 *
 * Every function restates, in strict IEEE-754 arithmetic (-fno-fast-math, no FMA contraction),
 * the algorithm of the reference function named in its comment (file:line into ha7ilm/csdr @6ef2a742).
 * It is pinned against the compiled, unmodified reference (oracle/_ref/libcsdr_ref.so, built by
 * `make -C oracle ref`) in tests/test_oracle.py and against the committed golden vectors in
 * tests/golden/ (generated from that same compiled reference by tests/golden/make_golden.py).
 *
 * FFT boundary: the reference calls FFTW3f (third-party, absent here; only pinned version anywhere
 * is fftw-3.3.3, reference Makefile:44).  No reference test pins results at that boundary, so the
 * FFT-based rows (apply_fir_fft_cc, fastddc) are "parity unpinned" at the library level: the oracle
 * uses the mathematical DFT evaluated in float64 and rounded to float.
 */
#ifndef CSDR_ORACLE_H
#define CSDR_ORACLE_H
#ifdef __cplusplus
extern "C" {
#endif

typedef struct { float i, q; } ocf32;                     /* libcsdr.h:46 complexf */

enum { ORACLE_WINDOW_BOXCAR = 0, ORACLE_WINDOW_BLACKMAN = 1, ORACLE_WINDOW_HAMMING = 2 };   /* libcsdr.h:70-75 */

/* sample-format conversion: libcsdr.c:2363-2366, 2373-2376, 2390-2398 */
void oracle_convert_u8_f(const unsigned char *in, float *out, int n);
void oracle_convert_s16_f(const short *in, float *out, int n);
void oracle_convert_f_s16(const float *in, short *out, int n);

/* filter design: libcsdr.c:76-90 (windows), 117-125, 127-142, 144-167, 169-174 */
int   oracle_firdes_filter_len(float transition_bw);
float oracle_window(int window, float rate);
void  oracle_firdes_lowpass_f(float *taps, int length, float cutoff_rate, int window);
void  oracle_firdes_bandpass_c(ocf32 *taps, int length, float lowcut, float highcut, int window);
int   oracle_next_pow2(int x);                           /* libcsdr.c next_pow2 */

/* NCO shift by phasor recursion: libcsdr_gpl.c:27-52, 81-89, 126-160 */
typedef struct { float sindelta, cosdelta, rate; } oracle_shift_t;            /* libcsdr_gpl.h:26-31 */
typedef struct { int decimation_remain; float starting_phase; int output_size; } oracle_dshift_status_t; /* :39-44 */
oracle_shift_t oracle_shift_addition_init(float rate);
float oracle_shift_addition_cc(const ocf32 *in, ocf32 *out, int n, oracle_shift_t d, float starting_phase);
oracle_shift_t oracle_decimating_shift_addition_init(float rate, int decimation);
oracle_dshift_status_t oracle_decimating_shift_addition_cc(const ocf32 *in, ocf32 *out, int n, oracle_shift_t d,
                                                          int decimation, oracle_dshift_status_t s);

/* decimating FIR, real taps on complex samples: libcsdr.c:528-549 */
int oracle_fir_decimate_cc(const ocf32 *in, ocf32 *out, int n, int decimation, const float *taps, int taps_length);

/* quadri-correlator FM demodulator: libcsdr.c:1021, 1040-1071 */
ocf32 oracle_fmdemod_quadri_cf(const ocf32 *in, float *out, int n, ocf32 last_sample);

/* fractional decimator (Lagrange, optional FIR prefilter): libcsdr.h:151-168, libcsdr.c:715-793 */
#define ORACLE_FD_MAX_POINTS 64
typedef struct {
    float where; int input_processed; int output_size;
    int num_poly_points, xifirst, xilast;
    float rate; float denom[ORACLE_FD_MAX_POINTS];
    const float *taps; int taps_length;
} oracle_fracdec_t;
void oracle_fractional_decimator_ff_init(oracle_fracdec_t *d, float rate, int num_poly_points,
                                         const float *taps, int taps_length);
void oracle_fractional_decimator_ff(const float *in, float *out, int n, oracle_fracdec_t *d);

/* block AGC with two blocks of look-ahead: libcsdr.h:118-128, libcsdr.c:944-991.
 * hist1/hist2 are the caller-owned delayed blocks (buffer_1/buffer_2); the call rotates their contents. */
typedef struct { float peak_1, peak_2, reference, last_gain; int block; } oracle_fastagc_t;
void oracle_fastagc_ff(oracle_fastagc_t *st, float *hist1, float *hist2, const float *in, float *out);

/* audio tail of the WFM/NFM graphs (SURVEY 8(f) rank 1): libcsdr.c:1081-1097 (1-pole de-emphasis IIR), 1130-1137 (hard limiter) */
float oracle_deemphasis_wfm_ff(const float *in, float *out, int n, float tau, int sample_rate, float last_output);
void  oracle_limit_ff(const float *in, float *out, int n, float max_amplitude);
int   oracle_deemphasis_nfm_ff(const float *in, float *out, int n, const float *taps, int taps_length);   /* libcsdr.c:1101-1128 */

/* spectrum side path + shift_unroll (SURVEY 8(f) ranks 3, 4): libcsdr.c:1245-1276 (windows), 1296-1314 (log power),
 * 283-315 (shift_unroll_init / shift_unroll_cc) */
void  oracle_precalculate_window(float *windowt, int size, int window);
void  oracle_apply_precalculated_window_c(const ocf32 *in, ocf32 *out, int size, const float *windowt);
void  oracle_logpower_cf(const ocf32 *in, float *out, int size, float add_db);
void  oracle_accumulate_power_cf(const ocf32 *in, float *acc, int size);
void  oracle_log_ff(const float *in, float *out, int size, float add_db);
float oracle_shift_unroll_init(float rate, int size, float *dsin, float *dcos);            /* returns phase_increment */
float oracle_shift_unroll_cc(const ocf32 *in, ocf32 *out, int n, const float *dsin, const float *dcos, float phase_increment, float starting_phase);

/* shift_math (SURVEY 8(f) rank 3): libcsdr.c:186-209 */
float oracle_shift_math_cc(const ocf32 *in, ocf32 *out, int n, float rate, float starting_phase);
/* shift_table (SURVEY 8(f) rank 3): libcsdr.c:210-260, pinned to the arithmetic of the reference's -ffast-math build (see oracle.c) */
void  oracle_shift_table_init(float *table, int size);
float oracle_shift_table_cc(const ocf32 *in, ocf32 *out, int n, float rate, const float *table, int table_size, float starting_phase, int *out_of_range);
/* shift_addfast (SURVEY 8(f) rank 3): libcsdr.h:189-197, libcsdr.c:307-317, 396-433.  d9 = dsin[4], dcos[4], phase_increment */
void  oracle_shift_addfast_init(float rate, float *d9);
float oracle_shift_addfast_cc(const ocf32 *in, ocf32 *out, int n, const float *d9, float starting_phase);
/* test helpers of tests/shift_ref.py: the phase chains and the seed phasors of the shift kernels (see oracle.c) */
float oracle_shift_chain(float inc, float phase, int n, int chunk, float *starts);
float oracle_shift_math_phases(float rate, float phase, int n, float *phases);
long  oracle_seed_phasors(const float *ph, long n, float *cs, float *alt, int ulps);

/* waterfall compression (SURVEY 8(f) rank 4): ima_adpcm.c:95-150, csdr.c:1739-1767 */
void oracle_encode_ima_adpcm_i16_u8(const short *in, unsigned char *out, int n, int *index, int *previous);
void oracle_compress_fft_adpcm_f_u8(const float *in, unsigned char *out, int fft_size);

/* mathematical DFT in float64, rounded once to float (stands in for FFTW3f; fft_fftw.c:6-41) */
void oracle_dft_c2c(const ocf32 *in, ocf32 *out, int n, int forward);

/* overlap-add FFT FIR step: libcsdr.c:814-849 (+ block loop csdr.c:1872-1883).
 * in_padded[fft_size] must hold input_size samples followed by zeros; result[fft_size] receives the
 * whole inverse transform with the previous tail added to its first overlap_size samples. */
void oracle_apply_fir_fft_cc(const ocf32 *in_padded, const ocf32 *taps_fft, const ocf32 *last_overlap,
                             int overlap_size, ocf32 *result, int fft_size);

/* fastddc geometry + inverse step: fastddc.h:5-24, fastddc.c:38-72, 91-104, 106-166 */
typedef struct {
    int pre_decimation, post_decimation, taps_length, taps_min_length, overlap_length;
    int fft_size, fft_inv_size, input_size, post_input_size;
    float pre_shift; int startbin, v, offsetbin; float post_shift; int scrap;
    oracle_shift_t dsadata;
} oracle_fastddc_t;
int  oracle_fastddc_init(oracle_fastddc_t *ddc, float transition_bw, int decimation, float shift_rate);
void oracle_fft_swap_sides(ocf32 *io, int fft_size);
/* taps_fft preparation exactly as csdr.c:2342-2351 does it (bandpass taps, zero pad, FFT, swap sides) */
void oracle_fastddc_make_taps_fft(const oracle_fastddc_t *ddc, float shift_rate, int decimation, int window, ocf32 *taps_fft);
/* spectrum[fft_size] is NOT modified (the reference swaps it in place, fastddc.c:123; we work on a copy) */
oracle_dshift_status_t oracle_fastddc_inv_cc(const ocf32 *spectrum, ocf32 *out, const oracle_fastddc_t *ddc,
                                             const ocf32 *taps_fft, oracle_dshift_status_t st);

#ifdef __cplusplus
}
#endif
#endif
