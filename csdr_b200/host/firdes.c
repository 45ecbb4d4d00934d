/*
 * firdes.c -- host-side filter design and geometry helpers of libcsdr_b200 (plain C, no CUDA).
 *
 * These run once at start-up, so they stay on the host exactly where the reference has them
 * (SURVEY.md 8(a) row a5, a11).  Same names, argument meaning and arithmetic promotions as
 *   libcsdr.c:57-174 (windows, firdes_*), :1220-1243 (log2n, next_pow2),
 *   libcsdr_gpl.c:81-89, 126-129 (shift_addition_init, decimating_shift_addition_init),
 *   fastddc.c:38-104 (fastddc_init, fastddc_print, fft_swap_sides).
 * Compiled with -fno-fast-math -ffp-contract=off: promotions below are the C language's, spelled out.
 */
#define _GNU_SOURCE                               /* sincosf */
#include "csdr_b200.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include "nfm_deemph_taps.h"

#define PI_F ((float)3.14159265358979323846)     /* libcsdr.h:65: PI is a float constant */

/* ---- windows (libcsdr.c:57-104) --------------------------------------------------------------- */
window_t firdes_get_window_from_string(char *input)
{
    static const struct { const char *name; window_t w; } table[] = {
        {"BOXCAR", WINDOW_BOXCAR}, {"BLACKMAN", WINDOW_BLACKMAN}, {"HAMMING", WINDOW_HAMMING}};
    for (size_t k = 0; k < sizeof table / sizeof table[0]; k++)
        if (input && !strcmp(input, table[k].name)) return table[k].w;
    return WINDOW_DEFAULT;
}

char *firdes_get_string_from_window(window_t window)
{
    switch (window) {
        case WINDOW_BOXCAR: return "BOXCAR";
        case WINDOW_BLACKMAN: return "BLACKMAN";
        case WINDOW_HAMMING: return "HAMMING";
    }
    return "INVALID";
}

static float remap_unit(float rate) { return (float)(0.5 + (double)(rate / 2)); }   /* [-1,1] -> [0,1] */

float firdes_wkernel_blackman(float rate)
{
    rate = remap_unit(rate);
    return (float)(0.42 - 0.5 * cos((double)(2 * PI_F * rate)) + 0.08 * cos((double)(4 * PI_F * rate)));
}

float firdes_wkernel_hamming(float rate)
{
    rate = remap_unit(rate);
    return (float)(0.54 - 0.46 * cos((double)(2 * PI_F * rate)));
}

float firdes_wkernel_boxcar(float rate) { (void)rate; return 1.0f; }

static float window_value(window_t window, float rate)
{
    if (window == WINDOW_BLACKMAN) return firdes_wkernel_blackman(rate);
    if (window == WINDOW_BOXCAR) return firdes_wkernel_boxcar(rate);
    return firdes_wkernel_hamming(rate);
}

/* ---- FIR design (libcsdr.c:117-174) ------------------------------------------------------------ */
int firdes_filter_len(float transition_bw)
{
    int len = (int)(4.0 / transition_bw);
    return len + (len % 2 == 0);
}

void firdes_lowpass_f(float *output, int length, float cutoff_rate, window_t window)
{
    const int centre = length / 2;
    output[centre] = 2 * PI_F * cutoff_rate * window_value(window, 0);
    for (int d = 1; d <= centre; d++) {
        const double sinc = sin((double)(2 * PI_F * cutoff_rate * d)) / d;
        const float tap = (float)(sinc * (double)window_value(window, (float)d / centre));
        output[centre + d] = tap;
        output[centre - d] = tap;
    }
    float dc_gain = 0;
    for (int k = 0; k < length; k++) dc_gain += output[k];
    for (int k = 0; k < length; k++) output[k] = output[k] / dc_gain;
}

/* rational_resampler_ff's anti-imaging / anti-aliasing lowpass (libcsdr.c:665-673): cutoff at half the lower of 1/I and 1/D */
void rational_resampler_get_lowpass_f(float *output, int output_size, int interpolation, int decimation, window_t window)
{
    const float for_interpolation = (float)(1.0 / interpolation), for_decimation = (float)(1.0 / decimation);
    const float cutoff = for_interpolation < for_decimation ? for_interpolation : for_decimation;
    firdes_lowpass_f(output, output_size, cutoff / 2, window);
}

void firdes_bandpass_c(complexf *output, int length, float lowcut, float highcut, window_t window)
{
    float *prototype = (float *)malloc(sizeof(float) * (size_t)(length > 0 ? length : 1));
    firdes_lowpass_f(prototype, length, (highcut - lowcut) / 2, window);
    const float centre_rate = (highcut + lowcut) / 2;
    float phase = 0;
    for (int k = 0; k < length; k++) {
        const float c = (float)cos((double)phase), s = (float)sin((double)phase);
        phase += 2 * PI_F * centre_rate;
        while (phase > 2 * PI_F) phase -= 2 * PI_F;
        while (phase < 0) phase += 2 * PI_F;
        output[k].i = c * prototype[k];
        output[k].q = s * prototype[k];
    }
    free(prototype);
}

/* ---- peak filter (libcsdr.c:2219-2258) as the reference's -O3 -ffast-math build computes it (DESIGN.md section 7) ----------------------
 * phase steps by (float)((double)-rate * 2pi) in float and wraps against 2pi in double; e_powj becomes sincosf of the float phase; the window
 * takes (float)(middle - i) times the float reciprocal of middle; the magnitudes sqrt((double)(i*i + q*q)) add in double and round to float
 * after every tap; the taps are multiplied by the float reciprocal of that sum. */
void firdes_add_peak_c(complexf *output, int length, float rate, window_t window, int add, int normalize)
{
    const int middle = length / 2;
    const float step = (float)((double)-rate * (2 * M_PI)), inv_middle = 1.0f / (float)middle;
    float phase = 0;
    for (int i = 0; i < length; i++) {
        float c, s;
        sincosf(phase, &s, &c);
        const float w = window_value(window, fabsf((float)(middle - i) * inv_middle));
        if (add) { output[i].i += c * w; output[i].q += s * w; }
        else { output[i].i = c * w; output[i].q = s * w; }
        phase += step;
        while ((double)phase > 2 * M_PI) phase = (float)((double)phase - 2 * M_PI);
        while (phase < 0) phase = (float)((double)phase + 2 * M_PI);
    }
    if (!normalize) return;
    float sum = 0;
    for (int i = 0; i < length; i++) sum = (float)((double)sum + sqrt((double)(output[i].i * output[i].i + output[i].q * output[i].q)));
    const float scale = 1.0f / sum;
    for (int i = 0; i < length; i++) { output[i].i *= scale; output[i].q *= scale; }
}

/* ---- integer helpers (libcsdr.c:1220-1243) ----------------------------------------------------- */
int log2n(int x)
{
    int found = -1;
    for (int b = 0; b < 31; b++)
        if ((x >> b) & 1) { if (found != -1) return -1; found = b; }
    return found;
}

int next_pow2(int x)
{
    for (int b = 0; b < 31; b++) if (x < (1 << b)) return 1 << b;
    return -1;
}

/* ---- NCO parameters (libcsdr_gpl.c:81-89, 126-129) --------------------------------------------- */
shift_addition_data_t shift_addition_init(float rate)
{
    /* One build-flag fact pinned on purpose: under the reference's -ffast-math gcc narrows sin()/cos() of this float argument to a single
     * sincosf() call (seen in every build of libcsdr_gpl.c:84-85).  glibc's sincosf is within an ulp of, but not always equal to, the
     * correctly rounded value (~3 % of rates differ), and the 1024-step phasor recursion turns one ulp in a delta into ~3e-5 of the
     * stream -- so we make the same libm call and get a co-located reference build's deltas bit for bit (tests/test_oracle.py). */
    shift_addition_data_t d;
    rate *= 2;
    sincosf(rate * PI_F, &d.sindelta, &d.cosdelta);
    d.rate = rate;
    return d;
}

shift_addition_data_t decimating_shift_addition_init(float rate, int decimation)
{
    return shift_addition_init(rate * decimation);
}

/* ---- shift_table quarter-wave sine table (libcsdr.c:210-222) ------------------------------------------------------------------ */
shift_table_data_t shift_table_init(int table_size)
{
    shift_table_data_t d;
    d.table_size = table_size;
    d.table = (float *)malloc(sizeof(float) * (size_t)(table_size > 0 ? table_size : 1));
    for (int i = 0; i < table_size; i++) d.table[i] = (float)sin((double)(((float)i / table_size) * (PI_F / 2)));
    return d;
}

void shift_table_deinit(shift_table_data_t table_data) { free(table_data.table); }

/* ---- shift_addfast steps (libcsdr.c:307-317): the phasor after 1..4 increments ---------------------------------- */
shift_addfast_data_t shift_addfast_init(float rate)
{
    shift_addfast_data_t d;
    d.phase_increment = 2 * rate * PI_F;
    for (int k = 0; k < 4; k++) {
        const float angle = d.phase_increment * (k + 1);
        d.dsin[k] = (float)sin((double)angle);
        d.dcos[k] = (float)cos((double)angle);
    }
    return d;
}

/* ---- fixed NFM de-emphasis FIRs (libcsdr.c:1099-1119 picks one by sample rate; tables: nfm_deemph_taps.h) ---------- */
const float *csdrb_deemphasis_nfm_taps(int sample_rate, int *taps_length)
{
    static const struct { int rate; const float *taps; int length; } table[] = {
        {48000, kNfmDeemph48000, (int)(sizeof kNfmDeemph48000 / sizeof(float))},
        {44100, kNfmDeemph44100, (int)(sizeof kNfmDeemph44100 / sizeof(float))},
        {8000, kNfmDeemph8000, (int)(sizeof kNfmDeemph8000 / sizeof(float))},
        {11025, kNfmDeemph11025, (int)(sizeof kNfmDeemph11025 / sizeof(float))}};
    for (size_t k = 0; k < sizeof table / sizeof table[0]; k++)
        if (table[k].rate == sample_rate) { if (taps_length) *taps_length = table[k].length; return table[k].taps; }
    if (taps_length) *taps_length = 0;
    return NULL;
}

/* ---- window table and shift_unroll table (libcsdr.c:1256-1267, 283-299): one-off host work ------------ */
float *precalculate_window(int size, window_t window)
{
    float *table = (float *)malloc(sizeof(float) * (size_t)(size > 0 ? size : 1));
    for (int k = 0; k < size; k++) {
        const float rate = (float)k / (size - 1);
        table[k] = window_value(window, (float)(2.0 * (double)rate + 1.0));
    }
    return table;
}

shift_unroll_data_t shift_unroll_init(float rate, int size)
{
    shift_unroll_data_t d;
    d.phase_increment = 2 * rate * PI_F;
    d.size = size;
    d.dsin = (float *)malloc(sizeof(float) * (size_t)(size > 0 ? size : 1));
    d.dcos = (float *)malloc(sizeof(float) * (size_t)(size > 0 ? size : 1));
    float phase = 0;
    for (int k = 0; k < size; k++) {
        phase += d.phase_increment;
        while (phase > PI_F) phase -= 2 * PI_F;
        while (phase < -PI_F) phase += 2 * PI_F;
        d.dsin[k] = (float)sin((double)phase);
        d.dcos[k] = (float)cos((double)phase);
    }
    return d;
}

/* ---- fastddc geometry (fastddc.c:38-104) ------------------------------------------------------- */
int fastddc_init(fastddc_t *ddc, float transition_bw, int decimation, float shift_rate)
{
    int pre = 1, post = decimation;
    while (post % 2 == 0 && post / 2 != 1) { post /= 2; pre *= 2; }      /* power-of-two part goes to the frequency domain */
    ddc->pre_decimation = pre;
    ddc->post_decimation = post;
    ddc->taps_min_length = firdes_filter_len(transition_bw);
    ddc->taps_length = next_pow2((int)(ceil(ddc->taps_min_length / (float)pre) * pre)) + 1;
    ddc->fft_size = next_pow2(ddc->taps_length * 4);
    while (ddc->fft_size < pre) ddc->fft_size *= 2;
    ddc->overlap_length = ddc->taps_length - 1;
    ddc->input_size = ddc->fft_size - ddc->overlap_length;
    ddc->fft_inv_size = ddc->fft_size / pre;
    ddc->v = ddc->fft_size / ddc->overlap_length;                         /* bin granularity of the coarse shift */
    const int mid = ddc->fft_size / 2;
    ddc->startbin = (int)(mid + mid * (-shift_rate) * 2);
    ddc->startbin = (int)(ddc->v * round(ddc->startbin / (float)ddc->v));
    ddc->offsetbin = ddc->startbin - mid;
    ddc->post_shift = pre * (shift_rate + ((float)ddc->offsetbin / ddc->fft_size));
    ddc->pre_shift = ddc->offsetbin / (float)ddc->fft_size;
    ddc->dsadata = decimating_shift_addition_init(ddc->post_shift, post);
    ddc->output_scrape = 0;
    ddc->scrap = ddc->overlap_length / pre;
    ddc->post_input_size = ddc->fft_inv_size - ddc->scrap;
    return ddc->fft_size <= 2;
}

void fastddc_print(fastddc_t *ddc, char *source)
{
    /* same stderr shape as fastddc.c:75-89 (scripts do not parse it, but drop-in means it looks the same) */
    fprintf(stderr,
            "%s: fastddc_print_sizes(): (fft_size = %d) = (taps_length = %d) + (input_size = %d) - 1\n"
            "  overlap     ::  (overlap_length = %d) = taps_length - 1, taps_min_length = %d\n"
            "  decimation  ::  decimation = (pre_decimation = %d) * (post_decimation = %d), fft_inv_size = %d\n"
            "  shift       ::  startbin = %d, offsetbin = %d, v = %d, pre_shift = %g, post_shift = %g\n"
            "  o&s         ::  post_input_size = %d, scrap = %d\n",
            source, ddc->fft_size, ddc->taps_length, ddc->input_size, ddc->overlap_length, ddc->taps_min_length,
            ddc->pre_decimation, ddc->post_decimation, ddc->fft_inv_size, ddc->startbin, ddc->offsetbin, ddc->v,
            ddc->pre_shift, ddc->post_shift, ddc->post_input_size, ddc->scrap);
}

void fft_swap_sides(complexf *io, int fft_size)
{
    const int half = fft_size / 2;
    for (int k = 0; k < half; k++) { complexf t = io[k]; io[k] = io[k + half]; io[k + half] = t; }
}
