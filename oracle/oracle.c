/*
 * oracle.c -- CPU restatement of the csdr block-DSP hot path.  TEST INFRASTRUCTURE (see oracle.h).
 *
 * Compiled strictly (gcc -O2 -fno-fast-math -ffp-contract=off): every float/double promotion below is
 * deliberate and mirrors the C promotion rules the reference source is subject to.  Comments of the
 * form [ref file:line] name the reference lines each block follows.
 */
#define _GNU_SOURCE                               /* sincosf */
#include "oracle.h"
#include <limits.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

static const float kPi = (float)3.14159265358979323846;          /* [ref libcsdr.h:65] PI is a float */

/* ------------------------------------------------------------------------------------------------
 * sample-format conversion
 * ---------------------------------------------------------------------------------------------- */

/* [ref libcsdr.c:2363-2366] byte -> float; the divide by 127.5 and the -1.0 happen in double. */
void oracle_convert_u8_f(const unsigned char *in, float *out, int n)
{
    for (int k = 0; k < n; k++) {
        double v = (double)(float)in[k];
        out[k] = (float)(v / (UCHAR_MAX / 2.0) - 1.0);
    }
}

/* [ref libcsdr.c:2373-2376] short -> float, `(float)x/SHRT_MAX`.  The reference's own build flags
 * (Makefile:38 -ffast-math) turn the divide into a multiply by the float-rounded reciprocal; that is
 * what every shipped libcsdr does, so it is what we pin (differs from a true divide by 1 ulp on 2.3 %
 * of the 65536 codes; verified bit-exact against oracle/_ref for all of them). */
void oracle_convert_s16_f(const short *in, float *out, int n)
{
    const float recip = 1.0f / (float)SHRT_MAX;
    for (int k = 0; k < n; k++) out[k] = (float)in[k] * recip;
}

/* [ref libcsdr.c:2390-2398] float -> short; single-precision multiply, truncation toward zero.
 * Out-of-range inputs follow what x86 does (cvttss2si to int32, keep the low 16 bits). */
void oracle_convert_f_s16(const float *in, short *out, int n)
{
    for (int k = 0; k < n; k++) {
        float scaled = in[k] * (float)SHRT_MAX;
        int wide = (scaled >= 2147483648.0f || scaled < -2147483648.0f || scaled != scaled) ? INT_MIN : (int)scaled;
        out[k] = (short)(unsigned short)(wide & 0xffff);
    }
}

/* ------------------------------------------------------------------------------------------------
 * filter design
 * ---------------------------------------------------------------------------------------------- */

/* [ref libcsdr.c:169-174] */
int oracle_firdes_filter_len(float transition_bw)
{
    int len = (int)(4.0 / transition_bw);
    return (len % 2 == 0) ? len + 1 : len;
}

/* [ref libcsdr.c:76-96] window kernels; argument in [-1,1] is remapped to [0,1] first. */
float oracle_window(int window, float rate)
{
    if (window == ORACLE_WINDOW_BOXCAR) return 1.0f;
    rate = (float)(0.5 + (double)(rate / 2));
    if (window == ORACLE_WINDOW_BLACKMAN)
        return (float)(0.42 - 0.5 * cos((double)(2 * kPi * rate)) + 0.08 * cos((double)(4 * kPi * rate)));
    return (float)(0.54 - 0.46 * cos((double)(2 * kPi * rate)));     /* HAMMING, also the default */
}

/* [ref libcsdr.c:117-125 normalize_fir_f, 127-142 firdes_lowpass_f] windowed sinc, unity DC gain. */
void oracle_firdes_lowpass_f(float *taps, int length, float cutoff_rate, int window)
{
    int mid = length / 2;
    taps[mid] = 2 * kPi * cutoff_rate * oracle_window(window, 0);
    for (int k = 1; k <= mid; k++) {
        double sinc = sin((double)(2 * kPi * cutoff_rate * k)) / k;
        float t = (float)(sinc * (double)oracle_window(window, (float)k / mid));
        taps[mid - k] = t;
        taps[mid + k] = t;
    }
    float sum = 0;
    for (int k = 0; k < length; k++) sum += taps[k];
    for (int k = 0; k < length; k++) taps[k] = taps[k] / sum;
}

/* [ref libcsdr.c:144-167] real low-pass of half the width, heterodyned to the band centre with a
 * float phase accumulator that is wrapped into [0, 2pi]. */
void oracle_firdes_bandpass_c(ocf32 *taps, int length, float lowcut, float highcut, int window)
{
    float *real_taps = malloc(sizeof(float) * (size_t)length);
    oracle_firdes_lowpass_f(real_taps, length, (highcut - lowcut) / 2, window);
    float centre = (highcut + lowcut) / 2;
    float phase = 0;
    for (int k = 0; k < length; k++) {
        float c = (float)cos((double)phase), s = (float)sin((double)phase);
        phase += 2 * kPi * centre;
        while (phase > 2 * kPi) phase -= 2 * kPi;
        while (phase < 0) phase += 2 * kPi;
        taps[k].i = c * real_taps[k];
        taps[k].q = s * real_taps[k];
    }
    free(real_taps);
}

/* [ref libcsdr.c:1234-1243] smallest power of two strictly greater than x. */
int oracle_next_pow2(int x)
{
    for (int b = 0; b < 31; b++) if (x < (1 << b)) return 1 << b;
    return -1;
}

/* ------------------------------------------------------------------------------------------------
 * NCO shift by phasor recursion
 * ---------------------------------------------------------------------------------------------- */

/* [ref libcsdr_gpl.c:81-89] */
oracle_shift_t oracle_shift_addition_init(float rate)
{
    /* The source says sin(rate*PI) / cos(rate*PI) with a float argument and a float destination; the reference's own build flags
     * (-ffast-math) let gcc narrow that pair to one sincosf() call, which is what every shipped libcsdr executes (objdump of
     * oracle/_ref: `call sincosf@plt`).  sincosf is within an ulp of the double evaluation but differs from it for ~3 % of rates, and the
     * recursion below amplifies one ulp in a delta to ~3e-5 over a 1024-sample call -- so the shipped behaviour is what we pin
     * (verified bit for bit against oracle/_ref over 22 000 rates in tests/test_oracle.py). */
    oracle_shift_t d;
    rate *= 2;
    sincosf(rate * kPi, &d.sindelta, &d.cosdelta);
    d.rate = rate;
    return d;
}

static float wrap_pm_pi(float phase)
{
    while (phase > kPi) phase -= 2 * kPi;
    while (phase < -kPi) phase += 2 * kPi;
    return phase;
}

/* [ref libcsdr_gpl.c:27-52] rotate by a phasor advanced with the angle-addition identities, all in
 * float; the phase returned is advanced arithmetically and wrapped to (-pi, pi]. */
float oracle_shift_addition_cc(const ocf32 *in, ocf32 *out, int n, oracle_shift_t d, float starting_phase)
{
    float c = (float)cos((double)starting_phase), s = (float)sin((double)starting_phase);
    for (int k = 0; k < n; k++) {
        float xi = in[k].i, xq = in[k].q;
        out[k].i = c * xi - s * xq;
        out[k].q = s * xi + c * xq;
        float c_next = c * d.cosdelta - s * d.sindelta;
        float s_next = s * d.cosdelta + c * d.sindelta;
        c = c_next; s = s_next;
    }
    return wrap_pm_pi(starting_phase + d.rate * kPi * n);
}

/* [ref libcsdr_gpl.c:126-129] */
oracle_shift_t oracle_decimating_shift_addition_init(float rate, int decimation)
{
    return oracle_shift_addition_init(rate * decimation);
}

/* [ref libcsdr_gpl.c:131-160] same rotation applied to every decimation-th sample only. */
oracle_dshift_status_t oracle_decimating_shift_addition_cc(const ocf32 *in, ocf32 *out, int n, oracle_shift_t d,
                                                          int decimation, oracle_dshift_status_t st)
{
    float c = (float)cos((double)st.starting_phase), s = (float)sin((double)st.starting_phase);
    int produced = 0, pos;
    for (pos = st.decimation_remain; pos < n; pos += decimation) {
        float xi = in[pos].i, xq = in[pos].q;
        out[produced].i = c * xi - s * xq;
        out[produced].q = s * xi + c * xq;
        produced++;
        float c_next = c * d.cosdelta - s * d.sindelta;
        float s_next = s * d.cosdelta + c * d.sindelta;
        c = c_next; s = s_next;
    }
    st.decimation_remain = pos - n;
    st.starting_phase = wrap_pm_pi(st.starting_phase + d.rate * kPi * produced);
    st.output_size = produced;
    return st;
}

/* ------------------------------------------------------------------------------------------------
 * decimating FIR
 * ---------------------------------------------------------------------------------------------- */

/* [ref libcsdr.c:528-549] one output per `decimation` inputs while a full tap window still fits;
 * I and Q are accumulated separately, taps in ascending order. */
int oracle_fir_decimate_cc(const ocf32 *in, ocf32 *out, int n, int decimation, const float *taps, int taps_length)
{
    int produced = 0;
    for (int start = 0; start < n && start + taps_length <= n; start += decimation) {
        float acc_i = 0, acc_q = 0;
        for (int t = 0; t < taps_length; t++) acc_i += in[start + t].i * taps[t];
        for (int t = 0; t < taps_length; t++) acc_q += in[start + t].q * taps[t];
        out[produced].i = acc_i;
        out[produced].q = acc_q;
        produced++;
    }
    return produced;
}

/* ------------------------------------------------------------------------------------------------
 * FM demodulator
 * ---------------------------------------------------------------------------------------------- */

/* [ref libcsdr.c:1021] */
static const double kQuadriK = 0.340447550238101026565118445432744920253753662109375;

/* [ref libcsdr.c:1040-1071] K*(I*dQ - Q*dI)/(I^2+Q^2); differences against the previous sample
 * (last_sample for the first one); 0 where the power is exactly 0; the final scale/divide is in double. */
ocf32 oracle_fmdemod_quadri_cf(const ocf32 *in, float *out, int n, ocf32 last_sample)
{
    ocf32 prev = last_sample;
    for (int k = 0; k < n; k++) {
        float dq = in[k].q - prev.q;
        float di = in[k].i - prev.i;
        float num = in[k].i * dq - in[k].q * di;
        float den = in[k].i * in[k].i + in[k].q * in[k].q;
        out[k] = den ? (float)(kQuadriK * (double)num / (double)den) : 0;
        prev = in[k];
    }
    return n > 0 ? in[n - 1] : last_sample;
}

/* ------------------------------------------------------------------------------------------------
 * fractional decimator
 * ---------------------------------------------------------------------------------------------- */

/* [ref libcsdr.c:715-748] */
void oracle_fractional_decimator_ff_init(oracle_fracdec_t *d, float rate, int num_poly_points,
                                         const float *taps, int taps_length)
{
    memset(d, 0, sizeof(*d));
    d->num_poly_points = num_poly_points & ~1;
    d->xifirst = -(num_poly_points / 2) + 1;
    d->xilast = num_poly_points / 2;
    int slot = 0;
    for (int xi = d->xifirst; xi <= d->xilast; xi++, slot++) {
        float prod = 1;
        for (int xj = d->xifirst; xj <= d->xilast; xj++)
            if (xi != xj) prod *= (float)(xi - xj);
        d->denom[slot] = prod;
    }
    d->where = (float)(-d->xifirst);
    d->rate = rate;
    d->taps = taps;
    d->taps_length = taps_length;
    d->input_processed = 0;
}

static float fir_dot(const float *x, const float *taps, int len)     /* [ref libcsdr.c fir_one_pass_ff] */
{
    float acc = 0;
    for (int t = 0; t < len; t++) acc += x[t] * taps[t];
    return acc;
}

/* [ref libcsdr.c:751-793] positions advance by a float accumulator; each output is a Lagrange
 * polynomial through num_poly_points neighbours of ceil(where)-1 (optionally FIR-prefiltered). */
void oracle_fractional_decimator_ff(const float *in, float *out, int n, oracle_fracdec_t *d)
{
    int produced = 0, index_high;
    float pts[ORACLE_FD_MAX_POINTS], coef[ORACLE_FD_MAX_POINTS];
    for (; (index_high = (int)ceilf(d->where)) + d->num_poly_points + d->taps_length < n; d->where += d->rate) {
        int low = index_high - 1;
        for (int w = 0; w < d->num_poly_points; w++)
            pts[w] = d->taps ? fir_dot(in + low + w, d->taps, d->taps_length) : in[low + w];
        float x = d->where - (float)low;
        int slot = 0;
        for (int xi = d->xifirst; xi <= d->xilast; xi++, slot++) {
            float prod = 1;
            for (int xj = d->xifirst; xj <= d->xilast; xj++)
                if (xi != xj) prod *= (x - (float)xj);
            coef[slot] = prod;
        }
        float acc = 0;
        for (int w = 0; w < d->num_poly_points; w++) acc += (coef[w] / d->denom[w]) * pts[w];
        out[produced++] = acc;
    }
    d->input_processed = (index_high - 1) + d->xifirst;
    d->where -= (float)d->input_processed;
    d->output_size = produced;
}

/* ------------------------------------------------------------------------------------------------
 * fastagc
 * ---------------------------------------------------------------------------------------------- */

/* [ref libcsdr.c:944-991] gain = reference / max(peak of this and the two previous blocks), capped
 * at 50, ramped linearly from the previous gain across the block that is two calls old. */
void oracle_fastagc_ff(oracle_fastagc_t *st, float *hist1, float *hist2, const float *in, float *out)
{
    int n = st->block;
    float peak_in = 0;
    for (int k = 0; k < n; k++) { float a = fabsf(in[k]); if (a > peak_in) peak_in = a; }
    float peak = peak_in;
    if (peak < st->peak_2) peak = st->peak_2;
    if (peak < st->peak_1) peak = st->peak_1;
    float target = st->reference / peak;
    if (target > 50) target = 50;                                /* FASTAGC_MAX_GAIN */
    for (int k = 0; k < n; k++) {
        float r = (float)k / n;
        float gain = (float)((double)st->last_gain * (1.0 - (double)r) + (double)(target * r));
        out[k] = hist1[k] * gain;
    }
    memcpy(hist1, hist2, sizeof(float) * (size_t)n);             /* buffer_1 <- buffer_2 <- input */
    memcpy(hist2, in, sizeof(float) * (size_t)n);
    st->peak_1 = st->peak_2;
    st->peak_2 = peak_in;
    st->last_gain = target;
}

/* ------------------------------------------------------------------------------------------------
 * audio tail
 * ---------------------------------------------------------------------------------------------- */

/* [ref libcsdr.c:1081-1097] y[i] = alpha*x[i] + (1-alpha)*y[i-1], alpha = dt/(tau+dt), dt = 1/sample_rate; everything in float
 * except the 1.0/sample_rate division; a NaN carry restarts from 0. */
float oracle_deemphasis_wfm_ff(const float *in, float *out, int n, float tau, int sample_rate, float last_output)
{
    float dt = (float)(1.0 / sample_rate);
    float alpha = dt / (tau + dt);
    float keep = 1 - alpha;
    if (last_output != last_output) last_output = 0.0f;
    float y = last_output;
    for (int k = 0; k < n; k++) { y = alpha * in[k] + keep * y; out[k] = y; }
    return n > 0 ? out[n - 1] : last_output;
}

/* [ref libcsdr.c:1101-1128] fixed-FIR NFM de-emphasis: out[i] = sum_t taps[t]*in[i+t] for i < n - taps_length, returns that count.
 * The reference picks `taps` by sample rate from predefined.h:56-68; the oracle takes them as an argument (tests pass the tables
 * read out of the compiled reference / the golden fixture) so that the product's own copy of the tables is checked, not trusted. */
int oracle_deemphasis_nfm_ff(const float *in, float *out, int n, const float *taps, int taps_length)
{
    if (taps_length <= 0) return 0;
    int i;
    for (i = 0; i < n - taps_length; i++) {
        float acc = 0;
        for (int t = 0; t < taps_length; t++) acc += taps[t] * in[i + t];
        out[i] = acc;
    }
    return i;
}

/* [ref libcsdr.c:1130-1137] clamp to +-max_amplitude.  The reference's own build flags (-ffast-math) compile the two selects to
 * minss/maxss, which return the non-NaN operand: a NaN sample leaves as +max_amplitude in every shipped libcsdr (verified against
 * oracle/_ref), so that is what we pin (the strict C expression would pass the NaN through). */
void oracle_limit_ff(const float *in, float *out, int n, float max_amplitude)
{
    for (int k = 0; k < n; k++) {
        float v = (in[k] != in[k]) ? max_amplitude : ((max_amplitude < in[k]) ? max_amplitude : in[k]);
        out[k] = (-max_amplitude > v) ? -max_amplitude : v;
    }
}

/* ------------------------------------------------------------------------------------------------
 * spectrum side path, shift_unroll
 * ---------------------------------------------------------------------------------------------- */

/* [ref libcsdr.c:1256-1267] window table over [-1, 1] mapped as 2*rate+1 with rate = i/(size-1) (the kernels then fold that back). */
void oracle_precalculate_window(float *windowt, int size, int window)
{
    for (int k = 0; k < size; k++) {
        float rate = (float)k / (size - 1);
        windowt[k] = oracle_window(window, (float)(2.0 * (double)rate + 1.0));
    }
}

/* [ref libcsdr.c:1269-1276] */
void oracle_apply_precalculated_window_c(const ocf32 *in, ocf32 *out, int size, const float *windowt)
{
    for (int k = 0; k < size; k++) { out[k].i = in[k].i * windowt[k]; out[k].q = in[k].q * windowt[k]; }
}

/* [ref libcsdr.c:1296-1303] 10*log10(I^2+Q^2) + add_db; the logarithm is the double libm one applied to a float. */
void oracle_logpower_cf(const ocf32 *in, float *out, int size, float add_db)
{
    for (int k = 0; k < size; k++) {
        float p = in[k].i * in[k].i + in[k].q * in[k].q;
        float l = (float)log10((double)p);
        out[k] = 10 * l + add_db;
    }
}

/* [ref libcsdr.c:1305-1308] */
void oracle_accumulate_power_cf(const ocf32 *in, float *acc, int size)
{
    for (int k = 0; k < size; k++) acc[k] += in[k].i * in[k].i + in[k].q * in[k].q;
}

/* [ref libcsdr.c:1310-1314] */
void oracle_log_ff(const float *in, float *out, int size, float add_db)
{
    for (int k = 0; k < size; k++) { float l = (float)log10((double)in[k]); out[k] = 10 * l + add_db; }
}

/* [ref libcsdr.c:283-299] table of the phasor after 1..size steps, built with a float phase accumulator wrapped to (-pi, pi]. */
float oracle_shift_unroll_init(float rate, int size, float *dsin, float *dcos)
{
    float inc = 2 * rate * kPi;
    float ph = 0;
    for (int k = 0; k < size; k++) {
        ph += inc;
        while (ph > kPi) ph -= 2 * kPi;
        while (ph < -kPi) ph += 2 * kPi;
        dsin[k] = (float)sin((double)ph);
        dcos[k] = (float)cos((double)ph);
    }
    return inc;
}

/* [ref libcsdr.c:301-320] every sample is rotated by (start phasor) x (table entry): no recursion, so no error growth inside a call. */
float oracle_shift_unroll_cc(const ocf32 *in, ocf32 *out, int n, const float *dsin, const float *dcos, float phase_increment, float starting_phase)
{
    float c0 = (float)cos((double)starting_phase), s0 = (float)sin((double)starting_phase);
    for (int k = 0; k < n; k++) {
        float c = c0 * dcos[k] - s0 * dsin[k];
        float s = s0 * dcos[k] + c0 * dsin[k];
        out[k].i = c * in[k].i - s * in[k].q;
        out[k].q = s * in[k].i + c * in[k].q;
    }
    return wrap_pm_pi(starting_phase + n * phase_increment);
}

/* [ref libcsdr.c:186-209] shift_math_cc: no recursion at all -- every sample is rotated by cos/sin of a float phase that advances by
 * one rounded addition per sample and is wrapped into [0, 2*PI] with the reference's while loops (2*PI is the float product). */
float oracle_shift_math_cc(const ocf32 *in, ocf32 *out, int n, float rate, float starting_phase)
{
    rate *= 2;
    float phase = starting_phase;
    const float inc = rate * kPi;
    for (int k = 0; k < n; k++) {
        const float c = (float)cos((double)phase), s = (float)sin((double)phase);
        out[k].i = c * in[k].i - s * in[k].q;
        out[k].q = s * in[k].i + c * in[k].q;
        phase += inc;
        while (phase > 2 * kPi) phase -= 2 * kPi;
        while (phase < 0) phase += 2 * kPi;
    }
    return phase;
}

/* [ref libcsdr.c:210-216] quarter-wave sine table: table[i] = sin((i/size) * PI/2), the quotient and product in float, sin in double */
void oracle_shift_table_init(float *table, int size)
{
    for (int i = 0; i < size; i++) table[i] = (float)sin((double)(((float)i / size) * (kPi / 2)));
}

/* [ref libcsdr.c:223-260] shift_table_cc AS THE REFERENCE'S OWN BUILD EXECUTES IT.  The source divides by PI/2 twice; under the Makefile's
 * -ffast-math gcc turns both divisions into multiplications by float constants (objdump of oracle/_ref: mulss by 0x3f22f983 = fl(1/fl(PI/2)),
 * and by fl((float)table_size * that)), and a table index moves the result by 2.4e-5 rad, so the shipped arithmetic is the only thing
 * worth pinning: quadrant = trunc(phase * K), vphase = phase - (float)quadrant * fl(PI/2), index = trunc(vphase * fl(size * K)).
 * The source reads table[size] / table[-1] when rounding pushes an index out of range (it is marked "RTODO"); such samples are reported
 * through *out_of_range (count) and computed with the index clamped, which is what the product does. */
float oracle_shift_table_cc(const ocf32 *in, ocf32 *out, int n, float rate, const float *table, int table_size, float starting_phase, int *out_of_range)
{
    const float K = 0.6366197466850281f;                                /* 0x3f22f983 */
    const float half_pi = kPi / 2;                                       /* 0x3fc90fdb */
    const float K2 = (float)table_size * K;
    float phase = starting_phase;
    const float inc = (rate * 2) * kPi;
    int bad = 0;
    for (int k = 0; k < n; k++) {
        const float qf = phase * K;
        const int quadrant = (int)qf;
        const float whole = (float)quadrant * half_pi;
        const float vphase = phase - whole;
        int sin_index = (int)(vphase * K2);
        int cos_index = table_size - 1 - sin_index;
        if (quadrant & 1) { int t = sin_index; sin_index = cos_index; cos_index = t; }
        if (sin_index < 0 || sin_index >= table_size || cos_index < 0 || cos_index >= table_size) {
            bad++;
            if (sin_index < 0) sin_index = 0; else if (sin_index >= table_size) sin_index = table_size - 1;
            if (cos_index < 0) cos_index = 0; else if (cos_index >= table_size) cos_index = table_size - 1;
        }
        const float sinval = (quadrant > 1 ? -1.0f : 1.0f) * table[sin_index];
        const float cosval = ((quadrant && quadrant < 3) ? -1.0f : 1.0f) * table[cos_index];
        out[k].i = cosval * in[k].i - sinval * in[k].q;
        out[k].q = sinval * in[k].i + cosval * in[k].q;
        phase += inc;
        while (phase > 2 * kPi) phase -= 2 * kPi;
        while (phase < 0) phase += 2 * kPi;
    }
    if (out_of_range) *out_of_range = bad;
    return phase;
}

/* [ref libcsdr.c:307-317] shift_addfast_init: the phasor after 1..4 steps of phase_increment = 2*rate*PI (float), each angle a float
 * product, sin/cos in double rounded to float.  out9 = dsin[4], dcos[4], phase_increment (libcsdr.h:189-194 member order). */
void oracle_shift_addfast_init(float rate, float *out9)
{
    float inc = 2 * rate * kPi;
    for (int k = 0; k < 4; k++) {
        out9[k] = (float)sin((double)(inc * (k + 1)));
        out9[4 + k] = (float)cos((double)(inc * (k + 1)));
    }
    out9[8] = inc;
}

/* [ref libcsdr.c:396-433, the plain-C branch every non-NEON build takes] groups of four samples: each group's four phasors come from
 * the LAST phasor of the previous group times the four fixed steps; the recursion therefore advances once per four samples.  Only
 * input_size/4 groups are touched (a tail of input_size%4 samples is left as it was); the float phase moves by input_size*increment. */
float oracle_shift_addfast_cc(const ocf32 *in, ocf32 *out, int n, const float *d9, float starting_phase)
{
    float c0 = (float)cos((double)starting_phase), s0 = (float)sin((double)starting_phase);
    for (int g = 0; g < n / 4; g++) {
        float c[4], s[4];
        for (int j = 0; j < 4; j++) {
            c[j] = c0 * d9[4 + j] - s0 * d9[j];
            s[j] = s0 * d9[4 + j] + c0 * d9[j];
        }
        for (int j = 0; j < 4; j++) {
            const ocf32 v = in[4 * g + j];
            out[4 * g + j].i = c[j] * v.i - s[j] * v.q;
            out[4 * g + j].q = s[j] * v.i + c[j] * v.q;
        }
        c0 = c[3]; s0 = s[3];
    }
    return wrap_pm_pi(starting_phase + n * d9[8]);
}

/* ------------------------------------------------------------------------------------------------
 * test helpers of the NCO shift checks (tests/shift_ref.py): the project's own restatement, not reference functions
 * ---------------------------------------------------------------------------------------------- */

/* The chunk-to-chunk phase chain of shift_addition_cc, shift_addfast_cc and shift_unroll_cc cut into calls of `chunk` samples (the last
 * one shorter): every call starts at starts[k] and moves the phase by fl(inc * len), wrapped to [-pi, pi] (inc = fl(fl(2 rate) * PI) for
 * all three).  Returns the phase after the last call. */
float oracle_shift_chain(float inc, float phase, int n, int chunk, float *starts)
{
    for (int k = 0, s = 0; s < n; k++, s += chunk) {
        const int len = n - s < chunk ? n - s : chunk;
        starts[k] = phase;
        phase = wrap_pm_pi(phase + inc * len);
    }
    return phase;
}

/* The per-sample phase of shift_math_cc and shift_table_cc: phases[k] is the phase sample k is rotated by.  Returns the carried phase. */
float oracle_shift_math_phases(float rate, float phase, int n, float *phases)
{
    rate *= 2;
    const float inc = rate * kPi;
    for (int k = 0; k < n; k++) {
        phases[k] = phase;
        phase += inc;
        while (phase > 2 * kPi) phase -= 2 * kPi;
        while (phase < 0) phase += 2 * kPi;
    }
    return phase;
}

/* (float)cos((double)ph), (float)sin((double)ph) for n phases, as every shift kernel seeds its phasor: cs[2k], cs[2k+1].  alt[] holds the
 * other float neighbour of a component whose double value lies within `ulps` double ulps of a float rounding midpoint (a libm within a few
 * ulps of this one may round it either way), and the component itself otherwise; returns how many components are that close. */
long oracle_seed_phasors(const float *ph, long n, float *cs, float *alt, int ulps)
{
    long close = 0;
    for (long k = 0; k < 2 * n; k++) {
        const double v = (k & 1) ? sin((double)ph[k >> 1]) : cos((double)ph[k >> 1]);
        const float f = (float)v;
        cs[k] = alt[k] = f;
        if (!isfinite(v) || (double)f == v) continue;
        const float other = nextafterf(f, (double)f < v ? INFINITY : -INFINITY);
        const double mid = ((double)f + (double)other) / 2;                   /* exact: two floats' sum has at most 25 significant bits */
        const double ulp = nextafter(fabs(v), INFINITY) - fabs(v);
        if (fabs(v - mid) <= ulps * ulp) { alt[k] = other; close++; }
    }
    return close;
}

/* ------------------------------------------------------------------------------------------------
 * waterfall compression (SURVEY 8(f) rank 4): IMA ADPCM, 4 bits per value
 * ---------------------------------------------------------------------------------------------- */

/* the IMA/DVI ADPCM standard's two tables (the reference carries the same numbers, ima_adpcm.c:75-93) */
static const int kImaIndexAdjust[8] = {-1, -1, -1, -1, 2, 4, 6, 8};
static const int kImaStep[89] = {7, 8, 9, 10, 11, 12, 13, 14, 16, 17, 19, 21, 23, 25, 28, 31, 34, 37, 41, 45, 50, 55, 60, 66, 73, 80, 88, 97, 107, 118, 130, 143, 157,
    173, 190, 209, 230, 253, 279, 307, 337, 371, 408, 449, 494, 544, 598, 658, 724, 796, 876, 963, 1060, 1166, 1282, 1411, 1552, 1707, 1878, 2066, 2272, 2499, 2749,
    3024, 3327, 3660, 4026, 4428, 4871, 5358, 5894, 6484, 7132, 7845, 8630, 9493, 10442, 11487, 12635, 13899, 15289, 16818, 18500, 20350, 22385, 24623, 27086,
    29794, 32767};

/* [ref ima_adpcm.c:95-139] one sample: quantise the difference to the predictor against the current step (sign + 3 magnitude bits by
 * successive comparison), then move the predictor exactly as a decoder would and adapt the step index. */
static unsigned ima_encode_one(int sample, int *index, int *previous)
{
    const int step = kImaStep[*index];
    int diff = sample - *previous, code = 0, s = step;
    if (diff < 0) { code = 8; diff = -diff; }
    if (diff >= s) { code |= 4; diff -= s; }
    s >>= 1;
    if (diff >= s) { code |= 2; diff -= s; }
    s >>= 1;
    if (diff >= s) code |= 1;
    int delta = step >> 3;
    if (code & 1) delta += step >> 2;
    if (code & 2) delta += step >> 1;
    if (code & 4) delta += step;
    *previous += (code & 8) ? -delta : delta;
    if (*previous > 32767) *previous = 32767; else if (*previous < -32768) *previous = -32768;
    *index += kImaIndexAdjust[code & 7];
    if (*index < 0) *index = 0; else if (*index > 88) *index = 88;
    return (unsigned)code;
}

/* [ref ima_adpcm.c:141-150] two samples per output byte, low nibble first; state = {index, previousValue} in and out */
void oracle_encode_ima_adpcm_i16_u8(const short *in, unsigned char *out, int n, int *index, int *previous)
{
    for (int k = 0; k < n / 2; k++) {
        unsigned lo = ima_encode_one(in[2 * k], index, previous);
        unsigned hi = ima_encode_one(in[2 * k + 1], index, previous);
        out[k] = (unsigned char)(lo | (hi << 4));
    }
}

/* [ref csdr.c:1739-1767] one waterfall line: ten copies of the first value in front (the encoder needs a few samples to settle), dB * 100
 * truncated to short like the C conversion on x86, ADPCM from a fresh state.  out receives (fft_size + 10) / 2 bytes. */
void oracle_compress_fft_adpcm_f_u8(const float *in, unsigned char *out, int fft_size)
{
    enum { PAD = 10 };
    int index = 0, previous = 0;
    short pair[2];
    for (int k = 0; k < (fft_size + PAD) / 2; k++) {
        for (int h = 0; h < 2; h++) {
            const int i = 2 * k + h;
            const float scaled = in[i < PAD ? 0 : i - PAD] * 100;
            const int wide = (scaled >= 2147483648.0f || scaled < -2147483648.0f || scaled != scaled) ? INT_MIN : (int)scaled;
            pair[h] = (short)(unsigned short)(wide & 0xffff);
        }
        unsigned lo = ima_encode_one(pair[0], &index, &previous), hi = ima_encode_one(pair[1], &index, &previous);
        out[k] = (unsigned char)(lo | (hi << 4));
    }
}

/* ------------------------------------------------------------------------------------------------
 * DFT (stands in for FFTW3f)
 * ---------------------------------------------------------------------------------------------- */

static void dft64(double *re, double *im, int n, int sign)
{
    if (n > 0 && (n & (n - 1)) == 0) {
        for (int a = 1, b = 0; a < n; a++) {
            int bit = n >> 1;
            for (; b & bit; bit >>= 1) b ^= bit;
            b ^= bit;
            if (a < b) { double t = re[a]; re[a] = re[b]; re[b] = t; t = im[a]; im[a] = im[b]; im[b] = t; }
        }
        for (int span = 2; span <= n; span <<= 1) {
            int half = span / 2, stride = n / span;
            for (int k = 0; k < half; k++) {
                double ang = sign * 2.0 * M_PI * (double)(k * stride) / (double)n;
                double wr = cos(ang), wi = sin(ang);
                for (int base = 0; base < n; base += span) {
                    int lo = base + k, hi = lo + half;
                    double tr = re[hi] * wr - im[hi] * wi, ti = re[hi] * wi + im[hi] * wr;
                    re[hi] = re[lo] - tr; im[hi] = im[lo] - ti;
                    re[lo] += tr; im[lo] += ti;
                }
            }
        }
        return;
    }
    double *yr = malloc(sizeof(double) * (size_t)n), *yi = malloc(sizeof(double) * (size_t)n);
    for (int k = 0; k < n; k++) {
        double sr = 0, si = 0;
        for (int t = 0; t < n; t++) {
            double ang = sign * 2.0 * M_PI * (double)(((long long)k * t) % n) / (double)n;
            sr += re[t] * cos(ang) - im[t] * sin(ang);
            si += re[t] * sin(ang) + im[t] * cos(ang);
        }
        yr[k] = sr; yi[k] = si;
    }
    memcpy(re, yr, sizeof(double) * (size_t)n); memcpy(im, yi, sizeof(double) * (size_t)n);
    free(yr); free(yi);
}

/* unnormalised DFT, exponent sign -1 when forward, +1 when backward [ref fft_fftw.c:9 FFTW_FORWARD/BACKWARD] */
void oracle_dft_c2c(const ocf32 *in, ocf32 *out, int n, int forward)
{
    double *re = malloc(sizeof(double) * 2 * (size_t)n), *im = re + n;
    for (int k = 0; k < n; k++) { re[k] = in[k].i; im[k] = in[k].q; }
    dft64(re, im, n, forward ? -1 : +1);
    for (int k = 0; k < n; k++) { out[k].i = (float)re[k]; out[k].q = (float)im[k]; }
    free(re);
}

/* ------------------------------------------------------------------------------------------------
 * overlap-add FFT filter
 * ---------------------------------------------------------------------------------------------- */

/* [ref libcsdr.c:814-849] spectrum x taps_fft, inverse, /N, then add the previous block's tail. */
void oracle_apply_fir_fft_cc(const ocf32 *in_padded, const ocf32 *taps_fft, const ocf32 *last_overlap,
                             int overlap_size, ocf32 *result, int fft_size)
{
    ocf32 *spec = malloc(sizeof(ocf32) * (size_t)fft_size);
    oracle_dft_c2c(in_padded, spec, fft_size, 1);
    for (int k = 0; k < fft_size; k++) {
        ocf32 x = spec[k], h = taps_fft[k];
        spec[k].i = x.i * h.i - x.q * h.q;
        spec[k].q = x.i * h.q + x.q * h.i;
    }
    oracle_dft_c2c(spec, result, fft_size, 0);
    for (int k = 0; k < fft_size; k++) { result[k].i /= (float)fft_size; result[k].q /= (float)fft_size; }
    for (int k = 0; k < overlap_size; k++) { result[k].i += last_overlap[k].i; result[k].q += last_overlap[k].q; }
    free(spec);
}

/* ------------------------------------------------------------------------------------------------
 * fastddc
 * ---------------------------------------------------------------------------------------------- */

/* [ref fastddc.c:38-72] */
int oracle_fastddc_init(oracle_fastddc_t *ddc, float transition_bw, int decimation, float shift_rate)
{
    ddc->pre_decimation = 1;
    ddc->post_decimation = decimation;
    while (ddc->post_decimation % 2 == 0 && ddc->post_decimation / 2 != 1) {     /* is_integer(post/2.f) */
        ddc->post_decimation /= 2;
        ddc->pre_decimation *= 2;
    }
    ddc->taps_min_length = oracle_firdes_filter_len(transition_bw);
    ddc->taps_length = oracle_next_pow2((int)(ceil(ddc->taps_min_length / (float)ddc->pre_decimation) * ddc->pre_decimation)) + 1;
    ddc->fft_size = oracle_next_pow2(ddc->taps_length * 4);
    while (ddc->fft_size < ddc->pre_decimation) ddc->fft_size *= 2;
    ddc->overlap_length = ddc->taps_length - 1;
    ddc->input_size = ddc->fft_size - ddc->overlap_length;
    ddc->fft_inv_size = ddc->fft_size / ddc->pre_decimation;
    ddc->v = ddc->fft_size / ddc->overlap_length;
    int middlebin = ddc->fft_size / 2;
    ddc->startbin = (int)(middlebin + middlebin * (-shift_rate) * 2);
    ddc->startbin = (int)(ddc->v * round(ddc->startbin / (float)ddc->v));
    ddc->offsetbin = ddc->startbin - middlebin;
    ddc->post_shift = (ddc->pre_decimation) * (shift_rate + ((float)ddc->offsetbin / ddc->fft_size));
    ddc->pre_shift = ddc->offsetbin / (float)ddc->fft_size;
    ddc->dsadata = oracle_decimating_shift_addition_init(ddc->post_shift, ddc->post_decimation);
    ddc->scrap = ddc->overlap_length / ddc->pre_decimation;
    ddc->post_input_size = ddc->fft_inv_size - ddc->scrap;
    return ddc->fft_size <= 2;
}

/* [ref fastddc.c:91-104] exchange the lower and upper halves (fftshift for even sizes). */
void oracle_fft_swap_sides(ocf32 *io, int fft_size)
{
    int half = fft_size / 2;
    for (int k = 0; k < half; k++) { ocf32 t = io[k]; io[k] = io[k + half]; io[k + half] = t; }
}

/* [ref csdr.c:2342-2351] */
void oracle_fastddc_make_taps_fft(const oracle_fastddc_t *ddc, float shift_rate, int decimation, int window, ocf32 *taps_fft)
{
    ocf32 *taps = calloc((size_t)ddc->fft_size, sizeof(ocf32));
    float half_bw = (float)(0.5 / decimation);
    oracle_firdes_bandpass_c(taps, ddc->taps_length, (-shift_rate) - half_bw, (-shift_rate) + half_bw, window);
    oracle_dft_c2c(taps, taps_fft, ddc->fft_size, 1);
    oracle_fft_swap_sides(taps_fft, ddc->fft_size);
    free(taps);
}

/* [ref fastddc.c:106-166] fold the (centre-swapped) wide spectrum times the filter response into
 * fft_inv_size aliasing bins, scale, un-swap, inverse transform, scale, discard the scrap, then
 * fine-shift and decimate in the time domain. */
oracle_dshift_status_t oracle_fastddc_inv_cc(const ocf32 *spectrum, ocf32 *out, const oracle_fastddc_t *ddc,
                                             const ocf32 *taps_fft, oracle_dshift_status_t st)
{
    int N = ddc->fft_size, M = ddc->fft_inv_size;
    ocf32 *wide = malloc(sizeof(ocf32) * (size_t)N);
    ocf32 *fold = calloc((size_t)M, sizeof(ocf32));
    ocf32 *time = malloc(sizeof(ocf32) * (size_t)M);
    memcpy(wide, spectrum, sizeof(ocf32) * (size_t)N);
    oracle_fft_swap_sides(wide, N);
    for (int b = 0; b < N; b++) {
        int dst = (N + b - ddc->offsetbin + M / 2) % M;
        fold[dst].i += wide[b].i * taps_fft[b].i - wide[b].q * taps_fft[b].q;
        fold[dst].q += wide[b].i * taps_fft[b].q + wide[b].q * taps_fft[b].i;
    }
    for (int b = 0; b < M; b++) { fold[b].i /= (float)ddc->pre_decimation; fold[b].q /= (float)ddc->pre_decimation; }
    oracle_fft_swap_sides(fold, M);
    oracle_dft_c2c(fold, time, M, 0);
    for (int b = 0; b < M; b++) { time[b].i /= (float)M; time[b].q /= (float)M; }
    st = oracle_decimating_shift_addition_cc(time + ddc->scrap, out, ddc->post_input_size, ddc->dsadata,
                                             ddc->post_decimation, st);
    free(wide); free(fold); free(time);
    return st;
}
