/*
 * am_ssb_oracle.c -- CPU restatement of the blocks of the AM and SSB receiver graphs (reference README.md:95, :110).
 * TEST INFRASTRUCTURE: compiled by tests/am_ssb/am_ssb.py into a temporary directory; the product never calls it.
 *
 * Like oracle/oracle.c, every function is plain IEEE-754 single precision (-fno-fast-math -ffp-contract=off).  The
 * reference always builds with -O3 -ffast-math (its Makefile:38), and for agc_ff and fastdcblock_ff that build does not
 * execute the source text: gcc reassociates and vectorises.  These functions restate the arithmetic of the compiled
 * build (read from `objdump -d` of oracle/_ref/libcsdr_ref.so), so that tests/test_oracle_am_ssb.py can pin them bit for
 * bit against that library.
 */
#include <math.h>

/* amdemod_cf, libcsdr.c:861-873: sqrt(i*i + q*q).  Two products and one sum, no FMA.  The reference build takes the square
 * root of its vectorised body with rsqrtps plus one Newton step (vendor-dependent bits); this is the correctly rounded
 * sqrt, which the GPU kernel computes too.  tests/test_oracle_am_ssb.py bounds the distance between the two. */
void am_oracle_amdemod_cf(const float *iq, float *out, int n)
{
    for (int k = 0; k < n; k++) {
        const float i = iq[2 * k], q = iq[2 * k + 1];
        const float ii = i * i, qq = q * q;
        out[k] = sqrtf(ii + qq);
    }
}

/* fastdcblock_ff, libcsdr.c:920-941, as the -O3 -ffast-math build computes it:
 *   sum : n >= 4: four partial sums from 0, lane l adds x[i], i = l (mod 4), i < 4*(n/4), in order; combined (s0+s2)+(s1+s3);
 *         then the n%4 leftover elements one by one.  n <= 3: one sum from 0, in order.
 *   avg = sum / (float)n;  k = (1.0f/(float)n) * (avg - last_dc)
 *   out[i] = (x[i] - last_dc) - (float)i*k,  except the last element of an odd n >= 3 (the scalar epilogue of the
 *   vectorised loop), which is (x[i] - (float)i*k) - last_dc.
 * Returns avg (0 for n <= 0).  in == out is allowed (the CLI works in place, csdr.c:963). */
float am_oracle_fastdcblock_ff(const float *in, float *out, int n, float last_dc)
{
    if (n <= 0) return 0.f;
    float sum;
    if (n >= 4) {
        float s[4] = {0.f, 0.f, 0.f, 0.f};
        const int q = n / 4;
        for (int j = 0; j < q; j++)
            for (int l = 0; l < 4; l++) s[l] = s[l] + in[4 * j + l];
        sum = (s[0] + s[2]) + (s[1] + s[3]);
        for (int i = 4 * q; i < n; i++) sum = sum + in[i];
    } else {
        sum = 0.f;
        for (int i = 0; i < n; i++) sum = sum + in[i];
    }
    const float nf = (float)n;
    const float avg = sum / nf;
    const float k0 = 1.0f / nf;
    const float k = k0 * (avg - last_dc);
    const int odd_tail = (n >= 3 && (n & 1)) ? n - 1 : -1;
    for (int i = 0; i < n; i++) {
        const float ik = (float)i * k;
        out[i] = i == odd_tail ? (in[i] - ik) - last_dc : (in[i] - last_dc) - ik;
    }
    return avg;
}

/* agc_ff, libcsdr_gpl.c:163-260, as the -O3 -ffast-math build computes it (gain and last_gain share one register):
 *   out[0] = last_gain*x[0]; counters 0; last_peak = reference/last_gain
 *   for i >= 1: v = g
 *     x == 0 or NaN (comiss/je): no update
 *     else err = reference/|x| - g
 *       0 > err: reload = |x| > last_peak; last_peak = last_peak > |x| ? last_peak : |x|  (maxss); reload -> awc = attack_wait
 *                awc > 0 ? awc-- : (v = err*attack_rate + g, hc = hang_time)
 *       else   : hc > 0 ? hc-- : v = err*decay_rate + g
 *     t = v < max_gain ? v : max_gain (minss);  t = t > 0 ? t : 0 (maxss)
 *     g = g*(1 - alpha) + t                     ((1 - alpha) rounded once per call)
 *     out[i] = x[i]*g
 * Returns g. */
float am_oracle_agc_ff(const float *in, float *out, int n, float reference, float attack_rate, float decay_rate, float max_gain,
                       short hang_time, short attack_wait_time, float alpha, float last_gain)
{
    if (n <= 0) return last_gain;
    float g = last_gain;
    float last_peak = reference / last_gain;
    const float one_minus_alpha = 1.0f - alpha;
    short hc = 0, awc = 0;
    out[0] = last_gain * in[0];
    for (int i = 1; i < n; i++) {
        const float x = in[i];
        float v = g;
        if (!(x == 0.f || x != x)) {
            const float a = fabsf(x);
            const float err = reference / a - g;
            if (0.f > err) {
                const int reload = a > last_peak;
                last_peak = last_peak > a ? last_peak : a;
                if (reload) awc = attack_wait_time;
                if (awc > 0) awc--;
                else { v = err * attack_rate + g; hc = hang_time; }
            } else {
                if (hc > 0) hc--;
                else v = err * decay_rate + g;
            }
        }
        float t = v < max_gain ? v : max_gain;
        t = t > 0.f ? t : 0.f;
        g = g * one_minus_alpha + t;
        out[i] = x * g;
    }
    return g;
}
