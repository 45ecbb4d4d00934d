/*
 * real_oracle.c -- CPU restatement of shift_addition_fc, the NCO shift of a REAL input (libcsdr_gpl.c:54-77), for the tests of the real-input
 * banks.  Strict IEEE float: compiled with -fno-fast-math -ffp-contract=off, so every product and sum below is one rounding, as in the reference's
 * x86 build.  The deltas come from oracle_shift_addition_init (oracle/oracle.c), passed in as a struct of the same layout.
 */
#define _GNU_SOURCE
#include <math.h>

typedef struct { float i, q; } real_oracle_cf32;
typedef struct { float sindelta, cosdelta, rate; } real_oracle_shift;

static const float kPi = 3.14159265358979323846f;       /* the reference's PI, a float */

/* one call: the phasor starts at (cos, sin) of the float phase and advances by the angle-addition identities, each product rounded on its own;
 * the sample is x times the phasor.  The returned phase moves on by rate*PI*n and is wrapped into [-pi, pi].
 * build_seed = 0: the seed is cos/sin evaluated in double, as the source writes it (and as the reference's shift_addition_cc runs);
 * build_seed = 1: one sincosf() of the float phase, what the reference's -ffast-math build of shift_addition_fc calls instead */
float oracle_shift_addition_fc(const float *in, real_oracle_cf32 *out, int n, real_oracle_shift d, float starting_phase, int build_seed)
{
    float c, s;
    if (build_seed) sincosf(starting_phase, &s, &c);
    else { c = (float)cos((double)starting_phase); s = (float)sin((double)starting_phase); }
    for (int k = 0; k < n; k++) {
        const float x = in[k];
        out[k].i = c * x;
        out[k].q = s * x;
        const float cn = c * d.cosdelta - s * d.sindelta;
        const float sn = s * d.cosdelta + c * d.sindelta;
        c = cn;
        s = sn;
    }
    float ph = starting_phase + d.rate * kPi * (float)n;
    while (ph > kPi) ph -= 2 * kPi;
    while (ph < -kPi) ph += 2 * kPi;
    return ph;
}
