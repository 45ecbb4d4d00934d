/* psk31_rates.c -- the rate table of psk31_interpolate_sine_cc as the reference's -O3 -ffast-math build computes it (libcsdr.c:1793-1808, its
 * disassembly): rec = 1.0f/(float)I, x = (float)(j+1)*rec, then in double sin(x*M_PI - M_PI/2), + 1.0, * 0.5, rounded to float.  The build's
 * vectorised loop takes j in pairs from 0 through glibc's libmvec _ZGVbN2v_sin and an odd last j through libm's sin.  libmvec's sin is not
 * correctly rounded, and near r = 0 the rounding of sin shows in the float: for 72 of the I in 1..8192 (the first is 1560) libm's sin gives another
 * table.  So the table is computed here, on the host, with the functions the build calls (tests/test_gpu_psk31_tx.py checks every I up to 8192). */
#define _GNU_SOURCE
#include <dlfcn.h>
#include <emmintrin.h>
#include <math.h>

typedef __m128d (*vsin_t)(__m128d);

static double arg(int j, float rec) { const float x = (float)(j + 1) * rec; return (double)x * M_PI - M_PI / 2; }
static float rate_of(double s) { return (float)((s + 1.0) * 0.5); }

/* rates[0..I-1]; 0, or -1 when libmvec cannot be loaded */
int csdrb_psk31_sine_rates(int I, float *rates)
{
    static vsin_t vsin = 0;
    if (!vsin) {
        void *h = dlopen("libmvec.so.1", RTLD_NOW | RTLD_LOCAL);
        vsin = h ? (vsin_t)dlsym(h, "_ZGVbN2v_sin") : 0;
        if (!vsin) return -1;
    }
    const float rec = 1.0f / (float)I;
    int j = 0;
    for (; j + 1 < I; j += 2) {
        double o[2];
        _mm_storeu_pd(o, vsin(_mm_set_pd(arg(j + 1, rec), arg(j, rec))));
        rates[j] = rate_of(o[0]);
        rates[j + 1] = rate_of(o[1]);
    }
    for (; j < I; j++) rates[j] = rate_of(sin(arg(j, rec)));
    return 0;
}
