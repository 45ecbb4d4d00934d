/*
 * tone_oracle.c -- CPU restatement of the reference's tone filters (apply_fir_cc, bfsk_demod_cf; libcsdr.c:2261-2273, 2335-2351).
 * TEST INFRASTRUCTURE: compiled by tests/tone/tone.py into a temporary directory; the product never calls it.
 *
 * Plain IEEE-754 arithmetic (-fno-fast-math -ffp-contract=off), in the orders DESIGN.md section 7 fixes for the kernels:
 *   apply_fir_cc as the reference's -O3 -ffast-math build computes it (objdump -d of oracle/_ref/libcsdr_ref.so): `ti` ascending, one
 *     accumulator, re = (x.i*t.i + re) - x.q*t.q and im = im + (x.i*t.q + t.i*x.q);
 *   bfsk_demod_cf in source order, since that build vectorises the `ti` sum: re += x.i*t.i - x.q*t.q, im += x.i*t.q + t.i*x.q, then
 *     -(s.i*s.i + s.q*s.q) + (m.i*m.i + m.q*m.q).
 */
typedef struct { float i, q; } cf;

/* n inputs -> n - L + 1 outputs (none when n < L); returns the output count */
int tone_oracle_apply_fir_cc(const cf *x, cf *out, int n, const cf *t, int L)
{
    int k;
    for (k = 0; k < n - L + 1; k++) {
        float re = 0.f, im = 0.f;
        for (int ti = 0; ti < L; ti++) {
            const cf a = x[k + ti], b = t[ti];
            re = (a.i * b.i + re) - a.q * b.q;
            im = im + (a.i * b.q + b.i * a.q);
        }
        out[k].i = re; out[k].q = im;
    }
    return k;
}

int tone_oracle_bfsk_demod_cf(const cf *x, float *out, int n, const cf *mark, const cf *space, int L)
{
    int k;
    for (k = 0; k < n - L + 1; k++) {
        float mi = 0.f, mq = 0.f, si = 0.f, sq = 0.f;
        for (int ti = 0; ti < L; ti++) {
            const cf a = x[k + ti], m = mark[ti], s = space[ti];
            mi += a.i * m.i - a.q * m.q;
            mq += a.i * m.q + m.i * a.q;
            si += a.i * s.i - a.q * s.q;
            sq += a.i * s.q + s.i * a.q;
        }
        out[k] = -(si * si + sq * sq) + (mi * mi + mq * mq);
    }
    return k;
}
