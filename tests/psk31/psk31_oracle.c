/*
 * psk31_oracle.c -- CPU restatement of the BPSK31 receive chain (simple_agc_cc, timing_recovery_cc, dbpsk_decoder_c_u8,
 * psk31_varicode_decoder_push).  TEST INFRASTRUCTURE: compiled by tests/psk31/psk31.py into a temporary directory; the product never calls it.
 *
 * Plain IEEE-754 single precision (-fno-fast-math -ffp-contract=off), restating the arithmetic of the reference's -O3 -ffast-math build as
 * read from `objdump -d` of oracle/_ref/libcsdr_ref.so (DESIGN.md section 7), so that tests/test_oracle_psk31.py can pin it against that
 * library.  The one deliberate difference: simple_agc_cc's reference/sqrt(s) is correctly rounded here, where the build uses rsqrtss and a
 * Newton step.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>

/* simple_agc_cc, libcsdr.c:2201-2217 */
void psk31_oracle_simple_agc_cc(const float *iq, float *out, int n, float rate, float reference, float max_gain, float *gain)
{
    const float one_minus_rate = 1.0f - rate;
    float g = *gain;
    for (int k = 0; k < n; k++) {
        const float i = iq[2 * k], q = iq[2 * k + 1];
        const float ii = i * i, qq = q * q, s = ii + qq;
        float ideal;
        if (s >= 1.17549435e-38f && s <= 3.40282347e38f) { const float r = sqrtf(s); ideal = reference / r; }
        else ideal = max_gain;                                   /* rsqrtss + Newton gives NaN for 0, subnormal, Inf, NaN; minss picks max_gain */
        ideal = ideal < max_gain ? ideal : max_gain;
        ideal = ideal > 0.f ? ideal : 0.f;
        const float a = (ideal - g) * rate, b = g * one_minus_rate;
        g = a + b;
        out[2 * k] = g * i;
        out[2 * k + 1] = g * q;
    }
    *gain = g;
}

/* timing_recovery_cc, libcsdr.c:1977-2072.  state[0] = last_correction_offset (in and out), state[1] = input_processed,
 * state[2] = output_size.  err / idx may be NULL. */
void psk31_oracle_timing_recovery_cc(const float *iq, float *out, int n, float *err, int *idx, int algorithm, int decimation, int use_q,
                                     float loop_gain, float max_error, int *state)
{
    const int h = decimation / 2, q = decimation / 4, wing = (int)((float)decimation * 0.25f);
    const double lo = (double)(-q) * 0.9, hi = (double)q * 0.9;
    int co = state[0], b = 0, si = 0;
    for (;;) {
        if (b + h * 3 >= n) break;
        if ((double)co <= lo || (double)co >= hi) co = 0;
        int l, m, r, s;
        if (algorithm == 1) { r = b + wing * 3; l = b + wing - co; m = b + h; s = m; }
        else if (algorithm == 0) { r = b + h * 3; l = b + h; m = b + h * 2; s = l; }
        else break;
        if (idx) idx[si] = s;
        out[2 * si] = iq[2 * s]; out[2 * si + 1] = iq[2 * s + 1];
        si++;
        float e = (iq[2 * r] - iq[2 * l]) * iq[2 * m];
        if (use_q) { const float eq = (iq[2 * r + 1] - iq[2 * l + 1]) * iq[2 * m + 1]; e = (e + eq) * 0.5f; }
        if (err) err[si - 1] = e;
        e = e < max_error ? e : max_error;                       /* minss */
        e = e > -max_error ? e : -max_error;                     /* maxss */
        const float step = (float)(algorithm == 0 ? -h : h);
        const float eg = e * loop_gain;
        co = (int)(eg * step);
        b += decimation + co;
        if (si >= n) break;
    }
    state[0] = co; state[1] = b; state[2] = si;
}

/* dbpsk_decoder_c_u8, libcsdr.c:2319-2333; last[0..1] is the previous sample (in and out) */
static float phase_of(float i, float q) { return (float)atan2((double)q, (double)i); }

void psk31_oracle_dbpsk_decoder_c_u8(const float *iq, unsigned char *out, int n, float *last)
{
    const float kPi = 3.14159274f, k2Pi = 6.28318548f, k3Pi = 9.42477798f, kHalfPi = 1.57079637f;
    float li = last[0], lq = last[1];
    for (int k = 0; k < n; k++) {
        const float i = iq[2 * k], q = iq[2 * k + 1];
        float d = phase_of(i, q) - phase_of(li, lq);
        if (d < -kPi) { float o; do { o = d; d = d + k2Pi; } while (o < -k3Pi); }
        else if (d >= kPi) { float o; do { o = d; d = d - k2Pi; } while (o >= k3Pi); }
        out[k] = (d > kHalfPi || !(d >= -kHalfPi)) ? 0 : 1;
        li = i; lq = q;
    }
    last[0] = li; last[1] = lq;
}

/* psk31_varicode_decoder_push, libcsdr.c:1536-1549, over a stream of bits (bytes, non-zero = 1).  The varicode of PSK31, ASCII 0..127, as
 * strings of code bits.  Returns the number of non-zero characters written to out; *hist is the shift register (in and out). */
static const char *kCodes[128] = {
    "1010101011", "1011011011", "1011101101", "1101110111", "1011101011", "1101011111", "1011101111", "1011111101", "1011111111", "11101111",
    "11101", "1101101111", "1011011101", "11111", "1101110101", "1110101011", "1011110111", "1011110101", "1110101101", "1110101111",
    "1101011011", "1101101011", "1101101101", "1101010111", "1101111011", "1101111101", "1110110111", "1101010101", "1101011101", "1110111011",
    "1011111011", "1101111111", "1", "111111111", "101011111", "111110101", "111011011", "1011010101", "1010111011", "101111111",
    "11111011", "11110111", "101101111", "111011111", "1110101", "110101", "1010111", "110101111", "10110111", "10111101",
    "11101101", "11111111", "101110111", "101011011", "101101011", "110101101", "110101011", "110110111", "11110101", "110111101",
    "111101101", "1010101", "111010111", "1010101111", "1010111101", "1111101", "11101011", "10101101", "10110101", "1110111",
    "11011011", "11111101", "101010101", "1111111", "111111101", "101111101", "11010111", "10111011", "11011101", "10101011",
    "11010101", "111011101", "10101111", "1101111", "1101101", "101010111", "110110101", "101011101", "101110101", "101111011",
    "1010101101", "111110111", "111101111", "111111011", "1010111111", "101101101", "1011011111", "1011", "1011111", "101111",
    "101101", "11", "111101", "1011011", "101011", "1101", "111101011", "10111111", "11011", "111011",
    "1111", "111", "111111", "110111111", "10101", "10111", "101", "110111", "1111011", "1101011",
    "11011111", "1011101", "111010101", "1010110111", "110111011", "1010110101", "1011010111", "1110110101",
};

int psk31_oracle_varicode_code(int ascii, int *bits)
{
    const char *s = kCodes[ascii & 127];
    int v = 0;
    for (const char *p = s; *p; p++) v = (v << 1) | (*p == '1');
    *bits = (int)strlen(s);
    return v;
}

int psk31_oracle_varicode_decode(const unsigned char *in, int n, unsigned char *out, uint64_t *hist)
{
    uint64_t shr = *hist;
    int cnt = 0;
    for (int k = 0; k < n; k++) {
        shr = (shr << 1) | (uint64_t)(in[k] != 0);
        for (int a = 0; a < 128; a++) {
            int bits;
            const uint64_t code = (uint64_t)psk31_oracle_varicode_code(a, &bits);
            const uint64_t mask = (bits + 4) >= 64 ? ~0ull : ((1ull << (bits + 4)) - 1ull);
            if ((code << 2) == (shr & mask)) { if (a) out[cnt++] = (unsigned char)a; break; }
        }
    }
    *hist = shr;
    return cnt;
}
