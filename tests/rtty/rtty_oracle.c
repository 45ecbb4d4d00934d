/*
 * rtty_oracle.c -- CPU restatement of the RTTY receive stages (serial_line_decoder_f_u8, rtty_baudot_decoder_lookup).
 * TEST INFRASTRUCTURE: compiled by tests/rtty/rtty.py into a temporary directory; the product never calls it.
 *
 * Plain IEEE-754 arithmetic (-fno-fast-math -ffp-contract=off), restating what the reference's -O3 -ffast-math build computes as read
 * from `objdump -d` of oracle/_ref/libcsdr_ref.so (DESIGN.md section 7), so that tests/test_oracle_rtty.py can pin it to that library
 * bit for bit.  Where the build differs from the source, the build is followed:
 *   - a window of 4 or more samples is summed in four partial sums (lane j takes samples j, j+4, ...), combined as (l0 + l2) + (l1 + l3),
 *     then the last (count mod 4) samples are added one by one; shorter windows are summed one by one from 0;
 *   - the stop-bit offsets are ((stopbits*spb)*0.5)*(1 -+ ratio) in double, the source's (stopbits*0.5*(1 -+ ratio))*spb reassociated;
 *   - 1 + ratio is formed in float like 1 - ratio;
 *   - the edge test is input[i] < 0 && !(input[i-1] <= 0): a NaN before a negative sample is an edge.
 */
#include <math.h>

static float window_sum(const float *x, int a, int b)
{
    float acc = 0.f;
    int k = a;
    if (b - a >= 4) {
        float l[4] = {0.f, 0.f, 0.f, 0.f};
        for (const int e = a + ((b - a) & ~3); k < e; k += 4)
            for (int j = 0; j < 4; j++) l[j] += x[k + j];
        acc = (l[0] + l[2]) + (l[1] + l[3]);
    }
    for (; k < b; k++) acc += x[k];
    return acc;
}

/* one serial_line_decoder_f_u8 call (libcsdr.c:1662-1729) on n samples, databits 1..8; st[0] = output_size, st[1] = input_used */
void rtty_oracle_serial_line_decoder(const float *x, unsigned char *out, int n, float spb, int databits, float stopbits, float ratio, int *st)
{
    const float all_bits = (float)(1 + databits) + stopbits;
    const double one_minus = (double)(1.0f - ratio), one_plus = (double)(ratio + 1.0f), spbd = (double)spb;
    const double data_lo = 0.5 * one_minus, data_hi = 0.5 * one_plus;
    const double stop_half = ((double)stopbits * spbd) * 0.5, stop_lo = one_minus * stop_half, stop_hi = stop_half * one_plus;
    int cnt = 0, used = 0;
    for (;;) {
        int sb = -1, i;
        for (i = 1; i < n; i++) if (x[i] < 0.f && !(x[i - 1] <= 0.f)) { sb = i; break; }
        if (sb < 0) { used += i; break; }                                 /* no edge: everything (at least 1) */
        const float sbf = (float)sb, span = spb * all_bits;
        if (span + sbf >= (float)n) { used += sb > 2 ? sb - 2 : 0; break; }       /* the character does not fit */
        unsigned shr = 0;
        for (int di = 0; di < databits; di++) {
            const double k = (double)(di + 1);
            const int a = (int)((k + data_lo) * spbd + (double)sb), b = (int)((k + data_hi) * spbd + (double)sb);
            shr = (shr << 1) | (window_sum(x, a, b) > 0.f);
        }
        const double base = (double)(spb * (float)(1 + databits) + sbf);
        const int a = (int)(stop_lo + base), b = (int)(base + stop_hi);
        if (window_sum(x, a, b) < 0.f) { used += n > sb ? sb + 1 : n; break; }     /* faulty stop bit */
        out[cnt++] = (unsigned char)shr;
        const float u = span + sbf, nf = (float)n;
        const int step = (int)(nf < u ? nf : u);                          /* minss */
        used += step; x += step; n -= step;
        if (!n) break;
    }
    st[0] = cnt; st[1] = used;
}

/* rtty_baudot_decoder_lookup (libcsdr.c:1608-1616): ITA2, letters and figures, indexed by the 5-bit code as the serial decoder assembles it
 * (first data bit most significant).  0 for code 0, for the shift codes FIGS (27) and LTRS (31), and for codes >= 32. */
static const unsigned char kLetters[32] = {0, 'T', '\r', 'O', ' ', 'H', 'N', 'M', '\n', 'L', 'R', 'G', 'I', 'P', 'C', 'V',
                                           'E', 'Z', 'D', 'B', 'S', 'Y', 'F', 'X', 'A', 'W', 'J', 0, 'U', 'Q', 'K', 0};
static const unsigned char kFigures[32] = {0, '5', '\r', '9', ' ', '$', ',', '.', '\n', ')', '4', '*', '8', '0', ':', '=',
                                           '3', '+', '#', '?', '\'', '6', '@', '/', '-', '2', '\a', 0, '7', '1', '(', 0};

int rtty_oracle_baudot_lookup(unsigned char *fig_mode, unsigned char c)
{
    if (c == 27) { *fig_mode = 1; return 0; }
    if (c == 31) { *fig_mode = 0; return 0; }
    if (c >= 32) return 0;
    return *fig_mode ? kFigures[c] : kLetters[c];
}

/* the lookup over a stream of codes: the non-zero characters go to out, their count is returned; *fig_mode carries over */
int rtty_oracle_baudot_decode(const unsigned char *in, int n, unsigned char *out, unsigned char *fig_mode)
{
    int cnt = 0;
    for (int k = 0; k < n; k++) {
        const int ch = rtty_oracle_baudot_lookup(fig_mode, in[k]);
        if (ch) out[cnt++] = (unsigned char)ch;
    }
    return cnt;
}
