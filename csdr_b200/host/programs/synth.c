/*
 * synth.c -- csdr-synth: many baseband channels into ONE wideband stream for a transmitter, in one process.
 *
 * What a transmit graph would otherwise run as one `csdr fir_interpolate_cc I | csdr shift_addition_cc RATE` chain per channel plus something
 * to add the chains' outputs (neither the reference nor the csdr CLI has a command that adds streams) is one synthesis bank
 * (csdrb_synth_bank_*): every block of every source goes to the GPU once, one launch interpolates, shifts and sums all channels, and the wideband
 * block comes back.  Plain C on the C ABI of libcsdr_b200 (no CUDA headers).
 *
 * usage: csdr-synth --interpolation I [--bw TBW] [--window W] [--chunk N] [--block N] RATE:SOURCE [RATE:SOURCE ...]
 *   --interpolation I  the factor from the baseband rate to the wideband rate (I >= 1)
 *   --bw TBW           transition bandwidth of the interpolation filter, 0 < TBW < 1 (default 0.05): the fir_interpolate_cc command's taps,
 *                      firdes_lowpass_f(taps, firdes_filter_len(TBW), 0.5 / I, W)
 *   --window W         HAMMING (default), BLACKMAN or BOXCAR
 *   --chunk N          samples per shift_addition_cc call on the wideband stream (default the CLI's 1024)
 *   --block N          baseband samples read from every source per block (default 16384)
 *   RATE               the channel's shift_addition_cc rate (fraction of the wideband sample rate)
 *   SOURCE             a cf32 baseband file or FIFO, or - for stdin (at most once)
 * The cf32 wideband stream goes to stdout, e.g. an FM modulator per channel into a 2.4 Msps transmitter at I = 50:
 *     csdr-synth --interpolation 50 -0.2:a.cf32 0.0:b.cf32 0.15:c.cf32 | csdr convert_f_s16 > tx.s16
 * Every block reads up to --block new samples from every source (blocking reads until the block is full or the source ends), runs one
 * csdrb_synth_bank_process and writes its outputs.  The program stops after the block in which any source ended.  stdout then holds the synthesis
 * bank run on all streams cut to the shortest source's length L, whatever --block is: max(0, L - h) * I samples, h = ceil((T - 1) / I) for T taps
 * (the CLI's per-process framing -- its zero preamble, its block-sized output steps -- is not reproduced).
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "csdr_b200.h"

static int fail(const char *msg, const char *arg)
{
    fprintf(stderr, "csdr-synth: %s%s%s\n", msg, arg ? ": " : "", arg ? arg : "");
    return 1;
}

static int usage(void)
{
    fprintf(stderr, "usage: csdr-synth --interpolation I [--bw TBW] [--window W] [--chunk N] [--block N] RATE:SOURCE [RATE:SOURCE ...]\n"
                    "  sums fir_interpolate_cc I | shift_addition_cc RATE over the channels into one cf32 wideband stream on stdout\n");
    return 1;
}

/* a whole int argument, or 0 with *ok cleared */
static int int_arg(const char *s, int *ok)
{
    char *end;
    long v = strtol(s, &end, 10);
    if (!*s || *end || v < -2147483647L || v > 2147483647L) { *ok = 0; return 0; }
    return (int)v;
}

/* blocking read of up to `want` complex samples; returns how many arrived (fewer only at the end of the source) */
static size_t read_full(FILE *f, complexf *dst, size_t want)
{
    size_t got = 0;
    while (got < want) {
        size_t r = fread(dst + got, sizeof(complexf), want - got, f);
        if (r == 0) break;
        got += r;
    }
    return got;
}

int main(int argc, char **argv)
{
    int interpolation = 0, chunk = 1024, block = 16384, ok = 1;
    float bw = 0.05f;
    window_t window = WINDOW_DEFAULT;
    int first = 1;
    for (; first < argc; first++) {
        const char *a = argv[first];
        if (strncmp(a, "--", 2) || !strcmp(a, "--")) break;
        if (!strcmp(a, "--help")) return usage();
        if (first + 1 >= argc) return fail("missing value of", a);
        const char *v = argv[++first];
        if (!strcmp(a, "--interpolation")) interpolation = int_arg(v, &ok);
        else if (!strcmp(a, "--chunk")) chunk = int_arg(v, &ok);
        else if (!strcmp(a, "--block")) block = int_arg(v, &ok);
        else if (!strcmp(a, "--bw")) { char *end; bw = strtof(v, &end); ok = ok && *v && !*end; }
        else if (!strcmp(a, "--window")) {
            if (strcmp(v, "HAMMING") && strcmp(v, "BLACKMAN") && strcmp(v, "BOXCAR")) return fail("unknown window (HAMMING, BLACKMAN or BOXCAR)", v);
            window = firdes_get_window_from_string((char *)v);
        } else return fail("unknown option", a);
        if (!ok) return fail("malformed value of", a);
    }
    if (first < argc && !strcmp(argv[first], "--")) first++;
    const int channels = argc - first;
    if (channels < 1) return fail("no channel: give at least one RATE:SOURCE", NULL);
    if (interpolation < 1) return fail("--interpolation must be at least 1", NULL);
    if (!(bw > 0.f && bw < 1.f)) return fail("--bw must lie in (0, 1)", NULL);
    if (chunk < 1) return fail("--chunk must be at least 1", NULL);
    if (block < 1) return fail("--block must be at least 1", NULL);

    float *rates = malloc(sizeof(float) * (size_t)channels);
    FILE **src = calloc((size_t)channels, sizeof(FILE *));
    int stdin_used = 0;
    for (int c = 0; c < channels; c++) {
        const char *spec = argv[first + c];
        const char *colon = strchr(spec, ':');
        char *end;
        if (!colon || colon == spec || !colon[1]) return fail("malformed RATE:SOURCE", spec);
        char num[64];
        if ((size_t)(colon - spec) >= sizeof num) return fail("malformed RATE:SOURCE", spec);
        memcpy(num, spec, (size_t)(colon - spec)); num[colon - spec] = 0;
        rates[c] = strtof(num, &end);
        if (*end) return fail("malformed RATE:SOURCE", spec);
        if (!strcmp(colon + 1, "-")) {
            if (stdin_used) return fail("stdin (-) can be the source of one channel only", NULL);
            stdin_used = 1;
            src[c] = stdin;
        }
    }
    for (int c = 0; c < channels; c++) {                               /* opened after every argument is checked (a FIFO open waits for its writer) */
        if (src[c]) continue;
        const char *path = strchr(argv[first + c], ':') + 1;
        if (!(src[c] = fopen(path, "rb"))) return fail("cannot open source", path);
    }

    const int taps_length = firdes_filter_len(bw);
    float *taps = malloc(sizeof(float) * (size_t)taps_length);
    firdes_lowpass_f(taps, taps_length, 0.5f / (float)interpolation, window);
    const int h = (taps_length - 1 + interpolation - 1) / interpolation;     /* inputs a group looks ahead: kept from one block to the next */
    const long cap = (long)block + h;
    csdrb_synth_bank_t *bank = csdrb_synth_bank_create(channels, rates, interpolation, taps, taps_length, chunk);
    if (!bank) return fail("bank create failed", csdrb_last_error());
    void *stream = csdrb_stream_create();
    complexf *h_in = csdrb_host_alloc(sizeof(complexf) * (size_t)cap * (size_t)channels);
    complexf *h_out = csdrb_host_alloc(sizeof(complexf) * (size_t)cap * (size_t)interpolation);
    complexf *d_in = csdrb_device_alloc(sizeof(complexf) * (size_t)cap * (size_t)channels);
    complexf *d_out = csdrb_device_alloc(sizeof(complexf) * (size_t)cap * (size_t)interpolation);
    if (!h_in || !h_out || !d_in || !d_out) return fail("out of memory", csdrb_last_error());

    long have = 0;                                                     /* inputs per channel carried in front of the next block */
    int ended = 0;
    long written = 0;
    while (!ended) {
        size_t m = (size_t)block;
        for (int c = 0; c < channels; c++) {
            const size_t got = read_full(src[c], h_in + (size_t)c * (size_t)cap + (size_t)have, (size_t)block);
            if (got < (size_t)block) ended = 1;
            if (got < m) m = got;
        }
        const long n = have + (long)m;                                 /* every channel is cut to the shortest source */
        if (csdrb_copy2d_h2d(d_in, sizeof(complexf) * (size_t)cap, h_in, sizeof(complexf) * (size_t)cap, sizeof(complexf) * (size_t)n,
                             (size_t)channels, stream) < 0)
            return fail("copy to the device failed", csdrb_last_error());
        const int produced = csdrb_synth_bank_process(bank, d_in, cap, (int)n, d_out, stream);
        if (produced < 0) return fail("synthesis bank failed", csdrb_last_error());
        if ((produced > 0 && csdrb_copy_d2h(h_out, d_out, sizeof(complexf) * (size_t)produced, stream) < 0) || csdrb_stream_synchronize(stream) < 0)
            return fail("copy from the device failed", csdrb_last_error());
        if (produced > 0) {
            if (fwrite(h_out, sizeof(complexf), (size_t)produced, stdout) != (size_t)produced) return fail("write to stdout failed", NULL);
            written += produced;
        }
        const long consumed = produced / interpolation;
        for (int c = 0; c < channels; c++)                             /* the inputs the last groups still look at start the next block */
            memmove(h_in + (size_t)c * (size_t)cap, h_in + (size_t)c * (size_t)cap + consumed, sizeof(complexf) * (size_t)(n - consumed));
        have = n - consumed;
    }
    fflush(stdout);
    fprintf(stderr, "csdr-synth: %d channels, %ld wideband samples\n", channels, written);
    csdrb_synth_bank_destroy(bank);
    csdrb_stream_destroy(stream);
    csdrb_device_free(d_in); csdrb_device_free(d_out);
    csdrb_host_free(h_in); csdrb_host_free(h_out);
    for (int c = 0; c < channels; c++) if (src[c] != stdin) fclose(src[c]);
    free(src); free(rates); free(taps);
    return 0;
}
