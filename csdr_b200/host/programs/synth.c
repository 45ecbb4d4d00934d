/*
 * synth.c -- csdr-synth: many baseband channels into ONE wideband stream for a transmitter, in one process.
 *
 * What a transmit graph would otherwise run as one `csdr fir_interpolate_cc I | csdr shift_addition_cc RATE` chain per channel plus something
 * to add the chains' outputs (neither the reference nor the csdr CLI has a command that adds streams) is one synthesis bank
 * (csdrb_synth_bank_*): every block of every source goes to the GPU once, one launch interpolates, shifts and sums all channels, and the wideband
 * block comes back.  Plain C on the C ABI of libcsdr_b200 (no CUDA headers).
 *
 * usage: csdr-synth --interpolation I [--bw TBW] [--window W] [--chunk N] [--block N] [--mod M [--gain G]] RATE:SOURCE [RATE:SOURCE ...]
 *   --interpolation I  the factor from the baseband rate to the wideband rate (I >= 1)
 *   --bw TBW           transition bandwidth of the interpolation filter, 0 < TBW < 1 (default 0.05): the fir_interpolate_cc command's taps,
 *                      firdes_lowpass_f(taps, firdes_filter_len(TBW), 0.5 / I, W)
 *   --window W         HAMMING (default), BLACKMAN or BOXCAR
 *   --chunk N          samples per shift_addition_cc call on the wideband stream (default the CLI's 1024)
 *   --block N          baseband samples read from every source per block (default 16384)
 *   RATE               the channel's shift_addition_cc rate (fraction of the wideband sample rate)
 *   --mod M            every SOURCE carries f32 audio at the baseband rate, modulated on the device before the synthesis bank by the reference's
 *                      pipe for M:  am   gain_ff G | dsb_fc | add_dcoffset_cc
 *                                   dsb  gain_ff G | dsb_fc
 *                                   usb  gain_ff G | dsb_fc | bandpass_fir_fft_cc 0 0.1 0.05      (csdr-bankd's usb tail filter)
 *                                   lsb  gain_ff G | dsb_fc | bandpass_fir_fft_cc -0.1 0 0.05
 *                                   fm   gain_ff G | fmmod_fc                                      (the phase carried per channel from 0)
 *   --gain G           the gain_ff factor of --mod (default 1); refused without --mod
 *   SOURCE             a cf32 baseband file or FIFO, or - for stdin (at most once); f32 audio with --mod
 * The cf32 wideband stream goes to stdout, e.g. an FM modulator per channel into a 2.4 Msps transmitter at I = 50:
 *     csdr-synth --interpolation 50 -0.2:a.cf32 0.0:b.cf32 0.15:c.cf32 | csdr convert_f_s16 > tx.s16
 * Every block reads up to --block new samples from every source (blocking reads until the block is full or the source ends), runs one
 * csdrb_synth_bank_process and writes its outputs.  The program stops after the block in which any source ended.  stdout then holds the synthesis
 * bank run on all streams cut to the shortest source's length L, whatever --block is: max(0, L - h) * I samples, h = ceil((T - 1) / I) for T taps
 * (the CLI's per-process framing -- its zero preamble, its block-sized output steps -- is not reproduced).  With --mod the same holds for the
 * synthesis bank run over the modulator banks composed on every stream cut to the shortest source's length L; for usb/lsb L is first cut to whole
 * units of the filter's input_size (the overlap-add runs on whole units, the rest of each channel's audio waits for the next block), so the
 * output does not depend on --block either.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "csdr_b200.h"
#include "../ssb_filter.h"

static int fail(const char *msg, const char *arg)
{
    fprintf(stderr, "csdr-synth: %s%s%s\n", msg, arg ? ": " : "", arg ? arg : "");
    return 1;
}

static long failed(const char *msg, const char *arg) { fail(msg, arg); return -1; }

static int usage(void)
{
    fprintf(stderr, "usage: csdr-synth --interpolation I [--bw TBW] [--window W] [--chunk N] [--block N] [--mod M [--gain G]] RATE:SOURCE [RATE:SOURCE ...]\n"
                    "  sums fir_interpolate_cc I | shift_addition_cc RATE over the channels into one cf32 wideband stream on stdout\n"
                    "  --mod am|dsb|usb|lsb|fm: the sources carry f32 audio, modulated first by gain_ff G (--gain, default 1) and\n"
                    "    am: dsb_fc | add_dcoffset_cc   dsb: dsb_fc   usb/lsb: dsb_fc | bandpass_fir_fft_cc 0 0.1 (-0.1 0) 0.05   fm: fmmod_fc\n"
                    "  the output is the bank run on every stream cut to the shortest source (usb/lsb: to whole filter units), whatever --block is\n");
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

/* blocking read of up to `want` items of `item` bytes; returns how many arrived (fewer only at the end of the source) */
static size_t read_full(FILE *f, void *dst, size_t item, size_t want)
{
    size_t got = 0;
    while (got < want) {
        size_t r = fread((char *)dst + got * item, item, want - got, f);
        if (r == 0) break;
        got += r;
    }
    return got;
}

/* cf32 baseband sources: every block goes to the device as it is read.  Returns the wideband samples written, or -1 (message printed). */
static long run_baseband(int channels, FILE **src, csdrb_synth_bank_t *bank, int interpolation, int h, int block, void *stream)
{
    const long cap = (long)block + h;
    complexf *h_in = csdrb_host_alloc(sizeof(complexf) * (size_t)cap * (size_t)channels);
    complexf *h_out = csdrb_host_alloc(sizeof(complexf) * (size_t)cap * (size_t)interpolation);
    complexf *d_in = csdrb_device_alloc(sizeof(complexf) * (size_t)cap * (size_t)channels);
    complexf *d_out = csdrb_device_alloc(sizeof(complexf) * (size_t)cap * (size_t)interpolation);
    if (!h_in || !h_out || !d_in || !d_out) return failed("out of memory", csdrb_last_error());

    long have = 0;                                                     /* inputs per channel carried in front of the next block */
    int ended = 0;
    long written = 0;
    while (!ended) {
        size_t m = (size_t)block;
        for (int c = 0; c < channels; c++) {
            const size_t got = read_full(src[c], h_in + (size_t)c * (size_t)cap + (size_t)have, sizeof(complexf), (size_t)block);
            if (got < (size_t)block) ended = 1;
            if (got < m) m = got;
        }
        const long n = have + (long)m;                                 /* every channel is cut to the shortest source */
        if (csdrb_copy2d_h2d(d_in, sizeof(complexf) * (size_t)cap, h_in, sizeof(complexf) * (size_t)cap, sizeof(complexf) * (size_t)n,
                             (size_t)channels, stream) < 0)
            return failed("copy to the device failed", csdrb_last_error());
        const int produced = csdrb_synth_bank_process(bank, d_in, cap, (int)n, d_out, stream);
        if (produced < 0) return failed("synthesis bank failed", csdrb_last_error());
        if ((produced > 0 && csdrb_copy_d2h(h_out, d_out, sizeof(complexf) * (size_t)produced, stream) < 0) || csdrb_stream_synchronize(stream) < 0)
            return failed("copy from the device failed", csdrb_last_error());
        if (produced > 0) {
            if (fwrite(h_out, sizeof(complexf), (size_t)produced, stdout) != (size_t)produced) return failed("write to stdout failed", NULL);
            written += produced;
        }
        const long consumed = produced / interpolation;
        for (int c = 0; c < channels; c++)                             /* the inputs the last groups still look at start the next block */
            memmove(h_in + (size_t)c * (size_t)cap, h_in + (size_t)c * (size_t)cap + consumed, sizeof(complexf) * (size_t)(n - consumed));
        have = n - consumed;
    }
    csdrb_device_free(d_in); csdrb_device_free(d_out);
    csdrb_host_free(h_in); csdrb_host_free(h_out);
    return written;
}

enum { MOD_NONE, MOD_AM, MOD_DSB, MOD_USB, MOD_LSB, MOD_FM };

/* --mod: every block reads up to `block` audio samples per source behind the audio carried from the block before, cuts every channel to the
 * shortest, and on the device runs gain_ff and the mode's stages over the whole units (unit 1, or the usb/lsb filter's input_size) into the
 * baseband rows behind the inputs the synthesis bank kept, then the bank.  Returns the wideband samples written, or -1 (message printed). */
static long run_modulated(int mod, float gain, int channels, FILE **src, csdrb_synth_bank_t *bank, int interpolation, int h, int block, void *stream)
{
    int fft_size = 0, unit = 1;
    complexf *d_taps_fft = NULL, *d_ola_tail = NULL, *d_mid = NULL;
    if (mod == MOD_USB || mod == MOD_LSB) {
        const float band[2][2] = {{0.0f, 0.1f}, {-0.1f, 0.0f}};
        d_taps_fft = ssb_taps_fft(band[mod == MOD_LSB][0], band[mod == MOD_LSB][1], &fft_size, &unit, stream);
        if (!d_taps_fft) return failed("SSB filter taps failed", csdrb_last_error());
    }
    const long acap = (long)block + unit;                              /* audio per channel: [carry (< unit) | new block] */
    const long cap = acap + h;                                         /* baseband per channel: [kept by the bank (<= h) | new whole units] */
    float *h_audio = csdrb_host_alloc(sizeof(float) * (size_t)acap * (size_t)channels);
    complexf *h_out = csdrb_host_alloc(sizeof(complexf) * (size_t)cap * (size_t)interpolation);
    float *d_audio = csdrb_device_alloc(sizeof(float) * (size_t)acap * (size_t)channels);
    complexf *d_bb = csdrb_device_alloc(sizeof(complexf) * (size_t)cap * (size_t)channels);
    complexf *d_carry = csdrb_device_alloc(sizeof(complexf) * (size_t)(h > 0 ? h : 1) * (size_t)channels);
    complexf *d_out = csdrb_device_alloc(sizeof(complexf) * (size_t)cap * (size_t)interpolation);
    float *d_phase = csdrb_device_alloc(sizeof(float) * (size_t)channels);                 /* zero-filled: fmmod_fc starts at phase 0 */
    if (fft_size) {
        d_mid = csdrb_device_alloc(sizeof(complexf) * (size_t)acap * (size_t)channels);
        d_ola_tail = csdrb_device_alloc(sizeof(complexf) * (size_t)fft_size * (size_t)channels);   /* zero-filled: the overlap tail at stream start */
    }
    if (!h_audio || !h_out || !d_audio || !d_bb || !d_carry || !d_out || !d_phase || (fft_size && (!d_mid || !d_ola_tail)))
        return failed("out of memory", csdrb_last_error());

    long have = 0, ahave = 0, written = 0;                             /* baseband kept by the bank, audio carried (usb/lsb) */
    int ended = 0;
    while (!ended) {
        size_t m = (size_t)block;
        for (int c = 0; c < channels; c++) {
            const size_t got = read_full(src[c], h_audio + (size_t)c * (size_t)acap + (size_t)ahave, sizeof(float), (size_t)block);
            if (got < (size_t)block) ended = 1;
            if (got < m) m = got;
        }
        const long na = ahave + (long)m, whole = na / unit * unit;
        complexf *bb = d_bb + have;
        int rc = 0;
        if (whole > 0) {
            rc = csdrb_copy2d_h2d(d_audio, sizeof(float) * (size_t)acap, h_audio, sizeof(float) * (size_t)acap, sizeof(float) * (size_t)whole,
                                  (size_t)channels, stream);
            if (rc >= 0) rc = csdrb_gain_bank_ff(d_audio, acap, d_audio, acap, channels, (int)whole, gain, stream);
            if (rc >= 0) switch (mod) {
                case MOD_AM:
                    rc = csdrb_dsb_bank_fc(d_audio, acap, bb, cap, channels, (int)whole, 0.f, stream);
                    if (rc >= 0) rc = csdrb_add_dcoffset_bank_cc(bb, cap, bb, cap, channels, (int)whole, stream);
                    break;
                case MOD_DSB: rc = csdrb_dsb_bank_fc(d_audio, acap, bb, cap, channels, (int)whole, 0.f, stream); break;
                case MOD_USB: case MOD_LSB:
                    rc = csdrb_dsb_bank_fc(d_audio, acap, d_mid, acap, channels, (int)whole, 0.f, stream);
                    if (rc >= 0) rc = csdrb_bandpass_fir_fft_bank_cc(d_mid, acap, bb, cap, channels, fft_size, unit, (int)(whole / unit), d_taps_fft, 0,
                                                                     d_ola_tail, stream);
                    break;
                default: rc = csdrb_fmmod_bank_fc(d_audio, acap, bb, cap, channels, (int)whole, d_phase, stream); break;
            }
            if (rc < 0) return failed("modulator banks failed", csdrb_last_error());
        }
        const long n = have + whole;
        const int produced = csdrb_synth_bank_process(bank, d_bb, cap, (int)n, d_out, stream);
        if (produced < 0) return failed("synthesis bank failed", csdrb_last_error());
        const long consumed = produced / interpolation, keep = n - consumed;
        if (consumed > 0 && keep > 0) {                                /* the inputs the last groups still look at start the next block */
            const size_t width = sizeof(complexf) * (size_t)keep;
            if (csdrb_copy2d_d2d(d_carry, width, d_bb + consumed, sizeof(complexf) * (size_t)cap, width, (size_t)channels, stream) < 0 ||
                csdrb_copy2d_d2d(d_bb, sizeof(complexf) * (size_t)cap, d_carry, width, width, (size_t)channels, stream) < 0)
                return failed("device copy failed", csdrb_last_error());
        }
        if ((produced > 0 && csdrb_copy_d2h(h_out, d_out, sizeof(complexf) * (size_t)produced, stream) < 0) || csdrb_stream_synchronize(stream) < 0)
            return failed("copy from the device failed", csdrb_last_error());
        if (produced > 0) {
            if (fwrite(h_out, sizeof(complexf), (size_t)produced, stdout) != (size_t)produced) return failed("write to stdout failed", NULL);
            written += produced;
        }
        have = keep;
        for (int c = 0; c < channels; c++)                             /* the audio short of a whole unit waits for the next block */
            memmove(h_audio + (size_t)c * (size_t)acap, h_audio + (size_t)c * (size_t)acap + whole, sizeof(float) * (size_t)(na - whole));
        ahave = na - whole;
    }
    csdrb_device_free(d_taps_fft); csdrb_device_free(d_ola_tail); csdrb_device_free(d_mid);
    csdrb_device_free(d_audio); csdrb_device_free(d_bb); csdrb_device_free(d_carry); csdrb_device_free(d_out); csdrb_device_free(d_phase);
    csdrb_host_free(h_audio); csdrb_host_free(h_out);
    return written;
}

int main(int argc, char **argv)
{
    int interpolation = 0, chunk = 1024, block = 16384, ok = 1, mod = MOD_NONE, gain_set = 0;
    float bw = 0.05f, gain = 1.f;
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
        else if (!strcmp(a, "--gain")) { char *end; gain = strtof(v, &end); ok = ok && *v && !*end; gain_set = 1; }
        else if (!strcmp(a, "--mod")) {
            static const char *const names[] = {"am", "dsb", "usb", "lsb", "fm"};    /* MOD_AM .. MOD_FM */
            mod = MOD_NONE;
            for (int k = 0; k < 5; k++) if (!strcmp(v, names[k])) mod = MOD_AM + k;
            if (mod == MOD_NONE) return fail("unknown --mod (am, dsb, usb, lsb or fm)", v);
        }
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
    if (gain_set && mod == MOD_NONE) return fail("--gain needs --mod", NULL);

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
    csdrb_synth_bank_t *bank = csdrb_synth_bank_create(channels, rates, interpolation, taps, taps_length, chunk);
    if (!bank) return fail("bank create failed", csdrb_last_error());
    void *stream = csdrb_stream_create();
    const long written = mod == MOD_NONE ? run_baseband(channels, src, bank, interpolation, h, block, stream)
                                         : run_modulated(mod, gain, channels, src, bank, interpolation, h, block, stream);
    if (written < 0) return 1;
    fflush(stdout);
    fprintf(stderr, "csdr-synth: %d channels, %ld wideband samples\n", channels, written);
    csdrb_synth_bank_destroy(bank);
    csdrb_stream_destroy(stream);
    for (int c = 0; c < channels; c++) if (src[c] != stdin) fclose(src[c]);
    free(src); free(rates); free(taps);
    return 0;
}
