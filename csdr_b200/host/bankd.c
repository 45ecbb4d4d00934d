/*
 * bankd.c -- csdr-bankd: a whole bank of NFM, WFM, AM, SSB, BPSK31 or RTTY receivers on ONE wideband IQ stream, in one process.
 *
 * SURVEY.md 8(f) rank 2.  What the reference does with processes -- `nmux` fanning the IQ stream out over TCP (nmux.cpp:246-353)
 * to one `csdr shift_addition_cc | csdr fir_decimate_cc | csdr fmdemod_quadri_cf | ...` chain per listener (ddcd_old.h:51-57,
 * README.md:87) -- becomes: read the stream once (stdin, or as a TCP client of an nmux server: nmux's wire format is the raw byte
 * stream, no framing), copy each block to the GPU once, run the fused bank kernel for all channels, and hand every channel's audio
 * to its own sink (file / FIFO / `tcp:PORT` listener).  Plain C on the C ABI of libcsdr_b200 (no CUDA headers).
 *
 * Per channel the sample stream is exactly the README graph's:
 *   convert_u8_f | shift_addition_cc r | fir_decimate_cc D bw W | fmdemod_quadri_cf [| limit_ff L | deemphasis_nfm_ff 48000 | fastagc_ff 1024 R | convert_f_s16]
 * as ONE continuous stream (the CLI's per-process block framing -- stale tail blocks at EOF, the zero block deemphasis_nfm_ff emits
 * first -- is process plumbing and is not reproduced; tests/test_gpu_zzz_bankd.py compares against the oracle run over the whole stream).
 *
 * usage: csdr-bankd [--in -|HOST:PORT] [--u8|--s8|--f32|--s16|--real-s16|--real-f32] [--decimation D] [--bw TRANSITION_BW] [--window W] [--block SAMPLES]
 *                   [--tail nfm|none|am|usb|lsb|iq|bpsk31|rtty|wfm] [--sps N] [--databits N] [--stopbits S] [--rtty-bufsize B] [--bfsk SPACING:LENGTH]
 *                   [--resample I:D[:BW]] [--fm-demod quadri|atan]
 *                   [--wfm-rate R] [--tau T]
 *                   [--limit L] [--agc-ref R] [--device N | --devices N0,N1,...]
 *                   [--waterfall SINK [--fft-size N] [--fft-every E] [--fft-averages A] [--fft-add-db X] [--fft-window W] [--fft-compression adpcm|none]
 *                    [--fft-real]]
 *                   RATE:SINK [RATE:SINK ...]
 *   --tail: nfm (default) the README.md:87 tail, s16; none the raw discriminator output, f32; am / usb / lsb the AM and SSB graphs of README.md:95 and :110
 *   behind the DDC's complex baseband (see bb_tail_t), s16; iq the complex baseband itself, cf32; bpsk31 the BPSK31 receive chain
 *   simple_agc_cc 0.001 R | timing_recovery_cc GARDNER N 0.5 2 --add_q | dbpsk_decoder_c_u8 | psk31_varicode_decoder_u8_u8 behind the baseband, the
 *   decoded text per channel (--sps N: samples per symbol at the baseband rate, > 4 and divisible by 4).  --limit is limit_ff's amplitude (default 1),
 *   --agc-ref the AGC reference (default: fastagc_ff's 1.0 for nfm, agc_ff's 0.2 for am/usb/lsb, simple_agc_cc's 0.5 for bpsk31).
 *   A PSK31 skimmer at 2.4 Msps: --decimation 300 --bw 0.001 gives 8 kHz baseband (4001 taps, M = 14 taps per output period: the fused bank serves it),
 *   and --sps 256 is 31.25 Bd:
 *     rtl_sdr -s 2400000 -f 14070000 - | csdr-bankd --decimation 300 --bw 0.001 --tail bpsk31 --sps 256 -0.1:ch1.txt 0.05:ch2.txt 0.2:ch3.txt
 *   rtty: the RTTY receive chain serial_line_decoder_f_u8 F N S | rtty_baudot2ascii_u8_u8 behind the discriminator (the bank runs with fmdemod),
 *   the decoded text per channel (--sps F: samples per bit at the baseband rate, a float; --databits N default 5, --stopbits S default 1.5).  The
 *   decoder runs in calls of exactly --rtty-bufsize B samples (default the CLI's 16384), so the text lags the signal by up to B baseband samples
 *   (about 8 s at 2 kHz); B must exceed F*(1 + N + S) + 2, or a call could not hold a character and the CLI would get stuck.  An RTTY skimmer
 *   at 2.4 Msps: --decimation 1200 --bw 0.001 gives 2 kHz baseband (4001 taps, M = 4 per output period, D*MP = 4800 <= 8000: the fused bank
 *   serves it), and --sps 44 is 45.45 Bd:
 *     rtl_sdr -s 2400000 -f 14080000 - | csdr-bankd --decimation 1200 --bw 0.001 --tail rtty --sps 44 -0.1:ch1.txt 0.05:ch2.txt 0.2:ch3.txt
 *   --bfsk SPACING:LENGTH demodulates with tone filters instead of the discriminator: the bank gives the complex baseband and each channel runs
 *   bfsk_demod_cf SPACING LENGTH (a Hamming peak filter of LENGTH taps on mark at +SPACING/2 and one on space at -SPACING/2 cycles per baseband
 *   sample, |mark|^2 - |space|^2 out) before the decoder; 170 Hz shift at 2 kHz baseband is --bfsk 0.085:44 (a filter about one bit long).
 *   wfm: broadcast FM, the README.md:66 graph's fractional_decimator_ff R | deemphasis_wfm_ff 48000 T | convert_f_s16 behind the discriminator (the bank
 *   runs with fmdemod), s16 audio per channel.  --wfm-rate R (default 5, above 1 and at most 16) brings wideband / D to 48 kHz, the de-emphasis rate;
 *   --tau T (default 50e-6; 75e-6 in the Americas).  Both run in the CLI's calls of 1024 samples (csdrb_wfm_audio_bank_f_s16), so every channel
 *   gets the bytes of that CLI pipe on the daemon's discriminator output.  No --resample: the fractional decimator is the rate converter.
 *   Three stations of a 2.4 Msps capture (240 kHz channels, 79 taps = 8 per output period, which the fused bank serves):
 *     rtl_sdr -s 2400000 -f 89300000 - | csdr-bankd --decimation 10 --bw 0.05 --tail wfm -0.085:a.s16 0.0:b.s16 0.2:c.s16
 *   and the whole 88-108 MHz band from a 20 Msps receiver, about 100 stations (250 kHz channels, 999 taps = 13 per output period):
 *     ... | csdr-bankd --decimation 80 --bw 0.004 --tail wfm --wfm-rate 5.2083333 -0.45:s1.s16 -0.44:s2.s16 ...
 *   --fm-demod quadri|atan picks the FM discriminator of the nfm, none, wfm and rtty tails.  quadri (default) is the bank's fmdemod_quadri_cf,
 *   K*|z[n-1]|/|z[n]|*sin(dphi) with K = 0.3404: sin() bends loud broadcast FM (75 kHz deviation in a 240 kHz channel takes dphi to 1.96 rad,
 *   harmonics about -13 dB below the tone).  atan runs the bank with the complex baseband (as --bfsk does) and fmdemod_atan_cf on it, dphi/pi,
 *   straight up to +-pi; per channel the stream is then ... | fir_decimate_cc D bw W | fmdemod_atan_cf | <the rest of the tail>, the phase
 *   carried from block to block.  At small deviation atan's level is 1/(pi*K) = 0.935 of quadri's, about 7 % lower on the none and wfm tails;
 *   the NFM AGC absorbs it.  Not with --bfsk, nor with the iq, am, usb, lsb and bpsk31 tails, which take the baseband.
 *   --decimation: any even D (default 50) whose filter the fused bank serves: M = ceil(taps / D) <= 24 and D * M (rounded up to the kernel's
 *   bucket) <= 8000 taps, see csdrb_ddc_bank in include/csdr_b200.h.  The NFM tail's deemphasis_nfm_ff stays at 48000 whatever D gives: where
 *   wideband rate / D is not 48 kHz, --resample I:D[:BW] puts rational_resampler_ff I D BW right behind the discriminator (tails nfm and none; see
 *   --help for the geometries it serves), e.g. 2.048 Msps with --decimation 32 --resample 3:4, or 10 Msps with --decimation 200 --resample 24:25:0.02.
 *   RATE  shift_addition_cc rate (fraction of the wideband sample rate), SINK a path (file or FIFO) or tcp:PORT (one listener).
 *   Input formats: --u8 (default) rtl_sdr's unsigned 8-bit IQ, --s8 HackRF's signed 8-bit IQ (convert_s8_f in front of the complex bank), --f32
 *   complex float, --s16 complex signed 16-bit (Airspy INT16_IQ, SDRplay, LimeSDR, PlutoSDR; convert_s16_f in front of the complex bank), and
 *   REAL streams as direct-sampling receivers (RX888 / SDDC, Airspy real modes, ADC boards) deliver them: --real-s16 (convert_s16_f) and --real-f32.  A real stream runs csdrb_ddc_bank_process_f, per channel
 *     convert_s16_f | shift_addition_fc r | fir_decimate_cc D bw W | <tail>
 *   and every tail works behind it.  A station at frequency f of a real stream sampled at fs is tuned with RATE = -f/fs (shift_addition_fc moves
 *   it to 0 Hz); +f/fs selects its mirror image, the conjugate: sidebands swapped and the discriminator negated.  E.g. 7.074 MHz FT8 from an RX888 at
 *   64.8 Msps, 48 kHz baseband: --real-s16 --decimation 1350 --bw 0.0008 --tail usb -0.10916667:ft8.s16.  --devices expands a real block to
 *   x + 0j on the host and runs the complex multi-GPU bank (the same outputs).  A real stream's waterfall is fft_fc's one-sided spectrum:
 *   --waterfall SINK --fft-real (below).
 *   --devices: the channels are sliced over several GPUs of this node (csdrb_multi_bank_*: the block goes to the first device once and on to
 *   the others by NCCL broadcast), one block of latency more (two blocks are kept in flight); the audio tail (nfm, am, usb, lsb), audio-rate work, runs on
 *   the first device for all channels, through the same kernels as without --devices; so do the bpsk31 and rtty decoders and the wfm tail.
 *   --waterfall SINK: the receiver server's other consumer of the wideband stream, OpenWebRX's waterfall
 *     fft_cc N E W | logaveragepower_cf X N A | fft_exchange_sides_ff N [| compress_fft_adpcm_f_u8 N]
 *   on every input sample (csdrb_spectrum_bank_cf on the block's cf32 samples, already on the device: no extra transfer; with --devices on the
 *   first device), so no nmux is needed in front of the daemon for it.  --fft-size N (default 2048), --fft-every E (default N), --fft-averages A
 *   (default 1), --fft-add-db X (default -70), --fft-window W (default HAMMING, fft_cc's), --fft-compression adpcm|none (default adpcm; none
 *   writes N floats of dB per line).  The sink gets the CLI pipe's lines on the whole stream, byte for byte.  At 2.4 Msps,
 *     rtl_sdr -s 2400000 - | csdr-bankd --waterfall wf.fifo --fft-size 4096 --fft-every 4096 --fft-averages 64 -0.1:ch1.s16 0.2:ch2.s16
 *   gives about 9 lines/s (2.4e6 / 4096 / 64).
 *   --fft-real (with --real-s16 | --real-f32): the waterfall of a real stream, fft_fc N E W | logaveragepower_cf X N A [| compress_fft_adpcm_f_u8 N]
 *   (csdrb_spectrum_bank_f on the block's real floats, where they already are on the device; with --devices the real floats of the host
 *   conversion go to the first device).  N counts bins (2N real samples per frame), --fft-every counts real samples and defaults to 2N, the lines
 *   run from DC up without a swap.  FT8 at 64.8 Msps with the whole HF waterfall beside it:
 *     csdr-bankd --real-s16 --decimation 1350 --bw 0.0008 --tail usb --waterfall wf.bin --fft-real --fft-size 16384 -0.10916667:ft8.s16
 * Sinks never hold the stream up: a sink that cannot take a block within 200 ms loses the rest of that block (counted on stderr at exit), one
 * that fails is dropped -- nmux's policy for slow clients (tsmpool.cpp:101-117, nmux.cpp:339-346).  The waterfall sink loses whole lines only
 * (a partial line would shift every later line): a line that cannot start within the block's 200 ms is dropped, one that started is finished.
 */
#define _GNU_SOURCE
#include "csdr_b200.h"
#include "ssb_filter.h"

#include <errno.h>
#include <fcntl.h>
#include <netdb.h>
#include <netinet/in.h>
#include <poll.h>
#include <signal.h>
#include <stdio.h>
#include <stdlib.h>
#include <limits.h>
#include <string.h>
#include <sys/socket.h>
#include <sys/types.h>
#include <unistd.h>

#define AGC_BLOCK 1024                                   /* fastagc_ff's default block (csdr.c:1382) */
#define NFM_RATE 48000                                   /* the README graph's audio rate: 2.4 Msps / 50 */

typedef struct { float rate; const char *sink; int fd; long dropped; } channel_t;

static int die(const char *what)
{
    fprintf(stderr, "csdr-bankd: %s", what);
    const char *e = csdrb_last_error();
    if (e && *e) fprintf(stderr, " (%s)", e);
    fprintf(stderr, "\n");
    exit(1);
}
#define OK(call) do { if ((call) < 0) die(#call " failed"); } while (0)

/* ---- input: stdin or a TCP client of an nmux server ------------------------------------------------------------------ */
static int open_input(const char *spec)
{
    if (!strcmp(spec, "-")) return STDIN_FILENO;
    char host[256];
    const char *colon = strrchr(spec, ':');
    if (!colon || (size_t)(colon - spec) >= sizeof host) die("--in wants - or HOST:PORT");
    memcpy(host, spec, (size_t)(colon - spec)); host[colon - spec] = 0;
    struct addrinfo hints = {0}, *res = NULL;
    hints.ai_family = AF_UNSPEC; hints.ai_socktype = SOCK_STREAM;
    if (getaddrinfo(host, colon + 1, &hints, &res) || !res) die("cannot resolve the --in address");
    int fd = -1;
    for (struct addrinfo *a = res; a; a = a->ai_next) {
        fd = socket(a->ai_family, a->ai_socktype, a->ai_protocol);
        if (fd < 0) continue;
        if (!connect(fd, a->ai_addr, a->ai_addrlen)) break;
        close(fd); fd = -1;
    }
    freeaddrinfo(res);
    if (fd < 0) die("cannot connect to the --in address");
    return fd;
}

/* all-or-EOF read: returns 1 when `bytes` bytes arrived, 0 at end of stream (a partial last block is dropped) */
static int read_block(int fd, unsigned char *dst, size_t bytes)
{
    size_t have = 0;
    while (have < bytes) {
        ssize_t got = read(fd, dst + have, bytes - have);
        if (got > 0) have += (size_t)got;
        else if (got == 0) return 0;
        else if (errno == EAGAIN || errno == EWOULDBLOCK) { struct pollfd p = {fd, POLLIN, 0}; poll(&p, 1, 1000); }   /* a non-blocking input: wait, do not spin */
        else if (errno != EINTR) return 0;
    }
    return 1;
}

/* ---- sinks ----------------------------------------------------------------------------------------------------------------- */
static int open_sink(const char *spec)
{
    if (!strncmp(spec, "tcp:", 4)) {                     /* one listener per channel, accepted before the stream starts */
        int ls = socket(AF_INET, SOCK_STREAM, 0), yes = 1;
        if (ls < 0) die("socket() failed");
        setsockopt(ls, SOL_SOCKET, SO_REUSEADDR, &yes, sizeof yes);
        struct sockaddr_in addr = {0};
        addr.sin_family = AF_INET; addr.sin_addr.s_addr = htonl(INADDR_ANY); addr.sin_port = htons((unsigned short)atoi(spec + 4));
        if (bind(ls, (struct sockaddr *)&addr, sizeof addr) || listen(ls, 1)) die("cannot listen on a tcp: sink");
        fprintf(stderr, "csdr-bankd: waiting for a listener on %s\n", spec);
        int fd = accept(ls, NULL, NULL);
        close(ls);
        if (fd < 0) die("accept() failed");
        return fd;
    }
    int fd = open(spec, O_WRONLY | O_CREAT | O_TRUNC, 0644);
    if (fd < 0) { fprintf(stderr, "csdr-bankd: cannot open %s: %s\n", spec, strerror(errno)); exit(1); }
    return fd;
}
static void sink_nonblocking(int fd) { const int fl = fcntl(fd, F_GETFL, 0); if (fl >= 0) fcntl(fd, F_SETFL, fl | O_NONBLOCK); }

/* a sink that fails (listener gone) is closed and skipped from then on, like nmux drops a client (nmux.cpp:339-346); one that is merely slow gets
 * 200 ms per block, then loses the rest of the block -- the other channels and the input never wait for it (nmux's readers are lossy too) */
static void write_sink(channel_t *ch, const void *data, size_t bytes)
{
    const unsigned char *p = data;
    int budget_ms = 200;
    while (ch->fd >= 0 && bytes) {
        ssize_t put = write(ch->fd, p, bytes);
        if (put > 0) { p += put; bytes -= (size_t)put; }
        else if (put < 0 && errno == EINTR) continue;
        else if (put < 0 && (errno == EAGAIN || errno == EWOULDBLOCK)) {
            if (budget_ms <= 0) { ch->dropped += (long)bytes; return; }
            struct pollfd pf = {ch->fd, POLLOUT, 0};
            poll(&pf, 1, 20); budget_ms -= 20;
        }
        else { fprintf(stderr, "csdr-bankd: sink %s closed\n", ch->sink); close(ch->fd); ch->fd = -1; }
    }
}

/* row c of the host rows at h (pitch bytes apart) to sink c: the whole row, or its first counts[c] bytes when counts is given */
static void write_rows(channel_t *chan, int C, const unsigned char *h, size_t pitch, const int *counts)
{
    for (int c = 0; c < C; c++) write_sink(&chan[c], h + pitch * (size_t)c, counts ? (size_t)(counts[c] > 0 ? counts[c] : 0) : pitch);
}

/* each of the C device rows at d_rows (pitch samples of esz bytes) keeps its n samples from `from` on, moved to the front through d_carry
 * (at least C x n samples): two copies on the stream, no synchronisation */
static void rows_to_front(void *d_rows, long pitch, int from, int n, size_t esz, void *d_carry, int C, void *stream)
{
    unsigned char *rows = d_rows;
    const size_t width = esz * (size_t)n;
    OK(csdrb_copy2d_d2d(d_carry, width, rows + esz * (size_t)from, esz * (size_t)pitch, width, (size_t)C, stream));
    OK(csdrb_copy2d_d2d(rows, esz * (size_t)pitch, d_carry, width, width, (size_t)C, stream));
}

/* a new stream on device dev, which stays the current device */
static void *device_stream(int dev)
{
    OK(csdrb_set_device(dev));
    void *stream = csdrb_stream_create();
    if (!stream) die("cannot create a stream");
    return stream;
}

/* ---- several GPUs: csdrb_multi_bank, raw discriminator output ------------------------------------------------------------------------ */
static int parse_devices(const char *list, int *dev, int max)
{
    int n = 0;
    for (const char *p = list; *p && n < max;) {
        char *e; long v = strtol(p, &e, 10);
        if (e == p) break;
        dev[n++] = (int)v;
        p = (*e == ',') ? e + 1 : e;
        if (*e && *e != ',') break;
    }
    return n;
}

/* ---- the NFM audio tail of README.md:87 behind the discriminator: limit_ff | deemphasis_nfm_ff 48000 | fastagc_ff | convert_f_s16 ------------------------
 * Device buffers of ONE device (the single-GPU path's own, the first device of --devices):
 *   demod   : [C][ds] float  : [Tn carried inputs of the de-emphasis FIR | new discriminator output]
 *   agc_in  : [C][gs] float  : [remainder (< AGC_BLOCK) | new de-emphasised samples]
 *   pcm     : [C][nb*AGC_BLOCK] s16 (contiguous so one flat copy serves all rows)
 * The caller puts n_new discriminator samples per channel at demod + a_have (pitch ds) and calls nfm_tail_push. */
typedef struct {
    int C, Tn, a_have, g_have;
    long ds, gs;
    float limit, agc_ref;
    float *d_demod, *d_carry, *d_agc_in;
    short *d_pcm;
    csdrb_fastagc_state_t *d_agc_state;
    float *d_agc_hist;
    void *d_agc_scratch;
    size_t agc_sb;
    unsigned char *h_out;
} nfm_tail_t;

static void nfm_tail_init(nfm_tail_t *t, int C, int out_cap, float limit, float agc_ref)
{
    t->C = C; t->limit = limit; t->agc_ref = agc_ref;
    if (!csdrb_deemphasis_nfm_taps(NFM_RATE, &t->Tn)) die("no de-emphasis table");
    t->ds = ((long)t->Tn + out_cap + 3) & ~3L;
    t->gs = ((long)AGC_BLOCK + out_cap + 3) & ~3L;
    t->d_demod = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)t->ds);
    t->d_carry = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)(AGC_BLOCK + t->Tn + 4));
    t->d_agc_in = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)t->gs);
    t->d_pcm = csdrb_device_alloc(sizeof(short) * (size_t)C * (size_t)t->gs + 16);
    t->d_agc_state = csdrb_device_alloc(sizeof(csdrb_fastagc_state_t) * (size_t)C);
    t->d_agc_hist = csdrb_device_alloc(sizeof(float) * (size_t)C * 2 * AGC_BLOCK);
    t->agc_sb = csdrb_fastagc_bank_scratch_bytes(C, (int)(t->gs / AGC_BLOCK) + 1);
    t->d_agc_scratch = csdrb_device_alloc(t->agc_sb + 16);
    t->h_out = csdrb_host_alloc((size_t)C * (size_t)t->gs * sizeof(float));
    if (!t->d_demod || !t->d_carry || !t->d_agc_in || !t->d_pcm || !t->d_agc_state || !t->d_agc_hist || !t->d_agc_scratch || !t->h_out) die("out of memory");
}

/* n_new fresh discriminator samples per channel sit at d_demod + a_have: de-emphasis (limiter fused), AGC + s16 over the whole AGC blocks, audio to the sinks */
static void nfm_tail_push(nfm_tail_t *t, channel_t *chan, int n_new, void *stream)
{
    const int C = t->C, Tn = t->Tn;
    const long ds = t->ds, gs = t->gs;
    const int a_n = t->a_have + n_new;
    /* limit_ff fused into deemphasis_nfm_ff: a_n inputs -> a_n - Tn outputs behind the AGC remainder; keep the last Tn inputs */
    int m = 0;
    if (a_n > Tn) {
        m = csdrb_deemphasis_nfm_bank_ff(t->d_demod, ds, t->d_agc_in + t->g_have, gs, C, a_n, NFM_RATE, t->limit, stream);
        if (m < 0) die("csdrb_deemphasis_nfm_bank_ff failed");
        rows_to_front(t->d_demod, ds, m, Tn, sizeof(float), t->d_carry, C, stream);
        t->a_have = Tn;
    } else t->a_have = a_n;
    /* fastagc_ff over the whole AGC blocks available, then convert_f_s16 (one pass); the remainder waits for the next block */
    const int g_n = t->g_have + m, nb = g_n / AGC_BLOCK, whole = nb * AGC_BLOCK;
    if (nb > 0) {
        OK(csdrb_fastagc_bank_f_s16(t->d_agc_in, gs, t->d_pcm, whole, C, AGC_BLOCK, nb, t->agc_ref, t->d_agc_state, t->d_agc_hist, t->d_agc_scratch, t->agc_sb + 16, stream));
        OK(csdrb_copy_d2h(t->h_out, t->d_pcm, sizeof(short) * (size_t)C * (size_t)whole, stream));
        const int rest = g_n - whole;
        rows_to_front(t->d_agc_in, gs, whole, rest, sizeof(float), t->d_carry, C, stream);
        t->g_have = rest;
        OK(csdrb_stream_synchronize(stream));
        write_rows(chan, C, t->h_out, sizeof(short) * (size_t)whole, NULL);
    } else {
        t->g_have = g_n;
        OK(csdrb_stream_synchronize(stream));
    }
}

/* ---- --resample I:D[:BW]: rational_resampler_ff I D BW right behind the discriminator (tails nfm and none) ---------------------------------------------------
 *   rs_in : [C][rs] float : [inputs the previous call left unconsumed (<= T/I) | new discriminator samples]
 * Each call ends because its input runs out, never on the output cap (resample_geometry_ok), so the state carries over exactly and every
 * channel's stream is the one a single rational_resampler_ff call over the whole discriminator stream gives. */
typedef struct {
    int C, I, D, T, ltd, have;
    long rs;
    float *taps, *d_in, *d_carry;
} rs_stage_t;

/* A call on n inputs computes outputs while the input lasts, floor((L*I + ltd) / D) + 1 of them with L = n - T/I - 1, and stops at the cap floor(n*I/D);
 * ending on the cap repeats that call's last output in the next call.  The input always runs out first when (T/I + 1)*I >= 2*D + I - 1, whatever n and
 * ltd < I (then (L*I + ltd)/D + 2 <= n*I/D); T >= 2*D + I - 2 is enough for that. */
static int resample_geometry_ok(int I, int D, int T) { return (long)(T / I + 1) * I >= 2L * D + I - 1; }

static void rs_init(rs_stage_t *r, int C, int I, int D, float bw, int in_cap)
{
    r->C = C; r->I = I; r->D = D; r->T = firdes_filter_len(bw);
    r->taps = malloc(sizeof(float) * (size_t)r->T);
    if (!r->taps) die("out of memory");
    rational_resampler_get_lowpass_f(r->taps, r->T, I, D, WINDOW_HAMMING);
    rational_resampler_ff_t st;                                      /* zero channels: the bank only checks the geometry */
    if (csdrb_rational_resampler_bank_ff(NULL, 0, NULL, 0, 0, 0, I, D, r->taps, r->T, 0, &st, NULL) < 0) die("--resample: the resampler refuses this geometry");
    r->rs = ((long)r->T / I + 2 + in_cap + 3) & ~3L;
    r->d_in = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)r->rs);
    r->d_carry = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)r->rs);
    if (!r->d_in || !r->d_carry) die("out of memory");
}

static int rs_out_cap(const rs_stage_t *r) { return (int)(r->rs * r->I / r->D) + 1; }

/* n_new fresh discriminator samples per channel sit at d_in + have: resample into dst (row pitch dst_pitch floats), keep what the call left unconsumed;
 * returns the outputs per channel */
static int rs_push(rs_stage_t *r, int n_new, float *dst, long dst_pitch, void *stream)
{
    const int n = r->have + n_new;
    rational_resampler_ff_t st;
    const int m = csdrb_rational_resampler_bank_ff(r->d_in, r->rs, dst, dst_pitch, r->C, n, r->I, r->D, r->taps, r->T, r->ltd, &st, stream);
    if (m < 0) die("csdrb_rational_resampler_bank_ff failed");
    const int keep = n - st.input_processed;
    if (keep > 0 && st.input_processed > 0) rows_to_front(r->d_in, r->rs, st.input_processed, keep, sizeof(float), r->d_carry, r->C, stream);
    r->have = keep; r->ltd = st.last_taps_delay;
    return m;
}

/* ---- --tail none and --tail iq: the bank's output itself, the discriminator (float) or the complex baseband (cf32) -----------------------------
 *   rows : [C][pitch] samples of esz bytes, the new ones from the front of every row; nothing is held back */
typedef struct { int C; size_t esz; long pitch; unsigned char *d_rows, *h_out; } raw_tail_t;

static void raw_tail_init(raw_tail_t *t, int C, int in_cap, size_t esz)
{
    t->C = C; t->esz = esz; t->pitch = ((long)in_cap + 3) & ~3L;
    t->d_rows = csdrb_device_alloc(esz * (size_t)C * (size_t)t->pitch);
    t->h_out = csdrb_host_alloc(esz * (size_t)C * (size_t)t->pitch);
    if (!t->d_rows || !t->h_out) die("out of memory");
}

/* n new samples per channel at the front of d_rows to the sinks */
static void raw_tail_push(raw_tail_t *t, channel_t *chan, int n, void *stream)
{
    const size_t width = t->esz * (size_t)n;
    OK(csdrb_copy2d_d2h(t->h_out, width, t->d_rows, t->esz * (size_t)t->pitch, width, (size_t)t->C, stream));
    OK(csdrb_stream_synchronize(stream));
    write_rows(chan, t->C, t->h_out, width, NULL);
}

/* ---- the AM and SSB audio tails (README.md:95, :110) behind the DDC bank's complex baseband ------------------------------------------------------------------
 *   am      : amdemod_cf | fastdcblock_ff 1024 | agc_ff | limit_ff L | convert_f_s16
 *   usb/lsb : bandpass_fir_fft_cc 0 0.1 0.05 (or -0.1 0 0.05) | realpart_cf | agc_ff | limit_ff L | convert_f_s16
 * agc_ff runs with the CLI defaults (csdr.c:1342-1361) and its 1024-sample calls; --agc-ref overrides the reference.  Device buffers of ONE device:
 *   bb   : [C][bs] complexf : [remainder (< unit samples) | new baseband]   unit = 1024 (am) or the overlap-add input size (usb/lsb)
 *   mid  : [C][bs] float (am: DC-blocked envelope) or complexf (usb/lsb: filtered baseband) over the whole units
 *   pcm  : [C][whole] s16 */

typedef struct {
    int C, unit, have, fft_size;                                  /* fft_size 0: am, else the usb/lsb bandpass */
    long bs;
    float limit;
    csdrb_agc_params_t agc;
    complexf *d_bb, *d_carry, *d_taps_fft, *d_ola_tail;
    void *d_mid;
    short *d_pcm;
    float *d_last_dc;
    csdrb_agc_state_t *d_agc_state;
    unsigned char *h_out;
} bb_tail_t;

/* band: the usb or lsb bandpass edges {lo, hi}; NULL for am */
static void bb_tail_init(bb_tail_t *t, int C, int out_cap, float limit, float agc_ref, const float *band, void *stream)
{
    t->C = C; t->limit = limit;
    const csdrb_agc_params_t p = {agc_ref, 0.01f, 0.0001f, 65536.0f, 200, 0, 0.999f, 1024};
    t->agc = p;
    t->unit = 1024;
    if (band) {                                                      /* bandpass_fir_fft_cc geometry and taps, ssb_filter.h */
        t->d_taps_fft = ssb_taps_fft(band[0], band[1], &t->fft_size, &t->unit, stream);
        if (!t->d_taps_fft) die("SSB filter taps failed");
        t->d_ola_tail = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->fft_size);   /* zero-filled: the overlap tail is zero at stream start (csdr.c:1860) */
        if (!t->d_ola_tail) die("out of memory");
    }
    t->bs = ((long)t->unit + out_cap + 3) & ~3L;
    t->d_bb = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->bs);
    t->d_carry = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->unit);
    t->d_mid = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->bs);
    t->d_pcm = csdrb_device_alloc(sizeof(short) * (size_t)C * (size_t)t->bs + 16);
    t->d_last_dc = csdrb_device_alloc(sizeof(float) * (size_t)C);                  /* zero-filled: last_dc_level starts at 0 (csdr.c:957) */
    t->d_agc_state = csdrb_device_alloc(sizeof(csdrb_agc_state_t) * (size_t)C);
    t->h_out = csdrb_host_alloc((size_t)C * (size_t)t->bs * sizeof(complexf));
    if (!t->d_bb || !t->d_carry || !t->d_mid || !t->d_pcm || !t->d_last_dc || !t->d_agc_state || !t->h_out) die("out of memory");
    csdrb_agc_state_t *h_st = calloc((size_t)C, sizeof *h_st);
    if (!h_st) die("out of memory");
    for (int c = 0; c < C; c++) h_st[c].gain = 1.0f;                 /* a stream starts at gain 1 (csdr.c:1363) */
    OK(csdrb_copy_h2d(t->d_agc_state, h_st, sizeof *h_st * (size_t)C, stream));
    OK(csdrb_stream_synchronize(stream));
    free(h_st);
}

/* n_new fresh baseband samples per channel sit at d_bb + have: run the tail over the whole units, audio to the sinks, keep the remainder */
static void bb_tail_push(bb_tail_t *t, channel_t *chan, int n_new, void *stream)
{
    const int C = t->C;
    const long bs = t->bs;
    const int n = t->have + n_new;
    const int nb = n / t->unit, whole = nb * t->unit, rest = n - whole;
    if (nb > 0) {
        if (!t->fft_size) {
            OK(csdrb_fastdcblock_bank_ff(t->d_bb, bs, 1, (float *)t->d_mid, bs, C, t->unit, nb, t->d_last_dc, stream));
            OK(csdrb_agc_bank_ff(t->d_mid, bs, 0, t->d_pcm, whole, 1, C, whole, &t->agc, t->d_agc_state, t->limit, stream));
        } else {
            OK(csdrb_bandpass_fir_fft_bank_cc(t->d_bb, bs, (complexf *)t->d_mid, bs, C, t->fft_size, t->unit, nb, t->d_taps_fft, 0, t->d_ola_tail, stream));
            OK(csdrb_agc_bank_ff(t->d_mid, bs, 1, t->d_pcm, whole, 1, C, whole, &t->agc, t->d_agc_state, t->limit, stream));
        }
        OK(csdrb_copy_d2h(t->h_out, t->d_pcm, sizeof(short) * (size_t)C * (size_t)whole, stream));
        if (rest > 0) rows_to_front(t->d_bb, bs, whole, rest, sizeof(complexf), t->d_carry, C, stream);
        OK(csdrb_stream_synchronize(stream));
        write_rows(chan, C, t->h_out, sizeof(short) * (size_t)whole, NULL);
    } else OK(csdrb_stream_synchronize(stream));
    t->have = rest;
}

/* ---- the BPSK31 tail: simple_agc_cc 0.001 R | timing_recovery_cc GARDNER N 0.5 2 --add_q | dbpsk_decoder_c_u8 | psk31_varicode_decoder_u8_u8 --------
 * Channels consume different amounts of baseband, so the timing recovery bank gets a start offset per channel.  Device buffers of ONE device:
 *   in   : [C][bs] complexf : the new baseband, from the front of every row
 *   tr   : [C][ts] complexf : AGC output; row c's unconsumed samples are [start[c], end) (end is the same for every row), new samples go to end
 *   sym  : [C][cap] complexf symbols, bits : [C][cap] dbpsk bits, chars : [C][cap] decoded text
 * Carried per channel: the AGC gain, the timing loop's correction offset and unconsumed baseband, the last dbpsk input, the varicode register.
 * The timing recovery leaves at most 3N/2 samples unconsumed, so every push first moves [min start, end) to the front of the rows. */
typedef struct {
    int C, sps, end, cap, last_cur;
    long bs, ts;
    float agc_ref;
    complexf *d_in, *d_tr, *d_carry, *d_sym, *d_last[2];
    unsigned char *d_bits, *d_chars;
    float *d_gain;
    int *d_start, *d_size, *d_counts, *d_char_count, *h_start, *h_size, *h_char_count;
    csdrb_timing_recovery_state_t *d_state, *h_state;
    unsigned long long *d_hist;
    unsigned char *h_chars;
} bpsk_tail_t;

static void bpsk_tail_init(bpsk_tail_t *t, int C, int sps, int in_cap, float agc_ref, void *stream)
{
    t->C = C; t->sps = sps; t->agc_ref = agc_ref;
    t->bs = ((long)in_cap + 3) & ~3L;
    t->ts = ((long)in_cap + 2L * sps + 3) & ~3L;
    t->cap = (int)(t->ts / (sps / 2) + 1);
    t->d_in = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->bs);
    t->d_tr = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->ts);
    t->d_carry = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->ts);
    t->d_sym = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->cap);
    t->d_last[0] = csdrb_device_alloc(sizeof(complexf) * (size_t)C);          /* zero-filled: dbpsk's previous sample starts at 0 */
    t->d_last[1] = csdrb_device_alloc(sizeof(complexf) * (size_t)C);
    t->d_bits = csdrb_device_alloc((size_t)C * (size_t)t->cap);
    t->d_chars = csdrb_device_alloc((size_t)C * (size_t)t->cap);
    t->d_gain = csdrb_device_alloc(sizeof(float) * (size_t)C);
    t->d_start = csdrb_device_alloc(sizeof(int) * (size_t)C * 2);            /* start[C] then size[C], one copy for both */
    t->d_size = t->d_start ? t->d_start + C : NULL;
    t->d_counts = csdrb_device_alloc(sizeof(int) * (size_t)C);
    t->d_char_count = csdrb_device_alloc(sizeof(int) * (size_t)C);
    t->d_state = csdrb_device_alloc(sizeof(csdrb_timing_recovery_state_t) * (size_t)C);   /* zero-filled: correction offset 0 */
    t->d_hist = csdrb_device_alloc(sizeof(unsigned long long) * (size_t)C);              /* zero-filled: status_shr = 0 */
    t->h_start = csdrb_host_alloc(sizeof(int) * (size_t)C * 3);
    t->h_state = csdrb_host_alloc(sizeof(csdrb_timing_recovery_state_t) * (size_t)C);
    t->h_chars = csdrb_host_alloc((size_t)C * (size_t)t->cap);
    if (!t->d_in || !t->d_tr || !t->d_carry || !t->d_sym || !t->d_last[0] || !t->d_last[1] || !t->d_bits || !t->d_chars || !t->d_gain || !t->d_start || !t->d_size ||
        !t->d_counts || !t->d_char_count || !t->d_state || !t->d_hist || !t->h_start || !t->h_state || !t->h_chars) die("out of memory");
    t->h_size = t->h_start + C; t->h_char_count = t->h_start + 2 * C;
    float *g = malloc(sizeof(float) * (size_t)C);
    if (!g) die("out of memory");
    for (int c = 0; c < C; c++) g[c] = 1.0f;                               /* simple_agc_cc's current_gain starts at 1 (csdr.c:2917) */
    OK(csdrb_copy_h2d(t->d_gain, g, sizeof(float) * (size_t)C, stream));
    OK(csdrb_stream_synchronize(stream));
    free(g);
}

/* n new baseband samples per channel at the front of d_in: the chain over them, the decoded text to the sinks */
static void bpsk_tail_push(bpsk_tail_t *t, channel_t *chan, int n, void *stream)
{
    const int C = t->C;
    int lo = t->end;
    for (int c = 0; c < C; c++) lo = t->h_start[c] < lo ? t->h_start[c] : lo;
    if (lo > 0 && t->end > lo) rows_to_front(t->d_tr, t->ts, lo, t->end - lo, sizeof(complexf), t->d_carry, C, stream);   /* the unconsumed samples */
    for (int c = 0; c < C; c++) t->h_start[c] -= lo;
    t->end -= lo;
    if (t->end + n > t->ts) die("bpsk31 tail: baseband buffer overflow");
    OK(csdrb_simple_agc_bank_cc(t->d_in, t->bs, t->d_tr + t->end, t->ts, C, n, 0.001f, t->agc_ref, 65535.0f, t->d_gain, stream));
    t->end += n;
    for (int c = 0; c < C; c++) t->h_size[c] = t->end - t->h_start[c];
    OK(csdrb_copy_h2d(t->d_start, t->h_start, sizeof(int) * (size_t)C * 2, stream));      /* h_start and h_size are adjacent */
    const csdrb_timing_recovery_params_t p = {0, t->sps, 1, 0.5f, 2.0f};  /* GARDNER <sps> 0.5 2 --add_q */
    OK(csdrb_timing_recovery_bank_cc(t->d_tr, t->ts, t->d_start, t->d_size, t->end, t->d_sym, t->cap, NULL, NULL, C, &p, t->d_state, stream));
    OK(csdrb_copy_d2h(t->h_state, t->d_state, sizeof(csdrb_timing_recovery_state_t) * (size_t)C, stream));
    OK(csdrb_stream_synchronize(stream));
    int *h_counts = t->h_size;                                              /* reused: the symbols each channel produced */
    int m = 0;
    for (int c = 0; c < C; c++) {
        t->h_start[c] += t->h_state[c].input_processed;
        h_counts[c] = t->h_state[c].output_size;
        m = h_counts[c] > m ? h_counts[c] : m;
    }
    if (m > 0) {
        OK(csdrb_copy_h2d(t->d_counts, h_counts, sizeof(int) * (size_t)C, stream));
        OK(csdrb_dbpsk_decoder_bank_c_u8(t->d_sym, t->cap, t->d_bits, t->cap, C, m, t->d_counts, t->d_last[t->last_cur], t->d_last[t->last_cur ^ 1], stream));
        t->last_cur ^= 1;
        OK(csdrb_psk31_varicode_decoder_bank_u8_u8(t->d_bits, t->cap, t->d_chars, t->cap, C, m, t->d_counts, t->d_hist, t->d_char_count, stream));
        OK(csdrb_copy_d2h(t->h_char_count, t->d_char_count, sizeof(int) * (size_t)C, stream));
        OK(csdrb_copy2d_d2h(t->h_chars, (size_t)m, t->d_chars, (size_t)t->cap, (size_t)m, (size_t)C, stream));
        OK(csdrb_stream_synchronize(stream));
        write_rows(chan, C, t->h_chars, (size_t)m, t->h_char_count);
    }
}

/* ---- the RTTY tail: serial_line_decoder_f_u8 F N S | rtty_baudot2ascii_u8_u8 behind the discriminator ---------------------------------------------
 * Channels consume different amounts of signal, so each row has its own start.  Device buffers of ONE device:
 *   rows  : [C][rs] float : discriminator output; row c's unconsumed samples are [start[c], end) (end is the same for every row), new ones go to end
 *   codes : [C][cap] ITA2 codes, chars : [C][cap] decoded text
 * The decoder bank runs calls of exactly B samples while B remain (the CLI's framing), so each row keeps fewer than B samples; after every push
 * [min start, end) moves to the front of the rows.  Carried per channel: the start, the FIGS/LTRS mode. */
typedef struct {
    int C, B, end, cap;
    long rs;
    csdrb_serial_line_params_t p;
    float *d_rows, *d_carry;
    unsigned char *d_codes, *d_chars, *d_mode, *h_chars;
    int *d_start, *d_count, *d_stuck, *d_char_count, *h_start;                 /* h_start: start[C], stuck[C], char_count[C] */
    /* --bfsk: the bank gives complexf baseband rows; bfsk_demod_cf with L taps turns them into the rows above.  bb: [C][bs] complexf, the
     * last L - 1 samples of the previous push (bb_have of them) and then the new ones; mark/space: the taps on the device */
    int L, bb_have;
    long bs;
    complexf *d_bb, *d_bb_carry, *d_mark, *d_space;
} rtty_tail_t;

static void rtty_tail_init(rtty_tail_t *t, int C, const csdrb_serial_line_params_t *p, int bufsize, int in_cap)
{
    t->C = C; t->B = bufsize; t->p = *p;
    t->rs = ((long)bufsize + in_cap + 3) & ~3L;
    t->cap = (int)(t->rs / (long)(p->samples_per_bits * ((float)(1 + p->databits) + p->stopbits)) + 1);   /* the bank's output bound */
    t->d_rows = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)t->rs);
    t->d_carry = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)bufsize);
    t->d_codes = csdrb_device_alloc((size_t)C * (size_t)t->cap);
    t->d_chars = csdrb_device_alloc((size_t)C * (size_t)t->cap);
    t->d_mode = csdrb_device_alloc((size_t)C);                               /* zero-filled: letters mode */
    t->d_start = csdrb_device_alloc(sizeof(int) * (size_t)C * 3);            /* start[C], stuck[C], char_count[C]: one copy back for all three */
    t->d_stuck = t->d_start ? t->d_start + C : NULL;
    t->d_char_count = t->d_start ? t->d_start + 2 * C : NULL;
    t->d_count = csdrb_device_alloc(sizeof(int) * (size_t)C);
    t->h_start = csdrb_host_alloc(sizeof(int) * (size_t)C * 3);
    t->h_chars = csdrb_host_alloc((size_t)C * (size_t)t->cap);
    if (!t->d_rows || !t->d_carry || !t->d_codes || !t->d_chars || !t->d_mode || !t->d_start || !t->d_count || !t->h_start || !t->h_chars)
        die("out of memory");
}

/* --bfsk SPACING:LENGTH: the taps of `csdr bfsk_demod_cf SPACING LENGTH` (csdr.c:3283-3286), and rows for LENGTH - 1 carried samples plus a push */
static void rtty_bfsk_init(rtty_tail_t *t, float spacing, int L, int in_cap, void *stream)
{
    const int C = t->C;
    t->L = L;
    t->bs = ((long)L - 1 + in_cap + 1) & ~1L;
    complexf *h = malloc(sizeof(complexf) * 2 * (size_t)L);
    t->d_bb = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->bs);
    t->d_bb_carry = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)L);
    t->d_mark = csdrb_device_alloc(sizeof(complexf) * 2 * (size_t)L);
    if (!h || !t->d_bb || !t->d_bb_carry || !t->d_mark) die("out of memory");
    t->d_space = t->d_mark + L;
    firdes_add_peak_c(h, L, spacing / 2, WINDOW_DEFAULT, 0, 1);
    firdes_add_peak_c(h + L, L, -spacing / 2, WINDOW_DEFAULT, 0, 1);
    OK(csdrb_copy_h2d(t->d_mark, h, sizeof(complexf) * 2 * (size_t)L, stream));
    OK(csdrb_stream_synchronize(stream));
    free(h);
}

/* n new discriminator samples per channel sit at d_rows + end: decode what fills whole calls, the text to the sinks, keep the rest */
static void rtty_tail_push(rtty_tail_t *t, channel_t *chan, int n, void *stream)
{
    const int C = t->C;
    t->end += n;
    if (t->end > t->rs) die("rtty tail: signal buffer overflow");
    OK(csdrb_serial_line_decoder_bank_f_u8(t->d_rows, t->rs, t->end, t->d_start, t->d_codes, t->cap, t->d_count, t->d_stuck, C, &t->p, t->B, stream));
    OK(csdrb_rtty_baudot2ascii_bank_u8_u8(t->d_codes, t->cap, t->d_chars, t->cap, C, t->cap, t->d_count, t->d_mode, t->d_char_count, stream));
    OK(csdrb_copy_d2h(t->h_start, t->d_start, sizeof(int) * (size_t)C * 3, stream));
    OK(csdrb_copy_d2h(t->h_chars, t->d_chars, (size_t)C * (size_t)t->cap, stream));
    OK(csdrb_stream_synchronize(stream));
    const int *stuck = t->h_start + C, *chars = t->h_start + 2 * C;
    int lo = t->end;
    for (int c = 0; c < C; c++) {
        if (stuck[c]) die("rtty tail: serial_line_decoder_f_u8 got stuck");   /* main() refuses the parameters that allow it */
        lo = t->h_start[c] < lo ? t->h_start[c] : lo;
    }
    write_rows(chan, C, t->h_chars, (size_t)t->cap, chars);
    if (lo > 0) {                                                           /* the unconsumed samples (fewer than B per row) to the front */
        if (t->end > lo) rows_to_front(t->d_rows, t->rs, lo, t->end - lo, sizeof(float), t->d_carry, C, stream);
        for (int c = 0; c < C; c++) t->h_start[c] -= lo;
        t->end -= lo;
        OK(csdrb_copy_h2d(t->d_start, t->h_start, sizeof(int) * (size_t)C, stream));
        OK(csdrb_stream_synchronize(stream));
    }
}

/* --bfsk: n new baseband samples per channel sit at d_bb + bb_have; the bfsk outputs of every complete window go to the decoder's rows */
static void rtty_bfsk_push(rtty_tail_t *t, channel_t *chan, int n, void *stream)
{
    const int have = t->bb_have + n;
    if (have < t->L) { t->bb_have = have; return; }
    if (t->end + (long)(have - t->L + 1) > t->rs) die("rtty tail: signal buffer overflow");
    const int m = csdrb_bfsk_demod_bank_cf(t->d_bb, t->bs, t->d_rows + t->end, t->rs, t->C, have, t->d_mark, t->d_space, t->L, stream);
    if (m < 0) die("csdrb_bfsk_demod_bank_cf failed");
    t->bb_have = t->L - 1;
    rows_to_front(t->d_bb, t->bs, have - t->bb_have, t->bb_have, sizeof(complexf), t->d_bb_carry, t->C, stream);
    rtty_tail_push(t, chan, m, stream);
}

/* ---- the WFM tail: fractional_decimator_ff R | deemphasis_wfm_ff 48000 TAU | convert_f_s16 behind the discriminator (README.md:66) --------------
 * The bank runs the decimator in the CLI's calls of WFM_BUFSIZE samples and consumes the same samples of every row.  Device buffers of ONE device:
 *   rows : [C][rs] float : [the unconsumed rest (< WFM_BUFSIZE) | new discriminator samples]
 *   pcm  : [C][cap] s16
 * Carried: the rest of every row, the host state {where, audio} and the de-emphasis carry of every channel. */
#define WFM_BUFSIZE 1024                                 /* the CLI's the_bufsize: the decimator's call size and the de-emphasis NaN-reset period */

typedef struct {
    int C, have, cap;
    long rs;
    csdrb_wfm_audio_params_t p;
    csdrb_wfm_audio_state_t s;
    float *d_rows, *d_carry, *d_last;
    short *d_pcm;
    unsigned char *h_pcm;
} wfm_tail_t;

static void wfm_tail_init(wfm_tail_t *t, int C, float rate, float tau, int in_cap)
{
    const csdrb_wfm_audio_params_t p = {rate, WFM_BUFSIZE, tau, NFM_RATE};
    t->C = C; t->p = p;
    t->rs = ((long)WFM_BUFSIZE + in_cap + 3) & ~3L;
    t->cap = (int)((double)t->rs / rate) + 2;                         /* every output advances the position by rate (> 1) */
    t->d_rows = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)t->rs);
    t->d_carry = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)WFM_BUFSIZE);
    t->d_last = csdrb_device_alloc(sizeof(float) * (size_t)C);           /* zero-filled: the de-emphasis starts from 0 */
    t->d_pcm = csdrb_device_alloc(sizeof(short) * (size_t)C * (size_t)t->cap);
    t->h_pcm = csdrb_host_alloc(sizeof(short) * (size_t)C * (size_t)t->cap);
    if (!t->d_rows || !t->d_carry || !t->d_last || !t->d_pcm || !t->h_pcm) die("out of memory");
}

/* n new discriminator samples per channel sit at d_rows + have: the audio of the whole decimator calls to the sinks, the rest to the front */
static void wfm_tail_push(wfm_tail_t *t, channel_t *chan, int n, void *stream)
{
    const int C = t->C, total = t->have + n;
    int consumed = 0;
    const int m = csdrb_wfm_audio_bank_outputs(&t->p, &t->s, total, &consumed);
    if (m < 0) die("csdrb_wfm_audio_bank_outputs failed");
    if (m > t->cap) die("wfm tail: more audio than the buffer holds");
    if (csdrb_wfm_audio_bank_f_s16(t->d_rows, t->rs, C, total, &t->p, &t->s, t->d_last, t->d_pcm, t->cap, &consumed, stream) != m)
        die("csdrb_wfm_audio_bank_f_s16 failed");
    const int rest = total - consumed;
    if (rest > 0 && consumed > 0) rows_to_front(t->d_rows, t->rs, consumed, rest, sizeof(float), t->d_carry, C, stream);
    t->have = rest;
    if (m > 0) OK(csdrb_copy2d_d2h(t->h_pcm, sizeof(short) * (size_t)m, t->d_pcm, sizeof(short) * (size_t)t->cap, sizeof(short) * (size_t)m, (size_t)C, stream));
    OK(csdrb_stream_synchronize(stream));
    write_rows(chan, C, t->h_pcm, sizeof(short) * (size_t)m, NULL);
}

/* ---- --waterfall SINK: fft_cc N E W | logaveragepower_cf X N A | fft_exchange_sides_ff N [| compress_fft_adpcm_f_u8 N] on the wideband stream ---
 * One row of csdrb_spectrum_bank_cf over the block's fresh cf32 samples: the bank carries the framing and the partial line from block to block, so
 * the sink gets the bytes of the CLI pipe on the whole stream.  Device buffers of ONE device (the single-GPU path's own, the first device of --devices);
 * d_in holds the block for --devices, whose samples arrive in host memory. */
typedef struct { int fft_size, every, averages, compress; float add_db; window_t window; int real; } waterfall_opts_t;   /* real: --fft-real */

typedef struct {
    csdrb_spectrum_params_t p;
    csdrb_spectrum_state_t s;
    size_t line_bytes, sb;
    long cap;                                                   /* lines one block can complete */
    int real;                                                   /* --fft-real: csdrb_spectrum_bank_f on real samples, d_hist / d_in hold floats */
    float *d_window, *d_acc;
    void *d_hist, *d_in;
    unsigned char *d_lines, *h_lines;
    void *d_scratch;
    channel_t sink;
    long lines_dropped;
} waterfall_t;

static void waterfall_init(waterfall_t *w, const waterfall_opts_t *o, int block, int need_in, void *stream)
{
    const int fft_size = o->fft_size, frame = o->real ? 2 * fft_size : fft_size;       /* fft_fc's frame is 2N real samples */
    const size_t ssz = o->real ? sizeof(float) : sizeof(complexf);
    const csdrb_spectrum_params_t p = {fft_size, o->every, o->averages, o->compress, o->add_db};
    w->p = p;
    w->real = o->real;
    w->s.consumed = 0; w->s.frames = 0;
    w->lines_dropped = 0;
    w->line_bytes = o->compress ? (size_t)(fft_size + 10) / 2 : sizeof(float) * (size_t)fft_size;
    w->cap = ((long)block + o->every - 1) / o->every / o->averages + 1;
    /* one launch per block when that takes at most 64 MB of scratch, else chunks of frames (same bytes) */
    size_t (*scratch_bytes)(int, long, const csdrb_spectrum_params_t *) = o->real ? csdrb_spectrum_bank_scratch_bytes_f : csdrb_spectrum_bank_scratch_bytes;
    const size_t full = scratch_bytes(1, block, &w->p), one = scratch_bytes(1, 1, &w->p), cap = (size_t)64 << 20;
    w->sb = full <= cap ? full : (one > cap ? one : cap);
    float *h_window = precalculate_window(frame, o->window);
    w->d_window = csdrb_device_alloc(sizeof(float) * (size_t)frame);
    w->d_acc = csdrb_device_alloc(sizeof(float) * (size_t)fft_size);            /* zero-filled: the first line starts from 0 */
    w->d_hist = csdrb_device_alloc(ssz * (size_t)frame);                        /* zero-filled: samples before the stream are 0 */
    w->d_in = need_in ? csdrb_device_alloc(ssz * (size_t)block) : NULL;
    w->d_lines = csdrb_device_alloc(w->line_bytes * (size_t)w->cap);
    w->h_lines = csdrb_host_alloc(w->line_bytes * (size_t)w->cap);
    w->d_scratch = csdrb_device_alloc(w->sb);
    if (!h_window || !w->d_window || !w->d_acc || !w->d_hist || (need_in && !w->d_in) || !w->d_lines || !w->h_lines || !w->d_scratch) die("out of memory");
    OK(csdrb_copy_h2d(w->d_window, h_window, sizeof(float) * (size_t)frame, stream));
    OK(csdrb_stream_synchronize(stream));
    free(h_window);
}

/* Only whole lines are dropped: a partial line would shift every later line of the fixed-size line stream.  A line that cannot start within the
 * block's 200 ms is dropped (counted); a line that started is finished. */
static void write_lines(waterfall_t *w, long lines)
{
    channel_t *ch = &w->sink;
    int budget_ms = 200;
    for (long k = 0; k < lines && ch->fd >= 0; k++) {
        const unsigned char *p = w->h_lines + (size_t)k * w->line_bytes;
        size_t left = w->line_bytes;
        while (ch->fd >= 0 && left) {
            ssize_t put = write(ch->fd, p, left);
            if (put > 0) { p += put; left -= (size_t)put; }
            else if (put < 0 && errno == EINTR) continue;
            else if (put < 0 && (errno == EAGAIN || errno == EWOULDBLOCK)) {
                const int started = left < w->line_bytes;
                if (!started && budget_ms <= 0) { w->lines_dropped++; break; }
                struct pollfd pf = {ch->fd, POLLOUT, 0};
                poll(&pf, 1, 20);
                if (!started) budget_ms -= 20;
            }
            else { fprintf(stderr, "csdr-bankd: sink %s closed\n", ch->sink); close(ch->fd); ch->fd = -1; }
        }
    }
}

/* n fresh wideband samples at d_fresh (on the stream's device; cf32, or f32 with --fft-real): the lines they complete to the waterfall sink */
static void waterfall_push(waterfall_t *w, const void *d_fresh, int n, void *stream)
{
    const long pitch = (long)(w->line_bytes * (size_t)w->cap);
    const int lines = w->real ? csdrb_spectrum_bank_f((const float *)d_fresh, n, 1, n, w->d_window, &w->p, (float *)w->d_hist, w->d_acc, &w->s, w->d_lines, pitch,
                                                      w->d_scratch, w->sb, stream)
                              : csdrb_spectrum_bank_cf((const complexf *)d_fresh, n, 1, n, w->d_window, &w->p, (complexf *)w->d_hist, w->d_acc, &w->s, w->d_lines,
                                                       pitch, w->d_scratch, w->sb, stream);
    if (lines < 0) die(w->real ? "csdrb_spectrum_bank_f failed" : "csdrb_spectrum_bank_cf failed");
    if (lines > w->cap) die("waterfall: more lines than the buffer holds");
    OK(csdrb_copy_d2h(w->h_lines, w->d_lines, w->line_bytes * (size_t)lines, stream));
    OK(csdrb_stream_synchronize(stream));
    write_lines(w, lines);
}

/* ---- sinks of both loops: opened last (a tcp: sink blocks until its listener arrives), losses reported at the end ------------------------------ */
static void open_sinks(channel_t *chan, int C, waterfall_t *wf)
{
    for (int c = 0; c < C; c++) { chan[c].fd = open_sink(chan[c].sink); sink_nonblocking(chan[c].fd); }
    if (wf) { wf->sink.fd = open_sink(wf->sink.sink); sink_nonblocking(wf->sink.fd); }
}

static void close_sinks(channel_t *chan, int C, waterfall_t *wf)
{
    for (int c = 0; c < C; c++) { if (chan[c].dropped) fprintf(stderr, "csdr-bankd: sink %s lost %ld bytes (too slow)\n", chan[c].sink, chan[c].dropped); if (chan[c].fd >= 0) close(chan[c].fd); }
    if (wf) {
        if (wf->lines_dropped) fprintf(stderr, "csdr-bankd: waterfall sink %s lost %ld lines (too slow)\n", wf->sink.sink, wf->lines_dropped);
        if (wf->sink.fd >= 0) close(wf->sink.fd);
    }
}

/* ---- options: main() parses and validates them, both loops read them ------------------------------------------------------------------------ */
/* wideband input formats (--u8 ...), their bytes per sample on the wire and their names */
enum { IN_U8, IN_F32, IN_S16, IN_REAL_S16, IN_REAL_F32, IN_S8 };
static const int kWireBytes[] = {2, 8, 4, 2, 4, 2};
static const char *kFormatNames[] = {"u8", "f32", "s16", "real s16", "real f32", "s8"};
#define S16_RECIP (1.0f / 32767.0f)                       /* convert_s16_f: the reference build multiplies by the float reciprocal (csdrb_convert_s16_f) */
#define S8_RECIP (1.0f / 127.0f)                          /* convert_s8_f: likewise (csdrb_convert_s8_f) */

/* the tails (--tail NAME): whether the bank demodulates for them (float discriminator rows, else cf32 baseband rows), whether --resample
 * may run in front of them, and their AGC reference when --agc-ref is not given: fastagc_ff's default (csdr.c:1388), agc_ff's (csdr.c:1342),
 * simple_agc_cc's in the OpenWebRX chain */
enum { TAIL_NFM, TAIL_NONE, TAIL_IQ, TAIL_AM, TAIL_USB, TAIL_LSB, TAIL_BPSK31, TAIL_RTTY, TAIL_WFM };
static const struct { const char *name; int demod, resample; float agc_ref; } kTails[] = {
    [TAIL_NFM] = {"nfm", 1, 1, 1.0f}, [TAIL_NONE] = {"none", 1, 1, 0.f}, [TAIL_IQ] = {"iq", 0, 0, 0.f}, [TAIL_AM] = {"am", 0, 0, 0.2f},
    [TAIL_USB] = {"usb", 0, 0, 0.2f}, [TAIL_LSB] = {"lsb", 0, 0, 0.2f}, [TAIL_BPSK31] = {"bpsk31", 0, 0, 0.5f}, [TAIL_RTTY] = {"rtty", 1, 0, 0.f},
    [TAIL_WFM] = {"wfm", 1, 0, 0.f},
};

typedef struct {
    const char *in_spec, *wf_sink;                                   /* --in; --waterfall SINK, NULL without a waterfall */
    int fmt, D, block, tail, device, ndev, devs[64];
    float bw, limit, agc_ref;                                        /* agc_ref 0: the tail's own default (kTails) */
    window_t window;
    int rs_I, rs_D, sps, rtty_B;                                     /* --resample I:D (rs_I 0: no resampler), --sps N of bpsk31, --rtty-bufsize */
    float rs_bw, wfm_rate, tau;                                      /* --resample's BW, --wfm-rate, --tau */
    csdrb_serial_line_params_t rtty;                                 /* --sps F, --databits, --stopbits of --tail rtty */
    float bfsk_spacing;                                              /* --bfsk SPACING:LENGTH of --tail rtty (bfsk_L 0: the discriminator) */
    int bfsk_L;
    int fm_atan;                                                     /* --fm-demod atan: fmdemod_atan_cf instead of the bank's quadri-correlator */
    waterfall_opts_t wf;
} opts_t;

/* --fm-demod atan: the bank gives complexf baseband rows, and fmdemod_atan_cf turns them into the discriminator rows of the resampler or the tail,
 * each channel's phase carried from call to call (phase[cur] in, phase[cur ^ 1] out: the bank's in and out must not alias; zero at stream start)
 *   bb : [C][bs] complexf, the new baseband samples from the front of every row */
typedef struct { complexf *d_bb; long bs; float *d_phase[2]; int cur; } atan_stage_t;

static void atan_stage_init(atan_stage_t *a, int C, int in_cap)
{
    a->bs = ((long)in_cap + 3) & ~3L;
    a->d_bb = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)a->bs);
    a->d_phase[0] = csdrb_device_alloc(sizeof(float) * (size_t)C);
    a->d_phase[1] = csdrb_device_alloc(sizeof(float) * (size_t)C);
    if (!a->d_bb || !a->d_phase[0] || !a->d_phase[1]) die("out of memory");
}

/* n new baseband samples per channel at the front of d_bb: their discriminator output to dst (row pitch in floats) */
static void atan_stage_push(atan_stage_t *a, int C, int n, float *dst, long pitch, void *stream)
{
    OK(csdrb_fmdemod_atan_bank_cf(a->d_bb, a->bs, dst, pitch, C, n, a->d_phase[a->cur], a->d_phase[a->cur ^ 1], stream));
    a->cur ^= 1;
}

/* ---- the tail interface: the only code past option validation that knows which tail runs ----------------------------------------------------
 * tail_in gives the device rows where the next bank outputs land (the resampler's input with --resample); tail_push runs the resampler if on
 * and the tail over the n samples per channel put there and writes the sinks; tail_push_host does both for rows in host memory (--devices).
 * All buffers are on ONE device: the single-GPU path's own, the first device of --devices. */
typedef struct {
    int kind, C, resample, atan;
    size_t esz;                                                      /* one bank output sample: float (demodulated) or complexf */
    atan_stage_t fm;
    rs_stage_t rs;
    union { nfm_tail_t nfm; raw_tail_t raw; bb_tail_t bb; bpsk_tail_t bpsk; rtty_tail_t rtty; wfm_tail_t wfm; } u;
} tail_t;

/* whether the bank demodulates: the tail's choice, except that --tail rtty --bfsk and --fm-demod atan take the complex baseband */
static int bank_demod(const opts_t *o) { return kTails[o->tail].demod && !o->bfsk_L && !o->fm_atan; }

/* --devices --tail none without --resample or --fm-demod atan: the rows collected on the host are the output, so that tail needs no device,
 * stream or buffer */
static int tail_host_fed(int kind, int resample, int atan) { return kind == TAIL_NONE && !resample && !atan; }

/* in_cap: the most samples per channel one block adds; stream NULL for a host-fed tail, which allocates nothing.  The per-tail inits fill the
 * state zeroed here. */
static void tail_init(tail_t *t, const opts_t *o, int C, int in_cap, void *stream)
{
    memset(t, 0, sizeof *t);
    t->kind = o->tail; t->C = C; t->resample = o->rs_I > 0; t->atan = o->fm_atan;
    t->esz = bank_demod(o) ? sizeof(float) : sizeof(complexf);
    if (!stream) return;
    if (t->atan) atan_stage_init(&t->fm, C, in_cap);
    if (t->resample) { rs_init(&t->rs, C, o->rs_I, o->rs_D, o->rs_bw, in_cap); in_cap = rs_out_cap(&t->rs); }
    switch (t->kind) {
    case TAIL_NFM: nfm_tail_init(&t->u.nfm, C, in_cap, o->limit, o->agc_ref); break;
    case TAIL_NONE: case TAIL_IQ: raw_tail_init(&t->u.raw, C, in_cap, t->kind == TAIL_NONE ? sizeof(float) : sizeof(complexf)); break;
    case TAIL_AM: bb_tail_init(&t->u.bb, C, in_cap, o->limit, o->agc_ref, NULL, stream); break;
    case TAIL_USB: bb_tail_init(&t->u.bb, C, in_cap, o->limit, o->agc_ref, (const float[2]){0.0f, 0.1f}, stream); break;
    case TAIL_LSB: bb_tail_init(&t->u.bb, C, in_cap, o->limit, o->agc_ref, (const float[2]){-0.1f, 0.0f}, stream); break;
    case TAIL_BPSK31: bpsk_tail_init(&t->u.bpsk, C, o->sps, in_cap, o->agc_ref, stream); break;
    case TAIL_RTTY:
        rtty_tail_init(&t->u.rtty, C, &o->rtty, o->rtty_B, in_cap);
        if (o->bfsk_L) rtty_bfsk_init(&t->u.rtty, o->bfsk_spacing, o->bfsk_L, in_cap, stream);
        break;
    case TAIL_WFM: wfm_tail_init(&t->u.wfm, C, o->wfm_rate, o->tau, in_cap); break;
    }
}

/* where the discriminator output (or, for iq, am, usb, lsb, bpsk31 and rtty --bfsk, the baseband) goes next */
static void *demod_in(tail_t *t, long *pitch)
{
    if (t->resample) { *pitch = t->rs.rs; return t->rs.d_in + t->rs.have; }
    switch (t->kind) {
    case TAIL_NFM: *pitch = t->u.nfm.ds; return t->u.nfm.d_demod + t->u.nfm.a_have;
    case TAIL_NONE: case TAIL_IQ: *pitch = t->u.raw.pitch; return t->u.raw.d_rows;
    case TAIL_AM: case TAIL_USB: case TAIL_LSB: *pitch = t->u.bb.bs; return t->u.bb.d_bb + t->u.bb.have;
    case TAIL_BPSK31: *pitch = t->u.bpsk.bs; return t->u.bpsk.d_in;
    case TAIL_RTTY:
        if (t->u.rtty.L) { *pitch = t->u.rtty.bs; return t->u.rtty.d_bb + t->u.rtty.bb_have; }
        *pitch = t->u.rtty.rs; return t->u.rtty.d_rows + t->u.rtty.end;
    case TAIL_WFM: default: *pitch = t->u.wfm.rs; return t->u.wfm.d_rows + t->u.wfm.have;
    }
}

static void *tail_in(tail_t *t, long *pitch)
{
    if (t->atan) { *pitch = t->fm.bs; return t->fm.d_bb; }
    return demod_in(t, pitch);
}

/* n new bank outputs per channel sit at tail_in: through the resampler if on, then the tail, output to the sinks */
static void tail_push(tail_t *t, channel_t *chan, int n, void *stream)
{
    if (t->atan) {
        long pitch;
        float *dst = demod_in(t, &pitch);
        atan_stage_push(&t->fm, t->C, n, dst, pitch, stream);
    }
    switch (t->kind) {
    case TAIL_NFM:
        if (t->resample) n = rs_push(&t->rs, n, t->u.nfm.d_demod + t->u.nfm.a_have, t->u.nfm.ds, stream);
        nfm_tail_push(&t->u.nfm, chan, n, stream);
        break;
    case TAIL_NONE: case TAIL_IQ:
        if (t->resample) n = rs_push(&t->rs, n, (float *)t->u.raw.d_rows, t->u.raw.pitch, stream);
        raw_tail_push(&t->u.raw, chan, n, stream);
        break;
    case TAIL_AM: case TAIL_USB: case TAIL_LSB: bb_tail_push(&t->u.bb, chan, n, stream); break;
    case TAIL_BPSK31: bpsk_tail_push(&t->u.bpsk, chan, n, stream); break;
    case TAIL_RTTY:
        if (t->u.rtty.L) rtty_bfsk_push(&t->u.rtty, chan, n, stream);
        else rtty_tail_push(&t->u.rtty, chan, n, stream);
        break;
    case TAIL_WFM: wfm_tail_push(&t->u.wfm, chan, n, stream); break;
    }
}

/* n bank outputs per channel in host rows of n samples: straight to the sinks for a host-fed tail, else to tail_in and tail_push */
static void tail_push_host(tail_t *t, channel_t *chan, const unsigned char *h_rows, int n, void *stream)
{
    const size_t width = t->esz * (size_t)n;
    if (tail_host_fed(t->kind, t->resample, t->atan)) { write_rows(chan, t->C, h_rows, width, NULL); return; }
    long pitch;
    void *d_in = tail_in(t, &pitch);
    OK(csdrb_copy2d_h2d(d_in, t->esz * (size_t)pitch, h_rows, width, width, (size_t)t->C, stream));
    tail_push(t, chan, n, stream);
}

static int run_multi(const opts_t *o, channel_t *chan, int C, const float *rates, const float *taps, int T, waterfall_t *wf)
{
    const int fmt = o->fmt, D = o->D, block = o->block;
    open_sinks(chan, C, wf);
    const int in_fd = open_input(o->in_spec);
    fprintf(stderr, "csdr-bankd: %d channels over %d devices, decimation %d, %d taps, %s input, blocks of %d samples, tail %s\n", C, o->ndev, D, T,
            kFormatNames[fmt], block, kTails[o->tail].name);
    csdrb_multi_bank_t *mb = csdrb_multi_bank_create(o->ndev, o->devs, C, rates, D, taps, T, bank_demod(o), 1024, block);
    if (!mb) die("cannot create the multi-GPU bank");
    const int n_out = (block - T) / D + 1, consumed = n_out * D, keep = block - consumed;
    /* the tail (and the resampler) is audio-rate work (C x the channel rate): the rows every device returned go to the FIRST device once more and
     * through the same tail as in the single-GPU path */
    tail_t tail;
    void *tail_stream = tail_host_fed(o->tail, o->rs_I > 0, o->fm_atan) ? NULL : device_stream(o->devs[0]);
    tail_init(&tail, o, C, n_out + 2, tail_stream);
    float lut[256];
    for (int i = 0; i < 256; i++) lut[i] = (float)((float)i / (UCHAR_MAX / 2.0) - 1.0);      /* convert_u8_f, libcsdr.c:2365 */
    complexf *h_wide[2] = {csdrb_host_alloc(sizeof(complexf) * (size_t)block), csdrb_host_alloc(sizeof(complexf) * (size_t)block)};
    unsigned char *h_out[2] = {csdrb_host_alloc(tail.esz * (size_t)C * (size_t)n_out), csdrb_host_alloc(tail.esz * (size_t)C * (size_t)n_out)};
    unsigned char *raw = malloc((size_t)block * (size_t)kWireBytes[fmt]);
    float *h_real = wf && o->wf.real ? csdrb_host_alloc(sizeof(float) * (size_t)block) : NULL;  /* --fft-real: the block's real samples */
    if (!h_wide[0] || !h_wide[1] || !h_out[0] || !h_out[1] || !raw || (wf && o->wf.real && !h_real)) die("out of memory");
    /* --waterfall: the block's fresh samples go to the first device once more, through the same bank as in the single-GPU path */
    void *wf_stream = wf ? device_stream(o->devs[0]) : NULL;
    if (wf) waterfall_init(wf, &o->wf, block, 1, wf_stream);
    long blocks = 0;
    int ticket[2] = {-1, -1};
    for (int first = 1;; first = 0) {
        const int slot = (int)(blocks & 1), fresh = first ? block : consumed;
        complexf *w = h_wide[slot];
        /* this buffer's previous block (two submits ago) must be done before it is overwritten; its results go out meanwhile */
        if (ticket[slot] >= 0) {
            if (csdrb_multi_bank_collect(mb, ticket[slot]) < 0) die("csdrb_multi_bank_collect failed");
            tail_push_host(&tail, chan, h_out[slot], n_out, tail_stream);
            ticket[slot] = -1;
        }
        if (!first) memcpy(w, h_wide[slot ^ 1] + consumed, sizeof(complexf) * (size_t)keep);   /* the unconsumed tail (csdr.c:1172-1174) */
        complexf *dst = w + (first ? 0 : keep);
        int ok;
        if (fmt == IN_F32) ok = read_block(in_fd, (unsigned char *)dst, sizeof(complexf) * (size_t)fresh);
        else {                                                     /* converted on the host: real samples become x + 0j */
            ok = read_block(in_fd, raw, (size_t)fresh * (size_t)kWireBytes[fmt]);
            const short *s16 = (const short *)raw;
            const float *f32 = (const float *)raw;
            const signed char *s8 = (const signed char *)raw;
            if (ok) for (int i = 0; i < fresh; i++) {
                if (fmt == IN_U8) { dst[i].i = lut[raw[2 * i]]; dst[i].q = lut[raw[2 * i + 1]]; }
                else if (fmt == IN_S8) { dst[i].i = (float)s8[2 * i] * S8_RECIP; dst[i].q = (float)s8[2 * i + 1] * S8_RECIP; }
                else if (fmt == IN_S16) { dst[i].i = (float)s16[2 * i] * S16_RECIP; dst[i].q = (float)s16[2 * i + 1] * S16_RECIP; }
                else if (fmt == IN_REAL_S16) { dst[i].i = (float)s16[i] * S16_RECIP; dst[i].q = 0.0f; }
                else { dst[i].i = f32[i]; dst[i].q = 0.0f; }
            }
        }
        if (!ok) break;
        if (wf && wf->real) {                                      /* the real floats the conversion produced, without the + 0j */
            for (int i = 0; i < fresh; i++) h_real[i] = dst[i].i;
            OK(csdrb_copy_h2d(wf->d_in, h_real, sizeof(float) * (size_t)fresh, wf_stream));
            waterfall_push(wf, wf->d_in, fresh, wf_stream);
        } else if (wf) {
            OK(csdrb_copy_h2d(wf->d_in, dst, sizeof(complexf) * (size_t)fresh, wf_stream));
            waterfall_push(wf, wf->d_in, fresh, wf_stream);
        }
        ticket[slot] = csdrb_multi_bank_submit(mb, w, block, h_out[slot], n_out);
        if (ticket[slot] < 0) die("csdrb_multi_bank_submit failed");
        blocks++;
    }
    for (int k = 0; k < 2; k++) {                                  /* drain in submission order */
        const int slot = (int)((blocks + k) & 1);
        if (ticket[slot] < 0) continue;
        if (csdrb_multi_bank_collect(mb, ticket[slot]) < 0) die("csdrb_multi_bank_collect failed");
        tail_push_host(&tail, chan, h_out[slot], n_out, tail_stream);
    }
    fprintf(stderr, "csdr-bankd: end of input after %ld blocks on %d devices, %ld kernel launches\n", blocks, o->ndev, csdrb_kernel_launches());
    if (wf_stream) csdrb_stream_destroy(wf_stream);
    csdrb_multi_bank_destroy(mb);
    close_sinks(chan, C, wf);
    return 0;
}

static int usage(void)
{
    fprintf(stderr,
            "usage: csdr-bankd [--in -|HOST:PORT] [--u8|--s8|--f32|--s16|--real-s16|--real-f32] [--decimation D] [--bw TRANSITION_BW] [--window W]\n"
            "                  [--block SAMPLES]\n"
            "                  [--tail nfm|none|am|usb|lsb|iq|bpsk31|rtty|wfm] [--sps N] [--databits N] [--stopbits S] [--rtty-bufsize B]\n"
            "                  [--bfsk SPACING:LENGTH] [--fm-demod quadri|atan]\n"
            "                  [--wfm-rate R] [--tau T] [--resample I:D[:BW]] [--limit L] [--agc-ref R] [--device N | --devices N0,N1,...]\n"
            "                  RATE:SINK [RATE:SINK ...]\n"
            "  --u8 | --f32 | --s16 the complex input: rtl_sdr's u8 IQ (default), complex float, or complex s16 (Airspy INT16_IQ, SDRplay, ...)\n"
            "  --s8                 HackRF's signed 8-bit IQ (hackrf_transfer -r -), convert_s8_f in front of the bank.  Three NFM channels\n"
            "                       at 10 Msps (50 kHz channels, resampled to 48 kHz):\n"
            "                       hackrf_transfer -r - -s 10000000 -f 145500000 | csdr-bankd --s8 --decimation 200 --resample 24:25\n"
            "                       -0.05:a.s16 0.0:b.s16 0.1:c.s16\n"
            "  --real-s16 | --real-f32  a REAL stream from a direct-sampling receiver (RX888 / SDDC, Airspy real modes, ADC boards): per channel\n"
            "                       convert_s16_f | shift_addition_fc RATE | fir_decimate_cc D bw | <tail>.  A station at f Hz of a real stream\n"
            "                       sampled at fs is tuned with RATE = -f/fs; +f/fs gives it conjugated (sidebands swapped, discriminator negated).\n"
            "                       FT8 at 7.074 MHz from an RX888 at 64.8 Msps, 48 kHz baseband:\n"
            "                       csdr-bankd --real-s16 --decimation 1350 --bw 0.0008 --tail usb -0.10916667:ft8.s16\n"
            "                       Its waterfall is fft_fc's one-sided spectrum: --waterfall SINK --fft-real (below).\n"
            "  --tail wfm           broadcast FM: per channel fmdemod_quadri_cf | fractional_decimator_ff R | deemphasis_wfm_ff 48000 T | convert_f_s16,\n"
            "                       in the CLI's calls of 1024 samples; the sinks get s16 audio.  --wfm-rate R (default 5, above 1 and at most 16)\n"
            "                       takes wideband/decimation to 48 kHz; --tau T (default 50e-6; 75e-6 in the Americas).  Not with --resample.\n"
            "                       Three stations at 2.4 Msps (240 kHz channels, 79 taps = 8 per output period, which the fused bank serves):\n"
            "                       rtl_sdr -s 2400000 -f 89300000 - | csdr-bankd --decimation 10 --bw 0.05 --tail wfm -0.085:a.s16 0.0:b.s16 0.2:c.s16\n"
            "                       The whole 88-108 MHz band at 20 Msps, about 100 stations (250 kHz channels, 999 taps = 13 per output period):\n"
            "                       ... | csdr-bankd --decimation 80 --bw 0.004 --tail wfm --wfm-rate 5.2083333 -0.45:s1.s16 -0.44:s2.s16 ...\n"
            "  --tail bpsk31 --sps N  per channel simple_agc_cc 0.001 R | timing_recovery_cc GARDNER N 0.5 2 --add_q | dbpsk_decoder_c_u8 |\n"
            "                       psk31_varicode_decoder_u8_u8 (R = --agc-ref, default 0.5) behind the baseband; the sinks get the decoded text.\n"
            "                       N is samples per symbol at the baseband rate, > 4 and divisible by 4.  A PSK31 skimmer at 2.4 Msps:\n"
            "                       csdr-bankd --decimation 300 --bw 0.001 --tail bpsk31 --sps 256 -0.1:ch1.txt 0.05:ch2.txt 0.2:ch3.txt\n"
            "                       (8 kHz baseband, 4001 taps = 14 per output period, which the fused bank serves; 31.25 Bd)\n"
            "  --tail rtty --sps F    per channel fmdemod_quadri_cf | serial_line_decoder_f_u8 F N S | rtty_baudot2ascii_u8_u8 (--databits N, default 5;\n"
            "                       --stopbits S, default 1.5); the sinks get the decoded text.  F is samples per bit at the baseband rate (a float).\n"
            "                       The decoder runs in calls of --rtty-bufsize B samples (default 16384, the CLI's), so the text lags the signal\n"
            "                       by up to B samples; B must exceed F*(1 + N + S) + 2.  An RTTY skimmer at 2.4 Msps:\n"
            "                       csdr-bankd --decimation 1200 --bw 0.001 --tail rtty --sps 44 -0.1:ch1.txt 0.05:ch2.txt 0.2:ch3.txt\n"
            "                       (2 kHz baseband, 4001 taps = 4 per output period, which the fused bank serves; 45.45 Bd; about 8 s of lag)\n"
            "  --bfsk SPACING:LENGTH  with --tail rtty: tone filters instead of the discriminator, bfsk_demod_cf SPACING LENGTH per channel on the\n"
            "                       complex baseband (peaks at +-SPACING/2 cycles per baseband sample, Hamming, LENGTH taps, 2..4096).  They hold\n"
            "                       up in noise below the discriminator's threshold.  170 Hz shift at 2 kHz baseband (2.4 Msps, --decimation 1200):\n"
            "                       csdr-bankd --decimation 1200 --bw 0.001 --tail rtty --sps 44 --bfsk 0.085:44 -0.1:ch1.txt 0.05:ch2.txt\n"
            "  --fm-demod quadri|atan  the FM discriminator of --tail nfm, none, wfm and rtty.  quadri (default): the bank's fmdemod_quadri_cf,\n"
            "                       K*|z[n-1]|/|z[n]|*sin(dphi) with K = 0.3404, which bends loud broadcast FM (75 kHz deviation at 240 kHz\n"
            "                       channels: harmonics about -13 dB).  atan: fmdemod_atan_cf on the bank's baseband, dphi/pi, straight up to\n"
            "                       +-pi.  At small deviation its level is about 7 %% lower than quadri's (1/pi against K): the none and wfm\n"
            "                       outputs come out that much quieter, the NFM AGC absorbs it.  Not with --bfsk or the baseband tails.  Broadcast FM:\n"
            "                       rtl_sdr -s 2400000 -f 89300000 - | csdr-bankd --decimation 10 --bw 0.05 --tail wfm --fm-demod atan 0.0:a.s16\n"
            "  --resample I:D[:BW]  rational_resampler_ff I D BW (BW default 0.05) right behind the discriminator, for --tail nfm and none: brings\n"
            "                       wideband/decimation to the 48 kHz the NFM de-emphasis is designed for (e.g. 2.048 Msps, --decimation 32,\n"
            "                       --resample 3:4).  With T = taps of BW, the daemon needs (T/I + 1)*I >= 2*D + I - 1 (T >= 2*D + I - 2 suffices),\n"
            "                       so that no resampler call ends on its output cap; other geometries are refused.\n"
            "  --waterfall SINK     the wideband waterfall beside the channels: fft_cc N E W | logaveragepower_cf X N A | fft_exchange_sides_ff N\n"
            "                       [| compress_fft_adpcm_f_u8 N] on the whole input stream, lines to SINK (a path, FIFO or tcp:PORT), with\n"
            "                       --fft-size N (default 2048, a power of two up to 16384), --fft-every E (default N), --fft-averages A\n"
            "                       (default 1), --fft-add-db X (default -70), --fft-window W (default HAMMING) and --fft-compression\n"
            "                       adpcm|none (default adpcm: (N + 10) / 2 bytes per line; none: N floats of dB).  A slow sink loses whole\n"
            "                       lines only.  At 2.4 Msps, about 9 lines/s of 4096 bins:\n"
            "                       csdr-bankd --waterfall wf.fifo --fft-size 4096 --fft-every 4096 --fft-averages 64 -0.1:ch1.s16 0.2:ch2.s16\n"
            "  --fft-real           with --real-s16 | --real-f32: the real stream's waterfall fft_fc N E W | logaveragepower_cf X N A\n"
            "                       [| compress_fft_adpcm_f_u8 N] instead: N bins (2N real samples per frame) from DC up, --fft-every E in\n"
            "                       real samples (default 2N).  The whole HF band from an RX888 beside an FT8 channel:\n"
            "                       csdr-bankd --real-s16 --decimation 1350 --bw 0.0008 --tail usb --waterfall wf.bin --fft-real --fft-size 16384\n"
            "                       -0.10916667:ft8.s16\n"
            "  see the head of csdr_b200/host/bankd.c for the other options\n");
    return 2;
}

int main(int argc, char **argv)
{
    const char *tail = "nfm";
    opts_t o = {.in_spec = "-", .fmt = IN_U8, .D = 50, .block = 1 << 18, .bw = 0.005f, .limit = 1.0f, .window = WINDOW_HAMMING,
                .rs_bw = 0.05f,                                      /* rational_resampler_ff's default transition bandwidth (csdr.c:1423) */
                .rtty = {0.f, 5, 1.5f, 0.4f}, .rtty_B = 16384,       /* bit_sampling_width_ratio (csdr.c:2510), the CLI's big buffer (csdr.c:190) */
                .wfm_rate = 5.0f, .tau = 50e-6f,                     /* the README.md:66 graph (75e-6 in the Americas) */
                .wf = {2048, 0, 1, 1, -70.0f, WINDOW_DEFAULT}};      /* --fft-every 0 stands for N */
    int rtty_opts = 0, wfm_opts = 0, wf_opts = 0;
    channel_t *chan = calloc((size_t)argc, sizeof *chan);
    int C = 0;
    for (int a = 1; a < argc; a++) {
        const char *arg = argv[a];
        const char *v = a + 1 < argc ? argv[a + 1] : NULL;
        if (!strcmp(arg, "--u8")) o.fmt = IN_U8;
        else if (!strcmp(arg, "--s8")) o.fmt = IN_S8;
        else if (!strcmp(arg, "--f32")) o.fmt = IN_F32;
        else if (!strcmp(arg, "--s16")) o.fmt = IN_S16;
        else if (!strcmp(arg, "--real-s16")) o.fmt = IN_REAL_S16;
        else if (!strcmp(arg, "--real-f32")) o.fmt = IN_REAL_F32;
        else if (!strcmp(arg, "--in") && v) { o.in_spec = v; a++; }
        else if (!strcmp(arg, "--decimation") && v) { o.D = atoi(v); a++; }
        else if (!strcmp(arg, "--bw") && v) { o.bw = (float)atof(v); a++; }
        else if (!strcmp(arg, "--window") && v) { o.window = firdes_get_window_from_string((char *)v); a++; }
        else if (!strcmp(arg, "--block") && v) { o.block = atoi(v); a++; }
        else if (!strcmp(arg, "--tail") && v) { tail = v; a++; }
        else if (!strcmp(arg, "--limit") && v) { o.limit = (float)atof(v); a++; }
        else if (!strcmp(arg, "--agc-ref") && v) { o.agc_ref = (float)atof(v); a++; }
        else if (!strcmp(arg, "--sps") && v) { o.sps = atoi(v); o.rtty.samples_per_bits = (float)atof(v); a++; }
        else if (!strcmp(arg, "--databits") && v) { o.rtty.databits = atoi(v); rtty_opts = 1; a++; }
        else if (!strcmp(arg, "--stopbits") && v) { o.rtty.stopbits = (float)atof(v); rtty_opts = 1; a++; }
        else if (!strcmp(arg, "--rtty-bufsize") && v) { o.rtty_B = atoi(v); rtty_opts = 1; a++; }
        else if (!strcmp(arg, "--bfsk") && v) {
            if (sscanf(v, "%f:%d", &o.bfsk_spacing, &o.bfsk_L) != 2) die("--bfsk takes SPACING:LENGTH, e.g. 0.085:44");
            if (!(o.bfsk_spacing > 0.f && o.bfsk_spacing < 1.f)) die("--bfsk SPACING is the mark-space shift in cycles per baseband sample, between 0 and 1");
            if (o.bfsk_L < 2 || o.bfsk_L > 4096) die("--bfsk LENGTH must be between 2 and 4096 taps");
            a++;
        }
        else if (!strcmp(arg, "--fm-demod") && v) {
            if (!strcmp(v, "atan")) o.fm_atan = 1;
            else if (!strcmp(v, "quadri")) o.fm_atan = 0;
            else die("--fm-demod is quadri or atan");
            a++;
        }
        else if (!strcmp(arg, "--wfm-rate") && v) { o.wfm_rate = (float)atof(v); wfm_opts = 1; a++; }
        else if (!strcmp(arg, "--tau") && v) { o.tau = (float)atof(v); wfm_opts = 1; a++; }
        else if (!strcmp(arg, "--waterfall") && v) { o.wf_sink = v; a++; }
        else if (!strcmp(arg, "--fft-size") && v) { o.wf.fft_size = atoi(v); wf_opts = 1; a++; }
        else if (!strcmp(arg, "--fft-every") && v) { o.wf.every = atoi(v); wf_opts = 1; if (o.wf.every < 1) die("--fft-every must be at least 1"); a++; }
        else if (!strcmp(arg, "--fft-averages") && v) { o.wf.averages = atoi(v); wf_opts = 1; a++; }
        else if (!strcmp(arg, "--fft-add-db") && v) { o.wf.add_db = (float)atof(v); wf_opts = 1; a++; }
        else if (!strcmp(arg, "--fft-real")) { o.wf.real = 1; wf_opts = 1; }
        else if (!strcmp(arg, "--fft-window") && v) { o.wf.window = firdes_get_window_from_string((char *)v); wf_opts = 1; a++; }
        else if (!strcmp(arg, "--fft-compression") && v) {
            if (!strcmp(v, "adpcm")) o.wf.compress = 1;
            else if (!strcmp(v, "none")) o.wf.compress = 0;
            else die("--fft-compression is adpcm or none");
            wf_opts = 1; a++;
        }
        else if (!strcmp(arg, "--device") && v) { o.device = atoi(v); a++; }
        else if (!strcmp(arg, "--devices") && v) { o.ndev = parse_devices(v, o.devs, 64); if (o.ndev <= 0) die("--devices wants N0,N1,..."); a++; }
        else if (!strcmp(arg, "--resample") && v) {
            if (sscanf(v, "%d:%d:%f", &o.rs_I, &o.rs_D, &o.rs_bw) < 2 || o.rs_I < 1 || o.rs_D < 1) die("--resample wants I:D[:BW] with positive integers I and D");
            a++;
        }
        else if (!strcmp(arg, "--help")) return usage();
        else if (strchr(arg, ':') && (arg[0] != '-' || arg[1] == '.' || (arg[1] >= '0' && arg[1] <= '9'))) {      /* RATE:SINK, RATE may be negative */
            char *end = NULL;
            chan[C].rate = strtof(arg, &end);
            if (!end || *end != ':') die("channels are RATE:SINK");
            chan[C].sink = end + 1; chan[C].fd = -1; chan[C].dropped = 0; C++;
        } else { fprintf(stderr, "csdr-bankd: unknown argument %s\n", arg); return 2; }
    }
    o.tail = -1;
    for (int k = 0; k < (int)(sizeof kTails / sizeof *kTails); k++) if (!strcmp(tail, kTails[k].name)) o.tail = k;
    if (o.tail < 0) die("--tail is nfm, none, iq, am, usb, lsb, bpsk31, rtty or wfm");
    if (o.tail == TAIL_BPSK31) {
        if (o.sps <= 4 || (o.sps & 3)) die("--tail bpsk31 needs --sps N with N > 4 and divisible by 4 (timing_recovery_cc's decimation)");
    } else if (o.tail == TAIL_RTTY) {
        const float spb = o.rtty.samples_per_bits;
        if (!(spb >= 1.f && spb <= 1e6f)) die("--tail rtty needs --sps F, samples per bit at the baseband rate, at least 1 (serial_line_decoder_f_u8's range)");
        if (spb < 5.f) fprintf(stderr, "csdr-bankd: warning: serial_line_decoder_f_u8 does not work well below 5 samples per bit\n");
        if (o.rtty.databits < 1 || o.rtty.databits > 8) die("--databits must be between 1 and 8");
        if (!(o.rtty.stopbits >= 1.f && o.rtty.stopbits <= 1000.f)) die("--stopbits must be at least 1");
        if (o.rtty_B < 1 || o.rtty_B > (1 << 22)) die("--rtty-bufsize must be between 1 and 4194304 samples");
        /* a character that starts at the third sample of a call and does not fit makes the call consume nothing: the CLI exits "stuck" */
        if (spb * ((float)(1 + o.rtty.databits) + o.rtty.stopbits) + 2.0f >= (float)o.rtty_B)
            die("--rtty-bufsize must exceed sps*(1 + databits + stopbits) + 2: a call could not hold one character and would get stuck");
    } else if (o.sps) die("--sps belongs to --tail bpsk31 and --tail rtty");
    if (o.tail != TAIL_RTTY && rtty_opts) die("--databits, --stopbits and --rtty-bufsize belong to --tail rtty");
    if (o.tail != TAIL_RTTY && o.bfsk_L) die("--bfsk belongs to --tail rtty");
    if (o.fm_atan && !kTails[o.tail].demod) die("--fm-demod atan works with --tail nfm, none, wfm and rtty only (the iq, am, usb, lsb and bpsk31 tails take the baseband)");
    if (o.fm_atan && o.bfsk_L) die("--fm-demod atan and --bfsk are two different demodulators: choose one");
    if (o.tail == TAIL_WFM) {
        /* above 16 a decimator call could consume more than its 1024 samples (the reference then memmoves a negative length): WFM needs about 5 */
        if (!(o.wfm_rate > 1.0f && o.wfm_rate <= 16.0f)) die("--wfm-rate must be above 1 and at most 16 (wideband rate / decimation / 48 kHz)");
        if (!(o.tau > 0.0f)) die("--tau must be positive (50e-6 in Europe, 75e-6 in the Americas)");
    } else if (wfm_opts) die("--wfm-rate and --tau belong to --tail wfm");
    if (o.agc_ref == 0.0f) o.agc_ref = kTails[o.tail].agc_ref;
    if (C == 0) die("no channels (RATE:SINK ...)");
    if (o.block <= 0 || (o.block & 1)) die("--block must be a positive even number of samples");
    if (o.D <= 0 || (o.D & 1)) die("--decimation must be a positive even number (the fused bank serves even decimations only)");
    if (!(o.bw > 0.f && o.bw < 0.5f)) die("--bw must be a transition bandwidth between 0 and 0.5");
    if (!(o.limit > 0.f) || !(o.agc_ref >= 0.f)) die("--limit and --agc-ref must be positive");
    if (o.rs_I > 0) {
        if (!kTails[o.tail].resample) die("--resample works with --tail nfm and --tail none only (the am, usb, lsb, iq, bpsk31, rtty and wfm tails are not resampled)");
        if (!(o.rs_bw > 0.f && o.rs_bw < 0.5f)) die("--resample: the transition bandwidth must be between 0 and 0.5");
        const int rs_T = firdes_filter_len(o.rs_bw);
        if (!resample_geometry_ok(o.rs_I, o.rs_D, rs_T)) {
            fprintf(stderr, "csdr-bankd: --resample %d:%d with %d taps: a resampler call could end on its output cap and repeat an output; "
                            "the daemon needs (T/I + 1)*I >= 2*D + I - 1 (T >= 2*D + I - 2 suffices): lower the transition bandwidth\n", o.rs_I, o.rs_D, rs_T);
            return 1;
        }
    }
    const int fmt = o.fmt, D = o.D, block = o.block, real = fmt == IN_REAL_S16 || fmt == IN_REAL_F32;
    if (real && o.wf_sink && !o.wf.real)
        die("--waterfall needs a complex input; the waterfall of a real stream is fft_fc's one-sided spectrum: add --fft-real");
    if (o.wf.real && !real) die("--fft-real takes a real input (--real-s16 or --real-f32)");
    if (wf_opts && !o.wf_sink) die("--fft-size, --fft-every, --fft-averages, --fft-add-db, --fft-window, --fft-compression and --fft-real belong to --waterfall");
    waterfall_t wf, *wfp = NULL;
    memset(&wf, 0, sizeof wf);
    if (o.wf_sink) {
        if (o.wf.every == 0) o.wf.every = o.wf.real ? 2 * o.wf.fft_size : o.wf.fft_size;      /* fft_fc's frame is 2N real samples */
        if (o.wf.averages < 1) die("--fft-averages must be at least 1");
        const csdrb_spectrum_params_t p = {o.wf.fft_size, o.wf.every, o.wf.averages, o.wf.compress, o.wf.add_db};
        const csdrb_spectrum_state_t s0 = {0, 0};
        if (csdrb_spectrum_bank_lines(&p, &s0, 0) < 0) die(o.wf.real ? "--fft-size must be a power of two from 2 to 16384 (bins)" : "--fft-size must be a power of two from 2 to 16384");
        wf.sink.rate = 0.f; wf.sink.sink = o.wf_sink; wf.sink.fd = -1;
        wfp = &wf;
    }
    signal(SIGPIPE, SIG_IGN);

    /* ---- filter and bank ---------------------------------------------------------------------------------------------------- */
    const int T = firdes_filter_len(o.bw);
    float *taps = malloc(sizeof(float) * (size_t)T);
    firdes_lowpass_f(taps, T, 0.5f / (float)D, o.window);
    if (block < 2 * T) die("--block is shorter than two filter lengths");
    float *rates = malloc(sizeof(float) * (size_t)C);
    for (int c = 0; c < C; c++) rates[c] = chan[c].rate;
    if (o.ndev > C) die("more devices than channels");
    if (o.ndev > 0) return run_multi(&o, chan, C, rates, taps, T, wfp);
    void *stream = device_stream(o.device);
    csdrb_ddc_bank_t *bank = csdrb_ddc_bank_create(C, rates, D, taps, T, bank_demod(&o), 1024);   /* 1024 = the CLI's shift_addition_cc call size (csdr.c:911) */
    if (!bank) die("cannot create the bank");

    /* ---- buffers ----------------------------------------------------------------------------------------------------------------
     * wide[2]  : [tail of the previous block | new block] cf32 (f32 for a real input), ping-pong so the tail copy never overlaps
     * raw      : the block as it arrived, for the formats converted on the device; stage: real s16 converted where the block lands unaligned
     * the bank writes straight into the tail's input rows (tail_in) */
    const size_t in_bytes = (size_t)block * (size_t)kWireBytes[fmt];
    const size_t ssz = real ? sizeof(float) : sizeof(complexf);   /* one wideband sample on the device */
    unsigned char *h_in = csdrb_host_alloc(in_bytes);
    const int wide_cap = block + T + D + 16;
    unsigned char *d_wide[2] = {csdrb_device_alloc(ssz * (size_t)wide_cap), csdrb_device_alloc(ssz * (size_t)wide_cap)};
    const int raw_in = fmt == IN_U8 || fmt == IN_S8 || fmt == IN_S16 || fmt == IN_REAL_S16;
    unsigned char *d_raw = raw_in ? csdrb_device_alloc(in_bytes + 16) : NULL;
    float *d_stage = fmt == IN_REAL_S16 ? csdrb_device_alloc(sizeof(float) * (size_t)block + 16) : NULL;
    const int out_cap = wide_cap / D + 2;                          /* bank outputs one block can add */
    tail_t tl;
    tail_init(&tl, &o, C, out_cap, stream);
    if (!h_in || !d_wide[0] || !d_wide[1] || (raw_in && !d_raw) || (fmt == IN_REAL_S16 && !d_stage)) die("out of memory");
    if (wfp) waterfall_init(wfp, &o.wf, block, 0, stream);

    open_sinks(chan, C, wfp);
    const int in_fd = open_input(o.in_spec);
    fprintf(stderr, "csdr-bankd: %d channels, decimation %d, %d taps, %s input, blocks of %d samples, tail %s\n", C, D, T, kFormatNames[fmt], block,
            kTails[o.tail].name);

    int cur = 0, keep = 0;
    long blocks = 0;
    /* Every call presents exactly `block` samples: the unconsumed tail plus as many new ones as the previous call consumed -- how csdr.c:1172-1174
     * feeds fir_decimate_cc.  A constant size keeps the bank's look-ahead pre-pass valid from block to block (a size that wobbles with
     * block % D made it miss, and re-run inline, on most blocks). */
    for (;;) {
        const int fresh_n = block - keep;                            /* first block: everything; later: what the last call consumed (even) */
        const size_t fresh_bytes = (size_t)fresh_n * (size_t)kWireBytes[fmt];
        if (!read_block(in_fd, h_in, fresh_bytes)) break;
        /* 1. the new samples land behind the unconsumed tail.  keep is even because block and D are: 16-byte alignment holds for complex samples,
         *    but a real block can land 8 bytes off, where convert_s16_f (16-byte aligned buffers) converts into the stage and the block is copied */
        float *fresh = (float *)(d_wide[cur] + ssz * (size_t)keep);
        if (raw_in) OK(csdrb_copy_h2d(d_raw, h_in, fresh_bytes, stream));
        if (fmt == IN_U8) OK(csdrb_convert_u8_f(d_raw, fresh, 2L * fresh_n, stream));
        else if (fmt == IN_S8) OK(csdrb_convert_s8_f((const signed char *)d_raw, fresh, 2L * fresh_n, stream));
        else if (fmt == IN_S16) OK(csdrb_convert_s16_f((const short *)d_raw, fresh, 2L * fresh_n, stream));
        else if (fmt == IN_REAL_S16 && !((size_t)fresh & 15)) OK(csdrb_convert_s16_f((const short *)d_raw, fresh, fresh_n, stream));
        else if (fmt == IN_REAL_S16) {
            OK(csdrb_convert_s16_f((const short *)d_raw, d_stage, fresh_n, stream));
            OK(csdrb_copy_d2d(fresh, d_stage, sizeof(float) * (size_t)fresh_n, stream));
        } else OK(csdrb_copy_h2d(fresh, h_in, fresh_bytes, stream));
        if (wfp) waterfall_push(wfp, fresh, fresh_n, stream);       /* the waterfall of the same samples (cf32, or f32 with --fft-real), lines to its sink */
        const int n_in = block;

        /* 2. shift | fir_decimate | fmdemod for every channel, the new outputs straight into the tail's input rows */
        long pitch;
        void *dst = tail_in(&tl, &pitch);
        const int n_out = real ? csdrb_ddc_bank_process_f(bank, (const float *)d_wide[cur], n_in, dst, pitch, stream)
                               : csdrb_ddc_bank_process(bank, (const complexf *)d_wide[cur], n_in, dst, pitch, stream);
        if (n_out < 0) die("csdrb_ddc_bank_process failed");
        const int consumed = n_out * D;
        keep = n_in - consumed;
        OK(csdrb_copy_d2d(d_wide[cur ^ 1], d_wide[cur] + ssz * (size_t)consumed, ssz * (size_t)keep, stream));
        cur ^= 1;

        /* 3. the resampler if on, the tail, its output to the sinks */
        tail_push(&tl, chan, n_out, stream);
        blocks++;
    }
    OK(csdrb_stream_synchronize(stream));
    fprintf(stderr, "csdr-bankd: end of input after %ld blocks, %ld kernel launches\n", blocks, csdrb_kernel_launches());
    close_sinks(chan, C, wfp);
    csdrb_ddc_bank_destroy(bank);
    csdrb_stream_destroy(stream);
    return 0;
}
