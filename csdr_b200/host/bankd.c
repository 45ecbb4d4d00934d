/*
 * bankd.c -- csdr-bankd: a whole bank of FM, AM or SSB receivers on ONE wideband IQ stream, in one process.
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
 * usage: csdr-bankd [--in -|HOST:PORT] [--u8|--f32] [--decimation D] [--bw TRANSITION_BW] [--window W] [--block SAMPLES]
 *                   [--tail nfm|none|am|usb|lsb|iq] [--limit L] [--agc-ref R] [--device N | --devices N0,N1,...]  RATE:SINK [RATE:SINK ...]
 *   --tail: nfm (default) the README.md:87 tail, s16; none the raw discriminator output, f32; am / usb / lsb the AM and SSB graphs of README.md:95 and :110
 *   behind the DDC's complex baseband (see bb_tail_t), s16; iq the complex baseband itself, cf32.  --limit is limit_ff's amplitude (default 1), --agc-ref
 *   the AGC reference (default: fastagc_ff's 1.0 for nfm, agc_ff's 0.2 for am/usb/lsb).
 *   RATE  shift_addition_cc rate (fraction of the wideband sample rate), SINK a path (file or FIFO) or tcp:PORT (one listener).
 *   --devices: the channels are sliced over several GPUs of this node (csdrb_multi_bank_*: the block goes to the first device once and on to
 *   the others by NCCL broadcast), one block of latency more (two blocks are kept in flight); the audio tail (nfm, am, usb, lsb), audio-rate work, runs on
 *   the first device for all channels, through the same kernels as without --devices.
 * Sinks never hold the stream up: a sink that cannot take a block within 200 ms loses the rest of that block (counted on stderr at exit), one
 * that fails is dropped -- nmux's policy for slow clients (tsmpool.cpp:101-117, nmux.cpp:339-346).
 */
#define _GNU_SOURCE
#include "csdr_b200.h"

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
    memset(t, 0, sizeof *t);
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
        OK(csdrb_copy2d_d2d(t->d_carry, sizeof(float) * (size_t)Tn, t->d_demod + m, sizeof(float) * (size_t)ds, sizeof(float) * (size_t)Tn, (size_t)C, stream));
        OK(csdrb_copy2d_d2d(t->d_demod, sizeof(float) * (size_t)ds, t->d_carry, sizeof(float) * (size_t)Tn, sizeof(float) * (size_t)Tn, (size_t)C, stream));
        t->a_have = Tn;
    } else t->a_have = a_n;
    /* fastagc_ff over the whole AGC blocks available, then convert_f_s16 (one pass); the remainder waits for the next block */
    const int g_n = t->g_have + m, nb = g_n / AGC_BLOCK, whole = nb * AGC_BLOCK;
    if (nb > 0) {
        OK(csdrb_fastagc_bank_f_s16(t->d_agc_in, gs, t->d_pcm, whole, C, AGC_BLOCK, nb, t->agc_ref, t->d_agc_state, t->d_agc_hist, t->d_agc_scratch, t->agc_sb + 16, stream));
        OK(csdrb_copy_d2h(t->h_out, t->d_pcm, sizeof(short) * (size_t)C * (size_t)whole, stream));
        const int rest = g_n - whole;
        OK(csdrb_copy2d_d2d(t->d_carry, sizeof(float) * (size_t)AGC_BLOCK, t->d_agc_in + whole, sizeof(float) * (size_t)gs, sizeof(float) * (size_t)rest, (size_t)C, stream));
        OK(csdrb_copy2d_d2d(t->d_agc_in, sizeof(float) * (size_t)gs, t->d_carry, sizeof(float) * (size_t)AGC_BLOCK, sizeof(float) * (size_t)rest, (size_t)C, stream));
        t->g_have = rest;
        OK(csdrb_stream_synchronize(stream));
        for (int c = 0; c < C; c++) write_sink(&chan[c], t->h_out + sizeof(short) * (size_t)c * (size_t)whole, sizeof(short) * (size_t)whole);
    } else {
        t->g_have = g_n;
        OK(csdrb_stream_synchronize(stream));
    }
}

/* ---- the AM and SSB audio tails (README.md:95, :110) behind the DDC bank's complex baseband ------------------------------------------------------------------
 *   am      : amdemod_cf | fastdcblock_ff 1024 | agc_ff | limit_ff L | convert_f_s16
 *   usb/lsb : bandpass_fir_fft_cc 0 0.1 0.05 (or -0.1 0 0.05) | realpart_cf | agc_ff | limit_ff L | convert_f_s16
 *   iq      : the baseband itself, cf32 (what either tail starts from)
 * agc_ff runs with the CLI defaults (csdr.c:1342-1361) and its 1024-sample calls; --agc-ref overrides the reference.  Device buffers of ONE device:
 *   bb   : [C][bs] complexf : [remainder (< unit samples) | new baseband]   unit = 1024 (am) or the overlap-add input size (usb/lsb)
 *   mid  : [C][bs] float (am: DC-blocked envelope) or complexf (usb/lsb: filtered baseband) over the whole units
 *   pcm  : [C][whole] s16 */
#define SSB_BW 0.05f                                      /* bandpass_fir_fft_cc transition bandwidth of README.md:110 */
enum { TAIL_NFM, TAIL_NONE, TAIL_IQ, TAIL_AM, TAIL_USB, TAIL_LSB };

typedef struct {
    int kind, C, unit, have, fft_size;
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

static void bb_tail_init(bb_tail_t *t, int kind, int C, int out_cap, float limit, float agc_ref, void *stream)
{
    memset(t, 0, sizeof *t);
    t->kind = kind; t->C = C; t->limit = limit;
    csdrb_agc_params_t p = {0.2f, 0.01f, 0.0001f, 65536.0f, 200, 0, 0.999f, 1024};
    if (agc_ref > 0.f) p.reference = agc_ref;
    t->agc = p;
    t->unit = 1024;
    if (kind == TAIL_USB || kind == TAIL_LSB) {                  /* bandpass_fir_fft_cc geometry, csdr.c:1822-1831 */
        const int T = firdes_filter_len(SSB_BW);
        int N = next_pow2(T);
        if (N - T < 200) N <<= 1;
        t->fft_size = N; t->unit = N - T + 1;
        complexf *h_taps = calloc((size_t)N, sizeof(complexf));
        if (!h_taps) die("out of memory");
        if (kind == TAIL_USB) firdes_bandpass_c(h_taps, T, 0.0f, 0.1f, WINDOW_HAMMING);
        else firdes_bandpass_c(h_taps, T, -0.1f, 0.0f, WINDOW_HAMMING);
        complexf *d_taps = csdrb_device_alloc(sizeof(complexf) * (size_t)N);
        t->d_taps_fft = csdrb_device_alloc(sizeof(complexf) * (size_t)N);
        t->d_ola_tail = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)N);
        if (!d_taps || !t->d_taps_fft || !t->d_ola_tail) die("out of memory");
        OK(csdrb_copy_h2d(d_taps, h_taps, sizeof(complexf) * (size_t)N, stream));
        OK(csdrb_fft_c2c_batch(d_taps, N, t->d_taps_fft, N, N, 1, 0, stream));       /* the forward FFT of the zero-padded taps (csdr.c:1869) */
        complexf *zeros = calloc((size_t)C * (size_t)N, sizeof(complexf));   /* the overlap tail is zero at stream start (csdr.c:1860) */
        if (!zeros) die("out of memory");
        OK(csdrb_copy_h2d(t->d_ola_tail, zeros, sizeof(complexf) * (size_t)C * (size_t)N, stream));
        OK(csdrb_stream_synchronize(stream));
        csdrb_device_free(d_taps); free(h_taps); free(zeros);
    }
    t->bs = ((long)t->unit + out_cap + 3) & ~3L;
    t->d_bb = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->bs);
    t->d_carry = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->unit);
    t->d_mid = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->bs);
    t->d_pcm = csdrb_device_alloc(sizeof(short) * (size_t)C * (size_t)t->bs + 16);
    t->d_last_dc = csdrb_device_alloc(sizeof(float) * (size_t)C);
    t->d_agc_state = csdrb_device_alloc(sizeof(csdrb_agc_state_t) * (size_t)C);
    t->h_out = csdrb_host_alloc((size_t)C * (size_t)t->bs * sizeof(complexf));
    if (!t->d_bb || !t->d_carry || !t->d_mid || !t->d_pcm || !t->d_last_dc || !t->d_agc_state || !t->h_out) die("out of memory");
    csdrb_agc_state_t *h_st = calloc((size_t)C, sizeof *h_st);
    if (!h_st) die("out of memory");
    for (int c = 0; c < C; c++) h_st[c].gain = 1.0f;                 /* a stream starts at gain 1 (csdr.c:1363) */
    OK(csdrb_copy_h2d(t->d_agc_state, h_st, sizeof *h_st * (size_t)C, stream));
    float *h_dc = calloc((size_t)C, sizeof(float));                     /* last_dc_level starts at 0 (csdr.c:957) */
    if (!h_dc) die("out of memory");
    OK(csdrb_copy_h2d(t->d_last_dc, h_dc, sizeof(float) * (size_t)C, stream));
    OK(csdrb_stream_synchronize(stream));
    free(h_st); free(h_dc);
}

/* n_new fresh baseband samples per channel sit at d_bb + have: run the tail over the whole units, audio to the sinks, keep the remainder */
static void bb_tail_push(bb_tail_t *t, channel_t *chan, int n_new, void *stream)
{
    const int C = t->C;
    const long bs = t->bs;
    const int n = t->have + n_new;
    if (t->kind == TAIL_IQ) {                                    /* raw baseband: nothing is held back */
        OK(csdrb_copy2d_d2h(t->h_out, sizeof(complexf) * (size_t)n, t->d_bb, sizeof(complexf) * (size_t)bs, sizeof(complexf) * (size_t)n, (size_t)C, stream));
        OK(csdrb_stream_synchronize(stream));
        for (int c = 0; c < C; c++) write_sink(&chan[c], t->h_out + sizeof(complexf) * (size_t)c * (size_t)n, sizeof(complexf) * (size_t)n);
        return;
    }
    const int nb = n / t->unit, whole = nb * t->unit, rest = n - whole;
    if (nb > 0) {
        if (t->kind == TAIL_AM) {
            OK(csdrb_fastdcblock_bank_ff(t->d_bb, bs, 1, (float *)t->d_mid, bs, C, t->unit, nb, t->d_last_dc, stream));
            OK(csdrb_agc_bank_ff(t->d_mid, bs, 0, t->d_pcm, whole, 1, C, whole, &t->agc, t->d_agc_state, t->limit, stream));
        } else {
            OK(csdrb_bandpass_fir_fft_bank_cc(t->d_bb, bs, (complexf *)t->d_mid, bs, C, t->fft_size, t->unit, nb, t->d_taps_fft, 0, t->d_ola_tail, stream));
            OK(csdrb_agc_bank_ff(t->d_mid, bs, 1, t->d_pcm, whole, 1, C, whole, &t->agc, t->d_agc_state, t->limit, stream));
        }
        OK(csdrb_copy_d2h(t->h_out, t->d_pcm, sizeof(short) * (size_t)C * (size_t)whole, stream));
        if (rest > 0) {
            OK(csdrb_copy2d_d2d(t->d_carry, sizeof(complexf) * (size_t)t->unit, t->d_bb + whole, sizeof(complexf) * (size_t)bs, sizeof(complexf) * (size_t)rest, (size_t)C, stream));
            OK(csdrb_copy2d_d2d(t->d_bb, sizeof(complexf) * (size_t)bs, t->d_carry, sizeof(complexf) * (size_t)t->unit, sizeof(complexf) * (size_t)rest, (size_t)C, stream));
        }
        OK(csdrb_stream_synchronize(stream));
        for (int c = 0; c < C; c++) write_sink(&chan[c], t->h_out + sizeof(short) * (size_t)c * (size_t)whole, sizeof(short) * (size_t)whole);
    } else OK(csdrb_stream_synchronize(stream));
    t->have = rest;
}

static int run_multi(int in_fd, int u8, const int *dev, int ndev, channel_t *chan, int C, const float *rates, int D, const float *taps, int T, int block,
                     int kind, float limit, float agc_ref)
{
    const int nfm = kind == TAIL_NFM, demod = kind == TAIL_NFM || kind == TAIL_NONE;
    const size_t osz = demod ? sizeof(float) : sizeof(complexf);
    csdrb_multi_bank_t *mb = csdrb_multi_bank_create(ndev, dev, C, rates, D, taps, T, demod, 1024, block);
    if (!mb) die("cannot create the multi-GPU bank");
    const int n_out = (block - T) / D + 1, consumed = n_out * D, keep = block - consumed;
    float lut[256];
    for (int i = 0; i < 256; i++) lut[i] = (float)((float)i / (UCHAR_MAX / 2.0) - 1.0);      /* convert_u8_f, libcsdr.c:2365 */
    complexf *h_wide[2] = {csdrb_host_alloc(sizeof(complexf) * (size_t)block), csdrb_host_alloc(sizeof(complexf) * (size_t)block)};
    unsigned char *h_out[2] = {csdrb_host_alloc(osz * (size_t)C * (size_t)n_out), csdrb_host_alloc(osz * (size_t)C * (size_t)n_out)};
    unsigned char *raw = malloc((size_t)block * 2);
    if (!h_wide[0] || !h_wide[1] || !h_out[0] || !h_out[1] || !raw) die("out of memory");
    /* --tail nfm: the audio tail is audio-rate work (C x 48 kHz): the discriminator rows every device returned go to the FIRST device once more and through
     * the same kernels as in the single-GPU path */
    nfm_tail_t tail_state; bb_tail_t bb; void *tail_stream = NULL;
    if (kind != TAIL_NONE) {
        OK(csdrb_set_device(dev[0]));
        tail_stream = csdrb_stream_create();
        if (!tail_stream) die("cannot create a stream");
        if (nfm) nfm_tail_init(&tail_state, C, n_out + 2, limit, agc_ref);
        else bb_tail_init(&bb, kind, C, n_out + 2, limit, agc_ref, tail_stream);
    }
#define EMIT(slot_) do { \
        if (nfm) { \
            OK(csdrb_copy2d_h2d(tail_state.d_demod + tail_state.a_have, sizeof(float) * (size_t)tail_state.ds, h_out[slot_], sizeof(float) * (size_t)n_out, \
                                sizeof(float) * (size_t)n_out, (size_t)C, tail_stream)); \
            nfm_tail_push(&tail_state, chan, n_out, tail_stream); \
        } else if (!demod) { \
            OK(csdrb_copy2d_h2d(bb.d_bb + bb.have, sizeof(complexf) * (size_t)bb.bs, h_out[slot_], sizeof(complexf) * (size_t)n_out, \
                                sizeof(complexf) * (size_t)n_out, (size_t)C, tail_stream)); \
            bb_tail_push(&bb, chan, n_out, tail_stream); \
        } else for (int c = 0; c < C; c++) write_sink(&chan[c], h_out[slot_] + osz * (size_t)c * (size_t)n_out, osz * (size_t)n_out); \
    } while (0)
    long blocks = 0;
    int ticket[2] = {-1, -1};
    for (int first = 1;; first = 0) {
        const int slot = (int)(blocks & 1), fresh = first ? block : consumed;
        complexf *w = h_wide[slot];
        /* this buffer's previous block (two submits ago) must be done before it is overwritten; its results go out meanwhile */
        if (ticket[slot] >= 0) {
            if (csdrb_multi_bank_collect(mb, ticket[slot]) < 0) die("csdrb_multi_bank_collect failed");
            EMIT(slot);
            ticket[slot] = -1;
        }
        if (!first) memcpy(w, h_wide[slot ^ 1] + consumed, sizeof(complexf) * (size_t)keep);   /* the unconsumed tail (csdr.c:1172-1174) */
        complexf *dst = w + (first ? 0 : keep);
        int ok;
        if (u8) {
            ok = read_block(in_fd, raw, (size_t)fresh * 2);
            if (ok) for (int i = 0; i < fresh; i++) { dst[i].i = lut[raw[2 * i]]; dst[i].q = lut[raw[2 * i + 1]]; }
        } else ok = read_block(in_fd, (unsigned char *)dst, sizeof(complexf) * (size_t)fresh);
        if (!ok) break;
        ticket[slot] = csdrb_multi_bank_submit(mb, w, block, h_out[slot], n_out);
        if (ticket[slot] < 0) die("csdrb_multi_bank_submit failed");
        blocks++;
    }
    for (int k = 0; k < 2; k++) {                                  /* drain in submission order */
        const int slot = (int)((blocks + k) & 1);
        if (ticket[slot] < 0) continue;
        if (csdrb_multi_bank_collect(mb, ticket[slot]) < 0) die("csdrb_multi_bank_collect failed");
        EMIT(slot);
    }
#undef EMIT
    fprintf(stderr, "csdr-bankd: end of input after %ld blocks on %d devices, %ld kernel launches\n", blocks, ndev, csdrb_kernel_launches());
    csdrb_multi_bank_destroy(mb);
    return 0;
}

int main(int argc, char **argv)
{
    const char *in_spec = "-", *tail = "nfm";
    int u8 = 1, D = 50, block = 1 << 18, device = 0, ndev = 0, devs[64];
    float bw = 0.005f, limit = 1.0f, agc_ref = 0.0f;                /* agc_ref 0: the tail's own default (fastagc_ff 1.0, agc_ff 0.2) */
    window_t window = WINDOW_HAMMING;
    channel_t *chan = calloc((size_t)argc, sizeof *chan);
    int C = 0;
    for (int a = 1; a < argc; a++) {
        const char *o = argv[a];
        const char *v = a + 1 < argc ? argv[a + 1] : NULL;
        if (!strcmp(o, "--u8")) u8 = 1;
        else if (!strcmp(o, "--f32")) u8 = 0;
        else if (!strcmp(o, "--in") && v) { in_spec = v; a++; }
        else if (!strcmp(o, "--decimation") && v) { D = atoi(v); a++; }
        else if (!strcmp(o, "--bw") && v) { bw = (float)atof(v); a++; }
        else if (!strcmp(o, "--window") && v) { window = firdes_get_window_from_string((char *)v); a++; }
        else if (!strcmp(o, "--block") && v) { block = atoi(v); a++; }
        else if (!strcmp(o, "--tail") && v) { tail = v; a++; }
        else if (!strcmp(o, "--limit") && v) { limit = (float)atof(v); a++; }
        else if (!strcmp(o, "--agc-ref") && v) { agc_ref = (float)atof(v); a++; }
        else if (!strcmp(o, "--device") && v) { device = atoi(v); a++; }
        else if (!strcmp(o, "--devices") && v) { ndev = parse_devices(v, devs, 64); if (ndev <= 0) die("--devices wants N0,N1,..."); a++; }
        else if (strchr(o, ':') && o[0] != '-' ) {
            char *end = NULL;
            chan[C].rate = strtof(o, &end);
            if (!end || *end != ':') die("channels are RATE:SINK");
            chan[C].sink = end + 1; chan[C].fd = -1; chan[C].dropped = 0; C++;
        } else if (o[0] == '-' && strchr(o + 1, ':') && (o[1] == '.' || (o[1] >= '0' && o[1] <= '9'))) {      /* negative rate */
            char *end = NULL;
            chan[C].rate = strtof(o, &end);
            if (!end || *end != ':') die("channels are RATE:SINK");
            chan[C].sink = end + 1; chan[C].fd = -1; chan[C].dropped = 0; C++;
        } else { fprintf(stderr, "csdr-bankd: unknown argument %s\n", o); return 2; }
    }
    static const char *kTails[] = {"nfm", "none", "iq", "am", "usb", "lsb"};
    int kind = -1;
    for (int k = 0; k < 6; k++) if (!strcmp(tail, kTails[k])) kind = k;
    if (kind < 0) die("--tail is nfm, none, iq, am, usb or lsb");
    const int nfm = kind == TAIL_NFM, demod = kind == TAIL_NFM || kind == TAIL_NONE;
    if (nfm && agc_ref == 0.0f) agc_ref = 1.0f;                      /* fastagc_ff's default reference (csdr.c:1388) */
    if (C == 0) die("no channels (RATE:SINK ...)");
    if (block <= 0 || (block & 1)) die("--block must be a positive even number of samples");
    if (D <= 0 || (D & 1)) die("--decimation must be a positive even number (the fused kernels exist for 10 and 50)");
    if (!(bw > 0.f && bw < 0.5f)) die("--bw must be a transition bandwidth between 0 and 0.5");
    if (!(limit > 0.f) || !(agc_ref >= 0.f)) die("--limit and --agc-ref must be positive");
    signal(SIGPIPE, SIG_IGN);

    /* ---- filter and bank ---------------------------------------------------------------------------------------------------- */
    const int T = firdes_filter_len(bw);
    float *taps = malloc(sizeof(float) * (size_t)T);
    firdes_lowpass_f(taps, T, 0.5f / (float)D, window);
    if (block < 2 * T) die("--block is shorter than two filter lengths");
    float *rates = malloc(sizeof(float) * (size_t)C);
    for (int c = 0; c < C; c++) rates[c] = chan[c].rate;
    if (ndev > 0) {
        if (ndev > C) die("more devices than channels");
        for (int c = 0; c < C; c++) { chan[c].fd = open_sink(chan[c].sink); sink_nonblocking(chan[c].fd); }
        const int fd = open_input(in_spec);
        fprintf(stderr, "csdr-bankd: %d channels over %d devices, decimation %d, %d taps, %s input, blocks of %d samples, tail %s\n", C, ndev, D, T, u8 ? "u8" : "f32", block, tail);
        const int rc = run_multi(fd, u8, devs, ndev, chan, C, rates, D, taps, T, block, kind, limit, agc_ref);
        for (int c = 0; c < C; c++) { if (chan[c].dropped) fprintf(stderr, "csdr-bankd: sink %s lost %ld bytes (too slow)\n", chan[c].sink, chan[c].dropped); if (chan[c].fd >= 0) close(chan[c].fd); }
        return rc;
    }
    OK(csdrb_set_device(device));
    csdrb_ddc_bank_t *bank = csdrb_ddc_bank_create(C, rates, D, taps, T, demod, 1024);   /* 1024 = the CLI's shift_addition_cc call size (csdr.c:911) */
    if (!bank) die("cannot create the bank");
    void *stream = csdrb_stream_create();
    if (!stream) die("cannot create a stream");

    /* ---- buffers ----------------------------------------------------------------------------------------------------------------
     * wide[2]  : [tail of the previous block | new block] cf32, ping-pong so the tail copy never overlaps
     * with the NFM tail the discriminator output goes straight into nfm_tail_t's demod rows; without it into a plain [C][ds] array */
    const size_t in_bytes = (size_t)block * (u8 ? 2 : 8);
    unsigned char *h_in = csdrb_host_alloc(in_bytes);
    const int wide_cap = block + T + D + 16;
    complexf *d_wide[2] = {csdrb_device_alloc(sizeof(complexf) * (size_t)wide_cap), csdrb_device_alloc(sizeof(complexf) * (size_t)wide_cap)};
    unsigned char *d_raw = u8 ? csdrb_device_alloc(in_bytes + 16) : NULL;
    const int out_cap = wide_cap / D + 2;                          /* discriminator samples one block can add */
    nfm_tail_t tl;
    bb_tail_t bb;
    long ds = ((long)out_cap + 3) & ~3L;
    float *d_demod = NULL;
    unsigned char *h_out = NULL;
    if (nfm) { nfm_tail_init(&tl, C, out_cap, limit, agc_ref); ds = tl.ds; d_demod = tl.d_demod; }
    else if (!demod) { bb_tail_init(&bb, kind, C, out_cap, limit, agc_ref, stream); ds = bb.bs; d_demod = (float *)bb.d_bb; }
    else {
        d_demod = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)ds);
        h_out = csdrb_host_alloc((size_t)C * (size_t)ds * sizeof(float));
    }
    if (!h_in || !d_wide[0] || !d_wide[1] || (u8 && !d_raw) || !d_demod || (kind == TAIL_NONE && !h_out)) die("out of memory");

    /* sinks last: tcp: sinks block until their listener arrives */
    for (int c = 0; c < C; c++) { chan[c].fd = open_sink(chan[c].sink); sink_nonblocking(chan[c].fd); }
    const int in_fd = open_input(in_spec);
    fprintf(stderr, "csdr-bankd: %d channels, decimation %d, %d taps, %s input, blocks of %d samples, tail %s\n", C, D, T, u8 ? "u8" : "f32", block, tail);

    int cur = 0, keep = 0;
    long blocks = 0;
    /* Every call presents exactly `block` samples: the unconsumed tail plus as many new ones as the previous call consumed -- how csdr.c:1172-1174
     * feeds fir_decimate_cc.  A constant size keeps the bank's look-ahead pre-pass valid from block to block (a size that wobbles with
     * block % D made it miss, and re-run inline, on most blocks). */
    for (;;) {
        const int fresh_n = block - keep;                            /* first block: everything; later: what the last call consumed (even) */
        const size_t fresh_bytes = (size_t)fresh_n * (u8 ? 2 : 8);
        if (!read_block(in_fd, h_in, fresh_bytes)) break;
        /* 1. the new samples land behind the unconsumed tail (keep is even because block and D are: 16-byte alignment holds) */
        complexf *fresh = d_wide[cur] + keep;
        if (u8) {
            OK(csdrb_copy_h2d(d_raw, h_in, fresh_bytes, stream));
            OK(csdrb_convert_u8_f(d_raw, (float *)fresh, 2L * fresh_n, stream));
        } else OK(csdrb_copy_h2d(fresh, h_in, fresh_bytes, stream));
        const int n_in = block;

        /* 2. shift | fir_decimate | fmdemod for every channel, new discriminator samples behind the de-emphasis FIR's carried inputs */
        void *dst = nfm ? (void *)(d_demod + tl.a_have) : !demod ? (void *)(bb.d_bb + bb.have) : (void *)d_demod;
        const int n_out = csdrb_ddc_bank_process(bank, d_wide[cur], n_in, dst, ds, stream);
        if (n_out < 0) die("csdrb_ddc_bank_process failed");
        const int consumed = n_out * D;
        keep = n_in - consumed;
        OK(csdrb_copy_d2d(d_wide[cur ^ 1], d_wide[cur] + consumed, sizeof(complexf) * (size_t)keep, stream));
        cur ^= 1;

        if (!demod) bb_tail_push(&bb, chan, n_out, stream);         /* baseband tails: am / usb / lsb audio, or the raw baseband */
        else if (!nfm) {                                           /* raw discriminator output, float */
            OK(csdrb_copy2d_d2h(h_out, sizeof(float) * (size_t)n_out, d_demod, sizeof(float) * (size_t)ds, sizeof(float) * (size_t)n_out, (size_t)C, stream));
            OK(csdrb_stream_synchronize(stream));
            for (int c = 0; c < C; c++) write_sink(&chan[c], h_out + sizeof(float) * (size_t)c * (size_t)n_out, sizeof(float) * (size_t)n_out);
        } else nfm_tail_push(&tl, chan, n_out, stream);           /* 3./4. limit | de-emphasis | AGC | s16, audio to the sinks */
        blocks++;
    }
    OK(csdrb_stream_synchronize(stream));
    fprintf(stderr, "csdr-bankd: end of input after %ld blocks, %ld kernel launches\n", blocks, csdrb_kernel_launches());
    for (int c = 0; c < C; c++) { if (chan[c].dropped) fprintf(stderr, "csdr-bankd: sink %s lost %ld bytes (too slow)\n", chan[c].sink, chan[c].dropped); if (chan[c].fd >= 0) close(chan[c].fd); }
    csdrb_ddc_bank_destroy(bank);
    csdrb_stream_destroy(stream);
    return 0;
}
