/*
 * bankd.c -- csdr-bankd: a whole bank of FM, AM, SSB or BPSK31 receivers on ONE wideband IQ stream, in one process.
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
 *                   [--tail nfm|none|am|usb|lsb|iq|bpsk31] [--sps N] [--resample I:D[:BW]] [--limit L] [--agc-ref R] [--device N | --devices N0,N1,...]
 *                   RATE:SINK [RATE:SINK ...]
 *   --tail: nfm (default) the README.md:87 tail, s16; none the raw discriminator output, f32; am / usb / lsb the AM and SSB graphs of README.md:95 and :110
 *   behind the DDC's complex baseband (see bb_tail_t), s16; iq the complex baseband itself, cf32; bpsk31 the BPSK31 receive chain
 *   simple_agc_cc 0.001 R | timing_recovery_cc GARDNER N 0.5 2 --add_q | dbpsk_decoder_c_u8 | psk31_varicode_decoder_u8_u8 behind the baseband, the
 *   decoded text per channel (--sps N: samples per symbol at the baseband rate, > 4 and divisible by 4).  --limit is limit_ff's amplitude (default 1),
 *   --agc-ref the AGC reference (default: fastagc_ff's 1.0 for nfm, agc_ff's 0.2 for am/usb/lsb, simple_agc_cc's 0.5 for bpsk31).
 *   A PSK31 skimmer at 2.4 Msps: --decimation 300 --bw 0.001 gives 8 kHz baseband (4001 taps, M = 14 taps per output period: the fused bank serves it),
 *   and --sps 256 is 31.25 Bd:
 *     rtl_sdr -s 2400000 -f 14070000 - | csdr-bankd --decimation 300 --bw 0.001 --tail bpsk31 --sps 256 -0.1:ch1.txt 0.05:ch2.txt 0.2:ch3.txt
 *   --decimation: any even D (default 50) whose filter the fused bank serves: M = ceil(taps / D) <= 24 and D * M (rounded up to the kernel's
 *   bucket) <= 8000 taps, see csdrb_ddc_bank in include/csdr_b200.h.  The NFM tail's deemphasis_nfm_ff stays at 48000 whatever D gives: where
 *   wideband rate / D is not 48 kHz, --resample I:D[:BW] puts rational_resampler_ff I D BW right behind the discriminator (tails nfm and none; see
 *   --help for the geometries it serves), e.g. 2.048 Msps with --decimation 32 --resample 3:4, or 10 Msps with --decimation 200 --resample 24:25:0.02.
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
    memset(r, 0, sizeof *r);
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
    if (keep > 0 && st.input_processed > 0) {
        const size_t row = sizeof(float) * (size_t)r->rs;
        OK(csdrb_copy2d_d2d(r->d_carry, row, r->d_in + st.input_processed, row, sizeof(float) * (size_t)keep, (size_t)r->C, stream));
        OK(csdrb_copy2d_d2d(r->d_in, row, r->d_carry, row, sizeof(float) * (size_t)keep, (size_t)r->C, stream));
    }
    r->have = keep; r->ltd = st.last_taps_delay;
    return m;
}

/* --tail none: n float samples per channel (device rows, pitch `pitch`) to the sinks */
static void raw_emit(const float *d_rows, long pitch, int n, unsigned char *h_out, channel_t *chan, int C, void *stream)
{
    OK(csdrb_copy2d_d2h(h_out, sizeof(float) * (size_t)n, d_rows, sizeof(float) * (size_t)pitch, sizeof(float) * (size_t)n, (size_t)C, stream));
    OK(csdrb_stream_synchronize(stream));
    for (int c = 0; c < C; c++) write_sink(&chan[c], h_out + sizeof(float) * (size_t)c * (size_t)n, sizeof(float) * (size_t)n);
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
enum { TAIL_NFM, TAIL_NONE, TAIL_IQ, TAIL_AM, TAIL_USB, TAIL_LSB, TAIL_BPSK31 };

/* ---- the BPSK31 tail: simple_agc_cc 0.001 R | timing_recovery_cc GARDNER N 0.5 2 --add_q | dbpsk_decoder_c_u8 | psk31_varicode_decoder_u8_u8 --------
 * Channels consume different amounts of baseband, so the timing recovery bank gets a start offset per channel.  Device buffers of ONE device:
 *   tr   : [C][ts] complexf : AGC output; row c's unconsumed samples are [start[c], end) (end is the same for every row), new samples go to end
 *   sym  : [C][cap] complexf symbols, bits : [C][cap] dbpsk bits, chars : [C][cap] decoded text
 * Carried per channel: the AGC gain, the timing loop's correction offset and unconsumed baseband, the last dbpsk input, the varicode register.
 * The timing recovery leaves at most 3N/2 samples unconsumed, so every push first moves [min start, end) to the front of the rows. */
typedef struct {
    int C, sps, end, cap, last_cur;
    long ts;
    float agc_ref;
    complexf *d_tr, *d_carry, *d_sym, *d_last[2];
    unsigned char *d_bits, *d_chars;
    float *d_gain;
    int *d_start, *d_size, *d_counts, *d_char_count, *h_start, *h_size, *h_char_count;
    csdrb_timing_recovery_state_t *d_state, *h_state;
    unsigned long long *d_hist;
    unsigned char *h_chars;
} bpsk_tail_t;

static void bpsk_tail_init(bpsk_tail_t *t, int C, int sps, int in_cap, float agc_ref, void *stream)
{
    memset(t, 0, sizeof *t);
    t->C = C; t->sps = sps; t->agc_ref = agc_ref;
    t->ts = ((long)in_cap + 2L * sps + 3) & ~3L;
    t->cap = (int)(t->ts / (sps / 2) + 1);
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
    if (!t->d_tr || !t->d_carry || !t->d_sym || !t->d_last[0] || !t->d_last[1] || !t->d_bits || !t->d_chars || !t->d_gain || !t->d_start || !t->d_size ||
        !t->d_counts || !t->d_char_count || !t->d_state || !t->d_hist || !t->h_start || !t->h_state || !t->h_chars) die("out of memory");
    t->h_size = t->h_start + C; t->h_char_count = t->h_start + 2 * C;
    float *g = malloc(sizeof(float) * (size_t)C);
    if (!g) die("out of memory");
    for (int c = 0; c < C; c++) g[c] = 1.0f;                               /* simple_agc_cc's current_gain starts at 1 (csdr.c:2917) */
    OK(csdrb_copy_h2d(t->d_gain, g, sizeof(float) * (size_t)C, stream));
    OK(csdrb_stream_synchronize(stream));
    free(g);
}

/* n new baseband samples per channel at d_bb (row pitch bs): the chain over them, the decoded text to the sinks */
static void bpsk_tail_push(bpsk_tail_t *t, channel_t *chan, const complexf *d_bb, long bs, int n, void *stream)
{
    const int C = t->C;
    const size_t row = sizeof(complexf) * (size_t)t->ts;
    int lo = t->end;
    for (int c = 0; c < C; c++) lo = t->h_start[c] < lo ? t->h_start[c] : lo;
    if (lo > 0 && t->end > lo) {                                            /* the unconsumed samples to the front of the rows */
        OK(csdrb_copy2d_d2d(t->d_carry, row, t->d_tr + lo, row, sizeof(complexf) * (size_t)(t->end - lo), (size_t)C, stream));
        OK(csdrb_copy2d_d2d(t->d_tr, row, t->d_carry, row, sizeof(complexf) * (size_t)(t->end - lo), (size_t)C, stream));
    }
    for (int c = 0; c < C; c++) t->h_start[c] -= lo;
    t->end -= lo;
    if (t->end + n > t->ts) die("bpsk31 tail: baseband buffer overflow");
    OK(csdrb_simple_agc_bank_cc(d_bb, bs, t->d_tr + t->end, t->ts, C, n, 0.001f, t->agc_ref, 65535.0f, t->d_gain, stream));
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
        for (int c = 0; c < C; c++) if (t->h_char_count[c] > 0) write_sink(&chan[c], t->h_chars + (size_t)c * (size_t)m, (size_t)t->h_char_count[c]);
    }
}

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
    bpsk_tail_t bpsk;
} bb_tail_t;

static void bb_tail_init(bb_tail_t *t, int kind, int C, int out_cap, float limit, float agc_ref, int sps, void *stream)
{
    memset(t, 0, sizeof *t);
    t->kind = kind; t->C = C; t->limit = limit;
    if (kind == TAIL_BPSK31) {                                       /* the baseband rows only pass the new samples on */
        t->unit = 1;
        t->bs = ((long)out_cap + 3) & ~3L;
        t->d_bb = csdrb_device_alloc(sizeof(complexf) * (size_t)C * (size_t)t->bs);
        if (!t->d_bb) die("out of memory");
        bpsk_tail_init(&t->bpsk, C, sps, out_cap, agc_ref, stream);
        return;
    }
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
    if (t->kind == TAIL_BPSK31) { bpsk_tail_push(&t->bpsk, chan, t->d_bb, bs, n, stream); t->have = 0; return; }
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
                     int kind, float limit, float agc_ref, int rs_I, int rs_D, float rs_bw, int sps)
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
    nfm_tail_t tail_state; bb_tail_t bb; rs_stage_t rsm; void *tail_stream = NULL;
    float *d_raw_out = NULL; unsigned char *h_raw_out = NULL;
    const int resample = rs_I > 0;
    if (kind != TAIL_NONE || resample) {
        OK(csdrb_set_device(dev[0]));
        tail_stream = csdrb_stream_create();
        if (!tail_stream) die("cannot create a stream");
        if (resample) rs_init(&rsm, C, rs_I, rs_D, rs_bw, n_out + 2);
        const int tail_cap = resample ? rs_out_cap(&rsm) : n_out + 2;
        if (nfm) nfm_tail_init(&tail_state, C, tail_cap, limit, agc_ref);
        else if (!demod) bb_tail_init(&bb, kind, C, tail_cap, limit, agc_ref, sps, tail_stream);
        else {
            d_raw_out = csdrb_device_alloc(sizeof(float) * (size_t)C * (size_t)tail_cap);
            h_raw_out = csdrb_host_alloc(sizeof(float) * (size_t)C * (size_t)tail_cap);
            if (!d_raw_out || !h_raw_out) die("out of memory");
        }
    }
    /* --resample: the discriminator rows go to the first device's resampler, its output into the tail (or straight to the sinks for --tail none) */
#define EMIT(slot_) do { \
        if (resample) { \
            OK(csdrb_copy2d_h2d(rsm.d_in + rsm.have, sizeof(float) * (size_t)rsm.rs, h_out[slot_], sizeof(float) * (size_t)n_out, \
                                sizeof(float) * (size_t)n_out, (size_t)C, tail_stream)); \
            if (nfm) nfm_tail_push(&tail_state, chan, rs_push(&rsm, n_out, tail_state.d_demod + tail_state.a_have, tail_state.ds, tail_stream), tail_stream); \
            else { const int m_ = rs_push(&rsm, n_out, d_raw_out, rs_out_cap(&rsm), tail_stream); raw_emit(d_raw_out, rs_out_cap(&rsm), m_, h_raw_out, chan, C, tail_stream); } \
        } else if (nfm) { \
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

static int usage(void)
{
    fprintf(stderr,
            "usage: csdr-bankd [--in -|HOST:PORT] [--u8|--f32] [--decimation D] [--bw TRANSITION_BW] [--window W] [--block SAMPLES]\n"
            "                  [--tail nfm|none|am|usb|lsb|iq|bpsk31] [--sps N] [--resample I:D[:BW]] [--limit L] [--agc-ref R] [--device N | --devices N0,N1,...]\n"
            "                  RATE:SINK [RATE:SINK ...]\n"
            "  --tail bpsk31 --sps N  per channel simple_agc_cc 0.001 R | timing_recovery_cc GARDNER N 0.5 2 --add_q | dbpsk_decoder_c_u8 |\n"
            "                       psk31_varicode_decoder_u8_u8 (R = --agc-ref, default 0.5) behind the baseband; the sinks get the decoded text.\n"
            "                       N is samples per symbol at the baseband rate, > 4 and divisible by 4.  A PSK31 skimmer at 2.4 Msps:\n"
            "                       csdr-bankd --decimation 300 --bw 0.001 --tail bpsk31 --sps 256 -0.1:ch1.txt 0.05:ch2.txt 0.2:ch3.txt\n"
            "                       (8 kHz baseband, 4001 taps = 14 per output period, which the fused bank serves; 31.25 Bd)\n"
            "  --resample I:D[:BW]  rational_resampler_ff I D BW (BW default 0.05) right behind the discriminator, for --tail nfm and none: brings\n"
            "                       wideband/decimation to the 48 kHz the NFM de-emphasis is designed for (e.g. 2.048 Msps, --decimation 32,\n"
            "                       --resample 3:4).  With T = taps of BW, the daemon needs (T/I + 1)*I >= 2*D + I - 1 (T >= 2*D + I - 2 suffices),\n"
            "                       so that no resampler call ends on its output cap; other geometries are refused.\n"
            "  see the head of csdr_b200/host/bankd.c for the other options\n");
    return 2;
}

int main(int argc, char **argv)
{
    const char *in_spec = "-", *tail = "nfm";
    int u8 = 1, D = 50, block = 1 << 18, device = 0, ndev = 0, devs[64];
    float bw = 0.005f, limit = 1.0f, agc_ref = 0.0f;                /* agc_ref 0: the tail's own default (fastagc_ff 1.0, agc_ff 0.2) */
    int rs_I = 0, rs_D = 0;                                          /* --resample I:D[:BW]; 0: no resampler */
    int sps = 0;                                                     /* --sps N of --tail bpsk31 */
    float rs_bw = 0.05f;                                             /* rational_resampler_ff's default transition bandwidth (csdr.c:1423) */
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
        else if (!strcmp(o, "--sps") && v) { sps = atoi(v); a++; }
        else if (!strcmp(o, "--device") && v) { device = atoi(v); a++; }
        else if (!strcmp(o, "--devices") && v) { ndev = parse_devices(v, devs, 64); if (ndev <= 0) die("--devices wants N0,N1,..."); a++; }
        else if (!strcmp(o, "--resample") && v) {
            if (sscanf(v, "%d:%d:%f", &rs_I, &rs_D, &rs_bw) < 2 || rs_I < 1 || rs_D < 1) die("--resample wants I:D[:BW] with positive integers I and D");
            a++;
        }
        else if (!strcmp(o, "--help")) return usage();
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
    static const char *kTails[] = {"nfm", "none", "iq", "am", "usb", "lsb", "bpsk31"};
    int kind = -1;
    for (int k = 0; k < 7; k++) if (!strcmp(tail, kTails[k])) kind = k;
    if (kind < 0) die("--tail is nfm, none, iq, am, usb, lsb or bpsk31");
    if (kind == TAIL_BPSK31) {
        if (sps <= 4 || (sps & 3)) die("--tail bpsk31 needs --sps N with N > 4 and divisible by 4 (timing_recovery_cc's decimation)");
        if (agc_ref == 0.0f) agc_ref = 0.5f;                         /* simple_agc_cc's reference in the OpenWebRX chain */
    } else if (sps) die("--sps belongs to --tail bpsk31");
    const int nfm = kind == TAIL_NFM, demod = kind == TAIL_NFM || kind == TAIL_NONE;
    if (nfm && agc_ref == 0.0f) agc_ref = 1.0f;                      /* fastagc_ff's default reference (csdr.c:1388) */
    if (C == 0) die("no channels (RATE:SINK ...)");
    if (block <= 0 || (block & 1)) die("--block must be a positive even number of samples");
    if (D <= 0 || (D & 1)) die("--decimation must be a positive even number (the fused bank serves even decimations only)");
    if (!(bw > 0.f && bw < 0.5f)) die("--bw must be a transition bandwidth between 0 and 0.5");
    if (!(limit > 0.f) || !(agc_ref >= 0.f)) die("--limit and --agc-ref must be positive");
    const int resample = rs_I > 0;
    if (resample) {
        if (!demod) die("--resample works with --tail nfm and --tail none only (the am, usb, lsb, iq and bpsk31 tails are not resampled)");
        if (!(rs_bw > 0.f && rs_bw < 0.5f)) die("--resample: the transition bandwidth must be between 0 and 0.5");
        const int rs_T = firdes_filter_len(rs_bw);
        if (!resample_geometry_ok(rs_I, rs_D, rs_T)) {
            fprintf(stderr, "csdr-bankd: --resample %d:%d with %d taps: a resampler call could end on its output cap and repeat an output; "
                            "the daemon needs (T/I + 1)*I >= 2*D + I - 1 (T >= 2*D + I - 2 suffices): lower the transition bandwidth\n", rs_I, rs_D, rs_T);
            return 1;
        }
    }
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
        const int rc = run_multi(fd, u8, devs, ndev, chan, C, rates, D, taps, T, block, kind, limit, agc_ref, rs_I, rs_D, rs_bw, sps);
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
    rs_stage_t rsm;
    if (resample) rs_init(&rsm, C, rs_I, rs_D, rs_bw, out_cap);
    const int tail_cap = resample ? rs_out_cap(&rsm) : out_cap;   /* samples one block can add behind the discriminator (and resampler) */
    long ds = ((long)tail_cap + 3) & ~3L;
    float *d_demod = NULL;
    unsigned char *h_out = NULL;
    if (nfm) { nfm_tail_init(&tl, C, tail_cap, limit, agc_ref); ds = tl.ds; d_demod = tl.d_demod; }
    else if (!demod) { bb_tail_init(&bb, kind, C, out_cap, limit, agc_ref, sps, stream); ds = bb.bs; d_demod = (float *)bb.d_bb; }
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
        void *dst = resample ? (void *)(rsm.d_in + rsm.have) : nfm ? (void *)(d_demod + tl.a_have) : !demod ? (void *)(bb.d_bb + bb.have) : (void *)d_demod;
        const int n_out = csdrb_ddc_bank_process(bank, d_wide[cur], n_in, dst, resample ? rsm.rs : ds, stream);
        if (n_out < 0) die("csdrb_ddc_bank_process failed");
        const int consumed = n_out * D;
        keep = n_in - consumed;
        OK(csdrb_copy_d2d(d_wide[cur ^ 1], d_wide[cur] + consumed, sizeof(complexf) * (size_t)keep, stream));
        cur ^= 1;

        /* 2b. --resample: the new discriminator samples through rational_resampler_ff, into the tail's rows */
        const int n_tail = resample ? rs_push(&rsm, n_out, nfm ? d_demod + tl.a_have : d_demod, ds, stream) : n_out;
        if (!demod) bb_tail_push(&bb, chan, n_out, stream);         /* baseband tails: am / usb / lsb audio, or the raw baseband */
        else if (!nfm) raw_emit(d_demod, ds, n_tail, h_out, chan, C, stream);   /* raw discriminator output, float */
        else nfm_tail_push(&tl, chan, n_tail, stream);             /* 3./4. limit | de-emphasis | AGC | s16, audio to the sinks */
        blocks++;
    }
    OK(csdrb_stream_synchronize(stream));
    fprintf(stderr, "csdr-bankd: end of input after %ld blocks, %ld kernel launches\n", blocks, csdrb_kernel_launches());
    for (int c = 0; c < C; c++) { if (chan[c].dropped) fprintf(stderr, "csdr-bankd: sink %s lost %ld bytes (too slow)\n", chan[c].sink, chan[c].dropped); if (chan[c].fd >= 0) close(chan[c].fd); }
    csdrb_ddc_bank_destroy(bank);
    csdrb_stream_destroy(stream);
    return 0;
}
