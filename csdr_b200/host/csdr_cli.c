/*
 * csdr_cli.c -- the `csdr` stdin/stdout command surface for the hot-path commands, host code in C over
 * libcsdr_b200.so (Part A of include/csdr_b200.h).  One process = one DSP block, raw samples on the pipes,
 * exactly like the reference CLI, so existing pipe graphs (csdr-fm:41, README.md:54-110) drop in unchanged.
 *
 * Behaviours reproduced from the reference (SURVEY.md 8(b); all citations into reference csdr.c):
 *   - block sizes: 1024 default / 16384 for the wideband commands, rounded up to a multiple of 4 (:189-190,
 *     :353-357), fir_decimate_cc grows its block to >= 2*taps (:1136); CSDR_FIXED_BUFSIZE,
 *     CSDR_DYNAMIC_BUFSIZE_ON, CSDR_PRINT_BUFSIZES (:394-417)
 *   - optional 8-byte "csdr"+int preamble in and out when dynamic buffer sizes are on (:330-339, :377-392)
 *   - EOF framing: the end-of-file test comes BEFORE the read, so a short final read is still processed and
 *     written as a whole block (:248 and every loop); the shift commands also stop on an empty read (:907)
 *   - fflush + sched_yield after every block (:198); F_SETPIPE_SZ 2 MiB, 4096 for small blocks (:427-428, :369-373)
 *   - runtime retune over --fifo <path> / --fd <n>: text lines, non-blocking, last complete line wins (:252-323)
 *   - the stderr lines the reference prints for these commands
 *   - psk31_varicode_encoder_u8_u8 as the reference's loop runs: after the first block it re-encodes that block once per read (:2797 refills
 *     the wrong buffer), so its bytes equal the reference CLI's for every input
 * Everything else the reference CLI offers (100+ other commands) is out of scope (SURVEY.md section 2.1 #6).
 */
#define _GNU_SOURCE
#include "csdr_b200.h"

#include <fcntl.h>
#include <math.h>
#include <sched.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>
#include <unistd.h>

/* ---- process-wide settings ---------------------------------------------------------------------- */
static struct {
    int fixed_small, fixed_big, dynamic_on, print_sizes, wideband;
    int argc; char **argv;
} G = {1024, 1024 * 16, 0, 0, 0, 0, NULL};

static void who(void) { fprintf(stderr, "%s%s%s: ", G.argv[0], G.argc >= 2 ? " " : "", G.argc >= 2 ? G.argv[1] : ""); }

static int complain(const char *why) { who(); fprintf(stderr, "%s\n", why); return -1; }

static void read_environment(void)
{
    const char *v = getenv("CSDR_DYNAMIC_BUFSIZE_ON");
    if (v) { G.dynamic_on = !!atoi(v); G.fixed_small = 0; }
    else if ((v = getenv("CSDR_FIXED_BUFSIZE"))) G.fixed_big = G.fixed_small = atoi(v);
    if ((v = getenv("CSDR_PRINT_BUFSIZES"))) G.print_sizes = atoi(v);
}

/* ---- buffer-size negotiation ------------------------------------------------------------------- */
static const char kPreamble[4] = {'c', 's', 'd', 'r'};

static int incoming_block_size(void)
{
    if (!G.dynamic_on) return G.wideband ? G.fixed_big : G.fixed_small;
    int head[2] = {0, 0};
    if (fread(head, sizeof(int), 2, stdin) != 2 || memcmp(head, kPreamble, 4) != 0) {
        complain("warning! Did not match preamble on the beginning of the stream. You should put \"csdr setbuf <buffer size>\" at the "
                 "beginning of the chain! Falling back to default buffer size: 1024");
        return 1024;
    }
    if (head[1] <= 0) { complain("warning! Invalid buffer size."); return 0; }
    return head[1];
}

static int round_to_unit(int n) { return n <= 0 ? 4 : ((n - 1) & ~3) + 4; }

static int block = 0;                                  /* samples (or values) per block of this process */

static int open_block(void)
{
    block = incoming_block_size();
    if (!block) return 0;
    block = round_to_unit(block);
    if (G.print_sizes) { who(); fprintf(stderr, "buffer size set to %d\n", block); }
    if (block <= 4096) { fcntl(STDIN_FILENO, F_SETPIPE_SZ, 4096); fcntl(STDOUT_FILENO, F_SETPIPE_SZ, 4096); }
    return block;
}

static int announce_block(int size)
{
    if (size <= 4096) fcntl(STDOUT_FILENO, F_SETPIPE_SZ, 4096);
    if (!G.dynamic_on) return G.fixed_small;
    if (G.print_sizes) { who(); fprintf(stderr, "next process proposed input buffer size is %d\n", size); }
    int head[2]; memcpy(head, kPreamble, 4); head[1] = size;
    fwrite(head, sizeof(int), 2, stdout);
    return size;
}

static void end_of_block(void) { fflush(stdout); sched_yield(); }

static void *must_alloc(size_t bytes) { void *p = calloc(1, bytes ? bytes : 1); if (!p) { complain("out of memory"); exit(-2); } return p; }

/* ---- runtime control channel (--fifo / --fd) ----------------------------------------------------- */
static int open_control(int argc, char **argv)
{
    if (argc < 4) return 0;
    int fd = 0;
    if (!strcmp(argv[2], "--fifo")) { who(); fprintf(stderr, "fifo control mode on\n"); fd = open(argv[3], O_RDONLY); }
    else if (!strcmp(argv[2], "--fd")) { if (sscanf(argv[3], "%d", &fd) <= 0) return 0; who(); fprintf(stderr, "fd control mode on, fd=%d\n", fd); }
    else return 0;
    fcntl(fd, F_SETFL, fcntl(fd, F_GETFL, 0) | O_NONBLOCK);
    return fd;
}

/* returns 1 when at least one complete line arrived; the LAST complete line is parsed with `format` */
static int poll_control(int fd, const char *format, ...)
{
    static char pending[1024];
    static int have = 0;
    if (!fd) return 0;
    int got = (int)read(fd, pending + have, sizeof pending - (size_t)have);
    if (got <= 0) return 0;
    int total = have + got, last_end = 0, prev_end = 0;
    for (int k = 0; k < total; k++) if (pending[k] == '\n') { prev_end = last_end; last_end = k + 1; }
    if (!last_end) { have = total; return 0; }
    va_list ap; va_start(ap, format); vsscanf(pending + prev_end, format, ap); va_end(ap);
    memmove(pending, pending + last_end, (size_t)(total - last_end));
    have = total - last_end;
    return 1;
}

/* the starting tuning: the first line on the control channel when there is one (waited for), else argv[2] (and argv[3] for b);
 * 0 when argv lacks it */
static int initial_tuning(int ctl, int argc, char **argv, const char *format, float *a, float *b)
{
    if (ctl) { while (!poll_control(ctl, format, a, b)) usleep(10000); return 1; }
    if (argc <= (b ? 3 : 2)) return 0;
    sscanf(argv[2], "%g", a);
    if (b) sscanf(argv[3], "%g", b);
    return 1;
}

/* ---- shared framing ------------------------------------------------------------------------------ */
/* One step call per block of the process on the whole buffer, written as out_count items.  The end-of-file test comes before the read, so a
 * short final read is still processed and written as a whole block, its tail left over from the block before (:248).  Some reference loops
 * also stop on an empty read (empty_read_stops = 1); fmdemod_atan_cf tests end of file right after its read, so a short final read is
 * dropped and only whole blocks come out (empty_read_stops = 2, :976). */
static int map_blocks(size_t in_item, size_t out_item, int out_count, int empty_read_stops, void (*step)(void *in, void *out, void *state), void *state)
{
    void *in = must_alloc(in_item * (size_t)block), *out = must_alloc(out_item * (size_t)out_count);
    for (;;) {
        if (feof(stdin)) return 0;
        if (!fread(in, in_item, (size_t)block, stdin) && empty_read_stops) return 0;
        if (empty_read_stops == 2 && feof(stdin)) return 0;
        step(in, out, state);
        fwrite(out, out_item, (size_t)out_count, stdout);
        end_of_block();
    }
}

/* keep the unconsumed tail of a buffer of `size` items at its front and read the `consumed` items behind it */
static void refill(void *buf, size_t item, int size, int consumed)
{
    memmove(buf, (char *)buf + item * (size_t)consumed, item * (size_t)(size - consumed));
    fread((char *)buf + item * (size_t)(size - consumed), item, (size_t)consumed, stdin);
}

/* the next FFT frame of `size` items, one starting every `every` items: overlapping frames slide, sparser ones are read whole and the rest
 * is skipped in pieces of at most one block of complexf samples (whatever the frame's item, see fft_fc) */
static void read_frame(void *in, size_t item, int size, int every, complexf *skip)
{
    if (every <= size) { refill(in, item, size, every); return; }
    fread(in, item, (size_t)size, stdin);
    for (int remain = every - size; remain > 0; remain -= block) fread(skip, sizeof(complexf), (size_t)(remain < block ? remain : block), stdin);
}

/* the pass-through special case of the resamplers (the reference's clone_): blocks of bytes copied through, the EOF test after the write */
static int clone_blocks(void)
{
    char *buf = must_alloc((size_t)block);
    for (;;) { fread(buf, 1, (size_t)block, stdin); fwrite(buf, 1, (size_t)block, stdout); end_of_block(); if (feof(stdin)) return 0; }
}

/* the optional window argument at argv[at]; without it the default window is named on stderr */
static window_t window_arg(int argc, char **argv, int at)
{
    if (argc > at) return firdes_get_window_from_string(argv[at]);
    who(); fprintf(stderr, "window = %s\n", firdes_get_string_from_window(WINDOW_DEFAULT));
    return WINDOW_DEFAULT;
}

/* ---- the retunable NCO loop of shift_addition_cc/_fc, shift_unroll_cc and shift_addfast_cc (csdr.c:749-849, :877-934, :3365-3410) ----
 * The rate comes from argv or the control channel.  Every block is shifted in calls of <= 1024 samples, the phasor re-seeded at each
 * (:911-918); an empty read ends the stream (:907).  A new rate is polled after a block is written and before it is flushed; it
 * re-initialises the NCO, and the phase carries on. */
typedef union { shift_addition_data_t addition; shift_unroll_data_t unroll; shift_addfast_data_t addfast; } nco_t;

static int nco_stream(int argc, char **argv, size_t in_item, void (*init)(nco_t *nco, float rate),
                      float (*step)(void *in, complexf *out, int n, nco_t *nco, float phase), void (*release)(nco_t *nco))
{
    G.wideband = 1;
    float phase = 0, rate = 0;
    int ctl = open_control(argc, argv);
    if (!initial_tuning(ctl, argc, argv, "%g\n", &rate, NULL)) return complain("need required parameter (rate)");
    if (!announce_block(open_block())) return -2;
    char *in = must_alloc(in_item * (size_t)block);
    complexf *out = must_alloc(sizeof(complexf) * (size_t)block);
    for (;;) {
        nco_t nco;
        init(&nco, rate);
        who(); fprintf(stderr, "reinitialized to %g\n", rate);
        for (;;) {
            if (feof(stdin)) return 0;
            if (!fread(in, in_item, (size_t)block, stdin)) break;
            for (int done = 0; done < block;) {
                int n = block - done > 1024 ? 1024 : block - done;
                phase = step(in + in_item * (size_t)done, out + done, n, &nco, phase);
                done += n;
            }
            fwrite(out, sizeof(complexf), (size_t)block, stdout);
            if (poll_control(ctl, "%g\n", &rate)) break;
            end_of_block();
        }
        if (release) release(&nco);
    }
}

/* ---- commands ------------------------------------------------------------------------------------ */
static void convert_u8_f_step(void *in, void *out, void *state) { (void)state; convert_u8_f(in, out, block); }
static void convert_s16_f_step(void *in, void *out, void *state) { (void)state; convert_s16_f(in, out, block); }
static void convert_f_s16_step(void *in, void *out, void *state) { (void)state; convert_f_s16(in, out, block); }

static int cmd_convert_u8_f(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(1, sizeof(float), block, 0, convert_u8_f_step, NULL);
}

static int cmd_convert_s16_f(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(short), sizeof(float), block, 0, convert_s16_f_step, NULL);
}

static int cmd_convert_f_s16(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(float), sizeof(short), block, 0, convert_f_s16_step, NULL);
}

/* convert_s8_f, convert_f_s8, convert_f_u8 (csdr.c:546-581) and convert_s24_f / convert_f_s24 [--bigendian] (:606-633): one call per block,
 * s24 values 3 bytes each.  `--bigendian` is the reference's flag, whose meaning on x86 is the opposite of its name (include/csdr_b200.h). */
static void convert_s8_f_step(void *in, void *out, void *state) { (void)state; convert_s8_f(in, out, block); }
static void convert_f_s8_step(void *in, void *out, void *state) { (void)state; convert_f_s8(in, out, block); }
static void convert_f_u8_step(void *in, void *out, void *state) { (void)state; convert_f_u8(in, out, block); }
static void convert_s24_f_step(void *in, void *out, void *bigendian) { convert_s24_f(in, out, block, *(int *)bigendian); }
static void convert_f_s24_step(void *in, void *out, void *bigendian) { convert_f_s24(in, out, block, *(int *)bigendian); }

static int cmd_convert_s8_f(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(1, sizeof(float), block, 0, convert_s8_f_step, NULL);
}

static int cmd_convert_f_s8(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(float), 1, block, 0, convert_f_s8_step, NULL);
}

static int cmd_convert_f_u8(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(float), 1, block, 0, convert_f_u8_step, NULL);
}

static int cmd_convert_s24_f(int argc, char **argv)
{
    int bigendian = argc > 2 && !strcmp(argv[2], "--bigendian");
    if (!announce_block(open_block())) return -2;
    return map_blocks(3, sizeof(float), block, 0, convert_s24_f_step, &bigendian);
}

static int cmd_convert_f_s24(int argc, char **argv)
{
    int bigendian = argc > 2 && !strcmp(argv[2], "--bigendian");
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(float), 3, block, 0, convert_f_s24_step, &bigendian);
}

static void addition_init(nco_t *nco, float rate) { nco->addition = shift_addition_init(rate); }
static float addition_cc(void *in, complexf *out, int n, nco_t *nco, float phase) { return shift_addition_cc(in, out, n, nco->addition, phase); }
static float addition_fc(void *in, complexf *out, int n, nco_t *nco, float phase) { return shift_addition_fc(in, out, n, nco->addition, phase); }

static int cmd_shift_addition_cc(int argc, char **argv) { return nco_stream(argc, argv, sizeof(complexf), addition_init, addition_cc, NULL); }

/* csdr.c:3365-3410: cmd_shift_addition_cc with real input -- the big buffer, 1024-sample calls, the stop on an empty read and the retune
 * between buffers are the same; only the input is one float per sample */
static int cmd_shift_addition_fc(int argc, char **argv) { return nco_stream(argc, argv, sizeof(float), addition_init, addition_fc, NULL); }

static int cmd_fir_decimate_cc(int argc, char **argv)
{
    G.wideband = 1;
    if (argc <= 2) return complain("need required parameter (decimation factor)");
    int factor = 0; sscanf(argv[2], "%d", &factor);
    float transition_bw = 0.05f; if (argc >= 4) sscanf(argv[3], "%g", &transition_bw);
    window_t window = WINDOW_DEFAULT;
    if (argc >= 5) window = firdes_get_window_from_string(argv[4]);
    else fprintf(stderr, "fir_decimate_cc: window = %s\n", firdes_get_string_from_window(window));
    int taps_length = firdes_filter_len(transition_bw);
    fprintf(stderr, "fir_decimate_cc: taps_length = %d\n", taps_length);
    while (G.fixed_big < taps_length * 2) G.fixed_big *= 2;
    if (!open_block()) return -2;
    announce_block(block / factor);
    float *taps = must_alloc(sizeof(float) * (size_t)taps_length);
    firdes_lowpass_f(taps, taps_length, 0.5f / (float)factor, window);
    complexf *in = must_alloc(sizeof(complexf) * (size_t)block), *out = must_alloc(sizeof(complexf) * (size_t)block);
    fread(in, sizeof(complexf), (size_t)block, stdin);
    for (;;) {
        if (feof(stdin)) return 0;
        int produced = fir_decimate_cc(in, out, block, factor, taps, taps_length);
        fwrite(out, sizeof(complexf), (size_t)produced, stdout);
        end_of_block();
        refill(in, sizeof(complexf), block, factor * produced);         /* keep the unconsumed tail, refill behind it (:1172-1174) */
    }
}

static void fmdemod_step(void *in, void *out, void *last) { *(complexf *)last = fmdemod_quadri_cf(in, out, block, NULL, *(complexf *)last); }

static int cmd_fmdemod_quadri_cf(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    complexf last = {0.f, 0.f};
    return map_blocks(sizeof(complexf), sizeof(float), block, 0, fmdemod_step, &last);
}

static void unroll_init(nco_t *nco, float rate) { nco->unroll = shift_unroll_init(rate, 1024); }
static float unroll_cc(void *in, complexf *out, int n, nco_t *nco, float phase) { return shift_unroll_cc(in, out, n, &nco->unroll, phase); }
static void unroll_release(nco_t *nco) { free(nco->unroll.dsin); free(nco->unroll.dcos); }

/* csdr.c:800-849 */
static int cmd_shift_unroll_cc(int argc, char **argv) { return nco_stream(argc, argv, sizeof(complexf), unroll_init, unroll_cc, unroll_release); }

typedef struct { float rate, phase; shift_table_data_t table; } shift_state_t;
static void shift_math_step(void *in, void *out, void *s) { shift_state_t *st = s; st->phase = shift_math_cc(in, out, block, st->rate, st->phase); }
static void shift_table_step(void *in, void *out, void *s) { shift_state_t *st = s; st->phase = shift_table_cc(in, out, block, st->rate, st->table, st->phase); }

static int cmd_shift_math_cc(int argc, char **argv)                        /* csdr.c:703-718 */
{
    if (argc <= 2) return complain("need required parameter (rate)");
    shift_state_t st = {0}; sscanf(argv[2], "%g", &st.rate);
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(complexf), sizeof(complexf), block, 1, shift_math_step, &st);
}

static int cmd_shift_table_cc(int argc, char **argv)                       /* csdr.c:725-747 */
{
    G.wideband = 1;
    if (argc <= 2) return complain("need required parameter (rate)");
    shift_state_t st = {0}; sscanf(argv[2], "%g", &st.rate);
    int table_size = 65536; if (argc > 3) sscanf(argv[3], "%d", &table_size);
    if (!announce_block(open_block())) return -2;
    st.table = shift_table_init(table_size);
    who(); fprintf(stderr, "LUT initialized\n");
    return map_blocks(sizeof(complexf), sizeof(complexf), block, 1, shift_table_step, &st);
}

static void addfast_init(nco_t *nco, float rate) { nco->addfast = shift_addfast_init(rate); }
static float addfast_cc(void *in, complexf *out, int n, nco_t *nco, float phase) { return shift_addfast_cc(in, out, n, &nco->addfast, phase); }

/* csdr.c:749-798 */
static int cmd_shift_addfast_cc(int argc, char **argv) { return nco_stream(argc, argv, sizeof(complexf), addfast_init, addfast_cc, NULL); }

static int cmd_decimating_shift_addition_cc(int argc, char **argv)         /* csdr.c:851-875 */
{
    G.wideband = 1;
    if (argc <= 2) return complain("need required parameter (rate)");
    float rate = 0; sscanf(argv[2], "%g", &rate);
    int decimation = 1; if (argc > 3) sscanf(argv[3], "%d", &decimation);
    if (!open_block()) return -2;
    announce_block(block / decimation);
    shift_addition_data_t nco = decimating_shift_addition_init(rate, decimation);
    decimating_shift_addition_status_t st = {0, 0.f, 0};
    complexf *in = must_alloc(sizeof(complexf) * (size_t)block), *out = must_alloc(sizeof(complexf) * (size_t)block);
    for (;;) {
        if (feof(stdin)) return 0;
        if (!fread(in, sizeof(complexf), (size_t)block, stdin)) return 0;
        st = decimating_shift_addition_cc(in, out, block, nco, decimation, st);
        fwrite(out, sizeof(complexf), (size_t)st.output_size, stdout);
        end_of_block();
    }
}

static int cmd_fft_cc(int argc, char **argv)                               /* csdr.c:1569-1643 (binary output; --octave is not part of this build) */
{
    if (argc <= 3) return complain("need required parameters (fft_size, out_of_every_n_samples)");
    int fft_size = 0; sscanf(argv[2], "%d", &fft_size);
    if (log2n(fft_size) == -1) return complain("fft_size should be power of 2");
    int every = 0; sscanf(argv[3], "%d", &every);
    window_t window = argc >= 5 ? firdes_get_window_from_string(argv[4]) : WINDOW_DEFAULT;
    if (!open_block()) return -2;
    announce_block(fft_size);
    complexf *in = fft_malloc(sizeof(complexf) * (size_t)fft_size), *win = fft_malloc(sizeof(complexf) * (size_t)fft_size);
    complexf *out = fft_malloc(sizeof(complexf) * (size_t)fft_size), *skip = must_alloc(sizeof(complexf) * (size_t)block);
    FFT_PLAN_T *plan = make_fft_c2c(fft_size, win, out, 1, 0);
    if (!plan) return complain("FFT size error.");
    float *table = precalculate_window(fft_size, window);
    memset(in, 0, sizeof(complexf) * (size_t)fft_size);
    for (;;) {
        if (feof(stdin)) return 0;
        read_frame(in, sizeof(complexf), fft_size, every, skip);
        apply_precalculated_window_c(in, win, fft_size, table);
        fft_execute(plan);
        fwrite(out, sizeof(complexf), (size_t)fft_size, stdout);
        end_of_block();
    }
}

/* csdr.c:3414-3498: the spectrum of a real stream, N bins of a 2N-point r2c transform per frame (no Nyquist bin, no half swap).  Frames overlap
 * like fft_cc's for E <= 2N; for E > 2N the reference reads 2N floats and then skips E - 2N COMPLEX samples (its skip counts floats but freads
 * sizeof(complexf) items), so frames start 2E - 2N samples apart -- reproduced here, as the pipes downstream expect.  The first frames of an
 * overlapped stream see zeros before the stream (the reference reads an uninitialised buffer there). */
static int cmd_fft_fc(int argc, char **argv)
{
    if (argc <= 3) return complain("need required parameters (fft_out_size, out_of_every_n_samples)");
    int out_size = 0; sscanf(argv[2], "%d", &out_size);
    if (log2n(out_size) == -1) return complain("fft_out_size should be power of 2");
    if (out_size < 2 || out_size > (1 << 20)) return complain("fft_out_size must be from 2 to 1048576 bins (a real transform of 4 to 2097152 points)");
    const int in_size = 2 * out_size;
    int every = 0; sscanf(argv[3], "%d", &every);
    if (every < 1) return complain("out_of_every_n_samples must be at least 1");
    window_t window = argc >= 5 ? firdes_get_window_from_string(argv[4]) : WINDOW_DEFAULT;
    if (!open_block()) return -2;
    announce_block(out_size);
    float *in = fft_malloc(sizeof(float) * (size_t)in_size), *win = fft_malloc(sizeof(float) * (size_t)in_size);
    complexf *out = fft_malloc(sizeof(complexf) * (size_t)(out_size + 1)), *skip = must_alloc(sizeof(complexf) * (size_t)block);   /* r2c: N + 1 bins */
    FFT_PLAN_T *plan = make_fft_r2c(in_size, win, out, 0);
    if (!plan) return complain("FFT size error.");
    float *table = precalculate_window(in_size, window);
    memset(in, 0, sizeof(float) * (size_t)in_size);
    for (;;) {
        if (feof(stdin)) return 0;
        read_frame(in, sizeof(float), in_size, every, skip);               /* the skip counts complexf samples, as above */
        apply_precalculated_window_f(in, win, in_size, table);
        fft_execute(plan);
        fwrite(out, sizeof(complexf), (size_t)out_size, stdout);
        end_of_block();
    }
}

static void logpower_step(void *in, void *out, void *add_db) { logpower_cf(in, out, block, *(float *)add_db); }

static int cmd_logpower_cf(int argc, char **argv)                          /* csdr.c:1645-1661 */
{
    float add_db = 0; if (argc >= 3) sscanf(argv[2], "%g", &add_db);
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(complexf), sizeof(float), block, 0, logpower_step, &add_db);
}

static int cmd_logaveragepower_cf(int argc, char **argv)                   /* csdr.c:1663-1695 */
{
    G.wideband = 1;
    if (argc <= 4) return complain("need required parameters (add_db, fft_size, avgnumber)");
    float add_db = 0; int fft_size = 0, avgnumber = 0;
    sscanf(argv[2], "%g", &add_db); sscanf(argv[3], "%d", &fft_size); sscanf(argv[4], "%d", &avgnumber);
    complexf *in = must_alloc(sizeof(complexf) * (size_t)fft_size);
    float *acc = must_alloc(sizeof(float) * (size_t)fft_size);
    add_db -= 10.0 * log10(avgnumber);
    for (;;) {
        memset(acc, 0, sizeof(float) * (size_t)fft_size);
        if (feof(stdin)) return 0;
        for (int n = 0; n < avgnumber; n++) { fread(in, sizeof(complexf), (size_t)fft_size, stdin); accumulate_power_cf(in, acc, fft_size); }
        log_ff(acc, acc, fft_size, add_db);
        fwrite(acc, sizeof(float), (size_t)fft_size, stdout);
        end_of_block();
    }
}

static int cmd_fft_exchange_sides_ff(int argc, char **argv)                /* csdr.c:1697-1715: pure I/O, the two halves of every line swap places */
{
    if (argc <= 2) return complain("need required parameters (fft_size)");
    int fft_size = 0; sscanf(argv[2], "%d", &fft_size);
    if (!incoming_block_size()) return -2;
    announce_block(fft_size);
    const size_t half = (size_t)(fft_size / 2);
    float *lower = must_alloc(sizeof(float) * half), *upper = must_alloc(sizeof(float) * half);
    for (;;) {
        if (feof(stdin)) return 0;
        fread(lower, sizeof(float), half, stdin);
        fread(upper, sizeof(float), half, stdin);
        fwrite(upper, sizeof(float), half, stdout);
        fwrite(lower, sizeof(float), half, stdout);
        end_of_block();
    }
}

static int cmd_compress_fft_adpcm_f_u8(int argc, char **argv)              /* csdr.c:1739-1767 */
{
    enum { PAD = 10 };                                                   /* the encoder needs a few values to settle: the line starts with ten copies of its first */
    if (argc <= 2) return complain("need required parameters (fft_size)");
    int fft_size = 0; sscanf(argv[2], "%d", &fft_size);
    const int line = fft_size + PAD;
    if (!incoming_block_size()) return -2;                               /* consumes a preamble if there is one (:1751) */
    announce_block(line);
    float *in = must_alloc(sizeof(float) * (size_t)line);
    short *scaled = must_alloc(sizeof(short) * (size_t)line);
    unsigned char *out = must_alloc((size_t)line / 2 + 1);
    const ima_adpcm_state_t fresh = {0, 0};
    for (;;) {
        if (feof(stdin)) return 0;
        fread(in + PAD, sizeof(float), (size_t)fft_size, stdin);
        for (int k = 0; k < PAD; k++) in[k] = in[PAD];
        for (int k = 0; k < line; k++) scaled[k] = (short)(in[k] * 100);   /* dB -> centi-dB, C conversion like the reference's */
        encode_ima_adpcm_i16_u8(scaled, out, line, fresh);               /* every line starts from the initial state (:1764) */
        fwrite(out, 1, (size_t)line / 2, stdout);
        end_of_block();
    }
}

static void adpcm_step(void *in, void *out, void *st) { *(ima_adpcm_state_t *)st = encode_ima_adpcm_i16_u8(in, out, block, *(ima_adpcm_state_t *)st); }

static int cmd_encode_ima_adpcm(int argc, char **argv)                     /* csdr.c:1891-1904 */
{
    (void)argc; (void)argv;
    if (!open_block()) return -2;
    announce_block(block / 2);
    ima_adpcm_state_t st = {0, 0};
    return map_blocks(sizeof(short), 1, block / 2, 0, adpcm_step, &st);
}

static void limit_step(void *in, void *out, void *max_amplitude) { limit_ff(in, out, block, *(float *)max_amplitude); }

static int cmd_limit_ff(int argc, char **argv)                              /* csdr.c:673-686 */
{
    float max_amplitude = 1.0f; if (argc >= 3) sscanf(argv[2], "%g", &max_amplitude);
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(float), sizeof(float), block, 0, limit_step, &max_amplitude);
}

typedef struct { float tau; int sample_rate; float last; } deemphasis_wfm_t;
static void deemphasis_wfm_step(void *in, void *out, void *s) { deemphasis_wfm_t *d = s; d->last = deemphasis_wfm_ff(in, out, block, d->tau, d->sample_rate, d->last); }

static int cmd_deemphasis_wfm_ff(int argc, char **argv)                     /* csdr.c:1014-1032 */
{
    if (argc <= 3) return complain("need required parameters (sample rate, tau)");
    if (!announce_block(open_block())) return -2;
    deemphasis_wfm_t d = {0, 0, 0};
    sscanf(argv[2], "%d", &d.sample_rate); sscanf(argv[3], "%g", &d.tau);
    who(); fprintf(stderr, "tau = %g, sample_rate = %d\n", d.tau, d.sample_rate);
    return map_blocks(sizeof(float), sizeof(float), block, 0, deemphasis_wfm_step, &d);
}

static int cmd_deemphasis_nfm_ff(int argc, char **argv)                     /* csdr.c:1068-1087 */
{
    if (argc <= 2) return complain("need required parameter (sample rate)");
    int sample_rate = 0; sscanf(argv[2], "%d", &sample_rate);
    if (!announce_block(open_block())) return -2;
    /* The reference filters its still-unread buffer once before the first read (processed starts at 0, :1075-1079), so the stream
     * is effectively prefixed by one block of whatever malloc returned -- zeros in practice, zeros by construction here. */
    float *in = must_alloc(sizeof(float) * (size_t)block), *out = must_alloc(sizeof(float) * (size_t)block);
    int produced = 0;
    for (;;) {
        if (feof(stdin)) return 0;
        fread(in + block - produced, sizeof(float), (size_t)produced, stdin);
        produced = deemphasis_nfm_ff(in, out, block, sample_rate);
        if (!produced) return complain("deemphasis_nfm_ff: invalid sample rate (this function works only with specific sample rates).");
        memmove(in, in + produced, sizeof(float) * (size_t)(block - produced));
        fwrite(out, sizeof(float), (size_t)produced, stdout);
        end_of_block();
    }
}

static int cmd_fractional_decimator_ff(int argc, char **argv)
{
    if (argc <= 2) return complain("need required parameters (rate)");
    float rate = 0; sscanf(argv[2], "%g", &rate);
    int points = 12; if (argc >= 4) sscanf(argv[3], "%d", &points);
    if (points & 1) return complain("num_poly_points should be even");
    if (points < 2) return complain("num_poly_points should be >= 2");
    int prefilter = 0; float transition_bw = 0.03f; window_t window = WINDOW_DEFAULT;
    if (argc >= 5) {
        if (!strcmp(argv[4], "--prefilter")) { who(); fprintf(stderr, "using prefilter with default values\n"); prefilter = 1; }
        else { sscanf(argv[4], "%g", &transition_bw); if (argc >= 6) window = firdes_get_window_from_string(argv[5]); }
    }
    who(); fprintf(stderr, "use_prefilter = %d, num_poly_points = %d, transition_bw = %g, window = %s\n", prefilter, points, transition_bw,
                   firdes_get_string_from_window(window));
    if (!open_block()) return -2;
    announce_block((int)(block / rate));
    if (rate == 1) return clone_blocks();                               /* pass-through special case (:1498, clone_) */
    float *in = must_alloc(sizeof(float) * (size_t)block), *out = must_alloc(sizeof(float) * (size_t)block);
    int taps_length = 0; float *taps = NULL;
    if (prefilter) {
        taps_length = firdes_filter_len(transition_bw);
        who(); fprintf(stderr, "taps_length = %d\n", taps_length);
        taps = must_alloc(sizeof(float) * (size_t)taps_length);
        firdes_lowpass_f(taps, taps_length, 0.5f / (rate - transition_bw), window);
    } else { who(); fprintf(stderr, "not using taps\n"); }
    fractional_decimator_ff_t d = fractional_decimator_ff_init(rate, points, taps, taps_length);
    for (;;) {
        if (feof(stdin)) return 0;
        if (d.input_processed == 0) d.input_processed = block;
        refill(in, sizeof(float), block, d.input_processed);
        fractional_decimator_ff(in, out, block, &d);
        fwrite(out, sizeof(float), (size_t)d.output_size, stdout);
        end_of_block();
    }
}

static int cmd_rational_resampler_ff(int argc, char **argv)                 /* csdr.c:1409-1462 */
{
    if (argc <= 3) return complain("need required parameters (interpolation, decimation)");
    int interpolation = 0, decimation = 0;
    sscanf(argv[2], "%d", &interpolation); sscanf(argv[3], "%d", &decimation);
    float transition_bw = 0.05f; if (argc >= 5) sscanf(argv[4], "%g", &transition_bw);
    window_t window = window_arg(argc, argv, 5);
    if (!open_block()) return -2;
    if (interpolation == 1 && decimation == 1) {                        /* pass-through special case (:1438, clone_) */
        announce_block(block);
        return clone_blocks();
    }
    if (interpolation < 1 || decimation < 1) return complain("interpolation and decimation must be positive integers");
    float *in = must_alloc(sizeof(float) * (size_t)block);
    const int out_size = (int)((long)block * interpolation / decimation);
    announce_block(out_size);
    float *out = must_alloc(sizeof(float) * (size_t)(out_size > 0 ? out_size : 1));
    const int taps_length = firdes_filter_len(transition_bw);
    float *taps = must_alloc(sizeof(float) * (size_t)taps_length);
    rational_resampler_get_lowpass_f(taps, taps_length, interpolation, decimation, window);
    rational_resampler_ff_t d = {0, 0, 0};                              /* the reference's static (.bss) state */
    for (;;) {
        if (feof(stdin)) return 0;
        if (d.input_processed == 0) d.input_processed = block;
        refill(in, sizeof(float), block, d.input_processed);
        d = rational_resampler_ff(in, out, block, interpolation, decimation, taps, taps_length, d.last_taps_delay);
        fwrite(out, sizeof(float), (size_t)d.output_size, stdout);
        end_of_block();
    }
}

static int cmd_fastagc_ff(int argc, char **argv)
{
    static fastagc_ff_t agc;                                            /* zero-initialised like the reference's .bss copy */
    agc.input_size = 1024; if (argc >= 3) sscanf(argv[2], "%d", &agc.input_size);
    incoming_block_size();                                              /* consumes the preamble if there is one (:1385) */
    announce_block(agc.input_size);
    agc.reference = 1.0f; if (argc >= 4) sscanf(argv[3], "%g", &agc.reference);
    agc.buffer_1 = must_alloc(sizeof(float) * (size_t)agc.input_size);
    agc.buffer_2 = must_alloc(sizeof(float) * (size_t)agc.input_size);
    agc.buffer_input = must_alloc(sizeof(float) * (size_t)agc.input_size);
    float *out = must_alloc(sizeof(float) * (size_t)agc.input_size);
    for (;;) {
        if (feof(stdin)) return 0;
        fread(agc.buffer_input, sizeof(float), (size_t)agc.input_size, stdin);
        fastagc_ff(&agc, out);
        fwrite(out, sizeof(float), (size_t)agc.input_size, stdout);
        end_of_block();
    }
}

static void amdemod_step(void *in, void *out, void *state) { (void)state; amdemod_cf(in, out, block); }

static int cmd_amdemod_cf(int argc, char **argv)                            /* csdr.c:1088-1100 */
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(complexf), sizeof(float), block, 0, amdemod_step, NULL);
}

/* fmdemod_atan_cf (csdr.c:970-983, whole blocks only), fmdemod_quadri_novect_cf (:999-1012), amdemod_estimator_cf (:1101-1112) and
 * dcblock_ff (:938-950): the carried phase, sample and filter state start at zero */
static void atan_step(void *in, void *out, void *last) { *(float *)last = fmdemod_atan_cf(in, out, block, *(float *)last); }
static void novect_step(void *in, void *out, void *last) { *(complexf *)last = fmdemod_quadri_novect_cf(in, out, block, *(complexf *)last); }
static void estimator_step(void *in, void *out, void *state) { (void)state; amdemod_estimator_cf(in, out, block, 0.f, 0.f); }
static void dcblock_step(void *in, void *out, void *dcp) { *(dcblock_preserve_t *)dcp = dcblock_ff(in, out, block, 0.f, *(dcblock_preserve_t *)dcp); }

static int cmd_fmdemod_atan_cf(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    float last_phase = 0.f;
    return map_blocks(sizeof(complexf), sizeof(float), block, 2, atan_step, &last_phase);
}

static int cmd_fmdemod_quadri_novect_cf(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    complexf last = {0.f, 0.f};
    return map_blocks(sizeof(complexf), sizeof(float), block, 0, novect_step, &last);
}

static int cmd_amdemod_estimator_cf(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(complexf), sizeof(float), block, 0, estimator_step, NULL);
}

static int cmd_dcblock_ff(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    dcblock_preserve_t dcp = {0.f, 0.f};
    return map_blocks(sizeof(float), sizeof(float), block, 0, dcblock_step, &dcp);
}

static void realpart_step(void *in, void *out, void *state) { (void)state; for (int i = 0; i < block; i++) ((float *)out)[i] = ((complexf *)in)[i].i; }

static int cmd_realpart_cf(int argc, char **argv)                           /* csdr.c:634-645: pure I/O, the I of every sample */
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(complexf), sizeof(float), block, 0, realpart_step, NULL);
}

static int cmd_fastdcblock_ff(int argc, char **argv)                        /* csdr.c:952-968: its own block size, in place */
{
    int size = 1024; if (argc >= 3) sscanf(argv[2], "%d", &size);
    if (size <= 0) return complain("block size must be positive");
    incoming_block_size();                                              /* consumes the preamble if there is one (:959) */
    announce_block(size);
    float *buf = must_alloc(sizeof(float) * (size_t)size);
    float last_dc = 0.0f;
    for (;;) {
        if (feof(stdin)) return 0;
        fread(buf, sizeof(float), (size_t)size, stdin);
        last_dc = fastdcblock_ff(buf, buf, size, last_dc);
        fwrite(buf, sizeof(float), (size_t)size, stdout);
        end_of_block();
    }
}

typedef struct { short hang_time, attack_wait; float reference, attack_rate, decay_rate, max_gain, filter_alpha, last_gain; } agc_args_t;
static void agc_step(void *in, void *out, void *s)
{
    agc_args_t *a = s;
    a->last_gain = agc_ff(in, out, block, a->reference, a->attack_rate, a->decay_rate, a->max_gain, a->hang_time, a->attack_wait, a->filter_alpha, a->last_gain);
}

static int cmd_agc_ff(int argc, char **argv)                                /* csdr.c:1337-1373: one agc_ff call per block */
{
    agc_args_t a = {200, 0, 0.2f, 0.01f, 0.0001f, 65536.0f, 0.999f, 1.0f};
    if (argc >= 3) sscanf(argv[2], "%hd", &a.hang_time);
    if (argc >= 4) sscanf(argv[3], "%g", &a.reference);
    if (argc >= 5) sscanf(argv[4], "%g", &a.attack_rate);
    if (argc >= 6) sscanf(argv[5], "%g", &a.decay_rate);
    if (argc >= 7) sscanf(argv[6], "%g", &a.max_gain);
    if (argc >= 8) sscanf(argv[7], "%hd", &a.attack_wait);
    if (argc >= 9) sscanf(argv[8], "%g", &a.filter_alpha);
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(float), sizeof(float), block, 0, agc_step, &a);
}

static int cmd_bandpass_fir_fft_cc(int argc, char **argv)
{
    float low_cut = 0, high_cut = 0, transition_bw = 0;
    int ctl = open_control(argc, argv);
    if (!initial_tuning(ctl, argc, argv, "%g %g\n", &low_cut, &high_cut) || argc <= 4)
        return complain(ctl ? "need more required parameters (transition_bw)" : "need required parameters (low_cut, high_cut, transition_bw)");
    sscanf(argv[4], "%g", &transition_bw);
    window_t window = window_arg(argc, argv, 5);
    int taps_length = firdes_filter_len(transition_bw);
    int fft_size = next_pow2(taps_length);
    if (fft_size - taps_length < 200) fft_size <<= 1;
    int input_size = fft_size - taps_length + 1, overlap = taps_length - 1;
    who(); fprintf(stderr, "(fft_size = %d) = (taps_length = %d) + (input_size = %d) - 1\n(overlap_length = %d) = taps_length - 1\n",
                   fft_size, taps_length, input_size, overlap);
    if (fft_size <= 2) return complain("FFT size error.");
    if (!announce_block(incoming_block_size())) return -2;
    complexf *taps = must_alloc(sizeof(complexf) * (size_t)fft_size), *taps_fft = must_alloc(sizeof(complexf) * (size_t)fft_size);
    FFT_PLAN_T *plan_taps = make_fft_c2c(fft_size, taps, taps_fft, 1, 0);
    complexf *in = fft_malloc(sizeof(complexf) * (size_t)fft_size), *spec = fft_malloc(sizeof(complexf) * (size_t)fft_size);
    complexf *prod = fft_malloc(sizeof(complexf) * (size_t)fft_size);
    complexf *res[2] = {fft_malloc(sizeof(complexf) * (size_t)fft_size), fft_malloc(sizeof(complexf) * (size_t)fft_size)};
    if (!plan_taps || !in || !spec || !prod || !res[0] || !res[1]) return complain("FFT size error.");
    FFT_PLAN_T *fwd = make_fft_c2c(fft_size, in, spec, 1, 1);
    FFT_PLAN_T *inv[2] = {make_fft_c2c(fft_size, prod, res[0], 0, 1), make_fft_c2c(fft_size, prod, res[1], 0, 1)};
    memset(res[1], 0, sizeof(complexf) * (size_t)fft_size);
    memset(in, 0, sizeof(complexf) * (size_t)fft_size);
    for (;;) {
        who(); fprintf(stderr, "filter initialized, low_cut = %g, high_cut = %g\n", low_cut, high_cut);
        firdes_bandpass_c(taps, taps_length, low_cut, high_cut, window);
        fft_execute(plan_taps);
        for (int odd = 0;; odd = !odd) {
            if (feof(stdin)) return 0;
            fread(in, sizeof(complexf), (size_t)input_size, stdin);
            apply_fir_fft_cc(fwd, inv[odd], taps_fft, res[!odd] + input_size, overlap);
            fwrite(res[odd], sizeof(complexf), (size_t)input_size, stdout);
            if (poll_control(ctl, "%g %g\n", &low_cut, &high_cut)) break;
            end_of_block();
        }
    }
}

static int cmd_fastddc_fwd_cc(int argc, char **argv)
{
    if (argc <= 2) return complain("need required parameter (decimation)");
    int decimation = 0; sscanf(argv[2], "%d", &decimation);
    float transition_bw = 0.05f; if (argc > 3) sscanf(argv[3], "%g", &transition_bw);
    window_arg(argc, argv, 4);                                          /* parsed, but the forward transform has no window (:2295) */
    fastddc_t ddc;
    if (fastddc_init(&ddc, transition_bw, decimation, 0)) { complain("error in fastddc_init()"); return 1; }
    fastddc_print(&ddc, "fastddc_fwd_cc");
    if (!open_block()) return -2;
    announce_block(ddc.fft_size);
    complexf *in = fft_malloc(sizeof(complexf) * (size_t)ddc.fft_size), *out = fft_malloc(sizeof(complexf) * (size_t)ddc.fft_size);
    memset(in, 0, sizeof(complexf) * (size_t)ddc.fft_size);
    who(); fprintf(stderr, "benchmarking FFT...");
    FFT_PLAN_T *plan = make_fft_c2c(ddc.fft_size, in, out, 1, 1);
    fprintf(stderr, " done\n");
    if (!plan) return complain("FFT size error.");
    for (;;) {
        if (feof(stdin)) return 0;
        refill(in, sizeof(complexf), ddc.fft_size, ddc.input_size);                             /* overlap-save (:2292) */
        fft_execute(plan);                                                                      /* no window (:2295) */
        fwrite(out, sizeof(complexf), (size_t)ddc.fft_size, stdout);
        end_of_block();
    }
}

static int cmd_fastddc_inv_cc(int argc, char **argv)
{
    float shift_rate = 0;
    int ctl = open_control(argc, argv);
    if (!initial_tuning(ctl, argc, argv, "%g\n", &shift_rate, NULL)) return complain("need required parameter (rate)");
    const int plus = ctl ? 1 : 0;                                        /* "--fd <fd>" takes the place of <shift_rate> */
    if (argc <= 3 + plus) return complain("need required parameter (decimation)");
    int decimation = 0; sscanf(argv[3 + plus], "%d", &decimation);
    float transition_bw = 0.05f; if (argc > 4 + plus) sscanf(argv[4 + plus], "%g", &transition_bw);
    window_t window = window_arg(argc, argv, 5 + plus);
    for (;;) {
        fastddc_t ddc;
        if (fastddc_init(&ddc, transition_bw, decimation, shift_rate)) { complain("error in fastddc_init()"); return 1; }
        fastddc_print(&ddc, "fastddc_inv_cc");
        if (!open_block()) return -2;
        announce_block(ddc.post_input_size / ddc.post_decimation);
        complexf *taps = must_alloc(sizeof(complexf) * (size_t)ddc.fft_size), *taps_fft = must_alloc(sizeof(complexf) * (size_t)ddc.fft_size);
        FFT_PLAN_T *plan_taps = make_fft_c2c(ddc.fft_size, taps, taps_fft, 1, 0);
        if (!plan_taps) return complain("FFT size error.");
        float half_bw = 0.5 / decimation;
        who(); fprintf(stderr, "preparing a bandpass filter of [%g, %g] cutoff rates. Real transition bandwidth is: %g\n",
                       (-shift_rate) - half_bw, (-shift_rate) + half_bw, 4.0 / ddc.taps_length);
        firdes_bandpass_c(taps, ddc.taps_length, (-shift_rate) - half_bw, (-shift_rate) + half_bw, window);
        fft_execute(plan_taps);
        fft_swap_sides(taps_fft, ddc.fft_size);
        complexf *inv_in = fft_malloc(sizeof(complexf) * (size_t)ddc.fft_inv_size), *inv_out = fft_malloc(sizeof(complexf) * (size_t)ddc.fft_inv_size);
        who(); fprintf(stderr, "benchmarking FFT...");
        FFT_PLAN_T *plan_inverse = make_fft_c2c(ddc.fft_inv_size, inv_in, inv_out, 0, 1);
        fprintf(stderr, " done\n");
        complexf *in = fft_malloc(sizeof(complexf) * (size_t)ddc.fft_size), *out = fft_malloc(sizeof(complexf) * (size_t)ddc.post_input_size);
        decimating_shift_addition_status_t st; memset(&st, 0, sizeof st);
        for (;;) {
            if (feof(stdin)) return 0;
            fread(in, sizeof(complexf), (size_t)ddc.fft_size, stdin);
            st = fastddc_inv_cc(in, out, &ddc, plan_inverse, taps_fft, st);
            fwrite(out, sizeof(complexf), (size_t)st.output_size, stdout);
            end_of_block();
            if (poll_control(ctl, "%g\n", &shift_rate)) break;
        }
        free(taps); free(taps_fft); fft_destroy(plan_taps); fft_destroy(plan_inverse);
        fft_free(inv_in); fft_free(inv_out); fft_free(in); fft_free(out);
    }
}

typedef struct { float rate, reference, max_gain, gain; } simple_agc_args_t;
static void simple_agc_step(void *in, void *out, void *s) { simple_agc_args_t *a = s; simple_agc_cc(in, out, block, a->rate, a->reference, a->max_gain, &a->gain); }

static int cmd_simple_agc_cc(int argc, char **argv)                          /* csdr.c:2902-2931 */
{
    simple_agc_args_t a = {0.f, 1.f, 65535.f, 1.f};
    if (argc <= 2) return complain("need required parameter (rate)");
    sscanf(argv[2], "%f", &a.rate);
    if (a.rate <= 0) return complain("rate should be > 0");
    if (argc > 3) sscanf(argv[3], "%f", &a.reference);
    if (a.reference <= 0) return complain("reference should be > 0");
    if (argc > 4) sscanf(argv[4], "%f", &a.max_gain);
    if (a.max_gain <= 0) return complain("max_gain should be > 0");
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(complexf), sizeof(complexf), block, 0, simple_agc_step, &a);
}

static int cmd_timing_recovery_cc(int argc, char **argv)                     /* csdr.c:2573-2637 */
{
    if (argc <= 2) return complain("need required parameter (algorithm)");
    timing_recovery_algorithm_t algorithm = !strcmp(argv[2], "EARLYLATE") ? TIMING_RECOVERY_ALGORITHM_EARLYLATE : TIMING_RECOVERY_ALGORITHM_GARDNER;
    if (argc <= 3) return complain("need required parameter (decimation factor)");
    int decimation = 0; sscanf(argv[3], "%d", &decimation);
    if (decimation <= 4 || decimation & 3) return complain("decimation factor should be a positive integer divisible by 4");
    float loop_gain = 0.5f; if (argc > 4) sscanf(argv[4], "%f", &loop_gain);
    float max_error = 2.f; if (argc > 5) sscanf(argv[5], "%f", &max_error);
    const int add_q = argc >= 7 && !strcmp(argv[6], "--add_q");
    /* like the reference, --octave / --octave_save select a debug mode only when their count follows (csdr.c:2600) */
    if (argc >= 8 + add_q && (!strcmp(argv[6 + add_q], "--octave") || !strcmp(argv[6 + add_q], "--octave_save")))
        return complain("the --octave and --octave_save debug outputs are not part of this build");
    if (!(fabs((double)loop_gain * (double)max_error) <= 2.0))
        return complain("|mu * max_error| must be at most 2: a larger correction can move a symbol back, before the start of its input");
    who(); fprintf(stderr, "--add_q mode on\n");                        /* printed whatever add_q is, like the reference */
    const int output_error = argc >= 7 + add_q && !strcmp(argv[6 + add_q], "--output_error");
    if (output_error) { who(); fprintf(stderr, "--output_error mode\n"); }
    const int output_indexes = argc >= 7 + add_q && !strcmp(argv[6 + add_q], "--output_indexes");
    if (output_indexes) { who(); fprintf(stderr, "--output_indexes mode\n"); }
    if (!open_block()) return -2;
    announce_block(block / decimation);
    complexf *in = must_alloc(sizeof(complexf) * (size_t)block), *out = must_alloc(sizeof(complexf) * (size_t)block);
    float *error = output_error ? must_alloc(sizeof(float) * (size_t)block) : NULL;
    unsigned *indexes = output_indexes ? must_alloc(sizeof(unsigned) * (size_t)block) : NULL;
    timing_recovery_state_t state = timing_recovery_init(algorithm, decimation, add_q, loop_gain, max_error, -1, NULL);
    fread(in, sizeof(complexf), (size_t)block, stdin);
    unsigned buffer_start_counter = 0;
    for (;;) {
        if (feof(stdin)) return 0;
        timing_recovery_cc(in, out, block, error, (int *)indexes, &state);
        if (error) fwrite(error, sizeof(float), (size_t)state.output_size, stdout);
        else if (indexes) {
            for (int i = 0; i < state.output_size; i++) indexes[i] += buffer_start_counter;
            fwrite(indexes, sizeof(unsigned), (size_t)state.output_size, stdout);
        } else fwrite(out, sizeof(complexf), (size_t)state.output_size, stdout);
        end_of_block();
        buffer_start_counter += (unsigned)state.input_processed;          /* keep the unconsumed tail, refill behind it */
        refill(in, sizeof(complexf), block, state.input_processed);
    }
}

static void dbpsk_step(void *in, void *out, void *state) { (void)state; dbpsk_decoder_c_u8(in, out, block); }

static int cmd_dbpsk_decoder_c_u8(int argc, char **argv)                     /* csdr.c:3256-3268 */
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(complexf), 1, block, 0, dbpsk_step, NULL);
}

/* The byte decoders on the GPU: every read() (whatever the pipe holds, up to one block) goes through one call of the decoder bank, which carries
 * its zero-initialised state_size bytes of state on the device, and the characters it decoded are written and flushed at once.  stdin is
 * unbuffered, so reading a preamble takes its 8 bytes and no more: whatever follows is left to read(). */
static int byte_decoder_stream(int (*bank)(const unsigned char *d_in, int n, unsigned char *d_out, void *d_state, int *d_count), size_t state_size)
{
    setvbuf(stdin, NULL, _IONBF, 0);
    if (!announce_block(open_block())) return -2;
    unsigned char *in = must_alloc((size_t)block), *out = must_alloc((size_t)block);
    unsigned char *d_in = csdrb_device_alloc((size_t)block), *d_out = csdrb_device_alloc((size_t)block);
    void *d_state = csdrb_device_alloc(state_size);                           /* zero-filled */
    int *d_count = csdrb_device_alloc(sizeof(int));
    if (!d_in || !d_out || !d_state || !d_count) { who(); fprintf(stderr, "%s\n", csdrb_last_error()); return -2; }
    for (;;) {
        const ssize_t got = read(STDIN_FILENO, in, (size_t)block);
        if (got <= 0) return 0;
        int count = 0;
        if (csdrb_copy_h2d(d_in, in, (size_t)got, NULL) < 0 || bank(d_in, (int)got, d_out, d_state, d_count) < 0 ||
            csdrb_copy_d2h(&count, d_count, sizeof count, NULL) < 0 || csdrb_stream_synchronize(NULL) < 0 ||
            (count > 0 && (csdrb_copy_d2h(out, d_out, (size_t)count, NULL) < 0 || csdrb_stream_synchronize(NULL) < 0))) {
            who(); fprintf(stderr, "%s\n", csdrb_last_error()); return -2;
        }
        if (count > 0) { fwrite(out, 1, (size_t)count, stdout); fflush(stdout); }
    }
}

static int varicode_bank(const unsigned char *d_in, int n, unsigned char *d_out, void *d_hist, int *d_count)
{
    return csdrb_psk31_varicode_decoder_bank_u8_u8(d_in, n, d_out, n, 1, n, NULL, d_hist, d_count, NULL);
}

/* csdr.c:2418-2430 pushes one getchar() at a time through psk31_varicode_decoder_push and flushes every character; here the varicode bank
 * decodes whole reads.  Its state is the reference's status_shr, 0 at the start. */
static int cmd_psk31_varicode_decoder_u8_u8(int argc, char **argv)
{
    (void)argc; (void)argv;
    return byte_decoder_stream(varicode_bank, sizeof(unsigned long long));
}

static int cmd_serial_line_decoder_f_u8(int argc, char **argv)               /* csdr.c:2490-2530 */
{
    G.wideband = 1;
    serial_line_t serial = {0};
    if (argc <= 2) return complain("need required parameter (samples_per_bits)");
    sscanf(argv[2], "%f", &serial.samples_per_bits);
    if (serial.samples_per_bits < 1) return complain("samples_per_bits should be at least 1.");
    if (serial.samples_per_bits < 5)
        fprintf(stderr, "%s: warning: this algorithm does not work well if samples_per_bits is too low. It should be at least 5.\n", argv[1]);
    serial.databits = 8; if (argc > 3) sscanf(argv[3], "%d", &serial.databits);
    if (serial.databits > 8 || serial.databits < 1) return complain("databits should be between 1 and 8.");
    serial.stopbits = 1; if (argc > 4) sscanf(argv[4], "%f", &serial.stopbits);
    if (serial.stopbits < 1) return complain("stopbits should be equal or above 1.");
    serial.bit_sampling_width_ratio = 0.4f;
    if (!announce_block(open_block())) return -2;
    float *in = must_alloc(sizeof(float) * (size_t)block);
    unsigned char *out = must_alloc((size_t)block);
    /* the reference keeps what a call left unconsumed at the front and refills behind it; after a short final read the buffer's tail still
     * holds the samples of the call before, and that last call is decoded and written like any other */
    for (;;) {
        if (feof(stdin)) return 0;
        refill(in, sizeof(float), block, serial.input_used ? serial.input_used : block);
        serial_line_decoder_f_u8(&serial, in, out, block);
        if (serial.input_used == 0) { who(); fprintf(stderr, "error: serial_line_decoder_f_u8() got stuck.\n"); return -3; }
        fwrite(out, 1, (size_t)serial.output_size, stdout);
        end_of_block();
    }
}

static int baudot_bank(const unsigned char *d_in, int n, unsigned char *d_out, void *d_mode, int *d_count)
{
    return csdrb_rtty_baudot2ascii_bank_u8_u8(d_in, n, d_out, n, 1, n, NULL, d_mode, d_count, NULL);
}

/* csdr.c:2461-2474 pushes one getchar() at a time through rtty_baudot_decoder_lookup and flushes every character; after the end of the input
 * it pushes up to 255 EOF values (0xFF), which give nothing.  Here the baudot bank decodes whole reads.  Its state is the letters (0) / figures
 * mode, letters at the start as fig_mode = 0. */
static int cmd_rtty_baudot2ascii_u8_u8(int argc, char **argv)
{
    (void)argc; (void)argv;
    return byte_decoder_stream(baudot_bank, 1);
}

/* ---- tone filters (csdr.c:2932-3017, 3271-3301) ---------------------------------------------------------------------------------
 * peaks_fir_cc and bfsk_demod_cf frame like the reference: one full read, then after every call the consumed output_size samples leave the
 * front of the buffer and as many are read behind the rest.  The end-of-file test comes before each call, so the output ends with the last
 * call whose refill was complete: a prefix of the valid convolution of the stream. */
static int tone_stream(int taps_length, const complexf *taps, const complexf *mark, const complexf *space)
{
    complexf *in = must_alloc(sizeof(complexf) * (size_t)block);
    void *out = must_alloc(sizeof(complexf) * (size_t)block);
    fread(in, sizeof(complexf), (size_t)block, stdin);
    for (;;) {
        if (feof(stdin)) return 0;
        int n;
        if (taps) { n = apply_fir_cc(in, out, block, (complexf *)taps, taps_length); fwrite(out, sizeof(complexf), (size_t)n, stdout); }
        else { n = bfsk_demod_cf(in, out, block, (complexf *)mark, (complexf *)space, taps_length); fwrite(out, sizeof(float), (size_t)n, stdout); }
        end_of_block();
        refill(in, sizeof(complexf), block, n);
    }
}

static int cmd_firdes_peak_c(int argc, char **argv)                         /* csdr.c:2932-2972 */
{
    if (argc <= 3) return complain("need required parameters (rate, length)");
    float rate; sscanf(argv[2], "%g", &rate);
    int length; sscanf(argv[3], "%d", &length);
    if (length % 2 == 0) return complain("number of symmetric FIR filter taps should be odd");
    window_t window = window_arg(argc, argv, 4);
    if (argc >= 6 && !strcmp(argv[5], "--octave")) return complain("--octave is not offered here (it plots the filter with GNU Octave)");
    if (length <= 0) return 0;                                              /* the reference's loops print nothing */
    complexf *taps = must_alloc(sizeof(complexf) * (size_t)length);
    firdes_add_peak_c(taps, length, rate, window, 0, 1);
    for (int i = 0; i < length; i++) printf("(%g)+(%g)*i ", taps[i].i, taps[i].q);
    return 0;
}

static int cmd_peaks_fir_cc(int argc, char **argv)                          /* csdr.c:2975-3017 */
{
    if (argc <= 2) return complain("need required parameter (taps_length)");
    int taps_length; sscanf(argv[2], "%d", &taps_length);
    const int num_peaks = argc - 3;
    float *peak_rate = must_alloc(sizeof(float) * (size_t)(num_peaks > 0 ? num_peaks : 1));
    for (int i = 0; i < num_peaks; i++) sscanf(argv[3 + i], "%f", peak_rate + i);
    if (num_peaks <= 0) return complain("need required parameter (peak_rate) once or multiple times");
    fflush(stderr);
    if (!open_block()) return -2;
    announce_block(block);
    if (block - taps_length <= 0) return complain("taps_length is below buffer size, decrease taps_length");
    if (taps_length < 2 || taps_length > 4096) return complain("taps_length must be between 2 and 4096");
    complexf *taps = must_alloc(sizeof(complexf) * (size_t)taps_length);     /* zero-filled: the peaks add up in it */
    for (int i = 0; i < num_peaks; i++) firdes_add_peak_c(taps, taps_length, peak_rate[i], WINDOW_DEFAULT, 1, i == num_peaks - 1);
    return tone_stream(taps_length, taps, NULL, NULL);
}

static int cmd_bfsk_demod_cf(int argc, char **argv)                         /* csdr.c:3271-3301 */
{
    if (argc <= 2) return complain("required parameter <frequency_shift> is missing.");
    float frequency_shift = 0; sscanf(argv[2], "%f", &frequency_shift);
    if (argc <= 3) return complain("required parameter <filter_length> is missing.");
    int filter_length = 0; sscanf(argv[3], "%d", &filter_length);
    if (!announce_block(open_block())) return -2;                           /* sendbufsize(initialize_buffers()) (:3286) */
    /* the reference designs NaN taps at length 1 (middle = 0) and computes a negative output count from a filter longer than the buffer */
    if (filter_length < 2 || filter_length > 4096 || filter_length >= block)
        return complain("filter_length must be between 2 and 4096 and below the buffer size");
    complexf *mark = must_alloc(sizeof(complexf) * (size_t)filter_length), *space = must_alloc(sizeof(complexf) * (size_t)filter_length);
    firdes_add_peak_c(mark, filter_length, frequency_shift / 2, WINDOW_DEFAULT, 0, 1);
    firdes_add_peak_c(space, filter_length, -frequency_shift / 2, WINDOW_DEFAULT, 0, 1);
    return tone_stream(filter_length, NULL, mark, space);
}

/* csdr.c:1179-1229: the big buffer (grown while below twice the taps), no read before the first call -- it interpolates the zero-filled buffer --
 * then one call per block, its output written, the consumed inputs (output / I) replaced behind the kept tail.  The next process is told the
 * block times I. */
static int cmd_fir_interpolate_cc(int argc, char **argv)
{
    G.wideband = 1;
    if (argc <= 2) return complain("need required parameter (interpolation factor)");
    int factor = 0; sscanf(argv[2], "%d", &factor);
    if (factor < 1) return complain("the interpolation factor must be at least 1");
    float transition_bw = 0.05f; if (argc >= 4) sscanf(argv[3], "%g", &transition_bw);
    if (!(transition_bw >= 0 && transition_bw < 1.f)) return complain("transition_bw must be in [0, 1)");
    window_t window = window_arg(argc, argv, 4);
    int taps_length = firdes_filter_len(transition_bw);
    who(); fprintf(stderr, "taps_length = %d\n", taps_length);
    while (G.fixed_big < taps_length * 2) G.fixed_big *= 2;
    if (!open_block()) return -2;
    announce_block(block * factor);
    float *taps = must_alloc(sizeof(float) * (size_t)taps_length);
    firdes_lowpass_f(taps, taps_length, 0.5f / (float)factor, window);
    complexf *in = must_alloc(sizeof(complexf) * (size_t)block), *out = must_alloc(sizeof(complexf) * (size_t)block * (size_t)factor);
    for (;;) {
        if (feof(stdin)) return 0;
        int produced = fir_interpolate_cc(in, out, block, factor, taps, taps_length);
        fwrite(out, sizeof(complexf), (size_t)produced, stdout);
        end_of_block();
        refill(in, sizeof(complexf), block, produced / factor);
    }
}

static void fmmod_step(void *in, void *out, void *phase) { *(float *)phase = fmmod_fc(in, out, block, *(float *)phase); }

static int cmd_fmmod_fc(int argc, char **argv)                               /* csdr.c:2142-2154 */
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    float phase = 0.f;
    return map_blocks(sizeof(float), sizeof(complexf), block, 0, fmmod_step, &phase);
}

/* ---- the amplitude modulators (csdr.c:658-671, 2084-2102, 2129-2140, 2156-2172): per-block maps of the reference's framing ----------------- */
static void gain_step(void *in, void *out, void *gain) { gain_ff(in, out, block, *(float *)gain); }

static int cmd_gain_ff(int argc, char **argv)
{
    if (argc <= 2) return complain("need required parameter (gain)");
    float gain = 0.f; sscanf(argv[2], "%g", &gain);
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(float), sizeof(float), block, 0, gain_step, &gain);
}

/* dsb_fc has no library function: the dsb bank on device copies of the block */
typedef struct { float q_value; float *d_in; complexf *d_out; } dsb_state_t;
static void dsb_step(void *in, void *out, void *s)
{
    dsb_state_t *d = s;
    if (csdrb_copy_h2d(d->d_in, in, sizeof(float) * (size_t)block, NULL) < 0 || csdrb_dsb_bank_fc(d->d_in, block, d->d_out, block, 1, block, d->q_value, NULL) < 0 ||
        csdrb_copy_d2h(out, d->d_out, sizeof(complexf) * (size_t)block, NULL) < 0 || csdrb_stream_synchronize(NULL) < 0) {
        who(); fprintf(stderr, "%s\n", csdrb_last_error()); exit(-2);
    }
}

static int cmd_dsb_fc(int argc, char **argv)
{
    dsb_state_t d = {0.f, NULL, NULL};
    if (argc >= 3) sscanf(argv[2], "%g", &d.q_value);
    if (!announce_block(open_block())) return -2;
    d.d_in = csdrb_device_alloc(sizeof(float) * (size_t)block); d.d_out = csdrb_device_alloc(sizeof(complexf) * (size_t)block);
    if (!d.d_in || !d.d_out) { who(); fprintf(stderr, "%s\n", csdrb_last_error()); return -2; }
    return map_blocks(sizeof(float), sizeof(complexf), block, 0, dsb_step, &d);
}

static void dcoffset_step(void *in, void *out, void *state) { (void)state; add_dcoffset_cc(in, out, block); }

static int cmd_add_dcoffset_cc(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(complexf), sizeof(complexf), block, 0, dcoffset_step, NULL);
}

static void fixed_amplitude_step(void *in, void *out, void *a) { fixed_amplitude_cc(in, out, block, *(float *)a); }

static int cmd_fixed_amplitude_cc(int argc, char **argv)
{
    if (argc <= 2) return complain("need required parameter (new_amplitude)");
    float new_amplitude = 0.f; sscanf(argv[2], "%g", &new_amplitude);
    if (!announce_block(open_block())) return -2;
    return map_blocks(sizeof(complexf), sizeof(complexf), block, 0, fixed_amplitude_step, &new_amplitude);
}

/* ---- BPSK31 transmit chain (csdr.c:2684-2701, 2727-2746, 2780-2800, 2816-2833) ---------------------------------------------------
 * psk31_varicode_encoder_u8_u8 | differential_encoder_u8_u8 | psk_modulator_u8_c 2 | psk31_interpolate_sine_cc <sps>, the pipe of the reference's
 * BER harness.  The codec, the modulator and the interpolator are per-block maps with their state carried; the next process is told the block
 * (codec, modulator) or the block times the interpolation. */
static void psk_modulator_step(void *in, void *out, void *n_psk) { psk_modulator_u8_c(in, out, block, *(int *)n_psk); }

static int cmd_psk_modulator_u8_c(int argc, char **argv)
{
    if (argc <= 2) return complain("need required parameter (n_psk)");
    int n_psk = 0; sscanf(argv[2], "%d", &n_psk);
    if (n_psk <= 0 || n_psk > 256) return complain("n_psk should be between 1 and 256");
    if (!announce_block(open_block())) return -2;
    return map_blocks(1, sizeof(complexf), block, 0, psk_modulator_step, &n_psk);
}

typedef struct { int interpolation; complexf last; } sine_state_t;
static void sine_step(void *in, void *out, void *s) { sine_state_t *st = s; st->last = psk31_interpolate_sine_cc(in, out, block, st->interpolation, st->last); }

static int cmd_psk31_interpolate_sine_cc(int argc, char **argv)
{
    if (argc <= 2) return complain("need required parameter (interpolation)");
    sine_state_t st = {0, {0.f, 0.f}}; sscanf(argv[2], "%d", &st.interpolation);
    if (st.interpolation <= 0) return complain("interpolation should be >0");
    if (!open_block()) return -2;
    announce_block(block * st.interpolation);
    return map_blocks(sizeof(complexf), sizeof(complexf), block * st.interpolation, 0, sine_step, &st);
}

typedef struct { int encode; unsigned char state; } codec_state_t;
static void codec_step(void *in, void *out, void *s) { codec_state_t *st = s; st->state = differential_codec(in, out, block, st->encode, st->state); }

static int codec_stream(int encode)
{
    if (!announce_block(open_block())) return -2;
    codec_state_t st = {encode, 0};
    return map_blocks(1, 1, block, 0, codec_step, &st);
}
static int cmd_differential_encoder_u8_u8(int argc, char **argv) { (void)argc; (void)argv; return codec_stream(1); }
static int cmd_differential_decoder_u8_u8(int argc, char **argv) { (void)argc; (void)argv; return codec_stream(0); }

/* The reference's encoder loop as it runs (csdr.c:2780-2800), so that a pipe graph keeps its bytes: one read into a zero-filled block, then
 * encode the block, write, the end-of-file test, and a refill that reads the consumed bytes into a buffer that is never encoded (csdr.c:2797
 * reads into input_buffer, not local_input_buffer).  Every block after the first therefore repeats the first block's bits, once per further
 * read, until the end of the input; a short first read encodes the zero padding as NUL characters.  Text longer than one block belongs to the
 * drop-in or the bank, which encode every byte. */
static int cmd_psk31_varicode_encoder_u8_u8(int argc, char **argv)
{
    (void)argc; (void)argv;
    if (!open_block()) return -2;
    announce_block(block * 8);
    const int output_max_size = block * 30;
    unsigned char *in = must_alloc((size_t)block), *out = must_alloc((size_t)output_max_size), *refilled = must_alloc((size_t)block);
    fread(in, 1, (size_t)block, stdin);
    for (;;) {
        int input_processed = 0, output_size = 0;
        psk31_varicode_encoder_u8_u8(in, out, block, output_max_size, &input_processed, &output_size);
        fwrite(out, 1, (size_t)output_size, stdout);
        if (feof(stdin)) return 0;
        memmove(in, in + input_processed, (size_t)(block - input_processed));
        fread(refilled, 1, (size_t)input_processed, stdin);
        end_of_block();
    }
}

/* ---- dispatch ------------------------------------------------------------------------------------ */
static const struct { const char *name; int (*run)(int, char **); const char *syntax; } kCommands[] = {
    {"convert_u8_f", cmd_convert_u8_f, "convert_u8_f"},
    {"convert_s16_f", cmd_convert_s16_f, "convert_s16_f"},
    {"convert_i16_f", cmd_convert_s16_f, "convert_i16_f"},
    {"convert_f_s16", cmd_convert_f_s16, "convert_f_s16"},
    {"convert_f_i16", cmd_convert_f_s16, "convert_f_i16"},
    {"convert_s8_f", cmd_convert_s8_f, "convert_s8_f"},
    {"convert_f_s8", cmd_convert_f_s8, "convert_f_s8"},
    {"convert_f_u8", cmd_convert_f_u8, "convert_f_u8"},
    {"convert_s24_f", cmd_convert_s24_f, "convert_s24_f [--bigendian]"},
    {"convert_f_s24", cmd_convert_f_s24, "convert_f_s24 [--bigendian]"},
    {"shift_addition_cc", cmd_shift_addition_cc, "shift_addition_cc <rate> | --fifo <fifo_path> | --fd <fd>"},
    {"shift_addition_fc", cmd_shift_addition_fc, "shift_addition_fc <rate> | --fifo <fifo_path> | --fd <fd>"},
    {"fir_decimate_cc", cmd_fir_decimate_cc, "fir_decimate_cc <decimation_factor> [transition_bw [window]]"},
    {"fmdemod_quadri_cf", cmd_fmdemod_quadri_cf, "fmdemod_quadri_cf"},
    {"fractional_decimator_ff", cmd_fractional_decimator_ff, "fractional_decimator_ff <decimation_rate> [num_poly_points ( [transition_bw [window]] | --prefilter )]"},
    {"rational_resampler_ff", cmd_rational_resampler_ff, "rational_resampler_ff <interpolation> <decimation> [transition_bw [window]]"},
    {"fastagc_ff", cmd_fastagc_ff, "fastagc_ff [block_size [reference]]"},
    {"limit_ff", cmd_limit_ff, "limit_ff [max_amplitude]"},
    {"amdemod_cf", cmd_amdemod_cf, "amdemod_cf"},
    {"amdemod_estimator_cf", cmd_amdemod_estimator_cf, "amdemod_estimator_cf"},
    {"fmdemod_atan_cf", cmd_fmdemod_atan_cf, "fmdemod_atan_cf"},
    {"fmdemod_quadri_novect_cf", cmd_fmdemod_quadri_novect_cf, "fmdemod_quadri_novect_cf"},
    {"dcblock_ff", cmd_dcblock_ff, "dcblock_ff"},
    {"realpart_cf", cmd_realpart_cf, "realpart_cf"},
    {"fastdcblock_ff", cmd_fastdcblock_ff, "fastdcblock_ff [block_size (<= 49152)]"},
    {"agc_ff", cmd_agc_ff, "agc_ff [hang_time [reference [attack_rate [decay_rate [max_gain [attack_wait [filter_alpha]]]]]]]"},
    {"fft_exchange_sides_ff", cmd_fft_exchange_sides_ff, "fft_exchange_sides_ff <fft_size>"},
    {"compress_fft_adpcm_f_u8", cmd_compress_fft_adpcm_f_u8, "compress_fft_adpcm_f_u8 <fft_size>"},
    {"encode_ima_adpcm_i16_u8", cmd_encode_ima_adpcm, "encode_ima_adpcm_i16_u8"},
    {"encode_ima_adpcm_s16_u8", cmd_encode_ima_adpcm, "encode_ima_adpcm_s16_u8"},
    {"shift_unroll_cc", cmd_shift_unroll_cc, "shift_unroll_cc <rate> | --fifo <fifo_path> | --fd <fd>"},
    {"shift_math_cc", cmd_shift_math_cc, "shift_math_cc <rate>"},
    {"shift_table_cc", cmd_shift_table_cc, "shift_table_cc <rate> [table_size]"},
    {"shift_addfast_cc", cmd_shift_addfast_cc, "shift_addfast_cc <rate> | --fifo <fifo_path> | --fd <fd>"},
    {"decimating_shift_addition_cc", cmd_decimating_shift_addition_cc, "decimating_shift_addition_cc <rate> [decimation]"},
    {"fft_cc", cmd_fft_cc, "fft_cc <fft_size> <out_of_every_n_samples> [window]"},
    {"fft_fc", cmd_fft_fc, "fft_fc <fft_out_size> <out_of_every_n_samples> [window]"},
    {"logpower_cf", cmd_logpower_cf, "logpower_cf [add_db]"},
    {"logaveragepower_cf", cmd_logaveragepower_cf, "logaveragepower_cf <add_db> <fft_size> <avgnumber>"},
    {"deemphasis_wfm_ff", cmd_deemphasis_wfm_ff, "deemphasis_wfm_ff <sample_rate> <tau>"},
    {"deemphasis_nfm_ff", cmd_deemphasis_nfm_ff, "deemphasis_nfm_ff <one_of_the_predefined_sample_rates>"},
    {"bandpass_fir_fft_cc", cmd_bandpass_fir_fft_cc, "bandpass_fir_fft_cc <low_cut> <high_cut> <transition_bw> [window] | --fifo <fifo_path> <transition_bw> [window]"},
    {"fastddc_fwd_cc", cmd_fastddc_fwd_cc, "fastddc_fwd_cc <decimation> [transition_bw [window]]"},
    {"simple_agc_cc", cmd_simple_agc_cc, "simple_agc_cc <rate> [reference [max_gain]]"},
    {"timing_recovery_cc", cmd_timing_recovery_cc, "timing_recovery_cc <algorithm> <decimation> [mu [max_error [--add_q [--output_error | --output_indexes]]]]"},
    {"dbpsk_decoder_c_u8", cmd_dbpsk_decoder_c_u8, "dbpsk_decoder_c_u8"},
    {"psk31_varicode_decoder_u8_u8", cmd_psk31_varicode_decoder_u8_u8, "psk31_varicode_decoder_u8_u8"},
    {"serial_line_decoder_f_u8", cmd_serial_line_decoder_f_u8, "serial_line_decoder_f_u8 <samples_per_bits> [databits [stopbits]]"},
    {"rtty_baudot2ascii_u8_u8", cmd_rtty_baudot2ascii_u8_u8, "rtty_baudot2ascii_u8_u8"},
    {"firdes_peak_c", cmd_firdes_peak_c, "firdes_peak_c <rate> <length> [window]"},
    {"peaks_fir_cc", cmd_peaks_fir_cc, "peaks_fir_cc <taps_length> <peak_rate> [peak_rate ...]"},
    {"bfsk_demod_cf", cmd_bfsk_demod_cf, "bfsk_demod_cf <spacing> <filter_length>"},
    {"fastddc_inv_cc", cmd_fastddc_inv_cc, "fastddc_inv_cc <shift_rate> <decimation> [transition_bw [window]] | --fifo <fifo_path> ... | --fd <fd> ..."},
    {"fir_interpolate_cc", cmd_fir_interpolate_cc, "fir_interpolate_cc <interpolation_factor> [transition_bw [window]]"},
    {"fmmod_fc", cmd_fmmod_fc, "fmmod_fc"},
    {"gain_ff", cmd_gain_ff, "gain_ff <gain>"},
    {"dsb_fc", cmd_dsb_fc, "dsb_fc [q_value]"},
    {"add_dcoffset_cc", cmd_add_dcoffset_cc, "add_dcoffset_cc"},
    {"fixed_amplitude_cc", cmd_fixed_amplitude_cc, "fixed_amplitude_cc <new_amplitude>"},
    {"psk31_varicode_encoder_u8_u8", cmd_psk31_varicode_encoder_u8_u8, "psk31_varicode_encoder_u8_u8"},
    {"differential_encoder_u8_u8", cmd_differential_encoder_u8_u8, "differential_encoder_u8_u8"},
    {"differential_decoder_u8_u8", cmd_differential_decoder_u8_u8, "differential_decoder_u8_u8"},
    {"psk_modulator_u8_c", cmd_psk_modulator_u8_c, "psk_modulator_u8_c <n_psk>"},
    {"psk31_interpolate_sine_cc", cmd_psk31_interpolate_sine_cc, "psk31_interpolate_sine_cc <interpolation>"},
};

static int usage(void)
{
    fprintf(stderr, "csdr (H100 hot-path build) - DSP blocks on stdin/stdout, computed by libcsdr_b200 on a CUDA device\nusage:\n");
    for (size_t k = 0; k < sizeof kCommands / sizeof kCommands[0]; k++) fprintf(stderr, "    csdr %s\n", kCommands[k].syntax);
    fprintf(stderr, "commands of the reference CLI outside this list are not part of this build\n");
    return -1;
}

int main(int argc, char **argv)
{
    read_environment();
    G.argc = argc; G.argv = argv;
    if (argc <= 1 || !strcmp(argv[1], "--help")) return usage();
    fcntl(STDIN_FILENO, F_SETPIPE_SZ, 65536 * 32);
    fcntl(STDOUT_FILENO, F_SETPIPE_SZ, 65536 * 32);
    for (size_t k = 0; k < sizeof kCommands / sizeof kCommands[0]; k++)
        if (!strcmp(argv[1], kCommands[k].name)) return kCommands[k].run(argc, argv);
    return complain("function name given in argument 1 does not exist (in this hot-path build). Possible causes: you have mistyped the commmand name, "
                    "or the command belongs to the reference CLI only.");
}
