// rtty.cu -- the RTTY receive chain of the reference,
//   fmdemod_quadri_cf | serial_line_decoder_f_u8 <samples_per_bit> 5 1.5 | rtty_baudot2ascii_u8_u8
// behind the discriminator, as banks, one row per channel:
//   serial_line_decoder_f_u8   one warp per channel: a ballot finds the next falling edge 32 samples at a time, then lane k < databits
//                              sums data bit k's window and lane databits the stop window, and the warp decides and advances together
//   rtty_baudot2ascii_u8_u8    one warp per channel: 32 codes per step, the FIGS/LTRS mode of each from a ballot over the shift codes,
//                              the table lookup, the characters compacted with a ballot
//
// The reference builds with -O3 -ffast-math (its Makefile:38).  DESIGN.md section 7 records the arithmetic of that build as read from its
// disassembly; the decoder follows it operation for operation, with explicit _rn intrinsics so that nothing is contracted into an FMA.
#include "common.cuh"
#include "kernels.h"

namespace csdrb {

#ifdef CSDRB_HOST_EMULATION
static inline double dadd_rn(double a, double b) { volatile double r = a + b; return r; }
static inline double dmul_rn(double a, double b) { volatile double r = a * b; return r; }
#else
__device__ __forceinline__ double dadd_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dmul_rn(double a, double b) { return __dmul_rn(a, b); }
#endif

// ---------------------------------------------------------------------------------------------- serial_line_decoder_f_u8
// libcsdr.c:1662-1729 as built.  One call on n samples x[0..n):
//   start bit: the first i >= 1 with x[i] < 0 && !(x[i-1] <= 0) (comiss: a NaN before a negative sample is an edge); none: consume
//     max(n, 1) and return
//   all_bits = (float)(1 + databits) + stopbits; when (float)(spb*all_bits) + (float)sb >= (float)n the character does not fit: consume
//     max(0, sb - 2) and return
//   data bit k: the window [(int)(((double)(k+1) + 0.5*(double)(1 - r)) * spb + sb), (int)(((double)(k+1) + 0.5*(double)(1 + r)) * spb + sb)),
//     1 - r and 1 + r in float, the rest in double; the bit is sum > 0 (a NaN sum is 0), the first bit most significant
//   stop bit: base = (double)(float)(spb*(float)(1 + databits) + (float)sb), half = ((double)stopbits * spb) * 0.5, the window
//     [(int)((double)(1 - r)*half + base), (int)(base + half*(double)(1 + r))); sum < 0 is a faulty stop bit: consume min(sb + 1, n) and return
//   otherwise emit the character, consume (int)min((float)n, (float)(spb*all_bits) + (float)sb) (minss) and go on with what remains
// A window of 4 or more samples is summed in four partial sums (lane j of the SSE register takes samples j, j+4, ...) combined as
// (l0 + l2) + (l1 + l3), then its last (count mod 4) samples one by one; a shorter window one by one from 0.
__device__ __forceinline__ float sld_window_sum(const float* __restrict__ x, int a, int b)
{
    float acc = 0.f;
    int k = a;
    if (b - a >= 4) {
        float l0 = 0.f, l1 = 0.f, l2 = 0.f, l3 = 0.f;
        for (const int e = a + ((b - a) & ~3); k < e; k += 4) {
            l0 = __fadd_rn(l0, x[k]); l1 = __fadd_rn(l1, x[k + 1]); l2 = __fadd_rn(l2, x[k + 2]); l3 = __fadd_rn(l3, x[k + 3]);
        }
        acc = __fadd_rn(__fadd_rn(l0, l2), __fadd_rn(l1, l3));
    }
    for (; k < b; k++) acc = __fadd_rn(acc, x[k]);
    return acc;
}

constexpr int SLD_WARPS = 4;

// Channel c's unconsumed samples are in[c][start[c] .. end).  While at least `bufsize` of them remain, one reference call runs on exactly
// bufsize samples from start[c] and start[c] advances by its input_used -- the CLI's memmove-and-refill framing (csdr.c:2517-2527).  A call
// that consumes nothing is the CLI's "got stuck": the row stops there with stuck[c] = 1.
__global__ void __launch_bounds__(SLD_WARPS * 32)
serial_line_bank_kernel(const float* __restrict__ in, long in_stride, int end, int* __restrict__ start_io, unsigned char* __restrict__ out,
                        long out_stride, int* __restrict__ count, int* __restrict__ stuck, int channels, SerialLineParams p, int bufsize)
{
    const int lane = threadIdx.x & 31, c = blockIdx.x * SLD_WARPS + (threadIdx.x >> 5);
    if (c >= channels) return;                                              // whole warps leave together
    const float* row = in + (long)c * in_stride;
    unsigned char* o = out + (long)c * out_stride;
    const int nbits = p.databits;
    const float spb = p.samples_per_bits;
    const float span = __fmul_rn(spb, __fadd_rn((float)(1 + nbits), p.stopbits));           // spb * all_bits
    const float data_span = __fmul_rn(spb, (float)(1 + nbits));
    const double spbd = (double)spb;
    const double one_minus = (double)__fsub_rn(1.0f, p.bit_sampling_width_ratio), one_plus = (double)__fadd_rn(p.bit_sampling_width_ratio, 1.0f);
    // this lane's window: data bit `lane` (its offsets from the start bit in bit periods), or the stop bit for lane == nbits
    const double data_lo = dadd_rn((double)(lane + 1), dmul_rn(0.5, one_minus)), data_hi = dadd_rn((double)(lane + 1), dmul_rn(0.5, one_plus));
    const double half = dmul_rn(dmul_rn((double)p.stopbits, spbd), 0.5);
    const double stop_lo = dmul_rn(one_minus, half), stop_hi = dmul_rn(half, one_plus);
    int pos = start_io[c], cnt = 0, stk = 0;
    while (end - pos >= bufsize) {
        const float* x = row + pos;
        int n = bufsize, used = 0;
        for (;;) {
            int sb = -1;
            for (int i0 = 1; i0 < n; i0 += 32) {
                const int i = i0 + lane;
                const unsigned m = __ballot_sync(0xffffffffu, i < n && x[i] < 0.f && !(x[i - 1] <= 0.f));
                if (m) { sb = i0 + __popc((m & (0u - m)) - 1u); break; }   // the lowest edge of the 32
            }
            if (sb < 0) { used += n > 1 ? n : 1; break; }
            const float sbf = (float)sb;
            if (__fadd_rn(span, sbf) >= (float)n) { used += sb > 2 ? sb - 2 : 0; break; }
            float acc = 0.f;
            if (lane <= nbits) {
                int a, b;
                if (lane < nbits) {
                    a = (int)dadd_rn(dmul_rn(data_lo, spbd), (double)sb);
                    b = (int)dadd_rn(dmul_rn(data_hi, spbd), (double)sb);
                } else {
                    const double base = (double)__fadd_rn(data_span, sbf);
                    a = (int)dadd_rn(stop_lo, base);
                    b = (int)dadd_rn(base, stop_hi);
                }
                acc = sld_window_sum(x, a, min(b, n));                      // b <= n always holds for bufsize <= 2^22 and 0 <= ratio <= 1
            }
            const unsigned ones = __ballot_sync(0xffffffffu, lane < nbits && acc > 0.f);
            const float stop = __shfl_sync(0xffffffffu, acc, nbits);
            if (stop < 0.f) { used += n > sb ? sb + 1 : n; break; }
            if (lane == 0) {
                unsigned shr = 0;
                for (int k = 0; k < nbits; k++) shr = (shr << 1) | ((ones >> k) & 1u);
                o[cnt] = (unsigned char)shr;
            }
            cnt++;
            const float u = __fadd_rn(span, sbf), nf = (float)n;
            const int step = (int)(nf < u ? nf : u);                        // minss
            used += step; x += step; n -= step;
            if (!n) break;
        }
        if (used == 0) { stk = 1; break; }
        pos += used;
    }
    if (lane == 0) { start_io[c] = pos; count[c] = cnt; stuck[c] = stk; }
}

int serial_line_max_outputs(float samples_per_bits, int databits, float stopbits, int input_size)
{
    const float span = samples_per_bits * ((float)(1 + databits) + stopbits);
    return input_size / (int)span + 1;
}

int launch_serial_line_bank(const float* d_in, long in_stride, int end, int* d_start_io, unsigned char* d_out, long out_stride, int* d_count,
                            int* d_stuck, int channels, const void* h_params_v, int bufsize, cudaStream_t st)
{
    if (!h_params_v) { set_error("serial_line bank: no parameters"); return -1; }
    const SerialLineParams& p = *static_cast<const SerialLineParams*>(h_params_v);
    if (p.databits < 1 || p.databits > 8) { set_error("serial_line bank: databits %d (1..8 are served, the CLI's range)", p.databits); return -1; }
    if (!(p.samples_per_bits >= 1.f && p.samples_per_bits <= 1e6f) || !(p.stopbits >= 1.f && p.stopbits <= 1e3f)) {
        set_error("serial_line bank: samples_per_bits must be in [1, 1e6] and stopbits in [1, 1000]");
        return -1;
    }
    if (!(p.bit_sampling_width_ratio >= 0.f && p.bit_sampling_width_ratio <= 1.f)) {
        set_error("serial_line bank: bit_sampling_width_ratio must be in [0, 1] (each window then lies inside its bit)");
        return -1;
    }
    if (bufsize < 1 || bufsize > (1 << 22)) { set_error("serial_line bank: bufsize %d outside 1..2^22", bufsize); return -1; }
    if (channels <= 0) return 0;
    if (end < 0 || in_stride < end) { set_error("serial_line bank: row stride shorter than the row"); return -1; }
    const int cap = serial_line_max_outputs(p.samples_per_bits, p.databits, p.stopbits, end);
    if (out_stride < cap) { set_error("serial_line bank: output rows need room for %d characters", cap); return -1; }
    serial_line_bank_kernel<<<(unsigned)((channels + SLD_WARPS - 1) / SLD_WARPS), SLD_WARPS * 32, 0, st>>>(d_in, in_stride, end, d_start_io, d_out,
                                                                                                      out_stride, d_count, d_stuck, channels, p, bufsize);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---------------------------------------------------------------------------------------------- rtty_baudot2ascii_u8_u8
// rtty_baudot_decoder_lookup (libcsdr.c:1608-1616) over a stream of codes: FIGS (27) and LTRS (31) set the mode and give nothing; a code
// below 32 gives its ITA2 character in the current mode, 0 (nothing) for code 0; 32 and above give nothing.  The table is ITA2 indexed by
// the code as serial_line_decoder_f_u8 assembles it (first data bit most significant), letters then figures.
__constant__ unsigned char kIta2[2][32] = {
    {0, 'T', '\r', 'O', ' ', 'H', 'N', 'M', '\n', 'L', 'R', 'G', 'I', 'P', 'C', 'V', 'E', 'Z', 'D', 'B', 'S', 'Y', 'F', 'X', 'A', 'W', 'J', 0, 'U', 'Q', 'K', 0},
    {0, '5', '\r', '9', ' ', '$', ',', '.', '\n', ')', '4', '*', '8', '0', ':', '=', '3', '+', '#', '?', '\'', '6', '@', '/', '-', '2', '\a', 0, '7', '1', '(', 0},
};
constexpr int BD_WARPS = 4;

__global__ void __launch_bounds__(BD_WARPS * 32)
baudot_bank_kernel(const unsigned char* __restrict__ in, long in_stride, unsigned char* __restrict__ out, long out_stride, int channels, int n,
                   const int* __restrict__ lengths, unsigned char* __restrict__ mode_io, int* __restrict__ count)
{
    const int lane = threadIdx.x & 31, c = blockIdx.x * BD_WARPS + (threadIdx.x >> 5);
    if (c >= channels) return;                                              // whole warps leave together
    const unsigned char* x = in + (long)c * in_stride;
    unsigned char* o = out + (long)c * out_stride;
    const int len = lengths ? min(lengths[c], n) : n;
    const unsigned below = (1u << lane) - 1u;
    unsigned mode = mode_io[c] ? 1u : 0u;
    int cnt = 0;
    for (int i0 = 0; i0 < len; i0 += 32) {
        const int i = i0 + lane;
        const unsigned code = i < len ? x[i] : 255u;
        const unsigned figs = __ballot_sync(0xffffffffu, code == 27u), ltrs = __ballot_sync(0xffffffffu, code == 31u);
        // the shift codes before this lane are disjoint bit sets: the later one is the larger mask
        const unsigned f = figs & below, l = ltrs & below;
        const unsigned m = (f | l) ? (f > l ? 1u : 0u) : mode;
        const unsigned char ch = code < 32u ? kIta2[m][code] : 0;
        const unsigned keep = __ballot_sync(0xffffffffu, ch != 0);
        if (ch) o[cnt + __popc(keep & below)] = ch;
        cnt += __popc(keep);
        if (figs | ltrs) mode = figs > ltrs ? 1u : 0u;
    }
    if (lane == 0) { mode_io[c] = (unsigned char)mode; count[c] = cnt; }
}

int launch_baudot_bank(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int n, const int* d_lengths,
                       unsigned char* d_mode_io, int* d_count, cudaStream_t st)
{
    if (channels <= 0) return 0;
    if (n < 0 || in_stride < n || out_stride < n) { set_error("baudot bank: row stride shorter than the row"); return -1; }
    baudot_bank_kernel<<<(unsigned)((channels + BD_WARPS - 1) / BD_WARPS), BD_WARPS * 32, 0, st>>>(d_in, in_stride, d_out, out_stride, channels, n,
                                                                                                   d_lengths, d_mode_io, d_count);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace csdrb
