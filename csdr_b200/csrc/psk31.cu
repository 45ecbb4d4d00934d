// psk31.cu -- the BPSK31 receive chain of the reference (csdr.c:130-159 usage; OpenWebRX runs it as
//   simple_agc_cc 0.001 0.5 | timing_recovery_cc GARDNER <sps> 0.5 2 --add_q | dbpsk_decoder_c_u8 | psk31_varicode_decoder_u8_u8)
// as banks, one row per channel:
//   simple_agc_cc                 one serial gain chain per channel, lane t of warp 0 walks channel t (the agc_bank_kernel scheme)
//   timing_recovery_cc            one thread per channel; the recursion is per symbol and reads three samples straight from global memory
//   dbpsk_decoder_c_u8            fully parallel: output i needs inputs i-1 and i
//   psk31_varicode_decoder_push   one thread per bit (the character at bit i is a function of the last 14 bits), ballot-compacted per channel
//
// The reference builds with -O3 -ffast-math (its Makefile:38).  DESIGN.md section 7 records the arithmetic of that build as read from its
// disassembly; these kernels follow it operation for operation, with explicit _rn intrinsics so that nothing is contracted into an FMA.
#include "common.cuh"
#include "kernels.h"
#include "varicode.cuh"

namespace csdrb {

// ---------------------------------------------------------------------------------------------- simple_agc_cc
// Per sample (libcsdr.c:2201-2217 as built): s = i*i + q*q; ideal = min(reference/sqrt(s), max_gain) then max(., 0), where a zero,
// subnormal, infinite or NaN s gives ideal = max_gain (the build's rsqrtss Newton step yields NaN there, and minss(NaN, max_gain) is
// max_gain); g = (ideal - g)*rate + g*(1 - rate); y = (g*i, g*q).  The reference/sqrt(s) is correctly rounded; the build's rsqrtss seed is
// a vendor-dependent approximation, so this one quotient is the only place where the kernel and the reference build differ (DESIGN 7).
//
// A CTA owns SAGC_CH = 32 channels.  Warps 1..3 stage tiles of 32 samples x 32 channels through shared memory (coalesced along the samples)
// and compute `ideal` for the tile (the next tile's loads are issued right after, into registers); lane t of warp 0 runs the gain chain of channel c0 + t over the tile and leaves the gain of every
// sample in place of its `ideal`; the staging warps then write y = g*x.  Three tiles rotate: at step k the stagers fill tile k and drain
// tile k-2 while the chain lane works through tile k-1.
constexpr int SAGC_CH = 32, SAGC_T = 32, SAGC_WARPS = 4, SAGC_PITCH = SAGC_T + 1;
constexpr int SAGC_STAGERS = (SAGC_WARPS - 1) * 32, SAGC_PER = (SAGC_CH * SAGC_T + SAGC_STAGERS - 1) / SAGC_STAGERS;

struct SimpleAgcTile { float2 x[SAGC_CH][SAGC_PITCH]; float g[SAGC_CH][SAGC_PITCH]; };

__device__ __forceinline__ float simple_agc_ideal(float2 v, float reference, float max_gain)
{
    const float s = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
    float ideal = (s >= 1.17549435e-38f && s <= 3.40282347e38f) ? __fdiv_rn(reference, sqrtf(s)) : max_gain;
    ideal = ideal < max_gain ? ideal : max_gain;                               // minss: a NaN quotient becomes max_gain
    return ideal > 0.f ? ideal : 0.f;                                          // maxss
}

__global__ void __launch_bounds__(SAGC_WARPS * 32)
simple_agc_bank_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride, int channels, int n,
                       float rate, float reference, float max_gain, float* __restrict__ gain_io)
{
    __shared__ SimpleAgcTile tiles[3];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int c0 = blockIdx.x * SAGC_CH;
    const int ntiles = (n + SAGC_T - 1) / SAGC_T;
    if (warp == 0) {
        const int c = c0 + lane;
        float g = c < channels ? gain_io[c] : 1.f;
        const float one_minus_rate = __fsub_rn(1.0f, rate);
        for (int k = 0; k <= ntiles + 1; k++) {
            const int t = k - 1;
            if (t >= 0 && t < ntiles && c < channels) {
                SimpleAgcTile& tl = tiles[t % 3];
                const int m = min(SAGC_T, n - t * SAGC_T);
                for (int i = 0; i < m; i++) {
                    g = __fadd_rn(__fmul_rn(__fsub_rn(tl.g[lane][i], g), rate), __fmul_rn(g, one_minus_rate));
                    tl.g[lane][i] = g;
                }
            }
            __syncthreads();
        }
        if (c < channels) gain_io[c] = g;
    } else {
        // each stager owns SAGC_PER elements of a tile; tile k+1 is loaded into registers while tile k-1's chain runs, so the loads are in
        // flight across the barrier instead of in front of the chain
        const int ltid = tid - 32;
        float2 v[SAGC_PER];
        auto load = [&](int k) {
#pragma unroll
            for (int j = 0; j < SAGC_PER; j++) {
                const int e = ltid + j * SAGC_STAGERS, ch = e / SAGC_T, i = e % SAGC_T, c = c0 + ch;
                const long pos = (long)k * SAGC_T + i;
                v[j] = (e < SAGC_CH * SAGC_T && c < channels && pos < n) ? in[(long)c * in_stride + pos] : make_float2(0.f, 0.f);
            }
        };
        if (ntiles > 0) load(0);
        for (int k = 0; k <= ntiles + 1; k++) {
            if (k < ntiles) {
                SimpleAgcTile& tl = tiles[k % 3];
#pragma unroll
                for (int j = 0; j < SAGC_PER; j++) {
                    const int e = ltid + j * SAGC_STAGERS;
                    if (e >= SAGC_CH * SAGC_T) continue;
                    tl.x[e / SAGC_T][e % SAGC_T] = v[j];
                    tl.g[e / SAGC_T][e % SAGC_T] = simple_agc_ideal(v[j], reference, max_gain);
                }
                if (k + 1 < ntiles) load(k + 1);
            }
            if (k >= 2) {
                SimpleAgcTile& tl = tiles[(k - 2) % 3];
                for (int e = ltid; e < SAGC_CH * SAGC_T; e += SAGC_STAGERS) {
                    const int ch = e / SAGC_T, i = e % SAGC_T, c = c0 + ch;
                    const long pos = (long)(k - 2) * SAGC_T + i;
                    if (c >= channels || pos >= n) continue;
                    const float g = tl.g[ch][i];
                    const float2 x = tl.x[ch][i];
                    out[(long)c * out_stride + pos] = make_float2(__fmul_rn(g, x.x), __fmul_rn(g, x.y));
                }
            }
            __syncthreads();
        }
    }
}

int launch_simple_agc_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, float rate, float reference,
                           float max_gain, float* d_gain_io, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (in_stride < n || out_stride < n) { set_error("simple_agc bank: row stride shorter than the row"); return -1; }
    simple_agc_bank_kernel<<<(unsigned)((channels + SAGC_CH - 1) / SAGC_CH), SAGC_WARPS * 32, 0, st>>>(d_in, in_stride, d_out, out_stride, channels, n,
                                                                                                      rate, reference, max_gain, d_gain_io);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---------------------------------------------------------------------------------------------- timing_recovery_cc
// libcsdr.c:1977-2072 as built.  Per symbol, with q = decimation/4, h = decimation/2 and the symbol starting at b:
//   stop when b + 3h >= size;  co = 0 when (double)co <= (double)(-q)*0.9 or (double)co >= (double)q*0.9
//   GARDNER:   left = b + h, mid = b + 2h, right = b + 3h, output input[left];  EARLYLATE: left = b + q - co, mid = b + h, right = b + 3q,
//              output input[mid]  (the early-late wing is (int)(decimation*0.25f) = q)
//   e = (r.i - l.i)*m.i;  use_q: e = (e + (r.q - l.q)*m.q)*0.5f     (the build multiplies by 0.5 where the source divides by 2)
//   e = max(min(e, max_error), -max_error) with minss/maxss semantics: a NaN error becomes max_error
//   co = (int)((e*loop_gain)*(float)(sign*h)), sign -1 for GARDNER;  b += decimation + co;  stop when the output count reaches size
// The launcher serves |loop_gain*max_error| <= 2: then |co| <= 2h = decimation, b never decreases and every read stays inside [b, b + 3h].
// Beyond 2 a correction can move b back, before the first sample.  Up to 1, b advances by at least h per symbol, so a call on n samples makes
// at most n/h + 1 symbols; above 1 it may stall, and only the reference's stop at n symbols bounds the count.
__global__ void __launch_bounds__(64)
timing_recovery_bank_kernel(const float2* __restrict__ in, long in_stride, const int* __restrict__ start, const int* __restrict__ size,
                            float2* __restrict__ out, long out_stride, float* __restrict__ err, int* __restrict__ idx, int channels, TrParams p,
                            TrState* __restrict__ state)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= channels) return;
    const float2* x = in + (long)c * in_stride + start[c];
    const int n = size[c];
    float2* y = out + (long)c * out_stride;
    const int bit = p.decimation, h = p.decimation / 2, q = p.decimation / 4;
    const double lo = (double)(-q) * 0.9, hi = (double)q * 0.9;
    const bool gardner = p.algorithm == 0;
    const float step = (float)(gardner ? -h : h);
    int co = state[c].last_correction_offset, b = 0, si = 0;
    for (;;) {
        if (b + 3 * h >= n) break;
        if ((double)co <= lo || (double)co >= hi) co = 0;
        int l, m, r, s;
        if (gardner) { l = b + h; m = b + 2 * h; r = b + 3 * h; s = l; }
        else { l = b + q - co; m = b + h; r = b + 3 * q; s = m; }
        const float2 xl = x[l], xm = x[m], xr = x[r];
        float e = __fmul_rn(__fsub_rn(xr.x, xl.x), xm.x);
        if (p.use_q) e = __fmul_rn(__fadd_rn(e, __fmul_rn(__fsub_rn(xr.y, xl.y), xm.y)), 0.5f);
        y[si] = x[s];
        if (idx) idx[(long)c * out_stride + si] = s;
        if (err) err[(long)c * out_stride + si] = e;
        si++;
        e = e < p.max_error ? e : p.max_error;
        e = e > -p.max_error ? e : -p.max_error;
        co = __float2int_rz(__fmul_rn(__fmul_rn(e, p.loop_gain), step));
        b += bit + co;
        if (si >= n) break;
    }
    state[c] = TrState{co, b, si};
}

int timing_recovery_max_outputs(int decimation, int input_size, float loop_gain, float max_error)
{
    return fabs((double)loop_gain) * fabs((double)max_error) <= 1.0 ? input_size / (decimation / 2) + 1 : (input_size > 1 ? input_size : 1);
}

int launch_timing_recovery_bank(const float2* d_in, long in_stride, const int* d_start, const int* d_size, float2* d_out, long out_stride, float* d_err,
                                int* d_idx, int channels, const void* h_params_v, void* d_state_v, int max_size, cudaStream_t st)
{
    if (!h_params_v) { set_error("timing_recovery bank: no parameters"); return -1; }
    const TrParams& p = *static_cast<const TrParams*>(h_params_v);
    TrState* d_state = static_cast<TrState*>(d_state_v);
    if (p.algorithm != 0 && p.algorithm != 1) { set_error("timing_recovery bank: algorithm must be GARDNER (0) or EARLYLATE (1)"); return -1; }
    if (p.decimation <= 4 || (p.decimation & 3)) { set_error("timing_recovery bank: decimation must be > 4 and divisible by 4"); return -1; }
    if (!(fabs((double)p.loop_gain) * fabs((double)p.max_error) <= 2.0)) {
        set_error("timing_recovery bank: |loop_gain * max_error| must be at most 2 (a larger correction can move a symbol back, before the input)");
        return -2;
    }
    if (channels <= 0) return 0;
    const int cap = timing_recovery_max_outputs(p.decimation, max_size, p.loop_gain, p.max_error);
    if (max_size < 0 || out_stride < cap) {
        set_error("timing_recovery bank: output rows need room for %d symbols", cap);
        return -1;
    }
    timing_recovery_bank_kernel<<<(unsigned)((channels + 63) / 64), 64, 0, st>>>(d_in, in_stride, d_start, d_size, d_out, out_stride, d_err, d_idx,
                                                                                  channels, p, d_state);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---------------------------------------------------------------------------------------------- dbpsk_decoder_c_u8
// libcsdr.c:2319-2333 as built: both phases are atan2 in double of the widened components, rounded to float; d = phase - last_phase in
// float.  The wrap loops run as the build rewrote them: d < -pi: repeat {old = d; d += 2pi} while old < -3pi; else d >= pi: repeat
// {old = d; d -= 2pi} while old >= 3pi (all float constants).  Output 0 when d > pi/2, d < -pi/2 or d is NaN (the build's comiss
// branches), else 1.
__device__ __forceinline__ float dbpsk_phase(float2 v) { return __double2float_rn(atan2((double)v.y, (double)v.x)); }

__device__ __forceinline__ unsigned char dbpsk_bit(float2 last, float2 cur)
{
    const float kPi = 3.14159274f, k2Pi = 6.28318548f, k3Pi = 9.42477798f, kHalfPi = 1.57079637f;
    float d = __fsub_rn(dbpsk_phase(cur), dbpsk_phase(last));
    if (d < -kPi) { float o; do { o = d; d = __fadd_rn(d, k2Pi); } while (o < -k3Pi); }
    else if (d >= kPi) { float o; do { o = d; d = __fsub_rn(d, k2Pi); } while (o >= k3Pi); }
    return (d > kHalfPi || !(d >= -kHalfPi)) ? 0 : 1;
}

__global__ void __launch_bounds__(256)
dbpsk_bank_kernel(const float2* __restrict__ in, long in_stride, unsigned char* __restrict__ out, long out_stride, int n, const int* __restrict__ lengths,
                  const float2* __restrict__ last_in, float2* __restrict__ last_out)
{
    const int c = blockIdx.y;
    const int len = lengths ? min(lengths[c], n) : n;
    const float2* x = in + (long)c * in_stride;
    const float2 prev0 = last_in ? last_in[c] : make_float2(0.f, 0.f);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < len; i += gridDim.x * blockDim.x) {
        out[(long)c * out_stride + i] = dbpsk_bit(i ? x[i - 1] : prev0, x[i]);
        if (last_out && i == len - 1) last_out[c] = x[i];
    }
    if (last_out && len <= 0 && blockIdx.x == 0 && threadIdx.x == 0) last_out[c] = prev0;
}

int launch_dbpsk_bank(const float2* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int n, const int* d_lengths,
                      const float2* d_last_in, float2* d_last_out, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (channels > 65535) { set_error("dbpsk bank: more than 65535 channels in one call"); return -1; }
    if (in_stride < n || out_stride < n) { set_error("dbpsk bank: row stride shorter than the row"); return -1; }
    if (d_last_in && d_last_in == d_last_out) { set_error("dbpsk bank: d_last_out must not alias d_last_in"); return -1; }
    const long blocks = (n + 255) / 256;
    dbpsk_bank_kernel<<<dim3((unsigned)(blocks < 64 ? blocks : 64), (unsigned)channels), 256, 0, st>>>(d_in, in_stride, d_out, out_stride, n, d_lengths,
                                                                                                       d_last_in, d_last_out);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---------------------------------------------------------------------------------------------- psk31_varicode_decoder
// psk31_varicode_decoder_push (libcsdr.c:1536-1549): shr = shr<<1 | (bit != 0); the character is the first table entry with
// (code << 2) == shr & (2^(bitcount+4) - 1), else 0.  Its early return tests `shr & (0xFFF == 0)`, i.e. `shr & 0`, and never fires.  The
// longest code has 10 bits, so the character at bit i is a function of bits i-13..i; bits before the call come from the carried register.
//
// The table, kVaricode, is shared with the encoder (varicode.cuh).
constexpr int kVaricodeWindow = 14;                                        // longest code (10 bits) + the two zero bits on either side

__device__ __forceinline__ unsigned char varicode_char(unsigned w)
{
    for (int k = 0; k < 128; k++) {
        const Varicode v = kVaricode[k];
        if (((unsigned)v.code << 2) == (w & ((1u << (v.bits + 4)) - 1u))) return (unsigned char)k;
    }
    return 0;
}

// one warp per channel: 32 bits per step, each lane assembles its 14-bit window and looks it up; the non-zero characters are compacted
// with a ballot and written in order.  d_hist_io[c] is the reference's status_shr (zero at stream start); d_count[c] receives the count.
constexpr int VC_WARPS = 4;

__global__ void __launch_bounds__(VC_WARPS * 32)
varicode_bank_kernel(const unsigned char* __restrict__ in, long in_stride, unsigned char* __restrict__ out, long out_stride, int channels, int n,
                     const int* __restrict__ lengths, unsigned long long* __restrict__ hist_io, int* __restrict__ count)
{
    const int lane = threadIdx.x & 31, c = blockIdx.x * VC_WARPS + (threadIdx.x >> 5);
    if (c >= channels) return;                                              // whole warps leave together
    const unsigned char* x = in + (long)c * in_stride;
    const int len = lengths ? min(lengths[c], n) : n;
    const unsigned long long h = hist_io[c];
    int cnt = 0;
    for (int i0 = 0; i0 < len; i0 += 32) {
        const int i = i0 + lane;
        unsigned char ch = 0;
        if (i < len) {
            unsigned w = 0;
            for (int k = kVaricodeWindow - 1; k >= 0; k--) {
                const int j = i - k;
                const unsigned b = j >= 0 ? (x[j] != 0) : (unsigned)((h >> (-j - 1)) & 1ull);
                w = (w << 1) | b;
            }
            ch = varicode_char(w);
        }
        const unsigned mask = __ballot_sync(0xffffffffu, ch != 0);
        if (ch) out[(long)c * out_stride + cnt + __popc(mask & ((1u << lane) - 1u))] = ch;
        cnt += __popc(mask);
    }
    if (lane == 0) {
        unsigned long long r = len >= 64 ? 0ull : h;
        for (int j = len >= 64 ? len - 64 : 0; j < len; j++) r = (r << 1) | (unsigned long long)(x[j] != 0);
        hist_io[c] = r;
        count[c] = cnt;
    }
}

int launch_varicode_bank(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int n, const int* d_lengths,
                         unsigned long long* d_hist_io, int* d_count, cudaStream_t st)
{
    if (channels <= 0) return 0;
    if (n < 0 || in_stride < n || out_stride < n) { set_error("varicode bank: row stride shorter than the row"); return -1; }
    varicode_bank_kernel<<<(unsigned)((channels + VC_WARPS - 1) / VC_WARPS), VC_WARPS * 32, 0, st>>>(d_in, in_stride, d_out, out_stride, channels, n,
                                                                                                      d_lengths, d_hist_io, d_count);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace csdrb
