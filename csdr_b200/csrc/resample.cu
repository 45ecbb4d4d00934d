// resample.cu -- rational_resampler_ff (libcsdr.c:607-636; state struct libcsdr.h:132-137) as a bank of float rows.
//
// The reference computes output oi from the closed-form index pair
//     startingi = (oi*D + I-1-ltd) / I,   delayi = (ltd + startingi*I - oi*D) % I
//     out[oi]   = I * sum_{i < (T-delayi)/I} in[startingi+i] * taps[delayi + i*I]
// and stops at the first output whose filter would run past the input (startingi + T/I + 1 > n) or at the output cap n*I/D.
// Nothing is carried from one output to the next, so the bank is fully parallel: one CTA covers a tile of consecutive outputs of one
// channel, stages the taps and the tile's input span in shared memory with coalesced loads, and every thread sums its outputs in the
// reference's order (i ascending, one accumulator, separately rounded products) -- bit for bit the sequential C loop.
// All channels run in lockstep (one shared last_taps_delay), so the state the call returns is a pure integer function of
// (n, I, D, T, ltd): rational_resampler_state() evaluates it on the host and the bank call never waits for the device.
#include "common.cuh"
#include "kernels.h"

#include <climits>

namespace csdrb {

constexpr int kRsThreads = 256;
constexpr long kRsMaxTile = 1024;                                  // outputs per CTA at most
constexpr long kRsSmemBudget = 200L * 1024;                        // taps + input span of one CTA (H100: 227 KB per block)

__device__ __forceinline__ long rs_starting(long oi, int I, int D, int ltd) { return (oi * D + I - 1 - ltd) / I; }

__global__ void __launch_bounds__(kRsThreads)
rational_resampler_kernel(const float* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride, long n_out, int I, int D,
                          const float* __restrict__ taps, int T, int taps_pad, int ltd, long tile)
{
    CSDRB_DYN_SMEM(smem);
    float* s_taps = reinterpret_cast<float*>(smem);
    float* s_in = s_taps + taps_pad;
    const long o0 = (long)blockIdx.x * tile;
    const long cnt = min(tile, n_out - o0);
    const long s0 = rs_starting(o0, I, D, ltd);
    // every output of the tile reads in[startingi .. startingi + T/I - 1], inside the row because startingi + T/I + 1 <= n
    const long span = rs_starting(o0 + cnt - 1, I, D, ltd) + T / I - s0;
    const float* row = in + (long)blockIdx.y * in_stride + s0;
    for (int t = threadIdx.x; t < T; t += kRsThreads) s_taps[t] = __ldg(taps + t);
    for (long j = threadIdx.x; j < span; j += kRsThreads) s_in[j] = __ldg(row + j);
    __syncthreads();
    float* orow = out + (long)blockIdx.y * out_stride;
    for (long k = threadIdx.x; k < cnt; k += kRsThreads) {
        const long oi = o0 + k;
        const long s = rs_starting(oi, I, D, ltd);
        const int delay = (int)((ltd + s * I - oi * D) % I);
        const int terms = (T - delay) / I;
        const float* x = s_in + (s - s0);
        const float* h = s_taps + delay;
        float acc = 0.f;
        for (int i = 0; i < terms; i++) acc = __fadd_rn(acc, __fmul_rn(x[i], h[i * I]));
        orow[oi] = __fmul_rn(acc, (float)I);
    }
}

// The reference loop's exit state without running it.  Output oi is computable while startingi(oi) <= L = n - T/I - 1, i.e. for
// oi <= (L*I + ltd) / D.  If the input runs out first the loop breaks at the first output it cannot compute and returns that output's
// pair; if the cap n*I/D ends it, the pair is the last output produced (the next call computes that output again).  With no output at
// all the reference returns uninitialised fields; here they are {0, 0, ltd}, what the first iteration would give.
int rational_resampler_state(int input_size, int interpolation, int decimation, int taps_length, int last_taps_delay, int* h_state)
{
    const long I = interpolation, D = decimation, ltd = last_taps_delay;
    const long cap = (long)input_size * I / D;
    const long L = (long)input_size - taps_length / interpolation - 1;
    const long fit = L >= 0 ? (L * I + ltd) / D + 1 : 0;
    if (cap <= 0) { h_state[0] = 0; h_state[1] = 0; h_state[2] = last_taps_delay; return 0; }
    const long produced = fit < cap ? fit : cap;
    const long k = fit < cap ? fit : cap - 1;
    const long s = (k * D + I - 1 - ltd) / I;
    h_state[0] = (int)s;
    h_state[1] = (int)produced;
    h_state[2] = (int)((ltd + s * I - k * D) % I);
    return (int)produced;
}

// outputs per channel (>= 0), -1 for invalid arguments, -2 for a geometry the bank does not serve
int launch_rational_resampler_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int input_size,
                                   int interpolation, int decimation, const float* h_taps, int taps_length, int last_taps_delay,
                                   int* h_state, cudaStream_t st)
{
    const int I = interpolation, D = decimation, T = taps_length;
    if (I <= 0 || D <= 0) { set_error("rational_resampler: interpolation and decimation must be positive"); return -1; }
    if (!h_taps || T <= 0) { set_error("rational_resampler: no taps"); return -1; }
    if (last_taps_delay < 0 || last_taps_delay >= I) { set_error("rational_resampler: last_taps_delay %d outside 0..%d", last_taps_delay, I - 1); return -1; }
    if (input_size < 0 || channels < 0) { set_error("rational_resampler: negative size"); return -1; }
    if ((long)input_size * I > INT_MAX) {
        set_error("rational_resampler: input_size * interpolation = %ld exceeds INT_MAX (the reference's int index arithmetic overflows)", (long)input_size * I);
        return -2;
    }
    if (T > kRsMaxTaps) { set_error("rational_resampler: %d taps (at most %d fit the shared-memory tile)", T, kRsMaxTaps); return -2; }
    const int taps_pad = (T + 3) & ~3;
    // the input span of `tile` outputs is at most ceil((tile-1)*D/I) + T/I samples; with T <= kRsMaxTaps one output always fits (room > 0)
    const long room = kRsSmemBudget / 4 - taps_pad - T / I - 1;
    long tile = room * I / D + 1;
    if (tile > kRsMaxTile) tile = kRsMaxTile;
    const int n_out = rational_resampler_state(input_size, I, D, T, last_taps_delay, h_state);
    if (channels == 0 || n_out == 0) return n_out;                  // zero channels: geometry check and state only
    if (!d_in || !d_out) { set_error("rational_resampler: null pointer"); return -1; }
    const long span_cap = ((tile - 1) * D + I - 1) / I + T / I + 1;
    const size_t smem = sizeof(float) * (size_t)(taps_pad + span_cap);
    float* d_taps = nullptr;                                            // stream-ordered copy of the host taps: the call never blocks
    CSDRB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&d_taps), sizeof(float) * (size_t)T, st));
    CSDRB_CUDA(cudaMemcpyAsync(d_taps, h_taps, sizeof(float) * (size_t)T, cudaMemcpyHostToDevice, st));
    const dim3 grid((unsigned)((n_out + tile - 1) / tile), (unsigned)channels);
    CSDRB_CUDA(launch_kernel(rational_resampler_kernel, grid, kRsThreads, smem, st, d_in, in_stride, d_out, out_stride, n_out, I, D, d_taps, T, taps_pad,
                             last_taps_delay, tile));
    CSDRB_CUDA(cudaFreeAsync(d_taps, st));
    return n_out;
}

}  // namespace csdrb
