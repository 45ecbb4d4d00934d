// interpolate.cu -- the two building blocks of a transmit graph, as bank kernels with one row per channel:
//   fir_interpolate_cc (libcsdr.c:579-602)   raise the rate by an integer factor I with a polyphase FIR
//   fmmod_fc           (libcsdr.c:1180-1192) the FM modulator: a float phase advanced by x*PI per sample, out (cos, sin)
//
// fir_interpolate_cc, the reference's arithmetic and framing, quirks included:
//   output i*I + ip  (ip = 0 .. I-1)  =  sum over si of x[i + si] * taps[ti],  ti = (I - ip) + si*I < T
//   The start index is I - ip without a "% I", so phase 0 starts at tap I and tap 0 is never used.  I and Q are summed separately, in tap order,
//   each product and sum rounded on its own (no FMA): the kernel's sum is bit for bit the source order, and within a float64 per-output bound of the
//   reference build, which may reorder under -ffast-math (tests/tx/tx.py).  A call stops at the first i with i*I + (I-1) + T > n*I, so a
//   row of n inputs gives G = n - ceil((T-1)/I) groups of I outputs (none when n is smaller), and the caller keeps n - G inputs for the next call.
// Layout: a CTA covers INTERP_TILE consecutive outputs of one row, one thread per output in turn, so that stores are coalesced whatever I is.  The taps
// are staged in shared memory when they fit (T <= INTERP_SMEM_TAPS); longer filters are read through the read-only cache.  Inputs are read through
// the read-only cache too: the I outputs of a group read the same few inputs, and neighbouring groups overlap by all but one.
//
// fmmod_fc: phase += x*PI (PI the float of libcsdr.h:65, the product rounded, then the sum); while (phase > PI) phase -= 2*PI; while (phase <= -PI)
// phase += 2*PI; out = (cos phase, sin phase).  The chain is serial and data dependent: one warp per channel walks it 32 samples at a time, every
// lane the same steps (the samples come by shuffle) and lane k keeps the phase of step k, so the warp then evaluates 32 cos/sin pairs in parallel
// and stores them coalesced.  The phase sequence is the reference build's bit for bit; how cos and sin are evaluated is in DESIGN.md section 7.
#include "common.cuh"
#include "kernels.h"

namespace csdrb {

constexpr int INTERP_THREADS = 256;
constexpr int INTERP_TILE = 2048;                            // outputs per CTA
constexpr int INTERP_SMEM_TAPS = 8192;                       // 32 KB of taps in shared memory; beyond, the read-only cache

template <bool SMEM_TAPS>
__global__ void __launch_bounds__(INTERP_THREADS)
fir_interpolate_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride, long nout, int I,
                       const float* __restrict__ taps, int T)
{
    CSDRB_DYN_SMEM(smem);
    const float* tp = taps;
    if constexpr (SMEM_TAPS) {
        float* s_taps = reinterpret_cast<float*>(smem);
        for (int k = threadIdx.x; k < T; k += INTERP_THREADS) s_taps[k] = taps[k];
        __syncthreads();
        tp = s_taps;
    }
    const float2* x = in + (long)blockIdx.y * in_stride;
    float2* y = out + (long)blockIdx.y * out_stride;
    const long o_end = min(nout, (long)(blockIdx.x + 1) * INTERP_TILE);
    for (long o = (long)blockIdx.x * INTERP_TILE + threadIdx.x; o < o_end; o += INTERP_THREADS) {
        const long i = o / I;
        const int ip = (int)(o - i * I);
        float acci = 0.f, accq = 0.f;
        const float2* xi = x + i;
        int si = 0;
        for (int ti = I - ip; ti < T; ti += I, si++) {
            const float t = SMEM_TAPS ? tp[ti] : __ldg(tp + ti);
            const float2 v = __ldg(xi + si);
            acci = __fadd_rn(acci, __fmul_rn(v.x, t));
            accq = __fadd_rn(accq, __fmul_rn(v.y, t));
        }
        y[o] = make_float2(acci, accq);
    }
}

int launch_fir_interpolate_bank_cc(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, int interpolation,
                                   const float* d_taps, int taps_length, cudaStream_t st)
{
    if (interpolation < 1 || taps_length < 1 || channels < 0 || n < 0) {
        set_error("fir_interpolate bank: needs interpolation >= 1, taps_length >= 1, channels >= 0 and n >= 0");
        return -1;
    }
    const long groups = interp_groups(n, interpolation, taps_length);
    const long nout = groups * interpolation;
    if (in_stride < n || out_stride < nout) { set_error("fir_interpolate bank: row strides below n inputs or the row's outputs"); return -1; }
    if (nout > 0x7fffffffL) { set_error("fir_interpolate bank: more than 2^31 - 1 outputs per row"); return -1; }
    if (channels == 0 || nout == 0) return (int)nout;
    const dim3 grid((unsigned)((nout + INTERP_TILE - 1) / INTERP_TILE), (unsigned)channels);
    if (taps_length <= INTERP_SMEM_TAPS)
        CSDRB_CUDA(launch_kernel(fir_interpolate_kernel<true>, grid, dim3(INTERP_THREADS), (size_t)taps_length * sizeof(float), st,
                                 d_in, in_stride, d_out, out_stride, nout, interpolation, d_taps, taps_length));
    else
        CSDRB_CUDA(launch_kernel(fir_interpolate_kernel<false>, grid, dim3(INTERP_THREADS), (size_t)0, st,
                                 d_in, in_stride, d_out, out_stride, nout, interpolation, d_taps, taps_length));
    return (int)nout;
}

// ---- fmmod_fc ---------------------------------------------------------------------------------------------------------------------------
// One step of the phase chain as the reference build runs it (its disassembly, DESIGN.md section 7): -ffast-math turns each wrap loop into a
// do-while that tests the value BEFORE the step against 3*PI (the float 9.424778), and the second loop is reached only when the first is not
// entered.  The loops are linear: a phase of magnitude P takes about P / 2*PI rounded steps (unscaled s16-range audio, x ~ 3e4, costs some 1e4
// per sample), as in the reference.  Below 2^27 every step still moves the phase (half the float spacing there is at most 4, less than 2*PI) and
// the loop ends as the reference's does; from 2^27 on a step of 2*PI rounds to no change and the reference never returns (at +-Inf neither).
// Such a phase is left as it is here.
constexpr float kThreePiF = 9.42477798461914062f;             // fl(3 * PI), the build's constant

__device__ __forceinline__ float fmmod_step(float ph, float x)
{
    ph = __fadd_rn(ph, __fmul_rn(x, kPiF));
    if (!(fabsf(ph) < 134217728.f)) return ph;
    float old;
    if (ph > kPiF) {
        do { old = ph; ph = __fsub_rn(ph, kTwoPiF); } while (old > kThreePiF);
    } else if (ph <= -kPiF) {
        do { old = ph; ph = __fadd_rn(ph, kTwoPiF); } while (old <= -kThreePiF);
    }
    return ph;
}

constexpr int FMMOD_WARPS = 4;

__global__ void __launch_bounds__(32 * FMMOD_WARPS)
fmmod_bank_kernel(const float* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride, int channels, int n,
                  float* __restrict__ phase_io)
{
    const int c = blockIdx.x * FMMOD_WARPS + (threadIdx.x >> 5);
    if (c >= channels) return;
    const int lane = threadIdx.x & 31;
    const float* x = in + (long)c * in_stride;
    float2* y = out + (long)c * out_stride;
    float ph = phase_io[c];
    __syncwarp();                                            // every lane has read the carried phase before lane 0 overwrites it
    for (int b = 0; b < n; b += 32) {
        const int m = min(32, n - b);
        const float v = lane < m ? x[b + lane] : 0.f;
        float mine = 0.f;
        for (int k = 0; k < m; k++) {                        // every lane walks the same steps; lane k keeps step k
            ph = fmmod_step(ph, __shfl_sync(0xffffffffu, v, k));
            if (k == lane) mine = ph;
        }
        if (lane < m) y[b + lane] = make_float2((float)cos((double)mine), (float)sin((double)mine));
    }
    if (lane == 0) phase_io[c] = ph;
}

int launch_fmmod_bank_fc(const float* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, float* d_phase_io, cudaStream_t st)
{
    if (channels < 0 || n < 0 || in_stride < n || out_stride < n) { set_error("fmmod bank: needs n >= 0 and row strides of at least n"); return -1; }
    if (channels == 0 || n == 0) return n;
    CSDRB_CUDA(launch_kernel(fmmod_bank_kernel, dim3((unsigned)((channels + FMMOD_WARPS - 1) / FMMOD_WARPS)), dim3(32 * FMMOD_WARPS), (size_t)0, st,
                             d_in, in_stride, d_out, out_stride, channels, n, d_phase_io));
    return n;
}

}  // namespace csdrb
