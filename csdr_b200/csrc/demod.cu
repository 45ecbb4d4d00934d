// demod.cu -- two demodulators of libcsdr as bank kernels, one row per channel:
//   fmdemod_atan_cf      (libcsdr.c:1004-1019)  y[i] = wrap(arg x[i] - arg x[i-1]) / pi, the phase difference itself
//   amdemod_estimator_cf (libcsdr.c:875-901)    y[i] = alpha*max(|I|,|Q|) + beta*min(|I|,|Q|)
// (dcblock_ff is the recursion kernel of audio.cu; fmdemod_quadri_novect_cf is K4 of elementwise.cu without its den != 0 guard.)
//
// Arithmetic, DESIGN.md section 7 "Phase-difference FM and the magnitude estimator":
//   atan: phase = (float)atan2((double)Q, (double)I), the reference's double atan2 rounded to float; d = phase - last in float, d += 2*PI where
//     d < -PI, else d -= 2*PI where d > PI (PI = (float)pi); y = d * 0x1.45f306p-2f, the float reciprocal of PI that the -ffast-math build
//     multiplies by.  No FMA.  CUDA's double atan2 is within 2 ulp (double), so the float phase can differ from glibc's where the double value
//     lies that close to a float rounding midpoint (about 1e-8 of samples); elsewhere the bits are the build's.
//   estimator: |I|, |Q| and the max/min selections are the build's comparisons, not fmaxf/fminf: maxss/minss (maxps/minps) return their second
//     operand when either is NaN, and the build orders the operands differently in its loops.  Calls of 2 samples or more run the SSE loops
//     (4 and 2 wide, and a last single sample), max(|I|,|Q|) and min(|I|,|Q|) with |Q| second: a NaN takes |Q|.  A call of one sample runs
//     the scalar loop, the source's selections with |I| second: a NaN takes |I|.  alpha == 0 selects the reference's defaults for alpha and beta.  Two rounded products and
//     a rounded sum, no FMA.
#include "common.cuh"
#include "kernels.h"

#include <algorithm>

namespace csdrb {

constexpr int ATAN_THREADS = 256, ATAN_PER_THREAD = 4, ATAN_TILE = ATAN_THREADS * ATAN_PER_THREAD;
constexpr float kPi = (float)3.14159265358979323846;
constexpr float kInvPi = 0x1.45f306p-2f;

__device__ __forceinline__ float phase_of(float2 v) { return (float)atan2((double)v.y, (double)v.x); }

__device__ __forceinline__ float atan_step(float phase, float last)
{
    float d = __fsub_rn(phase, last);
    if (d < -kPi) d = __fadd_rn(d, 2.f * kPi);
    else if (d > kPi) d = __fsub_rn(d, 2.f * kPi);
    return __fmul_rn(d, kInvPi);
}

// A CTA walks tiles of ATAN_TILE samples of one row; each thread owns ATAN_PER_THREAD consecutive samples and computes each of their phases
// once.  The phase before a thread's first sample is its left neighbour's last (a shuffle, across warps through shared memory); thread 0 takes
// one extra atan2 of the sample before the tile, or the carried phase at the row's start.
__global__ void __launch_bounds__(ATAN_THREADS)
fmdemod_atan_bank_kernel(const float2* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride, int n,
                         const float* __restrict__ last_in, float* __restrict__ last_out)
{
    __shared__ float warp_last[ATAN_THREADS / 32];
    const int ch = blockIdx.y;
    const float2* x = in + (long)ch * in_stride;
    float* y = out + (long)ch * out_stride;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
    for (long t0 = (long)blockIdx.x * ATAN_TILE; t0 < n; t0 += (long)gridDim.x * ATAN_TILE) {
        const long i0 = t0 + (long)threadIdx.x * ATAN_PER_THREAD;
        float ph[ATAN_PER_THREAD];
        if (vec && i0 + ATAN_PER_THREAD <= n) {
            const float4 a = reinterpret_cast<const float4*>(x + i0)[0], b = reinterpret_cast<const float4*>(x + i0)[1];
            ph[0] = phase_of(make_float2(a.x, a.y)); ph[1] = phase_of(make_float2(a.z, a.w));
            ph[2] = phase_of(make_float2(b.x, b.y)); ph[3] = phase_of(make_float2(b.z, b.w));
        } else {
#pragma unroll
            for (int k = 0; k < ATAN_PER_THREAD; k++) ph[k] = i0 + k < n ? phase_of(x[i0 + k]) : 0.f;
        }
        float before = __shfl_sync(0xffffffffu, ph[ATAN_PER_THREAD - 1], (lane + 31) & 31);   // lane 0's is replaced below
        if (lane == 31) warp_last[warp] = ph[ATAN_PER_THREAD - 1];
        __syncthreads();
        if (lane == 0) before = warp ? warp_last[warp - 1] : t0 ? phase_of(x[t0 - 1]) : last_in ? last_in[ch] : 0.f;
        __syncthreads();                                                  // warp_last is rewritten by the next tile
        float o[ATAN_PER_THREAD];
#pragma unroll
        for (int k = 0; k < ATAN_PER_THREAD; k++) { o[k] = atan_step(ph[k], before); before = ph[k]; }
        if (vec && i0 + ATAN_PER_THREAD <= n) reinterpret_cast<float4*>(y + i0)[0] = make_float4(o[0], o[1], o[2], o[3]);
        else {
#pragma unroll
            for (int k = 0; k < ATAN_PER_THREAD; k++) if (i0 + k < n) y[i0 + k] = o[k];
        }
        if (last_out) {
#pragma unroll
            for (int k = 0; k < ATAN_PER_THREAD; k++) if (i0 + k == n - 1) last_out[ch] = ph[k];
        }
    }
}

int launch_fmdemod_atan_bank(const float2* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, const float* d_last_in,
                             float* d_last_out, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (d_last_in && d_last_out == d_last_in) { set_error("fmdemod_atan bank: last_phase_in and last_phase_out must not alias"); return -1; }
    // about 16 CTAs per SM over the whole bank, at least one per row, no more than the row has tiles
    const long tiles = ((long)n + ATAN_TILE - 1) / ATAN_TILE;
    const unsigned gx = (unsigned)std::min(std::max(1L, kSmCount * 16 / channels), tiles);
    CSDRB_CUDA(launch_kernel(fmdemod_atan_bank_kernel, dim3(gx, channels), dim3(ATAN_THREADS), (size_t)0, st, d_in, in_stride, d_out, out_stride, n,
                             d_last_in, d_last_out));
    return 1;
}

// ---- amdemod_estimator_cf ---------------------------------------------------------------------------------------------------------------
constexpr int EST_THREADS = 256;

// sse: the selections of the build's SSE loops (a NaN takes |Q|), else of its scalar loop (a NaN takes |I|)
__device__ __forceinline__ float estimate(float2 v, float alpha, float beta, bool sse)
{
    const float ai = fabsf(v.x), aq = fabsf(v.y);
    const float mx = sse ? (ai > aq ? ai : aq) : (aq > ai ? aq : ai);
    const float mn = sse ? (ai < aq ? ai : aq) : (aq < ai ? aq : ai);
    return __fadd_rn(__fmul_rn(alpha, mx), __fmul_rn(beta, mn));
}

// two samples per thread per step (one 128-bit load, one 64-bit store) where the row allows it, one at a time otherwise
__global__ void __launch_bounds__(EST_THREADS)
amdemod_estimator_bank_kernel(const float2* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride, int channels, int n,
                              float alpha, float beta)
{
    const int stride = gridDim.x * EST_THREADS;
    const int t = blockIdx.x * EST_THREADS + threadIdx.x;
    const bool sse = n >= 2;
    for (int r = blockIdx.y; r < channels; r += gridDim.y) {
        const float2* x = in + (long)r * in_stride;
        float* y = out + (long)r * out_stride;
        int head = 0;
        if ((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 7) == 0) {
            const int np = n / 2;
            for (int v = t; v < np; v += stride) {
                const float4 q = reinterpret_cast<const float4*>(x)[v];
                reinterpret_cast<float2*>(y)[v] = make_float2(estimate(make_float2(q.x, q.y), alpha, beta, sse),
                                                              estimate(make_float2(q.z, q.w), alpha, beta, sse));
            }
            head = np * 2;
        }
        for (int i = head + t; i < n; i += stride) y[i] = estimate(x[i], alpha, beta, sse);
    }
}

int launch_amdemod_estimator_bank(const float2* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, float alpha, float beta,
                                  cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (alpha == 0.f) { alpha = 0.947543636291f; beta = 0.392485425092f; }   // libcsdr.c:881-885
    const long per_row = std::max(1L, kSmCount * 16 / channels);
    const unsigned gx = (unsigned)std::min(per_row, ((long)n / 2 + EST_THREADS) / EST_THREADS);
    const unsigned gy = (unsigned)std::min(channels, 65535);
    CSDRB_CUDA(launch_kernel(amdemod_estimator_bank_kernel, dim3(gx, gy), dim3(EST_THREADS), (size_t)0, st, d_in, in_stride, d_out, out_stride, channels,
                             n, alpha, beta));
    return 1;
}

}  // namespace csdrb
