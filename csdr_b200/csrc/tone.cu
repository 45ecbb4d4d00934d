// tone.cu -- the complex-tap FIR of the reference's tone filters, as one bank kernel family, one row per channel:
//   apply_fir_cc    (libcsdr.c:2261-2273)  one complex tap set -> complexf; peaks_fir_cc runs it
//   bfsk_demod_cf   (libcsdr.c:2335-2351)  a mark and a space tap set -> float -(|space|^2) + |mark|^2
// Row c gives the n - L + 1 outputs of the valid convolution of its n inputs; the caller carries the last L - 1 inputs between calls.
//
// Arithmetic (DESIGN.md section 7), every operation an explicit _rn intrinsic so that nothing is contracted into an FMA:
//   apply_fir_cc follows the reference's -O3 -ffast-math build, which keeps `ti` ascending and one accumulator but reassociates the real
//     part of cmultadd: re = (x.i*t.i + re) - x.q*t.q, im = im + (x.i*t.q + t.i*x.q).  Bit-exact with the library.
//   bfsk_demod_cf is vectorised by that build (four partial sums per accumulator, reduced in a tree, a tail in pairs), an order a
//     one-output-per-chain kernel cannot follow.  The kernel sums in source order instead: `ti` ascending, re += x.i*t.i - x.q*t.q,
//     im += x.i*t.q + t.i*x.q, then -(s.i*s.i + s.q*s.q) + (m.i*m.i + m.q*m.q).  Bit-exact with a strict-IEEE restatement, and within
//     the per-output bound of tests/test_tone_emulated.py of the library.
//
// Layout: a CTA computes TONE_TILE consecutive outputs of one row.  Its taps (both sets interleaved for bfsk) and its input tile with the
// L - 1 halo are staged in shared memory.  Thread k computes outputs k*R .. k*R + R - 1 and keeps the R inputs they read at tap ti in
// registers: one new input per tap, input m in register m mod R, so the rotation is resolved at compile time.  R is odd: the 64-bit
// loads of a half-warp then stride an odd number of complex samples and hit 16 distinct bank pairs.
#include "common.cuh"
#include "kernels.h"

namespace csdrb {

constexpr int TONE_THREADS = 128;
constexpr int TONE_R = 7;
constexpr int TONE_TILE = TONE_THREADS * TONE_R;

struct ToneApply {                                            // apply_fir_cc: complexf out
    using Tap = float2;
    using Acc = float2;
    using Out = float2;
    static __device__ __forceinline__ Tap load_tap(const float2* a, const float2*, int k) { return a[k]; }
    static __device__ __forceinline__ Acc zero() { return make_float2(0.f, 0.f); }
    static __device__ __forceinline__ void mac(Acc& acc, float2 x, Tap t)
    {
        acc.x = __fsub_rn(__fadd_rn(__fmul_rn(x.x, t.x), acc.x), __fmul_rn(x.y, t.y));
        acc.y = __fadd_rn(acc.y, __fadd_rn(__fmul_rn(x.x, t.y), __fmul_rn(t.x, x.y)));
    }
    static __device__ __forceinline__ Out finish(Acc a) { return a; }
};

struct ToneBfsk {                                             // bfsk_demod_cf: float out; the tap is (mark.i, mark.q, space.i, space.q)
    using Tap = float4;
    using Acc = float4;
    using Out = float;
    static __device__ __forceinline__ Tap load_tap(const float2* mark, const float2* space, int k)
    {
        const float2 m = mark[k], s = space[k];
        return make_float4(m.x, m.y, s.x, s.y);
    }
    static __device__ __forceinline__ Acc zero() { return make_float4(0.f, 0.f, 0.f, 0.f); }
    static __device__ __forceinline__ void mac(Acc& acc, float2 x, Tap t)
    {
        acc.x = __fadd_rn(acc.x, __fsub_rn(__fmul_rn(x.x, t.x), __fmul_rn(x.y, t.y)));
        acc.y = __fadd_rn(acc.y, __fadd_rn(__fmul_rn(x.x, t.y), __fmul_rn(t.x, x.y)));
        acc.z = __fadd_rn(acc.z, __fsub_rn(__fmul_rn(x.x, t.z), __fmul_rn(x.y, t.w)));
        acc.w = __fadd_rn(acc.w, __fadd_rn(__fmul_rn(x.x, t.w), __fmul_rn(t.z, x.y)));
    }
    static __device__ __forceinline__ Out finish(Acc a)
    {
        const float space = __fadd_rn(__fmul_rn(a.z, a.z), __fmul_rn(a.w, a.w)), mark = __fadd_rn(__fmul_rn(a.x, a.x), __fmul_rn(a.y, a.y));
        return __fadd_rn(-space, mark);
    }
};

template <class E>
__global__ void __launch_bounds__(TONE_THREADS)
tone_fir_kernel(const float2* __restrict__ in, long in_stride, typename E::Out* __restrict__ out, long out_stride, int n,
                const float2* __restrict__ ta, const float2* __restrict__ tb, int L)
{
    using Tap = typename E::Tap;
    CSDRB_DYN_SMEM(smem);
    Tap* s_taps = reinterpret_cast<Tap*>(smem);
    float2* s_x = reinterpret_cast<float2*>(smem + (size_t)L * sizeof(Tap));
    const int nout = n - L + 1;
    const long o0 = (long)blockIdx.x * TONE_TILE;
    const float2* row = in + (long)blockIdx.y * in_stride;
    const int span = TONE_TILE + L - 1 + TONE_R;              // the tile, its halo, and the R inputs the last tap step loads ahead
    for (int k = threadIdx.x; k < L; k += TONE_THREADS) s_taps[k] = E::load_tap(ta, tb, k);
    for (int k = threadIdx.x; k < span; k += TONE_THREADS) s_x[k] = o0 + k < n ? row[o0 + k] : make_float2(0.f, 0.f);
    __syncthreads();

    const int b = threadIdx.x * TONE_R;                        // this thread's first output in the tile
    if (o0 + b >= nout) return;                                // no barrier follows
    float2 w[TONE_R];                                          // input b + m sits in w[m mod R]
#pragma unroll
    for (int r = 0; r < TONE_R; r++) w[r] = s_x[b + r];
    typename E::Acc acc[TONE_R];
#pragma unroll
    for (int r = 0; r < TONE_R; r++) acc[r] = E::zero();
    int t0 = 0;
    for (; t0 + TONE_R <= L; t0 += TONE_R) {
#pragma unroll
        for (int j = 0; j < TONE_R; j++) {
            const Tap t = s_taps[t0 + j];
#pragma unroll
            for (int r = 0; r < TONE_R; r++) E::mac(acc[r], w[(r + j) % TONE_R], t);
            w[j] = s_x[b + t0 + j + TONE_R];                   // input b + t0 + j is read by no later tap; b + t0 + j + R takes its register
        }
    }
#pragma unroll
    for (int j = 0; j < TONE_R; j++) {
        if (t0 + j < L) {
            const Tap t = s_taps[t0 + j];
#pragma unroll
            for (int r = 0; r < TONE_R; r++) E::mac(acc[r], w[(r + j) % TONE_R], t);
            w[j] = s_x[b + t0 + j + TONE_R];
        }
    }
    typename E::Out* o = out + (long)blockIdx.y * out_stride;
#pragma unroll
    for (int r = 0; r < TONE_R; r++)
        if (o0 + b + r < nout) o[o0 + b + r] = E::finish(acc[r]);
}

template <class E>
static int launch_tone(const float2* d_in, long in_stride, typename E::Out* d_out, long out_stride, int channels, int n, const float2* ta,
                       const float2* tb, int L, const char* who, cudaStream_t st)
{
    if (L < 2 || L > kToneMaxTaps) { set_error("%s: %d taps (2..%d are served)", who, L, kToneMaxTaps); return -2; }
    if (channels < 0 || n < L || in_stride < n || out_stride < n - L + 1) {
        set_error("%s: needs n >= taps_length and row strides of at least n inputs and n - taps_length + 1 outputs", who);
        return -1;
    }
    const int nout = n - L + 1;
    if (channels == 0) return nout;
    const size_t smem = (size_t)L * sizeof(typename E::Tap) + (size_t)(TONE_TILE + L - 1 + TONE_R) * sizeof(float2);
    const dim3 grid((unsigned)((nout + TONE_TILE - 1) / TONE_TILE), (unsigned)channels);
    CSDRB_CUDA(launch_kernel(tone_fir_kernel<E>, grid, dim3(TONE_THREADS), smem, st, d_in, in_stride, d_out, out_stride, n, ta, tb, L));
    return nout;
}

int launch_apply_fir_bank_cc(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, const float2* d_taps, int L,
                             cudaStream_t st)
{
    return launch_tone<ToneApply>(d_in, in_stride, d_out, out_stride, channels, n, d_taps, nullptr, L, "apply_fir_cc bank", st);
}

int launch_bfsk_demod_bank_cf(const float2* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, const float2* d_mark,
                              const float2* d_space, int L, cudaStream_t st)
{
    return launch_tone<ToneBfsk>(d_in, in_stride, d_out, out_stride, channels, n, d_mark, d_space, L, "bfsk_demod_cf bank", st);
}

}  // namespace csdrb
