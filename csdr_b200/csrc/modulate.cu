// modulate.cu -- the amplitude-side modulator blocks of a transmit graph, as bank kernels with one row per channel:
//   gain_ff            (libcsdr.c:1139-1142)  y = gain*x
//   dsb_fc [q_value]   (csdr.c:2084-2102)     y = (x, q_value), a real signal as the I of a complex one (the CLI's loop; no library function)
//   add_dcoffset_cc    (libcsdr.c:1174-1178)  y = ((i + 1)*0.5, q*0.5)
//   fixed_amplitude_cc (libcsdr.c:1194-1208)  y = x * A/|x|, or 0 where |x| is not positive
// With fmmod_fc (interpolate.cu) they make the reference's AM, DSB, SSB and FM transmit pipes: `gain_ff G | dsb_fc [| add_dcoffset_cc]`,
// `... | bandpass_fir_fft_cc`, `gain_ff G | fmmod_fc`.
//
// Arithmetic, DESIGN.md section 7 "Transmit side: AM, DSB and SSB":
//   gain_ff, dsb_fc: one rounded product, a copy.  Bit for bit the reference build.
//   add_dcoffset_cc: the source reads 0.5 + i/2 in double; the -O3 -ffast-math build runs (i + 1.0f)*0.5f and q*0.5f in float, in its scalar and
//     its SSE loop alike.  That is what the kernel computes: bit for bit the build.
//   fixed_amplitude_cc: the build has no sqrt and no division (rsqrtss plus one Newton step, a CPU-dependent seed).  The kernel computes the
//     source's expression with correctly rounded operations and no FMA: s = i*i + q*q, a = sqrt(s) (sqrtf is sqrt.rn.f32 without
//     -use_fast_math; the source's double sqrt of a float rounds to the same float), g = a > 0 ? A/a : 0, y = (i*g, q*g).  Both lie within a
//     float64 bound of A*x/|x| where s > 0 (tests/modulate/modulate.py); NaN, Inf and zeros follow the restatement, not the build's path.
// Layout: grid.y walks the rows (a row per CTA row, grid-stride over rows beyond 65535), grid.x a grid-stride loop along the row.  A row whose
// input and output both start on 16 bytes moves 128 bits per load and per store; any other row, and a row's last few elements, go one element at
// a time.  Nothing is staged.  d_in == d_out (same strides) is allowed where the element types agree: every element is read and written by
// one thread, read first.
#include "common.cuh"
#include "kernels.h"

#include <algorithm>

namespace csdrb {

constexpr int MOD_THREADS = 256;

struct GainOp {
    float gain;
    __device__ __forceinline__ float operator()(float x) const { return __fmul_rn(gain, x); }
};
struct DsbOp {
    float q;
    __device__ __forceinline__ float2 operator()(float x) const { return make_float2(x, q); }
};
struct DcOffsetOp {
    __device__ __forceinline__ float2 operator()(float2 v) const { return make_float2(__fmul_rn(__fadd_rn(v.x, 1.0f), 0.5f), __fmul_rn(v.y, 0.5f)); }
};
struct FixedAmplitudeOp {
    float amplitude;
    __device__ __forceinline__ float2 operator()(float2 v) const
    {
        const float now = sqrtf(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)));
        const float g = now > 0.f ? __fdiv_rn(amplitude, now) : 0.f;
        return make_float2(__fmul_rn(v.x, g), __fmul_rn(v.y, g));
    }
};

// y[r][i] = op(x[r][i]) for i < n.  V inputs fill one 128-bit load, and their V outputs W 128-bit stores.
template <class In, class Out, class Op>
__global__ void __launch_bounds__(MOD_THREADS)
modulate_rows_kernel(const In* in, long in_stride, Out* out, long out_stride, int channels, int n, Op op)
{
    constexpr int V = 16 / (int)sizeof(In);
    constexpr int W = V * (int)sizeof(Out) / 16;
    const int stride = gridDim.x * MOD_THREADS;
    const int t = blockIdx.x * MOD_THREADS + threadIdx.x;
    for (int r = blockIdx.y; r < channels; r += gridDim.y) {
        const In* x = in + (long)r * in_stride;
        Out* y = out + (long)r * out_stride;
        int head = 0;
        if (((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0) {
            const int nv = n / V;
            for (int v = t; v < nv; v += stride) {
                union { float4 f4; In e[V]; } a;
                union { float4 f4[W]; Out e[V]; } b;
                a.f4 = reinterpret_cast<const float4*>(x)[v];
#pragma unroll
                for (int k = 0; k < V; k++) b.e[k] = op(a.e[k]);
#pragma unroll
                for (int w = 0; w < W; w++) reinterpret_cast<float4*>(y)[(long)v * W + w] = b.f4[w];
            }
            head = nv * V;
        }
        for (int i = head + t; i < n; i += stride) y[i] = op(x[i]);
    }
}

// argument checks shared by the four banks; 0 = go ahead, 1 = nothing to do, -1 = refused (nothing launched)
static int modulate_args(const char* who, const void* d_in, long in_stride, const void* d_out, long out_stride, int channels, int n, bool same_type)
{
    if (channels < 0 || n < 0 || in_stride < n || out_stride < n) { set_error("%s bank: needs channels >= 0, n >= 0 and row strides of at least n", who); return -1; }
    if (channels == 0 || n == 0) return 1;
    if (!d_in || !d_out) { set_error("%s bank: null pointer", who); return -1; }
    if (d_in == d_out && (!same_type || (channels > 1 && in_stride != out_stride))) {
        set_error("%s bank: in place only with equal input and output types and strides", who);
        return -1;
    }
    return 0;
}

template <class In, class Out, class Op>
static int launch_modulate(const char* who, const In* d_in, long in_stride, Out* d_out, long out_stride, int channels, int n, Op op, cudaStream_t st)
{
    const int rc = modulate_args(who, d_in, in_stride, d_out, out_stride, channels, n, sizeof(In) == sizeof(Out));
    if (rc) return rc < 0 ? rc : 0;
    if ((reinterpret_cast<uintptr_t>(d_in) & (alignof(In) - 1)) || (reinterpret_cast<uintptr_t>(d_out) & (alignof(Out) - 1))) {
        set_error("%s bank: misaligned pointer (complexf needs 8-byte, float 4-byte alignment)", who);
        return -1;
    }
    // about 16 CTAs per SM over the whole bank: a row gets its share, at least one CTA, and no more than its 128-bit steps fill
    const long steps = ((long)n * (long)sizeof(In) + 15) / 16;
    const long per_row = std::max(1L, kSmCount * 16 / channels);
    const unsigned gx = (unsigned)std::min(per_row, (steps + MOD_THREADS - 1) / MOD_THREADS);
    const unsigned gy = (unsigned)std::min(channels, 65535);
    CSDRB_CUDA(launch_kernel(modulate_rows_kernel<In, Out, Op>, dim3(gx, gy), dim3(MOD_THREADS), (size_t)0, st, d_in, in_stride, d_out, out_stride,
                             channels, n, op));
    return 1;
}

int launch_gain_bank_ff(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, float gain, cudaStream_t st)
{
    return launch_modulate("gain_ff", d_in, in_stride, d_out, out_stride, channels, n, GainOp{gain}, st);
}

int launch_dsb_bank_fc(const float* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, float q_value, cudaStream_t st)
{
    return launch_modulate("dsb_fc", d_in, in_stride, d_out, out_stride, channels, n, DsbOp{q_value}, st);
}

int launch_add_dcoffset_bank_cc(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, cudaStream_t st)
{
    return launch_modulate("add_dcoffset_cc", d_in, in_stride, d_out, out_stride, channels, n, DcOffsetOp{}, st);
}

int launch_fixed_amplitude_bank_cc(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, float amplitude,
                                   cudaStream_t st)
{
    return launch_modulate("fixed_amplitude_cc", d_in, in_stride, d_out, out_stride, channels, n, FixedAmplitudeOp{amplitude}, st);
}

}  // namespace csdrb
