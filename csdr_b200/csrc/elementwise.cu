// elementwise.cu -- K1 sample-format conversions and K4 fmdemod_quadri_cf.
//
// K1 replaces convert_u8_f / convert_s16_f / convert_f_s16 (libcsdr.c:2363-2366, 2373-2376, 2390-2398), and the other sample formats
// convert_s8_f / convert_f_s8 / convert_f_u8 / convert_s24_f / convert_f_s24 (libcsdr.c:2368-2437).
// K4 replaces fmdemod_quadri_cf (libcsdr.c:1040-1071) for C channels per launch.
// All are pure streaming kernels: 128-bit global accesses, grid-stride, nothing staged.
#include "common.cuh"
#include "kernels.h"

namespace csdrb {

// u8 -> f32.  The reference computes ((float)b)/(UCHAR_MAX/2.0) - 1.0 in double and rounds once.  For the 256 possible
// inputs that equals the correctly rounded float quotient (2b - 255)/255 (both operands exact in fp32, one IEEE division);
// identical for every code -- pinned by tests/test_gpu_parity.py::test_convert_u8_f_bit_exact against oracle and golden table.
__device__ __forceinline__ float u8_to_f(unsigned b) { return __fdiv_rn((float)(2 * (int)b - 255), 255.0f); }

// Access pattern of the widening conversions: a lane takes ONE 32-bit input word per step and writes ONE 128-bit output, so a
// warp reads 128 contiguous bytes and writes 512 contiguous bytes per instruction (fully coalesced on both sides); four steps
// are in flight per thread for memory-level parallelism.
__global__ void __launch_bounds__(256) convert_u8_f_kernel(const unsigned char* __restrict__ in, float* __restrict__ out, long n)
{
    const long nw = n / 4;                                             // whole 4-byte words
    const long stride = (long)gridDim.x * blockDim.x;
    long v = (long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; v + 3 * stride < nw; v += 4 * stride) {
        unsigned w[4];
#pragma unroll
        for (int u = 0; u < 4; u++) w[u] = __ldg(reinterpret_cast<const unsigned*>(in) + v + u * stride);
#pragma unroll
        for (int u = 0; u < 4; u++)
            st_na_f4(reinterpret_cast<float4*>(out) + v + u * stride,
                     make_float4(u8_to_f(w[u] & 255u), u8_to_f((w[u] >> 8) & 255u), u8_to_f((w[u] >> 16) & 255u), u8_to_f(w[u] >> 24)));
    }
    for (; v < nw; v += stride) {
        const unsigned w = __ldg(reinterpret_cast<const unsigned*>(in) + v);
        st_na_f4(reinterpret_cast<float4*>(out) + v, make_float4(u8_to_f(w & 255u), u8_to_f((w >> 8) & 255u), u8_to_f((w >> 16) & 255u), u8_to_f(w >> 24)));
    }
    for (long i = nw * 4 + (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = u8_to_f(in[i]);
}

__global__ void __launch_bounds__(256) convert_s16_f_kernel(const short* __restrict__ in, float* __restrict__ out, long n)
{
    // reference build (-ffast-math) multiplies by the float-rounded reciprocal of SHRT_MAX; see oracle.c
    const float recip = 1.0f / 32767.0f;
    const long nw = n / 4;                                             // 8-byte words of four shorts
    const long stride = (long)gridDim.x * blockDim.x;
    long v = (long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; v + 3 * stride < nw; v += 4 * stride) {
        uint2 w[4];
#pragma unroll
        for (int u = 0; u < 4; u++) w[u] = __ldg(reinterpret_cast<const uint2*>(in) + v + u * stride);
#pragma unroll
        for (int u = 0; u < 4; u++)
            st_na_f4(reinterpret_cast<float4*>(out) + v + u * stride,
                     make_float4(__fmul_rn((float)(short)(w[u].x & 0xffffu), recip), __fmul_rn((float)(short)(w[u].x >> 16), recip),
                                 __fmul_rn((float)(short)(w[u].y & 0xffffu), recip), __fmul_rn((float)(short)(w[u].y >> 16), recip)));
    }
    for (; v < nw; v += stride) {
        const uint2 w = __ldg(reinterpret_cast<const uint2*>(in) + v);
        st_na_f4(reinterpret_cast<float4*>(out) + v,
                 make_float4(__fmul_rn((float)(short)(w.x & 0xffffu), recip), __fmul_rn((float)(short)(w.x >> 16), recip),
                             __fmul_rn((float)(short)(w.y & 0xffffu), recip), __fmul_rn((float)(short)(w.y >> 16), recip)));
    }
    for (long i = nw * 4 + (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = __fmul_rn((float)in[i], recip);
}

// f32 -> s16: f_to_s16_bits (common.cuh) = float multiply by 32767, truncate toward zero, keep the low 16 bits of the int32
__global__ void __launch_bounds__(256) convert_f_s16_kernel(const float* __restrict__ in, short* __restrict__ out, long n)
{
    const long nvec = n / 8;
    const long stride = (long)gridDim.x * blockDim.x;
    for (long v = (long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
        const float4 a = reinterpret_cast<const float4*>(in)[2 * v], b = reinterpret_cast<const float4*>(in)[2 * v + 1];
        uint4 q;
        q.x = f_to_s16_bits(a.x) | (f_to_s16_bits(a.y) << 16);
        q.y = f_to_s16_bits(a.z) | (f_to_s16_bits(a.w) << 16);
        q.z = f_to_s16_bits(b.x) | (f_to_s16_bits(b.y) << 16);
        q.w = f_to_s16_bits(b.z) | (f_to_s16_bits(b.w) << 16);
        reinterpret_cast<uint4*>(out)[v] = q;
    }
    for (long i = nvec * 8 + (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (short)f_to_s16_bits(in[i]);
}

// ---- the other sample formats: convert_s8_f, convert_f_s8, convert_f_u8, convert_s24_f, convert_f_s24 (libcsdr.c:2368-2437) -------------
// The arithmetic of the reference's -O3 -ffast-math x86 build, value for value:
//   s8 -> f32   (float)b * (1.0f/127.0f): the build multiplies by the float-rounded reciprocal of SCHAR_MAX instead of dividing
//   f32 -> s8   x * 127.0f, truncated as cvttss2si does, low byte
//   f32 -> u8   (double)(x * 255.0f) * 0.5 + 128.0 (float product, double sum), truncated as cvttsd2si does, low byte
//   f32 -> s24  x * 8388607.0f (INT_MAX >> 8), truncated as cvttss2si does, low three bytes
//   s24 -> f32  the three bytes as the top of an int32 (exact as a float) times the build's constant 0x30000001 = (float)(1/2147483392.0f),
//               2147483392 being (float)(INT_MAX - 256)
// s24 byte order: the reference's `bigendian` flag names the opposite of what it does on x86.  Without it the most significant byte comes
// first (big-endian); with it the least significant one.  The kernels take the flag with the reference's meaning.
constexpr float kS8Recip = 1.0f / 127.0f;
constexpr float kS24Recip = 1.0f / 2147483392.0f;

__device__ __forceinline__ float s8_to_f(unsigned b) { return __fmul_rn((float)(int)(signed char)b, kS8Recip); }
__device__ __forceinline__ unsigned f_to_s8_bits(float x) { return (unsigned)x86_trunc_i32(__fmul_rn(x, 127.0f)) & 0xffu; }
// x*255 rounds once in float; *0.5 is exact in double, so the sum rounds once whether or not it is contracted into an FMA
__device__ __forceinline__ unsigned f_to_u8_bits(float x) { return (unsigned)x86_trunc_i32((double)__fmul_rn(x, 255.0f) * 0.5 + 128.0) & 0xffu; }

// v = the sample's three bytes in stream order, packed little-endian (b0 | b1 << 8 | b2 << 16).  LSB_FIRST = the reference's `bigendian`.
template <bool LSB_FIRST>
__device__ __forceinline__ float s24_to_f(unsigned v)
{
    const unsigned w = LSB_FIRST ? v << 8 : (v & 0xffu) << 24 | (v & 0xff00u) << 8 | (v & 0xff0000u) >> 8;
    return __fmul_rn((float)(int)w, kS24Recip);
}
// the sample's three bytes in stream order, packed the same way: the low three bytes of the truncated int32 (INT_MIN stores zeros)
template <bool LSB_FIRST>
__device__ __forceinline__ unsigned f_to_s24_bytes(float x)
{
    const unsigned t = (unsigned)x86_trunc_i32(__fmul_rn(x, 8388607.0f));
    return LSB_FIRST ? t & 0xffffffu : (t & 0xffu) << 16 | (t & 0xff00u) | (t >> 16 & 0xffu);
}

// Each format is a policy for one grid-stride loop: a lane converts a group of four values per step, four steps in flight, with whole-word
// global accesses -- one 32-bit word of s8 bytes, three of s24 bytes, one float4 of floats in; one float4, or one or three 32-bit words out.
// ngroups = 0 when a buffer lacks the alignment of its group accesses: then every value takes the per-value path (byte accesses).
struct S8ToF {
    using In = unsigned char; using Out = float; using Group = unsigned;
    static __device__ __forceinline__ Group load(const In* in, long g) { return __ldg(reinterpret_cast<const unsigned*>(in) + g); }
    static __device__ __forceinline__ void store(Out* out, long g, Group w)
    {
        st_na_f4(reinterpret_cast<float4*>(out) + g, make_float4(s8_to_f(w & 255u), s8_to_f((w >> 8) & 255u), s8_to_f((w >> 16) & 255u), s8_to_f(w >> 24)));
    }
    static __device__ __forceinline__ void one(const In* in, Out* out, long i) { out[i] = s8_to_f(in[i]); }
};

template <bool U8>
struct FToByte {
    using In = float; using Out = unsigned char; using Group = float4;
    static __device__ __forceinline__ unsigned bits(float x) { return U8 ? f_to_u8_bits(x) : f_to_s8_bits(x); }
    static __device__ __forceinline__ Group load(const In* in, long g) { return __ldg(reinterpret_cast<const float4*>(in) + g); }
    static __device__ __forceinline__ void store(Out* out, long g, Group a)
    {
        reinterpret_cast<unsigned*>(out)[g] = bits(a.x) | bits(a.y) << 8 | bits(a.z) << 16 | bits(a.w) << 24;
    }
    static __device__ __forceinline__ void one(const In* in, Out* out, long i) { out[i] = (unsigned char)bits(in[i]); }
};

struct Words3 { unsigned a, b, c; };                                      // 12 bytes: four s24 samples

template <bool LSB_FIRST>
struct S24ToF {
    using In = unsigned char; using Out = float; using Group = Words3;
    static __device__ __forceinline__ Group load(const In* in, long g)
    {
        const unsigned* p = reinterpret_cast<const unsigned*>(in) + 3 * g;
        return {__ldg(p), __ldg(p + 1), __ldg(p + 2)};
    }
    static __device__ __forceinline__ void store(Out* out, long g, Group w)
    {
        st_na_f4(reinterpret_cast<float4*>(out) + g,
                 make_float4(s24_to_f<LSB_FIRST>(w.a & 0xffffffu), s24_to_f<LSB_FIRST>(w.a >> 24 | (w.b & 0xffffu) << 8),
                             s24_to_f<LSB_FIRST>(w.b >> 16 | (w.c & 0xffu) << 16), s24_to_f<LSB_FIRST>(w.c >> 8)));
    }
    static __device__ __forceinline__ void one(const In* in, Out* out, long i)
    {
        const In* p = in + 3 * i;
        out[i] = s24_to_f<LSB_FIRST>((unsigned)p[0] | (unsigned)p[1] << 8 | (unsigned)p[2] << 16);
    }
};

template <bool LSB_FIRST>
struct FToS24 {
    using In = float; using Out = unsigned char; using Group = float4;
    static __device__ __forceinline__ Group load(const In* in, long g) { return __ldg(reinterpret_cast<const float4*>(in) + g); }
    static __device__ __forceinline__ void store(Out* out, long g, Group a)
    {
        const unsigned v0 = f_to_s24_bytes<LSB_FIRST>(a.x), v1 = f_to_s24_bytes<LSB_FIRST>(a.y), v2 = f_to_s24_bytes<LSB_FIRST>(a.z),
                       v3 = f_to_s24_bytes<LSB_FIRST>(a.w);
        unsigned* p = reinterpret_cast<unsigned*>(out) + 3 * g;
        p[0] = v0 | v1 << 24; p[1] = v1 >> 8 | v2 << 16; p[2] = v2 >> 16 | v3 << 8;
    }
    static __device__ __forceinline__ void one(const In* in, Out* out, long i)
    {
        const unsigned v = f_to_s24_bytes<LSB_FIRST>(in[i]);
        Out* p = out + 3 * i;
        p[0] = (Out)v; p[1] = (Out)(v >> 8); p[2] = (Out)(v >> 16);
    }
};

template <class P>
__global__ void __launch_bounds__(256) convert_groups_kernel(const typename P::In* __restrict__ in, typename P::Out* __restrict__ out, long n, long ngroups)
{
    const long stride = (long)gridDim.x * blockDim.x;
    long g = (long)blockIdx.x * blockDim.x + threadIdx.x;
    for (; g + 3 * stride < ngroups; g += 4 * stride) {
        typename P::Group w[4];
#pragma unroll
        for (int u = 0; u < 4; u++) w[u] = P::load(in, g + u * stride);
#pragma unroll
        for (int u = 0; u < 4; u++) P::store(out, g + u * stride, w[u]);
    }
    for (; g < ngroups; g += stride) P::store(out, g, P::load(in, g));
    for (long i = ngroups * 4 + (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) P::one(in, out, i);
}

// ---- waterfall compression (SURVEY 8(f) rank 4): IMA ADPCM, 4 bits per value ------------------------------------------------------------
// encode_ima_adpcm_i16_u8 (ima_adpcm.c:95-150) is a predictor/step-index recursion, sequential by definition; OpenWebRX runs one per audio stream and one
// per waterfall line (csdr.c:1745-1767, state reset every line), so the bank form is one thread per row.  Integer arithmetic: bit-exact.
__constant__ int c_ima_step[89] = {7, 8, 9, 10, 11, 12, 13, 14, 16, 17, 19, 21, 23, 25, 28, 31, 34, 37, 41, 45, 50, 55, 60, 66, 73, 80, 88, 97, 107, 118, 130, 143, 157,
    173, 190, 209, 230, 253, 279, 307, 337, 371, 408, 449, 494, 544, 598, 658, 724, 796, 876, 963, 1060, 1166, 1282, 1411, 1552, 1707, 1878, 2066, 2272, 2499, 2749,
    3024, 3327, 3660, 4026, 4428, 4871, 5358, 5894, 6484, 7132, 7845, 8630, 9493, 10442, 11487, 12635, 13899, 15289, 16818, 18500, 20350, 22385, 24623, 27086,
    29794, 32767};                                                       // the IMA/DVI ADPCM standard's step table

__device__ __forceinline__ unsigned ima_encode_one(int sample, int& index, int& previous)
{
    const int step = c_ima_step[index];
    int diff = sample - previous, s = step;
    unsigned code = 0;
    if (diff < 0) { code = 8; diff = -diff; }
    if (diff >= s) { code |= 4; diff -= s; }
    s >>= 1;
    if (diff >= s) { code |= 2; diff -= s; }
    s >>= 1;
    if (diff >= s) code |= 1;
    int delta = step >> 3;                                               // the decoder's reconstruction keeps encoder and decoder in step
    if (code & 1) delta += step >> 2;
    if (code & 2) delta += step >> 1;
    if (code & 4) delta += step;
    previous += (code & 8) ? -delta : delta;
    previous = min(32767, max(-32768, previous));
    index += (code & 4) ? 2 * (int)(code & 3) + 2 : -1;                  // index adjust table {-1,-1,-1,-1,2,4,6,8}
    index = min(88, max(0, index));
    return code;
}

struct ImaState { int index, previous; };                               // = ima_adpcm_state_t (ima_adpcm.h:35-38)

__global__ void adpcm_encode_rows_kernel(const short* __restrict__ in, long in_stride, unsigned char* __restrict__ out, long out_stride, int rows, int n,
                                         ImaState* __restrict__ state_io)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const short* x = in + (long)r * in_stride;
    unsigned char* y = out + (long)r * out_stride;
    int index = state_io[r].index, previous = state_io[r].previous;
    index = min(88, max(0, index));                                      // a caller's garbage must not index outside the table
    for (int k = 0; k < n / 2; k++) {
        const unsigned lo = ima_encode_one(x[2 * k], index, previous), hi = ima_encode_one(x[2 * k + 1], index, previous);
        y[k] = (unsigned char)(lo | (hi << 4));
    }
    state_io[r].index = index; state_io[r].previous = previous;
}

// one waterfall line per thread: ten copies of the first value in front, dB * 100 truncated to short (x86 cvttss2si + 16-bit store), fresh state
__global__ void compress_fft_adpcm_rows_kernel(const float* __restrict__ in, long in_stride, unsigned char* __restrict__ out, long out_stride, int rows, int fft_size)
{
    constexpr int PAD = 10;                                              // csdr.c:1739
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const float* x = in + (long)r * in_stride;
    unsigned char* y = out + (long)r * out_stride;
    int index = 0, previous = 0;
    for (int k = 0; k < (fft_size + PAD) / 2; k++) {
        unsigned code[2];
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int i = 2 * k + h;
            const int w = x86_trunc_i32(__fmul_rn(x[i < PAD ? 0 : i - PAD], 100.0f));
            code[h] = ima_encode_one((int)(short)(w & 0xffff), index, previous);
        }
        y[k] = (unsigned char)(code[0] | (code[1] << 4));
    }
}

static int grid_for(long work_items, int block)
{
    long g = (work_items + block - 1) / block;
    const long cap = kSmCount * 16;                              // 16 resident CTAs of 256 threads per SM is plenty
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

int launch_convert_u8_f(const unsigned char* d_in, float* d_out, long n, cudaStream_t st)
{
    if (n <= 0) return 0;
    if ((reinterpret_cast<uintptr_t>(d_in) & 15) || (reinterpret_cast<uintptr_t>(d_out) & 15)) { set_error("convert_u8_f: device buffers must be 16-byte aligned"); return -1; }
    convert_u8_f_kernel<<<grid_for(n / 16 + 1, 256), 256, 0, st>>>(d_in, d_out, n);
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}
int launch_convert_s16_f(const short* d_in, float* d_out, long n, cudaStream_t st)
{
    if (n <= 0) return 0;
    if ((reinterpret_cast<uintptr_t>(d_in) & 15) || (reinterpret_cast<uintptr_t>(d_out) & 15)) { set_error("convert_s16_f: device buffers must be 16-byte aligned"); return -1; }
    convert_s16_f_kernel<<<grid_for(n / 8 + 1, 256), 256, 0, st>>>(d_in, d_out, n);
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}
int launch_convert_f_s16(const float* d_in, short* d_out, long n, cudaStream_t st)
{
    if (n <= 0) return 0;
    if ((reinterpret_cast<uintptr_t>(d_in) & 15) || (reinterpret_cast<uintptr_t>(d_out) & 15)) { set_error("convert_f_s16: device buffers must be 16-byte aligned"); return -1; }
    convert_f_s16_kernel<<<grid_for(n / 8 + 1, 256), 256, 0, st>>>(d_in, d_out, n);
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}

// byte buffers at any address, float buffers 4-byte aligned: the group path where the input and output pointers have in_align / out_align, the per-value path otherwise
template <class P>
static int launch_convert_groups(const typename P::In* d_in, typename P::Out* d_out, long n, uintptr_t in_align, uintptr_t out_align, cudaStream_t st)
{
    if (n <= 0) return 0;
    const bool grouped = !(reinterpret_cast<uintptr_t>(d_in) & (in_align - 1)) && !(reinterpret_cast<uintptr_t>(d_out) & (out_align - 1));
    const long ngroups = grouped ? n / 4 : 0;
    convert_groups_kernel<P><<<grid_for(grouped ? n / 16 + 1 : n / 4 + 1, 256), 256, 0, st>>>(d_in, d_out, n, ngroups);
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}
int launch_convert_s8_f(const unsigned char* d_in, float* d_out, long n, cudaStream_t st) { return launch_convert_groups<S8ToF>(d_in, d_out, n, 4, 16, st); }
int launch_convert_f_s8(const float* d_in, unsigned char* d_out, long n, cudaStream_t st) { return launch_convert_groups<FToByte<false>>(d_in, d_out, n, 16, 4, st); }
int launch_convert_f_u8(const float* d_in, unsigned char* d_out, long n, cudaStream_t st) { return launch_convert_groups<FToByte<true>>(d_in, d_out, n, 16, 4, st); }
int launch_convert_s24_f(const unsigned char* d_in, float* d_out, long n, int bigendian, cudaStream_t st)
{
    return bigendian ? launch_convert_groups<S24ToF<true>>(d_in, d_out, n, 4, 16, st) : launch_convert_groups<S24ToF<false>>(d_in, d_out, n, 4, 16, st);
}
int launch_convert_f_s24(const float* d_in, unsigned char* d_out, long n, int bigendian, cudaStream_t st)
{
    return bigendian ? launch_convert_groups<FToS24<true>>(d_in, d_out, n, 16, 4, st) : launch_convert_groups<FToS24<false>>(d_in, d_out, n, 16, 4, st);
}

// ---- limit_ff (libcsdr.c:1130-1137): clamp to +-max; NaN -> +max like the reference build's minss/maxss (see oracle.c) ----
__global__ void __launch_bounds__(256) limit_ff_kernel(const float* __restrict__ in, float* __restrict__ out, long n, float max_amplitude)
{
    const long stride = (long)gridDim.x * blockDim.x;
    const long nvec = n / 4;
    for (long v = (long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(in) + v);
        st_na_f4(reinterpret_cast<float4*>(out) + v,
                 make_float4(fmaxf(-max_amplitude, fminf(max_amplitude, a.x)), fmaxf(-max_amplitude, fminf(max_amplitude, a.y)),
                             fmaxf(-max_amplitude, fminf(max_amplitude, a.z)), fmaxf(-max_amplitude, fminf(max_amplitude, a.w))));
    }
    for (long i = nvec * 4 + (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = fmaxf(-max_amplitude, fminf(max_amplitude, in[i]));
}

int launch_adpcm_encode_rows(const short* d_in, long in_stride, unsigned char* d_out, long out_stride, int rows, int n, void* d_state_io, cudaStream_t st)
{
    if (rows <= 0 || n < 2) return 0;
    adpcm_encode_rows_kernel<<<(rows + 63) / 64, 64, 0, st>>>(d_in, in_stride, d_out, out_stride, rows, n, static_cast<ImaState*>(d_state_io));
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

int launch_compress_fft_adpcm_rows(const float* d_in, long in_stride, unsigned char* d_out, long out_stride, int rows, int fft_size, cudaStream_t st)
{
    if (rows <= 0 || fft_size <= 0) return 0;
    compress_fft_adpcm_rows_kernel<<<(rows + 63) / 64, 64, 0, st>>>(d_in, in_stride, d_out, out_stride, rows, fft_size);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

int launch_limit_ff(const float* d_in, float* d_out, long n, float max_amplitude, cudaStream_t st)
{
    if (n <= 0) return 0;
    if ((reinterpret_cast<uintptr_t>(d_in) & 15) || (reinterpret_cast<uintptr_t>(d_out) & 15)) { set_error("limit_ff: device buffers must be 16-byte aligned"); return -1; }
    limit_ff_kernel<<<grid_for(n / 4 + 1, 256), 256, 0, st>>>(d_in, d_out, n, max_amplitude);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---- spectrum side path (8f rank 4): window multiply, log power (libcsdr.c:1269-1276, 1296-1314) ----------------------------
// rows of `size` complex values; the window table repeats per row (fft_cc applies one window per FFT frame)
__global__ void __launch_bounds__(256) apply_window_rows_kernel(const float2* __restrict__ in, float2* __restrict__ out, const float* __restrict__ w, int size, long total)
{
    const long stride = (long)gridDim.x * blockDim.x;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
        const float2 v = in[i]; const float g = __ldg(w + (int)(i % size));
        out[i] = make_float2(__fmul_rn(v.x, g), __fmul_rn(v.y, g));
    }
}
// mode 0: out = 10*log10(I^2+Q^2)+add_db   mode 1: acc += I^2+Q^2   mode 2: out = 10*log10(in_f)+add_db (log_ff)
__global__ void __launch_bounds__(256) power_kernel(const float2* __restrict__ in_c, const float* __restrict__ in_f, float* __restrict__ out, long n, float add_db, int mode)
{
    const long stride = (long)gridDim.x * blockDim.x;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
        float p;
        if (mode == 2) p = in_f[i];
        else { const float2 v = in_c[i]; p = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)); }
        if (mode == 1) out[i] = __fadd_rn(out[i], p);
        else out[i] = __fadd_rn(__fmul_rn(10.f, (float)log10((double)p)), add_db);      // log10 in double on the float value, like the C promotion
    }
}

int launch_apply_window_rows(const float2* d_in, float2* d_out, const float* d_window, int size, long rows, cudaStream_t st)
{
    if (size <= 0 || rows <= 0) return 0;
    apply_window_rows_kernel<<<grid_for((long)size * rows, 256), 256, 0, st>>>(d_in, d_out, d_window, size, (long)size * rows);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}
int launch_power(const float2* d_in_c, const float* d_in_f, float* d_out, long n, float add_db, int mode, cudaStream_t st)
{
    if (n <= 0) return 0;
    power_kernel<<<grid_for(n, 256), 256, 0, st>>>(d_in_c, d_in_f, d_out, n, add_db, mode);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---- K4 fmdemod_quadri_cf -------------------------------------------------------------------------
// out[i] = den ? K*(I*(Q-Qprev) - Q*(I-Iprev))/den : 0 with den = I*I+Q*Q; no FMA contraction so that
// every intermediate rounds like the reference's SSE code; the K*num/den tail is evaluated in double
// exactly as the C expression promotes it (libcsdr.c:1065).
#define FMDEMOD_K 0.340447550238101026565118445432744920253753662109375

__device__ __forceinline__ float quadri(float2 cur, float2 prev)
{
    const float dq = __fsub_rn(cur.y, prev.y), di = __fsub_rn(cur.x, prev.x);
    const float num = __fsub_rn(__fmul_rn(cur.x, dq), __fmul_rn(cur.y, di));
    const float den = __fadd_rn(__fmul_rn(cur.x, cur.x), __fmul_rn(cur.y, cur.y));
    return den != 0.f ? (float)(FMDEMOD_K * (double)num / (double)den) : 0.f;
}

__global__ void __launch_bounds__(256)
fmdemod_quadri_bank_kernel(const float2* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride, int n,
                           const float2* __restrict__ last_in, float2* __restrict__ last_out)
{
    const int ch = blockIdx.y;
    const float2* x = in + (long)ch * in_stride;
    float* y = out + (long)ch * out_stride;
    const float2 carry = last_in ? last_in[ch] : make_float2(0.f, 0.f);
    const int stride = gridDim.x * blockDim.x;
    // two samples per thread per step: one 128-bit load + the previous sample
    const int npair = n / 2;
    const bool vec_ok = ((reinterpret_cast<uintptr_t>(x) & 15) == 0);
    if (vec_ok) {
        for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < npair; v += stride) {
            const float4 q = reinterpret_cast<const float4*>(x)[v];
            const float2 a = make_float2(q.x, q.y), b = make_float2(q.z, q.w);
            const float2 p = v ? x[2 * v - 1] : carry;
            reinterpret_cast<float2*>(y)[v] = make_float2(quadri(a, p), quadri(b, a));   // y is 8-byte aligned when out_stride is even
        }
        if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) y[n - 1] = quadri(x[n - 1], n > 1 ? x[n - 2] : carry);
    } else {
        for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) y[i] = quadri(x[i], i ? x[i - 1] : carry);
    }
    if (last_out && blockIdx.x == 0 && threadIdx.x == 0 && n > 0) last_out[ch] = x[n - 1];
}

int launch_fmdemod_quadri_bank(const float2* d_in, long in_stride, float* d_out, long out_stride, int channels, int n,
                               const float2* d_last_in, float2* d_last_out, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if ((reinterpret_cast<uintptr_t>(d_out) & 7) || (out_stride & 1) ) {
        set_error("fmdemod_quadri bank: output must be 8-byte aligned with an even channel stride"); return -1;
    }
    if (d_last_in && d_last_out == d_last_in) {
        // in-place carry update is fine: each channel's carry is read before the single writer thread stores it?  No:
        // other blocks of the same channel may read it later.  Require distinct buffers.
        set_error("fmdemod_quadri bank: last_in and last_out must not alias"); return -1;
    }
    int gx = (n / 2 + 255) / 256; if (gx < 1) gx = 1; if (gx > 64) gx = 64;
    fmdemod_quadri_bank_kernel<<<dim3(gx, channels), 256, 0, st>>>(d_in, in_stride, d_out, out_stride, n, d_last_in, d_last_out);
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}

}  // namespace csdrb
