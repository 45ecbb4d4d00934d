// elementwise.cu -- K1 sample-format conversions and K4 fmdemod_quadri_cf.
//
// K1 replaces convert_u8_f / convert_s16_f / convert_f_s16 (libcsdr.c:2363-2366, 2373-2376, 2390-2398).
// K4 replaces fmdemod_quadri_cf (libcsdr.c:1040-1071) for C channels per launch.
// All are pure streaming kernels: 128-bit global accesses, grid-stride, nothing staged.
#include "common.cuh"
#include "kernels.h"
#include <limits.h>

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
            const float s = __fmul_rn(x[i < PAD ? 0 : i - PAD], 100.0f);
            const int w = (s >= 2147483648.0f || s < -2147483648.0f || s != s) ? INT_MIN : __float2int_rz(s);
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
