// fft_real.cuh -- forward real-to-complex FFT of 2M real points (fft_fc's make_fft_r2c plan, fft_fftw.c:16-24) through an M-point c2c.
//
// The standard packing: z[n] = x[2n] + i*x[2n+1], Z = FFT_M(z), then for k = 0..M (Z[M] = Z[0], W = exp(-2*pi*i/2M))
//     X[k] = (Z[k] + conj Z[M-k]) / 2  -  i * W^k * (Z[k] - conj Z[M-k]) / 2,     X[0] = Re Z[0] + Im Z[0],  X[M] = Re Z[0] - Im Z[0].
// One thread computes the pair X[k], X[M-k] (k = 0..M/2) from Z[k], Z[M-k] and one table entry W^k; W^(M-k) = -conj(W^k) exactly.  The table
// (M/2 + 1 entries) is computed in double and rounded once, cached per device and size (fft.cu: get_rfft_twiddles).
// rfft_split_pair is the only place that arithmetic lives: the single-CTA kernel below, the split kernel behind the four-step transform (fft.cu) and the
// real waterfall bank (spectrum.cu) all call it, so their bins agree bit for bit.
// Single CTA (M <= 16384, i.e. up to 32768 real points): the split reads Z from the FFT's own shared-memory buffer.  The transform's last pass
// ends its reads of that buffer with a barrier before it stores, so its sink writes Z back into the same slots; one more barrier and the split
// runs.  No second buffer: at M = 16384 the transform already takes 147 KB of shared memory.
#pragma once
#include "fft16.cuh"

namespace csdrb {

// X[k] from a = Z[k], b = Z[M-k] and w = W^k (all rounding spelled out: every caller gets the same bits)
__device__ __forceinline__ float2 rfft_split(float2 a, float2 b, float2 w)
{
    const float ex = __fmul_rn(0.5f, __fadd_rn(a.x, b.x)), ey = __fmul_rn(0.5f, __fsub_rn(a.y, b.y));     // (Z[k] + conj Z[M-k]) / 2
    const float ox = __fmul_rn(0.5f, __fsub_rn(a.x, b.x)), oy = __fmul_rn(0.5f, __fadd_rn(a.y, b.y));     // (Z[k] - conj Z[M-k]) / 2
    const float p = fmaf(w.x, ox, -__fmul_rn(w.y, oy)), q = fmaf(w.x, oy, __fmul_rn(w.y, ox));            // w * o = p + i q; i (p + i q) = -q + i p
    return make_float2(__fadd_rn(ex, q), __fsub_rn(ey, p));
}

// bins k and M - k (k = 0: bins 0 and M) of the 2M-point real transform to out.store(bin, value)
template <typename Out>
__device__ __forceinline__ void rfft_split_pair(int k, int M, float2 zk, float2 zmk, const float2* __restrict__ rtw, Out& out)
{
    if (k == 0) {
        out.store(0, make_float2(__fadd_rn(zk.x, zk.y), 0.f));
        out.store(M, make_float2(__fsub_rn(zk.x, zk.y), 0.f));
        return;
    }
    const float2 w = __ldg(rtw + k);
    out.store(k, rfft_split(zk, zmk, w));
    if (2 * k != M) out.store(M - k, rfft_split(zmk, zk, make_float2(-w.x, w.y)));
}

// 2M-point real transform: in.load(i) / in.load2(i) give packed elements (x[2i], x[2i+1]); out.store(k, X[k]) for k = 0..M.  `s` holds
// fft_smem_elems(M) slots; tw is the c2c table of M points (row_fft_twiddles), rtw the split table.  All fft_threads(M) threads must call.
template <int M, typename In, typename Out>
__device__ __forceinline__ void block_rfft_io(float2* __restrict__ s, const float2* __restrict__ tw, const float2* __restrict__ rtw, int tid, In& in, Out& out)
{
    constexpr int NT = fft_threads(M);
    struct ToShared {                                                   // Z back into the transform's buffer (the last pass has read all of it)
        float2* s;
        __device__ __forceinline__ void store(int i, float2 v) const { s[fft_pad(i)] = v; }
        __device__ __forceinline__ void store2(int i, float2 a, float2 b) const { *reinterpret_cast<float4*>(s + fft_pad(i)) = make_float4(a.x, a.y, b.x, b.y); }
    } z{s};
    block_row_fft_io<M, false>(s, tw, tid, in, z);
    __syncthreads();
    for (int k = tid; k <= M / 2; k += NT) rfft_split_pair(k, M, s[fft_pad(k)], s[fft_pad((M - k) & (M - 1))], rtw, out);
}

// one real row as packed input: element i = (x[2i], x[2i+1]), scalar loads (a row may start at any float)
struct RfftRowIn {
    const float* x;
    __device__ __forceinline__ float2 load(int i) const { return make_float2(__ldg(x + 2 * i), __ldg(x + 2 * i + 1)); }
    __device__ __forceinline__ float4 load2(int i) const { const float2 a = load(i), b = load(i + 1); return make_float4(a.x, a.y, b.x, b.y); }
};
// the same rows as input of the four-step transform (fft_large.cuh): element i of transform b
struct RfftLargeRowsIn {
    const float* x; long stride;
    __device__ __forceinline__ float2 at(int b, long i) const { const float* r = x + (long)b * stride + 2 * i; return make_float2(__ldg(r), __ldg(r + 1)); }
};
struct RfftRowOut {
    float2* y;
    __device__ __forceinline__ void store(int k, float2 v) const { y[k] = v; }
};

// csdrb_fft_r2c_batch up to 2*FFT_MAX_N real points: one CTA per row, M + 1 bins out
template <int M>
__global__ void __launch_bounds__(fft_threads(M))
fft_r2c_batch_kernel(const float* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride, const float2* __restrict__ tw,
                     const float2* __restrict__ rtw)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* s = reinterpret_cast<float2*>(smem_raw);
    RfftRowIn src{in + (long)blockIdx.x * in_stride};
    RfftRowOut dst{out + (long)blockIdx.x * out_stride};
    block_rfft_io<M>(s, tw, rtw, threadIdx.x, src, dst);
}

// host: W^k = exp(-2*pi*i*k / 2M), k = 0..M/2, in double and rounded once
inline void rfft_fill_twiddles(int M, float2* h)
{
    for (int k = 0; k <= M / 2; k++) {
        const double a = -3.14159265358979323846 * (double)k / (double)M;
        h[k] = make_float2((float)cos(a), (float)sin(a));
    }
}

}  // namespace csdrb
