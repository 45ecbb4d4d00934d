// fft_large.cuh -- batched c2c FFT for N = 2^15 .. 2^20 points: the four-step algorithm on top of the shared-memory transforms of fft16.cuh.
//
// N = N1*N2, n = n1*N2 + n2, k = k1 + N1*k2:
//     X[k1 + N1*k2] = sum_n2 w_N2^(n2*k2) * ( w_N^(k1*n2) * sum_n1 w_N1^(n1*k1) * x[n1*N2 + n2] )
//   step 1 (fft_large_step_kernel<N1, .., FIRST = true>): a CTA takes W adjacent columns n2, runs W transforms of length N1 over n1 (one group of
//       N1/16 threads per column, block_fft16_io), multiplies element (k1, n2) by w_N^(+-k1*n2) and writes the tile to the TRANSPOSED intermediate
//       t[n2*N1 + k1] -- W adjacent columns are W adjacent rows of it, one contiguous run of W*N1 values.
//   step 2 (FIRST = false): the same column transform on the intermediate, length N2 over n2 for W adjacent k1, stored straight from the last
//       pass's registers to X[k1 + N1*k2].
// W = 16 and the lanes of a warp walk the columns first, so every global load and every store of step 2 is a run of one 128-byte line; a CTA is
// 16 * F/16 = F threads (1024 for the 1024-point factor: 64 registers, no spills) on 144*F bytes of shared memory.  Column groups sit an odd
// number of elements apart there: the 16 lanes of a half warp hit 16 different bank pairs.
// Inter-step twiddles: m = k1*n2 < N splits as m = 1024*mh + ml, w_N^m = hi[mh] * lo[ml] with both tables computed in double and rounded once
// ((1024 + N/1024) * 8 bytes per size, at most 16 KiB, L1-resident); one float product on top of two correctly rounded factors keeps every
// twiddle within about 2 ulp -- the accuracy class of the products inside the shared-memory passes.
// The intermediate is stream-ordered scratch of at most kFftLargeScratchBytes (16 MiB): a batch runs in chunks of 2^21/N transforms.
// The kernels live here and their launchers in fft.cu, like fft_kernels.cuh (the CPU test tier executes both).
#pragma once
#include "fft16.cuh"

namespace csdrb {

constexpr int kFftLargeSplit = 1024;                                    // m = kFftLargeSplit*mh + ml
constexpr size_t kFftLargeScratchBytes = (size_t)16 << 20;

constexpr int kFftLargeTile = 16;                                       // W: columns per CTA
__host__ __device__ constexpr int fft_large_seg(int F) { return fft_smem_elems(F) | 1; }      // odd: see the bank remark above

// transform inputs: element i of transform b
struct LargeRowsIn {
    const float2* x; long stride;
    __device__ __forceinline__ float2 at(int b, long i) const { return __ldg(x + (long)b * stride + i); }
};
// fastddc forward step: block b is stream samples [b*input_size - overlap, (b+1)*input_size), the ones before the stream from the carried overlap
struct LargeSlideIn {
    const float2* in; const float2* ov; int input_size, overlap;
    __device__ __forceinline__ float2 at(int b, long i) const
    {
        const long p = (long)b * input_size - overlap + i;
        return p >= 0 ? __ldg(in + p) : ov[overlap + p];
    }
};

// F-point transforms down W adjacent columns of a [F][S] matrix (element (i, col) = in.at(b, i*S + col)).
// FIRST: times w_N^(k*col), N = F*S, to the transposed scratch row blockIdx.y; else: to out[b][k*S + col].
template <int F, bool INV, bool FIRST, typename In>
__global__ void __launch_bounds__(kFftLargeTile * (F / 16))
fft_large_step_kernel(In in, int in_b0, float2* __restrict__ out, long out_stride, int out_b0, int S, const float2* __restrict__ tw16,
                      const float2* __restrict__ tw_lo, const float2* __restrict__ tw_hi)
{
    CSDRB_DYN_SMEM(smem_raw);
    constexpr int W = kFftLargeTile, NT = F / 16, SEG = fft_large_seg(F);
    float2* const smem = reinterpret_cast<float2*>(smem_raw);
    const int g = threadIdx.x % W, tid = threadIdx.x / W;
    const int col = blockIdx.x * W + g;
    float2* const s = smem + g * SEG;
    struct ColIn {
        const In& in; int b, col, S;
        __device__ __forceinline__ float2 load(int i) const { return in.at(b, (long)i * S + col); }
    } src{in, in_b0 + (int)blockIdx.y, col, S};
    if constexpr (FIRST) {
        struct TwiddledBack {                                           // the last pass has read all of s before it stores: the result goes back into s
            float2* s; const float2* lo; const float2* hi; int col;
            __device__ __forceinline__ void store(int k, float2 v) const
            {
                const int m = k * col;
                const float2 w = cmul(__ldg(hi + m / kFftLargeSplit), __ldg(lo + m % kFftLargeSplit));
                s[fft_pad(k)] = cmul_w<INV>(v, w);
            }
        } dst{s, tw_lo, tw_hi, col};
        block_fft16_io<F, NT, INV>(s, tw16, tid, src, dst);
        __syncthreads();
        float2* const t = out + (long)(out_b0 + blockIdx.y) * out_stride + (long)blockIdx.x * (W * F);
        for (int e = threadIdx.x; e < W * F; e += W * NT) t[e] = smem[(e / F) * SEG + fft_pad(e % F)];
    } else {
        struct ColOut {
            float2* y; int col, S;
            __device__ __forceinline__ void store(int k, float2 v) const { y[(long)k * S + col] = v; }
        } dst{out + (long)(out_b0 + blockIdx.y) * out_stride, col, S};
        block_fft16_io<F, NT, INV>(s, tw16, tid, src, dst);
    }
}

// Y[i] = X[i] * H[i] with the rounding sequence of apply_fir_fft_cc (libcsdr.c:827-828: separate products, no FMA), in place
__global__ void __launch_bounds__(256)
fft_large_times_taps_kernel(float2* __restrict__ x, const float2* __restrict__ H, int n)
{
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
        const float2 a = x[i], h = __ldg(H + i);
        x[i] = make_float2(__fsub_rn(__fmul_rn(a.x, h.x), __fmul_rn(a.y, h.y)), __fadd_rn(__fmul_rn(a.x, h.y), __fmul_rn(a.y, h.x)));
    }
}

// y[i] = y[i]/N (+ last_overlap[i] for i < overlap_size), in place (libcsdr.c:837-847)
__global__ void __launch_bounds__(256)
fft_large_scale_overlap_kernel(float2* __restrict__ y, const float2* __restrict__ last_overlap, int overlap_size, float inv_n, int n)
{
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
        float2 v = make_float2(y[i].x * inv_n, y[i].y * inv_n);
        if (i < overlap_size) v = make_float2(__fadd_rn(v.x, last_overlap[i].x), __fadd_rn(v.y, last_overlap[i].y));
        y[i] = v;
    }
}

// dst[i] = sample total - overlap + i of (old overlap ++ in[0..total)), i < overlap
__global__ void __launch_bounds__(256)
fft_large_gather_overlap_kernel(const float2* __restrict__ in, const float2* __restrict__ overlap_old, float2* __restrict__ dst, int overlap, long total)
{
    for (int i = blockIdx.x * 256 + threadIdx.x; i < overlap; i += gridDim.x * 256) {
        const long p = total - overlap + i;
        dst[i] = p >= 0 ? in[p] : overlap_old[overlap + p];
    }
}

}  // namespace csdrb
