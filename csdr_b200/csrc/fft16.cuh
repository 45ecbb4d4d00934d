// fft16.cuh -- radix-16 passes for the block FFT.
//
// N = R0 * 16^k with R0 in {2, 4, 8, 16}: 4096 = 16*16*16 is three passes instead of four, 16384 = 4*16*16*16 four instead of five.  With the
// first pass reading the caller's data and the last pass writing it (fft.cuh: block_fft_io) a 4096-point transform touches shared memory
// 2R+2W times per point (round 1: 5R+5W, fused radix-8: 3R+3W).  One thread = one radix-16 butterfly per pass (16 points, 32 data
// registers); the first pass of the other sizes does 16/R0 small butterflies per thread.  Same index scheme as fft.cuh: butterfly j of a
// pass of radix R over sub-transforms of size NS reads elements j + r*N/R and writes (j/NS)*NS*R + j%NS + r*NS.
// Twiddles for a radix-16 pass: w^r, r = 1..15, w = exp(-2*pi*i*k/(16*NS)), k = j mod NS, from four planes w^1, w^2, w^4, w^8 at index
// NS + k (contiguous in k) and eleven products.
#pragma once
#include "fft.cuh"

namespace csdrb {

constexpr int fft16_first_radix(int n) { return ilog2_c(n) % 4 == 1 ? 2 : (ilog2_c(n) % 4 == 2 ? 4 : (ilog2_c(n) % 4 == 3 ? 8 : 16)); }

// host: four planes (w^1, w^2, w^4, w^8) of n entries each; a radix-16 pass over sub-size NS reads index NS + k, k < NS
inline void fft16_fill_twiddles(int n, float2* h)
{
    for (long i = 0; i < 4L * n; i++) h[i] = make_float2(1.f, 0.f);
    int ns = fft16_first_radix(n);
    for (; ns < n; ns *= 16)
        for (int k = 0; k < ns; k++)
            for (int c = 0; c < 4; c++) {
                const double a = -2.0 * 3.14159265358979323846 * (double)((1 << c) * k) / (double)(ns * 16);
                h[(size_t)c * n + ns + k] = make_float2((float)cos(a), (float)sin(a));
            }
}

// a * W16^M (forward) or a * conj(W16^M) (inverse), M a compile-time constant
template <bool INV, int M>
__device__ __forceinline__ float2 mul_w16(float2 a)
{
    constexpr float C1 = 0.923879532511286756f, S1 = 0.382683432365089772f, H = 0.707106781186547524f;
    constexpr float WR = M == 0 ? 1.f : M == 1 ? C1 : M == 2 ? H : M == 3 ? S1 : M == 4 ? 0.f : M == 6 ? -H : /* M == 9 */ -C1;
    constexpr float WI0 = M == 0 ? 0.f : M == 1 ? -S1 : M == 2 ? -H : M == 3 ? -C1 : M == 4 ? -1.f : M == 6 ? -H : /* M == 9 */ S1;
    constexpr float WI = INV ? -WI0 : WI0;
    if constexpr (M == 0) return a;
    else if constexpr (M == 4) return make_float2(-a.y * WI, a.x * WI);
    else return make_float2(fmaf(a.x, WR, -a.y * WI), fmaf(a.x, WI, a.y * WR));
}

template <bool INV>
__device__ __forceinline__ void dft16(float2 (&v)[16])
{
    // n = 4*n1 + n2, k = k1 + 4*k2:  X[k1 + 4 k2] = sum_n2 W4^(n2 k2) * W16^(n2 k1) * (sum_n1 W4^(n1 k1) x[4 n1 + n2])
    float2 y[4][4];                                                      // y[n2][k1]
#pragma unroll
    for (int n2 = 0; n2 < 4; n2++) {
        float2 a0 = v[n2], a1 = v[4 + n2], a2 = v[8 + n2], a3 = v[12 + n2];
        dft4<INV>(a0, a1, a2, a3);
        y[n2][0] = a0; y[n2][1] = a1; y[n2][2] = a2; y[n2][3] = a3;
    }
    y[1][1] = mul_w16<INV, 1>(y[1][1]); y[1][2] = mul_w16<INV, 2>(y[1][2]); y[1][3] = mul_w16<INV, 3>(y[1][3]);
    y[2][1] = mul_w16<INV, 2>(y[2][1]); y[2][2] = mul_w16<INV, 4>(y[2][2]); y[2][3] = mul_w16<INV, 6>(y[2][3]);
    y[3][1] = mul_w16<INV, 3>(y[3][1]); y[3][2] = mul_w16<INV, 6>(y[3][2]); y[3][3] = mul_w16<INV, 9>(y[3][3]);
#pragma unroll
    for (int k1 = 0; k1 < 4; k1++) {
        float2 b0 = y[0][k1], b1 = y[1][k1], b2 = y[2][k1], b3 = y[3][k1];
        dft4<INV>(b0, b1, b2, b3);
        v[k1] = b0; v[k1 + 4] = b1; v[k1 + 8] = b2; v[k1 + 12] = b3;
    }
}

template <int R, bool INV>
__device__ __forceinline__ void dft_any(float2 (&v)[R])
{
    if constexpr (R == 16) dft16<INV>(v);
    else dft_small<R, INV>(v);
}

__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x)); }

// twiddled radix-16 butterfly j of a pass over sub-transforms of size NS (> 1)
template <int N, int NS, bool INV>
__device__ __forceinline__ void fft16_butterfly(float2 (&v)[16], int j, const float2* __restrict__ tw)
{
    const int k = j % NS;
    float2 w[16];
    w[1] = __ldg(tw + NS + k); w[2] = __ldg(tw + N + NS + k); w[4] = __ldg(tw + 2 * N + NS + k); w[8] = __ldg(tw + 3 * N + NS + k);
    w[3] = cmul(w[1], w[2]); w[5] = cmul(w[1], w[4]); w[6] = cmul(w[2], w[4]); w[7] = cmul(w[3], w[4]);
    w[9] = cmul(w[1], w[8]); w[10] = cmul(w[2], w[8]); w[11] = cmul(w[3], w[8]); w[12] = cmul(w[4], w[8]);
    w[13] = cmul(w[5], w[8]); w[14] = cmul(w[6], w[8]); w[15] = cmul(w[7], w[8]);
#pragma unroll
    for (int r = 1; r < 16; r++) v[r] = cmul_w<INV>(v[r], w[r]);
    dft16<INV>(v);
}

// first pass (radix R0, no twiddles): in.load(j + r*N/R0) -> shared; every thread does 16/R0 butterflies (one when R0 = 16)
template <int N, int NT, int R0, bool INV, typename In>
__device__ __forceinline__ void fft16_pass_first(float2* __restrict__ s, int tid, In& in)
{
    constexpr int NB = N / R0;
    constexpr int PER = (NB + NT - 1) / NT;
    static_assert(PER * R0 <= 16, "one thread holds at most 16 points");
    float2 v[PER][R0];
#pragma unroll
    for (int b = 0; b < PER; b++) {
        const int j = tid + b * NT;
        if (NB % NT == 0 || j < NB) {
#pragma unroll
            for (int r = 0; r < R0; r++) v[b][r] = in.load(j + r * NB);
        }
    }
#pragma unroll
    for (int b = 0; b < PER; b++) {
        const int j = tid + b * NT;
        if (NB % NT == 0 || j < NB) {
            dft_any<R0, INV>(v[b]);
#pragma unroll
            for (int r = 0; r < R0; r++) s[fft_pad(j * R0 + r)] = v[b][r];
        }
    }
    __syncthreads();
}

template <int N, int NT, int NS, bool INV, bool LAST, typename Out>
__device__ __forceinline__ void fft16_pass(float2* __restrict__ s, const float2* __restrict__ tw, int tid, Out& out)
{
    constexpr int NB = N / 16;
    static_assert(!LAST || NS * 16 == N, "the last pass completes the transform");
    float2 v[16];
    const int j = tid;                                                   // NT >= N/16: at most one butterfly per thread
    const bool live = (NB >= NT) || j < NB;
    if (live) {
#pragma unroll
        for (int r = 0; r < 16; r++) v[r] = s[fft_pad(j + r * NB)];
        fft16_butterfly<N, NS, INV>(v, j, tw);
    }
    __syncthreads();                                                     // every read of s has happened
    if (live) {
        const int j0 = (j / NS) * NS * 16 + (j % NS);
#pragma unroll
        for (int r = 0; r < 16; r++) {
            if constexpr (LAST) out.store(j0 + r * NS, v[r]);
            else s[fft_pad(j0 + r * NS)] = v[r];
        }
    }
    if constexpr (!LAST) __syncthreads();
}

template <int N, int NT, int NS, bool INV, typename Out>
__device__ __forceinline__ void fft16_rest(float2* __restrict__ s, const float2* __restrict__ tw, int tid, Out& out)
{
    if constexpr (NS < N) {
        fft16_pass<N, NT, NS, INV, (NS * 16 == N)>(s, tw, tid, out);
        fft16_rest<N, NT, NS * 16, INV>(s, tw, tid, out);
    }
}

template <int N, int NT, int NS, bool INV>
__device__ __forceinline__ void fft16_rest_but_last(float2* __restrict__ s, const float2* __restrict__ tw, int tid)
{
    if constexpr (NS * 16 < N) {
        struct Nowhere { __device__ __forceinline__ void store(int, float2) const {} } nowhere;
        fft16_pass<N, NT, NS, INV, false>(s, tw, tid, nowhere);
        fft16_rest_but_last<N, NT, NS * 16, INV>(s, tw, tid);
    }
}

// N-point transform in.load(i) -> out.store(i), N >= 32 (smaller sizes stay on block_fft_io); `s` is scratch; NT = fft_threads(N)
template <int N, int NT, bool INV, typename In, typename Out>
__device__ __forceinline__ void block_fft16_io(float2* __restrict__ s, const float2* __restrict__ tw, int tid, In& in, Out& out)
{
    static_assert((N & (N - 1)) == 0 && N >= 32, "power of two sizes from 32");
    constexpr int R0 = fft16_first_radix(N);
    static_assert(R0 < N, "at least one radix-16 pass follows the first pass");
    fft16_pass_first<N, NT, R0, INV>(s, tid, in);
    fft16_rest<N, NT, R0, INV>(s, tw, tid, out);
}

// The one-CTA row transform of the batched c2c, r2c, fastddc forward and waterfall kernels: radix-16 passes from 32 points on (fewer passes over
// shared memory than radix 8: 4096 points take three instead of four, 16384 four instead of five), radix 8 below.  tw is the matching table
// (fft.cu: row_fft_twiddles); all fft_threads(N) threads must call.
template <int N, bool INV, typename In, typename Out>
__device__ __forceinline__ void block_row_fft_io(float2* __restrict__ s, const float2* __restrict__ tw, int tid, In& in, Out& out)
{
    if constexpr (N >= 32) block_fft16_io<N, fft_threads(N), INV>(s, tw, tid, in, out);
    else block_fft_io<N, fft_threads(N), INV>(s, tw, tid, in, out);
}

// FFT_N(in) -> map -> IFFT_N -> out for N = 16^k (256, 4096): the forward transform's last radix-16 pass leaves elements j + r*N/16 in the
// registers of thread j, which are exactly the inputs of the inverse transform's first pass -- the spectrum never returns to shared memory.
//   map.prefetch(r, i) / map.at(r, i, v): per-element data of slot r (element i = j + r*N/16), fetched while the butterfly runs.
template <int N, int NT, typename In, typename Map, typename Out>
__device__ __forceinline__ void block_fft16_map_ifft(float2* __restrict__ s, const float2* __restrict__ tw, int tid, In& in, Map& map, Out& out)
{
    static_assert(fft16_first_radix(N) == 16 && N >= 256, "register hand-over needs radix 16 at both ends");
    constexpr int NB = N / 16, NSL = N / 16;                              // last pass: sub-transform size N/16
    struct Nowhere { __device__ __forceinline__ void store(int, float2) const {} } nowhere;
    fft16_pass_first<N, NT, 16, false>(s, tid, in);
    if constexpr (N > 256) fft16_rest_but_last<N, NT, 16, false>(s, tw, tid);
    {   // forward last pass + map + inverse first pass, all in registers
        float2 v[16];
        const int j = tid;
        const bool live = (NB >= NT) || j < NB;
        if (live) {
#pragma unroll
            for (int r = 0; r < 16; r++) map.prefetch(r, j + r * NSL);
#pragma unroll
            for (int r = 0; r < 16; r++) v[r] = s[fft_pad(j + r * NB)];
            fft16_butterfly<N, NSL, false>(v, j, tw);
        }
        __syncthreads();                                                 // reads of s done
        if (live) {
#pragma unroll
            for (int r = 0; r < 16; r++) v[r] = map.at(r, j + r * NSL, v[r]);
            dft16<true>(v);                                              // inverse transform, first pass: inputs j + r*NB, no twiddles
#pragma unroll
            for (int r = 0; r < 16; r++) s[fft_pad(j * 16 + r)] = v[r];
        }
        __syncthreads();
    }
    fft16_rest<N, NT, 16, true>(s, tw, tid, out);
    (void)nowhere;
}

}  // namespace csdrb
