// fft.cuh -- K7: block-level Stockham autosort FFT in shared memory (no cuFFT), power-of-two sizes.
//
// Stands behind the reference's FFT abstraction (fft_fftw.c:6-41: unnormalised DFT, exponent sign -1
// forward / +1 backward).  One CTA transforms one N-point signal that already sits in shared memory.
//
// Pass structure (validated against numpy): radices are
// [2 or 4 (if log2 N is not a multiple of 3)] followed by radix-8 passes.  For a pass of radix R over
// sub-transforms of size Ns (Ns = product of the previous radices), butterfly j in [0, N/R):
//     k = j mod Ns;   v[r] = s[j + r*N/R] * W_N^(k*r*N/(Ns*R));   V = DFT_R(v);   s'[(j/Ns)*Ns*R + k + r*Ns] = V[r]
// All threads read their butterflies into registers, synchronise, then write: one buffer is enough
// (a thread holds at most 16 points per pass, so NT >= N/16 threads are required).
// Twiddles: for a radix-8 pass over sub-transforms of size NS the butterfly with k = j mod NS needs w^r, w = exp(-2*pi*i*k/(8*NS)).
// Three planes of a per-size table hold w^1, w^2, w^4 at index NS + k (the ranges [NS, 2NS) of the different passes do not
// overlap), computed in double on the host and rounded once to float; lanes with consecutive k read consecutive entries (seven
// scattered LDGs per butterfly would saturate L1TEX).  w^3, w^5, w^6, w^7 are one float product each, so every
// twiddle is within ~2 ulp and the whole transform stays ~1e-7*log2 N from the exact DFT.
#pragma once
#include "common.cuh"
#include <cmath>

namespace csdrb {

// Shared-memory layout: element i lives at i + 2*(i >> 4) (two pad slots per sixteen complex values, 12.5 % extra; even indices stay
// even so element pairs are 16-byte aligned).  A thread owns PAIRS of adjacent butterflies and moves them with 128-bit LDS/STS:
// in the first pass it writes 16 consecutive elements (lane stride 18 elements = 9 x 16 B, odd: conflict-free), in the later passes
// the pair lands at adjacent positions again (sub-transform sizes are even).
__host__ __device__ constexpr int fft_pad(int i) { return i + 2 * (i >> 4); }
__host__ __device__ constexpr int fft_smem_elems(int n) { return n + 2 * (n >> 4) + 2; }

template <bool INV>
__device__ __forceinline__ float2 cmul_w(float2 a, float2 w)
{
    // a * w (forward) or a * conj(w) (inverse)
    return INV ? make_float2(fmaf(a.x, w.x, a.y * w.y), fmaf(a.y, w.x, -a.x * w.y))
               : make_float2(fmaf(a.x, w.x, -a.y * w.y), fmaf(a.y, w.x, a.x * w.y));
}
template <bool INV>
__device__ __forceinline__ float2 mul_mi(float2 a)       // a * (-i) forward, a * (+i) inverse
{
    return INV ? make_float2(-a.y, a.x) : make_float2(a.y, -a.x);
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }

template <bool INV>
__device__ __forceinline__ void dft2(float2& a, float2& b) { float2 t = a; a = cadd(t, b); b = csub(t, b); }

template <bool INV>
__device__ __forceinline__ void dft4(float2& v0, float2& v1, float2& v2, float2& v3)
{
    const float2 a0 = cadd(v0, v2), a1 = csub(v0, v2), a2 = cadd(v1, v3), a3 = mul_mi<INV>(csub(v1, v3));
    v0 = cadd(a0, a2); v2 = csub(a0, a2); v1 = cadd(a1, a3); v3 = csub(a1, a3);
}

template <bool INV>
__device__ __forceinline__ void dft8(float2 (&v)[8])
{
    float2 e0 = v[0], e1 = v[2], e2 = v[4], e3 = v[6], o0 = v[1], o1 = v[3], o2 = v[5], o3 = v[7];
    dft4<INV>(e0, e1, e2, e3);
    dft4<INV>(o0, o1, o2, o3);
    const float h = 0.70710678118654752440f;
    // W8^1 = h*(1 -+ i), W8^2 = -+i, W8^3 = h*(-1 -+ i)
    const float2 t1 = INV ? make_float2(h * (o1.x - o1.y), h * (o1.x + o1.y)) : make_float2(h * (o1.x + o1.y), h * (o1.y - o1.x));
    const float2 t2 = mul_mi<INV>(o2);
    const float2 t3 = INV ? make_float2(-h * (o3.x + o3.y), h * (o3.x - o3.y)) : make_float2(h * (o3.y - o3.x), -h * (o3.x + o3.y));
    v[0] = cadd(e0, o0); v[4] = csub(e0, o0);
    v[1] = cadd(e1, t1); v[5] = csub(e1, t1);
    v[2] = cadd(e2, t2); v[6] = csub(e2, t2);
    v[3] = cadd(e3, t3); v[7] = csub(e3, t3);
}

template <int R, bool INV>
__device__ __forceinline__ void dft_small(float2 (&v)[R])
{
    if constexpr (R == 2) dft2<INV>(v[0], v[1]);
    else if constexpr (R == 4) dft4<INV>(v[0], v[1], v[2], v[3]);
    else dft8<INV>(v);
}

template <int N, int R, int NS, bool INV>
__device__ __forceinline__ void fft_butterfly(float2 (&v)[R], int j, const float2* __restrict__ tw)
{
    if constexpr (NS > 1) {
        static_assert(R == 8, "only the first pass may have a radix below 8");
        const int k = j % NS;
        const float2 w1 = __ldg(tw + NS + k), w2 = __ldg(tw + N + NS + k), w4 = __ldg(tw + 2 * N + NS + k);
        const float2 w3 = make_float2(fmaf(w1.x, w2.x, -w1.y * w2.y), fmaf(w1.x, w2.y, w1.y * w2.x));
        const float2 w5 = make_float2(fmaf(w1.x, w4.x, -w1.y * w4.y), fmaf(w1.x, w4.y, w1.y * w4.x));
        const float2 w6 = make_float2(fmaf(w2.x, w4.x, -w2.y * w4.y), fmaf(w2.x, w4.y, w2.y * w4.x));
        const float2 w7 = make_float2(fmaf(w3.x, w4.x, -w3.y * w4.y), fmaf(w3.x, w4.y, w3.y * w4.x));
        v[1] = cmul_w<INV>(v[1], w1); v[2] = cmul_w<INV>(v[2], w2); v[3] = cmul_w<INV>(v[3], w3);
        v[4] = cmul_w<INV>(v[4], w4); v[5] = cmul_w<INV>(v[5], w5); v[6] = cmul_w<INV>(v[6], w6);
        v[7] = cmul_w<INV>(v[7], w7);
    }
    dft_small<R, INV>(v);
}

template <int N, int NT, int R, int NS, bool INV>
__device__ __forceinline__ void fft_pass(float2* __restrict__ s, const float2* __restrict__ tw, int tid)
{
    constexpr int NB = N / R;
    constexpr int PER = (NB + NT - 1) / NT;
    static_assert(PER * R <= 16, "block_fft needs NT >= N/16 threads");
    constexpr bool PAIRED = (PER % 2 == 0) && (NB % (NT * PER) == 0);   // every thread owns whole pairs of adjacent butterflies
    float2 v[PER][R];
    if constexpr (PAIRED) {
#pragma unroll
        for (int b = 0; b < PER; b += 2) {
            const int j = tid * PER + b;                                // j even: (j, j+1) adjacent and 16-byte aligned in the padded array
#pragma unroll
            for (int r = 0; r < R; r++) {
                const float4 two = *reinterpret_cast<const float4*>(s + fft_pad(j + r * NB));
                v[b][r] = make_float2(two.x, two.y); v[b + 1][r] = make_float2(two.z, two.w);
            }
            fft_butterfly<N, R, NS, INV>(v[b], j, tw);
            fft_butterfly<N, R, NS, INV>(v[b + 1], j + 1, tw);
        }
        __syncthreads();
#pragma unroll
        for (int b = 0; b < PER; b += 2) {
            const int j = tid * PER + b;
            if constexpr (NS == 1) {
                // first pass: the two butterflies write 2R consecutive elements
#pragma unroll
                for (int r = 0; r < R; r += 2) {
                    *reinterpret_cast<float4*>(s + fft_pad(j * R + r)) = make_float4(v[b][r].x, v[b][r].y, v[b][r + 1].x, v[b][r + 1].y);
                    *reinterpret_cast<float4*>(s + fft_pad((j + 1) * R + r)) = make_float4(v[b + 1][r].x, v[b + 1][r].y, v[b + 1][r + 1].x, v[b + 1][r + 1].y);
                }
            } else {
                const int j0 = (j / NS) * NS * R + (j % NS);            // NS even: j and j+1 share the group, their outputs are adjacent
#pragma unroll
                for (int r = 0; r < R; r++)
                    *reinterpret_cast<float4*>(s + fft_pad(j0 + r * NS)) = make_float4(v[b][r].x, v[b][r].y, v[b + 1][r].x, v[b + 1][r].y);
            }
        }
        __syncthreads();
    } else {
#pragma unroll
        for (int b = 0; b < PER; b++) {
            const int j = tid + b * NT;
            if (NB % NT == 0 || j < NB) {
#pragma unroll
                for (int r = 0; r < R; r++) v[b][r] = s[fft_pad(j + r * NB)];
                fft_butterfly<N, R, NS, INV>(v[b], j, tw);
            }
        }
        __syncthreads();
#pragma unroll
        for (int b = 0; b < PER; b++) {
            const int j = tid + b * NT;
            if (NB % NT == 0 || j < NB) {
                const int j0 = (j / NS) * NS * R + (j % NS);
#pragma unroll
                for (int r = 0; r < R; r++) s[fft_pad(j0 + r * NS)] = v[b][r];
            }
        }
        __syncthreads();
    }
}

template <int N, int NT, int NS, bool INV>
__device__ __forceinline__ void fft_r8_passes(float2* __restrict__ s, const float2* __restrict__ tw, int tid)
{
    if constexpr (NS < N) {
        fft_pass<N, NT, 8, NS, INV>(s, tw, tid);
        fft_r8_passes<N, NT, NS * 8, INV>(s, tw, tid);
    }
}

constexpr int ilog2_c(int n) { return n <= 1 ? 0 : 1 + ilog2_c(n / 2); }

// In-place N-point transform of the PADDED array s (element i at s[fft_pad(i)], fft_smem_elems(N) slots) by a CTA of NT threads
// (all NT threads must call; a __syncthreads() must separate the last write to s from this call).
template <int N, int NT, bool INV>
__device__ __forceinline__ void block_fft(float2* __restrict__ s, const float2* __restrict__ tw, int tid)
{
    static_assert((N & (N - 1)) == 0 && N >= 2, "power of two sizes only");
    constexpr int LG = ilog2_c(N);
    if constexpr (LG % 3 == 1) { fft_pass<N, NT, 2, 1, INV>(s, tw, tid); fft_r8_passes<N, NT, 2, INV>(s, tw, tid); }
    else if constexpr (LG % 3 == 2) { fft_pass<N, NT, 4, 1, INV>(s, tw, tid); fft_r8_passes<N, NT, 4, INV>(s, tw, tid); }
    else fft_r8_passes<N, NT, 1, INV>(s, tw, tid);
}

// ---- transform with fused input / output -----------------------------------------------------------------------------------------
// The first pass needs no twiddles and reads element j + r*N/R: it can take its inputs straight from the caller (global memory, a
// zero-padded block, a product of two spectra ...) instead of from a staged copy, and the last pass (NS*8 == N) produces element
// j + r*N/8 per thread, which can go straight to the caller as well.  That removes one shared-memory write + read + barrier at each
// end of a transform (5R+5W -> 3R+3W shared accesses per point for a 4-pass size).  When first and last pass have the same radix
// (log2 N divisible by 3: 8, 64, 512, 4096) a thread's last-pass outputs are exactly its first-pass inputs of the next transform of
// the same size, so FFT -> pointwise product -> IFFT can hand over in registers (block_fft_chain below).
//
// IO concept (i = natural element index 0..N-1):  float2 load(int i);  float4 load2(int i)  = elements (i, i+1), i even;
//                                                  void store(int i, float2 v);  void store2(int i, float2 a, float2 b), i even.
// Barrier contract: nobody may still be reading `s` when a FIRST pass is entered (a LAST pass ends its reads with a barrier, so
// back-to-back transforms on the same buffer are safe); after a LAST pass the buffer is free.
template <int N, int NT, int R, bool INV, typename In>
__device__ __forceinline__ void fft_pass_first(float2* __restrict__ s, int tid, In& in)
{
    constexpr int NB = N / R;
    constexpr int PER = (NB + NT - 1) / NT;
    static_assert(PER * R <= 16, "block_fft needs NT >= N/16 threads");
    constexpr bool PAIRED = (PER % 2 == 0) && (NB % (NT * PER) == 0);
    float2 v[PER][R];
    if constexpr (PAIRED) {
#pragma unroll
        for (int b = 0; b < PER; b += 2) {
            const int j = tid * PER + b;
#pragma unroll
            for (int r = 0; r < R; r++) {
                const float4 two = in.load2(j + r * NB);                // elements (i, i+1), i even
                v[b][r] = make_float2(two.x, two.y); v[b + 1][r] = make_float2(two.z, two.w);
            }
        }
#pragma unroll
        for (int b = 0; b < PER; b++) dft_small<R, INV>(v[b]);
#pragma unroll
        for (int b = 0; b < PER; b += 2) {
            const int j = tid * PER + b;                                // the two butterflies write 2R consecutive elements
#pragma unroll
            for (int r = 0; r < R; r += 2) {
                *reinterpret_cast<float4*>(s + fft_pad(j * R + r)) = make_float4(v[b][r].x, v[b][r].y, v[b][r + 1].x, v[b][r + 1].y);
                *reinterpret_cast<float4*>(s + fft_pad((j + 1) * R + r)) = make_float4(v[b + 1][r].x, v[b + 1][r].y, v[b + 1][r + 1].x, v[b + 1][r + 1].y);
            }
        }
    } else {
#pragma unroll
        for (int b = 0; b < PER; b++) {
            const int j = tid + b * NT;
            if (NB % NT == 0 || j < NB) {
#pragma unroll
                for (int r = 0; r < R; r++) v[b][r] = in.load(j + r * NB);
            }
        }
#pragma unroll
        for (int b = 0; b < PER; b++) {
            const int j = tid + b * NT;
            if (NB % NT == 0 || j < NB) {
                dft_small<R, INV>(v[b]);
#pragma unroll
                for (int r = 0; r < R; r++) s[fft_pad(j * R + r)] = v[b][r];
            }
        }
    }
    __syncthreads();                                                    // writes visible to the next pass
}

// last pass: radix 8 over sub-transforms of size NS = N/8, so butterfly j (< N/8) produces elements j + r*N/8
template <int N, int NT, bool INV, typename Out>
__device__ __forceinline__ void fft_pass_last(float2* __restrict__ s, const float2* __restrict__ tw, int tid, Out& out)
{
    constexpr int R = 8, NB = N / 8, NS = N / 8;
    constexpr int PER = (NB + NT - 1) / NT;
    static_assert(PER * R <= 16, "block_fft needs NT >= N/16 threads");
    constexpr bool PAIRED = (PER % 2 == 0) && (NB % (NT * PER) == 0);
    float2 v[PER][R];
    if constexpr (PAIRED) {
#pragma unroll
        for (int b = 0; b < PER; b += 2) {
            const int j = tid * PER + b;
#pragma unroll
            for (int r = 0; r < R; r++) {
                const float4 two = *reinterpret_cast<const float4*>(s + fft_pad(j + r * NB));
                v[b][r] = make_float2(two.x, two.y); v[b + 1][r] = make_float2(two.z, two.w);
            }
            fft_butterfly<N, R, NS, INV>(v[b], j, tw);
            fft_butterfly<N, R, NS, INV>(v[b + 1], j + 1, tw);
        }
        __syncthreads();                                                // every read of s has happened: the buffer is free again
#pragma unroll
        for (int b = 0; b < PER; b += 2) {
            const int j = tid * PER + b;
#pragma unroll
            for (int r = 0; r < R; r++) out.store2(j + r * NS, v[b][r], v[b + 1][r]);     // elements (i, i+1), i even
        }
    } else {
#pragma unroll
        for (int b = 0; b < PER; b++) {
            const int j = tid + b * NT;
            if (NB % NT == 0 || j < NB) {
#pragma unroll
                for (int r = 0; r < R; r++) v[b][r] = s[fft_pad(j + r * NB)];
                fft_butterfly<N, R, NS, INV>(v[b], j, tw);
            }
        }
        __syncthreads();
#pragma unroll
        for (int b = 0; b < PER; b++) {
            const int j = tid + b * NT;
            if (NB % NT == 0 || j < NB) {
#pragma unroll
                for (int r = 0; r < R; r++) out.store(j + r * NS, v[b][r]);
            }
        }
    }
}

// fft_pass_last with the thread's compile-time slot handed to the sink: out.slot(b, r, i, v) gets butterfly b, leg r (i = j(b) + r*N/8), so a sink can
// keep per-element data it fetched EARLIER (before the middle passes) in registers indexed [b][r] -- out.prefetch() is the caller's business.
template <int N, int NT, bool INV, typename Out>
__device__ __forceinline__ void fft_pass_last_slots(float2* __restrict__ s, const float2* __restrict__ tw, int tid, Out& out)
{
    constexpr int R = 8, NB = N / 8, NS = N / 8;
    constexpr int PER = (NB + NT - 1) / NT;
    static_assert(PER * R <= 16, "block_fft needs NT >= N/16 threads");
    static_assert(NB % NT == 0, "slot sinks want every slot populated");
    float2 v[PER][R];
#pragma unroll
    for (int b = 0; b < PER; b++) {
        const int j = tid + b * NT;
#pragma unroll
        for (int r = 0; r < R; r++) v[b][r] = s[fft_pad(j + r * NB)];
        fft_butterfly<N, R, NS, INV>(v[b], j, tw);
    }
    __syncthreads();
#pragma unroll
    for (int b = 0; b < PER; b++) {
        const int j = tid + b * NT;
#pragma unroll
        for (int r = 0; r < R; r++) out.slot(b, r, j + r * NS, v[b][r]);
    }
}

template <int N, int NT, int NS, bool INV>
__device__ __forceinline__ void fft_r8_middle_passes(float2* __restrict__ s, const float2* __restrict__ tw, int tid)
{
    if constexpr (NS * 8 < N) {                                         // stop before the last pass
        fft_pass<N, NT, 8, NS, INV>(s, tw, tid);
        fft_r8_middle_passes<N, NT, NS * 8, INV>(s, tw, tid);
    }
}

constexpr int fft_first_radix(int n) { return ilog2_c(n) % 3 == 1 ? 2 : (ilog2_c(n) % 3 == 2 ? 4 : 8); }

// N-point transform in.load(i) -> out.store(i); `s` (fft_smem_elems(N) slots) is scratch only.  All NT threads must call.
template <int N, int NT, bool INV, typename In, typename Out>
__device__ __forceinline__ void block_fft_io(float2* __restrict__ s, const float2* __restrict__ tw, int tid, In& in, Out& out)
{
    static_assert((N & (N - 1)) == 0 && N >= 2, "power of two sizes only");
    constexpr int R0 = fft_first_radix(N);
    if constexpr (R0 == N) {                                            // 2, 4, 8 points: one butterfly, no shared memory at all
        if (tid == 0) {
            float2 v[R0];
#pragma unroll
            for (int r = 0; r < R0; r++) v[r] = in.load(r);
            dft_small<R0, INV>(v);
#pragma unroll
            for (int r = 0; r < R0; r++) out.store(r, v[r]);
        }
    } else {
        fft_pass_first<N, NT, R0, INV>(s, tid, in);
        fft_r8_middle_passes<N, NT, R0, INV>(s, tw, tid);
        fft_pass_last<N, NT, INV>(s, tw, tid, out);
    }
}

// Prologue copy global -> padded shared array.  All of a thread's loads are issued before the first store: a load-then-store loop
// serialises one DRAM round trip per element (16 for the 4096-point kernel).
template <int N, int NT, typename Fetch>
__device__ __forceinline__ void fft_stage_in(float2* __restrict__ s, int tid, Fetch fetch)
{
    constexpr int PER = (N + NT - 1) / NT;
    float2 t[PER];
#pragma unroll
    for (int k = 0; k < PER; k++) { const int i = tid + k * NT; t[k] = (N % NT == 0 || i < N) ? fetch(i) : make_float2(0.f, 0.f); }
#pragma unroll
    for (int k = 0; k < PER; k++) { const int i = tid + k * NT; if (N % NT == 0 || i < N) s[fft_pad(i)] = t[k]; }
}
// 128-bit variant for 16-byte aligned, fully dense rows (two samples per load; N >= 2*NT)
template <int N, int NT>
__device__ __forceinline__ void fft_stage_in_vec(float2* __restrict__ s, int tid, const float2* __restrict__ x)
{
    constexpr int PER = N / (2 * NT);
    float4 t[PER];
#pragma unroll
    for (int k = 0; k < PER; k++) t[k] = __ldg(reinterpret_cast<const float4*>(x) + tid + k * NT);
#pragma unroll
    for (int k = 0; k < PER; k++) *reinterpret_cast<float4*>(s + fft_pad(2 * (tid + k * NT))) = t[k];
}

// which butterflies the last pass (radix 8, N/8 butterflies) gives to thread `tid`: slot b -> butterfly index j
template <int N, int NT> struct FftLastPass {
    static constexpr int NB = N / 8;
    static constexpr int PER = (NB + NT - 1) / NT;
    static constexpr bool PAIRED = (PER % 2 == 0) && (NB % (NT * PER) == 0);
    static constexpr bool GUARD = !(NB % NT == 0 || PAIRED);           // some slots fall beyond the transform
    __device__ static __forceinline__ int j(int tid, int b) { return PAIRED ? tid * PER + b : tid + b * NT; }
};

// Last pass of a forward transform, a pointwise map, and the first pass of the inverse transform of the same size in one go, for
// sizes whose first pass is radix 8 (8^k): the thread that finishes elements j + r*N/8 of the spectrum is the thread that needs them.
//   map.at(b, r, i, v) -> the value of element i of the inverse transform's input (e.g. spectrum * taps_fft); (b, r) is the thread's
//   compile-time slot of that element (butterfly b, leg r: i = fft_last_pass_j(tid, b) + r*N/8), so a map can keep per-element data
//   in registers; map.prefetch(b, r, i) is called for every slot before the pass starts so that those loads overlap the butterflies.
//   map.any(i, v): the same without a slot (sizes that hand over through shared memory).
template <int N, int NT, typename Map>
__device__ __forceinline__ void fft_chain_fwd_last_inv_first(float2* __restrict__ s, const float2* __restrict__ tw, int tid, Map& map)
{
    static_assert(fft_first_radix(N) == 8 && N >= 64, "register hand-over needs radix 8 at both ends");
    constexpr int R = 8, NB = N / 8, NS = N / 8;
    constexpr int PER = (NB + NT - 1) / NT;
    static_assert(PER * R <= 16, "block_fft needs NT >= N/16 threads");
    constexpr bool PAIRED = (PER % 2 == 0) && (NB % (NT * PER) == 0);
    float2 v[PER][R];
#pragma unroll
    for (int b = 0; b < PER; b++) {                                     // let the map start fetching its per-element data (global/L2 latency
        const int j = PAIRED ? tid * PER + b : tid + b * NT;            // hides behind the butterflies below)
        if (NB % NT == 0 || PAIRED || j < NB) {
#pragma unroll
            for (int r = 0; r < R; r++) map.prefetch(b, r, j + r * NS);
        }
    }
    if constexpr (PAIRED) {
#pragma unroll
        for (int b = 0; b < PER; b += 2) {
            const int j = tid * PER + b;
#pragma unroll
            for (int r = 0; r < R; r++) {
                const float4 two = *reinterpret_cast<const float4*>(s + fft_pad(j + r * NB));
                v[b][r] = make_float2(two.x, two.y); v[b + 1][r] = make_float2(two.z, two.w);
            }
            fft_butterfly<N, R, NS, false>(v[b], j, tw);
            fft_butterfly<N, R, NS, false>(v[b + 1], j + 1, tw);
        }
        __syncthreads();                                                // reads of s done
#pragma unroll
        for (int b = 0; b < PER; b++) {
            const int j = tid * PER + b;
#pragma unroll
            for (int r = 0; r < R; r++) v[b][r] = map.at(b, r, j + r * NS, v[b][r]);    // b, r are compile-time after unrolling
            dft8<true>(v[b]);                                           // inverse transform, first pass: inputs j + r*NB, no twiddles
        }
#pragma unroll
        for (int b = 0; b < PER; b += 2) {
            const int j = tid * PER + b;
#pragma unroll
            for (int r = 0; r < R; r += 2) {
                *reinterpret_cast<float4*>(s + fft_pad(j * R + r)) = make_float4(v[b][r].x, v[b][r].y, v[b][r + 1].x, v[b][r + 1].y);
                *reinterpret_cast<float4*>(s + fft_pad((j + 1) * R + r)) = make_float4(v[b + 1][r].x, v[b + 1][r].y, v[b + 1][r + 1].x, v[b + 1][r + 1].y);
            }
        }
    } else {
#pragma unroll
        for (int b = 0; b < PER; b++) {
            const int j = tid + b * NT;
            if (NB % NT == 0 || j < NB) {
#pragma unroll
                for (int r = 0; r < R; r++) v[b][r] = s[fft_pad(j + r * NB)];
                fft_butterfly<N, R, NS, false>(v[b], j, tw);
            }
        }
        __syncthreads();
#pragma unroll
        for (int b = 0; b < PER; b++) {
            const int j = tid + b * NT;
            if (NB % NT == 0 || j < NB) {
#pragma unroll
                for (int r = 0; r < R; r++) v[b][r] = map.at(b, r, j + r * NS, v[b][r]);
                dft8<true>(v[b]);
#pragma unroll
                for (int r = 0; r < R; r++) s[fft_pad(j * R + r)] = v[b][r];
            }
        }
    }
    __syncthreads();                                                    // first inverse pass visible
}

// FFT_N(in) -> map -> IFFT_N -> out (unnormalised), `s` is scratch.  Register hand-over in the middle when N is a power of 8.
template <int N, int NT, typename In, typename Map, typename Out>
__device__ __forceinline__ void block_fft_map_ifft(float2* __restrict__ s, const float2* __restrict__ tw, int tid, In& in, Map& map, Out& out)
{
    constexpr int R0 = fft_first_radix(N);
    static_assert(N >= 16, "use two block_fft_io calls for tiny sizes");
    fft_pass_first<N, NT, R0, false>(s, tid, in);
    fft_r8_middle_passes<N, NT, R0, false>(s, tw, tid);
    if constexpr (R0 == 8) {
        fft_chain_fwd_last_inv_first<N, NT>(s, tw, tid, map);
    } else {
        struct ToShared {                                               // last forward pass writes map(spectrum) back into s ...
            float2* s; Map& map;
            __device__ __forceinline__ void store(int i, float2 v) const { s[fft_pad(i)] = map.any(i, v); }
            __device__ __forceinline__ void store2(int i, float2 a, float2 b) const
            {
                const float2 ma = map.any(i, a), mb = map.any(i + 1, b);
                *reinterpret_cast<float4*>(s + fft_pad(i)) = make_float4(ma.x, ma.y, mb.x, mb.y);
            }
        } mid{s, map};
        fft_pass_last<N, NT, false>(s, tw, tid, mid);
        __syncthreads();
        fft_pass<N, NT, R0, 1, true>(s, tw, tid);                      // ... and the inverse starts from shared memory
    }
    fft_r8_middle_passes<N, NT, R0, true>(s, tw, tid);
    fft_pass_last<N, NT, true>(s, tw, tid, out);
}

// dense global rows as transform input / output; 128-bit accesses when the row is 16-byte aligned
struct FftRowIn {
    const float2* x; bool vec;
    __device__ __forceinline__ explicit FftRowIn(const float2* p) : x(p), vec((reinterpret_cast<uintptr_t>(p) & 15) == 0) {}
    __device__ __forceinline__ float2 load(int i) const { return __ldg(x + i); }
    __device__ __forceinline__ float4 load2(int i) const
    {
        if (vec) return __ldg(reinterpret_cast<const float4*>(x + i));
        const float2 a = __ldg(x + i), b = __ldg(x + i + 1);
        return make_float4(a.x, a.y, b.x, b.y);
    }
};
struct FftRowOut {
    float2* y; bool vec;
    __device__ __forceinline__ explicit FftRowOut(float2* p) : y(p), vec((reinterpret_cast<uintptr_t>(p) & 15) == 0) {}
    __device__ __forceinline__ void store(int i, float2 v) const { y[i] = v; }
    __device__ __forceinline__ void store2(int i, float2 a, float2 b) const
    {
        if (vec) *reinterpret_cast<float4*>(y + i) = make_float4(a.x, a.y, b.x, b.y);
        else { y[i] = a; y[i + 1] = b; }
    }
};

// host: the three twiddle planes (w^1, w^2, w^4) of an n-point transform, 3*n entries; a radix-8 pass over sub-size NS reads index
// NS + k, k < NS.  Angles in double, rounded once to float.
inline void fft_fill_twiddles(int n, float2* h)
{
    for (long i = 0; i < 3L * n; i++) h[i] = make_float2(1.f, 0.f);
    int lg = 0; while ((1 << lg) < n) lg++;
    int ns = lg % 3 == 1 ? 2 : (lg % 3 == 2 ? 4 : 1);
    if (ns == 1) ns = 8;                                                // the first pass (NS = 1) needs no twiddles
    for (; ns < n; ns *= 8)
        for (int k = 0; k < ns; k++)
            for (int c = 0; c < 3; c++) {
                const double a = -2.0 * 3.14159265358979323846 * (double)((1 << c) * k) / (double)(ns * 8);
                h[(size_t)c * n + ns + k] = make_float2((float)cos(a), (float)sin(a));
            }
}

constexpr int fft_threads(int n) { return n / 16 < 32 ? 32 : n / 16; }
constexpr int FFT_MAX_N = 16384;
// every size of the single-CTA transforms, for the launchers' switches
#define CSDRB_FFT_SIZES(X) X(2) X(4) X(8) X(16) X(32) X(64) X(128) X(256) X(512) X(1024) X(2048) X(4096) X(8192) X(16384)

}  // namespace csdrb
