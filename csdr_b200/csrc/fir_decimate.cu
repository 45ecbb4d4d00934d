// fir_decimate.cu -- K3: decimating FIR bank, real taps on complex (cf32) streams.
//
// Replaces reference fir_decimate_cc (libcsdr.c:528-549):
//     for (i = 0; i + T <= N; i += D) out[oi++] = sum_{k<T} in[i+k] * taps[k]      (I and Q separately)
// for C independent channels in one launch (the reference runs one process per channel).
//
// Fast path (D % 4 == 2, e.g. 10 and 50; T <= D*M): polyphase register tiling, no tensor cores.
//   * taps travel as a __grid_constant__ kernel parameter, duplicated (h,h) so that one FFMA pair
//     (fma.rn.f32x2) multiplies the I and Q of a sample by the same real tap; ptxas keeps them in
//     UNIFORM registers (LDCU -> UR operand of FFMA pair): no vector registers, no shared-memory traffic.
//   * the input tile is copied global->shared by ONE bulk async copy (cp.async.bulk, SASS UBLKCP)
//     completing on an mbarrier; the layout in shared memory is the plain stream order.
//   * a thread owns R consecutive outputs.  Writing tap index k = m*D + p (phase p, sub-tap m), its
//     outputs need x[(r+m)*D + p]: for one phase that is a contiguous-in-(r+m) window of R+M-1 samples,
//     each reused by up to min(R,M) FFMA pair.  Phases are taken in PAIRS (p, p+1) so every window element
//     is one 128-bit LDS.  With D/2 odd and R odd the lane stride R*D/2 (in 16-byte units) is odd, so
//     the eight lanes of a quarter-warp hit eight different 16-byte bank groups: conflict-free, no padding.
//   * the tap range is split in two halves across the two warps of a warp pair (more resident warps per
//     shared-memory byte); partial sums meet in a small shared buffer and leave as coalesced 128-bit stores.
//
// Generic path: any D, T (taps read from shared memory); correct but not tuned.
#include "common.cuh"
#include "kernels.h"

namespace csdrb {

template <int D, int M, int R, int NPAIR>
struct FirCfg {
    static_assert(D % 4 == 2, "fast path needs D = 2 (mod 4)");
    static_assert(R % 2 == 1, "fast path needs an odd number of outputs per thread");
    static_assert(M % 2 == 0, "sub-tap count is split across a warp pair");
    static constexpr int MG = M / 2;                         // sub-taps per warp of a pair
    static constexpr int WIN = R + MG - 1;                   // window length per phase
    static constexpr int TPAD = D * M;                       // taps, zero padded
    static constexpr int OUT_PAIR = 32 * R;                  // outputs per warp pair
    static constexpr int OUT_TILE = NPAIR * OUT_PAIR;        // outputs per CTA
    static constexpr int IN_TILE = OUT_TILE * D + (M - 1) * D;   // samples the tile reads (even)
    static constexpr int THREADS = NPAIR * 64;
    static constexpr size_t SMEM_IN = (size_t)IN_TILE * sizeof(float2);
    static constexpr size_t SMEM_RED = (size_t)OUT_TILE * sizeof(float2);
    static constexpr size_t SMEM_BYTES = SMEM_IN + SMEM_RED + 16;
    static constexpr size_t SMEM_LUT = SMEM_BYTES;                   // u8 front end only: 256 floats behind the mbarrier
    static constexpr size_t SMEM_BYTES_U8 = SMEM_BYTES + 256 * sizeof(float);
};

template <int TPAD>
struct FirTaps { float2 hh[TPAD]; };                         // (h,h) pairs, zero beyond taps_length


// One warp's share of the tap range: sub-taps [0, MG) of every phase, taps at hh[TAP0 + m*D + p].
template <int D, int MG, int R, int WIN, int TAP0>
__device__ __forceinline__ void fir_accumulate(const float2* __restrict__ base, const float2* __restrict__ hh, float2 (&acc)[R])
{
#pragma unroll
    for (int r = 0; r < R; r++) acc[r] = make_float2(0.f, 0.f);
#pragma unroll 1
    for (int pp = 0; pp < D / 2; pp++) {
        float4 w[WIN];
#pragma unroll
        for (int j = 0; j < WIN; j++) w[j] = *reinterpret_cast<const float4*>(base + j * D + 2 * pp);
#pragma unroll
        for (int m = 0; m < MG; m++) {
            const float2 ha = hh[TAP0 + m * D + 2 * pp], hb = hh[TAP0 + m * D + 2 * pp + 1];
#pragma unroll
            for (int r = 0; r < R; r++) {
                acc[r] = ffma2(make_float2(w[r + m].x, w[r + m].y), ha, acc[r]);
                acc[r] = ffma2(make_float2(w[r + m].z, w[r + m].w), hb, acc[r]);
            }
        }
    }
}

// U8 = true: the input is rtl_sdr-style unsigned 8-bit IQ (2 bytes per sample, what csdr-fm:41 feeds convert_u8_f) and the conversion of
// libcsdr.c:2363-2366 happens on the way into the tile: the bytes arrive by the same bulk copy (a quarter of the HBM / PCIe traffic of cf32)
// at the tail of the tile buffer, every thread pulls its share into registers, and after a barrier writes the floats over the whole buffer.
// The 256 possible values come from a table filled with the reference's own expression in double, so the samples the FIR sees are bit-identical
// to convert_u8_f's output.
template <int D, int M, int R, int NPAIR, int MINB, bool U8>
__global__ void __launch_bounds__(NPAIR * 64, MINB)
fir_bank_fast_kernel(const void* __restrict__ in_v, long in_stride, float2* __restrict__ out, long out_stride,
                     int n_in, int n_out, const __grid_constant__ FirTaps<D * M> taps)
{
    using C = FirCfg<D, M, R, NPAIR>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float2* xs = reinterpret_cast<float2*>(smem_raw);
    float2* red = reinterpret_cast<float2*>(smem_raw + C::SMEM_IN);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + C::SMEM_IN + C::SMEM_RED);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pair = warp >> 1, half = warp & 1;
    const int tile = blockIdx.x, ch = blockIdx.y;
    const long s0 = (long)tile * C::OUT_TILE * D;            // first input sample of the tile
    int valid = n_in - s0 < C::IN_TILE ? (int)(n_in - s0) : C::IN_TILE;   // samples that exist

    if (tid == 0) { mbar_init(bar, 1); mbar_fence_init(); }
    if constexpr (U8) {
        float* lut = reinterpret_cast<float*>(smem_raw + C::SMEM_LUT);
        for (int i = tid; i < 256; i += C::THREADS) lut[i] = (float)((double)(float)i / (255 / 2.0) - 1.0);     // libcsdr.c:2365, same promotions
    }
    __syncthreads();
    if constexpr (!U8) {
        const float2* src = static_cast<const float2*>(in_v) + (long)ch * in_stride + s0;
        const int bulk_n = valid & ~1;
        if (tid == 0) {
            mbar_arrive_expect_tx(bar, (uint32_t)bulk_n * 8u);
            if (bulk_n) bulk_g2s(xs, src, (uint32_t)bulk_n * 8u, bar);
        }
        for (int s = bulk_n + tid; s < C::IN_TILE; s += C::THREADS)         // ragged end of the stream: zero fill
            xs[s] = s < valid ? src[s] : make_float2(0.f, 0.f);
        mbar_wait(bar, 0);
        __syncthreads();
    } else {
        // 2 bytes per sample; tile starts are multiples of OUT_TILE*D samples = a multiple of 16 bytes, row strides are checked by the launcher
        const unsigned char* src = static_cast<const unsigned char*>(in_v) + ((long)ch * in_stride + s0) * 2;
        unsigned char* stage = smem_raw + (((size_t)C::IN_TILE * 6) & ~(size_t)15);   // the last quarter of the float tile, 16-byte aligned for the bulk copy
        const int bulk_b = (2 * valid) & ~15;
        if (tid == 0) {
            mbar_arrive_expect_tx(bar, (uint32_t)bulk_b);
            if (bulk_b) bulk_g2s(stage, src, (uint32_t)bulk_b, bar);
        }
        for (int b = bulk_b + tid; b < 2 * valid; b += C::THREADS) stage[b] = src[b];
        mbar_wait(bar, 0);
        __syncthreads();
        // two samples (four bytes) per step: one 32-bit shared load, four table look-ups, one 128-bit shared store
        static_assert(C::IN_TILE % 2 == 0, "the tile holds whole sample pairs");
        constexpr int PAIRS = C::IN_TILE / 2, PER = (PAIRS + C::THREADS - 1) / C::THREADS;
        const int vpairs = valid >> 1;                                        // whole pairs that exist (a trailing odd sample is handled below)
        unsigned v[PER];
        const float* lut = reinterpret_cast<const float*>(smem_raw + C::SMEM_LUT);
        if (valid == C::IN_TILE) {                                           // a whole tile (all but the last of a row): no per-element checks
#pragma unroll
            for (int k = 0; k < PER; k++) { const int i = tid + k * C::THREADS; if (PAIRS % C::THREADS == 0 || i < PAIRS) v[k] = reinterpret_cast<const unsigned*>(stage)[i]; }
            __syncthreads();                                                 // everyone holds its bytes: the floats may now overwrite the staging area
#pragma unroll
            for (int k = 0; k < PER; k++) {
                const int i = tid + k * C::THREADS;
                if (PAIRS % C::THREADS == 0 || i < PAIRS)
                    reinterpret_cast<float4*>(xs)[i] = make_float4(lut[v[k] & 0xffu], lut[(v[k] >> 8) & 0xffu], lut[(v[k] >> 16) & 0xffu], lut[v[k] >> 24]);
            }
        } else {
#pragma unroll
            for (int k = 0; k < PER; k++) { const int i = tid + k * C::THREADS; v[k] = i < vpairs ? reinterpret_cast<const unsigned*>(stage)[i] : 0u; }
            const unsigned short odd = (valid & 1) ? reinterpret_cast<const unsigned short*>(stage)[valid - 1] : (unsigned short)0;
            __syncthreads();
#pragma unroll
            for (int k = 0; k < PER; k++) {                                  // (unrolled: a dynamic index would push v[] into local memory for the fast path too)
                const int i = tid + k * C::THREADS;
                if (i < PAIRS) {
                    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (i < vpairs) o = make_float4(lut[v[k] & 0xffu], lut[(v[k] >> 8) & 0xffu], lut[(v[k] >> 16) & 0xffu], lut[v[k] >> 24]);
                    else if (i == vpairs && (valid & 1)) { o.x = lut[odd & 0xffu]; o.y = lut[odd >> 8]; }
                    reinterpret_cast<float4*>(xs)[i] = o;
                }
            }
        }
        __syncthreads();
    }

    // ---- polyphase accumulate -------------------------------------------------------------------
    // The branch on `half` is warp-uniform; inside each arm every tap index depends only on the loop
    // counter, so ptxas keeps the taps in uniform registers (LDCU) instead of per-lane LDC loads.
    float2 acc[R];
    const float2* base = xs + (pair * C::OUT_PAIR + lane * R + half * C::MG) * D;
    if (half == 0) fir_accumulate<D, C::MG, R, C::WIN, 0>(base, taps.hh, acc);
    else           fir_accumulate<D, C::MG, R, C::WIN, C::MG * D>(base, taps.hh, acc);

    // ---- combine the two tap halves, store coalesced --------------------------------------------
    float2* myred = red + pair * C::OUT_PAIR + lane * R;
    if (half == 1) {
#pragma unroll
        for (int r = 0; r < R; r++) myred[r] = acc[r];
    }
    named_bar_sync(1 + pair, 64);
    if (half == 0) {
#pragma unroll
        for (int r = 0; r < R; r++) myred[r] = fadd2(acc[r], myred[r]);
    }
    named_bar_sync(1 + pair, 64);
    const int o0 = tile * C::OUT_TILE + pair * C::OUT_PAIR;  // first output of this pair (even)
    float2* dst = out + (long)ch * out_stride + o0;
    const float2* rsrc = red + pair * C::OUT_PAIR;
    const int t64 = tid & 63;
    const int avail = n_out - o0;                            // outputs that exist from o0 on
    if (avail >= C::OUT_PAIR && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
        for (int v = t64; v < C::OUT_PAIR / 2; v += 64)
            st_na_f4(reinterpret_cast<float4*>(dst) + v, reinterpret_cast<const float4*>(rsrc)[v]);
    } else {
        for (int v = t64; v < C::OUT_PAIR && v < avail; v += 64) dst[v] = rsrc[v];
    }
}

// Generic path: one output at a time per thread, taps and input tile in shared memory.
__global__ void __launch_bounds__(256)
fir_bank_generic_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride,
                        int n_in, int n_out, int D, const float* __restrict__ taps, long taps_stride, int T,
                        int out_tile)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* ts = reinterpret_cast<float*>(smem_raw);
    float2* xs = reinterpret_cast<float2*>(smem_raw + (((size_t)T * 4 + 15) & ~(size_t)15));
    const int ch = blockIdx.y, o0 = blockIdx.x * out_tile;
    const int n_here = min(out_tile, n_out - o0);
    if (n_here <= 0) return;
    const long s0 = (long)o0 * D;
    const int span = (n_here - 1) * D + T;                   // always <= n_in - s0 by construction of n_out
    const float2* src = in + (long)ch * in_stride + s0;
    for (int s = threadIdx.x; s < span; s += blockDim.x) xs[s] = src[s];
    for (int k = threadIdx.x; k < T; k += blockDim.x) ts[k] = taps[(long)ch * taps_stride + k];
    __syncthreads();
    for (int o = threadIdx.x; o < n_here; o += blockDim.x) {
        const float2* x = xs + o * D;
        float ai = 0.f, aq = 0.f;
        for (int k = 0; k < T; k++) { float h = ts[k]; float2 v = x[k]; ai = fmaf(v.x, h, ai); aq = fmaf(v.y, h, aq); }
        out[(long)ch * out_stride + o0 + o] = make_float2(ai, aq);
    }
}

// ---- host launchers ------------------------------------------------------------------------------
template <int D, int M, int R, int NPAIR, int MINB, bool U8 = false>
static int launch_fast(const void* in, long in_stride, float2* out, long out_stride, int channels, int n_in,
                       int n_out, const float* h_taps, int T, cudaStream_t st)
{
    using C = FirCfg<D, M, R, NPAIR>;
    static_assert(!U8 || (C::OUT_TILE * D * 2) % 16 == 0, "u8 tiles must start on 16-byte boundaries");
    auto kern = fir_bank_fast_kernel<D, M, R, NPAIR, MINB, U8>;
    constexpr size_t smem = U8 ? C::SMEM_BYTES_U8 : C::SMEM_BYTES;
    // per call, not cached: the attribute is per device and a process may switch devices (it costs ~1 us)
    CSDRB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    FirTaps<D * M> tp;
    for (int k = 0; k < D * M; k++) { float h = k < T ? h_taps[k] : 0.f; tp.hh[k] = make_float2(h, h); }
    dim3 grid((n_out + C::OUT_TILE - 1) / C::OUT_TILE, channels);
    kern<<<grid, C::THREADS, smem, st>>>(in, in_stride, out, out_stride, n_in, n_out, tp);
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}

// rows of u8 IQ at any alignment -> cf32 rows (the front end of the two-launch path for geometries without a fused tiling): libcsdr.c:2365 per value
__global__ void __launch_bounds__(256)
u8_rows_to_cf32_kernel(const unsigned char* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride, int n)
{
    const unsigned char* src = in + (long)blockIdx.y * in_stride * 2;
    float2* dst = out + (long)blockIdx.y * out_stride;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        dst[i] = make_float2((float)((double)(float)src[2 * i] / (255 / 2.0) - 1.0), (float)((double)(float)src[2 * i + 1] / (255 / 2.0) - 1.0));
}
int launch_u8_rows_to_cf32(const unsigned char* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    int gx = (n + 255) / 256; if (gx > 1024) gx = 1024;
    u8_rows_to_cf32_kernel<<<dim3(gx, channels), 256, 0, st>>>(d_in, in_stride, d_out, out_stride, n);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// u8 IQ in (2 bytes per sample, row stride in samples, a multiple of 8 so that rows start on 16-byte boundaries), cf32 out: convert_u8_f | fir_decimate_cc
// in one kernel.  Returns outputs per channel, or -2 when (D, T) has no fused tiling -- the caller then converts and filters in two launches.
int launch_fir_decimate_bank_u8(const unsigned char* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n_in,
                                int D, const float* h_taps, int T, cudaStream_t st)
{
    if (channels <= 0 || D <= 0 || T <= 0 || !h_taps) { set_error("fir_decimate u8 bank: bad geometry (C=%d D=%d T=%d)", channels, D, T); return -1; }
    const int n_out = n_in >= T ? (n_in - T) / D + 1 : 0;
    if (n_out == 0) return 0;
    if ((reinterpret_cast<uintptr_t>(d_in) & 15) || (in_stride % 8)) return -2;
    int rc = -2;
    if (D == 10 && T <= 80) rc = launch_fast<10, 8, 15, 2, 3, true>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st);
    else if (D == 10 && T <= 200) rc = launch_fast<10, 20, 13, 2, 3, true>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st);
    else if (D == 50 && T <= 900) rc = launch_fast<50, 18, 3, 2, 2, true>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st);
    else return -2;
    return rc < 0 ? rc : n_out;
}

int fir_bank_variant_count() { return 8; }

// variant: -1 = automatic choice; >= 0 selects one of the compiled tilings (tuning / benchmarking hook)
int launch_fir_decimate_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n_in,
                             int D, const float* h_taps, const float* d_taps, long taps_stride, int T, int variant,
                             cudaStream_t st)
{
    if (channels <= 0 || D <= 0 || T <= 0) { set_error("fir_decimate bank: bad geometry (C=%d D=%d T=%d)", channels, D, T); return -1; }
    if (variant >= fir_bank_variant_count()) { set_error("fir_decimate bank: tiling %d does not exist (0..%d, or < 0 for the automatic choice)", variant, fir_bank_variant_count() - 1); return -1; }
    const int n_out = n_in >= T ? (n_in - T) / D + 1 : 0;
    if (n_out == 0) return 0;
    const bool aligned = ((reinterpret_cast<uintptr_t>(d_in) & 15) == 0) && (in_stride % 2 == 0);
    const bool shared_taps = (taps_stride == 0) && h_taps != nullptr;
    if (aligned && shared_taps && D == 10 && T <= 80 && variant < 0) {
        // the CLI default (fir_decimate_cc 10 0.05 -> 79 taps): 8 sub-taps per phase instead of 20 zero-padded ones
        const int rc = launch_fast<10, 8, 15, 2, 3>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st);
        return rc < 0 ? rc : n_out;
    }
    if (aligned && shared_taps && D == 10 && T <= 200) {
        int rc;
        switch (variant) {
            case 1:  rc = launch_fast<10, 20, 15, 2, 2>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st); break;
            case 2:  rc = launch_fast<10, 20, 15, 4, 1>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st); break;
            case 3:  rc = launch_fast<10, 20, 9, 4, 2>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st); break;
            case 4:  rc = launch_fast<10, 20, 13, 1, 5>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st); break;
            case 5:  rc = launch_fast<10, 20, 9, 2, 4>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st); break;
            case 6:  rc = launch_fast<10, 20, 11, 2, 3>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st); break;
            case 7:  rc = launch_fast<10, 20, 17, 2, 2>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st); break;
            default: rc = launch_fast<10, 20, 13, 2, 3>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st); break;
        }
        return rc < 0 ? rc : n_out;
    }
    if (aligned && shared_taps && D == 50 && T <= 900) {
        // fir_decimate_cc 50 0.005 (801 taps), independent inputs: 3 outputs per thread keep the tile (150 samples per thread) in shared memory
        const int rc = launch_fast<50, 18, 3, 2, 2>(d_in, in_stride, d_out, out_stride, channels, n_in, n_out, h_taps, T, st);
        return rc < 0 ? rc : n_out;
    }
    // generic
    if (!d_taps) { set_error("fir_decimate bank: generic path needs device taps"); return -1; }
    size_t tap_bytes = ((size_t)T * 4 + 15) & ~(size_t)15;
    int out_tile = (int)(((size_t)96 * 1024 - tap_bytes) / 8 - (size_t)T) / D;
    if (out_tile < 1) { set_error("fir_decimate bank: taps_length %d too long for the generic kernel", T); return -1; }
    if (out_tile > 2048) out_tile = 2048;
    size_t smem = tap_bytes + ((size_t)(out_tile - 1) * D + T) * 8;
    CSDRB_CUDA(cudaFuncSetAttribute(fir_bank_generic_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    dim3 grid((n_out + out_tile - 1) / out_tile, channels);
    fir_bank_generic_kernel<<<grid, 256, smem, st>>>(d_in, in_stride, d_out, out_stride, n_in, n_out, D, d_taps, taps_stride, T, out_tile);
    CSDRB_CUDA(cudaGetLastError());
    return n_out;
}

}  // namespace csdrb
