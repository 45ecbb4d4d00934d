// ddc_bank.cu -- fused shared-input DDC / NFM bank (BASELINE config 4):
//     shift_addition_cc(rate_c)  ->  fir_decimate_cc(D, taps)  ->  [fmdemod_quadri_cf]        for C channels of ONE wideband stream
// i.e. what ddcd_old.h:51-57 runs as one `csdr shift_addition_cc --fd N | csdr fir_decimate_cc D bw` process chain per client.
//
// Mapping: LANE = CHANNEL.  All 32 lanes of a warp walk the same wideband samples in the same order, so
//   * the wideband sample is one broadcast load per warp (shared input: 8 B per sample, L1/L2 resident),
//   * the FIR tap for sample n and output o is the same for every lane -> taps live in uniform registers
//     (kernel parameter, duplicated (h,h) for FFMA pair), exactly like the independent-input bank kernel,
//   * each lane keeps its own NCO phasor (the reference's float recursion, re-seeded at every chunk boundary from the
//     replayed float phase chain) and its own M = ceil(T/D) running output accumulators in registers.
// Per wideband sample and channel: 4 flop rotation + 6 flop recursion + 2*M FFMA pair lanes; nothing goes through shared memory,
// the shifted stream never exists in HBM (the unfused chain writes and re-reads 8*C bytes per wideband sample).
// A warp owns a time segment of SEG outputs (plus M-1 trailing periods to finish its last outputs); segments are independent
// because the phasor of any sample depends only on its chunk's seed and its position inside the chunk.
//
// The float phase chain is a separate one-thread-per-channel pre-pass.  Folding it into this kernel as a ticketed producer CTA was
// tried and was slower: the whole grid is resident at once, so every segment needs
// its chunk phase at t = 0 and nothing overlaps, while the producer runs several times slower on a shared SM.  The remaining lever is to run the
// pre-pass of block k+1 on a side stream during the main kernel of block k (it only depends on the previous pre-pass).
//
// Bound: FP32 issue (SURVEY 8(d) cfg4): ~ (10 + 4*M) FMA-lane slots per (sample, channel).
#include "common.cuh"
#include "phase_table.cuh"
#include "kernels.h"
#include <cstdlib>
#include <type_traits>

namespace csdrb {

template <int TPAD>
struct alignas(16) DdcTaps { float4 hh2[TPAD / 2]; };               // rows of MP = M rounded up to even; one float4 = taps (j, j+1), each duplicated (h,h)

#define FMDEMOD_K_D 0.340447550238101026565118445432744920253753662109375

__device__ __forceinline__ float quadri_d(float2 cur, float2 prev)
{
    const float dq = __fsub_rn(cur.y, prev.y), di = __fsub_rn(cur.x, prev.x);
    const float num = __fsub_rn(__fmul_rn(cur.x, dq), __fmul_rn(cur.y, di));
    const float den = __fadd_rn(__fmul_rn(cur.x, cur.x), __fmul_rn(cur.y, cur.y));
    return den != 0.f ? (float)(FMDEMOD_K_D * (double)num / (double)den) : 0.f;
}

// seeds: (cos, sin) of every chunk's starting phase, evaluated in double like the reference does at each call
__global__ void ddc_seed_kernel(const float* __restrict__ chunk_phase, float2* __restrict__ seeds, long total)
{
    const long i = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const double ph = (double)chunk_phase[i];
    seeds[i] = make_float2((float)cos(ph), (float)sin(ph));
}

// phase chain over ABSOLUTE chunks: the block starts `offset` samples into chunk 0; phase_io holds the phase at the start of
// chunk 0 on entry and, on return, the phase at the start of the chunk that contains sample `advance` (the next block's start).
// Every step adds the same increment, so the wrap is a table lookup (phase_table.cuh): ~150 dependent cycles per chunk instead of ~1 200.
// One WARP per channel: lane 0 builds the table (32 different control flows in one warp would serialise), the chain itself keeps the table in
// registers across the lanes (wrap_after_add_warp) and stores 32 chunk phases at a time.
__global__ void __launch_bounds__(32)
ddc_wrap_tables_kernel(const float3* __restrict__ params, int chunk, WrapTable* __restrict__ tables, int channels)
{
    const int c = blockIdx.x;
    if (c < channels && threadIdx.x == 0) wrap_table_build(__fmul_rn(__fmul_rn(params[c].z, 3.14159265358979323846f), (float)chunk), tables + c);
}

// One warp walks DDC_CHAIN_CPW channels (1: more than one per warp does not interleave -- the wrap's branches and votes keep the chains in program order,
// as on the fastddc and shift chains).
constexpr int DDC_CHAIN_CPW = 1;
constexpr int DDC_CHAIN_WARPS = 1;                 // chains per CTA.  The pre-pass of block k+1 runs NEXT TO block k's main kernel, whose three CTAs leave ~10 K registers per SM: a one-warp
                                                   // CTA slips in, an eight-warp CTA has to wait for an SM to drain and the pre-pass serialises behind the main kernel

__global__ void __launch_bounds__(32 * DDC_CHAIN_WARPS)
ddc_phase_chain_kernel(const float3* __restrict__ params, float* __restrict__ phase_io, float* __restrict__ chunk_phase,
                       int channels, int nchunks, int chunk, int next_chunk, const WrapTable* __restrict__ tables)
{
    const int c0 = (blockIdx.x * DDC_CHAIN_WARPS + (threadIdx.x >> 5)) * DDC_CHAIN_CPW, lane = threadIdx.x & 31;
    if (c0 >= channels) return;
    const int nc = min(DDC_CHAIN_CPW, channels - c0);
    float inc[DDC_CHAIN_CPW], ph[DDC_CHAIN_CPW], keep[DDC_CHAIN_CPW], mine[DDC_CHAIN_CPW];
    WrapLanes w[DDC_CHAIN_CPW];
#pragma unroll
    for (int i = 0; i < DDC_CHAIN_CPW; i++) {
        const int c = min(c0 + i, channels - 1);                        // slots past the bank shadow its last channel (they compute, they do not store)
        inc[i] = __fmul_rn(__fmul_rn(params[c].z, 3.14159265358979323846f), (float)chunk);
        w[i] = wrap_lanes_load(tables + c, lane);
        ph[i] = phase_io[c]; keep[i] = ph[i]; mine[i] = 0.f;
    }
    __syncwarp();                                      // every lane has read the carried phases before lane 0 overwrites them
    for (int k = 0; k < nchunks; k++) {
        if ((k & 31) == lane) {
#pragma unroll
            for (int i = 0; i < DDC_CHAIN_CPW; i++) mine[i] = ph[i];
        }
        if (((k & 31) == 31 || k == nchunks - 1) && (k & ~31) + lane <= k) {                             // one coalesced store per channel and 32 steps
#pragma unroll
            for (int i = 0; i < DDC_CHAIN_CPW; i++) if (i < nc) chunk_phase[(long)(c0 + i) * nchunks + (k & ~31) + lane] = mine[i];
        }
        if (k == next_chunk) {
#pragma unroll
            for (int i = 0; i < DDC_CHAIN_CPW; i++) keep[i] = ph[i];
        }
#pragma unroll
        for (int i = 0; i < DDC_CHAIN_CPW; i++) ph[i] = wrap_after_add_warp(__fadd_rn(ph[i], inc[i]), w[i]);
    }
    if (next_chunk >= nchunks) {                       // the next block starts beyond the chunks this block touched
        for (int k = nchunks; k < next_chunk; k++) {
#pragma unroll
            for (int i = 0; i < DDC_CHAIN_CPW; i++) ph[i] = wrap_after_add_warp(__fadd_rn(ph[i], inc[i]), w[i]);
        }
#pragma unroll
        for (int i = 0; i < DDC_CHAIN_CPW; i++) keep[i] = ph[i];
    }
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < DDC_CHAIN_CPW; i++) if (i < nc) phase_io[c0 + i] = keep[i];
    }
}

// retune support: close the current chunk `n` samples in (every channel advances by n samples at its present rate), see csdrb_ddc_bank_process
__global__ void ddc_rechunk_kernel(const float3* __restrict__ params, float* __restrict__ phase_io, int channels, int n)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < channels) phase_io[c] = wrap_phase_pm_pi(__fadd_rn(phase_io[c], __fmul_rn(__fmul_rn(params[c].z, 3.14159265358979323846f), (float)n)));
}

// CPL = channels per lane.  A tap pair is loaded once per warp and sample phase (LDCU.128 fetches two of them: taps are stored
// [p][j] so the M taps that one sample meets are contiguous); with CPL = 2 every loaded tap feeds the FMAs of two channels and every
// wideband sample load feeds two channels, which halves the non-FMA issue slots per channel-sample (at CPL = 1 there is about one tap load per FMA pair).
template <int D, int M, int CPL, bool DEMOD>
__global__ void __launch_bounds__(128)
ddc_bank_fused_kernel(const float2* __restrict__ wide, int n_in, int offset, int chunk, int nchunks,
                      const float3* __restrict__ params, const float2* __restrict__ seeds, int channels,
                      void* __restrict__ out_v, long out_stride, int n_out, int seg_outputs,
                      const float2* __restrict__ last_in, float2* __restrict__ last_out,
                      const __grid_constant__ DdcTaps<D * ((M + 1) & ~1)> taps)
{
    constexpr int MP = (M + 1) & ~1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ch0 = (blockIdx.y * 4 + warp) * (32 * CPL) + lane;        // this lane's channels: ch0 + 32*u
    if (ch0 - lane >= channels) return;                                 // whole warp beyond the bank
    const int o_first = blockIdx.x * seg_outputs;                       // first output this warp emits
    if (o_first >= n_out) return;
    const int o_end = min(n_out, o_first + seg_outputs);
    // an output's window starts at its own first sample, so the walk can begin right at o_first (outputs before it are the
    // partial ones and are simply not emitted); the demodulator needs the previous baseband sample: start one output early.
    int o_start = o_first - (DEMOD ? 1 : 0);
    if (o_start < 0) o_start = 0;
    int chs[CPL]; bool live[CPL];
    float sind[CPL], cosd[CPL], c[CPL], s[CPL];
    float2 acc[CPL][M], prev[CPL];
    long n = (long)o_start * D;                                         // absolute chunk position = offset + n
    int kchunk = (int)((offset + n) / chunk);
    const int into = (int)((offset + n) % chunk);                       // samples already consumed in this chunk
#pragma unroll
    for (int u = 0; u < CPL; u++) {
        live[u] = ch0 + 32 * u < channels;
        chs[u] = live[u] ? ch0 + 32 * u : channels - 1;                 // dead lanes shadow a real channel (no divergence), never store
        const float3 p = params[chs[u]];
        sind[u] = p.x; cosd[u] = p.y;
#pragma unroll
        for (int j = 0; j < M; j++) acc[u][j] = make_float2(0.f, 0.f);
        prev[u] = (DEMOD && last_in) ? last_in[chs[u]] : make_float2(0.f, 0.f);
        const float2 cs = seeds[(long)chs[u] * nchunks + kchunk];
        c[u] = cs.x; s[u] = cs.y;
    }
    for (int t = 0; t < into; t++) {                                    // replay the recursion up to the segment start (< chunk steps, no data)
#pragma unroll
        for (int u = 0; u < CPL; u++) {
            const float cn = __fsub_rn(__fmul_rn(c[u], cosd[u]), __fmul_rn(s[u], sind[u]));
            const float sn = __fadd_rn(__fmul_rn(s[u], cosd[u]), __fmul_rn(c[u], sind[u]));
            c[u] = cn; s[u] = sn;
        }
    }
    int left = chunk - into;
    // acc[.][j] collects output q-j while the walk is in period q (samples qD .. qD+D-1): sample qD+p meets tap p + jD.
    for (int q = o_start; q < o_end + M - 1; q++) {
        const long base = (long)q * D;
        const bool inside = base + D <= n_in;                           // whole period inside the block: no per-load checks
        const float4* src = reinterpret_cast<const float4*>(wide + base);   // D even, base even: 16-byte aligned
#pragma unroll
        for (int pp = 0; pp < D; pp += 2) {
            float4 xx;                                                  // two wideband samples per 128-bit broadcast load
            if (inside) xx = __ldg(src + pp / 2);
            else {                                                      // samples past n_in only ever meet zero-padded taps: read as zeros
                const float2 a = base + pp < n_in ? wide[base + pp] : make_float2(0.f, 0.f);
                const float2 b = base + pp + 1 < n_in ? wide[base + pp + 1] : make_float2(0.f, 0.f);
                xx = make_float4(a.x, a.y, b.x, b.y);
            }
#pragma unroll
            for (int e = 0; e < 2; e++) {
                const int pidx = pp + e;
                const float xi = e ? xx.z : xx.x, xq = e ? xx.w : xx.y;
                if (left == 0) {                                        // chunk boundary: re-seed the phasors (warp-uniform branch)
                    if (kchunk < nchunks - 1) kchunk++;                 // (beyond the block the data are zeros; any phasor will do)
#pragma unroll
                    for (int u = 0; u < CPL; u++) { const float2 cs = seeds[(long)chs[u] * nchunks + kchunk]; c[u] = cs.x; s[u] = cs.y; }
                    left = chunk;
                }
                left--;
                float2 sh[CPL];
#pragma unroll
                for (int u = 0; u < CPL; u++) {
                    sh[u] = make_float2(fmaf(c[u], xi, -s[u] * xq), fmaf(s[u], xi, c[u] * xq));
                    const float cn = __fsub_rn(__fmul_rn(c[u], cosd[u]), __fmul_rn(s[u], sind[u]));
                    const float sn = __fadd_rn(__fmul_rn(s[u], cosd[u]), __fmul_rn(c[u], sind[u]));
                    c[u] = cn; s[u] = sn;
                }
#pragma unroll
                for (int j = 0; j < M; j += 2) {
                    const float4 h2 = taps.hh2[(pidx * MP + j) / 2];    // [p][j] layout, one 128-bit uniform load = two taps
#pragma unroll
                    for (int u = 0; u < CPL; u++) {
                        acc[u][j] = ffma2(sh[u], make_float2(h2.x, h2.y), acc[u][j]);
                        if (j + 1 < M) acc[u][j + 1] = ffma2(sh[u], make_float2(h2.z, h2.w), acc[u][j + 1]);
                    }
                }
            }
        }
        // period q done: output q-(M-1) is complete (its last tap block was j = M-1)
        const int o = q - (M - 1);
#pragma unroll
        for (int u = 0; u < CPL; u++) {
            const float2 y = acc[u][M - 1];
#pragma unroll
            for (int j = M - 1; j > 0; j--) acc[u][j] = acc[u][j - 1];
            acc[u][0] = make_float2(0.f, 0.f);
            if (o >= o_start) {
                if (DEMOD) {
                    if (o >= o_first && live[u]) static_cast<float*>(out_v)[(long)chs[u] * out_stride + o] = quadri_d(y, prev[u]);
                    prev[u] = y;
                    if (last_out && live[u] && o == n_out - 1) last_out[chs[u]] = y;
                } else if (o >= o_first && live[u]) {
                    static_cast<float2*>(out_v)[(long)chs[u] * out_stride + o] = y;
                }
            }
        }
    }
}


// ---- v2 (round 2): taps in shared memory, packed phasor arithmetic, ramp-aware tap ranges ---------------------------------------
// What the round-1 ncu profile of the kernel above showed: FMA pipe 29 %, issue 45 % -- neither saturated.  Three structural costs:
//  (1) every tap pair was an LDCU from a 7.2 KB kernel parameter walked once per period: far more than the uniform/constant L0 holds, so the
//      FFMA pair stream waited on constant-cache refills.  Here the CTA copies the taps once into shared memory ((h,h) pairs, [p][j] layout) and a
//      warp fetches two taps with one broadcast LDS.128 (one wavefront, 29-cycle fixed latency the compiler pipelines).
//  (2) rotation and recursion cost 10 scalar FMA-pipe slots per (sample, channel).  With the phasor kept twice, P = (c, s) and Q = (-s, c),
//          shifted = x.i * P + x.q * Q                        (FMUL pair + FFMA pair -- libcsdr_gpl.c:39-40 up to one fused product)
//          P'      = cosd * P + sind * Q                      (FMUL pair, FMUL pair, FADD, FADD: the reference's two rounded products and their sum, :42-45)
//          Q'      = (-P'.y, P'.x)                            (operand swizzle / negate modifiers of the packed instructions: free)
//      it is 6 slots; the phasor state stays bit-identical to the scalar sequence (negation commutes with rounding).
//  (3) a warp's time segment spends M-1 periods filling and M-1 periods draining its accumulators; with ~40-output segments that was a third of
//      all FFMA pair.  Here the head and tail periods only touch the accumulators that belong to emitted outputs, in groups of four taps
//      (template <JLO, JHI>), which removes ~80 % of that waste.
// Work decomposition: warp-granular 1-D grid; warp w owns (segment, channel set) = (w / sets, w % sets), a channel set = 32*CPL channels.
template <int D, int M, int CPL, bool DEMOD>
struct DdcWalk {
    static constexpr int MP = (M + 1) & ~1;
    float2 P[CPL], Q[CPL], cd2[CPL], sd2[CPL];
    float2 acc[CPL][MP];

    __device__ __forceinline__ void seed(int u, float2 cs)
    {
        P[u] = cs;
        Q[u] = make_float2(__uint_as_float(__float_as_uint(cs.y) ^ 0x80000000u), cs.x);
    }
    __device__ __forceinline__ void advance(int u)
    {
        // two rounded products and their rounded sum, as in the reference (the _rn helpers keep ptxas from fusing a product into the add)
        const float2 a = fmul2(P[u], cd2[u]), b = fmul2(Q[u], sd2[u]);
        const float2 pn = make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
        P[u] = pn;
        Q[u] = make_float2(__uint_as_float(__float_as_uint(pn.y) ^ 0x80000000u), pn.x);
    }
    // one wideband sample against the taps of its phase p (tp = taps of phase p, MP/2 float4), accumulators JLO..JHI-1 only
    // The taps come as SCALARS (two per 64-bit shared load) and multiply the I and the Q lane of the shifted sample: the tap operand is one register
    // for both channels of the lane, and four taps come with one 128-bit shared load (a copy duplicated (h, h) in shared memory needs twice the loads).
    template <int JLO, int JHI>
    __device__ __forceinline__ void sample(float xi, float xq, const float2* __restrict__ tp)
    {
        const float2 xi2 = make_float2(xi, xi), xq2 = make_float2(xq, xq);
        float2 sh[CPL];
#pragma unroll
        for (int u = 0; u < CPL; u++) {
            sh[u] = ffma2(P[u], xi2, fmul2(Q[u], xq2));             // one product rounded, the other fused (the data path has 1e-5 to spend; the phasor state has none)
            advance(u);
        }
#pragma unroll
        for (int j = JLO; j < JHI; j += 2) {
            const float2 h2 = tp[j / 2];
#pragma unroll
            for (int u = 0; u < CPL; u++) {
                acc[u][j] = ffma2(sh[u], make_float2(h2.x, h2.x), acc[u][j]);
                if (j + 1 < M) acc[u][j + 1] = ffma2(sh[u], make_float2(h2.y, h2.y), acc[u][j + 1]);
            }
        }
    }
};

template <int D, int M, int CPL, bool DEMOD>
__global__ void __launch_bounds__(128)
ddc_bank_fused2_kernel(const float2* __restrict__ wide, int n_in, int offset, int chunk, int nchunks,
                       const float3* __restrict__ params, const float2* __restrict__ seeds, int channels, int sets,
                       void* __restrict__ out_v, long out_stride, int n_out, int seg_outputs, int nsegs,
                       const float2* __restrict__ last_in, float2* __restrict__ last_out,
                       const __grid_constant__ DdcTaps<D * ((M + 1) & ~1)> taps)
{
    constexpr int MP = (M + 1) & ~1;
    constexpr int U = (D % 10 == 0) ? 10 : 2;                           // samples per unchecked group
    __shared__ float2 staps[D * MP / 2];                               // [p][j / 2] = taps (j, j+1) of phase p
    for (int i = threadIdx.x; i < D * MP / 2; i += 128) { const float4 hh = taps.hh2[i]; staps[i] = make_float2(hh.x, hh.z); }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const long wid = (long)blockIdx.x * 4 + (threadIdx.x >> 5);
    const int segi = (int)(wid / sets), set = (int)(wid % sets);
    if (segi >= nsegs) return;
    const int ch0 = set * (32 * CPL) + lane;
    const int o_first = segi * seg_outputs;
    if (o_first >= n_out) return;
    const int o_end = min(n_out, o_first + seg_outputs);
    int o_start = o_first - (DEMOD ? 1 : 0);                            // the discriminator needs the previous baseband sample
    if (o_start < 0) o_start = 0;

    DdcWalk<D, M, CPL, DEMOD> w;
    int chs[CPL]; bool live[CPL];
    float2 prev[CPL];
    const long n0 = (long)o_start * D;
    int kchunk = (int)((offset + n0) / chunk);
    const int into = (int)((offset + n0) % chunk);
#pragma unroll
    for (int u = 0; u < CPL; u++) {
        live[u] = ch0 + 32 * u < channels;
        chs[u] = live[u] ? ch0 + 32 * u : channels - 1;                 // dead lanes shadow a real channel (no divergence), never store
        const float3 p = params[chs[u]];
        w.sd2[u] = make_float2(p.x, p.x); w.cd2[u] = make_float2(p.y, p.y);
#pragma unroll
        for (int j = 0; j < MP; j++) w.acc[u][j] = make_float2(0.f, 0.f);
        prev[u] = (DEMOD && last_in) ? last_in[chs[u]] : make_float2(0.f, 0.f);
        w.seed(u, seeds[(long)chs[u] * nchunks + kchunk]);
    }
    for (int t = 0; t < into; t++) {                                    // replay the recursion up to the segment start (< chunk steps, no data)
#pragma unroll
        for (int u = 0; u < CPL; u++) w.advance(u);
    }
    int left = chunk - into;

    // one sample with the chunk-boundary and end-of-block checks (warp-uniform branches)
    auto checked = [&](auto jlo, auto jhi, long idx, int pidx) {
        if (left == 0) {
            if (kchunk < nchunks - 1) kchunk++;                         // (beyond the block the data are zeros; any phasor will do)
#pragma unroll
            for (int u = 0; u < CPL; u++) w.seed(u, seeds[(long)chs[u] * nchunks + kchunk]);
            left = chunk;
        }
        left--;
        const float2 x = idx < n_in ? __ldg(wide + idx) : make_float2(0.f, 0.f);   // samples past n_in only ever meet zero-padded taps
        w.template sample<decltype(jlo)::value, decltype(jhi)::value>(x.x, x.y, staps + pidx * (MP / 2));
    };
    // one period (D samples) restricted to accumulators [JLO, JHI)
    auto period = [&](auto jlo, auto jhi, int q) {
        constexpr int JLO = decltype(jlo)::value, JHI = decltype(jhi)::value;
        constexpr int UU = (JLO == 0 && JHI == MP) ? U : 2;             // the steady-state body is unrolled deeper than the ramps
        const long base = (long)q * D;
        // (fetching the next group's samples into registers while this one is multiplied was slower: the extra registers cost more
        // than the exposed L1 round trip)
#pragma unroll 1
        for (int p0 = 0; p0 < D; p0 += UU) {
            if (left >= UU && base + p0 + UU <= n_in) {
                const float4* src = reinterpret_cast<const float4*>(wide + base + p0);     // D, UU even: 16-byte aligned
                const float2* tp = staps + p0 * (MP / 2);
                float4 cur[UU / 2];
#pragma unroll
                for (int e = 0; e < UU / 2; e++) cur[e] = __ldg(src + e);
#pragma unroll
                for (int e = 0; e < UU; e += 2) {
                    const float4 xx = cur[e / 2];
                    w.template sample<JLO, JHI>(xx.x, xx.y, tp + e * (MP / 2));
                    w.template sample<JLO, JHI>(xx.z, xx.w, tp + (e + 1) * (MP / 2));
                }
                left -= UU;
            } else {
#pragma unroll 1
                for (int e = 0; e < UU; e++) checked(jlo, jhi, base + p0 + e, p0 + e);
            }
        }
    };
    // acc[.][j] collects output q-j while the walk is in period q (samples qD .. qD+D-1): sample qD+p meets tap p + jD.
    // Head: in period q only outputs >= o_start matter, i.e. j <= q - o_start.  Tail: only outputs < o_end, i.e. j >= q - o_end + 1.
    const int q_last = o_end + M - 2;
    for (int q = o_start; q <= q_last; q++) {
        const int need_hi = q - o_start + 1;                            // accumulators [0, need_hi) are live at the head
        const int need_lo = q - o_end + 1;                              // accumulators [need_lo, M) are live at the tail (<= 0: all)
        using I0 = std::integral_constant<int, 0>; using IM = std::integral_constant<int, MP>;
        if (need_hi <= 4 && 4 < MP) period(I0{}, std::integral_constant<int, 4>{}, q);
        else if (need_hi <= 8 && 8 < MP) period(I0{}, std::integral_constant<int, (8 < MP ? 8 : MP)>{}, q);
        else if (need_hi <= 12 && 12 < MP) period(I0{}, std::integral_constant<int, (12 < MP ? 12 : MP)>{}, q);
        else if (need_hi <= 16 && 16 < MP) period(I0{}, std::integral_constant<int, (16 < MP ? 16 : MP)>{}, q);
        else if (need_lo >= 16 && 16 < MP) period(std::integral_constant<int, (16 < MP ? 16 : 0)>{}, IM{}, q);
        else if (need_lo >= 12 && 12 < MP) period(std::integral_constant<int, (12 < MP ? 12 : 0)>{}, IM{}, q);
        else if (need_lo >= 8 && 8 < MP) period(std::integral_constant<int, (8 < MP ? 8 : 0)>{}, IM{}, q);
        else if (need_lo >= 4 && 4 < MP) period(std::integral_constant<int, (4 < MP ? 4 : 0)>{}, IM{}, q);
        else period(I0{}, IM{}, q);
        // period q done: output q-(M-1) is complete (its last tap block was j = M-1)
        const int o = q - (M - 1);
#pragma unroll
        for (int u = 0; u < CPL; u++) {
            const float2 y = w.acc[u][M - 1];
#pragma unroll
            for (int j = MP - 1; j > 0; j--) w.acc[u][j] = w.acc[u][j - 1];
            w.acc[u][0] = make_float2(0.f, 0.f);
            if (o >= o_start) {
                if (DEMOD) {
                    if (o >= o_first && live[u]) static_cast<float*>(out_v)[(long)chs[u] * out_stride + o] = quadri_d(y, prev[u]);
                    prev[u] = y;
                    if (last_out && live[u] && o == n_out - 1) last_out[chs[u]] = y;
                } else if (o >= o_first && live[u]) {
                    static_cast<float2*>(out_v)[(long)chs[u] * out_stride + o] = y;
                }
            }
        }
    }
}

size_t ddc_bank_scratch_bytes(int channels, int input_size, int chunk, int offset)
{
    if (chunk <= 0) chunk = input_size > 0 ? input_size : 1;
    const long nchunks = ((long)offset + input_size + chunk - 1) / chunk + 1;
    return (size_t)channels * (size_t)nchunks * (sizeof(float) + sizeof(float2)) + 64 + (size_t)channels * sizeof(WrapTable) + 16;
}
static inline size_t ddc_tables_offset(int channels, int nchunks)        // the per-call wrap tables sit behind the chunk phases and the seeds
{
    const size_t seeds_off = ((size_t)channels * nchunks * sizeof(float) + 15) & ~(size_t)15;
    return (seeds_off + (size_t)channels * nchunks * sizeof(float2) + 15) & ~(size_t)15;
}
int launch_ddc_rechunk(int channels, const float* d_params, float* d_phase_io, int n, cudaStream_t st)
{
    ddc_rechunk_kernel<<<(channels + 63) / 64, 64, 0, st>>>(reinterpret_cast<const float3*>(d_params), d_phase_io, channels, n);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}
size_t ddc_bank_tables_bytes(int channels) { return (size_t)channels * sizeof(WrapTable); }
int launch_ddc_tables(int channels, const float* d_params, int chunk, void* d_tables, cudaStream_t st)
{
    ddc_wrap_tables_kernel<<<channels, 32, 0, st>>>(reinterpret_cast<const float3*>(d_params), chunk, static_cast<WrapTable*>(d_tables), channels);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

template <int D, int M>
static int launch_fused(const float2* wide, int n_in, int offset, int chunk, int nchunks, const float3* params, const float2* seeds, int channels,
                        int demod, void* out, long out_stride, int n_out, const float2* last_in, float2* last_out, const float* h_taps, int T, cudaStream_t st)
{
    constexpr int MP = (M + 1) & ~1;
    DdcTaps<D * MP> tp;                                                 // tap k = jD + p stored at [p][j], duplicated for FFMA pair
    for (int p = 0; p < D; p++)
        for (int j = 0; j < MP; j++) {
            const int k = j * D + p; const float h = (j < M && k < T) ? h_taps[k] : 0.f;
            float4& slot = tp.hh2[(p * MP + j) / 2];
            if (j & 1) { slot.z = h; slot.w = h; } else { slot.x = h; slot.y = h; }
        }
    // tuning knobs: kernel generation (2 = shared-memory taps / packed phasor / ramp-aware, 1 = the round-1 kernel kept for A/B runs),
    // channels per lane and resident-warp target per SM
    static const int ver_env = getenv("CSDRB_DDC_V") ? atoi(getenv("CSDRB_DDC_V")) : 2;
    static const int cpl_env = getenv("CSDRB_DDC_CPL") ? atoi(getenv("CSDRB_DDC_CPL")) : (ver_env == 1 ? 1 : 2);
    static const int wps_env = getenv("CSDRB_DDC_WPS") ? atoi(getenv("CSDRB_DDC_WPS")) : (ver_env == 1 ? 24 : 12);
    const int cpl = cpl_env == 2 ? 2 : 1;
    const int warps_per_seg = (channels + 32 * cpl - 1) / (32 * cpl);
    // enough warps to fill the machine while keeping the M-1 trailing periods of every segment a small fraction
    long want_segments = (kSmCount * wps_env + warps_per_seg - 1) / warps_per_seg;
    int seg = (int)((n_out + want_segments - 1) / want_segments);
    if (seg < 2 * M) seg = 2 * M;
    const int nsegs = (n_out + seg - 1) / seg;
    if (ver_env != 1) {
        const long warps = (long)nsegs * warps_per_seg;
        const unsigned ctas = (unsigned)((warps + 3) / 4);
#define CSDRB_DDC_LAUNCH2(CPLV, DM) ddc_bank_fused2_kernel<D, M, CPLV, DM><<<ctas, 128, 0, st>>>(wide, n_in, offset, chunk, nchunks, params, seeds, channels, warps_per_seg, out, out_stride, n_out, seg, nsegs, last_in, last_out, tp)
        if (cpl == 2) { if (demod) CSDRB_DDC_LAUNCH2(2, true); else CSDRB_DDC_LAUNCH2(2, false); }
        else { if (demod) CSDRB_DDC_LAUNCH2(1, true); else CSDRB_DDC_LAUNCH2(1, false); }
#undef CSDRB_DDC_LAUNCH2
        CSDRB_CUDA(cudaGetLastError());
        return 0;
    }
    const int groups = (warps_per_seg + 3) / 4;
    dim3 grid(nsegs, groups);
#define CSDRB_DDC_LAUNCH(CPLV, DM) ddc_bank_fused_kernel<D, M, CPLV, DM><<<grid, 128, 0, st>>>(wide, n_in, offset, chunk, nchunks, params, seeds, channels, out, out_stride, n_out, seg, last_in, last_out, tp)
    if (cpl == 2) { if (demod) CSDRB_DDC_LAUNCH(2, true); else CSDRB_DDC_LAUNCH(2, false); }
    else { if (demod) CSDRB_DDC_LAUNCH(1, true); else CSDRB_DDC_LAUNCH(1, false); }
#undef CSDRB_DDC_LAUNCH
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}

// ---- the two halves of a block, exposed separately so a bank object can run the pre-pass of the NEXT block on a side stream ----
// pre-pass: float phase chain over the absolute chunks the block touches + the (cos, sin) seeds; advances d_phase_io to the chunk
// that contains the next block's first sample.
int launch_ddc_prepass(int input_size, int channels, const float* d_params, float* d_phase_io, int chunk, int offset, int decimation,
                       int taps_length, void* d_scratch, size_t scratch_bytes, const void* d_tables, cudaStream_t st)
{
    const int n_out = input_size >= taps_length ? (input_size - taps_length) / decimation + 1 : 0;
    if (n_out == 0) return 0;
    if (chunk <= 0) chunk = input_size;
    if (offset < 0 || offset >= chunk) { set_error("ddc bank: offset must be in [0, chunk)"); return -1; }
    if (scratch_bytes < ddc_bank_scratch_bytes(channels, input_size, chunk, offset) || !d_scratch) { set_error("ddc bank: scratch too small"); return -1; }
    const int nchunks = (int)(((long)offset + input_size + chunk - 1) / chunk) + 1;
    float* chunk_phase = static_cast<float*>(d_scratch);
    float2* seeds = reinterpret_cast<float2*>(static_cast<char*>(d_scratch) + (((size_t)channels * nchunks * sizeof(float) + 15) & ~(size_t)15));
    int launches = 2;
    if (!d_tables) {                                                    // no persistent tables (one-shot call): build them for this call
        void* tb = static_cast<char*>(d_scratch) + ddc_tables_offset(channels, nchunks);
        if (int rc = launch_ddc_tables(channels, d_params, chunk, tb, st); rc < 0) return rc;
        d_tables = tb; launches++;
    }
    const long advance = (long)n_out * decimation;                      // the next block starts here (the caller re-presents the tail)
    const int next_chunk = (int)((offset + advance) / chunk);
    ddc_phase_chain_kernel<<<(channels + DDC_CHAIN_CPW * DDC_CHAIN_WARPS - 1) / (DDC_CHAIN_CPW * DDC_CHAIN_WARPS), 32 * DDC_CHAIN_WARPS, 0, st>>>(reinterpret_cast<const float3*>(d_params), d_phase_io, chunk_phase, channels, nchunks, chunk, next_chunk,
                                                             static_cast<const WrapTable*>(d_tables));
    CSDRB_CUDA(cudaGetLastError());
    const long total = (long)channels * nchunks;
    ddc_seed_kernel<<<(int)((total + 255) / 256), 256, 0, st>>>(chunk_phase, seeds, total);
    CSDRB_CUDA(cudaGetLastError());
    return launches;
}

// main kernel: needs the seeds a matching launch_ddc_prepass() left in d_scratch
int launch_ddc_main(const float2* d_wide, int input_size, int channels, const float* d_params, int chunk, int offset, int decimation,
                    const float* h_taps, int taps_length, int demod, void* d_out, long out_stride, const float2* d_last_in, float2* d_last_out,
                    const void* d_scratch, cudaStream_t st)
{
    if (channels <= 0 || decimation <= 0 || taps_length <= 0) { set_error("ddc bank: bad geometry"); return -1; }
    const int n_out = input_size >= taps_length ? (input_size - taps_length) / decimation + 1 : 0;
    if (n_out == 0) return 0;
    if (chunk <= 0) chunk = input_size;
    if (reinterpret_cast<uintptr_t>(d_wide) & 15) { set_error("ddc bank: wideband input must be 16-byte aligned"); return -1; }
    const int nchunks = (int)(((long)offset + input_size + chunk - 1) / chunk) + 1;
    const float2* seeds = reinterpret_cast<const float2*>(static_cast<const char*>(d_scratch) + (((size_t)channels * nchunks * sizeof(float) + 15) & ~(size_t)15));
    int rc = -1;
    const float3* P = reinterpret_cast<const float3*>(d_params);
    if (decimation == 50 && taps_length <= 50 * 17) rc = launch_fused<50, 17>(d_wide, input_size, offset, chunk, nchunks, P, seeds, channels, demod, d_out, out_stride, n_out, d_last_in, d_last_out, h_taps, taps_length, st);
    else if (decimation == 10 && taps_length <= 10 * 8) rc = launch_fused<10, 8>(d_wide, input_size, offset, chunk, nchunks, P, seeds, channels, demod, d_out, out_stride, n_out, d_last_in, d_last_out, h_taps, taps_length, st);
    else if (decimation == 10 && taps_length <= 10 * 20) rc = launch_fused<10, 20>(d_wide, input_size, offset, chunk, nchunks, P, seeds, channels, demod, d_out, out_stride, n_out, d_last_in, d_last_out, h_taps, taps_length, st);
    else { set_error("ddc bank: no fused kernel for decimation %d / %d taps (compiled: d=50 T<=850, d=10 T<=200); run the unfused bank calls", decimation, taps_length); return -2; }
    return rc < 0 ? rc : n_out;
}

// one-shot: pre-pass and main kernel back to back on the caller's stream
int launch_ddc_bank(const float2* d_wide, int input_size, int channels, const float* d_params, float* d_phase_io, int chunk, int offset,
                    int decimation, const float* h_taps, int taps_length, int demod, void* d_out, long out_stride,
                    const float2* d_last_in, float2* d_last_out, void* d_scratch, size_t scratch_bytes, int* launches, cudaStream_t st)
{
    *launches = 0;
    if (channels <= 0 || decimation <= 0 || taps_length <= 0) { set_error("ddc bank: bad geometry"); return -1; }
    if (reinterpret_cast<uintptr_t>(d_wide) & 15) { set_error("ddc bank: wideband input must be 16-byte aligned"); return -1; }
    int rc = launch_ddc_prepass(input_size, channels, d_params, d_phase_io, chunk, offset, decimation, taps_length, d_scratch, scratch_bytes, nullptr, st);
    if (rc <= 0) return rc;
    const int pre = rc;
    rc = launch_ddc_main(d_wide, input_size, channels, d_params, chunk, offset, decimation, h_taps, taps_length, demod, d_out, out_stride, d_last_in, d_last_out, d_scratch, st);
    if (rc < 0) return rc;
    *launches = pre + 1;
    return rc;
}

}  // namespace csdrb
