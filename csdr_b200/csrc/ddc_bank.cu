// ddc_bank.cu -- fused shared-input DDC / NFM bank (BASELINE config 4):
//     shift_addition_cc(rate_c)  ->  fir_decimate_cc(D, taps)  ->  [fmdemod_quadri_cf]        for C channels of ONE wideband stream
// i.e. what ddcd_old.h:51-57 runs as one `csdr shift_addition_cc --fd N | csdr fir_decimate_cc D bw` process chain per client.
//
// Mapping: LANE = CHANNELS.  All 32 lanes of a warp walk the same wideband samples in the same order, so
//   * the wideband sample is one broadcast load per warp (shared input: 8 B per sample, L1/L2 resident),
//   * the FIR tap for sample n and output o is the same for every lane -> the CTA copies the taps into shared memory once and
//     a warp reads them with broadcast loads,
//   * each lane carries kDdcChannelsPerLane channels, each with its own NCO phasor (the reference's float recursion, re-seeded at
//     every chunk boundary from the replayed float phase chain) and its own M = ceil(T/D) running output accumulators in registers.
// Per wideband sample and channel: 4 flop rotation + 6 flop recursion + 2*M FFMA pair lanes; the shifted stream never exists in HBM
// (the unfused chain writes and re-reads 8*C bytes per wideband sample).
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
struct alignas(16) DdcTaps { float2 h2[TPAD / 2]; };                // [p][j / 2] = taps (j, j+1) of phase p; rows of MP = M rounded up to even

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
// registers across the lanes (chain_walk_warp) and stores 32 chunk phases at a time.
__global__ void __launch_bounds__(32)
ddc_wrap_tables_kernel(const float3* __restrict__ params, int chunk, WrapTable* __restrict__ tables, int channels)
{
    const int c = blockIdx.x;
    if (c < channels && threadIdx.x == 0) wrap_table_build(phase_increment(params[c].z, chunk), tables + c);
}

// Chains per CTA.  The pre-pass of block k+1 runs NEXT TO block k's main kernel, whose three CTAs leave ~10 K registers per SM: a one-warp
// CTA slips in, an eight-warp CTA has to wait for an SM to drain and the pre-pass serialises behind the main kernel.
constexpr int kDdcChainWarps = 1;

__global__ void __launch_bounds__(32 * kDdcChainWarps)
ddc_phase_chain_kernel(const float3* __restrict__ params, float* __restrict__ phase_io, float* __restrict__ chunk_phase,
                       int channels, int nchunks, int chunk, int next_chunk, const WrapTable* __restrict__ tables)
{
    const int c = blockIdx.x * kDdcChainWarps + (threadIdx.x >> 5);
    if (c >= channels) return;
    const float inc = phase_increment(params[c].z, chunk);
    const WrapLanes w = wrap_lanes_load(tables + c, threadIdx.x & 31);
    float keep = 0.f;
    const float ph = chain_walk_warp(phase_io[c], inc, &w, nchunks, chunk_phase + (long)c * nchunks, [&](int k, float p) { if (k == next_chunk) keep = p; });
    if (next_chunk >= nchunks) keep = chain_walk_warp(ph, inc, &w, next_chunk - nchunks, nullptr);   // the next block starts beyond the chunks this block touched
    if ((threadIdx.x & 31) == 0) phase_io[c] = keep;
}

// retune support: close the current chunk `n` samples in (every channel advances by n samples at its present rate), see csdrb_ddc_bank_process
__global__ void ddc_rechunk_kernel(const float3* __restrict__ params, float* __restrict__ phase_io, int channels, int n)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < channels) phase_io[c] = phase_step(phase_io[c], phase_increment(params[c].z, n));
}

// ---- the bank kernel: taps in shared memory, packed phasor arithmetic, ramp-aware tap ranges ---------------------------------------
//  (1) The taps (7.2 KB at D = 50) are walked once per period: far more than the uniform/constant cache holds, so read from a kernel parameter the
//      FFMA pair stream would wait on constant-cache refills.  The CTA copies them once into shared memory ([p][j] layout) and a warp fetches
//      several taps with one broadcast shared load.
//  (2) With the phasor kept twice, P = (c, s) and Q = (-s, c), rotation and recursion are packed operations:
//          shifted = x.i * P + x.q * Q                        (FMUL pair + FFMA pair -- libcsdr_gpl.c:39-40 up to one fused product)
//          P'      = cosd * P + sind * Q                      (FMUL pair, FMUL pair, FADD, FADD: the reference's two rounded products and their sum, :42-45)
//          Q'      = (-P'.y, P'.x)                            (operand swizzle / negate modifiers of the packed instructions: free)
//      and the phasor state stays bit-identical to the scalar sequence (negation commutes with rounding).
//  (3) A warp's time segment spends M-1 periods filling and M-1 periods draining its accumulators; with ~40-output segments a full-width walk
//      would spend a third of all FFMA pair there.  The head and tail periods only touch the accumulators that belong to emitted outputs, in
//      groups of four taps (template <JLO, JHI>), which removes ~80 % of that waste.
// Work decomposition: warp-granular 1-D grid; warp w owns (segment, channel set) = (w / sets, w % sets), a channel set = 32*CPL channels.
// CPL = channels per lane: with two, every loaded tap and every wideband sample feeds the FMAs of two channels, which halves the non-FMA issue
// slots per channel-sample against one channel per lane.  CSDRB_DDC_CPL=1 selects one channel per lane (DESIGN.md 8b: faster on an H100).
constexpr int kDdcChannelsPerLane = 2;
// Resident warps per SM the launcher sizes its segments for: three 4-warp CTAs at the ~165 registers per thread of the D = 50 and D = 10 / 20-tap
// kernels.  Fewer, longer segments would leave SMs idle; more, shorter ones spend a larger share on the M-1 trailing periods of each.
constexpr int kDdcWarpsPerSm = 12;

// Every other even decimation runs ddc_bank_generic_kernel<M, CPL, DEMOD>: D is a kernel argument and M a compile-time bucket, the smallest of
// kDdcBuckets >= ceil(T/D) (the taps of the blocks past ceil(T/D) are zero).  17 is a bucket of its own because T = firdes_filter_len(0.25/D) =
// 16D +- 1 -- a transition band of a quarter of the output rate, config 4's ratio -- has M = 16 or 17 at every D.
constexpr int kDdcBuckets[] = {4, 8, 12, 17, 20, 24};
constexpr int kDdcMaxM = 24;
// The generic kernel takes its taps as one fixed-size kernel parameter (no device buffer: csdrb_ddc_bank takes host taps and its scratch size knows
// neither D nor T).  All parameters together must stay within 32 764 bytes, so D * MP <= 8000 taps.
constexpr int kDdcTapCapacity = 8000;
// 4-warp CTAs per SM of each generic bucket (__launch_bounds__ caps the registers so that many fit; DESIGN.md 8b lists the registers): the
// launcher sizes its segments for that many resident warps.
__host__ __device__ constexpr int ddc_generic_ctas_per_sm(int M, int cpl)
{
    return cpl == 1 ? (M <= 8 ? 6 : M <= 12 ? 5 : M <= 20 ? 4 : 3) : (M <= 4 ? 5 : M <= 8 ? 4 : M <= 17 ? 3 : 2);
}

template <int M, int CPL>
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
    // one wideband sample against the taps of its phase p (tp = taps of phase p, MP/2 float2), accumulators JLO..JHI-1 only
    // The taps come as SCALARS (two per 64-bit shared load) and multiply the I and the Q lane of the shifted sample: the tap operand is one register
    // for both channels of the lane, and four taps come with one 128-bit shared load (a copy duplicated (h, h) in shared memory needs twice the loads).
    // LIM >= 0 (the guarded form): only taps jD + p < T are applied, lim = T - p -- the zero-padded taps past T meet samples outside the
    // output's window [oD, oD + T), and fma(sh, 0, acc) is NaN for a non-finite sh where the reference, which never reads them, stays finite.
    // For a finite sh the skipped fma(sh, 0, acc) is acc, so both forms give the same bits; the walk takes the unguarded one only for samples
    // it has checked to be small enough for sh to stay finite.
    // The shifted sample: complex x is one product rounded and the other fused (the data path has 1e-5 to spend; the phasor state has none);
    // real x (shift_addition_fc, libcsdr_gpl.c:66-67) is P * x, one rounded product per component -- the value ffma2(P, x, Q * 0) would give up to
    // the sign of a zero, without its extra multiply.
    __device__ __forceinline__ float2 shifted(int u, float2 x) const
    {
        return ffma2(P[u], make_float2(x.x, x.x), fmul2(Q[u], make_float2(x.y, x.y)));
    }
    __device__ __forceinline__ float2 shifted(int u, float x) const { return fmul2(P[u], make_float2(x, x)); }

    template <int JLO, int JHI, bool GUARD = false, class X>
    __device__ __forceinline__ void sample(X x, const float2* __restrict__ tp, int lim = 0, int D = 0)
    {
        float2 sh[CPL];
#pragma unroll
        for (int u = 0; u < CPL; u++) {
            sh[u] = shifted(u, x);
            advance(u);
        }
#pragma unroll
        for (int j = JLO; j < JHI; j += 2) {
            const float2 h2 = tp[j / 2];
            const bool la = !GUARD || j * D < lim, lb = j + 1 < M && (!GUARD || (j + 1) * D < lim);
#pragma unroll
            for (int u = 0; u < CPL; u++) {
                if (la) acc[u][j] = ffma2(sh[u], make_float2(h2.x, h2.x), acc[u][j]);
                if (lb) acc[u][j + 1] = ffma2(sh[u], make_float2(h2.y, h2.y), acc[u][j + 1]);
            }
        }
    }
};

// The walk of one warp, shared by both bank kernels.  DC > 0: the decimation is the compile-time DC (ddc_bank_fused2_kernel); DC = 0: it is the
// run-time d_rt (ddc_bank_generic_kernel).  U = samples per unchecked group of a full-width period: a period runs groups of U while U samples are
// left and the rest in groups of 2 (DC is a multiple of U).  staps = the taps in shared memory, [p][j / 2] = taps (j, j+1) of phase p.
// TIn = float2: complex wideband samples (shift_addition_cc); TIn = float: real ones (shift_addition_fc), read two per 8-byte load.
template <int DC, int M, int CPL, bool DEMOD, int U, class TIn = float2>
__device__ __forceinline__ void ddc_bank_walk(const TIn* __restrict__ wide, int n_in, int offset, int chunk, int nchunks,
                                              const float3* __restrict__ params, const float2* __restrict__ seeds, int channels, int sets,
                                              void* __restrict__ out_v, long out_stride, int n_out, int seg_outputs, int nsegs,
                                              const float2* __restrict__ last_in, float2* __restrict__ last_out, int T, int d_rt, const float2* staps)
{
    constexpr int MP = (M + 1) & ~1;
    static_assert(MP <= 24, "the head and tail ramps below step in fours up to 20");
    static_assert(DC % U == 0 && U % 2 == 0, "groups of U samples tile a period");
    const int D = DC > 0 ? DC : d_rt;
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

    DdcWalk<M, CPL> w;
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
        const TIn x = idx < n_in ? __ldg(wide + idx) : TIn{};       // samples past n_in only ever meet zero-padded taps
        w.template sample<decltype(jlo)::value, decltype(jhi)::value, true>(x, staps + pidx * (MP / 2), T - pidx, D);
    };
    // one period (D samples) restricted to accumulators [JLO, JHI)
    auto period = [&](auto jlo, auto jhi, int q) {
        constexpr int JLO = decltype(jlo)::value, JHI = decltype(jhi)::value;
        constexpr int UU = (JLO == 0 && JHI == MP) ? U : 2;             // the steady-state body is unrolled deeper than the ramps
        const long base = (long)q * D;
        // samples p0 .. p0+G-1 of the period
        auto group = [&](auto g, int p0) {
            constexpr int G = decltype(g)::value;
            // (fetching the next group's samples into registers while this one is multiplied was slower: the extra registers cost more
            // than the exposed L1 round trip)
            if (left >= G && base + p0 + G <= n_in) {
                // two samples per load: D, p0 even, so 16-byte aligned for complex samples and 8-byte aligned for real ones
                using Pair = std::conditional_t<std::is_same_v<TIn, float>, float2, float4>;
                const Pair* src = reinterpret_cast<const Pair*>(wide + base + p0);
                const float2* tp = staps + p0 * (MP / 2);
                Pair cur[G / 2];
                float mag = 0.f;                                        // sum of |x.i| + |x.q| over the group: NaN, Inf or huge -> guarded path
#pragma unroll
                for (int e = 0; e < G / 2; e++) {
                    cur[e] = __ldg(src + e);
                    if constexpr (std::is_same_v<TIn, float>) mag += fabsf(cur[e].x) + fabsf(cur[e].y);
                    else mag += fabsf(cur[e].x) + fabsf(cur[e].y) + fabsf(cur[e].z) + fabsf(cur[e].w);
                }
                // |P|, |Q| stay near 1, so below 2^126 every shifted sample of the group is finite and the padded taps add exactly nothing
                if (mag < 0x1p126f) {
#pragma unroll
                    for (int e = 0; e < G; e += 2) {
                        const Pair xx = cur[e / 2];
                        if constexpr (std::is_same_v<TIn, float>) {
                            w.template sample<JLO, JHI>(xx.x, tp + e * (MP / 2));
                            w.template sample<JLO, JHI>(xx.y, tp + (e + 1) * (MP / 2));
                        } else {
                            w.template sample<JLO, JHI>(make_float2(xx.x, xx.y), tp + e * (MP / 2));
                            w.template sample<JLO, JHI>(make_float2(xx.z, xx.w), tp + (e + 1) * (MP / 2));
                        }
                    }
                    left -= G;
                    return;
                }
            }
#pragma unroll 1
            for (int e = 0; e < G; e++) checked(jlo, jhi, base + p0 + e, p0 + e);   // chunk boundary, block end or a group that failed the check
        };
        const int d_main = DC > 0 ? D : D - D % UU;
#pragma unroll 1
        for (int p0 = 0; p0 < d_main; p0 += UU) group(std::integral_constant<int, UU>{}, p0);
        if constexpr (DC == 0 && UU > 2) {
#pragma unroll 1
            for (int p0 = d_main; p0 < D; p0 += 2) group(std::integral_constant<int, 2>{}, p0);
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
        else if (need_hi <= 20 && 20 < MP) period(I0{}, std::integral_constant<int, (20 < MP ? 20 : MP)>{}, q);
        else if (need_lo >= 20 && 20 < MP) period(std::integral_constant<int, (20 < MP ? 20 : 0)>{}, IM{}, q);
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

// D = 50 and D = 10: the taps in static shared memory, groups of 10 samples when D allows
template <int D, int M, int CPL, bool DEMOD>
__global__ void __launch_bounds__(128)
ddc_bank_fused2_kernel(const float2* __restrict__ wide, int n_in, int offset, int chunk, int nchunks,
                       const float3* __restrict__ params, const float2* __restrict__ seeds, int channels, int sets,
                       void* __restrict__ out_v, long out_stride, int n_out, int seg_outputs, int nsegs,
                       const float2* __restrict__ last_in, float2* __restrict__ last_out, int T,
                       const __grid_constant__ DdcTaps<D * ((M + 1) & ~1)> taps)
{
    constexpr int MP = (M + 1) & ~1;
    __shared__ float2 staps[D * MP / 2];
    for (int i = threadIdx.x; i < D * MP / 2; i += 128) staps[i] = taps.h2[i];
    __syncthreads();
    ddc_bank_walk<D, M, CPL, DEMOD, (D % 10 == 0) ? 10 : 2>(wide, n_in, offset, chunk, nchunks, params, seeds, channels, sets, out_v, out_stride, n_out,
                                                            seg_outputs, nsegs, last_in, last_out, T, D, staps);
}

static_assert(sizeof(DdcTaps<kDdcTapCapacity>) + 160 <= 32764, "the generic kernel's parameters must fit the 32 764-byte parameter space");

// the generic kernels' body: the taps into `staps` (D * MP floats of dynamic shared memory), then the walk with D a run-time argument
template <int M, int CPL, bool DEMOD, class TIn>
__device__ __forceinline__ void ddc_generic_body(const TIn* __restrict__ wide, int n_in, int offset, int chunk, int nchunks,
                                                 const float3* __restrict__ params, const float2* __restrict__ seeds, int channels, int sets,
                                                 void* __restrict__ out_v, long out_stride, int n_out, int seg_outputs, int nsegs,
                                                 const float2* __restrict__ last_in, float2* __restrict__ last_out, int T, int D,
                                                 const DdcTaps<kDdcTapCapacity>& taps, float2* staps)
{
    constexpr int MP = (M + 1) & ~1;
    for (int i = threadIdx.x; i < D * MP / 2; i += 128) staps[i] = taps.h2[i];
    __syncthreads();
    ddc_bank_walk<0, M, CPL, DEMOD, 8, TIn>(wide, n_in, offset, chunk, nchunks, params, seeds, channels, sets, out_v, out_stride, n_out,
                                            seg_outputs, nsegs, last_in, last_out, T, D, staps);
}

// any even D: D * MP floats of taps in dynamic shared memory (at most 32 000 bytes, no opt-in needed)
template <int M, int CPL, bool DEMOD>
__global__ void __launch_bounds__(128, ddc_generic_ctas_per_sm(M, CPL))
ddc_bank_generic_kernel(const float2* __restrict__ wide, int n_in, int offset, int chunk, int nchunks,
                        const float3* __restrict__ params, const float2* __restrict__ seeds, int channels, int sets,
                        void* __restrict__ out_v, long out_stride, int n_out, int seg_outputs, int nsegs,
                        const float2* __restrict__ last_in, float2* __restrict__ last_out, int T, int D,
                        const __grid_constant__ DdcTaps<kDdcTapCapacity> taps)
{
    CSDRB_DYN_SMEM(smem);
    ddc_generic_body<M, CPL, DEMOD, float2>(wide, n_in, offset, chunk, nchunks, params, seeds, channels, sets, out_v, out_stride, n_out, seg_outputs, nsegs,
                                            last_in, last_out, T, D, taps, reinterpret_cast<float2*>(smem));
}

// the same on real wideband samples (csdrb_ddc_bank_f), at every served geometry -- D = 50 and 10 too -- and kDdcChannelsPerLane channels per lane
template <int M, bool DEMOD>
__global__ void __launch_bounds__(128, ddc_generic_ctas_per_sm(M, kDdcChannelsPerLane))
ddc_bank_generic_real_kernel(const float* __restrict__ wide, int n_in, int offset, int chunk, int nchunks,
                             const float3* __restrict__ params, const float2* __restrict__ seeds, int channels, int sets,
                             void* __restrict__ out_v, long out_stride, int n_out, int seg_outputs, int nsegs,
                             const float2* __restrict__ last_in, float2* __restrict__ last_out, int T, int D,
                             const __grid_constant__ DdcTaps<kDdcTapCapacity> taps)
{
    CSDRB_DYN_SMEM(smem);
    ddc_generic_body<M, kDdcChannelsPerLane, DEMOD, float>(wide, n_in, offset, chunk, nchunks, params, seeds, channels, sets, out_v, out_stride, n_out,
                                                           seg_outputs, nsegs, last_in, last_out, T, D, taps, reinterpret_cast<float2*>(smem));
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

// tap k = jD + p stored at [p][j], rows of MP = M rounded up to even; taps past T (and rows past M) are zero
static void ddc_pack_taps(float2* h2, int D, int M, const float* h_taps, int T)
{
    const int MP = (M + 1) & ~1;
    for (int p = 0; p < D; p++)
        for (int j = 0; j < MP; j++) {
            const int k = j * D + p; const float h = (j < M && k < T) ? h_taps[k] : 0.f;
            float2& slot = h2[(p * MP + j) / 2];
            if (j & 1) slot.y = h; else slot.x = h;
        }
}

static int ddc_cpl_from_env() { return getenv("CSDRB_DDC_CPL") && atoi(getenv("CSDRB_DDC_CPL")) != kDdcChannelsPerLane ? 1 : kDdcChannelsPerLane; }

// Grid of a bank launch: one warp per (segment, channel set).  Enough segments to fill warps_per_sm resident warps on every SM, while keeping the
// M-1 trailing periods of every segment a small fraction (at least 2M outputs per segment).
struct DdcGrid { int sets, seg, nsegs; unsigned ctas; };
static DdcGrid ddc_grid(int channels, int n_out, int M, int cpl, int warps_per_sm)
{
    DdcGrid g;
    g.sets = (channels + 32 * cpl - 1) / (32 * cpl);
    const long want_segments = (kSmCount * warps_per_sm + g.sets - 1) / g.sets;
    g.seg = (int)((n_out + want_segments - 1) / want_segments);
    if (g.seg < 2 * M) g.seg = 2 * M;
    g.nsegs = (n_out + g.seg - 1) / g.seg;
    g.ctas = (unsigned)(((long)g.nsegs * g.sets + 3) / 4);
    return g;
}

template <int D, int M>
static int launch_fused(const float2* wide, int n_in, int offset, int chunk, int nchunks, const float3* params, const float2* seeds, int channels,
                        int demod, void* out, long out_stride, int n_out, const float2* last_in, float2* last_out, const float* h_taps, int T, cudaStream_t st)
{
    constexpr int MP = (M + 1) & ~1;
    DdcTaps<D * MP> tp;
    ddc_pack_taps(tp.h2, D, M, h_taps, T);
    static const int cpl = ddc_cpl_from_env();
    const DdcGrid g = ddc_grid(channels, n_out, M, cpl, kDdcWarpsPerSm);
#define CSDRB_DDC_LAUNCH(CPLV, DM) ddc_bank_fused2_kernel<D, M, CPLV, DM><<<g.ctas, 128, 0, st>>>(wide, n_in, offset, chunk, nchunks, params, seeds, channels, g.sets, out, out_stride, n_out, g.seg, g.nsegs, last_in, last_out, T, tp)
    if (cpl == kDdcChannelsPerLane) { if (demod) CSDRB_DDC_LAUNCH(kDdcChannelsPerLane, true); else CSDRB_DDC_LAUNCH(kDdcChannelsPerLane, false); }
    else { if (demod) CSDRB_DDC_LAUNCH(1, true); else CSDRB_DDC_LAUNCH(1, false); }
#undef CSDRB_DDC_LAUNCH
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}

// M = bucket; sized for the bucket's own resident warps (its registers allow fewer CTAs per SM than the D = 50 / 10 kernels' three at large M).
// Real input (TIn = float) runs at kDdcChannelsPerLane whatever CSDRB_DDC_CPL says: one instantiation per bucket and DEMOD.
template <int M, class TIn = float2>
static int launch_generic(const TIn* wide, int n_in, int offset, int chunk, int nchunks, const float3* params, const float2* seeds, int channels,
                          int demod, void* out, long out_stride, int n_out, const float2* last_in, float2* last_out, const float* h_taps, int T, int D,
                          cudaStream_t st)
{
    constexpr int MP = (M + 1) & ~1;
    DdcTaps<kDdcTapCapacity> tp;
    ddc_pack_taps(tp.h2, D, M, h_taps, T);
    static const int env_cpl = ddc_cpl_from_env();
    constexpr bool real = std::is_same_v<TIn, float>;
    const int cpl = real ? kDdcChannelsPerLane : env_cpl;
    const DdcGrid g = ddc_grid(channels, n_out, M, cpl, 4 * ddc_generic_ctas_per_sm(M, cpl));
    const size_t smem = (size_t)D * MP * sizeof(float);
#define CSDRB_DDC_ARGS wide, n_in, offset, chunk, nchunks, params, seeds, channels, g.sets, out, out_stride, n_out, g.seg, g.nsegs, last_in, last_out, T, D, tp
    if constexpr (real) {
        if (demod) ddc_bank_generic_real_kernel<M, true><<<g.ctas, 128, smem, st>>>(CSDRB_DDC_ARGS);
        else ddc_bank_generic_real_kernel<M, false><<<g.ctas, 128, smem, st>>>(CSDRB_DDC_ARGS);
    } else {
#define CSDRB_DDC_LAUNCH(CPLV, DM) ddc_bank_generic_kernel<M, CPLV, DM><<<g.ctas, 128, smem, st>>>(CSDRB_DDC_ARGS)
        if (cpl == kDdcChannelsPerLane) { if (demod) CSDRB_DDC_LAUNCH(kDdcChannelsPerLane, true); else CSDRB_DDC_LAUNCH(kDdcChannelsPerLane, false); }
        else { if (demod) CSDRB_DDC_LAUNCH(1, true); else CSDRB_DDC_LAUNCH(1, false); }
#undef CSDRB_DDC_LAUNCH
    }
#undef CSDRB_DDC_ARGS
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}

// the generic bucket of a geometry: the smallest of kDdcBuckets >= ceil(T/D) whose D * MP taps fit the capacity, or 0
static int ddc_bucket(int decimation, int taps_length)
{
    if (decimation <= 0 || (decimation & 1) || taps_length <= 0) return 0;
    const long m = ((long)taps_length + decimation - 1) / decimation;
    for (int b : kDdcBuckets)
        if (m <= b) return (long)decimation * ((b + 1) & ~1) <= kDdcTapCapacity ? b : 0;
    return 0;
}

int ddc_bank_geometry(int decimation, int taps_length)
{
    if (ddc_bucket(decimation, taps_length)) return 0;
    set_error("ddc bank: no fused kernel for decimation %d / %d taps (served: even decimation D, M = ceil(taps / D) <= %d, and D * MP <= %d taps, "
              "MP = the smallest of 4, 8, 12, 18, 20, 24 >= M); run the unfused bank calls", decimation, taps_length, kDdcMaxM, kDdcTapCapacity);
    return -2;
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
    ddc_phase_chain_kernel<<<chain_ctas(channels, kDdcChainWarps), 32 * kDdcChainWarps, 0, st>>>(reinterpret_cast<const float3*>(d_params), d_phase_io, chunk_phase, channels, nchunks, chunk, next_chunk,
                                                             static_cast<const WrapTable*>(d_tables));
    CSDRB_CUDA(cudaGetLastError());
    const long total = (long)channels * nchunks;
    ddc_seed_kernel<<<(int)((total + 255) / 256), 256, 0, st>>>(chunk_phase, seeds, total);
    CSDRB_CUDA(cudaGetLastError());
    return launches;
}

// the alignment the group loads need: two samples per load, 16 bytes for complex input, 8 for real
template <class TIn>
static bool ddc_wide_aligned(const TIn* d_wide)
{
    constexpr bool real = std::is_same_v<TIn, float>;
    if (!(reinterpret_cast<uintptr_t>(d_wide) & (real ? 7 : 15))) return true;
    set_error(real ? "ddc bank: real wideband input must be 8-byte aligned (an even sample of a 16-byte aligned buffer)"
                   : "ddc bank: wideband input must be 16-byte aligned");
    return false;
}

// main kernel: needs the seeds a matching launch_ddc_prepass() left in d_scratch.  Complex input: D = 50 and 10 run their own kernels; real input
// runs the generic kernel at every served geometry.
template <class TIn>
static int ddc_main(const TIn* d_wide, int input_size, int channels, const float* d_params, int chunk, int offset, int decimation,
                    const float* h_taps, int taps_length, int demod, void* d_out, long out_stride, const float2* d_last_in, float2* d_last_out,
                    const void* d_scratch, cudaStream_t st)
{
    if (channels <= 0 || decimation <= 0 || taps_length <= 0) { set_error("ddc bank: bad geometry"); return -1; }
    const int n_out = input_size >= taps_length ? (input_size - taps_length) / decimation + 1 : 0;
    if (n_out == 0) return 0;
    if (chunk <= 0) chunk = input_size;
    if (!ddc_wide_aligned(d_wide)) return -1;
    const int nchunks = (int)(((long)offset + input_size + chunk - 1) / chunk) + 1;
    const float2* seeds = reinterpret_cast<const float2*>(static_cast<const char*>(d_scratch) + (((size_t)channels * nchunks * sizeof(float) + 15) & ~(size_t)15));
    if (int rc = ddc_bank_geometry(decimation, taps_length); rc < 0) return rc;
    int rc = -1;
    const float3* P = reinterpret_cast<const float3*>(d_params);
#define CSDRB_DDC_ARGS d_wide, input_size, offset, chunk, nchunks, P, seeds, channels, demod, d_out, out_stride, n_out, d_last_in, d_last_out, h_taps, taps_length
    bool done = false;
    if constexpr (std::is_same_v<TIn, float2>) {
        done = true;
        if (decimation == 50 && taps_length <= 50 * 17) rc = launch_fused<50, 17>(CSDRB_DDC_ARGS, st);
        else if (decimation == 10 && taps_length <= 10 * 8) rc = launch_fused<10, 8>(CSDRB_DDC_ARGS, st);
        else if (decimation == 10 && taps_length <= 10 * 20) rc = launch_fused<10, 20>(CSDRB_DDC_ARGS, st);
        else done = false;
    }
    if (!done) switch (ddc_bucket(decimation, taps_length)) {
        case 4: rc = launch_generic<4, TIn>(CSDRB_DDC_ARGS, decimation, st); break;
        case 8: rc = launch_generic<8, TIn>(CSDRB_DDC_ARGS, decimation, st); break;
        case 12: rc = launch_generic<12, TIn>(CSDRB_DDC_ARGS, decimation, st); break;
        case 17: rc = launch_generic<17, TIn>(CSDRB_DDC_ARGS, decimation, st); break;
        case 20: rc = launch_generic<20, TIn>(CSDRB_DDC_ARGS, decimation, st); break;
        case 24: rc = launch_generic<24, TIn>(CSDRB_DDC_ARGS, decimation, st); break;
    }
#undef CSDRB_DDC_ARGS
    return rc < 0 ? rc : n_out;
}

int launch_ddc_main(const float2* d_wide, int input_size, int channels, const float* d_params, int chunk, int offset, int decimation,
                    const float* h_taps, int taps_length, int demod, void* d_out, long out_stride, const float2* d_last_in, float2* d_last_out,
                    const void* d_scratch, cudaStream_t st)
{
    return ddc_main(d_wide, input_size, channels, d_params, chunk, offset, decimation, h_taps, taps_length, demod, d_out, out_stride, d_last_in, d_last_out,
                    d_scratch, st);
}

int launch_ddc_main_f(const float* d_wide, int input_size, int channels, const float* d_params, int chunk, int offset, int decimation,
                      const float* h_taps, int taps_length, int demod, void* d_out, long out_stride, const float2* d_last_in, float2* d_last_out,
                      const void* d_scratch, cudaStream_t st)
{
    return ddc_main(d_wide, input_size, channels, d_params, chunk, offset, decimation, h_taps, taps_length, demod, d_out, out_stride, d_last_in, d_last_out,
                    d_scratch, st);
}

// one-shot: pre-pass and main kernel back to back on the caller's stream
template <class TIn>
static int ddc_bank(const TIn* d_wide, int input_size, int channels, const float* d_params, float* d_phase_io, int chunk, int offset,
                    int decimation, const float* h_taps, int taps_length, int demod, void* d_out, long out_stride,
                    const float2* d_last_in, float2* d_last_out, void* d_scratch, size_t scratch_bytes, int* launches, cudaStream_t st)
{
    *launches = 0;
    if (channels <= 0 || decimation <= 0 || taps_length <= 0) { set_error("ddc bank: bad geometry"); return -1; }
    if (!ddc_wide_aligned(d_wide)) return -1;
    if (input_size >= taps_length) {                                    // a refused geometry launches nothing (and leaves d_phase_io alone)
        if (int rc = ddc_bank_geometry(decimation, taps_length); rc < 0) return rc;
    }
    int rc = launch_ddc_prepass(input_size, channels, d_params, d_phase_io, chunk, offset, decimation, taps_length, d_scratch, scratch_bytes, nullptr, st);
    if (rc <= 0) return rc;
    const int pre = rc;
    rc = ddc_main(d_wide, input_size, channels, d_params, chunk, offset, decimation, h_taps, taps_length, demod, d_out, out_stride, d_last_in, d_last_out, d_scratch, st);
    if (rc < 0) return rc;
    *launches = pre + 1;
    return rc;
}

int launch_ddc_bank(const float2* d_wide, int input_size, int channels, const float* d_params, float* d_phase_io, int chunk, int offset,
                    int decimation, const float* h_taps, int taps_length, int demod, void* d_out, long out_stride,
                    const float2* d_last_in, float2* d_last_out, void* d_scratch, size_t scratch_bytes, int* launches, cudaStream_t st)
{
    return ddc_bank(d_wide, input_size, channels, d_params, d_phase_io, chunk, offset, decimation, h_taps, taps_length, demod, d_out, out_stride,
                    d_last_in, d_last_out, d_scratch, scratch_bytes, launches, st);
}

int launch_ddc_bank_f(const float* d_wide, int input_size, int channels, const float* d_params, float* d_phase_io, int chunk, int offset,
                      int decimation, const float* h_taps, int taps_length, int demod, void* d_out, long out_stride,
                      const float2* d_last_in, float2* d_last_out, void* d_scratch, size_t scratch_bytes, int* launches, cudaStream_t st)
{
    return ddc_bank(d_wide, input_size, channels, d_params, d_phase_io, chunk, offset, decimation, h_taps, taps_length, demod, d_out, out_stride,
                    d_last_in, d_last_out, d_scratch, scratch_bytes, launches, st);
}

}  // namespace csdrb
