// audio.cu -- K5 fractional_decimator_ff and K6 fastagc_ff (the per-channel audio-rate tail of the FM chain).
//
// K5 replaces fractional_decimator_ff (libcsdr.c:751-793; state struct libcsdr.h:151-168).
//    Output positions come from a float accumulator (`where += rate`) whose ceilf() picks sample indices,
//    so one ulp of difference flips an index (SURVEY.md section 7, hard part 3).  We therefore split the work:
//      fracdec_positions_kernel : one thread per channel replays the accumulator chain exactly and records
//                                 (index_high, xwhere) per output -- sequential by definition, tiny;
//      fracdec_interp_kernel    : one thread per output evaluates the Lagrange polynomial with the same
//                                 operation order as the reference (IEEE mul/div/add, no contraction).
// K6 replaces fastagc_ff (libcsdr.c:944-991; state struct libcsdr.h:118-128): fully parallel over (channel, block) -- the
//    gain only depends on a three-block window of peaks; linear gain ramp evaluated in double exactly as the C
//    expression promotes it, two blocks of latency.
#include "common.cuh"
#include "kernels.h"

#include <cmath>
#include <new>

namespace csdrb {

// ---------------------------------------------------------------------------------------------- K5
struct FracDecState { float where; int input_processed; int output_size; };

__global__ void fracdec_positions_kernel(FracDecState* __restrict__ state, int* __restrict__ idx_high, float* __restrict__ xwhere,
                                         int channels, int n, float rate, int num_poly_points, int xifirst, int taps_length, int cap)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= channels) return;
    float where = state[c].where;
    int produced = 0, index_high;
    for (; (index_high = (int)ceilf(where)) + num_poly_points + taps_length < n; where = __fadd_rn(where, rate)) {
        if (produced < cap) {
            idx_high[(long)c * cap + produced] = index_high;
            xwhere[(long)c * cap + produced] = __fsub_rn(where, (float)(index_high - 1));
        }
        produced++;
    }
    const int processed = (index_high - 1) + xifirst;
    state[c].input_processed = processed;
    state[c].where = __fsub_rn(where, (float)processed);
    state[c].output_size = produced < cap ? produced : cap;
}

constexpr int FD_MAX_POINTS = 64;
constexpr int FD_MAX_SEGS = 96;

// Closed form of the position chain.  While `where` stays inside one binade [2^E, 2^(E+1)) it is M*u (u = 2^(E-23)) and
// fl(where + rate) = (M + q)*u with a constant q = round(rate/u) (ties-to-even resolves to a constant step once M is even), as long
// as the exact sum stays inside the binade.  So the chain is a handful of arithmetic progressions ("segments") joined by single
// real float additions at the binade crossings; one thread per channel emits the segments (<= ~60 iterations instead of one
// per output), and every output then recomputes its own `where` exactly from its segment.  Bit-exact with the sequential loop
// (the K5 tests compare outputs with array_equal against the strict oracle).
struct FdSeg { int k0; unsigned M; unsigned q; int E; int cnt; };

__global__ void fracdec_segments_kernel(FracDecState* __restrict__ state, FdSeg* __restrict__ segs, int* __restrict__ nsegs, int channels, int n,
                                        float rate, int num_poly_points, int xifirst, int taps_length, int cap)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= channels) return;
    const long L = (long)n - num_poly_points - taps_length - 1;          // loop runs while ceil(where) <= L
    const unsigned rbits = __float_as_uint(rate);
    const int er = (int)((rbits >> 23) & 0xff) - 127;
    const unsigned R = (rbits & 0x7fffffu) | 0x800000u;                  // rate = R * 2^(er-23)
    float where = state[c].where;
    int k = 0, ns = 0;
    FdSeg* out = segs + (long)c * FD_MAX_SEGS;
    while ((long)ceilf(where) <= L && k < cap) {
        int cnt = 1;
        const unsigned wb = __float_as_uint(where);
        const int E = (int)((wb >> 23) & 0xff) - 127;
        const unsigned M = (wb & 0x7fffffu) | 0x800000u;
        unsigned q = 0;
        if (where > 0.f && E >= 0 && E <= 22 && ns < FD_MAX_SEGS - 2) {
            const int d = E - er;                                        // ulp(where) = 2^d * ulp(rate)
            unsigned cq = 0; bool regular = false;
            if (d <= 0) { if (d >= -6) { q = R << (-d); cq = q; regular = true; } }
            else if (d < 24) {
                const unsigned frac = R & ((1u << d) - 1u), I = R >> d, half = 1u << (d - 1);
                cq = I + (frac ? 1u : 0u);
                if (frac != half) { q = I + (frac > half ? 1u : 0u); regular = true; }
                else if ((M & 1u) == 0u) { q = I + (I & 1u); regular = true; }   // tie, M even: the sum always rounds to the even neighbour
            }
            if (regular && q > 0) {
                const long room = (long)(1u << 24) - 1 - (long)cq - (long)M;      // transitions that provably stay in the binade
                long jreg = room >= 0 ? room / (long)q : -1;
                const long lim = (L << (23 - E)) - (long)M;                        // where_j <= L  <=>  M + j*q <= L / u
                long jlim = lim >= 0 ? lim / (long)q : 0;
                long j = jreg < jlim ? jreg : jlim;
                if (j < 0) j = 0;
                if (j + 1 > (long)(cap - k)) j = cap - k - 1;
                cnt = (int)j + 1;
            }
        }
        FdSeg sg; sg.k0 = k; sg.M = M; sg.q = cnt > 1 ? q : 0u; sg.E = E; sg.cnt = cnt;
        if (cnt == 1) { sg.M = wb; sg.E = -1000; }                       // single output: keep the float itself
        if (ns < FD_MAX_SEGS) out[ns++] = sg;
        k += cnt;
        const float last = cnt > 1 ? __uint_as_float(((unsigned)(E + 127) << 23) | ((M + (unsigned)(cnt - 1) * q) & 0x7fffffu)) : where;
        where = __fadd_rn(last, rate);                                   // the crossing step (or a plain step) is a real float addition
    }
    const int index_high = (int)ceilf(where);
    const int processed = (index_high - 1) + xifirst;
    state[c].input_processed = processed;
    state[c].where = __fsub_rn(where, (float)processed);
    state[c].output_size = k;
    nsegs[c] = ns;
}

// PTS > 0: the point count is a compile-time constant (the CLI default is 12, libcsdr.c:717 / csdr.c:1476): the 16 x 16 predicated loop nest of the
// generic form (512 multiplies and 16 divisions per output, most of them masked) becomes PTS*(PTS-1) multiplies, PTS divisions and constant
// denominators -- same operations in the same order on the live points, so the result is unchanged bit for bit.
template <int PTS>
__global__ void __launch_bounds__(128)
fracdec_interp_seg_kernel(const float* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride,
                          const FracDecState* __restrict__ state, const FdSeg* __restrict__ segs, const int* __restrict__ nsegs,
                          int num_poly_points, int xifirst, int xilast, const float* __restrict__ taps, int taps_length)
{
    __shared__ FdSeg sseg[FD_MAX_SEGS];
    const int c = blockIdx.y;
    const int ns = nsegs[c];
    for (int i = threadIdx.x; i < ns; i += blockDim.x) sseg[i] = segs[(long)c * FD_MAX_SEGS + i];
    __syncthreads();
    const int produced = state[c].output_size;
    const float* x = in + (long)c * in_stride;
    for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < produced; o += gridDim.x * blockDim.x) {
        int si = 0;
        while (si + 1 < ns && sseg[si + 1].k0 <= o) si++;
        const FdSeg sg = sseg[si];
        float where;
        if (sg.E == -1000) where = __uint_as_float(sg.M);
        else where = __uint_as_float(((unsigned)(sg.E + 127) << 23) | ((sg.M + (unsigned)(o - sg.k0) * sg.q) & 0x7fffffu));
        const int low = (int)ceilf(where) - 1;
        const float xw = __fsub_rn(where, (float)low);
        float acc = 0.f;
        if (PTS > 0) {
            float pts[PTS > 0 ? PTS : 1], dxj[PTS > 0 ? PTS : 1];
#pragma unroll
            for (int w = 0; w < PTS; w++) { pts[w] = x[low + w]; dxj[w] = __fsub_rn(xw, (float)(1 - PTS / 2 + w)); }
#pragma unroll
            for (int wi = 0; wi < PTS; wi++) {
                float coef = 1.f, den = 1.f;
#pragma unroll
                for (int wj = 0; wj < PTS; wj++)
                    if (wj != wi) { coef = __fmul_rn(coef, dxj[wj]); den = __fmul_rn(den, (float)(wi - wj)); }     // den folds to a constant
                acc = __fadd_rn(acc, __fmul_rn(__fdiv_rn(coef, den), pts[wi]));
            }
        } else if (!taps && num_poly_points <= 16) {
            // common case (12 points, no prefilter): fetch all points and form all (xw - xj) first, then the products -- the loads are
            // independent of the accumulation chain, issuing them up front hides their latency once instead of once per point
            float pts[16], dxj[16];
#pragma unroll
            for (int w = 0; w < 16; w++) { pts[w] = w < num_poly_points ? x[low + w] : 0.f; dxj[w] = __fsub_rn(xw, (float)(xifirst + w)); }
#pragma unroll
            for (int wi = 0; wi < 16; wi++) {
                if (wi < num_poly_points) {
                    float coef = 1.f, den = 1.f;
#pragma unroll
                    for (int wj = 0; wj < 16; wj++)
                        if (wj < num_poly_points && wj != wi) { coef = __fmul_rn(coef, dxj[wj]); den = __fmul_rn(den, (float)(wi - wj)); }
                    acc = __fadd_rn(acc, __fmul_rn(__fdiv_rn(coef, den), pts[wi]));
                }
            }
        } else {
            int slot = 0;
            for (int xi = xifirst; xi <= xilast; xi++, slot++) {
                float coef = 1.f, den = 1.f;
                for (int xj = xifirst; xj <= xilast; xj++)
                    if (xi != xj) { coef = __fmul_rn(coef, __fsub_rn(xw, (float)xj)); den = __fmul_rn(den, (float)(xi - xj)); }
                float pt;
                if (taps) {
                    pt = 0.f;
                    const float* seg = x + low + slot;
                    for (int t = 0; t < taps_length; t++) pt = __fadd_rn(pt, __fmul_rn(seg[t], taps[t]));
                } else pt = x[low + slot];
                acc = __fadd_rn(acc, __fmul_rn(__fdiv_rn(coef, den), pt));
            }
        }
        out[(long)c * out_stride + o] = acc;
    }
}

__global__ void __launch_bounds__(128)
fracdec_interp_kernel(const float* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride,
                      const FracDecState* __restrict__ state, const int* __restrict__ idx_high, const float* __restrict__ xwhere,
                      int cap, int num_poly_points, int xifirst, int xilast, const float* __restrict__ taps, int taps_length)
{
    // fallback for blocks of 2^22 samples and more: positions were replayed sequentially by fracdec_positions_kernel
    const int c = blockIdx.y;
    const int produced = state[c].output_size;
    const float* x = in + (long)c * in_stride;
    for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < produced; o += gridDim.x * blockDim.x) {
        const int low = idx_high[(long)c * cap + o] - 1;
        const float xw = xwhere[(long)c * cap + o];
        float acc = 0.f;
        int slot = 0;
        for (int xi = xifirst; xi <= xilast; xi++, slot++) {
            float coef = 1.f, den = 1.f;
            for (int xj = xifirst; xj <= xilast; xj++)
                if (xi != xj) { coef = __fmul_rn(coef, __fsub_rn(xw, (float)xj)); den = __fmul_rn(den, (float)(xi - xj)); }
            float pt;
            if (taps) {
                pt = 0.f;
                const float* seg = x + low + slot;
                for (int t = 0; t < taps_length; t++) pt = __fadd_rn(pt, __fmul_rn(seg[t], taps[t]));
            } else pt = x[low + slot];
            acc = __fadd_rn(acc, __fmul_rn(__fdiv_rn(coef, den), pt));
        }
        out[(long)c * out_stride + o] = acc;
    }
}

size_t fracdec_scratch_bytes(int channels, int n, float rate)
{
    const int cap = (int)((double)n / (rate > 1.f ? rate : 1.0)) + 8;
    const size_t seq = (size_t)channels * cap * (sizeof(int) + sizeof(float));             // sequential fallback (n >= 2^22)
    const size_t par = (size_t)channels * (FD_MAX_SEGS * sizeof(FdSeg) + sizeof(int)) + 64;
    return seq > par ? seq : par;
}

int launch_fractional_decimator_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n,
                                     float rate, int num_poly_points, const float* d_taps, int taps_length, void* d_state,
                                     void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (!(rate > 1.0f)) { set_error("fractional_decimator: rate must be > 1.0 (reference asserts it, libcsdr.c:756)"); return -1; }
    num_poly_points &= ~1;
    if (num_poly_points < 2 || num_poly_points > FD_MAX_POINTS) { set_error("fractional_decimator: num_poly_points must be even, 2..64"); return -1; }
    const int cap = (int)((double)n / rate) + 8;
    if (!d_scratch || scratch_bytes < fracdec_scratch_bytes(channels, n, rate)) { set_error("fractional_decimator: scratch too small"); return -1; }
    const int xifirst = -(num_poly_points / 2) + 1, xilast = num_poly_points / 2;
    int* idx = static_cast<int*>(d_scratch);
    float* xw = reinterpret_cast<float*>(idx + (size_t)channels * cap);
    if (!d_taps) taps_length = 0;
    if (n < (1 << 22)) {                                                 // closed-form positions: fully parallel
        FdSeg* segs = static_cast<FdSeg*>(d_scratch);
        int* nsegs = reinterpret_cast<int*>(segs + (size_t)channels * FD_MAX_SEGS);
        fracdec_segments_kernel<<<(channels + 63) / 64, 64, 0, st>>>(static_cast<FracDecState*>(d_state), segs, nsegs, channels, n, rate, num_poly_points,
                                                                     xifirst, taps_length, cap);
        CSDRB_CUDA(cudaGetLastError());
        int gx2 = (cap + 127) / 128; if (gx2 > 2048) gx2 = 2048;
        if (!d_taps && num_poly_points == 12)
            fracdec_interp_seg_kernel<12><<<dim3(gx2, channels), 128, 0, st>>>(d_in, in_stride, d_out, out_stride, static_cast<const FracDecState*>(d_state), segs, nsegs,
                                                                               num_poly_points, xifirst, xilast, d_taps, taps_length);
        else
            fracdec_interp_seg_kernel<0><<<dim3(gx2, channels), 128, 0, st>>>(d_in, in_stride, d_out, out_stride, static_cast<const FracDecState*>(d_state), segs, nsegs,
                                                                              num_poly_points, xifirst, xilast, d_taps, taps_length);
        CSDRB_CUDA(cudaGetLastError());
        return 2;
    }
    fracdec_positions_kernel<<<(channels + 63) / 64, 64, 0, st>>>(static_cast<FracDecState*>(d_state), idx, xw, channels, n, rate, num_poly_points,
                                                                  xifirst, taps_length, cap);
    CSDRB_CUDA(cudaGetLastError());
    int gx = (cap + 127) / 128; if (gx > 1024) gx = 1024;
    fracdec_interp_kernel<<<dim3(gx, channels), 128, 0, st>>>(d_in, in_stride, d_out, out_stride, static_cast<const FracDecState*>(d_state), idx, xw, cap,
                                                              num_poly_points, xifirst, xilast, d_taps, taps_length);
    CSDRB_CUDA(cudaGetLastError());
    return 2;
}

// ---------------------------------------------------------------------------------------------- first-order recursions
// deemphasis_wfm_ff (libcsdr.c:1081-1097): y[i] = alpha*x[i] + (1-alpha)*y[i-1], and dcblock_ff (libcsdr.c:903-918): y[i] = (x[i] - x[i-1]) +
// a*y[i-1] -- float recursions whose rounding sequence is the result, so they stay sequential per channel: lane = channel, a warp moves 32
// channels through a padded shared tile so that global accesses are coalesced rows while each lane walks its own row (same scheme as the NCO
// kernel).  recursion_rows is that scheme; Step gives the per-channel State, how a carried state starts (begin) and one sample's step; every tile is read whole before it is
// written, so d_in == d_out with equal strides is allowed.
struct DeemphasisStep {
    using State = float;                                               // y[i-1]
    float alpha, keep;
    __device__ __forceinline__ State begin(State y) const { return y != y ? 0.f : y; }   // NaN carry restarts from 0 (libcsdr.c:1092)
    __device__ __forceinline__ float operator()(State& y, float x) const { y = __fadd_rn(__fmul_rn(alpha, x), __fmul_rn(keep, y)); return y; }
};
struct DcBlockStep {
    using State = DcBlockState;                                        // {x[i-1], y[i-1]}: dcblock_preserve_t
    float a;
    __device__ __forceinline__ State begin(State s) const { return s; }
    __device__ __forceinline__ float operator()(State& s, float x) const
    {
        s.last_output = __fadd_rn(__fsub_rn(x, s.last_input), __fmul_rn(a, s.last_output));
        s.last_input = x;
        return s.last_output;
    }
};

template <class Step>
__device__ __forceinline__ void recursion_rows(const float* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride, int channels,
                                               int n, Step step, typename Step::State* __restrict__ state_io)
{
    __shared__ float tile_all[4][32 * 33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* tile = tile_all[warp];
    const int c0 = (blockIdx.x * 4 + warp) * 32;
    if (c0 >= channels) return;
    const int rows = min(32, channels - c0);
    const bool live = lane < rows;
    typename Step::State s = live ? step.begin(state_io[c0 + lane]) : typename Step::State{};
    for (int t0 = 0; t0 < n; t0 += 32) {
        const int len = min(32, n - t0);
        for (int r0 = 0; r0 < rows; r0 += 8) {                       // eight rows' loads in flight before the first shared store
            float v[8];
#pragma unroll
            for (int u = 0; u < 8; u++) v[u] = (r0 + u < rows && lane < len) ? in[(long)(c0 + r0 + u) * in_stride + t0 + lane] : 0.f;
#pragma unroll
            for (int u = 0; u < 8; u++) if (r0 + u < rows) tile[(r0 + u) * 33 + lane] = v[u];
        }
        __syncwarp();
        if (live) {
            float* row = tile + lane * 33;
            for (int j = 0; j < len; j++) row[j] = step(s, row[j]);
        }
        __syncwarp();
        for (int r = 0; r < rows; r++) if (lane < len) out[(long)(c0 + r) * out_stride + t0 + lane] = tile[r * 33 + lane];
        __syncwarp();
    }
    if (live) state_io[c0 + lane] = s;
}

__global__ void __launch_bounds__(128)
deemphasis_wfm_bank_kernel(const float* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride, int channels, int n, DeemphasisStep step,
                           float* __restrict__ last_io)
{
    recursion_rows(in, in_stride, out, out_stride, channels, n, step, last_io);
}

__global__ void __launch_bounds__(128)
dcblock_bank_kernel(const float* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride, int channels, int n, DcBlockStep step,
                    DcBlockState* __restrict__ state_io)
{
    recursion_rows(in, in_stride, out, out_stride, channels, n, step, state_io);
}

int launch_deemphasis_wfm_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, float tau, int sample_rate,
                               float* d_last_io, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (sample_rate <= 0) { set_error("deemphasis_wfm: sample_rate must be positive"); return -1; }
    const float dt = (float)(1.0 / sample_rate);                        // same promotions as libcsdr.c:1090-1091
    const float alpha = dt / (tau + dt);
    const float keep = 1 - alpha;
    deemphasis_wfm_bank_kernel<<<(channels + 127) / 128, 128, 0, st>>>(d_in, in_stride, d_out, out_stride, channels, n, DeemphasisStep{alpha, keep}, d_last_io);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

int launch_dcblock_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, float a, void* d_state_io,
                        cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (a == 0.f) a = 0.999f;                                            // libcsdr.c:909
    dcblock_bank_kernel<<<(channels + 127) / 128, 128, 0, st>>>(d_in, in_stride, d_out, out_stride, channels, n, DcBlockStep{a},
                                                                  static_cast<DcBlockState*>(d_state_io));
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---------------------------------------------------------------------------------------------- WFM audio tail
// `fractional_decimator_ff R 12 | deemphasis_wfm_ff SR TAU | convert_f_s16` (README.md:66) per row, as the CLI runs it: the decimator in calls of
// exactly B samples (csdr.c:1510-1522: memmove of the unconsumed rest, `where -= input_processed` in float), the de-emphasis restarting a NaN carry
// at every B-th audio sample (libcsdr.c:1092, one call per B samples).  Every row shares the rate, the start and the framing, so the `where` chain,
// the sample positions and the 12 Lagrange weights of every output are the same for all rows: the host replays the chain (wfm_audio_replay, the
// reference's own float adds and ceilf) into a position table, and the kernel computes each output's weights once for all the rows of a warp.
struct WfmParams { float rate; int bufsize; float tau; int sample_rate; };   // layout of csdrb_wfm_audio_params_t
struct WfmState { float where; long long audio; };                           // layout of csdrb_wfm_audio_state_t; zeroed = stream start
struct WfmPos { int low; float xw; };                                         // first of the 12 input samples (row-relative), xwhere

constexpr int kWfmPoints = 12;
constexpr int kWfmXiFirst = 1 - kWfmPoints / 2;                               // -5: the reference starts at where = -xifirst (libcsdr.c:728)

// One warp per 32 rows (the deemphasis_wfm_bank_kernel scheme).  Per tile of 32 outputs: lane j forms the weights of output j once; for each of
// the warp's rows lane j sums w_i * x[low_j + i] into the padded tile; lane r then walks row r's recursion over the tile; the warp writes s16 rows.
__global__ void __launch_bounds__(128)
wfm_audio_bank_kernel(const float* __restrict__ in, long in_stride, short* __restrict__ out, long out_stride, int channels, int m,
                      const WfmPos* __restrict__ pos, float alpha, float keep, int bufsize, int phase0, float* __restrict__ last_io)
{
    __shared__ float tile_all[4][32 * 33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* tile = tile_all[warp];
    const int c0 = (blockIdx.x * 4 + warp) * 32;
    if (c0 >= channels) return;
    const int rows = min(32, channels - c0);
    const bool live = lane < rows;
    float y = live ? last_io[c0 + lane] : 0.f;
    int phase = phase0;                                                // audio index of the tile's first output, mod bufsize
    for (int t0 = 0; t0 < m; t0 += 32) {
        const int len = min(32, m - t0);
        const bool have = lane < len;
        float w[kWfmPoints];
        int low = 0;
        if (have) {
            const WfmPos p = pos[t0 + lane];
            low = p.low;
            float dxj[kWfmPoints];
#pragma unroll
            for (int k = 0; k < kWfmPoints; k++) dxj[k] = __fsub_rn(p.xw, (float)(kWfmXiFirst + k));
#pragma unroll
            for (int wi = 0; wi < kWfmPoints; wi++) {
                float coef = 1.f, den = 1.f;
#pragma unroll
                for (int wj = 0; wj < kWfmPoints; wj++)
                    if (wj != wi) { coef = __fmul_rn(coef, dxj[wj]); den = __fmul_rn(den, (float)(wi - wj)); }   // den folds to a constant
                w[wi] = __fdiv_rn(coef, den);
            }
        }
        for (int r0 = 0; r0 < rows; r0 += 8) {                          // eight rows' points in flight before the first sum
            float v[8][kWfmPoints];
#pragma unroll
            for (int u = 0; u < 8; u++) {
                const bool ok = have && r0 + u < rows;
                const float* x = in + (long)(c0 + (ok ? r0 + u : 0)) * in_stride + low;
#pragma unroll
                for (int k = 0; k < kWfmPoints; k++) v[u][k] = ok ? x[k] : 0.f;
            }
#pragma unroll
            for (int u = 0; u < 8; u++) {
                if (have && r0 + u < rows) {
                    float acc = 0.f;
#pragma unroll
                    for (int k = 0; k < kWfmPoints; k++) acc = __fadd_rn(acc, __fmul_rn(w[k], v[u][k]));
                    tile[(r0 + u) * 33 + lane] = acc;
                }
            }
        }
        __syncwarp();
        if (live) {
            float* row = tile + lane * 33;
            int q = phase;
            for (int j = 0; j < len; j++) {
                if (q == 0 && y != y) y = 0.f;                            // a new deemphasis_wfm_ff call: NaN carry restarts from 0
                y = __fadd_rn(__fmul_rn(alpha, row[j]), __fmul_rn(keep, y));
                row[j] = y;
                if (++q == bufsize) q = 0;
            }
        }
        phase = (phase + len) % bufsize;
        __syncwarp();
        for (int r = 0; r < rows; r++) if (have) out[(long)(c0 + r) * out_stride + t0 + lane] = (short)f_to_s16_bits(tile[r * 33 + lane]);
        __syncwarp();
    }
    if (live) last_io[c0 + lane] = y;
}

// Replays the reference's decimator calls over n samples from *s: returns the outputs and sets *consumed and *where_out; appends each output's
// position to `table` when given.  -1 for bad parameters or state, -2 for a call the CLI cannot run (it would consume nothing, or more than B).
int wfm_audio_replay(const void* h_params, const void* h_state, int n, int* consumed, float* where_out, std::vector<WfmPos>* table)
{
    const WfmParams* p = static_cast<const WfmParams*>(h_params);
    const WfmState* s = static_cast<const WfmState*>(h_state);
    if (!p || !s) { set_error("wfm_audio: null parameters or state"); return -1; }
    if (n < 0) { set_error("wfm_audio: negative sample count"); return -1; }
    if (!(p->rate > 1.0f)) { set_error("wfm_audio: rate must be > 1.0 (reference asserts it, libcsdr.c:756)"); return -1; }
    if (!std::isfinite(p->rate)) { set_error("wfm_audio: rate must be finite"); return -1; }
    if (!(p->tau > 0.0f)) { set_error("wfm_audio: tau must be positive"); return -1; }
    if (p->sample_rate <= 0) { set_error("wfm_audio: sample_rate must be positive"); return -1; }
    const bool start = s->where == 0.0f && s->audio == 0;
    if (!start && !(s->where >= 5.0f && s->where <= 6.0f && s->audio >= 0)) {
        set_error("wfm_audio: state {where %g, audio %lld} is neither a stream start nor one a call leaves (where in (5, 6])", (double)s->where, s->audio);
        return -1;
    }
    const int B = p->bufsize;
    if (B <= kWfmPoints) { set_error("wfm_audio: bufsize %d: a call needs more than %d samples", B, kWfmPoints); return -2; }
    float where = start ? (float)-kWfmXiFirst : s->where;
    const float rate = p->rate;
    int at = 0, m = 0;
    while (n - at >= B) {                                                 // one fractional_decimator_ff call on [at, at + B)
        double high;                                                      // ceilf(where) in double: exact, and no int overflow at huge rates
        for (; (high = (double)ceilf(where)) + kWfmPoints < (double)B; where += rate) {
            const int h = (int)high;                                      // < B here
            if (table) table->push_back(WfmPos{at + h - 1, where - (float)(h - 1)});
            m++;
        }
        const double processed = (high - 1) + kWfmXiFirst;
        if (!(processed >= 1 && processed <= (double)B)) {
            set_error("wfm_audio: a call at rate %g would consume %.0f of its %d samples, which the CLI cannot run", (double)rate, processed, B);
            return -2;
        }
        where -= (float)processed;
        at += (int)processed;
    }
    *consumed = at;
    *where_out = at > 0 ? where : s->where;                              // no call: the state stays as it was
    return m;
}

int wfm_audio_outputs(const void* h_params, const void* h_state, int n, int* consumed_out)
{
    int consumed = 0;
    float where = 0.f;
    const int m = wfm_audio_replay(h_params, h_state, n, &consumed, &where, nullptr);
    if (m >= 0 && consumed_out) *consumed_out = consumed;
    return m;
}

int launch_wfm_audio_bank(const float* d_in, long in_stride, int channels, int n, const void* h_params, void* h_state_io, float* d_last_io,
                          short* d_out, long out_stride, int* consumed_out, int* launches, cudaStream_t st)
{
    *launches = 0;
    if (channels < 1) { set_error("wfm_audio: channels must be at least 1"); return -1; }
    if (!d_in || !d_last_io || !d_out || !consumed_out) { set_error("wfm_audio: null pointer"); return -1; }
    if ((reinterpret_cast<uintptr_t>(d_in) & 3) || (reinterpret_cast<uintptr_t>(d_last_io) & 3) || (reinterpret_cast<uintptr_t>(d_out) & 1)) {
        set_error("wfm_audio: misaligned pointer (input and carry 4 bytes, output 2)"); return -1;
    }
    if (in_stride < n) { set_error("wfm_audio: input stride %ld below %d samples", in_stride, n); return -1; }
    std::vector<WfmPos> table;
    int consumed = 0;
    float where = 0.f;
    int m;
    try {
        m = wfm_audio_replay(h_params, h_state_io, n, &consumed, &where, &table);
    } catch (const std::bad_alloc&) {
        set_error("wfm_audio: no host memory for the position table of %d samples", n); return -1;
    }
    if (m < 0) return m;
    if (out_stride < m) { set_error("wfm_audio: output stride %ld below %d samples", out_stride, m); return -1; }
    WfmState* s = static_cast<WfmState*>(h_state_io);
    const WfmParams* p = static_cast<const WfmParams*>(h_params);
    if (m > 0) {
        const float dt = (float)(1.0 / p->sample_rate);                  // as launch_deemphasis_wfm_bank (libcsdr.c:1090-1091)
        const float alpha = dt / (p->tau + dt);
        const float keep = 1 - alpha;
        WfmPos* d_pos = nullptr;                                          // stream-ordered copy of the host table: the call never waits for the device
        CSDRB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&d_pos), sizeof(WfmPos) * (size_t)m, st));
        CSDRB_CUDA(cudaMemcpyAsync(d_pos, table.data(), sizeof(WfmPos) * (size_t)m, cudaMemcpyHostToDevice, st));
        wfm_audio_bank_kernel<<<(channels + 127) / 128, 128, 0, st>>>(d_in, in_stride, d_out, out_stride, channels, m, d_pos, alpha, keep, p->bufsize,
                                                                      (int)(s->audio % p->bufsize), d_last_io);
        CSDRB_CUDA(cudaGetLastError());
        CSDRB_CUDA(cudaFreeAsync(d_pos, st));
        *launches = 1;
    }
    s->where = where;
    s->audio += m;
    *consumed_out = consumed;
    return m;
}

// deemphasis_nfm_ff (libcsdr.c:1101-1128): a plain "valid" FIR over a real row, out[i] = sum_t taps[t] * in[i+t] for i < n - T
// (n - T outputs -- one fewer than a valid convolution has, exactly like the reference loop), taps picked by sample rate from the
// four fixed tables (host/nfm_deemph_taps.h).  One CTA = 1024 outputs of one channel: the 1024+T input window is staged in shared
// memory once (optionally clamped on the way in = the limit_ff that precedes this block in the NFM graph, README.md:87), the taps
// ride in as a __grid_constant__ parameter (uniform-index constant loads, no device-side table), and each thread owns four outputs
// 256 apart so that every shared read of a warp is 32 consecutive words.  Taps are accumulated in the reference's order (t ascending,
// one accumulator per output).
struct NfmTaps { float v[kNfmMaxTaps]; };

template <bool LIMIT>
__global__ void __launch_bounds__(256)
nfm_deemph_bank_kernel(const float* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride, int n, int T,
                       const __grid_constant__ NfmTaps taps, float limit_max)
{
    constexpr int kTile = 1024;
    __shared__ float win[kTile + kNfmMaxTaps];
    const int n_out = n - T;
    const int o0 = blockIdx.x * kTile;
    const float* row = in + (long)blockIdx.y * in_stride;
    for (int j = threadIdx.x; j < kTile + T; j += 256) {
        float v = o0 + j < n ? __ldg(row + o0 + j) : 0.f;
        if (LIMIT) v = fmaxf(-limit_max, fminf(limit_max, v));         // same expression as limit_ff_kernel (NaN -> +max)
        win[j] = v;
    }
    __syncthreads();
    float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f;
    const float* w = win + threadIdx.x;
#pragma unroll 4
    for (int t = 0; t < T; t++) {
        const float h = taps.v[t];
        acc0 = fmaf(h, w[t], acc0);
        acc1 = fmaf(h, w[t + 256], acc1);
        acc2 = fmaf(h, w[t + 512], acc2);
        acc3 = fmaf(h, w[t + 768], acc3);
    }
    float* orow = out + (long)blockIdx.y * out_stride;
    const int o = o0 + threadIdx.x;
    if (o < n_out) orow[o] = acc0;
    if (o + 256 < n_out) orow[o + 256] = acc1;
    if (o + 512 < n_out) orow[o + 512] = acc2;
    if (o + 768 < n_out) orow[o + 768] = acc3;
}

// returns the number of outputs per channel (n - T), 0 when the block is too short, < 0 on error
int launch_fir_valid_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, const float* h_taps, int T,
                          float limit_max, cudaStream_t st)
{
    if (!h_taps || T <= 0) { set_error("fir_valid bank: no taps"); return -1; }
    if (T > kNfmMaxTaps) { set_error("fir_valid bank: more than %d taps", kNfmMaxTaps); return -1; }
    if (channels <= 0 || n - T <= 0) return 0;
    if (channels > 65535) { set_error("fir_valid bank: more than 65535 channels in one call"); return -1; }
    NfmTaps taps;
    for (int t = 0; t < kNfmMaxTaps; t++) taps.v[t] = t < T ? h_taps[t] : 0.f;
    const dim3 grid((unsigned)((n - T + 1023) / 1024), (unsigned)channels);
    if (limit_max > 0.f) nfm_deemph_bank_kernel<true><<<grid, 256, 0, st>>>(d_in, in_stride, d_out, out_stride, n, T, taps, limit_max);
    else nfm_deemph_bank_kernel<false><<<grid, 256, 0, st>>>(d_in, in_stride, d_out, out_stride, n, T, taps, 0.f);
    CSDRB_CUDA(cudaGetLastError());
    return n - T;
}

// deemphasis_nfm_ff: the table of this sample rate, or 0 outputs when there is none (libcsdr.c:1119)
int launch_deemphasis_nfm_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, int sample_rate,
                               float limit_max, cudaStream_t st)
{
    int T = 0;
    const float* h = csdrb_deemphasis_nfm_taps(sample_rate, &T);
    if (!h || T <= 0) return 0;
    return launch_fir_valid_bank(d_in, in_stride, d_out, out_stride, channels, n, h, T, limit_max, st);
}

// ---------------------------------------------------------------------------------------------- K6
// The gain of block b is reference / max(peak_b, peak_{b-1}, peak_{b-2}) (capped), ramped from the gain of block b-1, applied to
// block b-2: nothing is sequential beyond a three-block window, so the bank runs fully parallel over (channel, block):
//   fastagc_peaks_kernel : |x| maximum of every block                                 (reads the input once)
//   fastagc_apply_kernel : recomputes target_b and target_{b-1} from the peaks window, writes block b-2 scaled by the ramp
//   fastagc_carry_kernel : new history (last two input blocks), peaks and last gain for the next call
struct FastAgcState { float peak_1, peak_2, last_gain; };

__global__ void __launch_bounds__(256)
fastagc_peaks_kernel(const float* __restrict__ in, long in_stride, int block, int nblocks, float* __restrict__ peaks)
{
    __shared__ float red[8];
    const int b = blockIdx.x, c = blockIdx.y, tid = threadIdx.x;
    const float* cur = in + (long)c * in_stride + (long)b * block;
    float m = 0.f;
    for (int i = tid; i < block; i += blockDim.x) m = fmaxf(m, fabsf(cur[i]));
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) red[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) { float t = red[0]; for (int w = 1; w < (int)(blockDim.x >> 5); w++) t = fmaxf(t, red[w]); peaks[(long)c * nblocks + b] = t; }
}

__device__ __forceinline__ float agc_peak_at(const float* pk, const FastAgcState& st, int b)
{
    // peak of the block that entered at call b; b = -1 / -2 are the two blocks before this launch (state.peak_2 / peak_1)
    return b >= 0 ? pk[b] : (b == -1 ? st.peak_2 : st.peak_1);
}
__device__ __forceinline__ float agc_target(const float* pk, const FastAgcState& st, int b, float reference)
{
    float t = agc_peak_at(pk, st, b);
    const float p2 = agc_peak_at(pk, st, b - 1), p1 = agc_peak_at(pk, st, b - 2);
    if (t < p2) t = p2;
    if (t < p1) t = p1;
    float g = __fdiv_rn(reference, t);
    if (g > 50.f) g = 50.f;                                            // FASTAGC_MAX_GAIN, libcsdr.c:944
    return g;
}

// S16 = true: the output leaves as convert_f_s16 of the scaled sample, as in fastagc_fused_kernel<true>
template <bool S16>
__global__ void __launch_bounds__(256)
fastagc_apply_kernel(const float* __restrict__ in, long in_stride, void* __restrict__ out_v, long out_stride, int block, int nblocks,
                     float reference, const FastAgcState* __restrict__ state, const float* __restrict__ hist, const float* __restrict__ peaks)
{
    const int b = blockIdx.x, c = blockIdx.y, tid = threadIdx.x;
    const FastAgcState st = state[c];
    const float* pk = peaks + (long)c * nblocks;
    const float target = agc_target(pk, st, b, reference);
    const float last_gain = b == 0 ? st.last_gain : agc_target(pk, st, b - 1, reference);
    const float* x = in + (long)c * in_stride;
    const float* h1 = hist + (long)c * 2 * block;
    const float* leaving = b >= 2 ? x + (long)(b - 2) * block : (b == 0 ? h1 : h1 + block);
    const long o = (long)c * out_stride + (long)b * block;
    for (int i = tid; i < block; i += blockDim.x) {
        const float r = __fdiv_rn((float)i, (float)block);
        const float gain = (float)((double)last_gain * (1.0 - (double)r) + (double)__fmul_rn(target, r));
        const float v = __fmul_rn(leaving[i], gain);
        if (S16) static_cast<short*>(out_v)[o + i] = (short)f_to_s16_bits(v); else static_cast<float*>(out_v)[o + i] = v;
    }
}

__global__ void __launch_bounds__(256)
fastagc_carry_kernel(const float* __restrict__ in, long in_stride, int block, int nblocks, float reference, FastAgcState* __restrict__ state,
                     float* __restrict__ hist, const float* __restrict__ peaks)
{
    const int c = blockIdx.x, tid = threadIdx.x;
    const float* x = in + (long)c * in_stride;
    float* h1 = hist + (long)c * 2 * block;
    float* h2 = h1 + block;
    if (nblocks >= 2) {
        for (int i = tid; i < block; i += blockDim.x) { h1[i] = x[(long)(nblocks - 2) * block + i]; h2[i] = x[(long)(nblocks - 1) * block + i]; }
    } else {
        for (int i = tid; i < block; i += blockDim.x) { const float keep = h2[i]; h1[i] = keep; h2[i] = x[i]; }
    }
    if (tid == 0) {
        const FastAgcState st = state[c];
        const float* pk = peaks + (long)c * nblocks;
        FastAgcState nx;
        nx.last_gain = agc_target(pk, st, nblocks - 1, reference);
        nx.peak_2 = agc_peak_at(pk, st, nblocks - 1);
        nx.peak_1 = agc_peak_at(pk, st, nblocks - 2);
        state[c] = nx;
    }
}

// Fused form for blocks of up to 1024 samples (the CLI default, csdr.c:1382): a CTA walks a run of consecutive blocks of one channel, computing
// each block's peak as it streams by and keeping the last two blocks in registers, so out[b] = in[b-2] * ramp(target_{b-1} -> target_b) leaves in the same
// pass.  Every input block is read once (plus three lead-in blocks per run for their peaks) instead of twice, and one launch replaces two.  Same
// arithmetic as the kernels above, element for element.  Peaks go to the scratch array for fastagc_carry_kernel.
constexpr int AGC_RUN = 16, AGC_PER = 4;

// S16 = true: the output leaves as convert_f_s16 of the scaled sample (libcsdr.c:2390-2398) -- the last two blocks of the README.md:87 NFM graph in one pass.
template <bool S16>
__global__ void __launch_bounds__(256)
fastagc_fused_kernel(const float* __restrict__ in, long in_stride, void* __restrict__ out_v, long out_stride, int block, int nblocks,
                     float reference, const FastAgcState* __restrict__ state, const float* __restrict__ hist, float* __restrict__ peaks)
{
    __shared__ float red[2][8];
    const int c = blockIdx.y, tid = threadIdx.x;
    const int b0 = blockIdx.x * AGC_RUN, b1 = min(nblocks, b0 + AGC_RUN);
    if (b0 >= nblocks) return;
    const FastAgcState st = state[c];
    const float* x = in + (long)c * in_stride;
    const float* h1 = hist + (long)c * 2 * block;
    float* pk_out = peaks + (long)c * nblocks;
    float* y = S16 ? nullptr : static_cast<float*>(out_v) + (long)c * out_stride;
    short* ys = S16 ? static_cast<short*>(out_v) + (long)c * out_stride : nullptr;
    float d2[AGC_PER], d1[AGC_PER], d0[AGC_PER];                        // data of blocks j-2, j-1, j
    float p3 = 0.f, p2 = 0.f, p1 = 0.f;                                 // peaks of blocks j-3, j-2, j-1
#pragma unroll
    for (int k = 0; k < AGC_PER; k++) d2[k] = d1[k] = 0.f;
    for (int j = b0 - 3; j < b1; j++) {
        // block j: from this call's input, from the carried history (j = -2, -1), or before it (only its peak matters: the state has it)
        float m = 0.f;
        if (j >= -2) {
            const float* src = j >= 0 ? x + (long)j * block : (j == -2 ? h1 : h1 + block);
#pragma unroll
            for (int k = 0; k < AGC_PER; k++) { const int i = tid + k * 256; d0[k] = i < block ? src[i] : 0.f; m = fmaxf(m, fabsf(d0[k])); }
        }
        float pj;
        if (j >= 0) {
            for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
            float* r = red[j & 1];
            if ((tid & 31) == 0) r[tid >> 5] = m;
            __syncthreads();
            pj = r[0];
#pragma unroll
            for (int w = 1; w < 8; w++) pj = fmaxf(pj, r[w]);
            if (j >= b0 && tid == 0) pk_out[j] = pj;
        } else pj = j == -1 ? st.peak_2 : (j == -2 ? st.peak_1 : 0.f);   // blocks before this call: their peaks are the carried state
        if (j >= b0) {
            // target_j from (p_j, p_{j-1}, p_{j-2}), target_{j-1} from (p_{j-1}, p_{j-2}, p_{j-3}); for j == 0 the previous target is the carried last_gain
            float t = pj; if (t < p1) t = p1; if (t < p2) t = p2;
            float target = __fdiv_rn(reference, t); if (target > 50.f) target = 50.f;
            float last_gain;
            if (j == 0) last_gain = st.last_gain;
            else { float u = p1; if (u < p2) u = p2; if (u < p3) u = p3; last_gain = __fdiv_rn(reference, u); if (last_gain > 50.f) last_gain = 50.f; }
#pragma unroll
            for (int k = 0; k < AGC_PER; k++) {
                const int i = tid + k * 256;
                if (i < block) {
                    const float r = __fdiv_rn((float)i, (float)block);
                    const float gain = (float)((double)last_gain * (1.0 - (double)r) + (double)__fmul_rn(target, r));
                    const float v = __fmul_rn(d2[k], gain);
                    if (S16) ys[(long)j * block + i] = (short)f_to_s16_bits(v); else y[(long)j * block + i] = v;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < AGC_PER; k++) { d2[k] = d1[k]; d1[k] = d0[k]; }
        p3 = p2; p2 = p1; p1 = pj;
    }
}

size_t fastagc_scratch_bytes(int channels, int nblocks) { return (size_t)channels * (size_t)(nblocks > 0 ? nblocks : 1) * sizeof(float); }

// blocks of up to 1024 samples: the fused kernel and the carry (2 launches); longer blocks: peaks, apply and the carry (3 launches).
// S16 = true: the output is convert_f_s16 of fastagc_ff's, short [channels][out_stride].
template <bool S16>
static int launch_fastagc(const float* d_in, long in_stride, void* d_out, long out_stride, int channels, int block, int nblocks,
                          float reference, void* d_state, float* d_hist, void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    if (channels <= 0 || nblocks <= 0) return 0;
    if (block <= 0) { set_error("fastagc: block size must be positive"); return -1; }
    if (!S16 && d_out == d_in) { set_error("fastagc: in-place operation is not supported (output lags input by two blocks)"); return -1; }
    if (!d_scratch || scratch_bytes < fastagc_scratch_bytes(channels, nblocks)) { set_error("fastagc: scratch too small"); return -1; }
    float* peaks = static_cast<float*>(d_scratch);
    int launches = 2;
    if (block <= 256 * AGC_PER) {
        fastagc_fused_kernel<S16><<<dim3((nblocks + AGC_RUN - 1) / AGC_RUN, channels), 256, 0, st>>>(d_in, in_stride, d_out, out_stride, block, nblocks, reference,
                                                                                                   static_cast<const FastAgcState*>(d_state), d_hist, peaks);
        CSDRB_CUDA(cudaGetLastError());
    } else {
        const dim3 grid(nblocks, channels);
        fastagc_peaks_kernel<<<grid, 256, 0, st>>>(d_in, in_stride, block, nblocks, peaks);
        CSDRB_CUDA(cudaGetLastError());
        fastagc_apply_kernel<S16><<<grid, 256, 0, st>>>(d_in, in_stride, d_out, out_stride, block, nblocks, reference, static_cast<const FastAgcState*>(d_state),
                                                        d_hist, peaks);
        CSDRB_CUDA(cudaGetLastError());
        launches = 3;
    }
    fastagc_carry_kernel<<<channels, 256, 0, st>>>(d_in, in_stride, block, nblocks, reference, static_cast<FastAgcState*>(d_state), d_hist, peaks);
    CSDRB_CUDA(cudaGetLastError());
    return launches;
}

// fastagc_ff | convert_f_s16 in one pass (blocks of up to 1024 samples); -2: the block size has no fused kernel
int launch_fastagc_bank_s16(const float* d_in, long in_stride, short* d_out, long out_stride, int channels, int block, int nblocks,
                            float reference, void* d_state, float* d_hist, void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    if (channels <= 0 || nblocks <= 0) return 0;
    if (block <= 0) { set_error("fastagc: block size must be positive"); return -1; }
    if (block > 256 * AGC_PER) return -2;
    return launch_fastagc<true>(d_in, in_stride, d_out, out_stride, channels, block, nblocks, reference, d_state, d_hist, d_scratch, scratch_bytes, st);
}

// the same for any block size: blocks over 1024 run peaks, apply with the s16 epilogue and carry (any row stride, no temporary)
int launch_fastagc_bank_s16_any(const float* d_in, long in_stride, short* d_out, long out_stride, int channels, int block, int nblocks,
                                float reference, void* d_state, float* d_hist, void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    return launch_fastagc<true>(d_in, in_stride, d_out, out_stride, channels, block, nblocks, reference, d_state, d_hist, d_scratch, scratch_bytes, st);
}

int launch_fastagc_bank(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int block, int nblocks,
                        float reference, void* d_state, float* d_hist, void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    return launch_fastagc<false>(d_in, in_stride, d_out, out_stride, channels, block, nblocks, reference, d_state, d_hist, d_scratch, scratch_bytes, st);
}

}  // namespace csdrb
