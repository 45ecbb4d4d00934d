// shift.cu -- K2: NCO frequency shift by phasor recursion, faithful to the reference's float arithmetic.
//
// Replaces shift_addition_cc (libcsdr_gpl.c:27-52) and decimating_shift_addition_cc (libcsdr_gpl.c:131-160).
//
// The reference's result IS its rounding sequence (SURVEY.md section 7, hard part 2): inside one call the
// phasor (cos phi, sin phi) is advanced by   c' = c*cosd - s*sind ;  s' = s*cosd + c*sind   in fp32 with
// separately rounded products (x86 SSE, no FMA); between calls the float phase is advanced by
// rate*PI*n and wrapped with while loops, and every call re-seeds the phasor from cos/sin of that float
// phase evaluated in double.  How a stream is cut into calls ("chunks", <= 1024 samples in the CLI,
// csdr.c:911-918) is therefore a parameter of the bank.
//
// Kernels:
//   shift_phase_chain_kernel : one thread per channel walks the chunk-to-chunk float phase chain
//                              (sequential by definition, a few thousand steps) and stores each chunk's seed phase.
//   shift_bank_kernel        : one lane per (channel, chunk) runs the <=chunk-step recursion; a warp owns 32
//                              consecutive chunks and moves data through a padded shared tile so that every
//                              global access is a coalesced 256-byte row while each lane walks its own row.
//   dshift_kernel            : decimating variant, one thread per channel (chains of a few hundred outputs).
// All products/sums use __fmul_rn/__fadd_rn/__fsub_rn so nvcc cannot contract them into FMAs.
#include "common.cuh"
#include "phase_table.cuh"
#include <climits>
#include "kernels.h"
#include "side_stream.cuh"
#include <cstdlib>

namespace csdrb {

#define PI_F 3.14159265358979323846f            // (float)3.14159265358979323846, libcsdr.h:65

__device__ __forceinline__ float wrap_pm_pi(float ph) { return wrap_phase_pm_pi(ph); }   // exact fast-forward, common.cuh
__device__ __forceinline__ float advance_phase(float ph, float rate2, int n)
{
    // starting_phase += d.rate*PI*input_size  (float*float -> float, * (float)int -> float, += float)
    return wrap_pm_pi(__fadd_rn(ph, __fmul_rn(__fmul_rn(rate2, PI_F), (float)n)));
}

// A chain of more than kChainTableMin steps first builds its increment's wrap table (phase_table.cuh: ~150 dependent cycles per step
// instead of ~1 200; the build costs about as much as thirty direct steps).  The last, shorter chunk has its own increment: direct.
constexpr int kChainTableMin = 96;

// chains of nchunks starting phases, one WARP per CHAIN_CPW channels: steps with the full-chunk increment go through the register-resident wrap tables
// (phase_table.cuh), the last, shorter chunk has its own increment (direct); 32 phases per channel are stored at a time.  `step(slot, ph, len)` is the direct
// form for slot's channel.  (Four channels per warp do not interleave: the wrap's branches and votes keep the chains in program order, so a
// warp per channel is faster; the constant stays 1.)
constexpr int CHAIN_CPW = 1;
constexpr int CHAIN_WARPS = 1;                    // chains per CTA: a chain slice runs next to the main kernel of the previous slice and must fit into what that leaves of an SM (see ddc_bank.cu)

template <class Step>
__device__ __forceinline__ void chain_walk(float* __restrict__ phase_io, float* __restrict__ dst, long dst_stride, int c0, int channels, int n, int chunk, int nchunks,
                                           const float (&inc_full)[CHAIN_CPW], WrapTable* __restrict__ tables, Step step, bool build_table = true)
{
    const int lane = threadIdx.x & 31;
    const int nc = min(CHAIN_CPW, channels - c0);
    const bool tab = tables != nullptr;
    WrapLanes w[CHAIN_CPW];
    if (tab) {
        if (build_table && lane < nc) {                                 // lane i builds channel c0 + i's table
            float inc = inc_full[0];
#pragma unroll
            for (int i = 1; i < CHAIN_CPW; i++) if (lane == i) inc = inc_full[i];
            wrap_table_build(inc, tables + c0 + lane);
        }
        __syncwarp();
#pragma unroll
        for (int i = 0; i < CHAIN_CPW; i++) w[i] = wrap_lanes_load(tables + min(c0 + i, channels - 1), lane);
    }
    float ph[CHAIN_CPW], mine[CHAIN_CPW];
#pragma unroll
    for (int i = 0; i < CHAIN_CPW; i++) { ph[i] = phase_io[min(c0 + i, channels - 1)]; mine[i] = 0.f; }   // slots past the bank shadow its last channel
    __syncwarp();                                                       // every lane has read the carried phases before lane 0 overwrites them
    for (int k = 0; k < nchunks; k++) {
        if ((k & 31) == lane) {
#pragma unroll
            for (int i = 0; i < CHAIN_CPW; i++) mine[i] = ph[i];
        }
        if (((k & 31) == 31 || k == nchunks - 1) && (k & ~31) + lane <= k) {
#pragma unroll
            for (int i = 0; i < CHAIN_CPW; i++) if (i < nc) dst[(long)(c0 + i) * dst_stride + (k & ~31) + lane] = mine[i];
        }
        const int len = min(chunk, n - k * chunk);
        if (tab && len == chunk) {
#pragma unroll
            for (int i = 0; i < CHAIN_CPW; i++) ph[i] = wrap_after_add_warp(__fadd_rn(ph[i], inc_full[i]), w[i]);
        } else {
#pragma unroll
            for (int i = 0; i < CHAIN_CPW; i++) ph[i] = step(i, ph[i], len);
        }
    }
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < CHAIN_CPW; i++) if (i < nc) phase_io[c0 + i] = ph[i];
    }
}

// One slice of the chain: chunks k_first .. k_first + k_count - 1 of every channel (the launcher cuts a long chain into slices so that the main kernel can
// start on slice 0 while slice 1 is still being walked); the carried phase in phase_io moves on slice by slice, the wrap table is built by the first one.
__global__ void __launch_bounds__(32 * CHAIN_WARPS)
shift_phase_chain_kernel(const float3* __restrict__ params, float* __restrict__ phase_io, float* __restrict__ chunk_phase,
                         int channels, int n, int chunk, int nchunks, WrapTable* __restrict__ tables, int k_first, int k_count)
{
    const int c0 = (blockIdx.x * CHAIN_WARPS + (threadIdx.x >> 5)) * CHAIN_CPW;
    if (c0 >= channels) return;
    const int count = min(k_count, nchunks - k_first);
    if (count <= 0) return;
    float rate2[CHAIN_CPW], inc[CHAIN_CPW];
#pragma unroll
    for (int i = 0; i < CHAIN_CPW; i++) { rate2[i] = params[min(c0 + i, channels - 1)].z; inc[i] = __fmul_rn(__fmul_rn(rate2[i], PI_F), (float)chunk); }
    chain_walk(phase_io, chunk_phase + k_first, nchunks, c0, channels, n - k_first * chunk, chunk, count, inc, tables,
               [&rate2](int i, float ph, int len) { return advance_phase(ph, rate2[i], len); }, k_first == 0);
}

constexpr int SH_TILE = 32;                       // samples per lane per sub-step

// Load `rows` rows of 32 consecutive samples into the padded tile: row r covers stream positions (k0 + r)*seg + t0 .. +31 (zeros past the row's
// length).  Eight rows' loads are issued before the first shared store -- a load-then-store loop serialises one DRAM/L2 round trip per row.
__device__ __forceinline__ void tile_load_rows(float2* __restrict__ tile, const float2* __restrict__ x, int rows, int k0, int seg, int n, int t0, int lane, int pitch)
{
    for (int r0 = 0; r0 < rows; r0 += 8) {
        float2 v[8];
#pragma unroll
        for (int u = 0; u < 8; u++) {
            const int r = r0 + u;
            const int len_r = r < rows ? min(seg, n - (k0 + r) * seg) : 0;
            v[u] = (t0 + lane < len_r) ? x[(long)(k0 + r) * seg + t0 + lane] : make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < 8; u++) if (r0 + u < rows) tile[(r0 + u) * pitch + lane] = v[u];
    }
}
constexpr int SH_PITCH = SH_TILE + 1;             // odd pitch in 8-byte units: row-wise walks are conflict-free

// (Two double-buffered forms were slower than this kernel -- the tile of step t+1 arriving by 8-byte cp.async while step t is rotated: 32 x 32
// tiles, 67 KB per CTA; 32 x 16 tiles in the same shared memory as here with the rotation in registers -- against this
// plain load / rotate / store form with its 24 resident warps per SM.)
__global__ void __launch_bounds__(128)
shift_bank_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride,
                  const float3* __restrict__ params, const float* __restrict__ chunk_phase, int n, int chunk, int nchunks, int k_first, int k_end)
{
    __shared__ float2 tile_all[4][32 * SH_PITCH];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2* tile = tile_all[warp];
    const int ch = blockIdx.y;
    const int k0 = k_first + (blockIdx.x * 4 + warp) * 32;    // first chunk of this warp; [k_first, k_end) is the launcher's slice of the chunk range
    if (k0 >= k_end) return;
    const float2* x = in + (long)ch * in_stride;
    float2* y = out + (long)ch * out_stride;
    const float3 p = params[ch];
    const float sind = p.x, cosd = p.y;
    const int k = k0 + lane;
    const bool live = k < k_end;
    const int my_len = live ? min(chunk, n - k * chunk) : 0;
    float c = 0.f, s = 0.f;
    if (live) {
        const double ph = (double)chunk_phase[(long)ch * nchunks + k];
        c = (float)cos(ph); s = (float)sin(ph);
    }
    const int rows = min(32, k_end - k0);
    const int max_len = min(chunk, n - k0 * chunk);          // the first chunk of the warp is never the short one
    for (int t0 = 0; t0 < max_len; t0 += SH_TILE) {
        // coalesced load: row r = chunk k0+r, 32 consecutive samples starting at t0
        tile_load_rows(tile, x, rows, k0, chunk, n, t0, lane, SH_PITCH);
        __syncwarp();
        if (live) {
            float2* row = tile + lane * SH_PITCH;
            const int steps = min(SH_TILE, my_len - t0);
            for (int j = 0; j < steps; j++) {
                const float2 v = row[j];
                row[j] = make_float2(__fsub_rn(__fmul_rn(c, v.x), __fmul_rn(s, v.y)), __fadd_rn(__fmul_rn(s, v.x), __fmul_rn(c, v.y)));
                const float cn = __fsub_rn(__fmul_rn(c, cosd), __fmul_rn(s, sind));
                const float sn = __fadd_rn(__fmul_rn(s, cosd), __fmul_rn(c, sind));
                c = cn; s = sn;
            }
        }
        __syncwarp();
        for (int r = 0; r < rows; r++) {
            const long pos = (long)(k0 + r) * chunk + t0 + lane;
            const int len_r = min(chunk, n - (k0 + r) * chunk);
            if (t0 + lane < len_r) y[pos] = tile[r * SH_PITCH + lane];
        }
        __syncwarp();
    }
}

// shift_addfast_cc (libcsdr.c:396-433, the plain-C branch): the same recursion advanced once per FOUR samples -- each group's phasors
// are the previous group's last phasor times four fixed steps (dsin/dcos[0..3] = 1..4 increments, shift_addfast_init :307-317).
// Same decomposition as above: a float phase chain between calls (n * phase_increment, wrapped to +-pi) and one lane per
// (channel, call) walking its own shared-memory row.  A call only touches input_size/4 groups: the n%4 tail is not written.
struct AddFastParams { float dsin[4], dcos[4], inc; };                 // = shift_addfast_data_t (libcsdr.h:189-194)

__global__ void __launch_bounds__(32 * CHAIN_WARPS)
addfast_phase_chain_kernel(const AddFastParams* __restrict__ params, float* __restrict__ phase_io, float* __restrict__ chunk_phase,
                           int channels, int n, int chunk, int nchunks, WrapTable* __restrict__ tables)
{
    const int c0 = (blockIdx.x * CHAIN_WARPS + (threadIdx.x >> 5)) * CHAIN_CPW;
    if (c0 >= channels) return;
    float inc1[CHAIN_CPW], inc[CHAIN_CPW];
#pragma unroll
    for (int i = 0; i < CHAIN_CPW; i++) { inc1[i] = params[min(c0 + i, channels - 1)].inc; inc[i] = __fmul_rn((float)chunk, inc1[i]); }
    // starting_phase += input_size * d->phase_increment  (:428)
    chain_walk(phase_io, chunk_phase, nchunks, c0, channels, n, chunk, nchunks, inc, tables,
               [&inc1](int i, float ph, int len) { return wrap_pm_pi(__fadd_rn(ph, __fmul_rn((float)len, inc1[i]))); });
}

__global__ void __launch_bounds__(128)
shift_addfast_bank_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride,
                          const AddFastParams* __restrict__ params, const float* __restrict__ chunk_phase, int n, int chunk, int nchunks)
{
    __shared__ float2 tile_all[4][32 * SH_PITCH];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2* tile = tile_all[warp];
    const int ch = blockIdx.y;
    const int k0 = (blockIdx.x * 4 + warp) * 32;              // first call ("chunk") of this warp
    if (k0 >= nchunks) return;
    const float2* x = in + (long)ch * in_stride;
    float2* y = out + (long)ch * out_stride;
    float ds[4], dc[4];
#pragma unroll
    for (int q = 0; q < 4; q++) { ds[q] = params[ch].dsin[q]; dc[q] = params[ch].dcos[q]; }
    const int k = k0 + lane;
    const bool live = k < nchunks;
    const int my_len = live ? (min(chunk, n - k * chunk) & ~3) : 0;   // whole groups of four only
    float c = 0.f, s = 0.f;
    if (live) {
        const double ph = (double)chunk_phase[(long)ch * nchunks + k];
        c = (float)cos(ph); s = (float)sin(ph);
    }
    const int rows = min(32, nchunks - k0);
    const int max_len = min(chunk, n - k0 * chunk);          // the first call of the warp is never the short one
    for (int t0 = 0; t0 < max_len; t0 += SH_TILE) {
        tile_load_rows(tile, x, rows, k0, chunk, n, t0, lane, SH_PITCH);
        __syncwarp();
        if (live) {
            float2* row = tile + lane * SH_PITCH;
            const int steps = min(SH_TILE, my_len - t0);     // a multiple of 4 (SH_TILE is), <= 0 past the end of a short call
            for (int j = 0; j < steps; j += 4) {
                float cg[4], sg[4];
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    cg[q] = __fsub_rn(__fmul_rn(c, dc[q]), __fmul_rn(s, ds[q]));
                    sg[q] = __fadd_rn(__fmul_rn(s, dc[q]), __fmul_rn(c, ds[q]));
                }
#pragma unroll
                for (int q = 0; q < 4; q++) {
                    const float2 v = row[j + q];
                    row[j + q] = make_float2(__fsub_rn(__fmul_rn(cg[q], v.x), __fmul_rn(sg[q], v.y)), __fadd_rn(__fmul_rn(sg[q], v.x), __fmul_rn(cg[q], v.y)));
                }
                c = cg[3]; s = sg[3];
            }
        }
        __syncwarp();
        for (int r = 0; r < rows; r++) {
            const long pos = (long)(k0 + r) * chunk + t0 + lane;
            const int len_r = min(chunk, n - (k0 + r) * chunk) & ~3;
            if (t0 + lane < len_r) y[pos] = tile[r * SH_PITCH + lane];
        }
        __syncwarp();
    }
}

// shift_math_cc (libcsdr.c:186-209): no phasor recursion -- each sample is rotated by cos/sin of a float phase that advances by ONE ROUNDED
// ADDITION PER SAMPLE and is wrapped into [0, 2*PI] by the reference's while loops.  That chain is sequential over the whole stream, so it
// is walked once per channel by one thread which drops a seed every MATH_SEG samples (shift_math_chain_kernel); the expensive part, a
// double-precision sincos per sample, then runs with one lane per (channel, segment) re-walking its MATH_SEG additions
// (shift_math_bank_kernel, same padded-tile data movement as shift_bank_kernel).  Bit-exact phases, samples within an ulp of the seed.
constexpr int MATH_SEG = 256;
#define TWO_PI_F 6.28318530717958647692f          // 2*PI in float arithmetic: (float)2 * PI_F rounds to this float

__device__ __forceinline__ float math_step(float ph, float inc)
{
    ph = __fadd_rn(ph, inc);
    if (!(fabsf(ph) < 67108864.f)) return ph;                 // the reference's loops would not terminate here either (2*PI below one ulp)
    while (ph > TWO_PI_F) ph = __fsub_rn(ph, TWO_PI_F);       // libcsdr.c:205-206, literally: a huge starting phase takes many rounded steps
    while (ph < 0.f) ph = __fadd_rn(ph, TWO_PI_F);
    return ph;
}

__global__ void shift_math_chain_kernel(const float* __restrict__ rates, float* __restrict__ phase_io, float* __restrict__ seg_phase,
                                        int channels, int n, int nseg)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= channels) return;
    const float inc = __fmul_rn(__fmul_rn(rates[c], 2.f), PI_F);     // rate *= 2; phase_increment = rate*PI  (:188,191)
    float ph = phase_io[c];
    for (int k = 0; k < nseg; k++) {
        seg_phase[(long)c * nseg + k] = ph;
        const int len = min(MATH_SEG, n - k * MATH_SEG);
        for (int j = 0; j < len; j++) ph = math_step(ph, inc);
    }
    phase_io[c] = ph;
}

__global__ void __launch_bounds__(128)
shift_math_bank_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride,
                       const float* __restrict__ rates, const float* __restrict__ seg_phase, int n, int nseg)
{
    __shared__ float2 tile_all[4][32 * SH_PITCH];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2* tile = tile_all[warp];
    const int ch = blockIdx.y;
    const int k0 = (blockIdx.x * 4 + warp) * 32;              // first segment of this warp
    if (k0 >= nseg) return;
    const float2* x = in + (long)ch * in_stride;
    float2* y = out + (long)ch * out_stride;
    const float inc = __fmul_rn(__fmul_rn(rates[ch], 2.f), PI_F);
    const int k = k0 + lane;
    const bool live = k < nseg;
    const int my_len = live ? min(MATH_SEG, n - k * MATH_SEG) : 0;
    float ph = live ? seg_phase[(long)ch * nseg + k] : 0.f;
    const int rows = min(32, nseg - k0);
    const int max_len = min(MATH_SEG, n - k0 * MATH_SEG);    // the first segment of the warp is never the short one
    for (int t0 = 0; t0 < max_len; t0 += SH_TILE) {
        tile_load_rows(tile, x, rows, k0, MATH_SEG, n, t0, lane, SH_PITCH);
        __syncwarp();
        if (live) {
            float2* row = tile + lane * SH_PITCH;
            const int steps = min(SH_TILE, my_len - t0);
            for (int j = 0; j < steps; j++) {
                const float c = (float)cos((double)ph), s = (float)sin((double)ph);
                const float2 v = row[j];
                row[j] = make_float2(__fsub_rn(__fmul_rn(c, v.x), __fmul_rn(s, v.y)), __fadd_rn(__fmul_rn(s, v.x), __fmul_rn(c, v.y)));
                ph = math_step(ph, inc);
            }
        }
        __syncwarp();
        for (int r = 0; r < rows; r++) {
            const long pos = (long)(k0 + r) * MATH_SEG + t0 + lane;
            const int len_r = min(MATH_SEG, n - (k0 + r) * MATH_SEG);
            if (t0 + lane < len_r) y[pos] = tile[r * SH_PITCH + lane];
        }
        __syncwarp();
    }
}

// shift_table_cc (libcsdr.c:223-260): the same per-sample phase chain as shift_math_cc (seeds from shift_math_chain_kernel), but cos/sin come
// from a quarter-wave table.  A table step is 2.4e-5 rad, far above the 1e-5 bar, so the index arithmetic has to be the reference BUILD's:
// under -ffast-math its two divisions by PI/2 are multiplications by float constants (see oracle.c).  Indices the source would read outside
// the table (it is marked "RTODO") are clamped.
__global__ void __launch_bounds__(128)
shift_table_bank_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride,
                        const float* __restrict__ rates, const float* __restrict__ seg_phase, const float* __restrict__ table, int table_size,
                        int n, int nseg)
{
    __shared__ float2 tile_all[4][32 * SH_PITCH];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2* tile = tile_all[warp];
    const int ch = blockIdx.y;
    const int k0 = (blockIdx.x * 4 + warp) * 32;
    if (k0 >= nseg) return;
    const float2* x = in + (long)ch * in_stride;
    float2* y = out + (long)ch * out_stride;
    const float inc = __fmul_rn(__fmul_rn(rates[ch], 2.f), PI_F);
    const float K = 0.6366197466850281f;                                 // fl(1 / fl(PI/2)), the constant the reference build multiplies by
    const float HALF_PI = 1.5707963705062866f;                           // fl(PI/2)
    const float K2 = __fmul_rn((float)table_size, K);
    const int k = k0 + lane;
    const bool live = k < nseg;
    const int my_len = live ? min(MATH_SEG, n - k * MATH_SEG) : 0;
    float ph = live ? seg_phase[(long)ch * nseg + k] : 0.f;
    const int rows = min(32, nseg - k0);
    const int max_len = min(MATH_SEG, n - k0 * MATH_SEG);
    for (int t0 = 0; t0 < max_len; t0 += SH_TILE) {
        for (int r = 0; r < rows; r++) {
            const long pos = (long)(k0 + r) * MATH_SEG + t0 + lane;
            const int len_r = min(MATH_SEG, n - (k0 + r) * MATH_SEG);
            tile[r * SH_PITCH + lane] = (t0 + lane < len_r) ? x[pos] : make_float2(0.f, 0.f);
        }
        __syncwarp();
        if (live) {
            float2* row = tile + lane * SH_PITCH;
            const int steps = min(SH_TILE, my_len - t0);
            for (int j = 0; j < steps; j++) {
                const float qf = __fmul_rn(ph, K);
                const int quadrant = (fabsf(qf) < 2147483648.0f) ? __float2int_rz(qf) : INT_MIN;     // cvttss2si
                const float vphase = __fsub_rn(ph, __fmul_rn((float)quadrant, HALF_PI));
                const float fi = __fmul_rn(vphase, K2);
                int si = (fabsf(fi) < 2147483648.0f) ? __float2int_rz(fi) : INT_MIN;
                int ci = table_size - 1 - si;
                if (quadrant & 1) { const int t = si; si = ci; ci = t; }
                si = min(table_size - 1, max(0, si)); ci = min(table_size - 1, max(0, ci));           // the source would read outside the table here
                const float s = (quadrant > 1 ? -1.0f : 1.0f) * __ldg(table + si);
                const float c = ((quadrant && quadrant < 3) ? -1.0f : 1.0f) * __ldg(table + ci);
                const float2 v = row[j];
                row[j] = make_float2(__fsub_rn(__fmul_rn(c, v.x), __fmul_rn(s, v.y)), __fadd_rn(__fmul_rn(s, v.x), __fmul_rn(c, v.y)));
                ph = math_step(ph, inc);
            }
        }
        __syncwarp();
        for (int r = 0; r < rows; r++) {
            const long pos = (long)(k0 + r) * MATH_SEG + t0 + lane;
            const int len_r = min(MATH_SEG, n - (k0 + r) * MATH_SEG);
            if (t0 + lane < len_r) y[pos] = tile[r * SH_PITCH + lane];
        }
        __syncwarp();
    }
}

// decimating variant: status per channel {decimation_remain, starting_phase, output_size} (libcsdr_gpl.h:39-44)
__global__ void dshift_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride,
                              const float3* __restrict__ params, int n, int decimation, int* __restrict__ remain_io,
                              float* __restrict__ phase_io, int* __restrict__ out_size, int channels)
{
    const int ch = blockIdx.x * blockDim.x + threadIdx.x;
    if (ch >= channels) return;
    const float2* x = in + (long)ch * in_stride;
    float2* y = out + (long)ch * out_stride;
    const float3 p = params[ch];
    const float ph0 = phase_io[ch];
    float c = (float)cos((double)ph0), s = (float)sin((double)ph0);
    int produced = 0, pos;
    for (pos = remain_io[ch]; pos < n; pos += decimation) {
        const float2 v = x[pos];
        y[produced++] = make_float2(__fsub_rn(__fmul_rn(c, v.x), __fmul_rn(s, v.y)), __fadd_rn(__fmul_rn(s, v.x), __fmul_rn(c, v.y)));
        const float cn = __fsub_rn(__fmul_rn(c, p.y), __fmul_rn(s, p.x));
        const float sn = __fadd_rn(__fmul_rn(s, p.y), __fmul_rn(c, p.x));
        c = cn; s = sn;
    }
    remain_io[ch] = pos - n;
    phase_io[ch] = advance_phase(ph0, p.z, produced);
    if (out_size) out_size[ch] = produced;
}

// shift_unroll_cc (libcsdr.c:301-320): every sample of a call is rotated by (phasor at the call's start) x (table entry i), no
// recursion -- fully parallel once the per-call start phases are known.  The phase chain between calls is the same float chain as
// shift_addition_cc's (n * phase_increment with phase_increment = 2*rate*PI), so the same pre-pass kernel serves both.
__global__ void __launch_bounds__(256)
shift_unroll_bank_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride,
                         const float* __restrict__ dsin, const float* __restrict__ dcos, long table_stride,
                         const float* __restrict__ chunk_phase, int n, int chunk, int nchunks)
{
    const int ch = blockIdx.y;
    const float2* x = in + (long)ch * in_stride;
    float2* y = out + (long)ch * out_stride;
    const float* ts = dsin + (long)ch * table_stride;
    const float* tc = dcos + (long)ch * table_stride;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int k = i / chunk, j = i - k * chunk;
        const double ph = (double)chunk_phase[(long)ch * nchunks + k];
        const float c0 = (float)cos(ph), s0 = (float)sin(ph);
        const float dc = __ldg(tc + j), ds = __ldg(ts + j);
        const float c = __fsub_rn(__fmul_rn(c0, dc), __fmul_rn(s0, ds));
        const float s = __fadd_rn(__fmul_rn(s0, dc), __fmul_rn(c0, ds));
        const float2 v = x[i];
        y[i] = make_float2(__fsub_rn(__fmul_rn(c, v.x), __fmul_rn(s, v.y)), __fadd_rn(__fmul_rn(s, v.x), __fmul_rn(c, v.y)));
    }
}

static inline WrapTable* chain_tables(void* d_scratch, size_t scratch_bytes, int channels, int nchunks);

int launch_shift_unroll_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n,
                             const float* d_params, const float* d_dsin, const float* d_dcos, long table_stride, int table_size,
                             float* d_phase_io, void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (table_size <= 0) { set_error("shift_unroll bank: table size must be positive"); return -1; }
    const int chunk = table_size < n ? table_size : n;                  // one reference call per `table_size` samples (csdr.c:834-841)
    const int nchunks = (n + chunk - 1) / chunk;
    if (scratch_bytes < (size_t)channels * nchunks * sizeof(float) || !d_scratch) { set_error("shift_unroll bank: scratch too small"); return -1; }
    float* chunk_phase = static_cast<float*>(d_scratch);
    shift_phase_chain_kernel<<<(channels + CHAIN_CPW * CHAIN_WARPS - 1) / (CHAIN_CPW * CHAIN_WARPS), 32 * CHAIN_WARPS, 0, st>>>(reinterpret_cast<const float3*>(d_params), d_phase_io, chunk_phase, channels, n, chunk, nchunks,
                                                               chain_tables(d_scratch, scratch_bytes, channels, nchunks), 0, nchunks);
    CSDRB_CUDA(cudaGetLastError());
    int gx = (n + 255) / 256; if (gx > 2048) gx = 2048;
    shift_unroll_bank_kernel<<<dim3(gx, channels), 256, 0, st>>>(d_in, in_stride, d_out, out_stride, d_dsin, d_dcos, table_stride, chunk_phase, n, chunk, nchunks);
    CSDRB_CUDA(cudaGetLastError());
    return 2;
}

// one reference call (n <= table size) from a known starting phase: the drop-in path of shift_unroll_cc
void shift_unroll_bank_single(const float2* d_in, float2* d_out, int n, const float* d_dsin, const float* d_dcos, const float* d_phase, cudaStream_t st)
{
    int gx = (n + 255) / 256; if (gx > 2048) gx = 2048;
    shift_unroll_bank_kernel<<<dim3(gx, 1), 256, 0, st>>>(d_in, 0, d_out, 0, d_dsin, d_dcos, 0, d_phase, n, n, 1);
}

size_t shift_bank_scratch_bytes(int channels, int n, int chunk)
{
    if (chunk <= 0 || chunk > n) chunk = n > 0 ? n : 1;
    const int nchunks = (n + chunk - 1) / chunk;
    const size_t phases = ((size_t)channels * (size_t)(nchunks > 0 ? nchunks : 1) * sizeof(float) + 15) & ~(size_t)15;
    return phases + (nchunks > kChainTableMin ? (size_t)channels * sizeof(WrapTable) : 0);
}
// the wrap tables sit behind the chunk phases when the caller's scratch has room for them (it has, if it was sized by the function above)
static inline WrapTable* chain_tables(void* d_scratch, size_t scratch_bytes, int channels, int nchunks)
{
    const size_t phases = ((size_t)channels * (size_t)nchunks * sizeof(float) + 15) & ~(size_t)15;
    if (nchunks <= kChainTableMin || scratch_bytes < phases + (size_t)channels * sizeof(WrapTable)) return nullptr;
    return reinterpret_cast<WrapTable*>(static_cast<char*>(d_scratch) + phases);
}

int launch_shift_addition_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n,
                               const float* d_params /*[C][3] sindelta,cosdelta,rate*/, float* d_phase_io, int chunk,
                               void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (chunk <= 0 || chunk > n) chunk = n;
    const int nchunks = (n + chunk - 1) / chunk;
    if (scratch_bytes < shift_bank_scratch_bytes(channels, n, chunk) || !d_scratch) { set_error("shift_addition bank: scratch too small"); return -1; }
    float* chunk_phase = static_cast<float*>(d_scratch);
    const float3* prm = reinterpret_cast<const float3*>(d_params);
    WrapTable* tables = chain_tables(d_scratch, scratch_bytes, channels, nchunks);
    constexpr size_t smem = 0;                                          // the tiles are static shared memory
    // The chain is one warp per channel and sequential: a long one is cut into up to three slices that run on a side stream, the main
    // kernel follows slice by slice on the caller's stream.  A slice must still fill the machine (a warp walks its 32 chunks tile after tile:
    // eight slices of 384 chunks x 64 channels run the main kernel at under half a wave and gain nothing).  CSDRB_SHIFT_SLICES=1: one stream.
    static const int max_slices = getenv("CSDRB_SHIFT_SLICES") ? atoi(getenv("CSDRB_SHIFT_SLICES")) : 3;
    static const long slice_min = getenv("CSDRB_SHIFT_SLICE_MIN") ? atol(getenv("CSDRB_SHIFT_SLICE_MIN")) : 768L * 64;   // chunk-channels a slice needs to fill the machine (the CPU tier lowers it)
    int slices = (int)(((long)nchunks * channels) / (slice_min > 0 ? slice_min : 1));
    if (slices > max_slices) slices = max_slices;
    if (slices > kSideSlices) slices = kSideSlices;
    if (slices < 2) {
        shift_phase_chain_kernel<<<(channels + CHAIN_CPW * CHAIN_WARPS - 1) / (CHAIN_CPW * CHAIN_WARPS), 32 * CHAIN_WARPS, 0, st>>>(prm, d_phase_io, chunk_phase, channels, n, chunk, nchunks, tables, 0, nchunks);
        CSDRB_CUDA(cudaGetLastError());
        shift_bank_kernel<<<dim3((nchunks + 127) / 128, channels), 128, smem, st>>>(d_in, in_stride, d_out, out_stride, prm, chunk_phase, n, chunk, nchunks, 0, nchunks);
        CSDRB_CUDA(cudaGetLastError());
        return 2;
    }
    SideStream* ss = side_stream();
    if (!ss) return -1;
    const int per = (((nchunks + slices - 1) / slices) + 127) / 128 * 128;           // whole CTAs (4 warps x 32 chunks) per slice
    std::lock_guard<std::mutex> lk(ss->mu);                             // the events are shared by every call on this device
    CSDRB_CUDA(cudaEventRecord(ss->fork, st));
    CSDRB_CUDA(cudaStreamWaitEvent(ss->stream, ss->fork, 0));
    int launches = 0;
    for (int i = 0; i < slices; i++) {
        const int k_first = i * per;
        if (k_first >= nchunks) break;
        const int k_end = k_first + per < nchunks ? k_first + per : nchunks;
        shift_phase_chain_kernel<<<(channels + CHAIN_CPW * CHAIN_WARPS - 1) / (CHAIN_CPW * CHAIN_WARPS), 32 * CHAIN_WARPS, 0, ss->stream>>>(prm, d_phase_io, chunk_phase, channels, n, chunk, nchunks, tables, k_first, k_end - k_first);
        CSDRB_CUDA(cudaGetLastError());
        CSDRB_CUDA(cudaEventRecord(ss->slice[i], ss->stream));
        CSDRB_CUDA(cudaStreamWaitEvent(st, ss->slice[i], 0));
        shift_bank_kernel<<<dim3((k_end - k_first + 127) / 128, channels), 128, smem, st>>>(d_in, in_stride, d_out, out_stride, prm, chunk_phase, n, chunk, nchunks, k_first, k_end);
        CSDRB_CUDA(cudaGetLastError());
        launches += 2;
    }
    return launches;
}

int launch_shift_addfast_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n,
                              const float* d_params /*[C][9] dsin[4],dcos[4],phase_increment*/, float* d_phase_io, int chunk,
                              void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (chunk <= 0 || chunk > n) chunk = n;
    const int nchunks = (n + chunk - 1) / chunk;
    if (scratch_bytes < shift_bank_scratch_bytes(channels, n, chunk) || !d_scratch) { set_error("shift_addfast bank: scratch too small"); return -1; }
    float* chunk_phase = static_cast<float*>(d_scratch);
    const AddFastParams* params = reinterpret_cast<const AddFastParams*>(d_params);
    addfast_phase_chain_kernel<<<(channels + CHAIN_CPW * CHAIN_WARPS - 1) / (CHAIN_CPW * CHAIN_WARPS), 32 * CHAIN_WARPS, 0, st>>>(params, d_phase_io, chunk_phase, channels, n, chunk, nchunks, chain_tables(d_scratch, scratch_bytes, channels, nchunks));
    CSDRB_CUDA(cudaGetLastError());
    dim3 grid((nchunks + 127) / 128, channels);
    shift_addfast_bank_kernel<<<grid, 128, 0, st>>>(d_in, in_stride, d_out, out_stride, params, chunk_phase, n, chunk, nchunks);
    CSDRB_CUDA(cudaGetLastError());
    return 2;
}

size_t shift_math_scratch_bytes(int channels, int n)
{
    const size_t nseg = (size_t)(((n > 0 ? n : 1) + MATH_SEG - 1) / MATH_SEG);
    return (size_t)(channels > 0 ? channels : 1) * nseg * sizeof(float) + 16;
}

int launch_shift_math_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, const float* d_rates,
                           float* d_phase_io, void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    const int nseg = (n + MATH_SEG - 1) / MATH_SEG;
    if (!d_scratch || scratch_bytes < (size_t)channels * nseg * sizeof(float)) { set_error("shift_math bank: scratch too small"); return -1; }
    float* seg_phase = static_cast<float*>(d_scratch);
    shift_math_chain_kernel<<<(channels + 63) / 64, 64, 0, st>>>(d_rates, d_phase_io, seg_phase, channels, n, nseg);
    CSDRB_CUDA(cudaGetLastError());
    dim3 grid((nseg + 127) / 128, channels);
    shift_math_bank_kernel<<<grid, 128, 0, st>>>(d_in, in_stride, d_out, out_stride, d_rates, seg_phase, n, nseg);
    CSDRB_CUDA(cudaGetLastError());
    return 2;
}

int launch_shift_table_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, const float* d_rates,
                            float* d_phase_io, const float* d_table, int table_size, void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    if (channels <= 0 || n <= 0) return 0;
    if (!d_table || table_size < 2) { set_error("shift_table bank: a table of at least two entries is needed"); return -1; }
    const int nseg = (n + MATH_SEG - 1) / MATH_SEG;
    if (!d_scratch || scratch_bytes < (size_t)channels * nseg * sizeof(float)) { set_error("shift_table bank: scratch too small"); return -1; }
    float* seg_phase = static_cast<float*>(d_scratch);
    shift_math_chain_kernel<<<(channels + 63) / 64, 64, 0, st>>>(d_rates, d_phase_io, seg_phase, channels, n, nseg);   // the same phase chain as shift_math_cc
    CSDRB_CUDA(cudaGetLastError());
    dim3 grid((nseg + 127) / 128, channels);
    shift_table_bank_kernel<<<grid, 128, 0, st>>>(d_in, in_stride, d_out, out_stride, d_rates, seg_phase, d_table, table_size, n, nseg);
    CSDRB_CUDA(cudaGetLastError());
    return 2;
}

int launch_decimating_shift_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n,
                                 const float* d_params, int decimation, int* d_remain_io, float* d_phase_io, int* d_out_size,
                                 cudaStream_t st)
{
    if (channels <= 0) return 0;
    if (decimation <= 0) { set_error("decimating_shift_addition bank: decimation must be positive"); return -1; }
    dshift_kernel<<<(channels + 63) / 64, 64, 0, st>>>(d_in, in_stride, d_out, out_stride, reinterpret_cast<const float3*>(d_params), n, decimation,
                                                       d_remain_io, d_phase_io, d_out_size, channels);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace csdrb
