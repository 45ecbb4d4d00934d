// agc.cu -- the blocks of the AM and SSB receiver graphs (reference README.md:95, :110) that follow the DDC bank:
//   amdemod_cf                     elementwise (libcsdr.c:861-873)
//   amdemod_cf | fastdcblock_ff    AM front over whole blocks, one CTA per (channel, run of blocks) (libcsdr.c:920-941)
//   [realpart_cf |] agc_ff [| limit_ff] [| convert_f_s16]    AGC tail, one serial chain per channel (libcsdr_gpl.c:163-260)
//
// The reference always builds with -O3 -ffast-math (its Makefile:38), and for fastdcblock_ff and agc_ff that build reassociates
// the source.  These kernels compute what the compiled build computes, operation for operation (DESIGN.md section 7; the CPU
// restatement is tests/am_ssb/am_ssb_oracle.c).  Every operation is an explicit _rn intrinsic so that no FMA contraction happens.
#include "common.cuh"
#include "kernels.h"

namespace csdrb {

// amdemod_cf: i*i + q*q is two separately rounded products and one sum (no FMA), then the correctly rounded square root (sqrtf is
// sqrt.rn.f32 without -use_fast_math).  The reference build's vectorised body uses rsqrtps + one Newton step instead, whose bits depend on
// the CPU vendor.
__device__ __forceinline__ float am_magnitude(float2 v) { return sqrtf(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y))); }

__global__ void __launch_bounds__(256) amdemod_cf_kernel(const float2* __restrict__ in, float* __restrict__ out, long n)
{
    const long stride = (long)gridDim.x * blockDim.x;
    for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = am_magnitude(in[i]);
}

int launch_amdemod_cf(const float2* d_in, float* d_out, long n, cudaStream_t st)
{
    if (n <= 0) return 0;
    const long blocks = (n + 255) / 256;
    amdemod_cf_kernel<<<(unsigned)(blocks < 8 * kSmCount ? blocks : 8 * kSmCount), 256, 0, st>>>(d_in, d_out, n);
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---------------------------------------------------------------------------------------------- AM front
// One CTA walks a run of DC_RUN consecutive blocks of one channel (plus the block before the run, whose average is the run's
// starting DC level).  Per block:
//   1. all threads stage the block's samples (magnitudes of cf32 input, or the float input) in shared memory, coalesced;
//   2. threads 0..3 each add one of the reference build's four interleaved partial sums, in order (lane l: elements i = l mod 4);
//      thread 0 combines them as (s0+s2)+(s1+s3) and adds the n%4 leftover elements one by one (n <= 3: one sum from 0);
//   3. avg = sum/n, k = (1/n)*(avg - last_dc); all threads write out[i] = (x[i] - last_dc) - i*k, in parallel.  The last element
//      of an odd n >= 3 comes from the build's scalar epilogue: (x[i] - i*k) - last_dc.
// The state (last_dc_level) of the channel is read by the first run and written by am_front_carry_kernel after the bank kernel.
constexpr int DC_RUN = 8, DC_THREADS = 256;

template <bool CF32>
__device__ __forceinline__ float dc_block_average(const void* __restrict__ row, long b, int block, float* __restrict__ xs, float* red)
{
    const int tid = threadIdx.x;
    for (int i = tid; i < block; i += DC_THREADS) {
        const long g = b * block + i;
        xs[i] = CF32 ? am_magnitude(static_cast<const float2*>(row)[g]) : static_cast<const float*>(row)[g];
    }
    __syncthreads();
    if (block >= 4) {
        if (tid < 4) {
            float s = 0.f;
            const int q = block >> 2;
            for (int j = 0; j < q; j++) s = __fadd_rn(s, xs[4 * j + tid]);
            red[tid] = s;
        }
        __syncthreads();
    }
    float sum;
    if (block >= 4) {
        sum = __fadd_rn(__fadd_rn(red[0], red[2]), __fadd_rn(red[1], red[3]));
        for (int i = block & ~3; i < block; i++) sum = __fadd_rn(sum, xs[i]);
    } else {
        sum = 0.f;
        for (int i = 0; i < block; i++) sum = __fadd_rn(sum, xs[i]);
    }
    return __fdiv_rn(sum, (float)block);
}

template <bool CF32>
__global__ void __launch_bounds__(DC_THREADS)
am_front_kernel(const void* __restrict__ in, long in_stride, float* __restrict__ out, long out_stride, int block, int nblocks,
                const float* __restrict__ last_dc_in)
{
    CSDRB_DYN_SMEM(smem);
    float* xs = reinterpret_cast<float*>(smem);
    __shared__ float red[4];
    const int c = blockIdx.y, tid = threadIdx.x;
    const int b0 = blockIdx.x * DC_RUN, b1 = min(nblocks, b0 + DC_RUN);
    const void* row = CF32 ? static_cast<const void*>(static_cast<const float2*>(in) + (long)c * in_stride)
                           : static_cast<const void*>(static_cast<const float*>(in) + (long)c * in_stride);
    float* y = out + (long)c * out_stride;
    float last = b0 == 0 ? last_dc_in[c] : dc_block_average<CF32>(row, b0 - 1, block, xs, red);
    const float k0 = __fdiv_rn(1.0f, (float)block);
    const int odd_tail = (block >= 3 && (block & 1)) ? block - 1 : -1;
    for (int b = b0; b < b1; b++) {
        __syncthreads();                                                   // xs / red of the previous block are consumed
        const float avg = dc_block_average<CF32>(row, b, block, xs, red);
        const float k = __fmul_rn(k0, __fsub_rn(avg, last));
        for (int i = tid; i < block; i += DC_THREADS) {
            const float ik = __fmul_rn((float)i, k);
            y[(long)b * block + i] = i == odd_tail ? __fsub_rn(__fsub_rn(xs[i], ik), last) : __fsub_rn(__fsub_rn(xs[i], last), ik);
        }
        last = avg;
    }
}

// the new last_dc_level of every channel: the average of its last block (one CTA per channel, after the bank kernel has read the old one)
template <bool CF32>
__global__ void __launch_bounds__(DC_THREADS)
am_front_carry_kernel(const void* __restrict__ in, long in_stride, int block, int nblocks, float* __restrict__ last_dc_out)
{
    CSDRB_DYN_SMEM(smem);
    float* xs = reinterpret_cast<float*>(smem);
    __shared__ float red[4];
    const int c = blockIdx.x;
    const void* row = CF32 ? static_cast<const void*>(static_cast<const float2*>(in) + (long)c * in_stride)
                           : static_cast<const void*>(static_cast<const float*>(in) + (long)c * in_stride);
    const float avg = dc_block_average<CF32>(row, nblocks - 1, block, xs, red);
    if (threadIdx.x == 0) last_dc_out[c] = avg;
}

constexpr int kDcMaxBlock = 49152;                                        // 192 KB of shared memory per CTA

// cf32 = 1: d_in is cf32 rows (amdemod_cf | fastdcblock_ff); 0: float rows (fastdcblock_ff).  Returns the launch count.
int launch_fastdcblock_bank(const void* d_in, long in_stride, int cf32, float* d_out, long out_stride, int channels, int block, int nblocks,
                            float* d_last_dc_io, cudaStream_t st)
{
    if (channels <= 0 || nblocks <= 0) return 0;
    if (block <= 0) { set_error("fastdcblock bank: block size must be positive"); return -1; }
    if (block > kDcMaxBlock) { set_error("fastdcblock bank: block size %d above the %d samples one CTA can stage", block, kDcMaxBlock); return -1; }
    if (channels > 65535) { set_error("fastdcblock bank: more than 65535 channels in one call"); return -1; }
    if (in_stride < (long)block * nblocks || out_stride < (long)block * nblocks) { set_error("fastdcblock bank: row stride shorter than the row"); return -1; }
    const size_t smem = (size_t)block * sizeof(float);
    const dim3 grid((unsigned)((nblocks + DC_RUN - 1) / DC_RUN), (unsigned)channels);
    CSDRB_CUDA(launch_kernel(cf32 ? am_front_kernel<true> : am_front_kernel<false>, grid, DC_THREADS, smem, st, d_in, in_stride, d_out, out_stride, block, nblocks,
                             d_last_dc_io));
    CSDRB_CUDA(launch_kernel(cf32 ? am_front_carry_kernel<true> : am_front_carry_kernel<false>, channels, DC_THREADS, smem, st, d_in, in_stride, block, nblocks,
                             d_last_dc_io));
    return 2;
}

// ---------------------------------------------------------------------------------------------- AGC tail
// agc_ff is a nonlinear feedback loop: sample i needs the gain after sample i-1, so each channel is one serial chain.  A CTA
// owns AGC_CH = 32 channels; lane t of warp 0 runs the chain of channel c0 + t.  The other warps keep that lane from waiting on
// global memory or on the division: they stage tiles of AGC_T samples x 32 channels through shared memory (coalesced along the
// samples), compute reference/|x| for the tile with the same __fdiv_rn, and write the finished tile back.  Three tile buffers
// rotate: at step k the loaders fill tile k and drain tile k-2 while the chain lane works through tile k-1.
//
// The per-sample chain is the reference build's (libcsdr_gpl.c:185-257 under -O3 -ffast-math; gain and last_gain share a register):
//   x == 0 or NaN: v = g                                                                    (comiss / je)
//   else err = reference/|x| - g;
//        0 > err: reload = |x| > last_peak; last_peak = last_peak > |x| ? last_peak : |x|;  reload: awc = attack_wait
//                 awc > 0 ? (awc--, v = g) : (v = err*attack_rate + g, hc = hang_time)
//        else   : hc > 0 ? (hc--, v = g) : v = err*decay_rate + g
//   g = g*(1 - alpha) + max(min(v, max_gain), 0);   y = x*g
// and the first sample of every agc_ff call (absolute multiples of `chunk` from stream start, csdr.c:1363-1372) is y = g*x with the
// counters reset and last_peak = reference/g.
constexpr int AGC_CH = 32, AGC_T = 32, AGC_WARPS = 4, AGC_PITCH = AGC_T + 1;

struct AgcTile { float x[AGC_CH][AGC_PITCH]; float r[AGC_CH][AGC_PITCH]; };

template <bool CF32, bool S16, bool LIMIT>
__global__ void __launch_bounds__(AGC_WARPS * 32)
agc_bank_kernel(const void* __restrict__ in, long in_stride, void* __restrict__ out, long out_stride, int channels, int n,
                AgcParams p, AgcState* __restrict__ state, float limit_max)
{
    __shared__ AgcTile tiles[3];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int c0 = blockIdx.x * AGC_CH;
    const int ntiles = (n + AGC_T - 1) / AGC_T;
    if (warp == 0) {
        const int c = c0 + lane;
        AgcState s = c < channels ? state[c] : AgcState{1.f, 0.f, 0, 0, 0};
        const float one_minus_alpha = __fsub_rn(1.0f, p.gain_filter_alpha);
        for (int k = 0; k <= ntiles + 1; k++) {
            const int t = k - 1;
            if (t >= 0 && t < ntiles && c < channels) {
                AgcTile& tl = tiles[t % 3];
                const int m = min(AGC_T, n - t * AGC_T);
                float g = s.gain;
                for (int i = 0; i < m; i++) {
                    const float x = tl.x[lane][i];
                    float y;
                    if (s.offset == 0) {                                        // first sample of an agc_ff call
                        s.hang_counter = 0; s.attack_wait_counter = 0;
                        s.last_peak = __fdiv_rn(p.reference, g);
                        y = __fmul_rn(g, x);
                    } else {
                        float v = g;
                        if (!(x == 0.f || x != x)) {
                            const float a = fabsf(x);
                            const float err = __fsub_rn(tl.r[lane][i], g);
                            if (0.f > err) {
                                const bool reload = a > s.last_peak;
                                s.last_peak = s.last_peak > a ? s.last_peak : a;
                                if (reload) s.attack_wait_counter = p.attack_wait_time;
                                if (s.attack_wait_counter > 0) s.attack_wait_counter--;
                                else { v = __fadd_rn(__fmul_rn(err, p.attack_rate), g); s.hang_counter = p.hang_time; }
                            } else {
                                if (s.hang_counter > 0) s.hang_counter--;
                                else v = __fadd_rn(__fmul_rn(err, p.decay_rate), g);
                            }
                        }
                        float cl = v < p.max_gain ? v : p.max_gain;
                        cl = cl > 0.f ? cl : 0.f;
                        g = __fadd_rn(__fmul_rn(g, one_minus_alpha), cl);
                        y = __fmul_rn(x, g);
                    }
                    if (++s.offset >= p.chunk) s.offset = 0;           // >=: a state carried from a call with a longer chunk
                    tl.x[lane][i] = y;
                }
                s.gain = g;
            }
            __syncthreads();
        }
        if (c < channels) state[c] = s;
    } else {
        const int ltid = tid - 32, nl = (AGC_WARPS - 1) * 32;
        for (int k = 0; k <= ntiles + 1; k++) {
            if (k < ntiles) {                                                   // fill tile k: x and reference/|x|
                AgcTile& tl = tiles[k % 3];
                for (int e = ltid; e < AGC_CH * AGC_T; e += nl) {
                    const int ch = e / AGC_T, i = e % AGC_T, c = c0 + ch;
                    const long pos = (long)k * AGC_T + i;
                    float x = 0.f;
                    if (c < channels && pos < n)
                        x = CF32 ? static_cast<const float2*>(in)[(long)c * in_stride + pos].x : static_cast<const float*>(in)[(long)c * in_stride + pos];
                    tl.x[ch][i] = x;
                    tl.r[ch][i] = __fdiv_rn(p.reference, fabsf(x));
                }
            }
            if (k >= 2) {                                                       // drain tile k-2: [limit_ff] [convert_f_s16]
                const int t = k - 2;
                AgcTile& tl = tiles[t % 3];
                for (int e = ltid; e < AGC_CH * AGC_T; e += nl) {
                    const int ch = e / AGC_T, i = e % AGC_T, c = c0 + ch;
                    const long pos = (long)t * AGC_T + i;
                    if (c >= channels || pos >= n) continue;
                    float y = tl.x[ch][i];
                    if (LIMIT) y = fmaxf(-limit_max, fminf(limit_max, y));            // limit_ff as launch_limit_ff computes it (NaN -> +max)
                    if (S16) static_cast<short*>(out)[(long)c * out_stride + pos] = (short)f_to_s16_bits(y);
                    else static_cast<float*>(out)[(long)c * out_stride + pos] = y;
                }
            }
            __syncthreads();
        }
    }
}

template <bool CF32, bool S16>
static void agc_launch_limit(dim3 grid, const void* d_in, long in_stride, void* d_out, long out_stride, int channels, int n, const AgcParams& p,
                             AgcState* d_state, float limit_max, cudaStream_t st)
{
    if (limit_max > 0.f) agc_bank_kernel<CF32, S16, true><<<grid, AGC_WARPS * 32, 0, st>>>(d_in, in_stride, d_out, out_stride, channels, n, p, d_state, limit_max);
    else agc_bank_kernel<CF32, S16, false><<<grid, AGC_WARPS * 32, 0, st>>>(d_in, in_stride, d_out, out_stride, channels, n, p, d_state, 0.f);
}

// cf32 = 1: d_in is cf32 rows of which only .i is read (realpart_cf); s16 = 1: d_out is short rows (convert_f_s16).  limit_max <= 0: no limit_ff.
int launch_agc_bank(const void* d_in, long in_stride, int cf32, void* d_out, long out_stride, int s16, int channels, int n, const void* h_params_v,
                    void* d_state_v, float limit_max, cudaStream_t st)
{
    const AgcParams* h_params = static_cast<const AgcParams*>(h_params_v);
    AgcState* d_state = static_cast<AgcState*>(d_state_v);
    if (!h_params) { set_error("agc bank: no parameters"); return -1; }
    if (h_params->chunk <= 0) { set_error("agc bank: chunk must be positive"); return -1; }
    if (channels <= 0 || n <= 0) return 0;
    if (in_stride < n || out_stride < n) { set_error("agc bank: row stride shorter than the row"); return -1; }
    const dim3 grid((unsigned)((channels + AGC_CH - 1) / AGC_CH));
    if (cf32) { if (s16) agc_launch_limit<true, true>(grid, d_in, in_stride, d_out, out_stride, channels, n, *h_params, d_state, limit_max, st);
                else agc_launch_limit<true, false>(grid, d_in, in_stride, d_out, out_stride, channels, n, *h_params, d_state, limit_max, st); }
    else      { if (s16) agc_launch_limit<false, true>(grid, d_in, in_stride, d_out, out_stride, channels, n, *h_params, d_state, limit_max, st);
                else agc_launch_limit<false, false>(grid, d_in, in_stride, d_out, out_stride, channels, n, *h_params, d_state, limit_max, st); }
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace csdrb
