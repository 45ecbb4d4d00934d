// fft_kernels.cuh -- the __global__ kernels of fft.cu (K7 batched c2c, K9 overlap-add bank, fastddc forward / inverse), kept apart from
// their launchers so that a host build can execute them thread by thread (tests/host_shim/cuda_emul.h: every CUDA thread a fiber,
// __syncthreads() a real barrier) in the CPU test tier.  The product includes this file from fft.cu only.
#pragma once
#include "fft.cuh"
#include "fft16.cuh"
#include "phase_table.cuh"

namespace csdrb {

// tw: row_fft_twiddles(N)
template <int N, bool INV>
__global__ void __launch_bounds__(fft_threads(N))
fft_c2c_batch_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride, const float2* __restrict__ tw)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* s = reinterpret_cast<float2*>(smem_raw);
    FftRowIn src(in + (long)blockIdx.x * in_stride); FftRowOut dst(out + (long)blockIdx.x * out_stride);
    block_row_fft_io<N, INV>(s, tw, threadIdx.x, src, dst);           // first pass reads the row, last pass writes it: no staging copies
}

template <int N>
__global__ void __launch_bounds__(fft_threads(N), (N <= 4096 ? 2 : 1))
olafir_bank_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride,
                   const float2* __restrict__ taps_fft, long taps_stride, float2* __restrict__ tail_io /*[C][N]*/,
                   int input_size, int nblocks, int blocks_per_cta, const float2* __restrict__ tw)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* s = reinterpret_cast<float2*>(smem_raw);
    float2* tail = s + fft_smem_elems(N);
    constexpr int NT = fft_threads(N);
    const int tid = threadIdx.x, ch = blockIdx.y;
    const int overlap = N - input_size;
    const int b_first = blockIdx.x * blocks_per_cta;
    if (b_first >= nblocks) return;
    const int b_last = min(nblocks, b_first + blocks_per_cta);
    const float2* x = in + (long)ch * in_stride;
    float2* y = out + (long)ch * out_stride;
    const float2* H = taps_fft + (long)ch * taps_stride;
    const float inv_n = 1.0f / (float)N;                           // N is a power of two: exact, same as /N
    // A block's result r[i] = ifft[i]/N + (i < overlap ? previous r[input_size + i] : 0)  (libcsdr.c:837-847 with the
    // ping-pong output buffers of csdr.c:1852-1878).  When overlap > input_size the carried tail chains through
    // ceil(overlap/input_size) earlier blocks, so a run that starts mid-stream recomputes that many lead-in blocks
    // from a zero tail; everything that zero start gets wrong has been shifted out by the first emitted block.
    const int lead = overlap > 0 ? (overlap + input_size - 1) / input_size : 0;
    const int b_start = b_first - lead > 0 ? b_first - lead : 0;
    for (int i = tid; i < overlap; i += NT) tail[i] = b_start == 0 ? tail_io[(long)ch * N + i] : make_float2(0.f, 0.f);
    for (int b = b_start; b < b_last; b++) {
        const bool emit = b >= b_first;
        { const float2* xb = x + (long)b * input_size;
          fft_stage_in<N, NT>(s, tid, [&](int i) { return i < input_size ? __ldg(xb + i) : make_float2(0.f, 0.f); }); }
        __syncthreads();
        block_fft<N, NT, false>(s, tw, tid);
        {
            constexpr int PERH = (N + NT - 1) / NT;
            float2 hh[PERH];                                            // all taps_fft loads first (L2 latency once, not PERH times)
#pragma unroll
            for (int k = 0; k < PERH; k++) { const int i = tid + k * NT; hh[k] = (N % NT == 0 || i < N) ? __ldg(H + i) : make_float2(0.f, 0.f); }
#pragma unroll
            for (int k = 0; k < PERH; k++) {
                const int i = tid + k * NT;
                if (N % NT == 0 || i < N) {
                    const float2 a = s[fft_pad(i)], h = hh[k];
                    // same rounding sequence as libcsdr.c:827-828 (separate products, no FMA)
                    s[fft_pad(i)] = make_float2(__fsub_rn(__fmul_rn(a.x, h.x), __fmul_rn(a.y, h.y)), __fadd_rn(__fmul_rn(a.x, h.y), __fmul_rn(a.y, h.x)));
                }
            }
        }
        __syncthreads();
        block_fft<N, NT, true>(s, tw, tid);
        for (int i = tid; i < N; i += NT) {
            const float2 raw = s[fft_pad(i)];
            float2 v = make_float2(raw.x * inv_n, raw.y * inv_n);
            if (i < overlap) v = make_float2(__fadd_rn(v.x, tail[i].x), __fadd_rn(v.y, tail[i].y));
            s[fft_pad(i)] = v;
            if (emit && i < input_size) y[(long)b * input_size + i] = v;
        }
        __syncthreads();
        for (int i = tid; i < overlap; i += NT) tail[i] = s[fft_pad(input_size + i)];
        __syncthreads();
    }
    if (b_last == nblocks) for (int i = tid; i < overlap; i += NT) tail_io[(long)ch * N + i] = tail[i];
}

// The fused overlap-add kernel on radix-16 passes, sizes 16^k (config 5's 4096): 4R+4W shared accesses per point and block
template <int N>
__global__ void __launch_bounds__(fft_threads(N), (N <= 4096 ? 2 : 1))
olafir_bank_fused16_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride,
                           const float2* __restrict__ taps_fft, long taps_stride, float2* __restrict__ tail_io /*[C][N]*/,
                           int input_size, int nblocks, int blocks_per_cta, const float2* __restrict__ tw16)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* s = reinterpret_cast<float2*>(smem_raw);
    constexpr int NT = fft_threads(N);
    const int tid = threadIdx.x, ch = blockIdx.y;
    const int overlap = N - input_size;
    float2* tail_cur = s + fft_smem_elems(N);
    float2* tail_next = tail_cur + overlap;
    const int b_first = blockIdx.x * blocks_per_cta;
    if (b_first >= nblocks) return;
    const int b_last = min(nblocks, b_first + blocks_per_cta);
    const float2* x = in + (long)ch * in_stride;
    float2* y = out + (long)ch * out_stride;
    const float2* H = taps_fft + (long)ch * taps_stride;
    const int lead = overlap > 0 ? (overlap + input_size - 1) / input_size : 0;      // see olafir_bank_kernel
    const int b_start = b_first - lead > 0 ? b_first - lead : 0;
    for (int i = tid; i < overlap; i += NT) tail_cur[i] = b_start == 0 ? tail_io[(long)ch * N + i] : make_float2(0.f, 0.f);
    struct TapsMap16 {                                                  // spectrum * taps_fft, rounding sequence of libcsdr.c:827-828
        const float2* H; float2 hh[16];
        __device__ __forceinline__ void prefetch(int r, int i) { hh[r] = __ldg(H + i); }
        __device__ __forceinline__ float2 at(int r, int, float2 a) const
        {
            const float2 h = hh[r];
            return make_float2(__fsub_rn(__fmul_rn(a.x, h.x), __fmul_rn(a.y, h.y)), __fadd_rn(__fmul_rn(a.x, h.y), __fmul_rn(a.y, h.x)));
        }
    } map;
    map.H = H;
    const float inv_n = 1.0f / (float)N;
    for (int b = b_start; b < b_last; b++) {
        struct BlockIn {
            const float2* xb; int input_size;
            __device__ __forceinline__ float2 load(int i) const { return i < input_size ? __ldg(xb + i) : make_float2(0.f, 0.f); }
        } src{x + (long)b * input_size, input_size};
        struct BlockOut {
            float2* yb; const float2* tail_cur; float2* tail_next; int input_size, overlap; float inv_n; bool emit;
            __device__ __forceinline__ void store(int i, float2 raw) const
            {
                float2 v = make_float2(raw.x * inv_n, raw.y * inv_n);
                if (i < overlap) v = make_float2(__fadd_rn(v.x, tail_cur[i].x), __fadd_rn(v.y, tail_cur[i].y));
                if (i < input_size) { if (emit) yb[i] = v; }
                else tail_next[i - input_size] = v;
            }
        } dst{y + (long)b * input_size, tail_cur, tail_next, input_size, overlap, inv_n, b >= b_first};
        block_fft16_map_ifft<N, NT>(s, tw16, tid, src, map, dst);
        float2* t = tail_cur; tail_cur = tail_next; tail_next = t;
    }
    __syncthreads();
    if (b_last == nblocks) for (int i = tid; i < overlap; i += NT) tail_io[(long)ch * N + i] = tail_cur[i];
}

// Same operation with the transforms' ends fused: the forward FFT's first pass reads the zero-padded block straight from global
// memory, its last pass hands the spectrum x taps_fft product to the inverse FFT's first pass in registers (4096 = 8^4; other sizes go
// through shared memory once), the inverse FFT's last pass scales, adds the carried tail and writes the result and the next tail.
// taps_fft is fetched (L2) into registers while the last forward butterflies run, tails ping-pong between two shared arrays.
template <int N>
__global__ void __launch_bounds__(fft_threads(N), (N <= 4096 ? 2 : 1))
olafir_bank_fused_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride,
                         const float2* __restrict__ taps_fft, long taps_stride, float2* __restrict__ tail_io /*[C][N]*/,
                         int input_size, int nblocks, int blocks_per_cta, const float2* __restrict__ tw)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* s = reinterpret_cast<float2*>(smem_raw);
    constexpr int NT = fft_threads(N);
    using LP = FftLastPass<N, NT>;
    const int tid = threadIdx.x, ch = blockIdx.y;
    const int overlap = N - input_size;
    float2* tail_cur = s + fft_smem_elems(N);
    float2* tail_next = tail_cur + overlap;
    const int b_first = blockIdx.x * blocks_per_cta;
    if (b_first >= nblocks) return;
    const int b_last = min(nblocks, b_first + blocks_per_cta);
    const float2* x = in + (long)ch * in_stride;
    float2* y = out + (long)ch * out_stride;
    const float2* H = taps_fft + (long)ch * taps_stride;
    const int lead = overlap > 0 ? (overlap + input_size - 1) / input_size : 0;      // see olafir_bank_kernel
    const int b_start = b_first - lead > 0 ? b_first - lead : 0;
    for (int i = tid; i < overlap; i += NT) tail_cur[i] = b_start == 0 ? tail_io[(long)ch * N + i] : make_float2(0.f, 0.f);

    struct TapsMap {                                                    // spectrum * taps_fft, rounding sequence of libcsdr.c:827-828
        const float2* H; float2 hh[LP::PER][8];
        __device__ __forceinline__ static float2 mul(float2 a, float2 h)
        {
            return make_float2(__fsub_rn(__fmul_rn(a.x, h.x), __fmul_rn(a.y, h.y)), __fadd_rn(__fmul_rn(a.x, h.y), __fmul_rn(a.y, h.x)));
        }
        __device__ __forceinline__ void prefetch(int b, int r, int i) { hh[b][r] = __ldg(H + i); }
        __device__ __forceinline__ float2 at(int b, int r, int, float2 v) const { return mul(v, hh[b][r]); }
        __device__ __forceinline__ float2 any(int i, float2 v) const { return mul(v, __ldg(H + i)); }
    } map;
    map.H = H;
    const float inv_n = 1.0f / (float)N;                               // N is a power of two: exact, same as /N
    for (int b = b_start; b < b_last; b++) {
        struct BlockIn {                                                // input_size samples followed by zeros (csdr.c:1872-1876)
            const float2* xb; int input_size;
            __device__ __forceinline__ float2 load(int i) const { return i < input_size ? __ldg(xb + i) : make_float2(0.f, 0.f); }
            __device__ __forceinline__ float4 load2(int i) const { const float2 a = load(i), c = load(i + 1); return make_float4(a.x, a.y, c.x, c.y); }
        } src{x + (long)b * input_size, input_size};
        struct BlockOut {                                               // r[i] = ifft[i]/N + (i < overlap ? previous r[input_size + i] : 0)
            float2* yb; const float2* tail_cur; float2* tail_next; int input_size, overlap; float inv_n; bool emit;
            __device__ __forceinline__ void store(int i, float2 raw) const
            {
                float2 v = make_float2(raw.x * inv_n, raw.y * inv_n);
                if (i < overlap) v = make_float2(__fadd_rn(v.x, tail_cur[i].x), __fadd_rn(v.y, tail_cur[i].y));
                if (i < input_size) { if (emit) yb[i] = v; }
                else tail_next[i - input_size] = v;
            }
            __device__ __forceinline__ void store2(int i, float2 a, float2 c) const { store(i, a); store(i + 1, c); }
        } dst{y + (long)b * input_size, tail_cur, tail_next, input_size, overlap, inv_n, b >= b_first};
        block_fft_map_ifft<N, NT>(s, tw, tid, src, map, dst);
        float2* t = tail_cur; tail_cur = tail_next; tail_next = t;       // the next block's first read of its tail is three barriers away
    }
    __syncthreads();
    if (b_last == nblocks) for (int i = tid; i < overlap; i += NT) tail_io[(long)ch * N + i] = tail_cur[i];
}

// tw: row_fft_twiddles(N)
template <int N>
__global__ void __launch_bounds__(fft_threads(N))
fastddc_fwd_kernel(const float2* __restrict__ in, float2* __restrict__ spectra, const float2* __restrict__ overlap_in,
                   int input_size, const float2* __restrict__ tw)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* s = reinterpret_cast<float2*>(smem_raw);
    const int b = blockIdx.x;
    const int overlap = N - input_size;
    // block b transforms stream samples [b*input_size - overlap, (b+1)*input_size); negative positions come from the carried overlap
    const long start = (long)b * input_size - overlap;
    struct SlideIn {                                                    // stream position start + i; before the stream: the carried overlap
        const float2* in; const float2* ov; long start; int overlap;
        __device__ __forceinline__ float2 load(int i) const { const long p = start + i; return p >= 0 ? __ldg(in + p) : ov[overlap + p]; }
        __device__ __forceinline__ float4 load2(int i) const { const float2 a = load(i), b = load(i + 1); return make_float4(a.x, a.y, b.x, b.y); }
    } src{in, overlap_in, start, overlap};
    FftRowOut dst(spectra + (long)b * N);
    block_row_fft_io<N, false>(s, tw, threadIdx.x, src, dst);
}

__global__ void __launch_bounds__(1024)
fastddc_carry_overlap_kernel(const float2* __restrict__ in, float2* __restrict__ overlap_io, int overlap, long total)
{
    // new carried overlap = last `overlap` samples of (old overlap ++ in[0..total)); one CTA, read everything, barrier, write
    float2 v[16];
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const int i = threadIdx.x + k * 1024;
        if (i < overlap) { const long p = total - overlap + i; v[k] = p >= 0 ? in[p] : overlap_io[overlap + p]; }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; k++) {
        const int i = threadIdx.x + k * 1024;
        if (i < overlap) overlap_io[i] = v[k];
    }
}

template <int N>
__global__ void __launch_bounds__(fft_threads(N))
apply_fir_fft_kernel(const float2* __restrict__ in, const float2* __restrict__ H, const float2* __restrict__ last_overlap, int overlap_size,
                     float2* __restrict__ out, const float2* __restrict__ tw)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* s = reinterpret_cast<float2*>(smem_raw);
    constexpr int NT = fft_threads(N);
    const int tid = threadIdx.x;
    fft_stage_in<N, NT>(s, tid, [&](int i) { return in[i]; });
    __syncthreads();
    block_fft<N, NT, false>(s, tw, tid);
    for (int i = tid; i < N; i += NT) {
        const float2 a = s[fft_pad(i)], h = H[i];
        s[fft_pad(i)] = make_float2(__fsub_rn(__fmul_rn(a.x, h.x), __fmul_rn(a.y, h.y)), __fadd_rn(__fmul_rn(a.x, h.y), __fmul_rn(a.y, h.x)));
    }
    __syncthreads();
    block_fft<N, NT, true>(s, tw, tid);
    const float inv_n = 1.0f / (float)N;
    for (int i = tid; i < N; i += NT) {
        float2 v = make_float2(s[fft_pad(i)].x * inv_n, s[fft_pad(i)].y * inv_n);
        if (i < overlap_size) v = make_float2(__fadd_rn(v.x, last_overlap[i].x), __fadd_rn(v.y, last_overlap[i].y));
        out[i] = v;
    }
}

struct DdcChan { int offsetbin; float sindelta, cosdelta, rate; };     // per channel: fastddc_t.offsetbin + dsadata

// Chains per CTA: the chains run NEXT TO other kernels (the fold, the IFFT step), and a guest warp slows its host SM's CTAs down -- eight warps per CTA put the 64
// chains of config 3 on 8 SMs instead of 64 (the fold's one CTA per SM leaves room for a 256-thread guest, which
// the fused NFM bank's three CTAs per SM do not: its chain kernel keeps one warp per CTA).
constexpr int kFastddcChainWarps = 8;

// Walk the block-to-block state of decimating_shift_addition_cc (libcsdr_gpl.c:154-158), one WARP per channel (a step is ~400 cycles of dependent latency).
__global__ void __launch_bounds__(32 * kFastddcChainWarps)
fastddc_state_chain_kernel(const DdcChan* __restrict__ chan, int* __restrict__ remain_io, float* __restrict__ phase_io,
                           int* __restrict__ blk_remain, float* __restrict__ blk_phase, int* __restrict__ blk_offset,
                           int* __restrict__ out_total, int channels, int nblocks, int post_input_size, int post_decimation,
                           WrapTable* __restrict__ tables, int build_tables)
{
    const int c = blockIdx.x * kFastddcChainWarps + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (c >= channels) return;
    const int k_const = post_input_size / post_decimation;
    int remain = remain_io[c], off = 0;
    float ph = phase_io[c];
    const float rate = chan[c].rate;
    const float adv_const = phase_increment(rate, k_const);
    // when post_decimation divides post_input_size (every fastddc geometry with an even scrap, e.g. 448/2) and the carried remainder is in range, both
    // the per-block output count and the remainder are constants: no integer division in the loop, and the phase chain runs on its increment's wrap table
    const bool steady = (post_input_size % post_decimation == 0) && remain >= 0 && remain < post_decimation;
    __syncwarp();                                                       // every lane has read the carried state before lane 0 overwrites it
    if (tables != nullptr && nblocks > kWrapTableMinSteps && steady) {
        // the table depends on the channel's increment only: a caller that keeps it (the plan object) has it built once
        if (build_tables && lane == 0) wrap_table_build(adv_const, tables + c);
        __syncwarp();
        const WrapLanes w = wrap_lanes_load(tables + c, lane);
        ph = chain_walk_warp(ph, adv_const, &w, nblocks, nullptr, [&](int b, float p) {
            if (lane == 0) {                                            // [block][channel] like the consumers index it
                const long at = (long)b * channels + c;
                blk_remain[at] = remain; blk_phase[at] = p; blk_offset[at] = b * k_const;
            }
        });
        off = nblocks * k_const;
    } else {                                                            // general form
        for (int b = 0; b < nblocks; b++) {
            if (lane == 0) {
                const long at = (long)b * channels + c;
                blk_remain[at] = remain; blk_phase[at] = ph; blk_offset[at] = off;
            }
            if (steady) {
                ph = phase_step(ph, adv_const);
                off += k_const;
            } else {
                int k = 0, pos = remain;
                if (pos < post_input_size) { k = (post_input_size - pos + post_decimation - 1) / post_decimation; pos += k * post_decimation; }
                remain = pos - post_input_size;
                ph = phase_step(ph, phase_increment(rate, k));
                off += k;
            }
        }
    }
    if (lane == 0) { remain_io[c] = remain; phase_io[c] = ph; out_total[c] = off; }
}

template <int M>
__global__ void __launch_bounds__(256)
fastddc_inv_kernel(const float2* __restrict__ spectra /*[nblocks][N]*/, const float2* __restrict__ taps_fft /*[C][N]*/, const DdcChan* __restrict__ chan,
                   const int* __restrict__ blk_remain, const float* __restrict__ blk_phase, const int* __restrict__ blk_offset,
                   float2* __restrict__ out, long out_stride, int N, int pre_decimation, int scrap, int post_input_size, int post_decimation,
                   int nblocks, const float2* __restrict__ tw)
{
    __shared__ float2 s[fft_smem_elems(M)];
    constexpr int NT = 256;
    static_assert(M <= 16 * NT, "fft_inv_size too large for this kernel");
    const int tid = threadIdx.x, b = blockIdx.x, c = blockIdx.y;
    const float2* X = spectra + (long)b * N;
    const float2* H = taps_fft + (long)c * N;
    const DdcChan cp = chan[c];
    const int half = N / 2;
    // fold: inv_input[(N + i - offsetbin + M/2) % M] += Xs[i] * H[i], Xs = spectrum with halves swapped (fastddc.c:123-141)
    // destination depends on i mod M only; each thread owns whole residue classes and adds in ascending i like the reference.
    const float inv_pre = 1.0f / (float)pre_decimation;            // power of two: exact
    for (int r = tid; r < M; r += NT) {
        float ai = 0.f, aq = 0.f;
        for (int i = r; i < N; i += M) {
            const float2 x = X[i < half ? i + half : i - half];
            const float2 h = H[i];
            ai = __fadd_rn(ai, __fsub_rn(__fmul_rn(x.x, h.x), __fmul_rn(x.y, h.y)));
            aq = __fadd_rn(aq, __fadd_rn(__fmul_rn(x.x, h.y), __fmul_rn(x.y, h.x)));
        }
        int dst = (N + r - cp.offsetbin + M / 2) % M;
        if (dst < 0) dst += M;
        // second swap (fastddc.c:150) folded into the store index
        const int d2 = dst < M / 2 ? dst + M / 2 : dst - M / 2;
        s[fft_pad(d2)] = make_float2(ai * inv_pre, aq * inv_pre);
    }
    __syncthreads();
    block_fft<M, NT, true>(s, tw, tid);
    // normalise, drop the scrap, post shift + decimate (sequential phasor chain: one thread)
    if (tid == 0) {
        const float inv_m = 1.0f / (float)M;
        const long bi = (long)b * gridDim.y + c;
        const double ph = (double)blk_phase[bi];
        float2 pc = make_float2((float)cos(ph), (float)sin(ph));
        const float2 d = make_float2(cp.cosdelta, cp.sindelta);
        float2* y = out + (long)c * out_stride + blk_offset[bi];
        int k = 0;
        for (int pos = blk_remain[bi]; pos < post_input_size; pos += post_decimation) {
            const float2 raw = s[fft_pad(scrap + pos)];
            const float2 v = make_float2(raw.x * inv_m, raw.y * inv_m);
            y[k++] = rotate_rn(pc, v);
            pc = rotate_rn(pc, d);
        }
    }
}

// Tiled variant for M <= 1024: one CTA folds CT channels x BT blocks at once, so every spectrum bin is fetched once per CT
// channels and every tap once per BT blocks (the untiled kernel moves 256 KB of L2 traffic per (channel, block) and runs
// at the L2 bandwidth limit).  The CT*BT inverse FFTs run four at a time (64 threads each); the CT*BT sequential post-shift
// chains run on CT*BT different lanes in parallel.  Summation order per destination bin is still ascending, as in the reference.
template <int M, int CT, int BT>
__global__ void __launch_bounds__(256)
fastddc_inv_tiled_kernel(const float2* __restrict__ spectra, const float2* __restrict__ taps_fft, const DdcChan* __restrict__ chan,
                         const int* __restrict__ blk_remain, const float* __restrict__ blk_phase, const int* __restrict__ blk_offset,
                         float2* __restrict__ out, long out_stride, int N, int pre_decimation, int scrap, int post_input_size, int post_decimation,
                         int nblocks, int channels, const float2* __restrict__ tw)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* s = reinterpret_cast<float2*>(smem_raw);                    // CT*BT padded arrays of M
    constexpr int NT = 256, NTG = 64, GROUPS = NT / NTG, ELEMS = fft_smem_elems(M), PERT = (M + NT - 1) / NT;
    static_assert(M <= 16 * NTG, "tiled fastddc_inv needs M <= 1024");
    const int tid = threadIdx.x;
    const int b0 = blockIdx.x * BT, c0 = blockIdx.y * CT;
    const int half = N / 2;
    const float inv_pre = 1.0f / (float)pre_decimation;                 // power of two: exact
    int cidx[CT], bidx[BT];
#pragma unroll
    for (int u = 0; u < CT; u++) cidx[u] = min(c0 + u, channels - 1);   // ragged edges shadow the last valid channel / block
#pragma unroll
    for (int v = 0; v < BT; v++) bidx[v] = min(b0 + v, nblocks - 1);
#pragma unroll 1
    for (int rr = 0; rr < PERT; rr++) {
        const int r = tid + rr * NT;
        if (r >= M) break;
        float2 acc[CT][BT];
#pragma unroll
        for (int u = 0; u < CT; u++)
#pragma unroll
            for (int v = 0; v < BT; v++) acc[u][v] = make_float2(0.f, 0.f);
        // two bins per step, all eight loads of both bins issued before the arithmetic of the first (r01: long_scoreboard dominated)
        for (int i = r; i < N; i += 2 * M) {
            const int i2 = i + M;                                       // N / M is even for every fastddc geometry (pre_decimation >= 2)
            const int xi = i < half ? i + half : i - half, xi2 = i2 < half ? i2 + half : i2 - half;
            float2 x[BT], h[CT], x2[BT], h2[CT];
#pragma unroll
            for (int v = 0; v < BT; v++) { x[v] = __ldg(spectra + (long)bidx[v] * N + xi); x2[v] = __ldg(spectra + (long)bidx[v] * N + xi2); }
#pragma unroll
            for (int u = 0; u < CT; u++) { h[u] = __ldg(taps_fft + (long)cidx[u] * N + i); h2[u] = __ldg(taps_fft + (long)cidx[u] * N + i2); }
#pragma unroll
            for (int u = 0; u < CT; u++)
#pragma unroll
                for (int v = 0; v < BT; v++) {
                    acc[u][v].x = __fadd_rn(acc[u][v].x, __fsub_rn(__fmul_rn(x[v].x, h[u].x), __fmul_rn(x[v].y, h[u].y)));
                    acc[u][v].y = __fadd_rn(acc[u][v].y, __fadd_rn(__fmul_rn(x[v].x, h[u].y), __fmul_rn(x[v].y, h[u].x)));
                }
#pragma unroll
            for (int u = 0; u < CT; u++)
#pragma unroll
                for (int v = 0; v < BT; v++) {
                    acc[u][v].x = __fadd_rn(acc[u][v].x, __fsub_rn(__fmul_rn(x2[v].x, h2[u].x), __fmul_rn(x2[v].y, h2[u].y)));
                    acc[u][v].y = __fadd_rn(acc[u][v].y, __fadd_rn(__fmul_rn(x2[v].x, h2[u].y), __fmul_rn(x2[v].y, h2[u].x)));
                }
        }
#pragma unroll
        for (int u = 0; u < CT; u++) {
            int dst = (N + r - chan[cidx[u]].offsetbin + M / 2) % M;
            if (dst < 0) dst += M;
            const int d2 = dst < M / 2 ? dst + M / 2 : dst - M / 2;   // second swap folded into the store index
#pragma unroll
            for (int v = 0; v < BT; v++) s[(u * BT + v) * ELEMS + fft_pad(d2)] = make_float2(acc[u][v].x * inv_pre, acc[u][v].y * inv_pre);
        }
    }
    __syncthreads();
    const int g = tid / NTG, tg = tid % NTG;
#pragma unroll 1
    for (int a = 0; a < CT * BT; a += GROUPS) block_fft<M, NTG, true>(s + (a + g) * ELEMS, tw, tg);   // CT*BT is a multiple of GROUPS
    if (tid < CT * BT) {
        const int u = tid / BT, v = tid % BT;
        if (c0 + u < channels && b0 + v < nblocks) {
            const DdcChan cp = chan[c0 + u];
            const float2* src = s + tid * ELEMS;
            const float inv_m = 1.0f / (float)M;
            const long bi = (long)(b0 + v) * channels + (c0 + u);
            const double ph = (double)blk_phase[bi];
            float2 pc = make_float2((float)cos(ph), (float)sin(ph));
            const float2 d = make_float2(cp.cosdelta, cp.sindelta);
            float2* y = out + (long)(c0 + u) * out_stride + blk_offset[bi];
            int k = 0;
            for (int pos = blk_remain[bi]; pos < post_input_size; pos += post_decimation) {
                const float2 raw = src[fft_pad(scrap + pos)];
                const float2 w = make_float2(raw.x * inv_m, raw.y * inv_m);
                y[k++] = rotate_rn(pc, w);
                pc = rotate_rn(pc, d);
            }
        }
    }
}


// ---- fastddc inverse: fold as a batched complex contraction + a separate IFFT / post-shift kernel ------------------------------------
// The tiled kernel above waits on the fold's global loads, and a 4x4 tile still pulls 1.07 GB through L2 per 64 ch x 256 blocks.  The fold is, per residue r of M,
//     F[c][b][r] = sum_{k < P}  Xs[b][r + k*M] * H[c][r + k*M],           P = N / M  (= pre_decimation)
// i.e. M independent complex (C x P) * (P x B) products.  fastddc_fold_kernel runs it like a GEMM: a CTA owns 64 residues x 16 channels x
// 16 blocks; per k-step the 16 spectrum rows and 16 tap rows (8 KB each) arrive by cp.async into a 4-stage ring, every value is read from
// shared memory by two thread groups, and a thread keeps an 8 x 8 accumulator tile for its residue (128 FFMA pair per 16 LDS.64).  L2 traffic
// drops to 0.27 GB, the inner loop is FMA-pipe bound.  Summation per destination bin is still ascending in the bin index, as in
// fastddc.c:126-141 (k ascending = bin index ascending); products and sums are fused (FFMA pair), inside the 1e-5 budget.
// The folded bins go to a scratch array (L2-sized: 64 ch x 256 blocks x 512 bins = 67 MB), fastddc_ifft_rows_kernel does IFFT_M, /M,
// scrap and the post shift; the block-to-block state chain runs on a side stream meanwhile (it is data-independent).
constexpr int FOLD_R = 64, FOLD_CT = 8, FOLD_BT = 8, FOLD_ST = 3;     // residues per CTA, thread tile (channels x blocks), pipeline stages
constexpr int FOLD_NT = 64 * 2 * 2;                                   // threads: a residue each, times two channel halves, times two block halves of the CTA tile

__global__ void __launch_bounds__(FOLD_NT, 1)
fastddc_fold_kernel(const float2* __restrict__ spectra /*[nblocks][N]*/, const float2* __restrict__ taps_fft /*[C][N]*/, const DdcChan* __restrict__ chan,
                    float2* __restrict__ folded /*[C][nblocks][M]*/, int N, int M, int nblocks, int channels, float inv_pre)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* sm = reinterpret_cast<float2*>(smem_raw);                   // FOLD_ST stages of { x[16][64], h[16][64] }
    constexpr int ROWS = 2 * FOLD_BT, STAGE = 2 * ROWS * FOLD_R;        // float2 per stage
    constexpr int NT = FOLD_NT, CPT = (2 * ROWS * (FOLD_R / 2)) / NT;  // 16-byte copies per thread and k-step
    const int tid = threadIdx.x;
    const int rl = tid & 63, g = tid >> 6, gc = g & 1, gb = g >> 1;
    const int r0 = blockIdx.x * FOLD_R, c0 = blockIdx.y * (2 * FOLD_CT), b0 = blockIdx.z * (2 * FOLD_BT);
    const int P = N / M, halfP = P / 2;                                 // the half swap of the spectrum (fastddc.c:123) is a rotation of k by P/2
    // this thread's CPT 16-byte copies per k-step: chunk ids tid + NT*q; 32 chunks per row, rows 0..15 = spectrum, 16..31 = taps
    const float2* src[CPT]; int dsto[CPT];
#pragma unroll
    for (int q = 0; q < CPT; q++) {
        const int id = tid + NT * q, row = id >> 5, col = (id & 31) * 2;
        if (row < ROWS) src[q] = spectra + (long)min(b0 + row, nblocks - 1) * N + r0 + col;          // ragged edges shadow the last valid row
        else src[q] = taps_fft + (long)min(c0 + row - ROWS, channels - 1) * N + r0 + col;
        dsto[q] = row * FOLD_R + col;
    }
    auto issue = [&](int k, int stage) {
        const int kx = k + halfP < P ? k + halfP : k + halfP - P;
#pragma unroll
        for (int q = 0; q < CPT; q++) cp_async16(sm + stage * STAGE + dsto[q], src[q] + (long)(q < CPT / 2 ? kx : k) * M);
    };
    // (a 4-stage ring with the next step's operands pulled into registers during the FMAs was slower: it needs ~230 registers)
    float2 acc[FOLD_CT][FOLD_BT];
#pragma unroll
    for (int u = 0; u < FOLD_CT; u++)
#pragma unroll
        for (int v = 0; v < FOLD_BT; v++) acc[u][v] = make_float2(0.f, 0.f);
#pragma unroll
    for (int s = 0; s < FOLD_ST - 1; s++) { if (s < P) issue(s, s); cp_async_commit(); }
    for (int k = 0; k < P; k++) {
        cp_async_wait<FOLD_ST - 2>();
        __syncthreads();                                                // stage k has landed for everyone; stage (k-1) is free again
        if (k + FOLD_ST - 1 < P) issue(k + FOLD_ST - 1, (k + FOLD_ST - 1) % FOLD_ST);
        cp_async_commit();
        const float2* xs = sm + (k % FOLD_ST) * STAGE + (gb * FOLD_BT) * FOLD_R + rl;
        const float2* hs = sm + (k % FOLD_ST) * STAGE + (ROWS + gc * FOLD_CT) * FOLD_R + rl;
        float2 x[FOLD_BT], h[FOLD_CT];
#pragma unroll
        for (int v = 0; v < FOLD_BT; v++) x[v] = xs[v * FOLD_R];
#pragma unroll
        for (int u = 0; u < FOLD_CT; u++) h[u] = hs[u * FOLD_R];
        // acc += x*h = xr*(hr, hi) + xi*(-hi, hr): two packed FMAs per accumulator, scalar-broadcast x against h and against h swapped/negated
        // (operand modifiers of FFMA pair: no register moves).  Two sweeps over the tile, so the two FMAs of one accumulator sit 64 instructions apart.
#pragma unroll
        for (int u = 0; u < FOLD_CT; u++)
#pragma unroll
            for (int v = 0; v < FOLD_BT; v++) acc[u][v] = ffma2(h[u], make_float2(x[v].x, x[v].x), acc[u][v]);
#pragma unroll
        for (int u = 0; u < FOLD_CT; u++)
#pragma unroll
            for (int v = 0; v < FOLD_BT; v++)
                acc[u][v] = ffma2(make_float2(__uint_as_float(__float_as_uint(h[u].y) ^ 0x80000000u), h[u].x), make_float2(x[v].y, x[v].y), acc[u][v]);
    }
    // /pre_decimation, and both half swaps (fastddc.c:143-150) folded into the destination index (r - offsetbin) mod M
    const int r = r0 + rl;
#pragma unroll
    for (int u = 0; u < FOLD_CT; u++) {
        const int c = c0 + gc * FOLD_CT + u;
        if (c >= channels) break;
        int d2 = (r - chan[c].offsetbin) % M;
        if (d2 < 0) d2 += M;
#pragma unroll
        for (int v = 0; v < FOLD_BT; v++) {
            const int b = b0 + gb * FOLD_BT + v;
            if (b < nblocks) folded[((long)c * nblocks + b) * M + d2] = make_float2(acc[u][v].x * inv_pre, acc[u][v].y * inv_pre);
        }
    }
}

// The post shift's phasors (libcsdr_gpl.c:131-160: seeded from the block's carried phase in double, advanced by the float recursion once per output) do not depend
// on the data: one lane per (channel, block) pair walks its <= kmax steps here, on the side stream behind the state chain and under the fold, and the table
// phasor[pair][k] is written 32 steps at a time through a padded shared tile, so both this kernel's stores and the IFFT kernel's loads are coalesced rows.
// The IFFT kernel then only multiplies -- every output in parallel instead of one lane per row.
// (Walking the recursion on the FP64 pipe instead -- bit-identical, 53 >= 2*24 + 2 bits make the double rounding innocuous -- to stay out of the fold kernel's
// FMA stream was slower under the fold than this form.)
__global__ void __launch_bounds__(128)
fastddc_phasor_kernel(const DdcChan* __restrict__ chan, const float* __restrict__ blk_phase, float2* __restrict__ phasor, int channels, int nblocks, int kmax)
{
    __shared__ float2 tile_all[4][32 * 33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2* tile = tile_all[warp];
    const long npairs = (long)channels * nblocks;
    const long p_first = ((long)blockIdx.x * 4 + warp) * 32;            // this warp's 32 pairs
    if (p_first >= npairs) return;
    const long p = min(p_first + lane, npairs - 1);                     // lanes past the end shadow the last pair (they compute, they do not store)
    const int c = (int)(p / nblocks), b = (int)(p % nblocks);
    const DdcChan cp = chan[c];
    const double ph = (double)blk_phase[(long)b * channels + c];
    float2 pc = make_float2((float)cos(ph), (float)sin(ph));
    const float2 d = make_float2(cp.cosdelta, cp.sindelta);
    const int rows = (int)min((long)32, npairs - p_first);
    for (int k0 = 0; k0 < kmax; k0 += 32) {
#pragma unroll 4
        for (int j = 0; j < 32; j++) {
            tile[lane * 33 + j] = pc;
            pc = rotate_rn(pc, d);
        }
        __syncwarp();
        for (int r = 0; r < rows; r++)
            if (k0 + lane < kmax) phasor[(p_first + r) * kmax + k0 + lane] = tile[r * 33 + lane];
        __syncwarp();
    }
}

// IFFT_M of the folded (channel, block) rows, /M, drop the scrap, decimate, post shift (the phasors come from fastddc_phasor_kernel; pairs are p = c * nblocks + b).
// A row is M/8 threads, a CTA is 128 threads = 1024/M rows; the first pass reads the folded row from global memory, the last pass hands every finished element
// to the sink below, which multiplies by the phasor fetched BEFORE the middle passes and stores: two shared-memory round trips per row, no staging copy, 8 KB of
// shared memory per CTA.  Earlier forms (a warp per row walking the recursion; sixteen rows per CTA,
// a lane per row; flat (row, output) items with precomputed phasors) were slower.
template <int M>
struct FastddcPostSink {
    float2* y; float2 ph[8]; int kk[8]; float inv_m;
    __device__ __forceinline__ void slot(int /*b*/, int r, int /*i*/, float2 v) const
    {
        if (kk[r] < 0) return;
        const float2 w = make_float2(v.x * inv_m, v.y * inv_m);
        y[kk[r]] = rotate_rn(ph[r], w);
    }
};

template <int M>
__global__ void __launch_bounds__(128)
fastddc_ifft_rows_kernel(const float2* __restrict__ folded, const int* __restrict__ blk_remain, const int* __restrict__ blk_offset, float2* __restrict__ out,
                         long out_stride, int scrap, int post_input_size, int post_decimation, int nblocks, int channels, const float2* __restrict__ tw,
                         const float2* __restrict__ phasor, int kmax, int step_k, int step_rem)
{
    CSDRB_DYN_SMEM(smem_raw);
    constexpr int NTG = M / 8, G = 128 / NTG, PITCH = fft_smem_elems(M), R0 = fft_first_radix(M);
    static_assert(M >= 64 && M <= 1024, "fastddc_ifft_rows_kernel: 64 <= M <= 1024");
    const int tid = threadIdx.x, g = tid / NTG, tg = tid % NTG;
    float2* s = reinterpret_cast<float2*>(smem_raw) + g * PITCH;
    const long npairs = (long)channels * nblocks, p = (long)blockIdx.x * G + g;
    const bool valid = p < npairs;
    const long pc = valid ? p : npairs - 1;                             // rows past the end shadow the last one (they take part in the barriers, they do not store)
    const int c = (int)(pc / nblocks), b = (int)(pc % nblocks);
    const long bi = (long)b * channels + c;
    const int first = __ldg(blk_remain + bi), off = __ldg(blk_offset + bi);       // in flight while the first pass loads the row
    FftRowIn src(folded + pc * M);
    fft_pass_first<M, NTG, R0, true>(s, tg, src);
    FastddcPostSink<M> sink;
    sink.inv_m = 1.0f / (float)M;
    sink.y = out + (long)c * out_stride + off;
    const int cnt = first < post_input_size ? (post_input_size - first + post_decimation - 1) / post_decimation : 0;
    // this thread's last-pass elements are tg + r*M/8, r = 0..7: which outputs are they (position q = k * post_decimation past the row's first kept sample), and
    // their phasors.  One integer division per thread; from leg to leg q grows by M/8 = step_k * post_decimation + step_rem (the launcher's division).
    const int q0 = tg - scrap - first;                                  // >= -(scrap + post_decimation): shift it non-negative for the division
    const int lift = scrap + first;                                     // any multiple count >= (scrap + first) / post_decimation will do
    int k = (q0 + lift * post_decimation) / post_decimation, rem = (q0 + lift * post_decimation) - k * post_decimation;
    k -= lift;
#pragma unroll
    for (int r = 0; r < 8; r++) {
        const bool keep = valid && rem == 0 && k >= 0 && k < cnt;
        sink.kk[r] = keep ? k : -1;
        sink.ph[r] = keep ? __ldg(phasor + pc * kmax + k) : make_float2(0.f, 0.f);
        k += step_k; rem += step_rem;
        if (rem >= post_decimation) { rem -= post_decimation; k++; }
    }
    fft_r8_middle_passes<M, NTG, R0, true>(s, tw, tg);
    fft_pass_last_slots<M, NTG, true>(s, tw, tg, sink);
}

}  // namespace csdrb
