// synth.cu -- the synthesis bank: C baseband channels raised to the wideband rate, each moved to its own frequency and summed into ONE stream,
//     y[n] = sum over c of  shift_addition_cc(fir_interpolate_cc(x_c, I, taps), rate_c)[n]
// the transmit mirror of the fused DDC bank (ddc_bank.cu).  The C upshifted intermediates never exist in memory.
//
// Contract, per channel bit for bit the composition of the project's own banks:
//   * fir_interpolate_cc exactly as fir_interpolate_kernel (interpolate.cu): output i*I + ip sums x[i + si] * taps[(I - ip) + si*I] over ascending si
//     while that index is below T (tap 0 is never used), I and Q separately, every product and sum rounded on its own; n inputs give
//     G = interp_groups(n, I, T) groups.
//   * shift_addition_cc exactly as shift_bank_kernel, with its chunks counted on the ABSOLUTE wideband stream as in the fused DDC bank: output 0
//     lies `offset` samples into chunk 0, every chunk seeds its phasor with (cos, sin) of its float start phase evaluated in double, inside a chunk
//     the phasor follows the reference's recursion.  The chunk start phases and seeds are the DDC bank's pre-pass (launch_ddc_prepass: the shared
//     phase chain on its wrap tables), run over the G*I outputs with decimation 1.
//   * The channels are summed in a fixed pairwise tree over the channel index, I and Q separately, each add rounded: level 0 pairs channels
//     (2k, 2k+1), level 1 those sums, and so on; a node with only one present child is that child, unchanged.  The order depends on C alone -- not on
//     block cuts, the grid or the device -- and no float atomics are used.
//
// Layout: lane = channel.  A warp is 32 consecutive channels (aligned to 32), a CTA W <= 8 warps = 32*W channels, walking one segment of whole
// NCO chunks of output positions in step.  Every lane is at the same output, so every lane reads the same tap: the taps sit in shared memory
// and each read is a broadcast.
//   * Fast path (1 <= h = ceil((T-1)/I) <= 8, I*h taps fit in shared memory): each lane keeps its channel's window x[i .. i+h-1] in registers
//     and forms all I phases of group i from it; the window slides by one input per group, the next input is loaded one group ahead.  The taps are
//     restaged as [ip][si] (entries past T are stored but never multiplied: phase ip sums exactly h or h-1 terms, both compile-time loops).
//   * General path (any other h): each term's input comes through the read-only cache, the taps from shared memory (T <= 8192) or from it too.
// The tree: every lane writes its rotated value into its row of a per-warp 32 x 32 tile of outputs (odd pitch); after 32 outputs lane t sums
// column t over the warp's present channels (levels 0-4 of the tree, pair_tree<32>); then warp 0 sums the W warp nodes of each output through
// shared memory (levels 5 .. 4 + log2 W) and stores 32 consecutive outputs.  With more than one CTA of channels per output, each CTA writes its node
// to a partial row in the scratch and synth_tree_kernel finishes the upper levels, in the same tree order.
#include "common.cuh"
#include "kernels.h"

namespace csdrb {

constexpr int kSynthWarps = 8;                                  // warps per CTA at most: 256 channels
constexpr int kSynthPitch = 33;                                 // tile row pitch in float2: a column walk is conflict-free
constexpr int kSynthMaxH = 8;                                   // register window of the fast path
constexpr int kSynthSmemTaps = 8192;                            // taps staged in shared memory (32 KB)
constexpr int kSynthSeg = 1024;                                 // outputs per CTA at least (whole chunks)

// Pairwise sum of v[lo*stride], v[(lo+1)*stride] ... over the N-wide aligned block at lo, restricted to indices below m (lo < m): the left half,
// plus the right half where it holds a present entry
template <int N>
__device__ __forceinline__ float2 pair_tree(const float2* v, int stride, int lo, int m)
{
    if constexpr (N == 1) {
        return v[lo * stride];
    } else {
        float2 a = pair_tree<N / 2>(v, stride, lo, m);
        if (lo + N / 2 < m) {
            const float2 b = pair_tree<N / 2>(v, stride, lo + N / 2, m);
            a = make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
        }
        return a;
    }
}

// K terms of one output from the register window: acc = (..((0 + w0 t0) + w1 t1) ..), I and Q apart, each product and sum rounded
template <int K, int H>
__device__ __forceinline__ float2 window_mac(const float2 (&win)[H], const float* __restrict__ tq)
{
    float ai = 0.f, aq = 0.f;
#pragma unroll
    for (int si = 0; si < K; si++) {
        const float t = tq[si];
        ai = __fadd_rn(ai, __fmul_rn(win[si].x, t));
        aq = __fadd_rn(aq, __fmul_rn(win[si].y, t));
    }
    return make_float2(ai, aq);
}

// H > 0: the fast path with an H-input register window (H = h exactly).  H = 0: the general path; SMEM_TAPS says whether the T taps fit in
// shared memory.  blockIdx.x = segment of seg_len absolute positions, blockIdx.y = CTA of channels; `out` row blockIdx.y * part_stride.
template <int H, bool SMEM_TAPS>
__global__ void __launch_bounds__(32 * kSynthWarps)
synth_bank_kernel(const float2* __restrict__ in, long in_stride, int n, int channels, int I, const float* __restrict__ taps, int T,
                  const float3* __restrict__ params, const float2* __restrict__ seeds, int nchunks, int chunk, int offset, long seg_len, long nout,
                  float2* __restrict__ out, long part_stride)
{
    CSDRB_DYN_SMEM(smem);
    const int W = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float2* tile = reinterpret_cast<float2*>(smem) + warp * 32 * kSynthPitch;
    float2* cross = reinterpret_cast<float2*>(smem) + W * 32 * kSynthPitch;            // [2][W][32]: warp nodes, double-buffered
    float* s_taps = reinterpret_cast<float*>(cross + 2 * W * 32);
    if constexpr (H > 0) {
        for (int k = threadIdx.x; k < I * H; k += blockDim.x) {                      // [ip][si] = taps[(I - ip) + si*I]
            const int ip = k / H, si = k - ip * H;
            const long ti = (long)(I - ip) + (long)si * I;
            s_taps[k] = ti < T ? taps[ti] : 0.f;
        }
    } else if constexpr (SMEM_TAPS) {
        for (int k = threadIdx.x; k < T; k += blockDim.x) s_taps[k] = taps[k];
    }
    __syncthreads();
    const float* tp = (H > 0 || SMEM_TAPS) ? s_taps : taps;

    const int cw = (blockIdx.y * W + warp) * 32;                                   // first channel of this warp
    const bool warp_live = cw < channels;
    const int rows = min(32, channels - cw);                                        // present channels of this warp
    const int c = cw + lane;
    const bool live = c < channels;
    const int wl = min(W, (channels - (int)blockIdx.y * W * 32 + 31) >> 5);        // present warps of this CTA
    const long a0 = (long)blockIdx.x * seg_len;                                    // absolute position of the segment
    const long o_begin = max(0L, a0 - offset), o_end = min(nout, a0 + seg_len - offset);
    const float2* x = in + (live ? (long)c * in_stride : 0L);

    // the phasor of output o_begin: the seed of its chunk, advanced to its place in it (only the first segment starts inside a chunk)
    float2 d = make_float2(0.f, 0.f), ph = make_float2(0.f, 0.f);
    const long a = offset + o_begin;
    int k = (int)(a / chunk), j = (int)(a - (long)k * chunk);
    if (live) {
        const float3 p = params[c];
        d = make_float2(p.y, p.x);                                                  // (cosd, sind)
        ph = seeds[(long)c * nchunks + k];
        for (int s = 0; s < j; s++) ph = rotate_rn(ph, d);
    }
    long i = o_begin / I;
    int ip = (int)(o_begin - i * I);
    constexpr int HW = H > 0 ? H : 1;
    float2 win[HW], nxt = make_float2(0.f, 0.f);
    if constexpr (H > 0) {
#pragma unroll
        for (int h = 0; h < H; h++) win[h] = live ? __ldg(x + i + h) : make_float2(0.f, 0.f);
        if (H > 1 && live && i + H < n) nxt = __ldg(x + i + H);           // one group ahead (at H = 1 the slide loads directly: ptxas spills otherwise)
    }
    const int ip_full = H * I - T + 1;                                             // fast path: phases ip >= ip_full sum H terms, the others H - 1

    int t = 0, buf = 0;
    for (long o = o_begin; o < o_end; o++) {
        if (warp_live) {
            float2 acc;
            if constexpr (H > 0) {
                const float* tq = tp + ip * H;
                acc = ip >= ip_full ? window_mac<H>(win, tq) : window_mac<H - 1>(win, tq);
            } else {
                float ai = 0.f, aq = 0.f;
                const float2* xi = x + i;
                int si = 0;
                for (long ti = I - ip; ti < T; ti += I, si++) {
                    const float tv = SMEM_TAPS ? tp[ti] : __ldg(tp + ti);
                    const float2 v = live ? __ldg(xi + si) : make_float2(0.f, 0.f);
                    ai = __fadd_rn(ai, __fmul_rn(v.x, tv));
                    aq = __fadd_rn(aq, __fmul_rn(v.y, tv));
                }
                acc = make_float2(ai, aq);
            }
            tile[lane * kSynthPitch + t] = rotate_rn(ph, acc);
            ph = rotate_rn(ph, d);
            if (++j == chunk) {                                                     // the next chunk: its own seed
                j = 0; k++;
                if (live) ph = seeds[(long)c * nchunks + k];
            }
            if (++ip == I) {                                                        // the next group: slide the window by one input
                ip = 0; i++;
                if constexpr (H > 0) {
#pragma unroll
                    for (int h = 0; h + 1 < H; h++) win[h] = win[h + 1];
                    if constexpr (H > 1) {
                        win[H - 1] = nxt;
                        if (live && i + H < n) nxt = __ldg(x + i + H);
                    } else if (live && i < n) {
                        win[0] = __ldg(x + i);
                    }
                }
            }
        }
        if (++t == 32 || o + 1 == o_end) {                                          // a tile of t outputs is complete: sum it over the channels
            __syncwarp();
            if (warp_live && lane < t) cross[(buf * W + warp) * 32 + lane] = pair_tree<32>(tile + lane, kSynthPitch, 0, rows);
            __syncthreads();
            if (warp == 0 && lane < t) out[(long)blockIdx.y * part_stride + (o + 1 - t) + lane] = pair_tree<kSynthWarps>(cross + buf * W * 32 + lane, 32, 0, wl);
            buf ^= 1;
            t = 0;
        }
    }
}

// The levels above one CTA of channels: output o of partial row b is the node of channels [256 b, 256 (b + 1)); the same pairwise tree over b,
// in place in the scratch
__global__ void __launch_bounds__(256)
synth_tree_kernel(float2* __restrict__ part, long nout, int nb, float2* __restrict__ out)
{
    const long o = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= nout) return;
    for (int s = 1; s < nb; s <<= 1)
        for (int b = 0; b + s < nb; b += 2 * s) {
            const float2 l = part[(long)b * nout + o], r = part[(long)(b + s) * nout + o];
            part[(long)b * nout + o] = make_float2(__fadd_rn(l.x, r.x), __fadd_rn(l.y, r.y));
        }
    out[o] = part[o];
}

static int synth_ctas(int channels) { return (channels + 32 * kSynthWarps - 1) / (32 * kSynthWarps); }

// warps per CTA: the smallest power of two that holds every channel, at most kSynthWarps
static int synth_warps(int channels)
{
    int w = 1;
    while (w < kSynthWarps && 32 * w < channels) w *= 2;
    return w;
}

size_t synth_bank_scratch_bytes(int channels, int n, int interpolation, int taps_length, int chunk, int offset)
{
    if (channels < 1 || n < 0 || interpolation < 1 || taps_length < 1 || chunk < 1 || offset < 0 || offset >= chunk) return 16;
    const long nout = interp_groups(n, interpolation, taps_length) * interpolation;
    if (nout > 0x7fffffffL) return 16;
    const size_t pre = (ddc_bank_scratch_bytes(channels, (int)nout, chunk, offset) + 15) & ~(size_t)15;
    const int nb = synth_ctas(channels);
    return pre + (nb > 1 ? (size_t)nb * (size_t)nout * sizeof(float2) : 0);
}

template <int H, bool SMEM_TAPS>
static cudaError_t synth_launch(dim3 grid, int warps, size_t smem, cudaStream_t st, const float2* d_in, long in_stride, int n, int channels, int I,
                                const float* d_taps, int T, const float3* params, const float2* seeds, int nchunks, int chunk, int offset, long seg_len,
                                long nout, float2* out, long part_stride)
{
    return launch_kernel(synth_bank_kernel<H, SMEM_TAPS>, grid, dim3(32 * warps), smem, st, d_in, in_stride, n, channels, I, d_taps, T, params, seeds,
                         nchunks, chunk, offset, seg_len, nout, out, part_stride);
}

int launch_synth_bank(const float2* d_in, long in_stride, int channels, int n, int interpolation, const float* d_taps, int taps_length,
                      const float* d_params, float* d_phase_io, int chunk, int offset, float2* d_out, void* d_scratch, size_t scratch_bytes,
                      int* launches, cudaStream_t st)
{
    *launches = 0;
    const int I = interpolation, T = taps_length;
    if (I < 1 || T < 1 || channels < 1 || n < 0 || chunk < 1) {
        set_error("synth bank: needs interpolation >= 1, taps_length >= 1, channels >= 1, input_size >= 0 and chunk >= 1");
        return -1;
    }
    if (offset < 0 || offset >= chunk) { set_error("synth bank: offset must be in [0, chunk)"); return -1; }
    if (in_stride < n) { set_error("synth bank: input row stride below input_size"); return -1; }
    const long nout = interp_groups(n, I, T) * I;
    if (nout > 0x7fffffffL) { set_error("synth bank: more than 2^31 - 1 outputs in one call"); return -1; }
    if (((long)offset + nout) / chunk + 2 > 0x7fffffffL) { set_error("synth bank: more than 2^31 - 2 NCO chunks in one call"); return -1; }
    if (!d_scratch || scratch_bytes < synth_bank_scratch_bytes(channels, n, I, T, chunk, offset)) { set_error("synth bank: scratch too small"); return -1; }
    if (nout == 0) return 0;
    // chunk start phases and seeds of every absolute chunk the outputs touch; d_phase_io moves to the chunk holding output nout
    int rc = launch_ddc_prepass((int)nout, channels, d_params, d_phase_io, chunk, offset, 1, 1, d_scratch, scratch_bytes, nullptr, st);
    if (rc < 0) return rc;
    *launches = rc;
    int nchunks;
    const float2* seeds = ddc_prepass_seeds(d_scratch, channels, (int)nout, chunk, offset, &nchunks);
    const int nb = synth_ctas(channels), warps = synth_warps(channels);
    float2* part = nb > 1 ? reinterpret_cast<float2*>(static_cast<char*>(d_scratch) + ((ddc_bank_scratch_bytes(channels, (int)nout, chunk, offset) + 15) & ~(size_t)15))
                          : d_out;
    const long seg_len = (long)chunk * ((kSynthSeg + chunk - 1) / chunk);          // whole chunks, about kSynthSeg outputs
    const long nseg = ((long)offset + nout + seg_len - 1) / seg_len;
    const dim3 grid((unsigned)nseg, (unsigned)nb);
    const long h = ((long)T - 1 + I - 1) / I;
    const size_t base = (size_t)warps * 32 * (kSynthPitch + 2) * sizeof(float2);    // tiles and the cross-warp buffers
    const float3* P = reinterpret_cast<const float3*>(d_params);
#define CSDRB_SYNTH_ARGS grid, warps, smem, st, d_in, in_stride, n, channels, I, d_taps, T, P, seeds, nchunks, chunk, offset, seg_len, nout, part, (long)(nb > 1 ? nout : 0)
    cudaError_t e;
    if (h >= 1 && h <= kSynthMaxH && (long)I * h <= kSynthSmemTaps) {
        const size_t smem = base + (size_t)I * h * sizeof(float);
        switch (h) {
            case 1: e = synth_launch<1, true>(CSDRB_SYNTH_ARGS); break;
            case 2: e = synth_launch<2, true>(CSDRB_SYNTH_ARGS); break;
            case 3: e = synth_launch<3, true>(CSDRB_SYNTH_ARGS); break;
            case 4: e = synth_launch<4, true>(CSDRB_SYNTH_ARGS); break;
            case 5: e = synth_launch<5, true>(CSDRB_SYNTH_ARGS); break;
            case 6: e = synth_launch<6, true>(CSDRB_SYNTH_ARGS); break;
            case 7: e = synth_launch<7, true>(CSDRB_SYNTH_ARGS); break;
            default: e = synth_launch<8, true>(CSDRB_SYNTH_ARGS); break;
        }
    } else if (T <= kSynthSmemTaps) {
        const size_t smem = base + (size_t)T * sizeof(float);
        e = synth_launch<0, true>(CSDRB_SYNTH_ARGS);
    } else {
        const size_t smem = base;
        e = synth_launch<0, false>(CSDRB_SYNTH_ARGS);
    }
#undef CSDRB_SYNTH_ARGS
    CSDRB_CUDA(e);
    *launches += 1;
    if (nb > 1) {
        synth_tree_kernel<<<(unsigned)((nout + 255) / 256), 256, 0, st>>>(part, nout, nb, d_out);
        CSDRB_CUDA(cudaGetLastError());
        *launches += 1;
    }
    return (int)nout;
}

}  // namespace csdrb
