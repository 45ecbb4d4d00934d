// psk31_tx.cu -- the BPSK31 transmit chain of the reference, the pipe its BER harness runs (grc_tests/bpsk31_ber.py):
//   psk31_varicode_encoder_u8_u8 | differential_encoder_u8_u8 | psk_modulator_u8_c 2 | psk31_interpolate_sine_cc <sps>
// as banks, one row per channel:
//   varicode_encoder_bank_kernel        one CTA per channel: a block-wide scan of per-byte bit counts, the bits scattered into the row
//   differential_codec_bank_kernel      one CTA per channel: encode is a prefix parity of the zero bytes (ballot + popc per 32 bytes), decode
//                                       compares each byte with the one before
//   psk_modulator_bank_kernel           a 256-entry constellation per CTA in shared memory, one lookup and one 8-byte store per symbol
//   psk31_interpolate_sine_bank_kernel  threads over outputs, the tile's inputs and the I rates in shared memory, coalesced float2 stores
//
// There is no fused modulator + interpolator: the symbols in between are 8 bytes each, the interpolator writes 8*I bytes per symbol (2 KiB at
// sps 256), so fusing would save under 1 % of the traffic for a second code path.  DESIGN.md section 7 records the arithmetic of the
// reference build that these kernels follow.
#include "common.cuh"
#include "kernels.h"
#include "varicode.cuh"

#include <map>
#include <mutex>
#include <vector>

namespace csdrb {

// ---------------------------------------------------------------------------------------------- psk31_varicode_encoder_u8_u8
// libcsdr.c:1551-1575: a byte b < 0x80 writes its code, most significant bit first, then two 0 bits; a byte >= 0x80 matches no table entry and
// is consumed without output.  A matched character that does not fit in what is left of output_max_size ends the call before it.  With S_k the
// running sum of (bits + 2) over the matched characters through byte k, input_processed is the first k with S_k > output_max_size (else the
// row's length) and output_size is S at the byte before it.  The CTA walks the row in chunks of ENC_THREADS * ENC_ITEMS bytes, each thread
// ENC_ITEMS consecutive ones, with an exclusive scan of the bit counts over the CTA and the offset carried between chunks.
constexpr int ENC_THREADS = 256, ENC_ITEMS = 4, ENC_WARPS = ENC_THREADS / 32, ENC_CHUNK = ENC_THREADS * ENC_ITEMS;

// exclusive scan of v over the CTA; *total receives the CTA's sum.  s_warp holds ENC_WARPS ints; the call ends with a barrier so that it can
// be reused at once.
__device__ __forceinline__ int enc_block_scan(int v, int* s_warp, int* total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int y = __shfl_sync(0xffffffffu, x, lane >= d ? lane - d : lane);
        if (lane >= d) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    int base = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < ENC_WARPS; w++) {
        const int t = s_warp[w];
        base += w < warp ? t : 0;
        tot += t;
    }
    __syncthreads();
    *total = tot;
    return base + x - v;
}

__global__ void __launch_bounds__(ENC_THREADS)
varicode_encoder_bank_kernel(const unsigned char* __restrict__ in, long in_stride, unsigned char* __restrict__ out, long out_stride, int n,
                             const int* __restrict__ lengths, int output_max_size, int* __restrict__ input_processed, int* __restrict__ output_size)
{
    __shared__ int s_warp[ENC_WARPS];
    const int c = blockIdx.x;
    const int len = lengths ? max(0, min(lengths[c], n)) : n;
    const unsigned char* x = in + (long)c * in_stride;
    unsigned char* y = out + (long)c * out_stride;
    long offset = 0;                                                       // bits written so far (at most output_max_size)
    int done = len;                                                        // input_processed
    for (int base = 0; base < len; base += ENC_CHUNK) {
        const int i0 = base + threadIdx.x * ENC_ITEMS;
        int cnt[ENC_ITEMS], mine = 0;
#pragma unroll
        for (int k = 0; k < ENC_ITEMS; k++) {
            const int i = i0 + k;
            const unsigned b = i < len ? x[i] : 0x80u;
            cnt[k] = b < 128u ? kVaricode[b].bits + 2 : 0;
            mine += cnt[k];
        }
        int chunk_bits;
        const int excl = enc_block_scan(mine, s_warp, &chunk_bits);
        // the items that fit form a prefix of the chunk: count them, and the bits they write
        int fit = 0, fit_bits = 0, pos = excl;
#pragma unroll
        for (int k = 0; k < ENC_ITEMS; k++) {
            const int i = i0 + k;
            // a byte >= 0x80 is consumed while no matched character before it failed: offset + pos <= max(output_max_size, 0)
            if (i < len && offset + pos + cnt[k] <= (cnt[k] ? (long)output_max_size : (long)max(output_max_size, 0))) {
                fit++;
                if (cnt[k]) {
                    const Varicode v = kVaricode[x[i]];
                    unsigned char* o = y + offset + pos;
                    for (int bi = 0; bi < v.bits; bi++) o[bi] = (unsigned char)((v.code >> (v.bits - 1 - bi)) & 1u);
                    o[v.bits] = 0;
                    o[v.bits + 1] = 0;
                }
                fit_bits += cnt[k];
            }
            pos += cnt[k];
        }
        int fit_all, bits_all;
        enc_block_scan(fit, s_warp, &fit_all);
        enc_block_scan(fit_bits, s_warp, &bits_all);
        offset += bits_all;
        if (fit_all < min(ENC_CHUNK, len - base)) { done = base + fit_all; break; }    // uniform over the CTA
    }
    if (threadIdx.x == 0) {
        input_processed[c] = done;
        output_size[c] = (int)offset;
    }
}

int launch_varicode_encoder_bank(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int n,
                                 const int* d_lengths, int output_max_size, int* d_input_processed, int* d_output_size, cudaStream_t st)
{
    if (channels < 0 || n < 0 || in_stride < n || out_stride < output_max_size) {
        set_error("varicode encoder bank: needs input_size >= 0, in_stride >= input_size and out_stride >= output_max_size");
        return -1;
    }
    if (channels == 0) return 0;
    CSDRB_CUDA(launch_kernel(varicode_encoder_bank_kernel, dim3((unsigned)channels), dim3(ENC_THREADS), (size_t)0, st, d_in, in_stride, d_out,
                             out_stride, n, d_lengths, output_max_size, d_input_processed, d_output_size));
    return 1;
}

// ---------------------------------------------------------------------------------------------- differential_codec
// libcsdr.c:1828-1843.  Encode: a zero byte sets state = !state, any other keeps it, out[i] = state.  After k zero bytes from state s the state
// is s (k = 0), s == 0 (k odd) or s != 0 (k even), so out[i] follows from the count of zero bytes in in[0..i]: a ballot per 32 bytes, popc,
// and the count carried across the warps of the CTA and its chunks.  Decode: out[i] = (in[i] == state), state = in[i]: the byte before, or
// the carried state at i = 0.  The state after the row is written back; an empty row leaves it alone.
constexpr int DC_THREADS = 256, DC_WARPS = DC_THREADS / 32, DC_GROUPS = 8, DC_CHUNK = DC_THREADS * DC_GROUPS;   // 32*DC_GROUPS bytes per warp

__device__ __forceinline__ unsigned char dc_state(unsigned char s, long zeros)
{
    return zeros == 0 ? s : (unsigned char)((zeros & 1) ? (s == 0) : (s != 0));
}

template <bool ENCODE>
__global__ void __launch_bounds__(DC_THREADS)
differential_codec_bank_kernel(const unsigned char* __restrict__ in, long in_stride, unsigned char* __restrict__ out, long out_stride, int n,
                               const int* __restrict__ lengths, unsigned char* __restrict__ state_io)
{
    __shared__ int s_zeros[DC_WARPS];
    const int c = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int len = lengths ? max(0, min(lengths[c], n)) : n;
    const unsigned char* x = in + (long)c * in_stride;
    unsigned char* y = out + (long)c * out_stride;
    const unsigned char s0 = state_io[c];
    long carried = 0;                                                      // zero bytes before the chunk
    for (int base = 0; base < len; base += DC_CHUNK) {
        const int w0 = base + warp * 32 * DC_GROUPS;
        if (ENCODE) {
            unsigned masks[DC_GROUPS];
            int zeros = 0;
#pragma unroll
            for (int g = 0; g < DC_GROUPS; g++) {
                const int i = w0 + g * 32 + lane;
                masks[g] = __ballot_sync(0xffffffffu, i < len && x[i] == 0);
                zeros += __popc(masks[g]);
            }
            if (lane == 0) s_zeros[warp] = zeros;
            __syncthreads();
            long before = carried, total = carried;
#pragma unroll
            for (int w = 0; w < DC_WARPS; w++) {
                before += w < warp ? s_zeros[w] : 0;
                total += s_zeros[w];
            }
            __syncthreads();
#pragma unroll
            for (int g = 0; g < DC_GROUPS; g++) {
                const int i = w0 + g * 32 + lane;
                const long z = before + __popc(masks[g] & (0xffffffffu >> (31 - lane)));     // zero bytes in in[0..i]
                if (i < len) y[i] = dc_state(s0, z);
                before += __popc(masks[g]);
            }
            carried = total;
        } else {
#pragma unroll
            for (int g = 0; g < DC_GROUPS; g++) {
                const int i = w0 + g * 32 + lane;
                if (i < len) y[i] = (unsigned char)(x[i] == (i ? x[i - 1] : s0));
            }
        }
    }
    __syncthreads();                                                       // every thread has read the state before it is replaced
    if (threadIdx.x == 0 && len > 0) state_io[c] = ENCODE ? dc_state(s0, carried) : x[len - 1];
}

int launch_differential_codec_bank(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int n,
                                   const int* d_lengths, int encode, unsigned char* d_state_io, cudaStream_t st)
{
    if (channels < 0 || n < 0 || in_stride < n || out_stride < n) {
        set_error("differential codec bank: needs input_size >= 0 and row strides of at least input_size");
        return -1;
    }
    if (channels == 0 || n == 0) return 0;
    if (encode)
        CSDRB_CUDA(launch_kernel(differential_codec_bank_kernel<true>, dim3((unsigned)channels), dim3(DC_THREADS), (size_t)0, st, d_in, in_stride,
                                 d_out, out_stride, n, d_lengths, d_state_io));
    else
        CSDRB_CUDA(launch_kernel(differential_codec_bank_kernel<false>, dim3((unsigned)channels), dim3(DC_THREADS), (size_t)0, st, d_in, in_stride,
                                 d_out, out_stride, n, d_lengths, d_state_io));
    return 1;
}

// ---------------------------------------------------------------------------------------------- psk_modulator_u8_c
// libcsdr.c:1772-1782 as built: inc = (float)((2*M_PI)/n_psk), formed in double and rounded once; the phase of byte b is fl((float)b * inc).
// The build evaluates cos/sin of it as sincosf on its scalar path and libm's vector cosf/sinf (_ZGVbN4v_) on its vectorised body, so its own
// bits depend on where a byte falls in the call.  Entry b of the constellation here is the float of the double cos/sin of the float phase:
// bit for bit both reference paths for n_psk 2, 4 and 8 with bytes below n_psk (BPSK is 1+0j and -1-8.742278e-08j), within 2 float ulps of
// them everywhere else (DESIGN.md section 7).
constexpr int PSK_THREADS = 256, PSK_PER_CTA = 8192;

__global__ void __launch_bounds__(PSK_THREADS)
psk_modulator_bank_kernel(const unsigned char* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride, int n,
                          const int* __restrict__ lengths, float inc)
{
    __shared__ float2 table[256];
    {
        const float ph = __fmul_rn((float)threadIdx.x, inc);
        table[threadIdx.x] = make_float2((float)cos((double)ph), (float)sin((double)ph));
    }
    __syncthreads();
    const int c = blockIdx.y;
    const int len = lengths ? max(0, min(lengths[c], n)) : n;
    const unsigned char* x = in + (long)c * in_stride;
    float2* y = out + (long)c * out_stride;
    for (long i = (long)blockIdx.x * PSK_THREADS + threadIdx.x; i < len; i += (long)gridDim.x * PSK_THREADS) y[i] = table[x[i]];
}

int launch_psk_modulator_bank(const unsigned char* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, const int* d_lengths,
                              int n_psk, cudaStream_t st)
{
    if (n_psk < 1 || n_psk > 256) { set_error("psk modulator bank: n_psk must be between 1 and 256"); return -1; }
    if (channels < 0 || n < 0 || in_stride < n || out_stride < n) {
        set_error("psk modulator bank: needs input_size >= 0 and row strides of at least input_size");
        return -1;
    }
    if (channels == 0 || n == 0) return 0;
    const float inc = (float)((2 * M_PI) / n_psk);
    const long blocks = (n + PSK_PER_CTA - 1) / PSK_PER_CTA;
    CSDRB_CUDA(launch_kernel(psk_modulator_bank_kernel, dim3((unsigned)blocks, (unsigned)channels), dim3(PSK_THREADS), (size_t)0, st, d_in, in_stride,
                             d_out, out_stride, n, d_lengths, inc));
    return 1;
}

// ---------------------------------------------------------------------------------------------- psk31_interpolate_sine_cc
// libcsdr.c:1793-1808 as built (its disassembly): rec = fl(1/(float)I); x = fl((float)(j+1) * rec); in double, sin(x*M_PI - M_PI/2), + 1.0,
// * 0.5, rounded to float: the rate r[j], j = 0..I-1.  Output i*I + j = fl(fl(in[i]*r[j]) + fl(last*fl(1 - r[j]))) per component, no FMA,
// last = in[i-1] (the carried last_input at i = 0); the last input of the row is carried out.  The build evaluates sin through libmvec for pairs
// of j and libm for an odd last one, and those roundings show in the table, so the table is computed on the host with the same functions
// (host/psk31_rates.c) and kept per device and I.
// Layout: a CTA covers SINE_TILE consecutive outputs of a row at a time, one thread per output in turn, so the float2 stores are coalesced for
// any I.  The I rates sit in shared memory when I <= SINE_SMEM_RATES (32 KB); beyond, the CTA copies the rates of each tile's outputs into
// shared memory before the tile.  The SINE_TILE/I + 2 inputs
// a tile reads are staged in shared memory first, so each is read from global memory about once per CTA.
constexpr int SINE_THREADS = 256, SINE_TILE = 2048, SINE_SMEM_RATES = 8192, SINE_MAX_CTAS_X = 1024;

// the table of one I on the current device, made on first use
struct SineRateTables { std::mutex mu; std::map<int, float*> tables; };

static int sine_rate_table(int I, const float** out)
{
    SineRateTables& t = per_device<SineRateTables>();
    std::lock_guard<std::mutex> lk(t.mu);
    auto it = t.tables.find(I);
    if (it == t.tables.end()) {
        std::vector<float> h((size_t)I);
        if (csdrb_psk31_sine_rates(I, h.data()) < 0) { set_error("psk31_interpolate_sine bank: libmvec (the reference's vector sin) not found"); return -1; }
        float* d = nullptr;
        CSDRB_CUDA(cudaMalloc(reinterpret_cast<void**>(&d), (size_t)I * sizeof(float)));
        CSDRB_CUDA(cudaMemcpy(d, h.data(), (size_t)I * sizeof(float), cudaMemcpyHostToDevice));
        it = t.tables.emplace(I, d).first;
    }
    *out = it->second;
    return 0;
}

template <bool SMEM_RATES>
__global__ void __launch_bounds__(SINE_THREADS)
psk31_interpolate_sine_bank_kernel(const float2* __restrict__ in, long in_stride, float2* __restrict__ out, long out_stride, int n,
                                   const int* __restrict__ lengths, int I, const float* __restrict__ rates, const float2* __restrict__ last_in)
{
    CSDRB_DYN_SMEM(smem);
    float* s_rate = reinterpret_cast<float*>(smem);
    float2* s_x = reinterpret_cast<float2*>(smem + (SMEM_RATES ? ((size_t)I * sizeof(float) + 7) / 8 * 8 : (size_t)SINE_TILE * sizeof(float)));
    if (SMEM_RATES) {
        for (int j = threadIdx.x; j < I; j += SINE_THREADS) s_rate[j] = rates[j];
    }
    const int c = blockIdx.y;
    const int len = lengths ? max(0, min(lengths[c], n)) : n;
    const float2* x = in + (long)c * in_stride;
    float2* y = out + (long)c * out_stride;
    const long nout = (long)len * I;
    for (long o0 = (long)blockIdx.x * SINE_TILE; o0 < nout; o0 += (long)gridDim.x * SINE_TILE) {
        const long o1 = min(nout, o0 + SINE_TILE);
        const long i0 = o0 / I, i1 = (o1 - 1) / I;                        // inputs i0 .. i1, and the one before i0
        const int t0 = (int)(o0 - i0 * I), span = (int)(o1 - i0 * I);      // the tile's outputs, counted from the first of input i0
        __syncthreads();                                                   // the previous tile is done with s_x (and the rates are in)
        if (!SMEM_RATES) {
            const int j0 = (int)(o0 % I);
#pragma unroll 1
            for (int t = threadIdx.x; t < span - t0; t += SINE_THREADS) {
                const int j = j0 + t;
                s_rate[t] = rates[j < I ? j : j - I];                      // a tile (< I outputs) wraps at most once
            }
        }
        for (long k = threadIdx.x; k <= i1 - i0 + 1; k += SINE_THREADS) {
            const long i = i0 - 1 + k;
            s_x[k] = i < 0 ? last_in[c] : x[i];
        }
        __syncthreads();
        for (int t = t0 + threadIdx.x; t < span; t += SINE_THREADS) {
            const int k = t / I, j = t - k * I;                            // input i0 + k, rate j
            const float r = s_rate[SMEM_RATES ? j : t - t0];
            const float omr = __fsub_rn(1.0f, r);
            const float2 v = s_x[k + 1], l = s_x[k];
            y[i0 * I + t] = make_float2(__fadd_rn(__fmul_rn(v.x, r), __fmul_rn(l.x, omr)), __fadd_rn(__fmul_rn(v.y, r), __fmul_rn(l.y, omr)));
        }
    }
}

// the carried input after the row: a launch of its own, stream-ordered after the tiles, every one of which may read the carried value
__global__ void __launch_bounds__(SINE_THREADS)
psk31_interpolate_sine_last_kernel(const float2* __restrict__ in, long in_stride, int channels, int n, const int* __restrict__ lengths,
                                   float2* __restrict__ last_io)
{
    const int c = blockIdx.x * SINE_THREADS + threadIdx.x;
    if (c >= channels) return;
    const int len = lengths ? max(0, min(lengths[c], n)) : n;
    if (len > 0) last_io[c] = in[(long)c * in_stride + len - 1];
}

int launch_psk31_interpolate_sine_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int n, const int* d_lengths,
                                       int interpolation, float2* d_last_io, cudaStream_t st)
{
    if (interpolation < 1) { set_error("psk31_interpolate_sine bank: interpolation must be at least 1"); return -1; }
    if (channels < 0 || n < 0 || in_stride < n) { set_error("psk31_interpolate_sine bank: needs input_size >= 0 and in_stride >= input_size"); return -1; }
    const long nout = (long)n * interpolation;                            // < 2^62
    if (channels > 1 && out_stride > 0x7fffffffffffffffL / channels) { set_error("psk31_interpolate_sine bank: the output rows overflow a long"); return -1; }
    if (out_stride < nout) { set_error("psk31_interpolate_sine bank: out_stride shorter than input_size * interpolation"); return -1; }
    if (channels == 0 || n == 0) return 0;
    const float* d_rates = nullptr;
    if (int rc = sine_rate_table(interpolation, &d_rates)) return rc;
    const long tiles = (nout + SINE_TILE - 1) / SINE_TILE;
    const dim3 grid((unsigned)(tiles < SINE_MAX_CTAS_X ? tiles : SINE_MAX_CTAS_X), (unsigned)channels);
    const size_t staged = (size_t)(SINE_TILE / interpolation + 3) * sizeof(float2);          // inputs of a tile (rates follow)
    if (interpolation <= SINE_SMEM_RATES)
        CSDRB_CUDA(launch_kernel(psk31_interpolate_sine_bank_kernel<true>, grid, dim3(SINE_THREADS),
                                 ((size_t)interpolation * sizeof(float) + 7) / 8 * 8 + staged, st, d_in, in_stride, d_out, out_stride, n, d_lengths,
                                 interpolation, d_rates, d_last_io));
    else
        CSDRB_CUDA(launch_kernel(psk31_interpolate_sine_bank_kernel<false>, grid, dim3(SINE_THREADS), (size_t)SINE_TILE * sizeof(float) + staged, st, d_in, in_stride, d_out, out_stride,
                                 n, d_lengths, interpolation, d_rates, d_last_io));
    CSDRB_CUDA(launch_kernel(psk31_interpolate_sine_last_kernel, dim3((unsigned)((channels + SINE_THREADS - 1) / SINE_THREADS)), dim3(SINE_THREADS),
                             (size_t)0, st, d_in, in_stride, channels, n, d_lengths, d_last_io));
    return 2;
}

}  // namespace csdrb
