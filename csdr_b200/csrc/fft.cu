// fft.cu -- K7 batched c2c FFT, K9 overlap-add FFT filter bank, a12 fastddc forward step, K8 fastddc inverse bank.
//
//   fft_c2c_batch_kernel  : fft_execute() of a make_fft_c2c plan (fft_fftw.c:6-41), one CTA per transform.
//   olafir_bank_kernel    : apply_fir_fft_cc (libcsdr.c:814-849) + the block loop of bandpass_fir_fft_cc
//                           (csdr.c:1872-1883): FFT_N(zero-padded block) * taps_fft -> IFFT_N -> /N -> first
//                           `overlap` outputs += previous block's tail.  A CTA walks a run of consecutive blocks
//                           of one channel keeping the tail in shared memory; a run that does not start at block 0
//                           first recomputes the tail of the block before it.
//   fastddc_fwd_kernel    : csdr.c:2288-2299 -- overlap-save forward FFT (slide `overlap` samples, append
//                           input_size new ones, no window), one CTA per block, all bins written.
//   fastddc_inv_kernel    : fastddc_inv_cc (fastddc.c:106-166) -- fold N bins x taps into M aliasing bins
//                           (same summation order as the reference: ascending bin index per destination),
//                           /pre_decimation, swap, IFFT_M, /M, drop `scrap`, post shift + decimate.
#include "fft_kernels.cuh"
#include "kernels.h"
#include "side_stream.cuh"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <mutex>
#include <vector>

namespace csdrb {

// Radix-16 passes (fft16.cuh) are the default: fewer passes over shared memory than radix 8 for the 4096- and 16384-point
// transforms, the fastddc forward FFT and the config-5 overlap-add bank.  CSDRB_FFT_RADIX16=0 selects the radix-8 kernels (kept for A/B runs and for sizes
// without a radix-16 plan).
static bool fft_radix16_enabled()
{
    const char* e = getenv("CSDRB_FFT_RADIX16");
    return !(e && e[0] == '0');
}

// ---- twiddle tables ------------------------------------------------------------------------------
static std::map<int, float2*> g_tw;
static std::mutex g_tw_mu;

int get_twiddles(int n, const float2** out, cudaStream_t st)
{
    std::lock_guard<std::mutex> lk(g_tw_mu);
    auto it = g_tw.find(n);
    if (it != g_tw.end()) { *out = it->second; return 0; }
    std::vector<float2> h((size_t)3 * n);
    fft_fill_twiddles(n, h.data());
    float2* d = nullptr;
    CSDRB_CUDA(cudaMalloc(&d, sizeof(float2) * h.size()));
    CSDRB_CUDA(cudaMemcpyAsync(d, h.data(), sizeof(float2) * h.size(), cudaMemcpyHostToDevice, st));
    CSDRB_CUDA(cudaStreamSynchronize(st));
    g_tw[n] = d;
    *out = d;
    return 0;
}

static std::map<int, float2*> g_tw16;
int get_twiddles16(int n, const float2** out, cudaStream_t st)
{
    std::lock_guard<std::mutex> lk(g_tw_mu);
    auto it = g_tw16.find(n);
    if (it != g_tw16.end()) { *out = it->second; return 0; }
    std::vector<float2> h((size_t)4 * n);
    fft16_fill_twiddles(n, h.data());
    float2* d = nullptr;
    CSDRB_CUDA(cudaMalloc(&d, sizeof(float2) * h.size()));
    CSDRB_CUDA(cudaMemcpyAsync(d, h.data(), sizeof(float2) * h.size(), cudaMemcpyHostToDevice, st));
    CSDRB_CUDA(cudaStreamSynchronize(st));
    g_tw16[n] = d;
    *out = d;
    return 0;
}

template <int N>
static int launch_c2c16_n(const float2* in, long is, float2* out, long os, int batch, bool inverse, const float2* tw16, cudaStream_t st)
{
    const size_t smem = sizeof(float2) * fft_smem_elems(N);
    if (inverse) {
        auto k = fft_c2c_batch16_kernel<N, true>;
        if (smem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k<<<batch, fft16_threads(N), smem, st>>>(in, is, out, os, tw16);
    } else {
        auto k = fft_c2c_batch16_kernel<N, false>;
        if (smem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k<<<batch, fft16_threads(N), smem, st>>>(in, is, out, os, tw16);
    }
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---- K7: batched c2c -------------------------------------------------------------------------------
template <int N>
static int launch_c2c_n(const float2* in, long is, float2* out, long os, int batch, bool inverse, const float2* tw, cudaStream_t st)
{
    const size_t smem = sizeof(float2) * fft_smem_elems(N);
    if (inverse) {
        auto k = fft_c2c_batch_kernel<N, true>;
        if (smem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k<<<batch, fft_threads(N), smem, st>>>(in, is, out, os, tw);
    } else {
        auto k = fft_c2c_batch_kernel<N, false>;
        if (smem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        k<<<batch, fft_threads(N), smem, st>>>(in, is, out, os, tw);
    }
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

#define CSDRB_FFT_SIZES(X) X(2) X(4) X(8) X(16) X(32) X(64) X(128) X(256) X(512) X(1024) X(2048) X(4096) X(8192) X(16384)

int launch_fft_c2c_batch(const float2* d_in, long in_stride, float2* d_out, long out_stride, int n, int batch, int inverse, cudaStream_t st)
{
    if (batch <= 0) return 0;
    if (n < 2 || n > FFT_MAX_N || (n & (n - 1))) { set_error("fft: size %d unsupported (power of two, 2..%d)", n, FFT_MAX_N); return -1; }
    static const bool radix16 = fft_radix16_enabled();
    if (radix16 && n >= 32) {
        const float2* tw16 = nullptr;
        if (int rc = get_twiddles16(n, &tw16, st)) return rc;
        switch (n) {
#define X(N) case N: if constexpr (N >= 32) return launch_c2c16_n<N>(d_in, in_stride, d_out, out_stride, batch, inverse != 0, tw16, st); break;
            CSDRB_FFT_SIZES(X)
#undef X
        }
    }
    const float2* tw = nullptr;
    if (int rc = get_twiddles(n, &tw, st)) return rc;
    switch (n) {
#define X(N) case N: return launch_c2c_n<N>(d_in, in_stride, d_out, out_stride, batch, inverse != 0, tw, st);
        CSDRB_FFT_SIZES(X)
#undef X
    }
    return -1;
}

// ---- K9: overlap-add FIR bank -------------------------------------------------------------------
int launch_olafir_bank(const float2* d_in, long in_stride, float2* d_out, long out_stride, int channels, int fft_size, int input_size,
                       int nblocks, const float2* d_taps_fft, long taps_stride, float2* d_tail_io, int blocks_per_cta, cudaStream_t st)
{
    if (channels <= 0 || nblocks <= 0) return 0;
    if (fft_size < 4 || fft_size > 8192 || (fft_size & (fft_size - 1))) { set_error("overlap-add FIR: fft_size %d unsupported (power of two, 4..8192)", fft_size); return -1; }
    if (input_size <= 0 || input_size > fft_size) { set_error("overlap-add FIR: bad input_size %d for fft_size %d", input_size, fft_size); return -1; }
    const float2* tw = nullptr;
    if (int rc = get_twiddles(fft_size, &tw, st)) return rc;
    if (blocks_per_cta <= 0) {
        // enough CTAs to fill the machine a few times over, but runs long enough that the recomputed lead-in block stays cheap
        long want = (kSmCount * 8 + channels - 1) / channels;
        blocks_per_cta = (int)((nblocks + want - 1) / want);
        if (blocks_per_cta < 16) blocks_per_cta = nblocks < 16 ? nblocks : 16;
    }
    const dim3 grid((nblocks + blocks_per_cta - 1) / blocks_per_cta, channels);
    static const bool staged = getenv("CSDRB_OLAFIR_STAGED") != nullptr;            // A/B switch: the first kernel, with staged copies
    static const bool radix16 = fft_radix16_enabled();
    if (radix16 && !staged && (fft_size == 256 || fft_size == 4096)) {
        const float2* tw16 = nullptr;
        if (int rc = get_twiddles16(fft_size, &tw16, st)) return rc;
        const size_t fsmem = sizeof(float2) * ((size_t)fft_smem_elems(fft_size) + 2 * (size_t)(fft_size - input_size));
        if (fft_size == 256) {
            auto k = olafir_bank_fused16_kernel<256>;
            k<<<grid, fft16_threads(256), fsmem, st>>>(d_in, in_stride, d_out, out_stride, d_taps_fft, taps_stride, d_tail_io, input_size, nblocks, blocks_per_cta, tw16);
        } else {
            auto k = olafir_bank_fused16_kernel<4096>;
            if (fsmem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
            k<<<grid, fft16_threads(4096), fsmem, st>>>(d_in, in_stride, d_out, out_stride, d_taps_fft, taps_stride, d_tail_io, input_size, nblocks, blocks_per_cta, tw16);
        }
        CSDRB_CUDA(cudaGetLastError());
        return 1;
    }
    if (fft_size >= 16 && !staged) {
        const size_t fsmem = sizeof(float2) * ((size_t)fft_smem_elems(fft_size) + 2 * (size_t)(fft_size - input_size));
        switch (fft_size) {
#define X(N) case N: if constexpr (N >= 16 && N <= 8192) { auto k = olafir_bank_fused_kernel<N>; \
            if (fsmem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem)); \
            k<<<grid, fft_threads(N), fsmem, st>>>(d_in, in_stride, d_out, out_stride, d_taps_fft, taps_stride, d_tail_io, input_size, nblocks, blocks_per_cta, tw); } break;
            CSDRB_FFT_SIZES(X)
#undef X
        }
        CSDRB_CUDA(cudaGetLastError());
        return 1;
    }
    const size_t smem = sizeof(float2) * ((size_t)fft_smem_elems(fft_size) + (size_t)fft_size);
    switch (fft_size) {
#define X(N) case N: if constexpr (N >= 4 && N <= 8192) { auto k = olafir_bank_kernel<N>; \
        if (smem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k<<<grid, fft_threads(N), smem, st>>>(d_in, in_stride, d_out, out_stride, d_taps_fft, taps_stride, d_tail_io, input_size, nblocks, blocks_per_cta, tw); } break;
        CSDRB_FFT_SIZES(X)
#undef X
    }
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---- fastddc forward -------------------------------------------------------------------------------
int launch_fastddc_fwd(const float2* d_in, float2* d_spectra, float2* d_overlap_io, int fft_size, int input_size, int nblocks, cudaStream_t st)
{
    if (nblocks <= 0) return 0;
    if (fft_size < 4 || fft_size > FFT_MAX_N || (fft_size & (fft_size - 1))) { set_error("fastddc_fwd: fft_size %d unsupported", fft_size); return -1; }
    static const bool radix16 = fft_radix16_enabled();
    if (radix16 && fft_size >= 32) {
        const float2* tw16 = nullptr;
        if (int rc = get_twiddles16(fft_size, &tw16, st)) return rc;
        const size_t smem16 = sizeof(float2) * (size_t)fft_smem_elems(fft_size);
        switch (fft_size) {
#define X(N) case N: if constexpr (N >= 32) { auto k = fastddc_fwd16_kernel<N>; \
            if (smem16 > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem16)); \
            k<<<nblocks, fft16_threads(N), smem16, st>>>(d_in, d_spectra, d_overlap_io, input_size, tw16); } break;
            CSDRB_FFT_SIZES(X)
#undef X
        }
        CSDRB_CUDA(cudaGetLastError());
        const int ov16 = fft_size - input_size;
        if (ov16 > 0) {
            fastddc_carry_overlap_kernel<<<1, 1024, 0, st>>>(d_in, d_overlap_io, ov16, (long)nblocks * input_size);
            CSDRB_CUDA(cudaGetLastError());
            return 2;
        }
        return 1;
    }
    const float2* tw = nullptr;
    if (int rc = get_twiddles(fft_size, &tw, st)) return rc;
    const size_t smem = sizeof(float2) * (size_t)fft_smem_elems(fft_size);
    switch (fft_size) {
#define X(N) case N: if constexpr (N >= 4) { auto k = fastddc_fwd_kernel<N>; \
        if (smem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k<<<nblocks, fft_threads(N), smem, st>>>(d_in, d_spectra, d_overlap_io, input_size, tw); } break;
        CSDRB_FFT_SIZES(X)
#undef X
    }
    CSDRB_CUDA(cudaGetLastError());
    const int overlap = fft_size - input_size;
    if (overlap > 0) {
        fastddc_carry_overlap_kernel<<<1, 1024, 0, st>>>(d_in, d_overlap_io, overlap, (long)nblocks * input_size);
        CSDRB_CUDA(cudaGetLastError());
        return 2;
    }
    return 1;
}

// ---- apply_fir_fft_cc drop-in (one block, explicit buffers) -------------------------------------------
int launch_apply_fir_fft(const float2* d_in, const float2* d_taps_fft, const float2* d_last_overlap, int overlap_size, float2* d_out,
                         int fft_size, cudaStream_t st)
{
    if (fft_size < 2 || fft_size > FFT_MAX_N || (fft_size & (fft_size - 1))) { set_error("apply_fir_fft: fft_size %d unsupported", fft_size); return -1; }
    const float2* tw = nullptr;
    if (int rc = get_twiddles(fft_size, &tw, st)) return rc;
    const size_t smem = sizeof(float2) * (size_t)fft_smem_elems(fft_size);
    switch (fft_size) {
#define X(N) case N: { auto k = apply_fir_fft_kernel<N>; \
        if (smem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        k<<<1, fft_threads(N), smem, st>>>(d_in, d_taps_fft, d_last_overlap, overlap_size, d_out, tw); } break;
        CSDRB_FFT_SIZES(X)
#undef X
    }
    CSDRB_CUDA(cudaGetLastError());
    return 1;
}

// ---- fastddc inverse bank ----------------------------------------------------------------------------
// device arrays of the data-independent half of an inverse-bank call
struct InvPrep { int* blk_remain; float* blk_phase; int* blk_offset; WrapTable* tables; float2* phasor; int kmax; };

// Geometries the fold path covers: whole 64-residue CTAs and an even pre-decimation (the half swap of the spectrum is then a rotation of the
// fold's k index).  CSDRB_INV_FOLD=0 sends everything to the round-1 kernels.
bool fastddc_inv_fold_ok(int fft_size, int fft_inv_size)
{
    static const bool fold_off = getenv("CSDRB_INV_FOLD") && getenv("CSDRB_INV_FOLD")[0] == '0';
    if (fold_off || fft_inv_size < 64 || fft_inv_size > 1024 || (fft_inv_size & (fft_inv_size - 1)) || fft_size % fft_inv_size) return false;
    const int P = fft_size / fft_inv_size;
    return P >= 2 && P % 2 == 0;
}

// The data-independent half of a call: block-to-block {remain, phase} chain (updates the carried state, writes the per-block state and the
// output counts) and the post-shift phasors of every (channel, block) row.  Everything on stream `s`.
int launch_fastddc_inv_prepare(const void* d_chan, int channels, int nblocks, int post_input_size, int post_decimation, int* d_remain_io, float* d_phase_io,
                               int* d_out_total, const InvPrep& p, cudaStream_t s, cudaEvent_t before_phasors = nullptr, bool build_tables = true)
{
    fastddc_state_chain_kernel<<<(channels + CHAIN_CPW * CHAIN_WARPS - 1) / (CHAIN_CPW * CHAIN_WARPS), 32 * CHAIN_WARPS, 0, s>>>(static_cast<const DdcChan*>(d_chan), d_remain_io, d_phase_io, p.blk_remain, p.blk_phase,
                                                       p.blk_offset, d_out_total, channels, nblocks, post_input_size, post_decimation, p.tables, build_tables ? 1 : 0);
    CSDRB_CUDA(cudaGetLastError());
    // the chain (votes, shuffles, a double add per step) shares an SM with a running fold at no cost to either; the phasor walk is FMUL/FADD and does not --
    // a caller that has a fold in flight passes the event behind it
    if (before_phasors) CSDRB_CUDA(cudaStreamWaitEvent(s, before_phasors, 0));
    fastddc_phasor_kernel<<<(unsigned)(((long)channels * nblocks + 127) / 128), 128, 0, s>>>(static_cast<const DdcChan*>(d_chan), p.blk_phase, p.phasor, channels, nblocks, p.kmax);
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}

// The data half: fold on `st`, then (after `prepared`, if given) IFFT + post shift.  `after_fold`, if given, is recorded between the two.
int launch_fastddc_inv_apply(const float2* d_spectra, int nblocks, const float2* d_taps_fft, const void* d_chan, int channels, int fft_size, int fft_inv_size,
                             int pre_decimation, int scrap, int post_input_size, int post_decimation, const InvPrep& p, float2* folded, float2* d_out,
                             long out_stride, cudaEvent_t prepared, cudaEvent_t after_fold, cudaStream_t st)
{
    const float2* tw = nullptr;
    if (int rc = get_twiddles(fft_inv_size, &tw, st)) return rc;
    const size_t fsmem = sizeof(float2) * (size_t)FOLD_ST * 2 * (2 * FOLD_BT) * FOLD_R;
    static const bool wide_cta = getenv("CSDRB_FOLD_BT") && getenv("CSDRB_FOLD_BT")[0] == '4';     // A/B: 512-thread CTAs with 8 x 4 thread tiles
    static const bool x_first = getenv("CSDRB_FOLD_HFIRST") && getenv("CSDRB_FOLD_HFIRST")[0] == '0';   // A/B: the sample, not the tap pair, as first multiplicand
    const dim3 fgrid(fft_inv_size / FOLD_R, (channels + 2 * FOLD_CT - 1) / (2 * FOLD_CT), (nblocks + 2 * FOLD_BT - 1) / (2 * FOLD_BT));
    if (fgrid.y > 65535u || fgrid.z > 65535u) { set_error("fastddc_inv: bank too large for one call"); return -1; }
    const float inv_pre = 1.0f / (float)pre_decimation;
    const DdcChan* dc = static_cast<const DdcChan*>(d_chan);
    // (the attribute belongs to the current device's context: set per call, not latched per process)
    if (wide_cta) CSDRB_CUDA(cudaFuncSetAttribute(fastddc_fold_kernel<4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
    else if (x_first) CSDRB_CUDA(cudaFuncSetAttribute(fastddc_fold_kernel<8, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
    else CSDRB_CUDA(cudaFuncSetAttribute(fastddc_fold_kernel<8, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem));
    if (wide_cta) fastddc_fold_kernel<4, true><<<fgrid, 512, fsmem, st>>>(d_spectra, d_taps_fft, dc, folded, fft_size, fft_inv_size, nblocks, channels, inv_pre);
    else if (x_first) fastddc_fold_kernel<8, false><<<fgrid, 256, fsmem, st>>>(d_spectra, d_taps_fft, dc, folded, fft_size, fft_inv_size, nblocks, channels, inv_pre);
    else fastddc_fold_kernel<8, true><<<fgrid, 256, fsmem, st>>>(d_spectra, d_taps_fft, dc, folded, fft_size, fft_inv_size, nblocks, channels, inv_pre);
    CSDRB_CUDA(cudaGetLastError());
    if (after_fold) CSDRB_CUDA(cudaEventRecord(after_fold, st));
    if (prepared) CSDRB_CUDA(cudaStreamWaitEvent(st, prepared, 0));
    const long npairs = (long)channels * nblocks;
    const int rows_per_cta = 1024 / fft_inv_size;
    const size_t rsmem = sizeof(float2) * (size_t)rows_per_cta * (size_t)fft_smem_elems(fft_inv_size);
    switch (fft_inv_size) {
#define X(M) case M: if constexpr (M >= 64 && M <= 1024) { \
        fastddc_ifft_rows_kernel<M><<<(unsigned)((npairs + rows_per_cta - 1) / rows_per_cta), 128, rsmem, st>>>(folded, p.blk_remain, p.blk_offset, d_out, out_stride, \
                                                        scrap, post_input_size, post_decimation, nblocks, channels, tw, p.phasor, p.kmax, \
                                                        (M / 8) / post_decimation, (M / 8) % post_decimation); } break;
        CSDRB_FFT_SIZES(X)
#undef X
    }
    CSDRB_CUDA(cudaGetLastError());
    return 0;
}

size_t fastddc_inv_scratch_bytes(int channels, int nblocks)
{
    return (((size_t)channels * nblocks * 12 + 64 + 15) & ~(size_t)15) + (nblocks > 96 ? (size_t)channels * sizeof(WrapTable) : 0);
}

int launch_fastddc_inv_bank(const float2* d_spectra, int nblocks, const float2* d_taps_fft, const void* d_chan, int channels,
                            int fft_size, int fft_inv_size, int pre_decimation, int scrap, int post_input_size, int post_decimation,
                            int* d_remain_io, float* d_phase_io, float2* d_out, long out_stride, int* d_out_total,
                            void* d_scratch, size_t scratch_bytes, cudaStream_t st)
{
    if (channels <= 0 || nblocks <= 0) return 0;
    if (fft_inv_size < 2 || fft_inv_size > 4096 || (fft_inv_size & (fft_inv_size - 1)) || fft_size % fft_inv_size) {
        set_error("fastddc_inv: fft_inv_size %d unsupported (power of two, 2..4096, dividing fft_size %d)", fft_inv_size, fft_size); return -1;
    }
    if (!d_scratch || scratch_bytes < fastddc_inv_scratch_bytes(channels, nblocks)) { set_error("fastddc_inv: scratch too small"); return -1; }
    const float2* tw = nullptr;
    if (int rc = get_twiddles(fft_inv_size, &tw, st)) return rc;
    int* blk_remain = static_cast<int*>(d_scratch);
    float* blk_phase = reinterpret_cast<float*>(blk_remain + (size_t)channels * nblocks);
    int* blk_offset = reinterpret_cast<int*>(blk_phase + (size_t)channels * nblocks);
    WrapTable* tables = nblocks > 96 ? reinterpret_cast<WrapTable*>(static_cast<char*>(d_scratch) + (((size_t)channels * nblocks * 12 + 64 + 15) & ~(size_t)15)) : nullptr;
    // Round-2 path: fold as a batched contraction (fastddc_fold_kernel), IFFT + post shift in a second kernel, and the data-independent
    // block-to-block state chain + phasor walk on a side stream meanwhile.  Anything fastddc_inv_fold_ok() refuses takes the round-1 kernels below.
    if (fastddc_inv_fold_ok(fft_size, fft_inv_size)) {
        SideStream* ss = side_stream();
        if (!ss) return -1;
        float2* folded = nullptr;
        const int kmax = (post_input_size + post_decimation - 1) / post_decimation;      // outputs one block can emit
        const size_t folded_elems = (size_t)channels * nblocks * fft_inv_size, phasor_elems = (size_t)channels * nblocks * (size_t)kmax;
        CSDRB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&folded), sizeof(float2) * (folded_elems + phasor_elems), st));
        InvPrep pr; pr.blk_remain = blk_remain; pr.blk_phase = blk_phase; pr.blk_offset = blk_offset; pr.tables = tables; pr.phasor = folded + folded_elems; pr.kmax = kmax;
        // CSDRB_INV_TRACE=1 (tools only): timestamps around the pieces of this call, printed after a synchronize.
        static const bool trace = getenv("CSDRB_INV_TRACE") && getenv("CSDRB_INV_TRACE")[0] == '1';
        cudaEvent_t tev[4] = {};
        if (trace) for (auto& e : tev) CSDRB_CUDA(cudaEventCreate(&e));
        int rc = 0;
        {
            std::lock_guard<std::mutex> lk(ss->mu);                     // the fork/join events are shared by every call on this device
            CSDRB_CUDA(cudaEventRecord(ss->fork, st));
            if (trace) CSDRB_CUDA(cudaEventRecord(tev[0], st));
            CSDRB_CUDA(cudaStreamWaitEvent(ss->stream, ss->fork, 0));
            rc = launch_fastddc_inv_prepare(d_chan, channels, nblocks, post_input_size, post_decimation, d_remain_io, d_phase_io, d_out_total, pr, ss->stream);
            if (rc < 0) return rc;
            CSDRB_CUDA(cudaEventRecord(ss->join, ss->stream));
            if (trace) CSDRB_CUDA(cudaEventRecord(tev[1], ss->stream));
            rc = launch_fastddc_inv_apply(d_spectra, nblocks, d_taps_fft, d_chan, channels, fft_size, fft_inv_size, pre_decimation, scrap, post_input_size, post_decimation,
                                          pr, folded, d_out, out_stride, ss->join, trace ? tev[2] : nullptr, st);
            if (rc < 0) return rc;
        }
        if (trace) {
            CSDRB_CUDA(cudaEventRecord(tev[3], st));
            CSDRB_CUDA(cudaStreamSynchronize(st));
            float t[4] = {};
            for (int i = 1; i < 4; ++i) cudaEventElapsedTime(&t[i], tev[0], tev[i]);
            fprintf(stderr, "[inv trace] us from call start: chain + phasors done %.1f | fold done %.1f, post done %.1f\n", t[1] * 1e3f, t[2] * 1e3f, t[3] * 1e3f);
            for (auto& e : tev) cudaEventDestroy(e);
        }
        CSDRB_CUDA(cudaFreeAsync(folded, st));
        return 4;
    }
    fastddc_state_chain_kernel<<<(channels + CHAIN_CPW * CHAIN_WARPS - 1) / (CHAIN_CPW * CHAIN_WARPS), 32 * CHAIN_WARPS, 0, st>>>(static_cast<const DdcChan*>(d_chan), d_remain_io, d_phase_io, blk_remain, blk_phase,
                                                                    blk_offset, d_out_total, channels, nblocks, post_input_size, post_decimation, tables, 1);
    CSDRB_CUDA(cudaGetLastError());
    if (fft_inv_size <= 1024 && fft_inv_size >= 8 && (fft_size / fft_inv_size) % 2 == 0) {
        // Tile = CT channels x BT blocks per CTA (each spectrum bin fetched once per CT channels, each tap once per BT blocks).  Big tiles
        // save L2 traffic but a bank of 64 channels x 16 blocks is only 64 CTAs of 4x4 on the whole GPU (the launch is latency-bound),
        // so the tile shrinks until the grid covers the machine about twice.  CSDRB_INV_TILE=44|22 forces one for A/B runs.
        static const char* forced = getenv("CSDRB_INV_TILE");
        const long ctas44 = (long)((nblocks + 3) / 4) * ((channels + 3) / 4);
        const bool small_tile = forced ? (forced[0] == '2') : (ctas44 < 2 * kSmCount);
        const int CTv = small_tile ? 2 : 4, BTv = small_tile ? 2 : 4;
        const dim3 tgrid((nblocks + BTv - 1) / BTv, (channels + CTv - 1) / CTv);
        const size_t smem = sizeof(float2) * (size_t)CTv * BTv * fft_smem_elems(fft_inv_size);
        switch (fft_inv_size) {
#define X(M) case M: if constexpr (M >= 8 && M <= 1024) { \
            if (small_tile) { auto k = fastddc_inv_tiled_kernel<M, 2, 2>; \
                if (smem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
                k<<<tgrid, 256, smem, st>>>(d_spectra, d_taps_fft, static_cast<const DdcChan*>(d_chan), blk_remain, blk_phase, blk_offset, d_out, out_stride, \
                                           fft_size, pre_decimation, scrap, post_input_size, post_decimation, nblocks, channels, tw); } \
            else { auto k = fastddc_inv_tiled_kernel<M, 4, 4>; \
                if (smem > 48 * 1024) CSDRB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
                k<<<tgrid, 256, smem, st>>>(d_spectra, d_taps_fft, static_cast<const DdcChan*>(d_chan), blk_remain, blk_phase, blk_offset, d_out, out_stride, \
                                           fft_size, pre_decimation, scrap, post_input_size, post_decimation, nblocks, channels, tw); } } break;
            CSDRB_FFT_SIZES(X)
#undef X
        }
        CSDRB_CUDA(cudaGetLastError());
        return 2;
    }
    const dim3 grid(nblocks, channels);
    switch (fft_inv_size) {
#define X(M) case M: if constexpr (M <= 4096) { fastddc_inv_kernel<M><<<grid, 256, 0, st>>>(d_spectra, d_taps_fft, static_cast<const DdcChan*>(d_chan), blk_remain, \
        blk_phase, blk_offset, d_out, out_stride, fft_size, pre_decimation, scrap, post_input_size, post_decimation, nblocks, tw); } break;
        CSDRB_FFT_SIZES(X)
#undef X
    }
    CSDRB_CUDA(cudaGetLastError());
    return 2;
}


// ---- fastddc inverse bank with look-ahead ---------------------------------------------------------------------------------------------
// The stateless call above has the chain + phasor walk inside every call, next to a fold that
// keeps the FMA pipe busy: the post step waits for them after the fold is done.  They depend on nothing
// but the channel parameters and the carried state, so a plan object that OWNS that state prepares call k+1 while call k's IFFT/post step
// and the caller's next forward FFT run: two sets of {state, per-block arrays, phasors}, set q is written by the side stream while set p is
// read by the main stream.  Same kernels, same order of operations per channel: the outputs are those of the stateless call, bit for bit
// (tests/test_kernels_emulated.py, tests/test_gpu_round2.py).
struct FastddcInvPlan {
    int dev = 0, channels = 0, nblocks = 0, kmax = 0;
    int fft_size = 0, fft_inv_size = 0, pre_decimation = 0, scrap = 0, post_input_size = 0, post_decimation = 0;
    DdcChan* d_chan = nullptr;
    int* d_remain[2] = {}; float* d_phase[2] = {}; int* d_total[2] = {};
    void* prep_mem[2] = {}; InvPrep prep[2];
    float2* folded = nullptr;
    cudaStream_t side = nullptr;
    cudaEvent_t ready[2] = {}, post_done[2] = {}, fold_done = nullptr, chan_set = nullptr;
    int cur = 0;                    // the set the NEXT run reads
    bool ahead = false;             // ... has already been enqueued on the side stream
    bool chan_dirty = false;        // a retune is in flight on the side stream: the next fold waits for it
    WrapTable* tables = nullptr;    // one wrap table per channel, shared by both sets (they depend on the channel's increment only)
    bool tables_built = false;
    std::mutex mu;
};

static size_t plan_prep_bytes(int channels, int nblocks, int kmax)
{
    return fastddc_inv_scratch_bytes(channels, nblocks) + 16 + sizeof(float2) * (size_t)channels * nblocks * (size_t)kmax;
}

static int plan_enqueue_prepare(FastddcInvPlan* pl, int q, cudaEvent_t before_phasors = nullptr)
{
    // state of set q := state of the other set (what the previous preparation left), then the chain advances it in place
    CSDRB_CUDA(cudaMemcpyAsync(pl->d_remain[q], pl->d_remain[1 - q], sizeof(int) * pl->channels, cudaMemcpyDeviceToDevice, pl->side));
    CSDRB_CUDA(cudaMemcpyAsync(pl->d_phase[q], pl->d_phase[1 - q], sizeof(float) * pl->channels, cudaMemcpyDeviceToDevice, pl->side));
    if (int rc = launch_fastddc_inv_prepare(pl->d_chan, pl->channels, pl->nblocks, pl->post_input_size, pl->post_decimation, pl->d_remain[q], pl->d_phase[q],
                                            pl->d_total[q], pl->prep[q], pl->side, before_phasors, !pl->tables_built)) return rc;
    pl->tables_built = true;
    CSDRB_CUDA(cudaEventRecord(pl->ready[q], pl->side));
    return 0;
}

void fastddc_inv_plan_destroy(void* plan)
{
    auto* pl = static_cast<FastddcInvPlan*>(plan);
    if (!pl) return;
    int prev = 0; cudaGetDevice(&prev); cudaSetDevice(pl->dev);
    if (pl->side) cudaStreamSynchronize(pl->side);
    cudaDeviceSynchronize();
    cudaFree(pl->d_chan); cudaFree(pl->folded); cudaFree(pl->tables);
    for (int i = 0; i < 2; i++) {
        cudaFree(pl->d_remain[i]); cudaFree(pl->d_phase[i]); cudaFree(pl->d_total[i]); cudaFree(pl->prep_mem[i]);
        if (pl->ready[i]) cudaEventDestroy(pl->ready[i]);
        if (pl->post_done[i]) cudaEventDestroy(pl->post_done[i]);
    }
    if (pl->fold_done) cudaEventDestroy(pl->fold_done);
    if (pl->chan_set) cudaEventDestroy(pl->chan_set);
    if (pl->side) cudaStreamDestroy(pl->side);
    cudaSetDevice(prev);
    delete pl;
}

int fastddc_inv_plan_create(void** out_plan, const void* h_chan, int channels, int nblocks, int fft_size, int fft_inv_size, int pre_decimation, int scrap,
                            int post_input_size, int post_decimation)
{
    if (!out_plan || !h_chan || channels <= 0 || nblocks <= 0 || post_decimation <= 0 || post_input_size <= 0) { set_error("fastddc_inv_plan: bad arguments"); return -1; }
    if (!fastddc_inv_fold_ok(fft_size, fft_inv_size)) {
        set_error("fastddc_inv_plan: geometry %d/%d is not covered by the fold path (fft_inv_size 64..1024, even pre-decimation): use csdrb_fastddc_inv_bank_cc", fft_size, fft_inv_size);
        return -1;
    }
    auto* pl = new FastddcInvPlan();
    CSDRB_CUDA(cudaGetDevice(&pl->dev));
    pl->channels = channels; pl->nblocks = nblocks; pl->fft_size = fft_size; pl->fft_inv_size = fft_inv_size; pl->pre_decimation = pre_decimation; pl->scrap = scrap;
    pl->post_input_size = post_input_size; pl->post_decimation = post_decimation;
    pl->kmax = (post_input_size + post_decimation - 1) / post_decimation;
    bool ok = cudaMalloc(reinterpret_cast<void**>(&pl->d_chan), sizeof(DdcChan) * channels) == cudaSuccess &&
              cudaMalloc(reinterpret_cast<void**>(&pl->folded), sizeof(float2) * (size_t)channels * nblocks * fft_inv_size) == cudaSuccess &&
              cudaMalloc(reinterpret_cast<void**>(&pl->tables), sizeof(WrapTable) * channels) == cudaSuccess &&
              cudaStreamCreateWithFlags(&pl->side, cudaStreamNonBlocking) == cudaSuccess &&
              cudaEventCreateWithFlags(&pl->fold_done, (getenv("CSDRB_INV_TRACE") && getenv("CSDRB_INV_TRACE")[0] == '1') ? cudaEventDefault : cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&pl->chan_set, cudaEventDisableTiming) == cudaSuccess;
    const size_t state_part = fastddc_inv_scratch_bytes(channels, nblocks);
    for (int i = 0; i < 2 && ok; i++) {
        ok = cudaMalloc(reinterpret_cast<void**>(&pl->d_remain[i]), sizeof(int) * channels) == cudaSuccess && cudaMalloc(reinterpret_cast<void**>(&pl->d_phase[i]), sizeof(float) * channels) == cudaSuccess &&
             cudaMalloc(reinterpret_cast<void**>(&pl->d_total[i]), sizeof(int) * channels) == cudaSuccess && cudaMalloc(&pl->prep_mem[i], plan_prep_bytes(channels, nblocks, pl->kmax)) == cudaSuccess &&
             cudaEventCreateWithFlags(&pl->ready[i], cudaEventDisableTiming) == cudaSuccess && cudaEventCreateWithFlags(&pl->post_done[i], cudaEventDisableTiming) == cudaSuccess;
        if (!ok) break;
        char* base = static_cast<char*>(pl->prep_mem[i]);
        InvPrep& pr = pl->prep[i];
        pr.blk_remain = reinterpret_cast<int*>(base);
        pr.blk_phase = reinterpret_cast<float*>(pr.blk_remain + (size_t)channels * nblocks);
        pr.blk_offset = reinterpret_cast<int*>(pr.blk_phase + (size_t)channels * nblocks);
        pr.tables = nblocks > 96 ? pl->tables : nullptr;
        pr.phasor = reinterpret_cast<float2*>(base + ((state_part + 15) & ~(size_t)15));
        pr.kmax = pl->kmax;
        ok = cudaMemset(pl->d_remain[i], 0, sizeof(int) * channels) == cudaSuccess && cudaMemset(pl->d_phase[i], 0, sizeof(float) * channels) == cudaSuccess &&
             cudaMemset(pl->d_total[i], 0, sizeof(int) * channels) == cudaSuccess;
    }
    ok = ok && cudaMemcpy(pl->d_chan, h_chan, sizeof(DdcChan) * channels, cudaMemcpyHostToDevice) == cudaSuccess;
    if (!ok) { set_error("fastddc_inv_plan: device allocation failed (%s)", cudaGetErrorString(cudaGetLastError())); fastddc_inv_plan_destroy(pl); return -1; }
    pl->cur = 0; pl->ahead = false;                                       // the carried state (zeros) sits in set 1, the first preparation goes to set 0
    *out_plan = pl;
    return 0;
}

int fastddc_inv_plan_run(void* plan, const float2* d_spectra, const float2* d_taps_fft, float2* d_out, long out_stride, int* d_out_total, cudaStream_t st)
{
    auto* pl = static_cast<FastddcInvPlan*>(plan);
    if (!pl || !d_spectra || !d_taps_fft || !d_out || !d_out_total) { set_error("fastddc_inv_plan_run: null pointer"); return -1; }
    std::lock_guard<std::mutex> lk(pl->mu);
    int dev_now = -1;
    if (cudaGetDevice(&dev_now) != cudaSuccess || dev_now != pl->dev) { set_error("fastddc_inv_plan_run: the plan lives on device %d, the current device is %d", pl->dev, dev_now); return -1; }
    const int p = pl->cur;
    static const bool trace = getenv("CSDRB_INV_TRACE") && getenv("CSDRB_INV_TRACE")[0] == '1';      // tools only: timeline of this run, printed after a synchronize
    cudaEvent_t tev[5] = {};
    if (trace) { for (auto& e : tev) CSDRB_CUDA(cudaEventCreate(&e)); CSDRB_CUDA(cudaEventRecord(tev[0], st)); }
    if (!pl->ahead) {                                                     // first run, or the look-ahead was dropped by a retune / set_state
        if (int rc = plan_enqueue_prepare(pl, p)) return rc;
    }
    if (pl->chan_dirty) { CSDRB_CUDA(cudaStreamWaitEvent(st, pl->chan_set, 0)); pl->chan_dirty = false; }
    if (int rc = launch_fastddc_inv_apply(d_spectra, pl->nblocks, d_taps_fft, pl->d_chan, pl->channels, pl->fft_size, pl->fft_inv_size, pl->pre_decimation, pl->scrap,
                                          pl->post_input_size, pl->post_decimation, pl->prep[p], pl->folded, d_out, out_stride, pl->ready[p], pl->fold_done, st)) return rc;
    CSDRB_CUDA(cudaMemcpyAsync(d_out_total, pl->d_total[p], sizeof(int) * pl->channels, cudaMemcpyDeviceToDevice, st));
    CSDRB_CUDA(cudaEventRecord(pl->post_done[p], st));
    if (trace) CSDRB_CUDA(cudaEventRecord(tev[2], st));
    // look-ahead: the next run's chain and phasor walk, on the side stream
    const int q = 1 - p;
    CSDRB_CUDA(cudaStreamWaitEvent(pl->side, pl->post_done[q], 0));       // set q was last read two runs ago (a never-recorded event does not block)
    if (trace) CSDRB_CUDA(cudaEventRecord(tev[3], pl->side));
    // A chain walked NEXT TO the fold stretches the fold (one chain warp per channel, 64 SMs with a guest
    // that holds up every barrier of the fold CTA there), so chain and walk go behind the fold, next to the IFFT step and the caller's next forward FFT
    // ('f', the default).  CSDRB_PLAN_ORDER for A/B: 'd' = chain at once, walk behind the fold; 'i' = chain at once, walk behind the IFFT step; 's' = both behind the IFFT step.
    static const char order = getenv("CSDRB_PLAN_ORDER") ? getenv("CSDRB_PLAN_ORDER")[0] : 'f';
    if (order == 'f') CSDRB_CUDA(cudaStreamWaitEvent(pl->side, pl->fold_done, 0));
    if (order == 's') CSDRB_CUDA(cudaStreamWaitEvent(pl->side, pl->post_done[p], 0));
    if (int rc = plan_enqueue_prepare(pl, q, order == 'i' ? pl->post_done[p] : (order == 'd' ? pl->fold_done : nullptr))) return rc;
    pl->cur = q; pl->ahead = true;
    if (trace) {
        CSDRB_CUDA(cudaEventRecord(tev[4], pl->side));
        CSDRB_CUDA(cudaStreamSynchronize(st)); CSDRB_CUDA(cudaStreamSynchronize(pl->side));
        float t[5] = {};
        for (int i = 2; i < 5; ++i) cudaEventElapsedTime(&t[i], tev[0], tev[i]);
        cudaEventElapsedTime(&t[1], tev[0], pl->fold_done);
        fprintf(stderr, "[plan trace] us from run start: fold done %.1f, IFFT done %.1f | look-ahead for the next run: starts %.1f, done %.1f\n", t[1] * 1e3f, t[2] * 1e3f, t[3] * 1e3f, t[4] * 1e3f);
        for (auto& e : tev) cudaEventDestroy(e);
    }
    return pl->nblocks;
}

// Retune channel c from the next run on (the caller replaces that channel's taps_fft on its own stream).  Drops the look-ahead.
int fastddc_inv_plan_set_channel(void* plan, int c, const void* h_chan_one)
{
    auto* pl = static_cast<FastddcInvPlan*>(plan);
    if (!pl || !h_chan_one || c < 0 || c >= pl->channels) { set_error("fastddc_inv_plan_set_channel: bad arguments"); return -1; }
    std::lock_guard<std::mutex> lk(pl->mu);
    // the last run's kernels read d_chan: the copy goes behind them (post_done of the set read last), the next fold behind the copy (chan_set)
    CSDRB_CUDA(cudaStreamWaitEvent(pl->side, pl->post_done[1 - pl->cur], 0));
    CSDRB_CUDA(cudaMemcpyAsync(pl->d_chan + c, h_chan_one, sizeof(DdcChan), cudaMemcpyHostToDevice, pl->side));
    CSDRB_CUDA(cudaStreamSynchronize(pl->side));                          // h_chan_one may be a stack variable of the caller
    CSDRB_CUDA(cudaEventRecord(pl->chan_set, pl->side));
    pl->chan_dirty = true;
    pl->ahead = false;                                                    // set cur was prepared with the old parameters; the state it started from is still in the other set
    pl->tables_built = false;
    return 0;
}

// The carried state {remain, phase} per channel BEFORE the next run (what decimating_shift_addition_status_t carries, libcsdr_gpl.c:154-158).
int fastddc_inv_plan_get_state(void* plan, int* h_remain, float* h_phase)
{
    auto* pl = static_cast<FastddcInvPlan*>(plan);
    if (!pl || !h_remain || !h_phase) { set_error("fastddc_inv_plan_get_state: null pointer"); return -1; }
    std::lock_guard<std::mutex> lk(pl->mu);
    CSDRB_CUDA(cudaStreamSynchronize(pl->side));
    const int src = 1 - pl->cur;
    CSDRB_CUDA(cudaMemcpy(h_remain, pl->d_remain[src], sizeof(int) * pl->channels, cudaMemcpyDeviceToHost));
    CSDRB_CUDA(cudaMemcpy(h_phase, pl->d_phase[src], sizeof(float) * pl->channels, cudaMemcpyDeviceToHost));
    return 0;
}

int fastddc_inv_plan_set_state(void* plan, const int* h_remain, const float* h_phase)
{
    auto* pl = static_cast<FastddcInvPlan*>(plan);
    if (!pl || !h_remain || !h_phase) { set_error("fastddc_inv_plan_set_state: null pointer"); return -1; }
    std::lock_guard<std::mutex> lk(pl->mu);
    CSDRB_CUDA(cudaStreamSynchronize(pl->side));
    const int dst = 1 - pl->cur;
    CSDRB_CUDA(cudaMemcpy(pl->d_remain[dst], h_remain, sizeof(int) * pl->channels, cudaMemcpyHostToDevice));
    CSDRB_CUDA(cudaMemcpy(pl->d_phase[dst], h_phase, sizeof(float) * pl->channels, cudaMemcpyHostToDevice));
    pl->ahead = false;
    return 0;
}

}  // namespace csdrb
