// fft.cu -- K7 batched c2c FFT (and its four-step form above 16384 points), K9 overlap-add FFT filter bank, a12 fastddc forward step, K8 fastddc inverse bank.
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
//   fft_r2c_batch_kernel  : fft_execute() of a make_fft_r2c plan (fft_fftw.c:16-24) up to 32768 real points, one CTA per row (fft_real.cuh);
//   fft_r2c_split_kernel    above that, the four-step transform of the packed rows and this split in place.
#include "fft_kernels.cuh"
#include "fft_large.cuh"
#include "fft_real.cuh"
#include "kernels.h"
#include "side_stream.cuh"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <mutex>
#include <vector>

namespace csdrb {

// ---- device tables -------------------------------------------------------------------------------
// Every twiddle table the FFT kernels read, per device (a process may csdrb_set_device() between calls), kind and size: filled on the host in
// double and rounded once, uploaded on first use.
enum FftTableKind { kTwRadix8, kTwRadix16, kTwLargeStep, kTwRfftSplit };

struct FftTables { std::mutex mu; std::map<std::pair<int, int>, float2*> by_kind_n; };

static int fft_table(FftTableKind kind, int n, const float2** out, cudaStream_t st)
{
    FftTables& c = per_device<FftTables>();
    std::lock_guard<std::mutex> lk(c.mu);
    auto it = c.by_kind_n.find({kind, n});
    if (it == c.by_kind_n.end()) {
        std::vector<float2> h;
        switch (kind) {
        case kTwRadix8: h.resize((size_t)3 * n); fft_fill_twiddles(n, h.data()); break;
        case kTwRadix16: h.resize((size_t)4 * n); fft16_fill_twiddles(n, h.data()); break;
        case kTwLargeStep:                                              // four-step inter-step twiddles: kFftLargeSplit low powers, then n / kFftLargeSplit high ones
            h.resize((size_t)kFftLargeSplit + n / kFftLargeSplit);
            for (int m = 0; m < (int)h.size(); m++) {
                const double a = -2.0 * 3.14159265358979323846 * (m < kFftLargeSplit ? (double)m : (double)kFftLargeSplit * (m - kFftLargeSplit)) / (double)n;
                h[(size_t)m] = make_float2((float)cos(a), (float)sin(a));
            }
            break;
        case kTwRfftSplit: h.resize((size_t)n / 2 + 1); rfft_fill_twiddles(n, h.data()); break;
        }
        float2* d = nullptr;
        CSDRB_CUDA(cudaMalloc(&d, sizeof(float2) * h.size()));
        CSDRB_CUDA(cudaMemcpyAsync(d, h.data(), sizeof(float2) * h.size(), cudaMemcpyHostToDevice, st));
        CSDRB_CUDA(cudaStreamSynchronize(st));                           // h leaves scope; once per device, kind and size
        it = c.by_kind_n.emplace(std::make_pair((int)kind, n), d).first;
    }
    *out = it->second;
    return 0;
}

int row_fft_twiddles(int n, const float2** out, cudaStream_t st) { return fft_table(n >= 32 ? kTwRadix16 : kTwRadix8, n, out, st); }
int get_rfft_twiddles(int m, const float2** out, cudaStream_t st) { return fft_table(kTwRfftSplit, m, out, st); }

// ---- K7: batched c2c -------------------------------------------------------------------------------
int launch_fft_c2c_batch(const float2* d_in, long in_stride, float2* d_out, long out_stride, int n, int batch, int inverse, cudaStream_t st)
{
    if (batch <= 0) return 0;
    if (n < 2 || n > FFT_MAX_N || (n & (n - 1))) { set_error("fft: size %d unsupported (power of two, 2..%d)", n, FFT_MAX_N); return -1; }
    const float2* tw = nullptr;
    if (int rc = row_fft_twiddles(n, &tw, st)) return rc;
    switch (n) {
#define X(N) case N: CSDRB_CUDA(launch_kernel(inverse ? fft_c2c_batch_kernel<N, true> : fft_c2c_batch_kernel<N, false>, batch, fft_threads(N), \
                                              sizeof(float2) * fft_smem_elems(N), st, d_in, in_stride, d_out, out_stride, tw)); return 1;
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
    if (blocks_per_cta <= 0) {
        // enough CTAs to fill the machine a few times over, but runs long enough that the recomputed lead-in block stays cheap
        long want = (kSmCount * 8 + channels - 1) / channels;
        blocks_per_cta = (int)((nblocks + want - 1) / want);
        if (blocks_per_cta < 16) blocks_per_cta = nblocks < 16 ? nblocks : 16;
    }
    const dim3 grid((nblocks + blocks_per_cta - 1) / blocks_per_cta, channels);
    const size_t fsmem = sizeof(float2) * ((size_t)fft_smem_elems(fft_size) + 2 * (size_t)(fft_size - input_size));
    // fused kernels: radix-16 passes at 256 and 4096 points, radix-8 passes at the other sizes from 16 on; 4 and 8 points take the staged kernel
    const bool r16 = fft_size == 256 || fft_size == 4096;
    const float2* tw = nullptr;
    if (int rc = fft_table(r16 ? kTwRadix16 : kTwRadix8, fft_size, &tw, st)) return rc;
    switch (fft_size) {
#define X(N) case N: \
        if constexpr (N == 256 || N == 4096) CSDRB_CUDA(launch_kernel(olafir_bank_fused16_kernel<N>, grid, fft_threads(N), fsmem, st, d_in, in_stride, d_out, out_stride, \
                                                                      d_taps_fft, taps_stride, d_tail_io, input_size, nblocks, blocks_per_cta, tw)); \
        else if constexpr (N >= 16 && N <= 8192) CSDRB_CUDA(launch_kernel(olafir_bank_fused_kernel<N>, grid, fft_threads(N), fsmem, st, d_in, in_stride, d_out, out_stride, \
                                                                           d_taps_fft, taps_stride, d_tail_io, input_size, nblocks, blocks_per_cta, tw)); \
        else if constexpr (N == 4 || N == 8) CSDRB_CUDA(launch_kernel(olafir_bank_kernel<N>, grid, fft_threads(N), sizeof(float2) * (size_t)(fft_smem_elems(N) + N), st, \
                                                                      d_in, in_stride, d_out, out_stride, d_taps_fft, taps_stride, d_tail_io, input_size, nblocks, blocks_per_cta, tw)); \
        break;
        CSDRB_FFT_SIZES(X)
#undef X
    }
    return 1;
}

// ---- fastddc forward -------------------------------------------------------------------------------
int launch_fastddc_fwd(const float2* d_in, float2* d_spectra, float2* d_overlap_io, int fft_size, int input_size, int nblocks, cudaStream_t st)
{
    if (nblocks <= 0) return 0;
    if (fft_size > FFT_MAX_N) return launch_fastddc_fwd_large(d_in, d_spectra, d_overlap_io, fft_size, input_size, nblocks, st);
    if (fft_size < 4 || (fft_size & (fft_size - 1))) { set_error("fastddc_fwd: fft_size %d unsupported (power of two, 4..%d)", fft_size, kFftLargeMaxN); return -1; }
    const float2* tw = nullptr;
    if (int rc = row_fft_twiddles(fft_size, &tw, st)) return rc;
    switch (fft_size) {
#define X(N) case N: if constexpr (N >= 4) CSDRB_CUDA(launch_kernel(fastddc_fwd_kernel<N>, nblocks, fft_threads(N), sizeof(float2) * fft_smem_elems(N), st, \
                                                                d_in, d_spectra, d_overlap_io, input_size, tw)); break;
        CSDRB_FFT_SIZES(X)
#undef X
    }
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
    if (fft_size > FFT_MAX_N) return launch_apply_fir_fft_large(d_in, d_taps_fft, d_last_overlap, overlap_size, d_out, fft_size, st);
    if (fft_size < 2 || (fft_size & (fft_size - 1))) { set_error("apply_fir_fft: fft_size %d unsupported (power of two, 2..%d)", fft_size, kFftLargeMaxN); return -1; }
    const float2* tw = nullptr;
    if (int rc = fft_table(kTwRadix8, fft_size, &tw, st)) return rc;
    switch (fft_size) {
#define X(N) case N: CSDRB_CUDA(launch_kernel(apply_fir_fft_kernel<N>, 1, fft_threads(N), sizeof(float2) * fft_smem_elems(N), st, \
                                              d_in, d_taps_fft, d_last_overlap, overlap_size, d_out, tw)); break;
        CSDRB_FFT_SIZES(X)
#undef X
    }
    return 1;
}

// ---- fastddc inverse bank ----------------------------------------------------------------------------
// device arrays of the data-independent half of an inverse-bank call
struct InvPrep { int* blk_remain; float* blk_phase; int* blk_offset; WrapTable* tables; float2* phasor; int kmax; };

// Geometries the fold path covers: whole 64-residue CTAs and an even pre-decimation (the half swap of the spectrum is then a rotation of the
// fold's k index).
bool fastddc_inv_fold_ok(int fft_size, int fft_inv_size)
{
    if (fft_inv_size < 64 || fft_inv_size > 1024 || (fft_inv_size & (fft_inv_size - 1)) || fft_size % fft_inv_size) return false;
    const int P = fft_size / fft_inv_size;
    return P >= 2 && P % 2 == 0;
}

// The data-independent half of a call: block-to-block {remain, phase} chain (updates the carried state, writes the per-block state and the
// output counts) and the post-shift phasors of every (channel, block) row.  Everything on stream `s`.
int launch_fastddc_inv_prepare(const void* d_chan, int channels, int nblocks, int post_input_size, int post_decimation, int* d_remain_io, float* d_phase_io,
                               int* d_out_total, const InvPrep& p, cudaStream_t s, bool build_tables = true)
{
    fastddc_state_chain_kernel<<<chain_ctas(channels, kFastddcChainWarps), 32 * kFastddcChainWarps, 0, s>>>(static_cast<const DdcChan*>(d_chan), d_remain_io, d_phase_io, p.blk_remain, p.blk_phase,
                                                       p.blk_offset, d_out_total, channels, nblocks, post_input_size, post_decimation, p.tables, build_tables ? 1 : 0);
    CSDRB_CUDA(cudaGetLastError());
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
    if (int rc = fft_table(kTwRadix8, fft_inv_size, &tw, st)) return rc;
    const size_t fsmem = sizeof(float2) * (size_t)FOLD_ST * 2 * (2 * FOLD_BT) * FOLD_R;
    const dim3 fgrid(fft_inv_size / FOLD_R, (channels + 2 * FOLD_CT - 1) / (2 * FOLD_CT), (nblocks + 2 * FOLD_BT - 1) / (2 * FOLD_BT));
    if (fgrid.y > 65535u || fgrid.z > 65535u) { set_error("fastddc_inv: bank too large for one call"); return -1; }
    const float inv_pre = 1.0f / (float)pre_decimation;
    const DdcChan* dc = static_cast<const DdcChan*>(d_chan);
    CSDRB_CUDA(launch_kernel(fastddc_fold_kernel, fgrid, FOLD_NT, fsmem, st, d_spectra, d_taps_fft, dc, folded, fft_size, fft_inv_size, nblocks, channels, inv_pre));
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
    return (((size_t)channels * nblocks * 12 + 64 + 15) & ~(size_t)15) + (nblocks > kWrapTableMinSteps ? (size_t)channels * sizeof(WrapTable) : 0);
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
    if (int rc = fft_table(kTwRadix8, fft_inv_size, &tw, st)) return rc;
    int* blk_remain = static_cast<int*>(d_scratch);
    float* blk_phase = reinterpret_cast<float*>(blk_remain + (size_t)channels * nblocks);
    int* blk_offset = reinterpret_cast<int*>(blk_phase + (size_t)channels * nblocks);
    WrapTable* tables = nblocks > kWrapTableMinSteps ? reinterpret_cast<WrapTable*>(static_cast<char*>(d_scratch) + (((size_t)channels * nblocks * 12 + 64 + 15) & ~(size_t)15)) : nullptr;
    // Fold path: fold as a batched contraction (fastddc_fold_kernel), IFFT + post shift in a second kernel, and the data-independent
    // block-to-block state chain + phasor walk on a side stream meanwhile.  Anything fastddc_inv_fold_ok() refuses takes the single-kernel forms below.
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
    fastddc_state_chain_kernel<<<chain_ctas(channels, kFastddcChainWarps), 32 * kFastddcChainWarps, 0, st>>>(static_cast<const DdcChan*>(d_chan), d_remain_io, d_phase_io, blk_remain, blk_phase,
                                                                    blk_offset, d_out_total, channels, nblocks, post_input_size, post_decimation, tables, 1);
    CSDRB_CUDA(cudaGetLastError());
    if (fft_inv_size >= 8 && fft_inv_size <= 32 && (fft_size / fft_inv_size) % 2 == 0) {          // (64..1024 with an even P is the fold path's)
        // Tile = CT channels x BT blocks per CTA (each spectrum bin fetched once per CT channels, each tap once per BT blocks).  Big tiles
        // save L2 traffic but a bank of 64 channels x 16 blocks is only 64 CTAs of 4x4 on the whole GPU (the launch is latency-bound),
        // so the tile shrinks until the grid covers the machine about twice.
        const long ctas44 = (long)((nblocks + 3) / 4) * ((channels + 3) / 4);
        const bool small_tile = ctas44 < 2 * kSmCount;
        const int CTv = small_tile ? 2 : 4, BTv = small_tile ? 2 : 4;
        const dim3 tgrid((nblocks + BTv - 1) / BTv, (channels + CTv - 1) / CTv);
        const size_t smem = sizeof(float2) * (size_t)CTv * BTv * fft_smem_elems(fft_inv_size);
        switch (fft_inv_size) {
#define X(M) case M: if constexpr (M >= 8 && M <= 32) \
            CSDRB_CUDA(launch_kernel(small_tile ? fastddc_inv_tiled_kernel<M, 2, 2> : fastddc_inv_tiled_kernel<M, 4, 4>, tgrid, 256, smem, st, d_spectra, d_taps_fft, \
                                     static_cast<const DdcChan*>(d_chan), blk_remain, blk_phase, blk_offset, d_out, out_stride, fft_size, pre_decimation, scrap, \
                                     post_input_size, post_decimation, nblocks, channels, tw)); break;
            CSDRB_FFT_SIZES(X)
#undef X
        }
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

static int plan_enqueue_prepare(FastddcInvPlan* pl, int q)
{
    // state of set q := state of the other set (what the previous preparation left), then the chain advances it in place
    CSDRB_CUDA(cudaMemcpyAsync(pl->d_remain[q], pl->d_remain[1 - q], sizeof(int) * pl->channels, cudaMemcpyDeviceToDevice, pl->side));
    CSDRB_CUDA(cudaMemcpyAsync(pl->d_phase[q], pl->d_phase[1 - q], sizeof(float) * pl->channels, cudaMemcpyDeviceToDevice, pl->side));
    if (int rc = launch_fastddc_inv_prepare(pl->d_chan, pl->channels, pl->nblocks, pl->post_input_size, pl->post_decimation, pl->d_remain[q], pl->d_phase[q],
                                            pl->d_total[q], pl->prep[q], pl->side, !pl->tables_built)) return rc;
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
        pr.tables = nblocks > kWrapTableMinSteps ? pl->tables : nullptr;
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
    // that holds up every barrier of the fold CTA there), so chain and walk go behind the fold, next to the IFFT step and the caller's next forward FFT.
    CSDRB_CUDA(cudaStreamWaitEvent(pl->side, pl->fold_done, 0));
    if (int rc = plan_enqueue_prepare(pl, q)) return rc;
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

// ==== four-step transforms above FFT_MAX_N points (kernels: fft_large.cuh) ==========================================================================
// ---- launchers -------------------------------------------------------------------------------------------------------------------------------------
template <int F, bool FIRST, typename In>
static int launch_step(In in, int in_b0, float2* out, long out_stride, int out_b0, int S, int count, bool inverse, const float2* lo, const float2* hi, cudaStream_t st)
{
    constexpr int W = kFftLargeTile;
    const float2* tw16 = nullptr;
    if (int rc = fft_table(kTwRadix16, F, &tw16, st)) return rc;
    CSDRB_CUDA(launch_kernel(inverse ? fft_large_step_kernel<F, true, FIRST, In> : fft_large_step_kernel<F, false, FIRST, In>, dim3(S / W, count), W * (F / 16),
                             sizeof(float2) * (size_t)W * fft_large_seg(F), st, in, in_b0, out, out_stride, out_b0, S, tw16, lo, hi));
    return 0;
}

// N = 2^LG = N1 * N2; the longer factor goes first
#define CSDRB_FFT_LARGE_SIZES(X) X(15, 256, 128) X(16, 256, 256) X(17, 512, 256) X(18, 512, 512) X(19, 1024, 512) X(20, 1024, 1024)

static bool fft_large_size_ok(int n) { return n >= kFftLargeMinN && n <= kFftLargeMaxN && (n & (n - 1)) == 0; }

// `batch` transforms in.at(b, .) -> d_out + b*out_stride, in chunks that keep the intermediate within kFftLargeScratchBytes; returns the launches
template <typename In>
static int fft_large_run(In in, float2* d_out, long out_stride, int n, int batch, bool inverse, cudaStream_t st)
{
    const float2* lo = nullptr;
    if (int rc = fft_table(kTwLargeStep, n, &lo, st)) return rc;
    const float2* hi = lo + kFftLargeSplit;
    const int chunk = (int)(kFftLargeScratchBytes / (sizeof(float2) * (size_t)n));
    float2* t = nullptr;
    CSDRB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&t), sizeof(float2) * (size_t)n * (size_t)(batch < chunk ? batch : chunk), st));
    int launches = 0, rc = 0;
    for (int b0 = 0; b0 < batch && rc == 0; b0 += chunk) {
        const int count = batch - b0 < chunk ? batch - b0 : chunk;
        switch (n) {
#define X(LG, N1, N2) case 1 << LG: \
            rc = launch_step<N1, true>(in, b0, t, (long)n, 0, N2, count, inverse, lo, hi, st); \
            if (rc == 0) rc = launch_step<N2, false>(LargeRowsIn{t, (long)n}, 0, d_out, out_stride, b0, N1, count, inverse, lo, hi, st); \
            break;
            CSDRB_FFT_LARGE_SIZES(X)
#undef X
        }
        launches += 2;
    }
    const cudaError_t freed = cudaFreeAsync(t, st);
    if (rc) return rc;
    CSDRB_CUDA(freed);
    return launches;
}

int launch_fft_c2c_large_batch(const float2* d_in, long in_stride, float2* d_out, long out_stride, int n, int batch, int inverse, cudaStream_t st)
{
    if (!fft_large_size_ok(n)) { set_error("fft (large): size %d unsupported (power of two, %d..%d)", n, kFftLargeMinN, kFftLargeMaxN); return -1; }
    if (batch <= 0) return 0;
    return fft_large_run(LargeRowsIn{d_in, in_stride}, d_out, out_stride, n, batch, inverse != 0, st);
}

int launch_fastddc_fwd_large(const float2* d_in, float2* d_spectra, float2* d_overlap_io, int fft_size, int input_size, int nblocks, cudaStream_t st)
{
    if (!fft_large_size_ok(fft_size)) { set_error("fastddc_fwd: fft_size %d unsupported (power of two, 4..%d)", fft_size, kFftLargeMaxN); return -1; }
    if (input_size <= 0 || input_size > fft_size) { set_error("fastddc_fwd: bad input_size %d for fft_size %d", input_size, fft_size); return -1; }
    const int overlap = fft_size - input_size;
    int launches = fft_large_run(LargeSlideIn{d_in, d_overlap_io, input_size, overlap}, d_spectra, (long)fft_size, fft_size, nblocks, false, st);
    if (launches < 0 || overlap == 0) return launches;
    // carry: the last `overlap` samples of (old overlap ++ new input).  A call shorter than the overlap shifts the old overlap, which a
    // many-CTA copy cannot do in place: it goes through a stream-ordered buffer.
    const long total = (long)nblocks * input_size;
    const unsigned ctas = (unsigned)((overlap + 255) / 256 < 1024 ? (overlap + 255) / 256 : 1024);
    if (total >= overlap) {
        fft_large_gather_overlap_kernel<<<ctas, 256, 0, st>>>(d_in, d_overlap_io, d_overlap_io, overlap, total);
        CSDRB_CUDA(cudaGetLastError());
    } else {
        float2* tmp = nullptr;
        CSDRB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&tmp), sizeof(float2) * (size_t)overlap, st));
        fft_large_gather_overlap_kernel<<<ctas, 256, 0, st>>>(d_in, d_overlap_io, tmp, overlap, total);
        CSDRB_CUDA(cudaGetLastError());
        CSDRB_CUDA(cudaMemcpyAsync(d_overlap_io, tmp, sizeof(float2) * (size_t)overlap, cudaMemcpyDeviceToDevice, st));
        CSDRB_CUDA(cudaFreeAsync(tmp, st));
    }
    return launches + 1;
}

// ==== real-to-complex transforms (kernels: fft_real.cuh) ===========================================================================================
// the split behind the four-step transform, in place: row r holds Z[0..M) and gets X[0..M]; thread k reads and writes only bins k and M - k
// (and M for k = 0, which no thread reads)
__global__ void __launch_bounds__(256)
fft_r2c_split_kernel(float2* __restrict__ y, long stride, int M, int rows, const float2* __restrict__ rtw)
{
    const int k = blockIdx.x * 256 + threadIdx.x;
    if (k > M / 2) return;
    for (int r = blockIdx.y; r < rows; r += gridDim.y) {
        RfftRowOut dst{y + (long)r * stride};
        rfft_split_pair(k, M, dst.y[k], dst.y[(M - k) & (M - 1)], rtw, dst);
    }
}

int launch_fft_r2c_batch(const float* d_in, long in_stride, float2* d_out, long out_stride, int n, int batch, cudaStream_t st)
{
    if (n < 4 || n > 2 * kFftLargeMaxN || (n & (n - 1))) { set_error("fft r2c: size %d unsupported (power of two, 4..%d)", n, 2 * kFftLargeMaxN); return -1; }
    if (batch <= 0) return 0;
    const int m = n / 2;
    if (batch > 1 && (in_stride < n || out_stride < m + 1)) {
        set_error("fft r2c: rows overlap (in_stride %ld < %d real points or out_stride %ld < %d bins)", in_stride, n, out_stride, m + 1); return -1;
    }
    const float2* rtw = nullptr;
    if (int rc = get_rfft_twiddles(m, &rtw, st)) return rc;
    if (m >= kFftLargeMinN) {
        // Z of the packed rows straight into the output rows (m of their m + 1 bins), then the split in place
        const int launches = fft_large_run(RfftLargeRowsIn{d_in, in_stride}, d_out, out_stride, m, batch, false, st);
        if (launches < 0) return launches;
        fft_r2c_split_kernel<<<dim3((unsigned)((m / 2 + 256) / 256), (unsigned)(batch < 65535 ? batch : 65535)), 256, 0, st>>>(d_out, out_stride, m, batch, rtw);
        CSDRB_CUDA(cudaGetLastError());
        return launches + 1;
    }
    const float2* tw = nullptr;
    if (int rc = row_fft_twiddles(m, &tw, st)) return rc;
    switch (m) {
#define X(M) case M: CSDRB_CUDA(launch_kernel(fft_r2c_batch_kernel<M>, batch, fft_threads(M), sizeof(float2) * fft_smem_elems(M), st, \
                                              d_in, in_stride, d_out, out_stride, tw, rtw)); return 1;
        CSDRB_FFT_SIZES(X)
#undef X
    }
    return -1;
}

int launch_apply_fir_fft_large(const float2* d_in, const float2* d_taps_fft, const float2* d_last_overlap, int overlap_size, float2* d_out,
                               int fft_size, cudaStream_t st)
{
    if (!fft_large_size_ok(fft_size)) { set_error("apply_fir_fft: fft_size %d unsupported (power of two, 2..%d)", fft_size, kFftLargeMaxN); return -1; }
    float2* spec = nullptr;
    CSDRB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&spec), sizeof(float2) * (size_t)fft_size, st));
    int rc = fft_large_run(LargeRowsIn{d_in, (long)fft_size}, spec, (long)fft_size, fft_size, 1, false, st);
    if (rc >= 0) {
        fft_large_times_taps_kernel<<<(fft_size + 255) / 256, 256, 0, st>>>(spec, d_taps_fft, fft_size);
        rc = fft_large_run(LargeRowsIn{spec, (long)fft_size}, d_out, (long)fft_size, fft_size, 1, true, st);
    }
    const cudaError_t freed = cudaFreeAsync(spec, st);
    if (rc < 0) return rc;
    CSDRB_CUDA(freed);
    fft_large_scale_overlap_kernel<<<(fft_size + 255) / 256, 256, 0, st>>>(d_out, d_last_overlap, overlap_size, 1.0f / (float)fft_size, fft_size);
    CSDRB_CUDA(cudaGetLastError());
    return 6;
}

}  // namespace csdrb
