// spectrum.cu -- the OpenWebRX waterfall chain as one streaming bank (SURVEY 8(f) rank 4):
//
//     fft_cc N E [window] | logaveragepower_cf ADD_DB N A | fft_exchange_sides_ff N [| compress_fft_adpcm_f_u8 N]
//
// on many independent streams (rows) at once, carrying fft_cc's framing and logaveragepower_cf's partial line between calls.
//   spectrum_frames_kernel<N> : one CTA per (row, frame): window -> N-point forward FFT -> bin power, the FFT being the device function of
//                               csdrb_fft_c2c_batch (block_row_fft_io) with the window in the first pass's
//                               loads and the power in the last pass's stores, so a frame's power has the bits of the composition
//                               apply_window_rows -> fft_c2c_batch -> accumulate_power.
//   spectrum_lines_kernel     : one thread per (row, bin pair b, b + N/2): sums the call's frames in frame order onto the carried accumulator,
//                               and at every line end writes 10*log10(acc) + add_db to the swapped positions and restarts from 0.
//   spectrum_history_kernel   : one CTA per row: the last N samples of the stream so far, for the frames of the next call.
// The real-input bank, `fft_fc N E W | logaveragepower_cf ADD_DB N A [| compress_fft_adpcm_f_u8 N]`, is the same host side and the same lines,
// history and ADPCM stages with two differences, the framing formula and the missing half swap:
//   spectrum_frames_real_kernel<N> : one CTA per (row, frame) of 2N real samples: the window in the loads of the packed N-point transform, the
//                               r2c split of fft_real.cuh (block_rfft_io, the device function of csdrb_fft_r2c_batch) and the power of bins 0..N-1.
// Frames are independent, so a single wideband row still spreads over the whole GPU; only the A-frame sums run in frame order, one thread per bin.
#include "fft_real.cuh"
#include "kernels.h"

namespace csdrb {

// frame k of a stream covers [(k+1)E - N, (k+1)E) when E <= N (fft_cc's memmove-and-refill, csdr.c:1608-1628), [kE, kE + N) when E > N
__host__ __device__ __forceinline__ long long spectrum_frame_start(long long k, int N, int E) { return E <= N ? (k + 1) * E - N : k * E; }

// samples before the call come from the carried history (the last N samples of the stream so far), samples before the stream are 0
struct SpectrumFrameIn {
    const float2* x; const float2* hist; const float* w; long long rel, s0; int N;
    __device__ __forceinline__ float2 load(int i) const
    {
        const long long q = rel + i;
        float2 v = make_float2(0.f, 0.f);
        if (q >= 0) v = __ldg(x + q);
        else if (s0 + i >= 0) v = hist[N + q];
        const float g = __ldg(w + i);
        return make_float2(__fmul_rn(v.x, g), __fmul_rn(v.y, g));       // apply_window_rows_kernel's rounding
    }
    __device__ __forceinline__ float4 load2(int i) const { const float2 a = load(i), b = load(i + 1); return make_float4(a.x, a.y, b.x, b.y); }
};

// frame k of a real stream (2N samples) covers [(k+1)E - 2N, (k+1)E) when E <= 2N.  When E > 2N fft_fc reads 2N floats and then skips E - 2N
// COMPLEX samples (csdr.c:3462-3470: the skip counts floats but freads sizeof(complexf) items), so frame k starts at k(2E - 2N).
__host__ __device__ __forceinline__ long long spectrum_frame_start_f(long long k, int N, int E)
{
    return E <= 2 * N ? (k + 1) * E - 2LL * N : k * (2LL * E - 2LL * N);
}

// packed element i of a real frame: the windowed samples 2i and 2i + 1 (scalar loads: a frame may start at an odd sample)
struct SpectrumRealFrameIn {
    const float* x; const float* hist; const float* w; long long rel, s0; int L;
    __device__ __forceinline__ float sample(int j) const
    {
        const long long q = rel + j;
        float v = 0.f;
        if (q >= 0) v = __ldg(x + q);
        else if (s0 + j >= 0) v = hist[L + q];
        return __fmul_rn(v, __ldg(w + j));                              // apply_precalculated_window_f's rounding
    }
    __device__ __forceinline__ float2 load(int i) const { return make_float2(sample(2 * i), sample(2 * i + 1)); }
    __device__ __forceinline__ float4 load2(int i) const { return make_float4(sample(2 * i), sample(2 * i + 1), sample(2 * i + 2), sample(2 * i + 3)); }
};

struct SpectrumPowerOut {                                               // accumulate_power_cf's term, one per bin
    float* p;
    __device__ __forceinline__ static float power(float2 v) { return __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)); }
    __device__ __forceinline__ void store(int i, float2 v) const { p[i] = power(v); }
    __device__ __forceinline__ void store2(int i, float2 a, float2 b) const { *reinterpret_cast<float2*>(p + i) = make_float2(power(a), power(b)); }
};

// tw: row_fft_twiddles(N), the table csdrb_fft_c2c_batch uses at this size
template <int N>
__global__ void __launch_bounds__(fft_threads(N))
spectrum_frames_kernel(const float2* __restrict__ in, long in_stride, const float2* __restrict__ hist /*[rows][N]*/, const float* __restrict__ window,
                       float* __restrict__ power /*[rows][frames][N]*/, long long consumed, int every, long long first_frame, int frames,
                       const float2* __restrict__ tw)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* s = reinterpret_cast<float2*>(smem_raw);
    const int f = blockIdx.x, r = blockIdx.y;
    const long long s0 = spectrum_frame_start(first_frame + f, N, every);
    SpectrumFrameIn src{in + (long)r * in_stride, hist + (long)r * N, window, s0 - consumed, s0, N};
    SpectrumPowerOut dst{power + ((long)r * frames + f) * N};
    block_row_fft_io<N, false>(s, tw, threadIdx.x, src, dst);
}

// bins 0..N-1 of a real frame (fft_fc writes no Nyquist bin)
struct SpectrumRealPowerOut {
    float* p; int N;
    __device__ __forceinline__ void store(int k, float2 v) const { if (k < N) p[k] = SpectrumPowerOut::power(v); }
};

// rtw: the split table of get_rfft_twiddles(N); tw as for spectrum_frames_kernel<N>
template <int N>
__global__ void __launch_bounds__(fft_threads(N))
spectrum_frames_real_kernel(const float* __restrict__ in, long in_stride, const float* __restrict__ hist /*[rows][2N]*/, const float* __restrict__ window,
                            float* __restrict__ power /*[rows][frames][N]*/, long long consumed, int every, long long first_frame, int frames,
                            const float2* __restrict__ tw, const float2* __restrict__ rtw)
{
    CSDRB_DYN_SMEM(smem_raw);
    float2* s = reinterpret_cast<float2*>(smem_raw);
    const int f = blockIdx.x, r = blockIdx.y;
    const long long s0 = spectrum_frame_start_f(first_frame + f, N, every);
    SpectrumRealFrameIn src{in + (long)r * in_stride, hist + (long)r * 2 * N, window, s0 - consumed, s0, 2 * N};
    SpectrumRealPowerOut dst{power + ((long)r * frames + f) * N, N};
    block_rfft_io<N>(s, tw, rtw, threadIdx.x, src, dst);
}

// One thread per (row, b < N/2) owns bins b and b + N/2, so the half swap of fft_exchange_sides_ff stays inside the thread (SWAP = false: the real
// bank's lines, in bin order).  Line j ends at
// frame jA + A - 1; its dB values go to out_f (row pitch out_stride floats, line j - line0 of the call) or, for the ADPCM stage, to db
// ([rows][lines_here][N], line j - chunk_line0).
template <bool SWAP>
__global__ void __launch_bounds__(256)
spectrum_lines_kernel(const float* __restrict__ power, int rows, int frames, int N, int averages, long long first_frame, float* __restrict__ acc_io,
                      float add_db, float* __restrict__ out_f, long out_stride, long long line0, float* __restrict__ db, int lines_here)
{
    const int half = N / 2;
    const long t = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (long)rows * half) return;
    const int r = (int)(t / half), b = (int)(t % half), b2 = b + half;
    const long long chunk_line0 = first_frame / averages;
    float a0 = acc_io[(long)r * N + b], a1 = acc_io[(long)r * N + b2];
    const float* p = power + (long)r * frames * N;
    for (int f = 0; f < frames; f++) {
        a0 = __fadd_rn(a0, p[(long)f * N + b]);
        a1 = __fadd_rn(a1, p[(long)f * N + b2]);
        const long long g = first_frame + f;
        if ((g + 1) % averages == 0) {
            const long long j = (g + 1) / averages - 1;
            const float d0 = __fadd_rn(__fmul_rn(10.f, (float)log10((double)a0)), add_db);     // log_ff (power_kernel mode 2)
            const float d1 = __fadd_rn(__fmul_rn(10.f, (float)log10((double)a1)), add_db);
            float* y = db ? db + ((long)r * lines_here + (long)(j - chunk_line0)) * N : out_f + (long)r * out_stride + (long)(j - line0) * N;
            if (SWAP) { y[b2] = d0; y[b] = d1; }                        // the two halves of the line swap places
            else { y[b] = d0; y[b2] = d1; }
            a0 = 0.f; a1 = 0.f;
        }
    }
    acc_io[(long)r * N + b] = a0; acc_io[(long)r * N + b2] = a1;
}

// new history = last H samples of [old history | n new samples]; element i reads position n + i >= i, so ascending chunks of one CTA,
// each read completely before it is written, never overwrite what a later chunk still reads
template <typename T>
__global__ void __launch_bounds__(256)
spectrum_history_kernel(const T* __restrict__ in, long in_stride, T* hist_io, int N, long n)
{
    const int r = blockIdx.x;
    const T* x = in + (long)r * in_stride;
    T* h = hist_io + (long)r * N;
    for (int base = 0; base < N; base += blockDim.x) {
        const int i = base + threadIdx.x;
        T v{};
        if (i < N) { const long c = n + i; v = c < N ? h[c] : x[c - N]; }
        __syncthreads();
        if (i < N) h[i] = v;
        __syncthreads();
    }
}

// ---- host side (both banks) ------------------------------------------------------------------------------------------------------------
static bool spectrum_size_ok(int N) { return N >= 2 && N <= FFT_MAX_N && (N & (N - 1)) == 0; }

long long spectrum_frames_at(int N, int E, long long total)            // frames a stream of `total` samples completes
{
    if (E <= N) return total / E;
    return total >= N ? (total - N) / E + 1 : 0;
}

long long spectrum_frames_at_f(int N, int E, long long total)          // the same for fft_fc: frames of 2N real samples, starts as spectrum_frame_start_f
{
    const long long L = 2LL * N;
    if (E <= L) return total / E;
    return total >= L ? (total - L) / (2LL * E - L) + 1 : 0;
}

static long long frames_at(const SpectrumParams* p, int real, long long total)
{
    return real ? spectrum_frames_at_f(p->fft_size, p->every, total) : spectrum_frames_at(p->fft_size, p->every, total);
}

static int spectrum_check_params(const SpectrumParams* p)
{
    if (!p) { set_error("spectrum bank: null parameters"); return -1; }
    if (p->every < 1 || p->averages < 1) { set_error("spectrum bank: every (%d) and averages (%d) must be at least 1", p->every, p->averages); return -1; }
    if (!spectrum_size_ok(p->fft_size)) { set_error("spectrum bank: fft_size %d unsupported (power of two, 2..%d)", p->fft_size, FFT_MAX_N); return -2; }
    return 0;
}

long spectrum_lines(const void* h_params_v, const void* h_state_v, long n, int real)
{
    const SpectrumParams* p = static_cast<const SpectrumParams*>(h_params_v);
    const SpectrumState* s = static_cast<const SpectrumState*>(h_state_v);
    if (int rc = spectrum_check_params(p)) return rc;
    if (!s || n < 0 || s->consumed < 0) { set_error("spectrum bank: bad state or n < 0"); return -1; }
    const long long f0 = frames_at(p, real, s->consumed), f1 = frames_at(p, real, s->consumed + n);
    return (long)(f1 / p->averages - f0 / p->averages);
}

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
static size_t spectrum_line_bytes(const SpectrumParams* p) { return p->compress ? (size_t)(p->fft_size + 10) / 2 : sizeof(float) * (size_t)p->fft_size; }

// scratch of a chunk of F frames per row: the bin powers, and for the ADPCM stage the dB lines and their bytes
static size_t spectrum_chunk_bytes(int rows, long long F, const SpectrumParams* p)
{
    const size_t N = (size_t)p->fft_size;
    size_t b = align256(sizeof(float) * (size_t)rows * (size_t)F * N);
    if (p->compress) {
        const size_t L = (size_t)((F + p->averages - 1) / p->averages);                 // lines that end in F consecutive frames
        b += align256(sizeof(float) * (size_t)rows * L * N) + align256((size_t)rows * L * spectrum_line_bytes(p));
    }
    return b;
}

// the same for both banks: frames start at least `every` samples apart
size_t spectrum_scratch_bytes(int rows, long n, const void* h_params_v)
{
    const SpectrumParams* p = static_cast<const SpectrumParams*>(h_params_v);
    if (!p || p->every < 1 || p->averages < 1 || !spectrum_size_ok(p->fft_size) || rows < 1 || n < 0) return 0;
    const long long F = (n + p->every - 1) / p->every;                   // the most frames n samples can complete
    return spectrum_chunk_bytes(rows, F > 1 ? F : 1, p);
}

// One body for both banks.  real = 0: d_in / d_hist_io are float2 (N-sample history); real = 1: float (2N-sample history), fft_fc's framing, no swap.
static int spectrum_bank_run(const void* d_in, long in_stride, int rows, long n, const float* d_window, const void* h_params_v, void* d_hist_io,
                             float* d_acc_io, void* h_state_io, void* d_out, long out_stride_bytes, void* d_scratch, size_t scratch_bytes, int* launches,
                             int real, cudaStream_t st)
{
    const SpectrumParams* p = static_cast<const SpectrumParams*>(h_params_v);
    SpectrumState* s = static_cast<SpectrumState*>(h_state_io);
    *launches = 0;
    if (!p) { set_error("spectrum bank: null parameters"); return -1; }
    if (rows < 1 || rows > 65535 || n < 0 || in_stride < 0 || out_stride_bytes < 0) { set_error("spectrum bank: bad rows (%d), n (%ld) or strides", rows, n); return -1; }
    if (int rc = spectrum_check_params(p)) return rc;
    const int N = p->fft_size, E = p->every, A = p->averages;
    if (!s || s->consumed < 0 || s->frames != frames_at(p, real, s->consumed)) { set_error("spectrum bank: the state does not belong to these parameters"); return -1; }
    if ((n > 0 && !d_in) || !d_window || !d_hist_io || !d_acc_io || !d_out || !d_scratch) { set_error("spectrum bank: null pointer"); return -1; }
    auto mis = [](const void* q, uintptr_t a) { return (reinterpret_cast<uintptr_t>(q) & (a - 1)) != 0; };
    const uintptr_t sample_align = real ? 4 : 8;
    if ((n > 0 && mis(d_in, sample_align)) || mis(d_hist_io, sample_align) || mis(d_acc_io, 4) || mis(d_window, 4) || mis(d_scratch, 16) ||
        (!p->compress && (mis(d_out, 4) || (out_stride_bytes & 3)))) {
        set_error(real ? "spectrum bank: misaligned pointer (input, history, accumulator, window and float output 4 bytes, scratch 16)"
                       : "spectrum bank: misaligned pointer (input and history 8 bytes, accumulator, window and float output 4, scratch 16)");
        return -1;
    }
    if (scratch_bytes < spectrum_chunk_bytes(rows, 1, p)) { set_error("spectrum bank: scratch too small (%zu bytes, one frame per row needs %zu)", scratch_bytes, spectrum_chunk_bytes(rows, 1, p)); return -1; }
    const long long f_first = s->frames, f_end = frames_at(p, real, s->consumed + n), line0 = f_first / A;
    const long lines = (long)(f_end / A - line0);
    // frames per chunk: as many as the scratch holds (never fewer than one per row); the chunking changes the launch count, not the bits
    long long F = f_end - f_first;
    {
        long long lo = 1, hi = F > 1 ? F : 1;
        while (lo < hi) { const long long mid = (lo + hi + 1) / 2; if (spectrum_chunk_bytes(rows, mid, p) <= scratch_bytes) lo = mid; else hi = mid - 1; }
        F = lo < 0x7fffffff ? lo : 0x7fffffff;
    }
    const float2 *tw = nullptr, *rtw = nullptr;
    if (f_end > f_first) {
        if (int rc = row_fft_twiddles(N, &tw, st)) return rc;
        if (real) { if (int rc = get_rfft_twiddles(N, &rtw, st)) return rc; }
    }
    const float add_db = (float)((double)p->add_db - 10.0 * log10((double)A));        // logaveragepower_cf's add_db -= 10*log10(avgnumber) on a float
    const size_t line_bytes = spectrum_line_bytes(p);
    float* power = static_cast<float*>(d_scratch);
    const float *xf = static_cast<const float*>(d_in), *hf = static_cast<const float*>(d_hist_io);
    const float2 *xc = static_cast<const float2*>(d_in), *hc = static_cast<const float2*>(d_hist_io);
    const size_t smem = sizeof(float2) * fft_smem_elems(N);
    for (long long g0 = f_first; g0 < f_end; g0 += F) {
        const int Fc = (int)(f_end - g0 < F ? f_end - g0 : F);
        const dim3 grid(Fc, rows);
        cudaError_t e = cudaSuccess;
        switch (N) {
#define X(M) case M: e = real ? launch_kernel(spectrum_frames_real_kernel<M>, grid, fft_threads(M), smem, st, xf, in_stride, hf, d_window, power, s->consumed, E, g0, Fc, tw, rtw) \
                              : launch_kernel(spectrum_frames_kernel<M>, grid, fft_threads(M), smem, st, xc, in_stride, hc, d_window, power, s->consumed, E, g0, Fc, tw); break;
            CSDRB_FFT_SIZES(X)
#undef X
        }
        CSDRB_CUDA(e);
        ++*launches;
        const int Lc = (int)((g0 + Fc) / A - g0 / A);
        float* db = nullptr;
        unsigned char* bytes = nullptr;
        if (p->compress) {
            db = reinterpret_cast<float*>(static_cast<char*>(d_scratch) + align256(sizeof(float) * (size_t)rows * (size_t)F * N));
            bytes = reinterpret_cast<unsigned char*>(db) + align256(sizeof(float) * (size_t)rows * (size_t)((F + A - 1) / A) * N);
        }
        const long threads = (long)rows * (N / 2);
        auto lines_kernel = real ? spectrum_lines_kernel<false> : spectrum_lines_kernel<true>;
        lines_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(power, rows, Fc, N, A, g0, d_acc_io, add_db, static_cast<float*>(d_out),
                                                                       out_stride_bytes / 4, line0, db, Lc);
        CSDRB_CUDA(cudaGetLastError());
        ++*launches;
        if (p->compress && Lc > 0) {
            // compress_fft_adpcm_f_u8 on every finished line (one launch for all rows), then the lines to their rows of d_out
            if (int rc = launch_compress_fft_adpcm_rows(db, N, bytes, (long)line_bytes, rows * Lc, N, st); rc < 0) return rc;
            ++*launches;
            char* dst = static_cast<char*>(d_out) + (size_t)(g0 / A - line0) * line_bytes;
            CSDRB_CUDA(cudaMemcpy2DAsync(dst, (size_t)out_stride_bytes, bytes, (size_t)Lc * line_bytes, (size_t)Lc * line_bytes, (size_t)rows,
                                         cudaMemcpyDeviceToDevice, st));
        }
    }
    if (n > 0) {
        if (real) spectrum_history_kernel<float><<<rows, 256, 0, st>>>(static_cast<const float*>(d_in), in_stride, static_cast<float*>(d_hist_io), 2 * N, n);
        else spectrum_history_kernel<float2><<<rows, 256, 0, st>>>(static_cast<const float2*>(d_in), in_stride, static_cast<float2*>(d_hist_io), N, n);
        CSDRB_CUDA(cudaGetLastError());
        ++*launches;
    }
    s->consumed += n;
    s->frames = f_end;
    return (int)lines;
}

int launch_spectrum_bank(const float2* d_in, long in_stride, int rows, long n, const float* d_window, const void* h_params_v, float2* d_hist_io,
                         float* d_acc_io, void* h_state_io, void* d_out, long out_stride_bytes, void* d_scratch, size_t scratch_bytes, int* launches,
                         cudaStream_t st)
{
    return spectrum_bank_run(d_in, in_stride, rows, n, d_window, h_params_v, d_hist_io, d_acc_io, h_state_io, d_out, out_stride_bytes, d_scratch,
                             scratch_bytes, launches, 0, st);
}

int launch_spectrum_bank_f(const float* d_in, long in_stride, int rows, long n, const float* d_window, const void* h_params_v, float* d_hist_io,
                           float* d_acc_io, void* h_state_io, void* d_out, long out_stride_bytes, void* d_scratch, size_t scratch_bytes, int* launches,
                           cudaStream_t st)
{
    return spectrum_bank_run(d_in, in_stride, rows, n, d_window, h_params_v, d_hist_io, d_acc_io, h_state_io, d_out, out_stride_bytes, d_scratch,
                             scratch_bytes, launches, 1, st);
}

}  // namespace csdrb
