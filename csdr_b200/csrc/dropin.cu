// dropin.cu -- Part A of the C ABI of libcsdr_b200.so (see include/csdr_b200.h): the libcsdr-named drop-ins on HOST buffers.
//
// Each call stages its buffers through the current device's workspace (grow-only device buffers, one private stream), runs the
// Part B entry point of capi.cu on them and waits for the result: synchronous per call, what a drop-in for a CPU library has to be.
#include "common.cuh"
#include "kernels.h"
#include "csdr_b200.h"

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <vector>

namespace csdrb {
namespace {

[[noreturn]] void die(const char* who)
{
    const char* e = csdrb_last_error();
    fprintf(stderr, "libcsdr_b200: %s failed: %s\n", who, e[0] ? e : "(no detail)");
    abort();
}

struct Workspace {
    struct Buffer { void* p = nullptr; size_t cap = 0; };
    std::mutex mu;
    cudaStream_t stream = nullptr;
    std::vector<Buffer> bufs;
};

// One drop-in call on the current device's workspace, whose mutex it holds for its lifetime.  The k-th alloc() of a call takes the
// workspace's k-th buffer.  A drop-in has no error return (the reference's contract), so a failure prints
// `libcsdr_b200: <who> failed: <detail>` and aborts.
class Staging {
public:
    explicit Staging(const char* who) : who_(who), ws_(per_device<Workspace>()), lock_(ws_.mu)
    {
        if (ws_.stream) return;
        int n = 0;
        cuda(cudaGetDeviceCount(&n), "cudaGetDeviceCount");
        if (n <= 0) { set_error("no CUDA device visible"); die(who_); }
        cuda(cudaStreamCreateWithFlags(&ws_.stream, cudaStreamNonBlocking), "cudaStreamCreateWithFlags");
    }
    cudaStream_t stream() const { return ws_.stream; }

    // room for n elements (none for n <= 0) and kSlack bytes more; a buffer that has to grow gets half as much again plus 4 KiB
    template <class T>
    T* alloc(long n)
    {
        const size_t bytes = (size_t)(n > 0 ? n : 0) * sizeof(T) + kSlack;
        if (next_ == ws_.bufs.size()) ws_.bufs.emplace_back();
        Workspace::Buffer& b = ws_.bufs[next_++];
        if (bytes > b.cap) {
            if (b.p) cuda(cudaFree(b.p), "cudaFree");
            b = {};
            cuda(cudaMalloc(&b.p, bytes + bytes / 2 + 4096), "cudaMalloc");
            b.cap = bytes + bytes / 2 + 4096;
        }
        return static_cast<T*>(b.p);
    }
    // copies of n <= 0 elements are skipped
    template <class T>
    void put(T* dev, const T* host, long n)
    {
        if (n > 0) cuda(cudaMemcpyAsync(dev, host, (size_t)n * sizeof(T), cudaMemcpyHostToDevice, ws_.stream), "cudaMemcpyAsync to the device");
    }
    template <class T>
    T* up(const T* host, long n)
    {
        T* dev = alloc<T>(n);
        put(dev, host, n);
        return dev;
    }
    template <class T>
    void get(T* host, const T* dev, long n)
    {
        if (n > 0) cuda(cudaMemcpyAsync(host, dev, (size_t)n * sizeof(T), cudaMemcpyDeviceToHost, ws_.stream), "cudaMemcpyAsync to the host");
    }
    int check(int rc) const
    {
        if (rc < 0) die(who_);
        return rc;
    }
    void sync() const { cuda(cudaStreamSynchronize(ws_.stream), "cudaStreamSynchronize"); }

private:
    static constexpr size_t kSlack = 64;            // kernels may read whole vectors past the last element
    void cuda(cudaError_t e, const char* what) const
    {
        if (e == cudaSuccess) return;
        cuda_fail(e, what, __FILE__, __LINE__);
        die(who_);
    }
    const char* who_;
    Workspace& ws_;
    std::lock_guard<std::mutex> lock_;
    size_t next_ = 0;
};

// the drop-ins that turn n values into n values with one Part B call f(d_in, d_out, n, stream); a value is in_items In elements on the way in
// and out_items Out elements on the way out (3 bytes of s24)
template <class In, class Out, class F>
void elementwise(const char* who, const In* input, Out* output, int n, F f, int in_items = 1, int out_items = 1)
{
    if (n <= 0) return;
    Staging st(who);
    const In* d_in = st.up(input, (long)n * in_items);
    Out* d_out = st.alloc<Out>((long)n * out_items);
    st.check(f(d_in, d_out, n, st.stream()));
    st.get(output, d_out, (long)n * out_items);
    st.sync();
}

struct csdrb_plan_impl { unsigned magic; int forward; };
const unsigned kPlanMagic = 0xC5D2B200u;
const unsigned kPlanMagicR2C = 0xC5D2B2F1u;                                // make_fft_r2c's plans (always forward)

}  // namespace
}  // namespace csdrb

using namespace csdrb;

extern "C" {

void convert_u8_f(unsigned char* input, float* output, int input_size) { elementwise("convert_u8_f", input, output, input_size, csdrb_convert_u8_f); }
void convert_s16_f(short* input, float* output, int input_size) { elementwise("convert_s16_f", input, output, input_size, csdrb_convert_s16_f); }
void convert_i16_f(short* input, float* output, int input_size) { convert_s16_f(input, output, input_size); }
void convert_f_s16(float* input, short* output, int input_size) { elementwise("convert_f_s16", input, output, input_size, csdrb_convert_f_s16); }
void convert_f_i16(float* input, short* output, int input_size) { convert_f_s16(input, output, input_size); }
void convert_s8_f(signed char* input, float* output, int input_size) { elementwise("convert_s8_f", input, output, input_size, csdrb_convert_s8_f); }
void convert_f_s8(float* input, signed char* output, int input_size) { elementwise("convert_f_s8", input, output, input_size, csdrb_convert_f_s8); }
void convert_f_u8(float* input, unsigned char* output, int input_size) { elementwise("convert_f_u8", input, output, input_size, csdrb_convert_f_u8); }
void convert_f_s24(float* input, unsigned char* output, int input_size, int bigendian)
{
    elementwise("convert_f_s24", input, output, input_size,
                [bigendian](const float* d_in, unsigned char* d_out, long n, void* s) { return csdrb_convert_f_s24(d_in, d_out, n, bigendian, s); }, 1, 3);
}
void convert_s24_f(unsigned char* input, float* output, int input_size, int bigendian)
{
    elementwise("convert_s24_f", input, output, input_size,
                [bigendian](const unsigned char* d_in, float* d_out, long n, void* s) { return csdrb_convert_s24_f(d_in, d_out, n, bigendian, s); }, 3, 1);
}

int fir_decimate_cc(complexf* input, complexf* output, int input_size, int decimation, float* taps, int taps_length)
{
    if (input_size < taps_length || input_size <= 0) return 0;
    Staging st("fir_decimate_cc");
    const int n_out = (input_size - taps_length) / decimation + 1;
    const complexf* d_in = st.up(input, input_size);
    complexf* d_out = st.alloc<complexf>(n_out);
    const int rc = st.check(csdrb_fir_decimate_bank_cc(d_in, (input_size + 1) & ~1, d_out, (n_out + 1) & ~1, 1, input_size, decimation, taps, taps_length, -1,
                                                       st.stream()));
    st.get(output, d_out, rc);
    st.sync();
    return rc;
}

complexf fmdemod_quadri_cf(complexf* input, float* output, int input_size, float* temp, complexf last_sample)
{
    (void)temp;
    if (input_size <= 0) return last_sample;
    Staging st("fmdemod_quadri_cf");
    const complexf* d_in = st.up(input, input_size);
    const complexf* d_last = st.up(&last_sample, 1);
    float* d_out = st.alloc<float>(input_size);
    st.check(csdrb_fmdemod_quadri_bank_cf(d_in, (input_size + 1) & ~1, d_out, (input_size + 1) & ~1, 1, input_size, d_last, nullptr, st.stream()));
    st.get(output, d_out, input_size);
    st.sync();
    return input[input_size - 1];
}

complexf fmdemod_quadri_novect_cf(complexf* input, float* output, int input_size, complexf last_sample)
{
    if (input_size <= 0) return last_sample;
    Staging st("fmdemod_quadri_novect_cf");
    const complexf* d_in = st.up(input, input_size);
    const complexf* d_last = st.up(&last_sample, 1);
    float* d_out = st.alloc<float>(input_size);
    st.check(csdrb_fmdemod_quadri_novect_bank_cf(d_in, (input_size + 1) & ~1, d_out, (input_size + 1) & ~1, 1, input_size, d_last, nullptr, st.stream()));
    st.get(output, d_out, input_size);
    st.sync();
    return input[input_size - 1];
}

float fmdemod_atan_cf(complexf* input, float* output, int input_size, float last_phase)
{
    if (input_size <= 0) return last_phase;
    Staging st("fmdemod_atan_cf");
    const complexf* d_in = st.up(input, input_size);
    float* d_phase = st.up(&last_phase, 1);                               // in: the carried phase; out: the last sample's
    float* d_out = st.alloc<float>(input_size);
    float* d_phase_out = st.alloc<float>(1);
    st.check(csdrb_fmdemod_atan_bank_cf(d_in, input_size, d_out, input_size, 1, input_size, d_phase, d_phase_out, st.stream()));
    st.get(output, d_out, input_size);
    st.get(&last_phase, d_phase_out, 1);
    st.sync();
    return last_phase;
}

void amdemod_estimator_cf(complexf* input, float* output, int input_size, float alpha, float beta)
{
    elementwise("amdemod_estimator_cf", input, output, input_size, [=](const complexf* in, float* out, long n, void* s) {
        return csdrb_amdemod_estimator_bank_cf(in, n, out, n, 1, (int)n, alpha, beta, s);
    });
}

// input == output gives what separate buffers give, not libcsdr's in-place result (include/csdr_b200.h)
dcblock_preserve_t dcblock_ff(float* input, float* output, int input_size, float a, dcblock_preserve_t preserved)
{
    if (input_size <= 0) return preserved;
    Staging st("dcblock_ff");
    const float* d_in = st.up(input, input_size);
    dcblock_preserve_t* d_state = st.up(&preserved, 1);
    float* d_out = st.alloc<float>(input_size);
    st.check(csdrb_dcblock_bank_ff(d_in, input_size, d_out, input_size, 1, input_size, a, d_state, st.stream()));
    st.get(output, d_out, input_size);
    st.get(&preserved, d_state, 1);
    st.sync();
    return preserved;
}

// ---- shift / fractional decimator / fastagc ----------------------------------------------------------
float shift_addition_cc(complexf* input, complexf* output, int input_size, shift_addition_data_t d, float starting_phase)
{
    if (input_size <= 0) return starting_phase;      // the reference still wraps the phase; with n = 0 nothing changes unless |phase| > pi
    Staging st("shift_addition_cc");
    struct State { shift_addition_data_t params; float phase; } s = {d, starting_phase};
    State* d_s = st.up(&s, 1);
    const complexf* d_in = st.up(input, input_size);
    complexf* d_out = st.alloc<complexf>(input_size);
    const size_t sb = csdrb_shift_addition_bank_scratch_bytes(1, input_size, input_size);
    void* scratch = st.alloc<char>(sb);
    st.check(csdrb_shift_addition_bank_cc(d_in, 0, d_out, 0, 1, input_size, &d_s->params, &d_s->phase, input_size, scratch, sb, st.stream()));
    st.get(output, d_out, input_size);
    st.get(&s.phase, &d_s->phase, 1);
    st.sync();
    return s.phase;
}

// The reference BUILD seeds shift_addition_fc's phasor with one sincosf() of the float phase (-ffast-math narrows the source's cos/sin pair of
// libcsdr_gpl.c:64-65 to it; objdump of the built libcsdr: `call sincosf@plt`), not with the double evaluation its shift_addition_cc keeps.  The
// two differ by an ulp for a few per cent of phases, and the recursion carries that through the call, so the drop-in seeds the call on the host
// with the same sincosf and gives the reference's bytes; the rest of the call is the bank kernel's.
float shift_addition_fc(float* input, complexf* output, int input_size, shift_addition_data_t d, float starting_phase)
{
    if (input_size <= 0) return starting_phase;      // as shift_addition_cc above
    Staging st("shift_addition_fc");
    struct State { shift_addition_data_t params; float phase; float2 seed; } s = {d, starting_phase, {0.f, 0.f}};
    sincosf(starting_phase, &s.seed.y, &s.seed.x);
    State* d_s = st.up(&s, 1);
    const float* d_in = st.up(input, input_size);
    complexf* d_out = st.alloc<complexf>(input_size);
    const size_t sb = csdrb_shift_addition_bank_scratch_bytes(1, input_size, input_size);
    void* scratch = st.alloc<char>(sb);
    const int rc = launch_shift_addition_fc_seeded(d_in, reinterpret_cast<float2*>(d_out), input_size, reinterpret_cast<const float*>(&d_s->params),
                                                   &d_s->phase, &d_s->seed, scratch, sb, st.stream());
    st.check(rc < 0 ? rc : counted(0, rc));
    st.get(output, d_out, input_size);
    st.get(&s.phase, &d_s->phase, 1);
    st.sync();
    return s.phase;
}

float shift_table_cc(complexf* input, complexf* output, int input_size, float rate, shift_table_data_t table_data, float starting_phase)
{
    if (input_size <= 0 || !table_data.table || table_data.table_size < 2) return starting_phase;
    Staging st("shift_table_cc");
    struct State { float rate, phase; } s = {rate, starting_phase};
    State* d_s = st.up(&s, 1);
    const complexf* d_in = st.up(input, input_size);
    complexf* d_out = st.alloc<complexf>(input_size);
    // the table is sent with every call (256 KB for the default size): a host pointer is no proof that the contents are the ones sent last time
    const float* d_table = st.up(table_data.table, table_data.table_size);
    const size_t sb = csdrb_shift_math_bank_scratch_bytes(1, input_size);
    void* scratch = st.alloc<char>(sb);
    st.check(csdrb_shift_table_bank_cc(d_in, 0, d_out, 0, 1, input_size, &d_s->rate, &d_s->phase, d_table, table_data.table_size, scratch, sb, st.stream()));
    st.get(output, d_out, input_size);
    st.get(&s.phase, &d_s->phase, 1);
    st.sync();
    return s.phase;
}

float shift_math_cc(complexf* input, complexf* output, int input_size, float rate, float starting_phase)
{
    if (input_size <= 0) return starting_phase;
    Staging st("shift_math_cc");
    struct State { float rate, phase; } s = {rate, starting_phase};
    State* d_s = st.up(&s, 1);
    const complexf* d_in = st.up(input, input_size);
    complexf* d_out = st.alloc<complexf>(input_size);
    const size_t sb = csdrb_shift_math_bank_scratch_bytes(1, input_size);
    void* scratch = st.alloc<char>(sb);
    st.check(csdrb_shift_math_bank_cc(d_in, 0, d_out, 0, 1, input_size, &d_s->rate, &d_s->phase, scratch, sb, st.stream()));
    st.get(output, d_out, input_size);
    st.get(&s.phase, &d_s->phase, 1);
    st.sync();
    return s.phase;
}

float shift_addfast_cc(complexf* input, complexf* output, int input_size, shift_addfast_data_t* d, float starting_phase)
{
    if (input_size <= 0 || !d) return starting_phase;
    Staging st("shift_addfast_cc");
    struct State { shift_addfast_data_t params; float phase; } s = {*d, starting_phase};
    State* d_s = st.up(&s, 1);
    const complexf* d_in = st.up(input, input_size);
    complexf* d_out = st.alloc<complexf>(input_size);
    const size_t sb = csdrb_shift_addition_bank_scratch_bytes(1, input_size, input_size);
    void* scratch = st.alloc<char>(sb);
    st.check(csdrb_shift_addfast_bank_cc(d_in, 0, d_out, 0, 1, input_size, &d_s->params, &d_s->phase, input_size, scratch, sb, st.stream()));
    st.get(output, d_out, input_size & ~3);                             // the n%4 tail of `output` is left alone, like the reference
    st.get(&s.phase, &d_s->phase, 1);
    st.sync();
    return s.phase;
}

decimating_shift_addition_status_t decimating_shift_addition_cc(complexf* input, complexf* output, int input_size, shift_addition_data_t d,
                                                                int decimation, decimating_shift_addition_status_t s)
{
    Staging st("decimating_shift_addition_cc");
    struct State { shift_addition_data_t params; int remain; float phase; int output_size; } h = {d, s.decimation_remain, s.starting_phase, 0};
    State* d_h = st.up(&h, 1);
    const complexf* d_in = st.up(input, input_size);
    complexf* d_out = st.alloc<complexf>(input_size / (decimation > 0 ? decimation : 1) + 2);
    st.check(csdrb_decimating_shift_addition_bank_cc(d_in, 0, d_out, 0, 1, input_size, &d_h->params, decimation, &d_h->remain, &d_h->phase,
                                                     &d_h->output_size, st.stream()));
    st.get(&h, d_h, 1);
    st.sync();
    if (h.output_size > 0) { st.get(output, d_out, h.output_size); st.sync(); }
    s.decimation_remain = h.remain; s.starting_phase = h.phase; s.output_size = h.output_size;
    return s;
}

fractional_decimator_ff_t fractional_decimator_ff_init(float rate, int num_poly_points, float* taps, int taps_length)
{
    // libcsdr.c:715-748 -- same field values; the three scratch arrays are kept so the struct stays layout- and
    // ownership-compatible with callers that free them.
    fractional_decimator_ff_t d;
    d.num_poly_points = num_poly_points & ~1;
    d.poly_precalc_denomiator = (float*)malloc(sizeof(float) * (size_t)(d.num_poly_points > 0 ? d.num_poly_points : 1));
    d.xifirst = -(num_poly_points / 2) + 1;
    d.xilast = num_poly_points / 2;
    int slot = 0;
    for (int xi = d.xifirst; xi <= d.xilast && slot < d.num_poly_points; xi++, slot++) {
        float prod = 1;
        for (int xj = d.xifirst; xj <= d.xilast; xj++) if (xi != xj) prod *= (float)(xi - xj);
        d.poly_precalc_denomiator[slot] = prod;
    }
    d.where = (float)(-d.xifirst);
    d.coeffs_buf = (float*)malloc(sizeof(float) * (size_t)(d.num_poly_points > 0 ? d.num_poly_points : 1));
    d.filtered_buf = (float*)malloc(sizeof(float) * (size_t)(d.num_poly_points > 0 ? d.num_poly_points : 1));
    d.rate = rate; d.taps = taps; d.taps_length = taps_length; d.input_processed = 0; d.output_size = 0;
    return d;
}

void fractional_decimator_ff(float* input, float* output, int input_size, fractional_decimator_ff_t* d)
{
    if (input_size <= 0) { d->output_size = 0; return; }
    Staging st("fractional_decimator_ff");
    csdrb_fracdec_state_t s = {d->where, 0, 0};
    csdrb_fracdec_state_t* d_s = st.up(&s, 1);
    const float* d_in = st.up(input, input_size);
    float* d_out = st.alloc<float>((int)((double)input_size / (d->rate > 1.f ? d->rate : 1.0)) + 8);
    const int tl = d->taps ? d->taps_length : 0;
    const float* d_taps = tl > 0 ? st.up(d->taps, tl) : nullptr;
    const size_t sb = csdrb_fractional_decimator_bank_scratch_bytes(1, input_size, d->rate);
    void* scratch = st.alloc<char>(sb);
    st.check(csdrb_fractional_decimator_bank_ff(d_in, 0, d_out, 0, 1, input_size, d->rate, d->num_poly_points, d_taps, tl, d_s, scratch, sb, st.stream()));
    st.get(&s, d_s, 1);
    st.sync();
    if (s.output_size > 0) { st.get(output, d_out, s.output_size); st.sync(); }
    d->where = s.where; d->input_processed = s.input_processed; d->output_size = s.output_size;
}

rational_resampler_ff_t rational_resampler_ff(float* input, float* output, int input_size, int interpolation, int decimation, float* taps,
                                              int taps_length, int last_taps_delay)
{
    Staging st("rational_resampler_ff");
    const long cap = interpolation > 0 && decimation > 0 && input_size > 0 ? (long)input_size * interpolation / decimation : 0;
    const float* d_in = st.up(input, input_size);
    float* d_out = st.alloc<float>(cap);
    rational_resampler_ff_t s;
    const int n = st.check(csdrb_rational_resampler_bank_ff(d_in, input_size, d_out, cap, 1, input_size, interpolation, decimation, taps, taps_length,
                                                            last_taps_delay, &s, st.stream()));
    st.get(output, d_out, n);
    st.sync();
    return s;
}

void fastagc_ff(fastagc_ff_t* a, float* output)
{
    const int n = a->input_size;
    if (n <= 0) return;
    Staging st("fastagc_ff");
    csdrb_fastagc_state_t s = {a->peak_1, a->peak_2, a->last_gain};
    csdrb_fastagc_state_t* d_s = st.up(&s, 1);
    const float* d_in = st.up(a->buffer_input, n);
    float* d_hist = st.alloc<float>(2L * n);                            // the two previous blocks, buffer_1 first
    st.put(d_hist, a->buffer_1, n);
    st.put(d_hist + n, a->buffer_2, n);
    float* d_out = st.alloc<float>(n);
    const size_t sb = csdrb_fastagc_bank_scratch_bytes(1, 1);
    void* scratch = st.alloc<char>(sb);
    st.check(csdrb_fastagc_bank_ff(d_in, 0, d_out, 0, 1, n, 1, a->reference, d_s, d_hist, scratch, sb, st.stream()));
    st.get(output, d_out, n);
    st.get(&s, d_s, 1);
    st.sync();
    // rotate the three caller-owned buffers exactly like libcsdr.c:981-989
    float* recycled = a->buffer_1;
    a->buffer_1 = a->buffer_2; a->buffer_2 = a->buffer_input; a->buffer_input = recycled;
    a->peak_1 = s.peak_1; a->peak_2 = s.peak_2; a->last_gain = s.last_gain;
}

// ---- spectrum, shift_unroll, ADPCM ------------------------------------------------------------------
void apply_precalculated_window_c(complexf* input, complexf* output, int size, float* windowt)
{
    if (size <= 0) return;
    Staging st("apply_precalculated_window_c");
    const complexf* d_in = st.up(input, size);
    const float* d_window = st.up(windowt, size);
    complexf* d_out = st.alloc<complexf>(size);
    st.check(csdrb_apply_window_rows_c(d_in, d_out, d_window, size, 1, st.stream()));
    st.get(output, d_out, size);
    st.sync();
}

// fft_fc windows its frames on the host (csdr.c:3478) right before fft_execute stages them: an O(n) multiply that a device round trip would only
// slow down.  The float product is the one the real waterfall bank computes on the device (__fmul_rn).
void apply_precalculated_window_f(float* input, float* output, int size, float* windowt)
{
    for (int i = 0; i < size; i++) output[i] = input[i] * windowt[i];
}

void apply_window_c(complexf* input, complexf* output, int size, window_t window)
{
    float* table = precalculate_window(size, window);                    // the table itself is one-off host work, like every filter design step
    apply_precalculated_window_c(input, output, size, table);
    free(table);
}

void logpower_cf(complexf* input, float* output, int size, float add_db)
{
    elementwise("logpower_cf", input, output, size, [=](const complexf* in, float* out, long n, void* s) { return csdrb_logpower_cf(in, out, n, add_db, s); });
}

void accumulate_power_cf(complexf* input, float* output, int size)
{
    if (size <= 0) return;
    Staging st("accumulate_power_cf");
    const complexf* d_in = st.up(input, size);
    float* d_acc = st.up(output, size);
    st.check(csdrb_accumulate_power_cf(d_in, d_acc, size, st.stream()));
    st.get(output, d_acc, size);
    st.sync();
}

void log_ff(float* input, float* output, int size, float add_db)
{
    elementwise("log_ff", input, output, size, [=](const float* in, float* out, long n, void* s) { return csdrb_log_ff(in, out, n, add_db, s); });
}

float shift_unroll_cc(complexf* input, complexf* output, int input_size, shift_unroll_data_t* d, float starting_phase)
{
    const char* who = "shift_unroll_cc";
    if (input_size <= 0) return starting_phase;
    if (!d || input_size > d->size) { set_error("input_size %d exceeds the table size %d", input_size, d ? d->size : 0); die(who); }
    Staging st(who);
    const complexf* d_in = st.up(input, input_size);
    const float* d_phase = st.up(&starting_phase, 1);                    // single call = single chunk: chunk_phase[0] is the starting phase itself
    const float* d_dsin = st.up(d->dsin, d->size);
    const float* d_dcos = st.up(d->dcos, d->size);
    complexf* d_out = st.alloc<complexf>(input_size);
    shift_unroll_bank_single(reinterpret_cast<const float2*>(d_in), reinterpret_cast<float2*>(d_out), input_size, d_dsin, d_dcos, d_phase, st.stream());
    counted(0, 1);
    st.get(output, d_out, input_size);
    st.sync();
    // one call = one chunk: the phase carried to the next call is one float multiply-add and a wrap -- done right here on the host
    float new_phase = starting_phase + input_size * d->phase_increment;
    while (new_phase > kPiF) new_phase -= 2 * kPiF;
    while (new_phase < -kPiF) new_phase += 2 * kPiF;
    return new_phase;
}

ima_adpcm_state_t encode_ima_adpcm_i16_u8(short* input, unsigned char* output, int input_length, ima_adpcm_state_t state)
{
    if (input_length < 2) return state;
    Staging st("encode_ima_adpcm_i16_u8");
    const short* d_in = st.up(input, input_length);
    ima_adpcm_state_t* d_state = st.up(&state, 1);
    unsigned char* d_out = st.alloc<unsigned char>(input_length / 2);
    st.check(csdrb_encode_ima_adpcm_rows_i16_u8(d_in, input_length, d_out, input_length / 2, 1, input_length, d_state, st.stream()));
    st.get(output, d_out, input_length / 2);
    st.get(&state, d_state, 1);
    st.sync();
    return state;
}

// ---- audio tail, AM / SSB --------------------------------------------------------------------------
void limit_ff(float* input, float* output, int input_size, float max_amplitude)
{
    elementwise("limit_ff", input, output, input_size, [=](const float* in, float* out, long n, void* s) { return csdrb_limit_ff(in, out, n, max_amplitude, s); });
}

void amdemod_cf(complexf* input, float* output, int input_size) { elementwise("amdemod_cf", input, output, input_size, csdrb_amdemod_cf); }

// one call = one block; returns the block's average like libcsdr.c:940 (0 for input_size <= 0, as the reference build does).  input == output is allowed.
float fastdcblock_ff(float* input, float* output, int input_size, float last_dc_level)
{
    if (input_size <= 0) return 0.f;
    Staging st("fastdcblock_ff");
    const float* d_in = st.up(input, input_size);
    float* d_dc = st.up(&last_dc_level, 1);                              // in: the previous block's average; out: this block's
    float* d_out = st.alloc<float>(input_size);
    st.check(csdrb_fastdcblock_bank_ff(d_in, input_size, 0, d_out, input_size, 1, input_size, 1, d_dc, st.stream()));
    st.get(output, d_out, input_size);
    float avg = 0.f;
    st.get(&avg, d_dc, 1);
    st.sync();
    return avg;
}

// one call = one agc_ff call of input_size samples; returns the last gain (libcsdr_gpl.c:259)
float agc_ff(float* input, float* output, int input_size, float reference, float attack_rate, float decay_rate, float max_gain,
             short hang_time, short attack_wait_time, float gain_filter_alpha, float last_gain)
{
    if (input_size <= 0) return last_gain;
    Staging st("agc_ff");
    const float* d_in = st.up(input, input_size);
    csdrb_agc_state_t s = {last_gain, 0.f, 0, 0, 0};
    csdrb_agc_state_t* d_s = st.up(&s, 1);
    float* d_out = st.alloc<float>(input_size);
    const csdrb_agc_params_t p = {reference, attack_rate, decay_rate, max_gain, hang_time, attack_wait_time, gain_filter_alpha, input_size};
    st.check(csdrb_agc_bank_ff(d_in, input_size, 0, d_out, input_size, 0, 1, input_size, &p, d_s, 0.f, st.stream()));
    st.get(output, d_out, input_size);
    st.get(&s, d_s, 1);
    st.sync();
    return s.gain;
}

float deemphasis_wfm_ff(float* input, float* output, int input_size, float tau, int sample_rate, float last_output)
{
    if (input_size <= 0) return last_output;
    Staging st("deemphasis_wfm_ff");
    const float* d_in = st.up(input, input_size);
    float* d_last = st.up(&last_output, 1);
    float* d_out = st.alloc<float>(input_size);
    st.check(csdrb_deemphasis_wfm_bank_ff(d_in, input_size, d_out, input_size, 1, input_size, tau, sample_rate, d_last, st.stream()));
    st.get(output, d_out, input_size);
    st.sync();
    return output[input_size - 1];
}

int deemphasis_nfm_ff(float* input, float* output, int input_size, int sample_rate)
{
    int taps_length = 0;
    if (!csdrb_deemphasis_nfm_taps(sample_rate, &taps_length)) return 0;          // libcsdr.c:1119: no table for this rate
    if (input_size - taps_length <= 0) return 0;
    Staging st("deemphasis_nfm_ff");
    const float* d_in = st.up(input, input_size);
    float* d_out = st.alloc<float>(input_size);
    const int produced = st.check(csdrb_deemphasis_nfm_bank_ff(d_in, input_size, d_out, input_size, 1, input_size, sample_rate, 0.f, st.stream()));
    st.get(output, d_out, produced);
    st.sync();
    return produced;
}

// ---- FFT abstraction, overlap-add step, fastddc ---------------------------------------------------------
FFT_PLAN_T* make_fft_c2c(int size, complexf* input, complexf* output, int forward, int benchmark)
{
    (void)benchmark;
    if (size < 2 || size > kFftLargeMaxN || (size & (size - 1))) {
        fprintf(stderr, "libcsdr_b200: make_fft_c2c: size %d unsupported (power of two, 2..%d)\n", size, kFftLargeMaxN);
        return nullptr;
    }
    FFT_PLAN_T* p = (FFT_PLAN_T*)malloc(sizeof(FFT_PLAN_T));
    csdrb_plan_impl* impl = (csdrb_plan_impl*)malloc(sizeof(csdrb_plan_impl));
    impl->magic = kPlanMagic; impl->forward = forward ? 1 : 0;
    p->size = size; p->input = input; p->output = output; p->plan = impl;
    return p;
}

FFT_PLAN_T* make_fft_r2c(int size, float* input, complexf* output, int benchmark)
{
    (void)benchmark;
    if (size < 4 || size > 2 * kFftLargeMaxN || (size & (size - 1))) {
        fprintf(stderr, "libcsdr_b200: make_fft_r2c: size %d unsupported (power of two, 4..%d)\n", size, 2 * kFftLargeMaxN);
        return nullptr;
    }
    FFT_PLAN_T* p = (FFT_PLAN_T*)malloc(sizeof(FFT_PLAN_T));
    csdrb_plan_impl* impl = (csdrb_plan_impl*)malloc(sizeof(csdrb_plan_impl));
    impl->magic = kPlanMagicR2C; impl->forward = 1;
    p->size = size; p->input = input; p->output = output; p->plan = impl;
    return p;
}

// size real points in, size/2 + 1 bins out, like FFTW's r2c
static void fft_execute_r2c(FFT_PLAN_T* plan)
{
    Staging st("fft_execute");
    const int n = plan->size;
    const float* d_in = st.up(static_cast<const float*>(plan->input), n);
    complexf* d_out = st.alloc<complexf>(n / 2 + 1);
    st.check(csdrb_fft_r2c_batch(d_in, n, d_out, n / 2 + 1, n, 1, st.stream()));
    st.get(static_cast<complexf*>(plan->output), d_out, n / 2 + 1);
    st.sync();
}

void fft_execute(FFT_PLAN_T* plan)
{
    const char* who = "fft_execute";
    if (!plan) return;
    if (plan->plan && ((csdrb_plan_impl*)plan->plan)->magic == kPlanMagicR2C) { fft_execute_r2c(plan); return; }
    if (!plan->plan || ((csdrb_plan_impl*)plan->plan)->magic != kPlanMagic) {
        set_error("plan was not created by libcsdr_b200's make_fft_c2c or make_fft_r2c (c2r plans are outside the hot path)"); die(who);
    }
    const int inverse = ((csdrb_plan_impl*)plan->plan)->forward ? 0 : 1;
    elementwise(who, static_cast<const complexf*>(plan->input), static_cast<complexf*>(plan->output), plan->size,
                [=](const complexf* in, complexf* out, long n, void* s) {
                    return n < kFftLargeMinN ? csdrb_fft_c2c_batch(in, n, out, n, (int)n, 1, inverse, s) : csdrb_fft_c2c_large_batch(in, n, out, n, (int)n, 1, inverse, s);
                });
}

void fft_destroy(FFT_PLAN_T* plan) { if (plan) { free(plan->plan); free(plan); } }
void* csdrb_fft_malloc(size_t bytes) { void* p = nullptr; return posix_memalign(&p, 64, bytes ? bytes : 64) ? nullptr : p; }
void csdrb_fft_free(void* p) { free(p); }

void apply_fir_fft_cc(FFT_PLAN_T* plan, FFT_PLAN_T* plan_inverse, complexf* taps_fft, complexf* last_overlap, int overlap_size)
{
    // libcsdr.c:814-849 in one fused kernel (above 16384 points: transform, product, transform, overlap add as separate launches): the intermediate
    // spectrum (plan->output) and product (plan_inverse->input) never leave the GPU, so those two caller buffers are NOT written (no caller in the
    // reference reads them).
    Staging st("apply_fir_fft_cc");
    const int n = plan->size;
    const complexf* d_in = st.up(static_cast<const complexf*>(plan->input), n);
    const complexf* d_taps = st.up(taps_fft, n);
    const complexf* d_overlap = st.up(last_overlap, overlap_size);
    complexf* d_out = st.alloc<complexf>(n);
    const int launches = st.check(launch_apply_fir_fft(reinterpret_cast<const float2*>(d_in), reinterpret_cast<const float2*>(d_taps), reinterpret_cast<const float2*>(d_overlap),
                                                       overlap_size, reinterpret_cast<float2*>(d_out), n, st.stream()));
    counted(0, launches);
    st.get(static_cast<complexf*>(plan_inverse->output), d_out, n);
    st.sync();
}

decimating_shift_addition_status_t fastddc_inv_cc(complexf* input, complexf* output, fastddc_t* ddc, FFT_PLAN_T* plan_inverse, complexf* taps_fft,
                                                  decimating_shift_addition_status_t shift_stat)
{
    (void)plan_inverse;
    {
        Staging st("fastddc_inv_cc");
        struct State { csdrb_fastddc_chan_t chan; int remain; float phase; int total; } s =
            {{ddc->offsetbin, ddc->dsadata.sindelta, ddc->dsadata.cosdelta, ddc->dsadata.rate}, shift_stat.decimation_remain, shift_stat.starting_phase, 0};
        State* d_s = st.up(&s, 1);
        const complexf* d_in = st.up(input, ddc->fft_size);
        const complexf* d_taps = st.up(taps_fft, ddc->fft_size);
        complexf* d_out = st.alloc<complexf>(ddc->post_input_size);
        const size_t sb = csdrb_fastddc_inv_bank_scratch_bytes(1, 1);
        void* scratch = st.alloc<char>(sb);
        st.check(csdrb_fastddc_inv_bank_cc(d_in, 1, d_taps, &d_s->chan, 1, ddc, &d_s->remain, &d_s->phase, d_out, ddc->post_input_size, &d_s->total,
                                           scratch, sb, st.stream()));
        st.get(&s, d_s, 1);
        st.sync();
        if (s.total > 0) { st.get(output, d_out, s.total); st.sync(); }
        shift_stat.decimation_remain = s.remain; shift_stat.starting_phase = s.phase; shift_stat.output_size = s.total;
    }
    fft_swap_sides(input, ddc->fft_size);            // the reference leaves its input swapped in place (fastddc.c:123), once the workspace is released
    return shift_stat;
}

// ---- BPSK31 receive chain ---------------------------------------------------------------------------------
void simple_agc_cc(complexf* input, complexf* output, int input_size, float rate, float reference, float max_gain, float* current_gain)
{
    if (input_size <= 0) return;
    Staging st("simple_agc_cc");
    const complexf* d_in = st.up(input, input_size);
    float* d_gain = st.up(current_gain, 1);
    complexf* d_out = st.alloc<complexf>(input_size);
    st.check(csdrb_simple_agc_bank_cc(d_in, input_size, d_out, input_size, 1, input_size, rate, reference, max_gain, d_gain, st.stream()));
    st.get(output, d_out, input_size);
    st.get(current_gain, d_gain, 1);
    st.sync();
}

// the reference's `static complexf last_input` (libcsdr.c:2321), zero at process start
static std::mutex g_dbpsk_mu;
static complexf g_dbpsk_last = {0.f, 0.f};

void dbpsk_decoder_c_u8(complexf* input, unsigned char* output, int input_size)
{
    if (input_size <= 0) return;
    std::lock_guard<std::mutex> lk(g_dbpsk_mu);
    Staging st("dbpsk_decoder_c_u8");
    const complexf* d_in = st.up(input, input_size);
    const complexf* d_last_in = st.up(&g_dbpsk_last, 1);
    unsigned char* d_out = st.alloc<unsigned char>(input_size);
    st.check(csdrb_dbpsk_decoder_bank_c_u8(d_in, input_size, d_out, input_size, 1, input_size, nullptr, d_last_in, nullptr, st.stream()));
    st.get(output, d_out, input_size);
    st.sync();
    g_dbpsk_last = input[input_size - 1];
}

timing_recovery_state_t timing_recovery_init(timing_recovery_algorithm_t algorithm, int decimation_rate, int use_q, float loop_gain, float max_error,
                                             int debug_every_nth, char* debug_writefiles_path)
{
    timing_recovery_state_t s = {};                                        // libcsdr.c:1960-1973
    s.algorithm = algorithm; s.decimation_rate = decimation_rate; s.loop_gain = loop_gain; s.max_error = max_error; s.use_q = use_q;
    s.debug_phase = s.debug_every_nth = debug_every_nth; s.last_correction_offset = 0; s.earlylate_ratio = 0.25f;
    s.debug_writefiles_path = debug_writefiles_path;
    return s;
}

void timing_recovery_cc(complexf* input, complexf* output, int input_size, float* timing_error, int* sampled_indexes, timing_recovery_state_t* state)
{
    if (state->debug_every_nth >= 0) { set_error("the octave debug output (debug_every_nth >= 0) is not part of this build"); die("timing_recovery_cc"); }
    if (state->earlylate_ratio != 0.25f) { set_error("earlylate_ratio other than timing_recovery_init's 0.25 is not served"); die("timing_recovery_cc"); }
    const csdrb_timing_recovery_params_t p = {(int)state->algorithm, state->decimation_rate, state->use_q, state->loop_gain, state->max_error};
    csdrb_timing_recovery_state_t s = {state->last_correction_offset, 0, 0};
    const int n = input_size > 0 ? input_size : 0;
    const int cap = p.decimation >= 2 ? timing_recovery_max_outputs(p.decimation, n, p.loop_gain, p.max_error) : 1;
    Staging st("timing_recovery_cc");
    const complexf* d_in = st.up(input, n);
    struct Call { int start, size; csdrb_timing_recovery_state_t state; } call = {0, n, s};
    Call* d_call = st.up(&call, 1);
    complexf* d_out = st.alloc<complexf>(cap);
    float* d_err = timing_error ? st.alloc<float>(cap) : nullptr;
    int* d_idx = sampled_indexes ? st.alloc<int>(cap) : nullptr;
    st.check(csdrb_timing_recovery_bank_cc(d_in, n, &d_call->start, &d_call->size, n, d_out, cap, d_err, d_idx, 1, &p, &d_call->state, st.stream()));
    st.get(&call, d_call, 1);
    st.sync();
    const int m = call.state.output_size;
    st.get(output, d_out, m);
    if (timing_error) st.get(timing_error, d_err, m);
    if (sampled_indexes) st.get(sampled_indexes, d_idx, m);
    st.sync();
    state->input_processed = call.state.input_processed;
    state->output_size = m;
    state->last_correction_offset = call.state.last_correction_offset;
}

// ---- tone filters (libcsdr.c:2261-2273, 2335-2351) ---------------------------------------------------------
int apply_fir_cc(complexf* input, complexf* output, int input_size, complexf* taps, int taps_length)
{
    if (input_size < taps_length) return 0;
    Staging st("apply_fir_cc");
    const complexf* d_in = st.up(input, input_size);
    const complexf* d_taps = st.up(taps, taps_length);
    complexf* d_out = st.alloc<complexf>(input_size - taps_length + 1);
    const int n_out = st.check(csdrb_apply_fir_bank_cc(d_in, input_size, d_out, input_size, 1, input_size, d_taps, taps_length, st.stream()));
    st.get(output, d_out, n_out);
    st.sync();
    return n_out;
}

int fir_interpolate_cc(complexf* input, complexf* output, int input_size, int interpolation, float* taps, int taps_length)
{
    if (input_size <= 0) return 0;
    Staging st("fir_interpolate_cc");
    const complexf* d_in = st.up(input, input_size);
    const float* d_taps = st.up(taps, taps_length);
    const long groups = (long)input_size - ((long)taps_length - 1 + interpolation - 1) / (interpolation > 0 ? interpolation : 1);
    complexf* d_out = st.alloc<complexf>(groups > 0 ? groups * interpolation : 0);
    const int n_out = st.check(csdrb_fir_interpolate_bank_cc(d_in, input_size, d_out, groups > 0 ? groups * interpolation : 0, 1, input_size,
                                                             interpolation, d_taps, taps_length, st.stream()));
    st.get(output, d_out, n_out);
    st.sync();
    return n_out;
}

float fmmod_fc(float* input, complexf* output, int input_size, float last_phase)
{
    if (input_size <= 0) return last_phase;
    Staging st("fmmod_fc");
    const float* d_in = st.up(input, input_size);
    float* d_phase = st.up(&last_phase, 1);
    complexf* d_out = st.alloc<complexf>(input_size);
    st.check(csdrb_fmmod_bank_fc(d_in, input_size, d_out, input_size, 1, input_size, d_phase, st.stream()));
    st.get(output, d_out, input_size);
    st.get(&last_phase, d_phase, 1);
    st.sync();
    return last_phase;
}

// ---- the other modulators (libcsdr.c:1139-1142, 1174-1178, 1194-1208): one-row banks; input == output is staged like any other call ----------
void gain_ff(float* input, float* output, int input_size, float gain)
{
    elementwise("gain_ff", input, output, input_size,
                [=](const float* in, float* out, long n, void* s) { return csdrb_gain_bank_ff(in, n, out, n, 1, (int)n, gain, s); });
}

void add_dcoffset_cc(complexf* input, complexf* output, int input_size)
{
    elementwise("add_dcoffset_cc", input, output, input_size,
                [](const complexf* in, complexf* out, long n, void* s) { return csdrb_add_dcoffset_bank_cc(in, n, out, n, 1, (int)n, s); });
}

void fixed_amplitude_cc(complexf* input, complexf* output, int input_size, float new_amplitude)
{
    elementwise("fixed_amplitude_cc", input, output, input_size, [=](const complexf* in, complexf* out, long n, void* s) {
        return csdrb_fixed_amplitude_bank_cc(in, n, out, n, 1, (int)n, new_amplitude, s);
    });
}

// ---- BPSK31 transmit chain (libcsdr.c:1551-1575, 1828-1843, 1772-1782, 1793-1808) ------------------------------------------------
void psk31_varicode_encoder_u8_u8(unsigned char* input, unsigned char* output, int input_size, int output_max_size, int* input_processed,
                                  int* output_size)
{
    *input_processed = 0;
    *output_size = 0;
    if (input_size <= 0) return;
    Staging st("psk31_varicode_encoder_u8_u8");
    const unsigned char* d_in = st.up(input, input_size);
    const int room = output_max_size > 0 ? output_max_size : 0;
    unsigned char* d_out = st.alloc<unsigned char>(room);
    int* d_counts = st.alloc<int>(2);
    st.check(csdrb_psk31_varicode_encoder_bank_u8_u8(d_in, input_size, d_out, room, 1, input_size, nullptr, output_max_size, d_counts, d_counts + 1,
                                                     st.stream()));
    int counts[2];
    st.get(counts, d_counts, 2);
    st.sync();
    st.get(output, d_out, counts[1]);
    st.sync();
    *input_processed = counts[0];
    *output_size = counts[1];
}

unsigned char differential_codec(unsigned char* input, unsigned char* output, int input_size, int encode, unsigned char state)
{
    if (input_size <= 0) return state;
    Staging st("differential_codec");
    const unsigned char* d_in = st.up(input, input_size);
    unsigned char* d_state = st.up(&state, 1);
    unsigned char* d_out = st.alloc<unsigned char>(input_size);
    st.check(csdrb_differential_codec_bank_u8_u8(d_in, input_size, d_out, input_size, 1, input_size, nullptr, encode, d_state, st.stream()));
    st.get(output, d_out, input_size);
    st.get(&state, d_state, 1);
    st.sync();
    return state;
}

void psk_modulator_u8_c(unsigned char* input, complexf* output, int input_size, int n_psk)
{
    if (input_size <= 0) return;
    Staging st("psk_modulator_u8_c");
    const unsigned char* d_in = st.up(input, input_size);
    complexf* d_out = st.alloc<complexf>(input_size);
    st.check(csdrb_psk_modulator_bank_u8_c(d_in, input_size, d_out, input_size, 1, input_size, nullptr, n_psk, st.stream()));
    st.get(output, d_out, input_size);
    st.sync();
}

complexf psk31_interpolate_sine_cc(complexf* input, complexf* output, int input_size, int interpolation, complexf last_input)
{
    if (input_size <= 0) return last_input;
    Staging st("psk31_interpolate_sine_cc");
    const complexf* d_in = st.up(input, input_size);
    complexf* d_last = st.up(&last_input, 1);
    const long nout = (long)input_size * (interpolation > 0 ? interpolation : 0);
    complexf* d_out = st.alloc<complexf>(nout);
    st.check(csdrb_psk31_interpolate_sine_bank_cc(d_in, input_size, d_out, nout, 1, input_size, nullptr, interpolation, d_last, st.stream()));
    st.get(output, d_out, nout);
    st.get(&last_input, d_last, 1);
    st.sync();
    return last_input;
}

int bfsk_demod_cf(complexf* input, float* output, int input_size, complexf* mark_filter, complexf* space_filter, int taps_length)
{
    if (input_size < taps_length) return input_size - taps_length + 1;     // the reference returns the count it would have written
    Staging st("bfsk_demod_cf");
    const complexf* d_in = st.up(input, input_size);
    const complexf* d_mark = st.up(mark_filter, taps_length);
    const complexf* d_space = st.up(space_filter, taps_length);
    float* d_out = st.alloc<float>(input_size - taps_length + 1);
    const int n_out = st.check(csdrb_bfsk_demod_bank_cf(d_in, input_size, d_out, input_size, 1, input_size, d_mark, d_space, taps_length, st.stream()));
    st.get(output, d_out, n_out);
    st.sync();
    return n_out;
}

// ---- RTTY receive chain -----------------------------------------------------------------------------------
void serial_line_decoder_f_u8(serial_line_t* s, float* input, unsigned char* output, int input_size)
{
    const SerialLineParams p = {s->samples_per_bits, s->databits, s->stopbits, s->bit_sampling_width_ratio};
    if (p.databits < 1 || p.databits > 8) {
        set_error("databits %d: 1..8 are served (the CLI's range; wider characters are written as 16 or 32 bits)", p.databits);
        die("serial_line_decoder_f_u8");
    }
    s->output_size = 0;
    if (input_size <= 0) { s->input_used = 1; return; }                  // the edge search's i = 1 with nothing to read (libcsdr.c:1676-1678)
    Staging st("serial_line_decoder_f_u8");
    const float* d_in = st.up(input, input_size);
    struct Row { int start, count, stuck; } row = {0, 0, 0};
    Row* d_row = st.up(&row, 1);
    const int cap = serial_line_max_outputs(p.samples_per_bits, p.databits, p.stopbits, input_size);
    unsigned char* d_out = st.alloc<unsigned char>(cap);
    st.check(csdrb_serial_line_decoder_bank_f_u8(d_in, input_size, input_size, &d_row->start, d_out, cap, &d_row->count, &d_row->stuck, 1,
                                                 reinterpret_cast<const csdrb_serial_line_params_t*>(&p), input_size, st.stream()));
    st.get(&row, d_row, 1);
    st.sync();
    st.get(output, d_out, row.count);
    st.sync();
    s->output_size = row.count;
    s->input_used = row.start;
}

}  // extern "C"
