// capi.cu -- the C ABI of libcsdr_b200.so (see include/csdr_b200.h).
//
// Part B (csdrb_*) entry points are thin: validate, launch on the caller's stream, count the launch.
// Part A (the libcsdr-named drop-ins on host buffers) lives in dropin.cu and calls these.
#include "common.cuh"
#include "kernels.h"
#include "csdr_b200.h"

#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>
#include <sched.h>

namespace csdrb {

static thread_local char g_err[512] = "";
static std::atomic<long> g_launches{0};

void set_error(const char* fmt, ...)
{
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap);
}
int cuda_fail(cudaError_t e, const char* what, const char* file, int line)
{
    set_error("CUDA error %d (%s) at %s:%d in `%s`", (int)e, cudaGetErrorString(e), file, line, what);
    return -(1000 + (int)e);
}
static inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }
int counted(int rc, int n) { if (rc >= 0) g_launches += n; return rc; }

// CSDRB_TRACE=1: report at exit how many kernels this process launched (lets a caller verify that a
// preloaded/linked libcsdr_b200 really did the work instead of some other libcsdr).
struct ExitReport {
    ~ExitReport()
    {
        const char* t = getenv("CSDRB_TRACE");
        if (t && *t && *t != '0') fprintf(stderr, "libcsdr_b200: %ld kernel launches in this process\n", g_launches.load());
    }
};
static ExitReport g_exit_report;

}  // namespace csdrb

using namespace csdrb;

extern "C" {

// =====================================================================================================
// Part B
// =====================================================================================================
const char* csdrb_last_error(void) { return g_err; }
const char* csdrb_version(void) { return "csdr_b200 0.1 (sm_90a)"; }
int csdrb_device_count(void)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) return cuda_fail(e, "cudaGetDeviceCount", __FILE__, __LINE__);
    return n;
}
int csdrb_set_device(int device) { CSDRB_CUDA(cudaSetDevice(device)); return 0; }
int csdrb_stream_synchronize(void* stream) { CSDRB_CUDA(cudaStreamSynchronize(S(stream))); return 0; }
long csdrb_kernel_launches(void) { return g_launches.load(); }

// channels ride in gridDim.y (limit 65535) in the bank kernels: refuse larger banks with a message instead of an "invalid configuration" launch error
static inline bool too_many_channels(int channels, const char* who)
{
    if (channels <= 65535) return false;
    set_error("%s: %d channels in one call (at most 65535; split the bank)", who, channels);
    return true;
}
static inline bool misaligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }
static inline bool null_io(const void* in, const void* out, const char* who) { if (in && out) return false; set_error("%s: null pointer", who); return true; }
int csdrb_convert_u8_f(const unsigned char* d_in, float* d_out, long n, void* stream)
{
    return null_io(d_in, d_out, "convert_u8_f") ? -1 : counted(launch_convert_u8_f(d_in, d_out, n, S(stream)));
}
int csdrb_convert_s16_f(const short* d_in, float* d_out, long n, void* stream)
{
    return null_io(d_in, d_out, "convert_s16_f") ? -1 : counted(launch_convert_s16_f(d_in, d_out, n, S(stream)));
}
int csdrb_convert_f_s16(const float* d_in, short* d_out, long n, void* stream)
{
    return null_io(d_in, d_out, "convert_f_s16") ? -1 : counted(launch_convert_f_s16(d_in, d_out, n, S(stream)));
}
// the other sample formats: byte buffers at any address, float buffers 4-byte aligned; a null pointer, a misaligned float buffer or n < 0 is
// refused before anything is launched
static inline bool bad_io(const void* in, const void* out, const float* floats, long n, const char* who)
{
    if (null_io(in, out, who)) return true;
    if (misaligned(floats, 4)) { set_error("%s: float buffer not 4-byte aligned", who); return true; }
    if (n >= 0) return false;
    set_error("%s: negative count %ld", who, n);
    return true;
}
int csdrb_convert_s8_f(const signed char* d_in, float* d_out, long n, void* stream)
{
    return bad_io(d_in, d_out, d_out, n, "convert_s8_f") ? -1 : counted(launch_convert_s8_f(reinterpret_cast<const unsigned char*>(d_in), d_out, n, S(stream)), n > 0);
}
int csdrb_convert_f_s8(const float* d_in, signed char* d_out, long n, void* stream)
{
    return bad_io(d_in, d_out, d_in, n, "convert_f_s8") ? -1 : counted(launch_convert_f_s8(d_in, reinterpret_cast<unsigned char*>(d_out), n, S(stream)), n > 0);
}
int csdrb_convert_f_u8(const float* d_in, unsigned char* d_out, long n, void* stream)
{
    return bad_io(d_in, d_out, d_in, n, "convert_f_u8") ? -1 : counted(launch_convert_f_u8(d_in, d_out, n, S(stream)), n > 0);
}
int csdrb_convert_s24_f(const unsigned char* d_in, float* d_out, long n, int bigendian, void* stream)
{
    return bad_io(d_in, d_out, d_out, n, "convert_s24_f") ? -1 : counted(launch_convert_s24_f(d_in, d_out, n, bigendian, S(stream)), n > 0);
}
int csdrb_convert_f_s24(const float* d_in, unsigned char* d_out, long n, int bigendian, void* stream)
{
    return bad_io(d_in, d_out, d_in, n, "convert_f_s24") ? -1 : counted(launch_convert_f_s24(d_in, d_out, n, bigendian, S(stream)), n > 0);
}

int csdrb_fir_bank_variants(void) { return fir_bank_variant_count(); }

int csdrb_fir_decimate_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels,
                               int input_size, int decimation, const float* h_taps, int taps_length, int variant, void* stream)
{
    if (too_many_channels(channels, "fir_decimate bank")) return -1;
    if (!d_in || !d_out || !h_taps) { set_error("fir_decimate bank: null pointer"); return -1; }
    // the generic kernel reads its taps from device memory: a stream-ordered allocation per call, so that two callers on different streams (or
    // devices) never share a buffer that one of them is still reading
    float* dt = nullptr;
    const bool fast = ((decimation == 10 && taps_length <= 200) || (decimation == 50 && taps_length <= 900)) && (in_stride % 2 == 0) &&
                      ((reinterpret_cast<uintptr_t>(d_in) & 15) == 0);
    if (!fast) {
        CSDRB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&dt), sizeof(float) * (size_t)taps_length, S(stream)));
        CSDRB_CUDA(cudaMemcpyAsync(dt, h_taps, sizeof(float) * (size_t)taps_length, cudaMemcpyHostToDevice, S(stream)));
        CSDRB_CUDA(cudaStreamSynchronize(S(stream)));       // h_taps is the caller's (possibly pageable) memory: it may change once we return
    }
    const int rc = counted(launch_fir_decimate_bank(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride,
                                                    channels, input_size, decimation, h_taps, dt, 0, taps_length, variant, S(stream)));
    if (dt) CSDRB_CUDA(cudaFreeAsync(dt, S(stream)));
    return rc;
}

// convert_u8_f | fir_decimate_cc in one launch for rtl_sdr-style input: d_in holds interleaved unsigned 8-bit I,Q (2 bytes per sample), in_stride counts
// SAMPLES between channel rows.  Fused for the compiled tilings (d=10 T<=200, d=50 T<=900) when rows start on 16-byte boundaries (in_stride % 8 == 0);
// any other geometry converts into a stream-ordered temporary and runs the cf32 bank.
int csdrb_fir_decimate_bank_u8_cc(const unsigned char* d_in, long in_stride, complexf* d_out, long out_stride, int channels,
                                  int input_size, int decimation, const float* h_taps, int taps_length, void* stream)
{
    if (too_many_channels(channels, "fir_decimate u8 bank")) return -1;
    if (!d_in || !d_out || !h_taps) { set_error("fir_decimate u8 bank: null pointer"); return -1; }
    int rc = launch_fir_decimate_bank_u8(d_in, in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, input_size, decimation, h_taps, taps_length, S(stream));
    if (rc != -2) return counted(rc);
    const long fstride = (input_size + 1) & ~1L;
    float* tmp = nullptr;
    CSDRB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&tmp), sizeof(float) * 2 * (size_t)fstride * channels, S(stream)));
    rc = launch_u8_rows_to_cf32(d_in, in_stride, reinterpret_cast<float2*>(tmp), fstride, channels, input_size, S(stream));
    if (rc < 0) { cudaFreeAsync(tmp, S(stream)); return rc; }
    g_launches += 1;
    rc = csdrb_fir_decimate_bank_cc(reinterpret_cast<const complexf*>(tmp), fstride, d_out, out_stride, channels, input_size, decimation, h_taps, taps_length, -1, stream);
    CSDRB_CUDA(cudaFreeAsync(tmp, S(stream)));
    return rc;
}

int csdrb_fmdemod_quadri_bank_cf(const complexf* d_in, long in_stride, float* d_out, long out_stride, int channels,
                                 int input_size, const complexf* d_last_in, complexf* d_last_out, void* stream)
{
    if (too_many_channels(channels, "fmdemod_quadri bank")) return -1;
    if (!d_in || !d_out) { set_error("fmdemod_quadri bank: null pointer"); return -1; }
    if (channels <= 0 || input_size <= 0) return 0;                  // nothing to do: no launch to count
    return counted(launch_fmdemod_quadri_bank(reinterpret_cast<const float2*>(d_in), in_stride, d_out, out_stride, channels, input_size,
                                              reinterpret_cast<const float2*>(d_last_in), reinterpret_cast<float2*>(d_last_out), S(stream)));
}


// ---- host-buffer bank call: the e2e path -------------------------------------------------------------
// Streams a [channels][input_size] HOST bank through the device in channel chunks on three streams so
// that the H2D copy of chunk i+1, the kernel of chunk i and the D2H copy of chunk i-1 overlap (PCIe is
// full duplex).  Host buffers should be page-locked (csdrb_host_alloc) -- pageable memory works but is
// staged by the driver.  Synchronous: returns when h_out is complete.
} // extern C (reopened below)
namespace csdrb {
struct HostBank {
    static constexpr int NS = 3;
    cudaStream_t st[NS] = {nullptr, nullptr, nullptr};
    void* din[NS] = {nullptr, nullptr, nullptr};
    void* dout[NS] = {nullptr, nullptr, nullptr};
    size_t cin = 0, cout = 0;
    std::mutex mu;
    int ensure(size_t bin, size_t bout)
    {
        for (int k = 0; k < NS; k++) if (!st[k]) CSDRB_CUDA(cudaStreamCreateWithFlags(&st[k], cudaStreamNonBlocking));
        if (bin > cin) {
            for (int k = 0; k < NS; k++) { if (din[k]) CSDRB_CUDA(cudaFree(din[k])); CSDRB_CUDA(cudaMalloc(&din[k], bin)); }
            cin = bin;
        }
        if (bout > cout) {
            for (int k = 0; k < NS; k++) { if (dout[k]) CSDRB_CUDA(cudaFree(dout[k])); CSDRB_CUDA(cudaMalloc(&dout[k], bout)); }
            cout = bout;
        }
        return 0;
    }
};

// Page-locked memory on the NUMA node the current device hangs off.  cudaHostAlloc places the pages where the calling thread runs; with one
// process per GPU on a two-socket host half the ranks would otherwise stream their H2D traffic across the socket interconnect.
// The thread is moved onto the device's node for the duration of the allocation (sysfs: the PCI device's numa_node and that node's cpulist), then gets its old affinity back.  Any failure along the way just leaves the default placement.
static bool cpus_of_device_node(cpu_set_t* set)
{
    int dev = 0; char bus[32] = "";
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetPCIBusId(bus, sizeof bus, dev) != cudaSuccess) return false;
    for (char* p = bus; *p; p++) if (*p >= 'A' && *p <= 'Z') *p = (char)(*p - 'A' + 'a');
    char path[128]; snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r"); if (!f) return false;
    int node = -1; const int got = fscanf(f, "%d", &node); fclose(f);
    if (got != 1 || node < 0) return false;
    snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
    f = fopen(path, "r"); if (!f) return false;
    char list[4096] = ""; const bool ok = fgets(list, sizeof list, f) != nullptr; fclose(f);
    if (!ok) return false;
    CPU_ZERO(set);
    int n = 0;
    for (char* p = list; *p && *p != '\n';) {                         // "0-31,64-95"
        char* e; long a = strtol(p, &e, 10); if (e == p) break; long b = a;
        if (*e == '-') { p = e + 1; b = strtol(p, &e, 10); }
        for (long c = a; c <= b && c < CPU_SETSIZE; c++) { CPU_SET((int)c, set); n++; }
        p = (*e == ',') ? e + 1 : e;
    }
    return n > 0;
}
}  // namespace csdrb
extern "C" {

void* csdrb_host_alloc(size_t bytes)
{
    cpu_set_t old_set, node_set;
    const bool have_old = sched_getaffinity(0, sizeof old_set, &old_set) == 0;
    const bool moved = have_old && !(getenv("CSDRB_NO_NUMA") && getenv("CSDRB_NO_NUMA")[0] == '1') && cpus_of_device_node(&node_set) &&
                       sched_setaffinity(0, sizeof node_set, &node_set) == 0;
    void* p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault);
    if (e == cudaSuccess && moved) memset(p, 0, bytes ? bytes : 1);  // first touch from the node, in case the driver only reserved the range
    if (moved) sched_setaffinity(0, sizeof old_set, &old_set);
    if (e != cudaSuccess) { cuda_fail(e, "cudaHostAlloc", __FILE__, __LINE__); return nullptr; }
    return p;
}
void csdrb_host_free(void* p) { if (p) cudaFreeHost(p); }

// in_bytes = bytes per input sample: 8 (cf32) or 2 (u8 IQ, converted inside the FIR kernel)
static int fir_bank_host(const void* h_in, int in_bytes, long in_stride, complexf* h_out, long out_stride, int channels,
                         int input_size, int decimation, const float* h_taps, int taps_length, int chunk_channels)
{
    if (!h_in || !h_out || !h_taps || channels <= 0 || decimation <= 0 || taps_length <= 0) { set_error("fir_decimate host bank: bad argument"); return -1; }
    const int n_out = input_size >= taps_length ? (input_size - taps_length) / decimation + 1 : 0;
    if (n_out == 0) return 0;
    HostBank& hb = per_device<HostBank>();
    std::lock_guard<std::mutex> lk(hb.mu);
    const long dstride_in = in_bytes == 2 ? (input_size + 7) & ~7L : (input_size + 1) & ~1L, dstride_out = (n_out + 1) & ~1L;
    if (chunk_channels <= 0) {                                 // ~192 MiB of cf32 input (48 MiB of u8) per chunk keeps all three stages busy
        chunk_channels = (int)((192L << 20) / (dstride_in * 8));
        if (chunk_channels < 1) chunk_channels = 1;
    }
    if (chunk_channels > channels) chunk_channels = channels;
    if (int rc = hb.ensure((size_t)chunk_channels * dstride_in * in_bytes, (size_t)chunk_channels * dstride_out * 8)) return rc;
    int slot = 0;
    for (int c0 = 0; c0 < channels; c0 += chunk_channels, slot = (slot + 1) % HostBank::NS) {
        const int nc = channels - c0 < chunk_channels ? channels - c0 : chunk_channels;
        cudaStream_t s = hb.st[slot];
        CSDRB_CUDA(cudaMemcpy2DAsync(hb.din[slot], (size_t)dstride_in * in_bytes, static_cast<const char*>(h_in) + (long)c0 * in_stride * in_bytes,
                                     (size_t)in_stride * in_bytes, (size_t)input_size * in_bytes, nc, cudaMemcpyHostToDevice, s));
        int rc = in_bytes == 2
            ? csdrb_fir_decimate_bank_u8_cc((const unsigned char*)hb.din[slot], dstride_in, (complexf*)hb.dout[slot], dstride_out, nc, input_size, decimation, h_taps, taps_length, s)
            : csdrb_fir_decimate_bank_cc((const complexf*)hb.din[slot], dstride_in, (complexf*)hb.dout[slot], dstride_out, nc, input_size, decimation, h_taps, taps_length, -1, s);
        if (rc < 0) return rc;
        CSDRB_CUDA(cudaMemcpy2DAsync(h_out + (long)c0 * out_stride, (size_t)out_stride * 8, hb.dout[slot], (size_t)dstride_out * 8,
                                     (size_t)n_out * 8, nc, cudaMemcpyDeviceToHost, s));
    }
    for (int k = 0; k < HostBank::NS; k++) CSDRB_CUDA(cudaStreamSynchronize(hb.st[k]));
    return n_out;
}

int csdrb_fir_decimate_bank_cc_host(const complexf* h_in, long in_stride, complexf* h_out, long out_stride, int channels,
                                    int input_size, int decimation, const float* h_taps, int taps_length, int chunk_channels)
{
    return fir_bank_host(h_in, 8, in_stride, h_out, out_stride, channels, input_size, decimation, h_taps, taps_length, chunk_channels);
}

// the same with rtl_sdr-style u8 IQ on the host side (2 bytes per sample over PCIe instead of 8): convert_u8_f | fir_decimate_cc, csdr-fm:41
int csdrb_fir_decimate_bank_u8_host(const unsigned char* h_in, long in_stride, complexf* h_out, long out_stride, int channels,
                                    int input_size, int decimation, const float* h_taps, int taps_length, int chunk_channels)
{
    return fir_bank_host(h_in, 2, in_stride, h_out, out_stride, channels, input_size, decimation, h_taps, taps_length, chunk_channels);
}

// =====================================================================================================
// Part B, continued: K2, K5-K9
// =====================================================================================================
size_t csdrb_shift_addition_bank_scratch_bytes(int channels, int input_size, int chunk) { return shift_bank_scratch_bytes(channels, input_size, chunk); }

int csdrb_shift_addition_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int input_size,
                                 const shift_addition_data_t* d_params, float* d_phase_io, int chunk, void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (too_many_channels(channels, "shift_addition bank")) return -1;
    if (!d_in || !d_out || !d_params || !d_phase_io) { set_error("shift_addition bank: null pointer"); return -1; }
    int rc = launch_shift_addition_bank(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, input_size,
                                        reinterpret_cast<const float*>(d_params), d_phase_io, chunk, d_scratch, scratch_bytes, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_shift_addition_bank_fc(const float* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int input_size,
                                 const shift_addition_data_t* d_params, float* d_phase_io, int chunk, void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (too_many_channels(channels, "shift_addition_fc bank")) return -1;
    if (!d_in || !d_out || !d_params || !d_phase_io) { set_error("shift_addition_fc bank: null pointer"); return -1; }
    int rc = launch_shift_addition_bank_fc(d_in, in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, input_size,
                                           reinterpret_cast<const float*>(d_params), d_phase_io, chunk, d_scratch, scratch_bytes, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

size_t csdrb_shift_math_bank_scratch_bytes(int channels, int input_size) { return shift_math_scratch_bytes(channels, input_size); }

int csdrb_shift_math_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int input_size,
                             const float* d_rates, float* d_phase_io, void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (too_many_channels(channels, "shift_math bank")) return -1;
    if (!d_in || !d_out || !d_rates || !d_phase_io) { set_error("shift_math bank: null pointer"); return -1; }
    int rc = launch_shift_math_bank(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, input_size,
                                    d_rates, d_phase_io, d_scratch, scratch_bytes, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_shift_table_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int input_size,
                              const float* d_rates, float* d_phase_io, const float* d_table, int table_size, void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (too_many_channels(channels, "shift_table bank")) return -1;
    if (!d_in || !d_out || !d_rates || !d_phase_io || !d_table) { set_error("shift_table bank: null pointer"); return -1; }
    int rc = launch_shift_table_bank(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, input_size,
                                     d_rates, d_phase_io, d_table, table_size, d_scratch, scratch_bytes, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_shift_addfast_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int input_size,
                                const shift_addfast_data_t* d_params, float* d_phase_io, int chunk, void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (too_many_channels(channels, "shift_addfast bank")) return -1;
    if (!d_in || !d_out || !d_params || !d_phase_io) { set_error("shift_addfast bank: null pointer"); return -1; }
    int rc = launch_shift_addfast_bank(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, input_size,
                                       reinterpret_cast<const float*>(d_params), d_phase_io, chunk, d_scratch, scratch_bytes, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_decimating_shift_addition_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int input_size,
                                            const shift_addition_data_t* d_params, int decimation, int* d_remain_io, float* d_phase_io, int* d_out_size, void* stream)
{
    if (!d_in || !d_out || !d_params || !d_remain_io || !d_phase_io) { set_error("decimating_shift_addition bank: null pointer"); return -1; }
    int rc = launch_decimating_shift_bank(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, input_size,
                                          reinterpret_cast<const float*>(d_params), decimation, d_remain_io, d_phase_io, d_out_size, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

size_t csdrb_fractional_decimator_bank_scratch_bytes(int channels, int input_size, float rate) { return fracdec_scratch_bytes(channels, input_size, rate); }

int csdrb_fractional_decimator_bank_ff(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int input_size, float rate,
                                       int num_poly_points, const float* d_taps, int taps_length, csdrb_fracdec_state_t* d_state,
                                       void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (too_many_channels(channels, "fractional_decimator bank")) return -1;
    if (!d_in || !d_out || !d_state) { set_error("fractional_decimator bank: null pointer"); return -1; }
    int rc = launch_fractional_decimator_bank(d_in, in_stride, d_out, out_stride, channels, input_size, rate, num_poly_points, d_taps, taps_length, d_state,
                                              d_scratch, scratch_bytes, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_rational_resampler_bank_ff(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int input_size, int interpolation,
                                     int decimation, const float* h_taps, int taps_length, int last_taps_delay, rational_resampler_ff_t* h_state_out,
                                     void* stream)
{
    if (too_many_channels(channels, "rational_resampler bank")) return -1;
    if (!h_state_out) { set_error("rational_resampler bank: null state pointer"); return -1; }
    static_assert(sizeof(rational_resampler_ff_t) == 3 * sizeof(int), "state layout");
    int rc = launch_rational_resampler_bank(d_in, in_stride, d_out, out_stride, channels, input_size, interpolation, decimation, h_taps, taps_length,
                                            last_taps_delay, reinterpret_cast<int*>(h_state_out), S(stream));
    if (rc > 0 && channels > 0) counted(0, 1);
    return rc;
}

size_t csdrb_fastagc_bank_scratch_bytes(int channels, int nblocks) { return fastagc_scratch_bytes(channels, nblocks); }

int csdrb_fastagc_bank_ff(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int block, int nblocks, float reference,
                          csdrb_fastagc_state_t* d_state, float* d_hist, void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (too_many_channels(channels, "fastagc bank")) return -1;
    if (!d_in || !d_out || !d_state || !d_hist) { set_error("fastagc bank: null pointer"); return -1; }
    int rc = launch_fastagc_bank(d_in, in_stride, d_out, out_stride, channels, block, nblocks, reference, d_state, d_hist, d_scratch, scratch_bytes, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

// fastagc_ff | convert_f_s16 fused (the last two blocks of the NFM graph, README.md:87), at every block size
int csdrb_fastagc_bank_f_s16(const float* d_in, long in_stride, short* d_out, long out_stride, int channels, int block, int nblocks, float reference,
                             csdrb_fastagc_state_t* d_state, float* d_hist, void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (too_many_channels(channels, "fastagc bank")) return -1;
    if (!d_in || !d_out || !d_state || !d_hist) { set_error("fastagc s16 bank: null pointer"); return -1; }
    int rc = launch_fastagc_bank_s16_any(d_in, in_stride, d_out, out_stride, channels, block, nblocks, reference, d_state, d_hist, d_scratch, scratch_bytes,
                                         S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

// amdemod_cf (libcsdr.c:861-873) over n samples
int csdrb_amdemod_cf(const complexf* d_in, float* d_out, long n, void* stream)
{
    if (!d_in || !d_out) { set_error("amdemod_cf: null pointer"); return -1; }
    int rc = launch_amdemod_cf(reinterpret_cast<const float2*>(d_in), d_out, n, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

// [amdemod_cf |] fastdcblock_ff over whole blocks (libcsdr.c:861-873, 920-941; csdr.c:952-968)
int csdrb_fastdcblock_bank_ff(const void* d_in, long in_stride, int cf32_in, float* d_out, long out_stride, int channels, int block, int nblocks,
                              float* d_last_dc_io, void* stream)
{
    if (too_many_channels(channels, "fastdcblock bank")) return -1;
    if (!d_in || !d_out || !d_last_dc_io) { set_error("fastdcblock bank: null pointer"); return -1; }
    int rc = launch_fastdcblock_bank(d_in, in_stride, cf32_in, d_out, out_stride, channels, block, nblocks, d_last_dc_io, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

// [realpart_cf |] agc_ff [| limit_ff] [| convert_f_s16] (csdr.c:634-645, 1337-1373; libcsdr_gpl.c:163-260; libcsdr.c:1130-1137, 2390-2398)
int csdrb_agc_bank_ff(const void* d_in, long in_stride, int cf32_in, void* d_out, long out_stride, int s16_out, int channels, int n,
                      const csdrb_agc_params_t* params, csdrb_agc_state_t* d_state, float limit_max, void* stream)
{
    static_assert(sizeof(csdrb_agc_params_t) == sizeof(AgcParams) && sizeof(csdrb_agc_state_t) == sizeof(AgcState), "AGC structs mirror kernels.h");
    if (too_many_channels(channels, "agc bank")) return -1;
    if (!d_in || !d_out || !params || !d_state) { set_error("agc bank: null pointer"); return -1; }
    AgcParams p;
    memcpy(&p, params, sizeof p);
    p.hang_time = (short)p.hang_time;                                   // the reference's parameters are `short` (libcsdr_gpl.h:37)
    p.attack_wait_time = (short)p.attack_wait_time;
    int rc = launch_agc_bank(d_in, in_stride, cf32_in, d_out, out_stride, s16_out, channels, n, &p, d_state, limit_max, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

// BPSK31 receive chain (psk31.cu; libcsdr.c:2201-2217, 1977-2072, 2319-2333, 1536-1549)
int csdrb_simple_agc_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int input_size, float rate,
                             float reference, float max_gain, float* d_gain_io, void* stream)
{
    if (too_many_channels(channels, "simple_agc bank")) return -1;
    if (!d_in || !d_out || !d_gain_io) { set_error("simple_agc bank: null pointer"); return -1; }
    int rc = launch_simple_agc_bank(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, input_size,
                                    rate, reference, max_gain, d_gain_io, S(stream));
    return rc < 0 ? rc : counted(input_size > 0 ? input_size : 0, rc);
}

int csdrb_timing_recovery_bank_cc(const complexf* d_in, long in_stride, const int* d_start, const int* d_size, int max_size, complexf* d_out,
                                  long out_stride, float* d_error, int* d_indexes, int channels, const csdrb_timing_recovery_params_t* params,
                                  csdrb_timing_recovery_state_t* d_state, void* stream)
{
    static_assert(sizeof(csdrb_timing_recovery_params_t) == sizeof(TrParams) && sizeof(csdrb_timing_recovery_state_t) == sizeof(TrState),
                  "timing recovery structs mirror kernels.h");
    if (too_many_channels(channels, "timing_recovery bank")) return -1;
    if (!d_in || !d_start || !d_size || !d_out || !params || !d_state) { set_error("timing_recovery bank: null pointer"); return -1; }
    int rc = launch_timing_recovery_bank(reinterpret_cast<const float2*>(d_in), in_stride, d_start, d_size, reinterpret_cast<float2*>(d_out), out_stride,
                                         d_error, d_indexes, channels, params, d_state, max_size, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_dbpsk_decoder_bank_c_u8(const complexf* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int input_size,
                                  const int* d_lengths, const complexf* d_last_in, complexf* d_last_out, void* stream)
{
    if (null_io(d_in, d_out, "dbpsk bank")) return -1;
    int rc = launch_dbpsk_bank(reinterpret_cast<const float2*>(d_in), in_stride, d_out, out_stride, channels, input_size, d_lengths,
                               reinterpret_cast<const float2*>(d_last_in), reinterpret_cast<float2*>(d_last_out), S(stream));
    return rc < 0 ? rc : counted(input_size > 0 ? input_size : 0, rc);
}

int csdrb_psk31_varicode_decoder_bank_u8_u8(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels,
                                            int input_size, const int* d_lengths, unsigned long long* d_hist_io, int* d_count, void* stream)
{
    if (null_io(d_in, d_out, "varicode bank")) return -1;
    if (!d_hist_io || !d_count) { set_error("varicode bank: null pointer"); return -1; }
    int rc = launch_varicode_bank(d_in, in_stride, d_out, out_stride, channels, input_size, d_lengths, d_hist_io, d_count, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

// BPSK31 transmit chain (psk31_tx.cu; libcsdr.c:1551-1575, 1828-1843, 1772-1782, 1793-1808)
int csdrb_psk31_varicode_encoder_bank_u8_u8(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels,
                                            int input_size, const int* d_lengths, int output_max_size, int* d_input_processed, int* d_output_size,
                                            void* stream)
{
    if (null_io(d_in, d_out, "varicode encoder bank")) return -1;
    if (!d_input_processed || !d_output_size) { set_error("varicode encoder bank: null pointer"); return -1; }
    int rc = launch_varicode_encoder_bank(d_in, in_stride, d_out, out_stride, channels, input_size, d_lengths, output_max_size, d_input_processed,
                                          d_output_size, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_differential_codec_bank_u8_u8(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels,
                                        int input_size, const int* d_lengths, int encode, unsigned char* d_state_io, void* stream)
{
    if (null_io(d_in, d_out, "differential codec bank")) return -1;
    if (!d_state_io) { set_error("differential codec bank: null pointer"); return -1; }
    int rc = launch_differential_codec_bank(d_in, in_stride, d_out, out_stride, channels, input_size, d_lengths, encode, d_state_io, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_psk_modulator_bank_u8_c(const unsigned char* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int input_size,
                                  const int* d_lengths, int n_psk, void* stream)
{
    if (too_many_channels(channels, "psk modulator bank")) return -1;
    if (!d_in || !d_out || misaligned(d_out, 8)) { set_error("psk modulator bank: null or misaligned pointer (complexf needs 8-byte alignment)"); return -1; }
    int rc = launch_psk_modulator_bank(d_in, in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, input_size, d_lengths, n_psk, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_psk31_interpolate_sine_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int input_size,
                                         const int* d_lengths, int interpolation, complexf* d_last_io, void* stream)
{
    if (too_many_channels(channels, "psk31_interpolate_sine bank")) return -1;
    if (!d_in || !d_out || !d_last_io || misaligned(d_in, 8) || misaligned(d_out, 8) || misaligned(d_last_io, 8)) {
        set_error("psk31_interpolate_sine bank: null or misaligned pointer (complexf needs 8-byte alignment)");
        return -1;
    }
    int rc = launch_psk31_interpolate_sine_bank(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels,
                                                input_size, d_lengths, interpolation, reinterpret_cast<float2*>(d_last_io), S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

// RTTY receive chain (rtty.cu; libcsdr.c:1662-1729, 1608-1616)
int csdrb_serial_line_decoder_bank_f_u8(const float* d_in, long in_stride, int end, int* d_start_io, unsigned char* d_out, long out_stride, int* d_count,
                                        int* d_stuck, int channels, const csdrb_serial_line_params_t* params, int bufsize, void* stream)
{
    static_assert(sizeof(csdrb_serial_line_params_t) == sizeof(SerialLineParams), "serial line params mirror kernels.h");
    if (too_many_channels(channels, "serial_line bank")) return -1;
    if (!d_in || !d_start_io || !d_out || !d_count || !d_stuck || !params) { set_error("serial_line bank: null pointer"); return -1; }
    int rc = launch_serial_line_bank(d_in, in_stride, end, d_start_io, d_out, out_stride, d_count, d_stuck, channels, params, bufsize, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_rtty_baudot2ascii_bank_u8_u8(const unsigned char* d_in, long in_stride, unsigned char* d_out, long out_stride, int channels, int input_size,
                                       const int* d_lengths, unsigned char* d_fig_mode_io, int* d_count, void* stream)
{
    if (null_io(d_in, d_out, "baudot bank")) return -1;
    if (!d_fig_mode_io || !d_count) { set_error("baudot bank: null pointer"); return -1; }
    int rc = launch_baudot_bank(d_in, in_stride, d_out, out_stride, channels, input_size, d_lengths, d_fig_mode_io, d_count, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

// tone filters (tone.cu; libcsdr.c:2261-2273, 2335-2351)

int csdrb_apply_fir_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int n, const complexf* d_taps,
                            int taps_length, void* stream)
{
    if (too_many_channels(channels, "apply_fir_cc bank")) return -1;
    if (!d_in || !d_out || !d_taps || misaligned(d_in, 8) || misaligned(d_out, 8) || misaligned(d_taps, 8)) {
        set_error("apply_fir_cc bank: null or misaligned pointer (complexf needs 8-byte alignment)");
        return -1;
    }
    int rc = launch_apply_fir_bank_cc(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, n,
                                      reinterpret_cast<const float2*>(d_taps), taps_length, S(stream));
    return rc < 0 ? rc : counted(rc, channels > 0 ? 1 : 0);
}

int csdrb_bfsk_demod_bank_cf(const complexf* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, const complexf* d_mark,
                             const complexf* d_space, int taps_length, void* stream)
{
    if (too_many_channels(channels, "bfsk_demod_cf bank")) return -1;
    if (!d_in || !d_out || !d_mark || !d_space || misaligned(d_in, 8) || misaligned(d_out, 4) || misaligned(d_mark, 8) || misaligned(d_space, 8)) {
        set_error("bfsk_demod_cf bank: null or misaligned pointer (complexf needs 8-byte, float 4-byte alignment)");
        return -1;
    }
    int rc = launch_bfsk_demod_bank_cf(reinterpret_cast<const float2*>(d_in), in_stride, d_out, out_stride, channels, n,
                                       reinterpret_cast<const float2*>(d_mark), reinterpret_cast<const float2*>(d_space), taps_length, S(stream));
    return rc < 0 ? rc : counted(rc, channels > 0 ? 1 : 0);
}

// transmit banks (interpolate.cu; libcsdr.c:579-602, 1180-1192)
int csdrb_fir_interpolate_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int n, int interpolation,
                                  const float* d_taps, int taps_length, void* stream)
{
    if (too_many_channels(channels, "fir_interpolate bank")) return -1;
    if (!d_in || !d_out || !d_taps || misaligned(d_in, 8) || misaligned(d_out, 8) || misaligned(d_taps, 4)) {
        set_error("fir_interpolate bank: null or misaligned pointer (complexf needs 8-byte, float 4-byte alignment)");
        return -1;
    }
    int rc = launch_fir_interpolate_bank_cc(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, n,
                                            interpolation, d_taps, taps_length, S(stream));
    return rc < 0 ? rc : counted(rc, channels > 0 && rc > 0 ? 1 : 0);
}

int csdrb_fmmod_bank_fc(const float* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int n, float* d_phase_io, void* stream)
{
    if (too_many_channels(channels, "fmmod bank")) return -1;
    if (!d_in || !d_out || !d_phase_io || misaligned(d_in, 4) || misaligned(d_out, 8) || misaligned(d_phase_io, 4)) {
        set_error("fmmod bank: null or misaligned pointer (complexf needs 8-byte, float 4-byte alignment)");
        return -1;
    }
    int rc = launch_fmmod_bank_fc(d_in, in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, n, d_phase_io, S(stream));
    return rc < 0 ? rc : counted(rc, channels > 0 && n > 0 ? 1 : 0);
}

// amplitude modulator banks (modulate.cu; libcsdr.c:1139-1142, 1174-1178, 1194-1208, csdr.c:2084-2102): the launcher returns its launches
int csdrb_gain_bank_ff(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int n, float gain, void* stream)
{
    const int rc = launch_gain_bank_ff(d_in, in_stride, d_out, out_stride, channels, n, gain, S(stream));
    return rc < 0 ? rc : counted(n, rc);
}

int csdrb_dsb_bank_fc(const float* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int n, float q_value, void* stream)
{
    const int rc = launch_dsb_bank_fc(d_in, in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, n, q_value, S(stream));
    return rc < 0 ? rc : counted(n, rc);
}

int csdrb_add_dcoffset_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int n, void* stream)
{
    const int rc = launch_add_dcoffset_bank_cc(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels,
                                               n, S(stream));
    return rc < 0 ? rc : counted(n, rc);
}

int csdrb_fixed_amplitude_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int n, float new_amplitude,
                                  void* stream)
{
    const int rc = launch_fixed_amplitude_bank_cc(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride,
                                                  channels, n, new_amplitude, S(stream));
    return rc < 0 ? rc : counted(n, rc);
}

// synthesis bank (synth.cu): fir_interpolate_cc | shift_addition_cc per channel, summed over the channels in a fixed pairwise tree
size_t csdrb_synth_bank_scratch_bytes(int channels, int input_size, int interpolation, int taps_length, int chunk, int offset)
{
    return synth_bank_scratch_bytes(channels, input_size, interpolation, taps_length, chunk, offset);
}

int csdrb_synth_bank_cc(const complexf* d_in, long in_stride, int channels, int input_size, int interpolation, const float* d_taps, int taps_length,
                        const shift_addition_data_t* d_params, float* d_phase_io, int chunk, int offset, complexf* d_out, void* d_scratch,
                        size_t scratch_bytes, void* stream)
{
    if (!d_in || !d_taps || !d_params || !d_phase_io || !d_out || misaligned(d_in, 8) || misaligned(d_out, 8) || misaligned(d_taps, 4) ||
        misaligned(d_params, 4) || misaligned(d_phase_io, 4)) {
        set_error("synth bank: null or misaligned pointer (complexf needs 8-byte, float 4-byte alignment)");
        return -1;
    }
    int launches = 0;
    int rc = launch_synth_bank(reinterpret_cast<const float2*>(d_in), in_stride, channels, input_size, interpolation, d_taps, taps_length,
                               reinterpret_cast<const float*>(d_params), d_phase_io, chunk, offset, reinterpret_cast<float2*>(d_out), d_scratch,
                               scratch_bytes, &launches, S(stream));
    return rc < 0 ? rc : counted(rc, launches);
}

// streaming synthesis bank: the state of csdrb_synth_bank_cc between blocks (phases, offset inside the NCO chunk) and its buffers
struct csdrb_synth_bank_s {
    int channels = 0, interpolation = 0, taps_length = 0, chunk = 0, offset = 0;
    float* d_params = nullptr;                        // shift_addition_data_t per channel
    float* d_taps = nullptr;
    float* d_phase = nullptr;                         // phase at the start of the chunk holding the next block's first output
    void* d_scratch = nullptr;
    size_t scratch_cap = 0;
};

csdrb_synth_bank_t* csdrb_synth_bank_create(int channels, const float* h_rates, int interpolation, const float* h_taps, int taps_length, int chunk)
{
    if (channels < 1 || !h_rates || !h_taps || interpolation < 1 || taps_length < 1 || chunk < 1) {
        set_error("synth bank create: needs channels >= 1, rates, taps, interpolation >= 1, taps_length >= 1 and chunk >= 1");
        return nullptr;
    }
    auto* b = new csdrb_synth_bank_s();
    b->channels = channels; b->interpolation = interpolation; b->taps_length = taps_length; b->chunk = chunk;
    std::vector<shift_addition_data_t> params((size_t)channels);
    for (int c = 0; c < channels; c++) params[(size_t)c] = shift_addition_init(h_rates[c]);
    bool ok = cudaMalloc(&b->d_params, sizeof(shift_addition_data_t) * (size_t)channels) == cudaSuccess;
    ok = ok && cudaMalloc(&b->d_taps, sizeof(float) * (size_t)taps_length) == cudaSuccess;
    ok = ok && cudaMalloc(&b->d_phase, sizeof(float) * (size_t)channels) == cudaSuccess;
    ok = ok && cudaMemcpy(b->d_params, params.data(), sizeof(shift_addition_data_t) * (size_t)channels, cudaMemcpyHostToDevice) == cudaSuccess;
    ok = ok && cudaMemcpy(b->d_taps, h_taps, sizeof(float) * (size_t)taps_length, cudaMemcpyHostToDevice) == cudaSuccess;
    ok = ok && cudaMemset(b->d_phase, 0, sizeof(float) * (size_t)channels) == cudaSuccess;
    if (!ok) { set_error("synth bank create: CUDA allocation failed (%s)", cudaGetErrorString(cudaGetLastError())); csdrb_synth_bank_destroy(b); return nullptr; }
    return b;
}

void csdrb_synth_bank_destroy(csdrb_synth_bank_t* b)
{
    if (!b) return;
    cudaFree(b->d_params); cudaFree(b->d_taps); cudaFree(b->d_phase); cudaFree(b->d_scratch);
    delete b;
}

int csdrb_synth_bank_process(csdrb_synth_bank_t* b, const complexf* d_in, long in_stride, int input_size, complexf* d_out, void* stream)
{
    if (!b) { set_error("synth bank process: null bank"); return -1; }
    const size_t need = synth_bank_scratch_bytes(b->channels, input_size, b->interpolation, b->taps_length, b->chunk, b->offset);
    if (need > b->scratch_cap) {                      // grow: the previous block may still read the old buffer
        CSDRB_CUDA(cudaStreamSynchronize(S(stream)));
        if (b->d_scratch) CSDRB_CUDA(cudaFree(b->d_scratch));
        b->d_scratch = nullptr; b->scratch_cap = 0;
        CSDRB_CUDA(cudaMalloc(&b->d_scratch, need));
        b->scratch_cap = need;
    }
    const int rc = csdrb_synth_bank_cc(d_in, in_stride, b->channels, input_size, b->interpolation, b->d_taps, b->taps_length,
                                       reinterpret_cast<const shift_addition_data_t*>(b->d_params), b->d_phase, b->chunk, b->offset, d_out,
                                       b->d_scratch, b->scratch_cap, stream);
    if (rc > 0) b->offset = (int)(((long)b->offset + rc) % b->chunk);
    return rc;
}

int csdrb_fft_c2c_batch(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int size, int batch, int inverse, void* stream)
{
    if (!d_in || !d_out) { set_error("fft: null pointer"); return -1; }
    int rc = launch_fft_c2c_batch(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, size, batch, inverse, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_fft_c2c_large_batch(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int size, int batch, int inverse, void* stream)
{
    if (!d_in || !d_out) { set_error("fft (large): null pointer"); return -1; }
    int rc = launch_fft_c2c_large_batch(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, size, batch, inverse, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_fft_r2c_batch(const float* d_in, long in_stride, complexf* d_out, long out_stride, int size, int batch, void* stream)
{
    if (!d_in || !d_out) { set_error("fft r2c: null pointer"); return -1; }
    int rc = launch_fft_r2c_batch(d_in, in_stride, reinterpret_cast<float2*>(d_out), out_stride, size, batch, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_bandpass_fir_fft_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int fft_size, int input_size,
                                   int nblocks, const complexf* d_taps_fft, long taps_stride, complexf* d_tail_io, void* stream)
{
    if (too_many_channels(channels, "bandpass_fir_fft bank")) return -1;
    if (!d_in || !d_out || !d_taps_fft || !d_tail_io) { set_error("bandpass_fir_fft bank: null pointer"); return -1; }
    int rc = launch_olafir_bank(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, fft_size, input_size,
                                nblocks, reinterpret_cast<const float2*>(d_taps_fft), taps_stride, reinterpret_cast<float2*>(d_tail_io), 0, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_fastddc_fwd_cc(const complexf* d_in, complexf* d_spectra, complexf* d_overlap_io, int fft_size, int input_size, int nblocks, void* stream)
{
    if (!d_in || !d_spectra || !d_overlap_io) { set_error("fastddc_fwd: null pointer"); return -1; }
    int rc = launch_fastddc_fwd(reinterpret_cast<const float2*>(d_in), reinterpret_cast<float2*>(d_spectra), reinterpret_cast<float2*>(d_overlap_io),
                                fft_size, input_size, nblocks, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

size_t csdrb_fastddc_inv_bank_scratch_bytes(int channels, int nblocks) { return fastddc_inv_scratch_bytes(channels, nblocks); }

int csdrb_fastddc_inv_bank_cc(const complexf* d_spectra, int nblocks, const complexf* d_taps_fft, const csdrb_fastddc_chan_t* d_chan, int channels,
                              const fastddc_t* g, int* d_remain_io, float* d_phase_io, complexf* d_out, long out_stride, int* d_out_total,
                              void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (too_many_channels(channels, "fastddc_inv bank")) return -1;
    if (!d_spectra || !d_taps_fft || !d_chan || !g || !d_remain_io || !d_phase_io || !d_out || !d_out_total) { set_error("fastddc_inv bank: null pointer"); return -1; }
    int rc = launch_fastddc_inv_bank(reinterpret_cast<const float2*>(d_spectra), nblocks, reinterpret_cast<const float2*>(d_taps_fft), d_chan, channels,
                                     g->fft_size, g->fft_inv_size, g->pre_decimation, g->scrap, g->post_input_size, g->post_decimation,
                                     d_remain_io, d_phase_io, reinterpret_cast<float2*>(d_out), out_stride, d_out_total, d_scratch, scratch_bytes, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

struct csdrb_fastddc_inv_plan { void* impl; };

csdrb_fastddc_inv_plan_t* csdrb_fastddc_inv_plan_create(const csdrb_fastddc_chan_t* chan, int channels, const fastddc_t* g, int nblocks)
{
    if (too_many_channels(channels, "fastddc_inv plan")) return nullptr;
    if (!chan || !g) { set_error("fastddc_inv_plan_create: null pointer"); return nullptr; }
    void* impl = nullptr;
    if (fastddc_inv_plan_create(&impl, chan, channels, nblocks, g->fft_size, g->fft_inv_size, g->pre_decimation, g->scrap, g->post_input_size, g->post_decimation) < 0) return nullptr;
    auto* p = new csdrb_fastddc_inv_plan_t{impl};
    return p;
}

int csdrb_fastddc_inv_plan_run(csdrb_fastddc_inv_plan_t* plan, const complexf* d_spectra, const complexf* d_taps_fft, complexf* d_out, long out_stride,
                               int* d_out_total, void* stream)
{
    if (!plan) { set_error("fastddc_inv_plan_run: null plan"); return -1; }
    int rc = fastddc_inv_plan_run(plan->impl, reinterpret_cast<const float2*>(d_spectra), reinterpret_cast<const float2*>(d_taps_fft), reinterpret_cast<float2*>(d_out),
                                  out_stride, d_out_total, S(stream));
    return rc < 0 ? rc : counted(rc, 4);
}

int csdrb_fastddc_inv_plan_set_channel(csdrb_fastddc_inv_plan_t* plan, int channel, const csdrb_fastddc_chan_t* chan)
{
    if (!plan) { set_error("fastddc_inv_plan_set_channel: null plan"); return -1; }
    return fastddc_inv_plan_set_channel(plan->impl, channel, chan);
}

int csdrb_fastddc_inv_plan_get_state(csdrb_fastddc_inv_plan_t* plan, int* remain, float* phase)
{
    if (!plan) { set_error("fastddc_inv_plan_get_state: null plan"); return -1; }
    return fastddc_inv_plan_get_state(plan->impl, remain, phase);
}

int csdrb_fastddc_inv_plan_set_state(csdrb_fastddc_inv_plan_t* plan, const int* remain, const float* phase)
{
    if (!plan) { set_error("fastddc_inv_plan_set_state: null plan"); return -1; }
    return fastddc_inv_plan_set_state(plan->impl, remain, phase);
}

void csdrb_fastddc_inv_plan_destroy(csdrb_fastddc_inv_plan_t* plan)
{
    if (!plan) return;
    fastddc_inv_plan_destroy(plan->impl);
    delete plan;
}

int csdrb_apply_window_rows_c(const complexf* d_in, complexf* d_out, const float* d_window, int size, long rows, void* stream)
{
    if (!d_in || !d_out || !d_window) { set_error("apply_window: null pointer"); return -1; }
    int rc = launch_apply_window_rows(reinterpret_cast<const float2*>(d_in), reinterpret_cast<float2*>(d_out), d_window, size, rows, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}
int csdrb_logpower_cf(const complexf* d_in, float* d_out, long n, float add_db, void* stream)
{
    if (!d_in || !d_out) { set_error("logpower_cf: null pointer"); return -1; }
    int rc = launch_power(reinterpret_cast<const float2*>(d_in), nullptr, d_out, n, add_db, 0, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}
int csdrb_accumulate_power_cf(const complexf* d_in, float* d_acc, long n, void* stream)
{
    if (!d_in || !d_acc) { set_error("accumulate_power_cf: null pointer"); return -1; }
    int rc = launch_power(reinterpret_cast<const float2*>(d_in), nullptr, d_acc, n, 0.f, 1, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}
int csdrb_log_ff(const float* d_in, float* d_out, long n, float add_db, void* stream)
{
    if (!d_in || !d_out) { set_error("log_ff: null pointer"); return -1; }
    int rc = launch_power(nullptr, d_in, d_out, n, add_db, 2, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}
// waterfall bank (spectrum.cu): fft_cc | logaveragepower_cf | fft_exchange_sides_ff [| compress_fft_adpcm_f_u8] per row
long csdrb_spectrum_bank_lines(const csdrb_spectrum_params_t* p, const csdrb_spectrum_state_t* s, long n) { return spectrum_lines(p, s, n, 0); }
size_t csdrb_spectrum_bank_scratch_bytes(int rows, long n, const csdrb_spectrum_params_t* p) { return spectrum_scratch_bytes(rows, n, p); }
int csdrb_spectrum_bank_cf(const complexf* d_in, long in_stride, int rows, long n, const float* d_window, const csdrb_spectrum_params_t* p,
                           complexf* d_hist_io, float* d_acc_io, csdrb_spectrum_state_t* state_io, void* d_out, long out_stride_bytes,
                           void* d_scratch, size_t scratch_bytes, void* stream)
{
    static_assert(sizeof(csdrb_spectrum_params_t) == sizeof(SpectrumParams) && sizeof(csdrb_spectrum_state_t) == sizeof(SpectrumState),
                  "spectrum structs mirror kernels.h");
    int launches = 0;
    int rc = launch_spectrum_bank(reinterpret_cast<const float2*>(d_in), in_stride, rows, n, d_window, p, reinterpret_cast<float2*>(d_hist_io), d_acc_io,
                                  state_io, d_out, out_stride_bytes, d_scratch, scratch_bytes, &launches, S(stream));
    return rc < 0 ? rc : counted(rc, launches);
}
// real-input waterfall bank (spectrum.cu): fft_fc | logaveragepower_cf [| compress_fft_adpcm_f_u8] per row
long csdrb_spectrum_bank_lines_f(const csdrb_spectrum_params_t* p, const csdrb_spectrum_state_t* s, long n) { return spectrum_lines(p, s, n, 1); }
size_t csdrb_spectrum_bank_scratch_bytes_f(int rows, long n, const csdrb_spectrum_params_t* p) { return spectrum_scratch_bytes(rows, n, p); }
int csdrb_spectrum_bank_f(const float* d_in, long in_stride, int rows, long n, const float* d_window, const csdrb_spectrum_params_t* p,
                          float* d_hist_io, float* d_acc_io, csdrb_spectrum_state_t* state_io, void* d_out, long out_stride_bytes,
                          void* d_scratch, size_t scratch_bytes, void* stream)
{
    int launches = 0;
    int rc = launch_spectrum_bank_f(d_in, in_stride, rows, n, d_window, p, d_hist_io, d_acc_io, state_io, d_out, out_stride_bytes, d_scratch, scratch_bytes,
                                    &launches, S(stream));
    return rc < 0 ? rc : counted(rc, launches);
}
int csdrb_shift_unroll_bank_cc(const complexf* d_in, long in_stride, complexf* d_out, long out_stride, int channels, int input_size,
                               const shift_addition_data_t* d_params, const float* d_dsin, const float* d_dcos, long table_stride, int table_size,
                               float* d_phase_io, void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (too_many_channels(channels, "shift_unroll bank")) return -1;
    if (!d_in || !d_out || !d_params || !d_dsin || !d_dcos || !d_phase_io) { set_error("shift_unroll bank: null pointer"); return -1; }
    int rc = launch_shift_unroll_bank(reinterpret_cast<const float2*>(d_in), in_stride, reinterpret_cast<float2*>(d_out), out_stride, channels, input_size,
                                      reinterpret_cast<const float*>(d_params), d_dsin, d_dcos, table_stride, table_size, d_phase_io, d_scratch, scratch_bytes, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

// ---- device memory / streams for CUDA-header-free hosts ------------------------------------------------------------------
void* csdrb_device_alloc(size_t bytes)
{
    void* p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes ? bytes : 16);
    if (e == cudaSuccess) e = cudaMemset(p, 0, bytes ? bytes : 16);
    if (e != cudaSuccess) { cuda_fail(e, "cudaMalloc/cudaMemset", __FILE__, __LINE__); if (p) cudaFree(p); return nullptr; }
    return p;
}
void csdrb_device_free(void* d_ptr) { if (d_ptr) cudaFree(d_ptr); }
void* csdrb_stream_create(void)
{
    cudaStream_t st = nullptr;
    cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    if (e != cudaSuccess) { cuda_fail(e, "cudaStreamCreateWithFlags", __FILE__, __LINE__); return nullptr; }
    return st;
}
void csdrb_stream_destroy(void* stream) { if (stream) cudaStreamDestroy(S(stream)); }
int csdrb_copy_h2d(void* d_dst, const void* h_src, size_t bytes, void* stream)
{
    if (!bytes) return 0;
    if (null_io(h_src, d_dst, "copy_h2d")) return -1;
    CSDRB_CUDA(cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, S(stream)));
    return 0;
}
int csdrb_copy_d2h(void* h_dst, const void* d_src, size_t bytes, void* stream)
{
    if (!bytes) return 0;
    if (null_io(d_src, h_dst, "copy_d2h")) return -1;
    CSDRB_CUDA(cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, S(stream)));
    return 0;
}
int csdrb_copy_d2d(void* d_dst, const void* d_src, size_t bytes, void* stream)
{
    if (!bytes) return 0;
    if (null_io(d_src, d_dst, "copy_d2d")) return -1;
    CSDRB_CUDA(cudaMemcpyAsync(d_dst, d_src, bytes, cudaMemcpyDeviceToDevice, S(stream)));
    return 0;
}
int csdrb_copy2d_d2d(void* d_dst, size_t dst_pitch_bytes, const void* d_src, size_t src_pitch_bytes, size_t width_bytes, size_t rows, void* stream)
{
    if (!width_bytes || !rows) return 0;
    if (null_io(d_src, d_dst, "copy2d_d2d")) return -1;
    CSDRB_CUDA(cudaMemcpy2DAsync(d_dst, dst_pitch_bytes, d_src, src_pitch_bytes, width_bytes, rows, cudaMemcpyDeviceToDevice, S(stream)));
    return 0;
}
int csdrb_copy2d_h2d(void* d_dst, size_t dst_pitch_bytes, const void* h_src, size_t src_pitch_bytes, size_t width_bytes, size_t rows, void* stream)
{
    if (!width_bytes || !rows) return 0;
    if (null_io(h_src, d_dst, "copy2d_h2d")) return -1;
    CSDRB_CUDA(cudaMemcpy2DAsync(d_dst, dst_pitch_bytes, h_src, src_pitch_bytes, width_bytes, rows, cudaMemcpyHostToDevice, S(stream)));
    return 0;
}
int csdrb_copy2d_d2h(void* h_dst, size_t dst_pitch_bytes, const void* d_src, size_t src_pitch_bytes, size_t width_bytes, size_t rows, void* stream)
{
    if (!width_bytes || !rows) return 0;
    if (null_io(d_src, h_dst, "copy2d_d2h")) return -1;
    CSDRB_CUDA(cudaMemcpy2DAsync(h_dst, dst_pitch_bytes, d_src, src_pitch_bytes, width_bytes, rows, cudaMemcpyDeviceToHost, S(stream)));
    return 0;
}

int csdrb_encode_ima_adpcm_rows_i16_u8(const short* d_in, long in_stride, unsigned char* d_out, long out_stride, int rows, int input_length,
                                       ima_adpcm_state_t* d_state_io, void* stream)
{
    if (!d_in || !d_out || !d_state_io) { set_error("encode_ima_adpcm rows: null pointer"); return -1; }
    int rc = launch_adpcm_encode_rows(d_in, in_stride, d_out, out_stride, rows, input_length, d_state_io, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_compress_fft_adpcm_rows_f_u8(const float* d_in, long in_stride, unsigned char* d_out, long out_stride, int rows, int fft_size, void* stream)
{
    if (!d_in || !d_out) { set_error("compress_fft_adpcm rows: null pointer"); return -1; }
    int rc = launch_compress_fft_adpcm_rows(d_in, in_stride, d_out, out_stride, rows, fft_size, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_limit_ff(const float* d_in, float* d_out, long n, float max_amplitude, void* stream)
{
    if (!d_in || !d_out) { set_error("limit_ff: null pointer"); return -1; }
    int rc = launch_limit_ff(d_in, d_out, n, max_amplitude, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}

int csdrb_deemphasis_wfm_bank_ff(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int input_size, float tau,
                                 int sample_rate, float* d_last_io, void* stream)
{
    if (!d_in || !d_out || !d_last_io) { set_error("deemphasis_wfm bank: null pointer"); return -1; }
    int rc = launch_deemphasis_wfm_bank(d_in, in_stride, d_out, out_stride, channels, input_size, tau, sample_rate, d_last_io, S(stream));
    return rc < 0 ? rc : counted(0, rc);
}
// WFM audio tail (audio.cu): fractional_decimator_ff R 12 | deemphasis_wfm_ff SR TAU | convert_f_s16 per row, in the CLI's B-sample calls
int csdrb_wfm_audio_bank_outputs(const csdrb_wfm_audio_params_t* params, const csdrb_wfm_audio_state_t* state, int n, int* consumed_out)
{
    return wfm_audio_outputs(params, state, n, consumed_out);
}
int csdrb_wfm_audio_bank_f_s16(const float* d_in, long in_stride, int channels, int n, const csdrb_wfm_audio_params_t* params,
                               csdrb_wfm_audio_state_t* state_io, float* d_last_io, short* d_out, long out_stride, int* consumed_out, void* stream)
{
    static_assert(sizeof(csdrb_wfm_audio_params_t) == 16 && sizeof(csdrb_wfm_audio_state_t) == 16, "wfm structs mirror audio.cu");
    if (too_many_channels(channels, "wfm_audio bank")) return -1;
    int launches = 0;
    int rc = launch_wfm_audio_bank(d_in, in_stride, channels, n, params, state_io, d_last_io, d_out, out_stride, consumed_out, &launches, S(stream));
    return rc < 0 ? rc : counted(rc, launches);
}

int csdrb_fir_valid_bank_ff(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int input_size, const float* taps,
                            int taps_length, float limit_max, void* stream)
{
    if (!d_in || !d_out || !taps) { set_error("fir_valid bank: null pointer"); return -1; }
    int rc = launch_fir_valid_bank(d_in, in_stride, d_out, out_stride, channels, input_size, taps, taps_length, limit_max, S(stream));
    if (rc > 0) counted(0, 1);
    return rc;
}

int csdrb_deemphasis_nfm_bank_ff(const float* d_in, long in_stride, float* d_out, long out_stride, int channels, int input_size, int sample_rate,
                                 float limit_max, void* stream)
{
    if (!d_in || !d_out) { set_error("deemphasis_nfm bank: null pointer"); return -1; }
    int rc = launch_deemphasis_nfm_bank(d_in, in_stride, d_out, out_stride, channels, input_size, sample_rate, limit_max, S(stream));
    if (rc > 0) counted(0, 1);
    return rc;
}

size_t csdrb_ddc_bank_scratch_bytes(int channels, int input_size, int chunk, int offset) { return ddc_bank_scratch_bytes(channels, input_size, chunk, offset); }

int csdrb_ddc_bank(const complexf* d_wide, int input_size, int channels, const shift_addition_data_t* d_params, float* d_phase_io, int chunk, int offset,
                   int decimation, const float* h_taps, int taps_length, int demod, void* d_out, long out_stride,
                   const complexf* d_last_in, complexf* d_last_out, void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (!d_wide || !d_params || !d_phase_io || !h_taps || !d_out) { set_error("ddc bank: null pointer"); return -1; }
    int launches = 0;
    int rc = launch_ddc_bank(reinterpret_cast<const float2*>(d_wide), input_size, channels, reinterpret_cast<const float*>(d_params), d_phase_io, chunk, offset,
                             decimation, h_taps, taps_length, demod, d_out, out_stride, reinterpret_cast<const float2*>(d_last_in),
                             reinterpret_cast<float2*>(d_last_out), d_scratch, scratch_bytes, &launches, S(stream));
    if (rc >= 0) g_launches += launches;
    return rc;
}

int csdrb_ddc_bank_f(const float* d_wide, int input_size, int channels, const shift_addition_data_t* d_params, float* d_phase_io, int chunk, int offset,
                     int decimation, const float* h_taps, int taps_length, int demod, void* d_out, long out_stride,
                     const complexf* d_last_in, complexf* d_last_out, void* d_scratch, size_t scratch_bytes, void* stream)
{
    if (!d_wide || !d_params || !d_phase_io || !h_taps || !d_out) { set_error("ddc bank: null pointer"); return -1; }
    int launches = 0;
    int rc = launch_ddc_bank_f(d_wide, input_size, channels, reinterpret_cast<const float*>(d_params), d_phase_io, chunk, offset,
                               decimation, h_taps, taps_length, demod, d_out, out_stride, reinterpret_cast<const float2*>(d_last_in),
                               reinterpret_cast<float2*>(d_last_out), d_scratch, scratch_bytes, &launches, S(stream));
    if (rc >= 0) g_launches += launches;
    return rc;
}

// ---- streaming DDC/NFM bank object ---------------------------------------------------------------------
// Owns every piece of per-channel state (NCO parameters, chunk-start phases, discriminator history, position inside the current
// chunk) so that a stream is processed block by block with one call per block, and hides the serial float phase chain: while the
// caller's stream runs the main kernel of block k, a private side stream already runs the pre-pass of block k+1 (it depends only on
// the previous pre-pass).  Two scratch/phase buffers alternate; a retune or a block of a different size simply drops the look-ahead.
struct csdrb_ddc_bank_s {
    int channels = 0, decimation = 0, taps_length = 0, demod = 0, chunk = 0;
    std::vector<float> taps;
    std::vector<shift_addition_data_t> h_params;
    float* d_params = nullptr;
    float* d_phase[2] = {nullptr, nullptr};          // phase at the start of the chunk holding the next block's first sample (ping-pong)
    float2* d_last[2] = {nullptr, nullptr};          // previous baseband sample per channel (ping-pong across blocks)
    void* d_scratch[2] = {nullptr, nullptr};
    void* d_tables = nullptr;                         // phase-wrap tables (phase_table.cuh), one per channel; rebuilt when a rate changes
    size_t scratch_cap = 0;
    int cur = 0;                                      // which phase/scratch buffer holds the state for the NEXT process() call
    int last_sel = 0;
    int offset = 0;                                   // position of the next block's first sample inside its chunk
    bool ahead_valid = false; int ahead_input_size = 0; // a pre-pass for the next block (of this size) is already in flight/done
    cudaStream_t side = nullptr;
    cudaEvent_t ev_prepass = nullptr, ev_pre_inline = nullptr, ev_main[2] = {nullptr, nullptr};
    long blocks = 0;
    bool params_dirty = false;
};

csdrb_ddc_bank_t* csdrb_ddc_bank_create(int channels, const float* h_rates, int decimation, const float* h_taps, int taps_length, int demod, int chunk)
{
    if (channels <= 0 || !h_rates || !h_taps || decimation <= 0 || taps_length <= 0) { set_error("ddc bank create: bad argument"); return nullptr; }
    if (ddc_bank_geometry(decimation, taps_length) < 0) return nullptr;
    auto* b = new csdrb_ddc_bank_s();
    b->channels = channels; b->decimation = decimation; b->taps_length = taps_length; b->demod = demod ? 1 : 0; b->chunk = chunk > 0 ? chunk : 1024;
    b->taps.assign(h_taps, h_taps + taps_length);
    b->h_params.resize((size_t)channels);
    for (int c = 0; c < channels; c++) b->h_params[(size_t)c] = shift_addition_init(h_rates[c]);
    bool ok = cudaMalloc(&b->d_params, sizeof(shift_addition_data_t) * (size_t)channels) == cudaSuccess;
    for (int k = 0; k < 2 && ok; k++) {
        ok = ok && cudaMalloc(&b->d_phase[k], sizeof(float) * (size_t)channels) == cudaSuccess;
        ok = ok && cudaMalloc(&b->d_last[k], sizeof(float2) * (size_t)channels) == cudaSuccess;
        if (ok) { cudaMemset(b->d_phase[k], 0, sizeof(float) * (size_t)channels); cudaMemset(b->d_last[k], 0, sizeof(float2) * (size_t)channels); }
    }
    ok = ok && cudaMemcpy(b->d_params, b->h_params.data(), sizeof(shift_addition_data_t) * (size_t)channels, cudaMemcpyHostToDevice) == cudaSuccess;
    ok = ok && cudaMalloc(&b->d_tables, ddc_bank_tables_bytes(channels)) == cudaSuccess;
    ok = ok && launch_ddc_tables(channels, b->d_params, b->chunk, b->d_tables, nullptr) >= 0 && cudaStreamSynchronize(nullptr) == cudaSuccess;
    ok = ok && cudaStreamCreateWithFlags(&b->side, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&b->ev_prepass, cudaEventDisableTiming) == cudaSuccess;
    ok = ok && cudaEventCreateWithFlags(&b->ev_pre_inline, cudaEventDisableTiming) == cudaSuccess;
    for (int k = 0; k < 2; k++) ok = ok && cudaEventCreateWithFlags(&b->ev_main[k], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) { set_error("ddc bank create: CUDA allocation failed (%s)", cudaGetErrorString(cudaGetLastError())); csdrb_ddc_bank_destroy(b); return nullptr; }
    return b;
}

void csdrb_ddc_bank_destroy(csdrb_ddc_bank_t* b)
{
    if (!b) return;
    if (b->side) { cudaStreamSynchronize(b->side); cudaStreamDestroy(b->side); }
    if (b->ev_prepass) cudaEventDestroy(b->ev_prepass);
    if (b->ev_pre_inline) cudaEventDestroy(b->ev_pre_inline);
    for (int k = 0; k < 2; k++) if (b->ev_main[k]) cudaEventDestroy(b->ev_main[k]);
    cudaFree(b->d_params); cudaFree(b->d_tables);
    for (int k = 0; k < 2; k++) { cudaFree(b->d_phase[k]); cudaFree(b->d_last[k]); cudaFree(b->d_scratch[k]); }
    delete b;
}

int csdrb_ddc_bank_set_rate(csdrb_ddc_bank_t* b, int channel, float rate)
{
    if (!b || channel < 0 || channel >= b->channels) { set_error("ddc bank set_rate: bad channel"); return -1; }
    b->h_params[(size_t)channel] = shift_addition_init(rate);
    b->params_dirty = true;                           // uploaded, and the look-ahead dropped, at the next process()
    return 0;
}

// close the current NCO chunk at the next block's first sample without changing a rate (what a retune does to every channel of the bank): lets
// several banks that share a stream stay chunk-aligned with each other when only one of them retunes (csrc/multi.cu)
int csdrb_ddc_bank_rechunk(csdrb_ddc_bank_t* b)
{
    if (!b) { set_error("ddc bank rechunk: null pointer"); return -1; }
    b->params_dirty = true;
    return 0;
}

int csdrb_ddc_bank_offset(const csdrb_ddc_bank_t* b) { return b ? b->offset : -1; }

// one block of complex (real = false) or real (real = true) wideband samples; the bank's state does not depend on which, so a stream may even switch
static int ddc_bank_process(csdrb_ddc_bank_t* b, const void* d_wide, bool real, int input_size, void* d_out, long out_stride, void* stream)
{
    if (!b || !d_wide || !d_out) { set_error("ddc bank process: null pointer"); return -1; }
    cudaStream_t st = S(stream);
    const int n_out = input_size >= b->taps_length ? (input_size - b->taps_length) / b->decimation + 1 : 0;
    if (n_out == 0) return 0;
    const size_t need = csdrb_ddc_bank_scratch_bytes(b->channels, input_size, b->chunk, b->chunk - 1) + 64;
    if (need > b->scratch_cap) {                      // grow both scratch buffers (drops any look-ahead)
        CSDRB_CUDA(cudaStreamSynchronize(b->side));
        CSDRB_CUDA(cudaStreamSynchronize(st));
        for (int k = 0; k < 2; k++) { if (b->d_scratch[k]) CSDRB_CUDA(cudaFree(b->d_scratch[k])); CSDRB_CUDA(cudaMalloc(&b->d_scratch[k], need)); }
        b->scratch_cap = need; b->ahead_valid = false;
    }
    int launches = 0;
    if (b->params_dirty) {                            // retune: a pre-pass made with the old deltas is void
        CSDRB_CUDA(cudaStreamSynchronize(b->side));
        // the look-ahead already advanced phase[cur^1] from phase[cur]; phase[cur] is still the state before it: just forget it
        b->ahead_valid = false;
        // The phase stays continuous across a retune only if the new deltas start from the phase AT the retune sample.  phase[cur] is the
        // phase at the start of the current chunk, `offset` samples back: close that chunk here -- advance every channel by `offset` samples
        // at its OLD rate, exactly what the reference does when a caller hands shift_addition_cc a shorter buffer (libcsdr_gpl.c:48-50) -- and
        // start a fresh chunk at this block's first sample.
        if (b->offset > 0) {
            int rc = launch_ddc_rechunk(b->channels, b->d_params, b->d_phase[b->cur], b->offset, st);
            if (rc < 0) return rc;
            launches += rc;
            b->offset = 0;
        }
        CSDRB_CUDA(cudaMemcpyAsync(b->d_params, b->h_params.data(), sizeof(shift_addition_data_t) * (size_t)b->channels, cudaMemcpyHostToDevice, st));
        { int rc = launch_ddc_tables(b->channels, b->d_params, b->chunk, b->d_tables, st); if (rc < 0) return rc; launches += rc; }
        CSDRB_CUDA(cudaStreamSynchronize(st));        // h_params may change again as soon as we return; the side stream reads the new tables next
        b->params_dirty = false;
    }
    int sel;                                          // scratch buffer holding this block's seeds
    if (b->ahead_valid && b->ahead_input_size == input_size) {
        sel = b->cur ^ 1;                             // the side stream produced seeds[sel] and advanced phase[sel] from phase[cur]
        CSDRB_CUDA(cudaStreamWaitEvent(st, b->ev_prepass, 0));
    } else {
        if (b->ahead_valid) CSDRB_CUDA(cudaStreamSynchronize(b->side));   // a mismatching look-ahead: let it finish, then ignore it
        sel = b->cur ^ 1;
        // phase[sel] <- phase[cur], then run the pre-pass on the caller's stream (it advances phase[sel])
        CSDRB_CUDA(cudaMemcpyAsync(b->d_phase[sel], b->d_phase[b->cur], sizeof(float) * (size_t)b->channels, cudaMemcpyDeviceToDevice, st));
        int rc = launch_ddc_prepass(input_size, b->channels, b->d_params, b->d_phase[sel], b->chunk, b->offset, b->decimation, b->taps_length,
                                    b->d_scratch[sel], b->scratch_cap, b->d_tables, st);
        if (rc < 0) return rc;
        launches += rc;
        CSDRB_CUDA(cudaEventRecord(b->ev_pre_inline, st));             // the look-ahead below starts from the phases this pre-pass produced
        CSDRB_CUDA(cudaStreamWaitEvent(b->side, b->ev_pre_inline, 0));
    }
    b->ahead_valid = false;
    // main kernel of this block: discriminator history ping-pongs last[last_sel] -> last[last_sel^1]
    int rc = real ? launch_ddc_main_f(static_cast<const float*>(d_wide), input_size, b->channels, b->d_params, b->chunk, b->offset, b->decimation, b->taps.data(),
                                      b->taps_length, b->demod, d_out, out_stride, b->d_last[b->last_sel], b->d_last[b->last_sel ^ 1], b->d_scratch[sel], st)
                  : launch_ddc_main(static_cast<const float2*>(d_wide), input_size, b->channels, b->d_params, b->chunk, b->offset, b->decimation, b->taps.data(),
                                    b->taps_length, b->demod, d_out, out_stride, b->d_last[b->last_sel], b->d_last[b->last_sel ^ 1], b->d_scratch[sel], st);
    if (rc < 0) return rc;
    launches += 1;
    b->last_sel ^= 1;
    CSDRB_CUDA(cudaEventRecord(b->ev_main[b->blocks & 1], st));
    // state for the next block now lives in phase[sel]; its first sample sits `offset` samples into that chunk
    b->cur = sel;
    b->offset = (int)(((long)b->offset + (long)n_out * b->decimation) % b->chunk);
    // look-ahead: pre-pass of the next block (assumed to have the same size) on the side stream into the other buffer, CONCURRENT
    // with the main kernel just launched.  It only has to wait for (a) this block's pre-pass (ordered above / same stream) and
    // (b) the main kernel of the PREVIOUS block, the last reader of the scratch buffer it is about to overwrite.
    {
        const int nxt = b->cur ^ 1;
        if (b->blocks > 0) CSDRB_CUDA(cudaStreamWaitEvent(b->side, b->ev_main[(b->blocks - 1) & 1], 0));
        CSDRB_CUDA(cudaMemcpyAsync(b->d_phase[nxt], b->d_phase[b->cur], sizeof(float) * (size_t)b->channels, cudaMemcpyDeviceToDevice, b->side));
        int rp = launch_ddc_prepass(input_size, b->channels, b->d_params, b->d_phase[nxt], b->chunk, b->offset, b->decimation, b->taps_length,
                                    b->d_scratch[nxt], b->scratch_cap, b->d_tables, b->side);
        if (rp < 0) return rp;
        launches += rp;
        CSDRB_CUDA(cudaEventRecord(b->ev_prepass, b->side));
        b->ahead_valid = true; b->ahead_input_size = input_size;
    }
    b->blocks++;
    g_launches += launches;
    return n_out;
}

int csdrb_ddc_bank_process(csdrb_ddc_bank_t* b, const complexf* d_wide, int input_size, void* d_out, long out_stride, void* stream)
{
    return ddc_bank_process(b, d_wide, false, input_size, d_out, out_stride, stream);
}

int csdrb_ddc_bank_process_f(csdrb_ddc_bank_t* b, const float* d_wide, int input_size, void* d_out, long out_stride, void* stream)
{
    return ddc_bank_process(b, d_wide, true, input_size, d_out, out_stride, stream);
}

}  // extern "C"
