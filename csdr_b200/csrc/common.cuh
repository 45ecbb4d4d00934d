// common.cuh -- shared device helpers for the csdr_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>
#include <vector>

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "csdr_b200 kernels are written for sm_90a (H100) only"
#endif

// dynamic shared memory of a kernel; the CPU-tier emulator (tests/host_shim/cuda_emul.h) supplies its own definition
#ifndef CSDRB_DYN_SMEM
#define CSDRB_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif

namespace csdrb {

// SMs of an H100 SXM: the launch-size heuristics aim at whole waves of this many SMs
constexpr long kSmCount = 132;

// ---- error plumbing (host) ---------------------------------------------------------------------
// Every C-ABI entry point returns >= 0 on success and a negative csdrb_status on failure; the text of
// the last failure is kept per thread (csdrb_last_error()).
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);
#define CSDRB_CUDA(call)                                                                  \
    do {                                                                                  \
        cudaError_t e_ = (call);                                                          \
        if (e_ != cudaSuccess) return ::csdrb::cuda_fail(e_, #call, __FILE__, __LINE__);  \
    } while (0)
// adds n to the process's kernel-launch count (csdrb_kernel_launches, CSDRB_TRACE) when rc >= 0; returns rc
int counted(int rc, int n = 1);

// The T of the current device, created on first use: host-side state whose device buffers and streams belong to one device
// (a process may csdrb_set_device() between calls).
template <class T>
T& per_device()
{
    static std::mutex mu;
    static std::vector<T*> per_dev;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0) dev = 0;
    std::lock_guard<std::mutex> lk(mu);
    if ((size_t)dev >= per_dev.size()) per_dev.resize((size_t)dev + 1, nullptr);
    if (!per_dev[(size_t)dev]) per_dev[(size_t)dev] = new T();
    return *per_dev[(size_t)dev];
}

// k<<<grid, block, smem, st>>>(args...), returning the launch's error.  Above 47 KB of dynamic shared memory the kernel's limit is raised first, on
// every call: the attribute belongs to the current device's context, and the 48 KB default also has to hold the kernel's static shared memory.
#if defined(__CUDACC__) || defined(CSDRB_HOST_EMULATION)
template <typename K, typename... A>
cudaError_t launch_kernel(K k, dim3 grid, dim3 block, size_t smem, cudaStream_t st, A... args)
{
    if (smem > 47 * 1024) {
        if (cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) return e;
    }
#ifdef CSDRB_HOST_EMULATION
    ::cuda_emul::cfg(grid, block, smem, st).run(k, args...);         // what tests/host_shim/emul_build.py makes of a launch in a .cu file
#else
    k<<<grid, block, smem, st>>>(args...);
#endif
    return cudaGetLastError();
}
#endif

// The inline-PTX helpers below have C++ models in tests/host_shim/cuda_emul.h (CPU test tier); the product never defines this macro.
#ifndef CSDRB_HOST_EMULATION
// ---- complex-lane FP32 pairs ------------------------------------------------------------------
// The I and the Q lane of a complex sample.  Hopper has no packed FP32 instruction, so each helper is two
// scalar IEEE-754 fp32 operations (round-to-nearest-even); the _rn intrinsics keep ptxas from contracting
// a separately rounded product into a later add.
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c)
{
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fsub2(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// ---- mbarrier + bulk async copy (the 1-D TMA path: SASS UBLKCP) ----------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-byte aligned; completes on `bar`.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// streaming global store that does not pollute L1
__device__ __forceinline__ void st_na_f4(float4* p, float4 v)
{
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads)
{
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// Ampere-style 16-byte asynchronous copies global -> shared (SASS LDGSTS), for tiles too ragged for one bulk copy
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
// 8-byte form (one complex sample): for tiles whose rows have an odd pitch in shared memory (conflict-free row walks) and cannot take 16-byte pieces
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gmem_src)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(PENDING) : "memory"); }

#endif  // CSDRB_HOST_EMULATION

// ---- convert_f_s16 of one value (libcsdr.c:2390-2398): float multiply by 32767, truncate toward zero, keep the low 16 bits of the int32 ----
// (what cvttss2si + a 16-bit store do on the reference's x86 build; out-of-range / NaN -> INT_MIN -> 0)
__device__ __forceinline__ unsigned f_to_s16_bits(float x)
{
    const float s = __fmul_rn(x, 32767.0f);
    const int w = (s >= 2147483648.0f || s < -2147483648.0f || s != s) ? (-2147483647 - 1) : __float2int_rz(s);
    return (unsigned)w & 0xffffu;
}

// ---- the reference's complex rotation: two rounded products, then a rounded difference / sum ----------------------------
//   (p.x*v.x - p.y*v.y, p.y*v.x + p.x*v.y)   e.g. libcsdr_gpl.c:39-45: the sample times the phasor, and the phasor recursion with v = (cosd, sind)
__device__ __forceinline__ float2 rotate_rn(float2 p, float2 v)
{
    return make_float2(__fsub_rn(__fmul_rn(p.x, v.x), __fmul_rn(p.y, v.y)), __fadd_rn(__fmul_rn(p.y, v.x), __fmul_rn(p.x, v.y)));
}

// the reference's PI (libcsdr.h:65) as a float; 2*PI in float arithmetic is exactly twice it
constexpr float kPiF = 3.14159265358979323846f;
constexpr float kTwoPiF = 2.f * kPiF;

// ---- exact fast-forward of the reference's phase wrap ----------------------------------------------
//   while (ph >  PI) ph -= 2*PI;   while (ph < -PI) ph += 2*PI;        (libcsdr_gpl.c:49-50)
// Every subtraction rounds, so the loop cannot be replaced by fmod.  But while |ph| stays in one binade
// [2^E, 2^(E+1)), E >= 4, ph = M*u (u = 2^(E-23), M a 24-bit integer) and fl(ph - c) = (M - q)*u with
// q = round(c/u) independent of M (c/u is never a tie for the float 2*pi = 0xC90FDB * 2^-21, checked for all E),
// as long as the exact difference stays in the binade, i.e. M >= 2^23 + ceil(c/u).  So whole runs of iterations
// collapse into one integer multiply; the binade-crossing steps are done with a real float subtraction.
// Bit-exact with the loop (tests/test_gpu_parity2.py::test_phase_wrap_fast_forward_is_exact on the GPU; tests/test_phase_wrap_host.py compiles
// this very function for the host and sweeps every binade on the CPU tier), ~25 steps instead of ~400.
template <int E>
__device__ __forceinline__ float wrap_binade_step(float a)
{
    // Branch-free (lanes = channels sit in different binades; predication keeps the warp converged).
    // a in [2^E, 2^(E+1)): collapse every subtraction that provably stays in this binade, then cross with real subtractions.
    constexpr unsigned MC = 0xC90FDBu;
    constexpr int sh = E - 2;
    constexpr unsigned q = (MC + (1u << (sh - 1))) >> sh;                                         // round(c/u)
    constexpr unsigned mmin = (1u << 23) + ((MC + (1u << sh) - 1u) >> sh);                        // 2^23 + ceil(c/u)
    const float lo = __uint_as_float((unsigned)(E + 127) << 23);                                  // 2^E
    const unsigned M = (__float_as_uint(a) & 0x7fffffu) | 0x800000u;
    const int span = (int)M - (int)mmin;
    const unsigned k = span >= 0 ? (unsigned)span / q + 1u : 0u;                                  // division by a compile-time constant
    const float bulk = __uint_as_float(((unsigned)(E + 127) << 23) | ((M - k * q) & 0x7fffffu));
    a = a >= lo ? bulk : a;
    // after the bulk step a < 2^E + c + u, so at most two real (rounded) subtractions cross the boundary
    a = a >= lo ? __fsub_rn(a, kTwoPiF) : a;
    a = a >= lo ? __fsub_rn(a, kTwoPiF) : a;
    return a;
}

// The wrapped phase from the wrapped magnitude a = |result|: the sign of x, except that a wrap landing exactly on zero gives +0, as the
// reference's loop does (fl(-2*pi + 2*pi) = +0); only an input of -0.0, which no loop step touches, stays -0.0.
__device__ __forceinline__ float wrap_sign(float x, float a)
{
    return (__float_as_uint(x) >> 31) && (a != 0.f || x == 0.f) ? -a : a;
}

__device__ __forceinline__ float wrap_phase_pm_pi(float ph)
{
    float a = fabsf(ph);
    if (!(a < 67108864.f)) return ph;                // |ph| >= 2^26 (or nan): subtracting 2*pi no longer changes it; the reference would spin
    if (a >= 1048576.f) {                            // 2^20 and up: rare
        a = wrap_binade_step<25>(a); a = wrap_binade_step<24>(a); a = wrap_binade_step<23>(a);
        a = wrap_binade_step<22>(a); a = wrap_binade_step<21>(a); a = wrap_binade_step<20>(a);
    }
    if (a >= 8192.f) {                               // 2^13 .. 2^20
        a = wrap_binade_step<19>(a); a = wrap_binade_step<18>(a); a = wrap_binade_step<17>(a); a = wrap_binade_step<16>(a);
        a = wrap_binade_step<15>(a); a = wrap_binade_step<14>(a); a = wrap_binade_step<13>(a);
    }
    if (a >= 16.f) {                                 // the common range: one 1024-sample chunk advances the phase by < 2^12 rad
        a = wrap_binade_step<12>(a); a = wrap_binade_step<11>(a); a = wrap_binade_step<10>(a);
        a = wrap_binade_step<9>(a);  a = wrap_binade_step<8>(a);  a = wrap_binade_step<7>(a);
        a = wrap_binade_step<6>(a);  a = wrap_binade_step<5>(a);  a = wrap_binade_step<4>(a);
    }
    while (a > kPiF) a = __fsub_rn(a, kTwoPiF);                                            // below 16: at most three plain steps
    return wrap_sign(ph, a);
}

// The reference's phase advance over n samples, starting_phase += rate*PI*n (libcsdr_gpl.c:48, :154): fl(fl(rate*PI)*n) ...
__device__ __forceinline__ float phase_increment(float rate, int n) { return __fmul_rn(__fmul_rn(rate, kPiF), (float)n); }
// ... added to the phase and wrapped into [-PI, PI]: one step of the chain ph <- wrap(fl(ph + inc))
__device__ __forceinline__ float phase_step(float ph, float inc) { return wrap_phase_pm_pi(__fadd_rn(ph, inc)); }

// groups of I outputs one fir_interpolate_cc call on n inputs gives (libcsdr.c:579-602): interpolate.cu's bank and synth.cu's synthesis bank
__host__ __device__ inline long interp_groups(int n, int I, int T)
{
    const long h = ((long)T - 1 + I - 1) / I;                // ceil((T-1)/I): inputs each group looks ahead
    return n > h ? (long)n - h : 0;
}

}  // namespace csdrb
