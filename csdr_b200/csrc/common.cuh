// common.cuh -- shared device helpers for the csdr_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

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

// ---- exact fast-forward of the reference's phase wrap ----------------------------------------------
//   while (ph >  PI) ph -= 2*PI;   while (ph < -PI) ph += 2*PI;        (libcsdr_gpl.c:49-50, PI = (float)3.14159...)
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
    a = a >= lo ? __fsub_rn(a, 6.28318530717958647692f) : a;
    a = a >= lo ? __fsub_rn(a, 6.28318530717958647692f) : a;
    return a;
}

__device__ __forceinline__ float wrap_phase_pm_pi(float ph)
{
    const float PI_F32 = 3.14159265358979323846f, TWO_PI_F32 = 6.28318530717958647692f;   // float(2)*PI rounds to the same float
    const bool neg = (__float_as_uint(ph) >> 31) != 0u;   // sign bit, so that -0.0 stays -0.0 like the loop leaves it
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
    while (a > PI_F32) a = __fsub_rn(a, TWO_PI_F32);                                       // below 16: at most three plain steps
    return neg ? -a : a;
}

}  // namespace csdrb
