// cuda_emul.h -- TEST INFRASTRUCTURE: run the shipped CUDA kernels thread by thread on the CPU (CPU test tier only).
//
// Not a CPU fallback: nothing under csdr_b200/ can reach this file; it exists so that kernels which cannot be run in this container
// (no GPU) are still EXECUTED, with their real index arithmetic, barriers and rounding, before GPU minutes are spent on them.
// Model: one CTA at a time; every CUDA thread of the CTA is a ucontext fiber on one OS thread; __syncthreads(), __syncwarp(), named
// barriers (bar.sync id, n) and mbarrier waits are real barriers between fibers (a fiber that reaches one yields until the others have
// arrived); the order in which fibers run between barriers alternates / reverses / is shuffled (CUDA_EMUL_ORDER) so that a missing
// barrier shows as a wrong result; threadIdx/blockIdx/blockDim/gridDim are per-fiber values; dynamic shared memory is one buffer per CTA
// pre-filled with a NaN pattern; IEEE single-precision intrinsics map onto the same operations (fmaf is a true FMA on the host too);
// __shfl_xor_sync goes through a per-warp exchange; the inline-PTX helpers of csrc/common.cuh have C++ models here (ffma2 = two FMAs,
// cp.async.bulk = alignment-checked memcpy that completes an mbarrier, st.global.L1::no_allocate = alignment-checked store); launch
// configurations the hardware would refuse (gridDim.y/z > 65535, > 1024 threads, > 227 KB shared) fail like they would on the GPU.
// Not modelled: the memory model (fibers switch only at barriers, so a race that needs true concurrency can go unnoticed), occupancy and
// register limits, alignment of plain vector loads (build with CUDA_EMUL_SANITIZE=1 for that), atomics, partial-warp votes, clusters, tensor cores.
#pragma once
#define CSDRB_HOST_EMULATION 1
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <functional>
#include <vector>
#include <ucontext.h>

#include <cuda_runtime.h>                       // float2/float4/dim3/uint3, make_float2 ... (host-usable headers of the toolkit)

namespace cuda_emul {

struct Fiber {
    ucontext_t ctx;
    unsigned char* stack = nullptr;              // from a pool that lives as long as the library (never zeroed, never freed)
    uint3 tid;
    bool done = false;
};
inline unsigned char* fiber_stack(size_t index, size_t bytes)
{
    static std::vector<unsigned char*> pool;
    while (pool.size() <= index) pool.push_back(static_cast<unsigned char*>(std::malloc(bytes)));
    return pool[index];
}

struct State {
    ucontext_t sched;
    std::vector<Fiber> fibers;
    Fiber* cur = nullptr;
    dim3 block, grid;
    uint3 bid;
    std::function<void()> body;
    int live = 0, arrived = 0;
    unsigned long generation = 0;
    std::vector<int> warp_live, warp_arrived;
    std::vector<unsigned long> warp_generation;
    std::vector<unsigned char> smem;
    long barriers = 0, switches = 0;
    int order_mode = 0;                       // 0 alternate, 1 reverse, 2 random, 3 forward
    bool launch_error = false;                // a launch configuration the hardware would refuse; cleared by cudaGetLastError()
    unsigned long long rng = 88172645463325252ULL;
};
inline State& st()
{
    static State s;
    static bool init = false;
    if (!init) {
        init = true;
        const char* o = getenv("CUDA_EMUL_ORDER");
        if (o) s.order_mode = !strcmp(o, "reverse") ? 1 : !strcmp(o, "random") ? 2 : !strcmp(o, "forward") ? 3 : 0;
    }
    return s;
}

inline void yield() { State& s = st(); s.switches++; swapcontext(&s.cur->ctx, &s.sched); }

inline void sync_threads()
{
    State& s = st();
    const unsigned long my = s.generation;
    if (++s.arrived == s.live) { s.arrived = 0; s.generation++; s.barriers++; return; }
    while (s.generation == my) yield();
}

inline int linear_tid(const Fiber* f) { State& s = st(); return (int)(f->tid.x + s.block.x * (f->tid.y + s.block.y * f->tid.z)); }

inline void sync_warp()
{
    State& s = st();
    const int w = linear_tid(s.cur) / 32;
    const unsigned long my = s.warp_generation[w];
    if (++s.warp_arrived[w] == s.warp_live[w]) { s.warp_arrived[w] = 0; s.warp_generation[w]++; return; }
    while (s.warp_generation[w] == my) yield();
}

inline void trampoline()
{
    State& s = st();
    s.body();
    Fiber* f = s.cur;
    f->done = true;
    s.live--;
    s.warp_live[linear_tid(f) / 32]--;
    // a barrier the others are waiting in may have become complete by this thread's exit
    if (s.live > 0 && s.arrived == s.live) { s.arrived = 0; s.generation++; }
    const int w = linear_tid(f) / 32;
    if (s.warp_live[w] > 0 && s.warp_arrived[w] == s.warp_live[w]) { s.warp_arrived[w] = 0; s.warp_generation[w]++; }
    swapcontext(&f->ctx, &s.sched);
}

inline unsigned char* dyn_smem() { return st().smem.data(); }

// run `kernel(args...)` for every thread of every CTA of the grid
template <typename K, typename... A>
void launch(dim3 grid, dim3 block, size_t smem_bytes, K kernel, A... args)
{
    State& s = st();
    // what cudaLaunchKernel would refuse on sm_90 (cudaErrorInvalidConfiguration / invalid value): recorded for cudaGetLastError()
    if (grid.x == 0 || grid.y == 0 || grid.z == 0 || grid.y > 65535u || grid.z > 65535u || grid.x > 2147483647u || block.x * block.y * block.z == 0 ||
        block.x * block.y * block.z > 1024u || block.x > 1024u || block.y > 1024u || block.z > 64u || smem_bytes > 227u * 1024u) {
        s.launch_error = true;
        return;
    }
    s.grid = grid; s.block = block;
    const int nthreads = (int)(block.x * block.y * block.z);
    const size_t stack_bytes = 256 * 1024;
    s.body = [=]() { kernel(args...); };
    for (unsigned bz = 0; bz < grid.z; bz++)
        for (unsigned by = 0; by < grid.y; by++)
            for (unsigned bx = 0; bx < grid.x; bx++) {
                s.bid = make_uint3(bx, by, bz);
                s.smem.assign(smem_bytes + 64, 0xFF);                 // NaN pattern: reading shared memory nobody wrote shows up
                s.fibers.clear(); s.fibers.resize((size_t)nthreads);
                s.live = nthreads; s.arrived = 0; s.generation = 0;
                const int nwarps = (nthreads + 31) / 32;
                s.warp_live.assign((size_t)nwarps, 0); s.warp_arrived.assign((size_t)nwarps, 0); s.warp_generation.assign((size_t)nwarps, 0);
                for (int t = 0; t < nthreads; t++) {
                    Fiber& f = s.fibers[(size_t)t];
                    f.tid = make_uint3((unsigned)t % block.x, ((unsigned)t / block.x) % block.y, (unsigned)t / (block.x * block.y));
                    f.stack = fiber_stack((size_t)t, stack_bytes);
                    getcontext(&f.ctx);
                    f.ctx.uc_stack.ss_sp = f.stack; f.ctx.uc_stack.ss_size = stack_bytes; f.ctx.uc_link = nullptr;
                    makecontext(&f.ctx, (void (*)())trampoline, 0);
                    s.warp_live[(size_t)(t / 32)]++;
                }
                // Between two barriers the fibers run one after the other, so a missing barrier only shows when the victim happens to run
                // in the unlucky order: CUDA_EMUL_ORDER = forward | reverse | random (default: alternate forward / reverse every sweep,
                // which exposes read-after-write and write-after-read hazards in both directions).
                std::vector<int> order((size_t)nthreads);
                for (int t = 0; t < nthreads; t++) order[(size_t)t] = t;
                unsigned long sweep = 0;
                while (s.live > 0) {
                    if (s.order_mode == 1 || (s.order_mode == 0 && (sweep & 1))) std::reverse(order.begin(), order.end());
                    else if (s.order_mode == 2) for (int t = nthreads - 1; t > 0; t--) { s.rng = s.rng * 6364136223846793005ULL + 1442695040888963407ULL; std::swap(order[(size_t)t], order[(size_t)((s.rng >> 33) % (unsigned long)(t + 1))]); }
                    for (int k = 0; k < nthreads; k++) {
                        Fiber& f = s.fibers[(size_t)order[(size_t)k]];
                        if (f.done) continue;
                        s.cur = &f;
                        swapcontext(&s.sched, &f.ctx);
                    }
                    if (s.order_mode == 1 || (s.order_mode == 0 && (sweep & 1))) std::reverse(order.begin(), order.end());
                    sweep++;
                }
            }
}

// `k<<<grid, block, smem, stream>>>(args...)` of a launcher is rewritten (tests/host_shim/emul_build.py) to cfg(grid, block, smem, stream).run(k, args...)
struct Cfg {
    dim3 grid, block; size_t smem;
    template <typename K, typename... A> void run(K kernel, A... args) const { launch(grid, block, smem, kernel, args...); }
};
inline Cfg cfg(dim3 grid, dim3 block, size_t smem = 0, void* /*stream*/ = nullptr) { return Cfg{grid, block, smem}; }

// ---- warp shuffle: lanes publish, meet at a warp barrier, read their partner, meet again -----------------------------------------
inline unsigned char* warp_scratch() { static unsigned char buf[64][32][16]; return &buf[0][0][0]; }
template <typename T> T shfl_xor(T v, int lane_mask)
{
    static_assert(sizeof(T) <= 16, "shuffle payload");
    State& s = st();
    const int t = linear_tid(s.cur), w = t / 32, l = t % 32;
    unsigned char* base = warp_scratch() + ((size_t)w * 32) * 16;
    std::memcpy(base + (size_t)l * 16, &v, sizeof(T));
    sync_warp();
    T r; std::memcpy(&r, base + (size_t)(l ^ lane_mask) * 16, sizeof(T));
    sync_warp();
    return r;
}

// warp-wide exchange of one value per lane: every lane publishes, all meet, every lane reads what it wants, all meet again
template <typename T, typename F> auto warp_exchange(T v, F pick)
{
    static_assert(sizeof(T) <= 16, "exchange payload");
    State& s = st();
    const int t = linear_tid(s.cur), w = t / 32, l = t % 32;
    unsigned char* base = warp_scratch() + ((size_t)w * 32) * 16;
    std::memcpy(base + (size_t)l * 16, &v, sizeof(T));
    sync_warp();
    auto r = pick(reinterpret_cast<const unsigned char*>(base), l);
    sync_warp();
    return r;
}
template <typename T> T shfl_idx(T v, int src)
{
    return warp_exchange(v, [src](const unsigned char* base, int) { T r; std::memcpy(&r, base + (size_t)(src & 31) * 16, sizeof(T)); return r; });
}
inline unsigned ballot(int pred)                 // full, converged warps only (what the kernels use): a lane that has exited would hang the barrier on the GPU too
{
    return warp_exchange(pred, [](const unsigned char* base, int) { unsigned m = 0; for (int i = 0; i < 32; i++) { int p; std::memcpy(&p, base + (size_t)i * 16, 4); if (p) m |= 1u << i; } return m; });
}

// ---- named barriers (bar.sync id, count) --------------------------------------------------------------------------------------------
struct NamedBar { int arrived = 0; unsigned long generation = 0; };
inline NamedBar& named_bar(int id) { static NamedBar b[16]; return b[id & 15]; }
inline void named_sync(int id, int nthreads)
{
    NamedBar& b = named_bar(id);
    const unsigned long my = b.generation;
    if (++b.arrived == nthreads) { b.arrived = 0; b.generation++; return; }
    while (b.generation == my) yield();
}

inline bool take_launch_error() { State& s = st(); const bool e = s.launch_error; s.launch_error = false; return e; }

}  // namespace cuda_emul

extern "C" int cuda_emul_take_launch_error(void);     // cuda_emul_runtime.cpp asks through this (defined once per library, below or in the harness)

// ---- the CUDA surface the kernels use ----------------------------------------------------------------------------------------
#define threadIdx (::cuda_emul::st().cur->tid)
#define blockIdx (::cuda_emul::st().bid)
#define blockDim (::cuda_emul::st().block)
#define gridDim (::cuda_emul::st().grid)
#define __syncthreads() ::cuda_emul::sync_threads()
#define __syncwarp() ::cuda_emul::sync_warp()
#define CSDRB_DYN_SMEM(name) unsigned char* name = ::cuda_emul::dyn_smem()
#define __launch_bounds__(...)
#define __grid_constant__
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))
#endif
#undef __global__
#define __global__
#undef __shared__
#define __shared__ static                       /* one CTA runs at a time, so a function-level static is CTA-shared */

template <typename T> static inline T __ldg(const T* p) { return *p; }
static inline float __uint_as_float(unsigned u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline unsigned __float_as_uint(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }
static inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
static inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
static inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
static inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
static inline size_t __cvta_generic_to_shared(const void*) { return 0; }
static inline int __float2int_rz(float f) { return (int)f; }                       // callers guard the range, as they must on the GPU
static inline int __float2int_rn(float f) { return (int)nearbyintf(f); }
static inline float __int2float_rn(int i) { return (float)i; }
static inline float __double2float_rn(double d) { return (float)d; }         // round to nearest even (the default rounding mode of the host)
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
template <typename T> static inline cudaError_t cudaFuncSetAttribute(T*, cudaFuncAttribute, int) { return cudaSuccess; }
template <typename T> static inline T __shfl_xor_sync(unsigned, T v, int lane_mask) { return ::cuda_emul::shfl_xor(v, lane_mask); }
template <typename T> static inline T __shfl_sync(unsigned, T v, int src_lane) { return ::cuda_emul::shfl_idx(v, src_lane); }
static inline unsigned __ballot_sync(unsigned, int pred) { return ::cuda_emul::ballot(pred); }
static inline int __popc(unsigned v) { return __builtin_popcount(v); }

// ---- C++ models of the inline-PTX helpers of csdr_b200/csrc/common.cuh (which steps aside under CSDRB_HOST_EMULATION) ------------
namespace csdrb {
static inline float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }     // two IEEE FMAs
static inline float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
static inline float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
static inline float2 fsub2(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
static inline uint32_t smem_u32(const void*) { return 0; }
// one-phase mbarrier model: word 0 = arrivals still expected, word 1 = transaction bytes still in flight; complete when both are 0
static inline void mbar_init(uint64_t* bar, uint32_t count) { int32_t* w = reinterpret_cast<int32_t*>(bar); w[0] = (int32_t)count; w[1] = 0; }
static inline void mbar_fence_init() {}
static inline void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) { int32_t* w = reinterpret_cast<int32_t*>(bar); w[1] += (int32_t)bytes; w[0] -= 1; }
static inline void mbar_arrive(uint64_t* bar) { reinterpret_cast<int32_t*>(bar)[0] -= 1; }
static inline void mbar_wait(uint64_t* bar, uint32_t parity)
{
    if (parity != 0) { std::fprintf(stderr, "cuda_emul: only phase 0 of an mbarrier is modelled\n"); std::abort(); }
    volatile int32_t* w = reinterpret_cast<volatile int32_t*>(bar);
    while (w[0] != 0 || w[1] != 0) ::cuda_emul::yield();
}
static inline void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar)
{
    if ((reinterpret_cast<uintptr_t>(smem_dst) & 15) || (reinterpret_cast<uintptr_t>(gmem_src) & 15) || (bytes & 15)) {
        std::fprintf(stderr, "cuda_emul: cp.async.bulk needs 16-byte aligned addresses and size\n"); std::abort();          // the GPU would fault here
    }
    std::memcpy(smem_dst, gmem_src, bytes);
    reinterpret_cast<int32_t*>(bar)[1] -= (int32_t)bytes;
}
static inline void st_na_f4(float4* p, float4 v)
{
    if (reinterpret_cast<uintptr_t>(p) & 15) { std::fprintf(stderr, "cuda_emul: misaligned 128-bit store\n"); std::abort(); }
    *p = v;
}
static inline void named_bar_sync(int id, int nthreads) { ::cuda_emul::named_sync(id, nthreads); }
// cp.async: the copy happens at once (alignment checked like the hardware would); commit / wait are no-ops, so a MISSING wait goes unnoticed here
static inline void cp_async16(void* smem_dst, const void* gmem_src)
{
    if ((reinterpret_cast<uintptr_t>(smem_dst) & 15) || (reinterpret_cast<uintptr_t>(gmem_src) & 15)) {
        std::fprintf(stderr, "cuda_emul: cp.async 16 needs 16-byte aligned addresses\n"); std::abort();
    }
    std::memcpy(smem_dst, gmem_src, 16);
}
static inline void cp_async8(void* smem_dst, const void* gmem_src)
{
    if ((reinterpret_cast<uintptr_t>(smem_dst) & 7) || (reinterpret_cast<uintptr_t>(gmem_src) & 7)) {
        std::fprintf(stderr, "cuda_emul: cp.async 8 needs 8-byte aligned addresses\n"); std::abort();
    }
    std::memcpy(smem_dst, gmem_src, 8);
}
static inline void cp_async_commit() {}
template <int PENDING> static inline void cp_async_wait() {}
}  // namespace csdrb

// the CUDA runtime calls launchers and the C ABI make are stubbed in cuda_emul_runtime.cpp (one copy per emulated library)
