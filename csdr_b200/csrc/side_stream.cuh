// side_stream.cuh -- one private side stream + fork/join/slice events per device and translation unit, for work that is independent of the data path
// of a call (phase chains, state chains): forked from the caller's stream, joined back into it.
#pragma once
#include "common.cuh"
#include <map>
#include <mutex>

namespace csdrb {

constexpr int kSideSlices = 8;
struct SideStream { cudaStream_t stream = nullptr; cudaEvent_t fork = nullptr, join = nullptr, slice[kSideSlices] = {}; std::mutex mu; };

static SideStream* side_stream()
{
    static std::map<int, SideStream*> per_dev;
    static std::mutex mu;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { set_error("cudaGetDevice failed"); return nullptr; }
    std::lock_guard<std::mutex> lk(mu);
    auto it = per_dev.find(dev);
    if (it != per_dev.end()) return it->second;
    auto* s = new SideStream();
    bool ok = cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking) == cudaSuccess && cudaEventCreateWithFlags(&s->fork, cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&s->join, cudaEventDisableTiming) == cudaSuccess;
    for (int i = 0; i < kSideSlices && ok; i++) ok = cudaEventCreateWithFlags(&s->slice[i], cudaEventDisableTiming) == cudaSuccess;
    if (!ok) { set_error("side stream: CUDA object creation failed"); delete s; return nullptr; }
    // stream-ordered scratch (cudaMallocAsync) must not go back to the OS at every synchronisation: keep the pool's memory (re-mapping the fastddc
    // scratch at every call costs more than the kernels)
    cudaMemPool_t pool = nullptr;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) { unsigned long long keep = ~0ULL; cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep); }
    per_dev[dev] = s;
    return s;
}

}  // namespace csdrb
