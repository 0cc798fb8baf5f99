#include <atomic>
#include <map>
#include <mutex>
#include <stdio.h>
#include <string.h>
#include <tuple>

#include "../../include/serl_b200.h"
#include "common.cuh"

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

int serl_fail(int code, const char* msg)
{
    snprintf(g_err, sizeof(g_err), "%s", msg);
    return code;
}

int serl_fail_cuda(cudaError_t e, const char* where)
{
    snprintf(g_err, sizeof(g_err), "%s: %s", where, cudaGetErrorString(e));
    // consume the runtime's record of an error reported here (e.g. a refused shared-memory opt-in), so that the caller's
    // next CUDA call does not fail with it again
    cudaGetLastError();
    return SERL_ERR_CUDA;
}

void serl_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }

extern "C" int64_t serl_launch_count(void) { return (int64_t)g_launches.load(); }
extern "C" const char* serl_last_error(void) { return g_err; }

int serl_device_sms()
{
    static int num_sms = 0;
    if (num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        if (cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || num_sms <= 0) num_sms = 132;
    }
    return num_sms;
}

// One grow-only buffer per (device, purpose, stream), kept for the life of the process.  Launches on one stream are
// ordered, so they can share it; launches on different streams (the Agent's side-stream episodes next to the population
// rollout) get their own.  No stream-ordered allocator here: growing its pool maps memory, which waits for kernels in
// flight on OTHER streams.
cudaError_t serl_scratch(int purpose, cudaStream_t s, size_t bytes, void** out)
{
    struct Buf { void* p; size_t bytes; };
    static std::mutex mu;
    static std::map<std::tuple<int, int, cudaStream_t>, Buf> pool;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lk(mu);
    Buf& b = pool[std::make_tuple(dev, purpose, s)];
    if (b.bytes < bytes) {
        if (b.p) { cudaStreamSynchronize(s); cudaFree(b.p); b.p = nullptr; b.bytes = 0; }
        const size_t want = bytes + bytes / 4;
        cudaError_t e = cudaMalloc(&b.p, want);
        if (e != cudaSuccess) return e;
        b.bytes = want;
    }
    *out = b.p;
    return cudaSuccess;
}
