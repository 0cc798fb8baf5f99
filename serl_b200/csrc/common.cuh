// Shared host-side helpers of the C-ABI: error reporting, launch accounting, the SM count and the launch scratch pool.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

#include "../../include/serl_b200.h"

int serl_fail(int code, const char* msg);
int serl_fail_cuda(cudaError_t e, const char* where);
void serl_count_launch();

// shared memory a CTA may opt in to on sm_90a (static + dynamic)
constexpr size_t SERL_SMEM_OPTIN = 227 * 1024;

// SMs of the current device (cached after the first call; 132 = H100 SXM if the query fails)
int serl_device_sms();

// what a scratch buffer holds; launches of different purposes never share one
enum { SERL_SCRATCH_K1 = 0, SERL_SCRATCH_K6 = 1, SERL_SCRATCH_TC = 2, SERL_SCRATCH_TD3 = 3 };
// a device buffer of at least `bytes` for launches of `purpose` on stream `s` of the current device
cudaError_t serl_scratch(int purpose, cudaStream_t s, size_t bytes, void** out);

#ifdef __CUDACC__
// Every kernel launch of the library: raises the kernel's dynamic shared-memory limit to `smem` when it uses any (the
// 48 KB default counts the kernel's static shared memory too), launches, counts the launch once (serl_launch_count)
// and reports a CUDA error as SERL_ERR_CUDA with `what`.
template <typename... P, typename... A>
int serl_launch(const char* what, void (*k)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, A... args)
{
    if (smem > 0) {
        const cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return serl_fail_cuda(e, what);
    }
    k<<<grid, block, smem, s>>>(args...);
    serl_count_launch();
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? SERL_OK : serl_fail_cuda(e, what);
}
#endif
