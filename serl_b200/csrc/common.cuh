// Shared host-side helpers of the C-ABI: error reporting, launch accounting, the SM count and the launch scratch pool.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>

int serl_fail(int code, const char* msg);
int serl_fail_cuda(cudaError_t e, const char* where);
void serl_count_launch();

// SMs of the current device (cached after the first call; 132 = H100 SXM if the query fails)
int serl_device_sms();

// what a scratch buffer holds; launches of different purposes never share one
enum { SERL_SCRATCH_K1 = 0, SERL_SCRATCH_K6 = 1, SERL_SCRATCH_TC = 2 };
// a device buffer of at least `bytes` for launches of `purpose` on stream `s` of the current device
cudaError_t serl_scratch(int purpose, cudaStream_t s, size_t bytes, void** out);
