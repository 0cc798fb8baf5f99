// The priority tree of prioritized replay (include/serl_td3_per.h): the kernels that insert rows, rebuild the tree, draw a
// batch and re-prioritise rows outside K7.  The draw and the re-prioritising are per.cuh's, the code K7's PER learner runs.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/serl_td3_per.h"
#include "common.cuh"
#include "per.cuh"

namespace {

constexpr int NT = 256, NT_MAX = 1024;

// the largest stored priority (1.0 when nothing is stored) on to the leaves of the n rows from `start` (mod capacity).
// One CTA: a max reduction over the stored leaves, then the writes.  Writing the max never lowers the max, so this equals
// n single adds of the reference buffer, each giving its row the max of the priorities stored before it.
__global__ void __launch_bounds__(NT_MAX) per_insert_kernel(double* t, int leaves, int capacity, int n_valid, int start, int n)
{
    __shared__ double red[NT_MAX / 32];
    double m = 0.0;
    for (int i = threadIdx.x; i < n_valid; i += NT_MAX) m = fmax(m, t[2 * (leaves + i)]);
#pragma unroll
    for (int o = 16; o; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = 0.0;
    for (int w = 0; w < NT_MAX / 32; ++w) m = fmax(m, red[w]);
    const double p = n_valid ? m : 1.0;
    for (int i = threadIdx.x; i < n; i += NT_MAX) {
        const int r = (start + i) % capacity;
        t[2 * (leaves + r)] = p;
        t[2 * (leaves + r) + 1] = p;
    }
}

// the nodes [first, 2 first) of one level from their children
__global__ void per_level_kernel(double* t, int first)
{
    for (int v = first + blockIdx.x * NT + threadIdx.x; v < 2 * first; v += gridDim.x * NT) {
        t[2 * v] = t[4 * v] + t[4 * v + 2];
        t[2 * v + 1] = fmin(t[4 * v + 1], t[4 * v + 3]);
    }
}

__global__ void __launch_bounds__(NT) per_update_kernel(double* t, int leaves, const int* rows, const float* td, int n, double alpha)
{
    per_reprioritise(t, leaves, rows, td, n, alpha);
}

__global__ void per_sample_kernel(const double* t, int leaves, int n_valid, int batch, unsigned long long seed, long long it,
                                  double beta, int* rows, float* w)
{
    const int j = blockIdx.x * NT + threadIdx.x;
    if (j >= batch) return;
    const int r = per_draw(t, leaves, seed, it, j);
    rows[j] = r;
    w[j] = per_weight(t, leaves, n_valid, r, beta);
}

int rebuild(double* t, int leaves, cudaStream_t s)
{
    for (int first = leaves / 2; first >= 1; first /= 2) {
        const int grid = (first + NT - 1) / NT < 1024 ? (first + NT - 1) / NT : 1024;
        if (const int rc = serl_launch("per_level_kernel", per_level_kernel, dim3(grid), dim3(NT), 0, s, t, first)) return rc;
    }
    return SERL_OK;
}

bool capacity_ok(int32_t c) { return c >= 1 && c <= SERL_PER_MAX_CAPACITY; }

}  // namespace

extern "C" int64_t serl_per_tree_doubles(int32_t capacity)
{
    if (!capacity_ok(capacity)) return serl_fail(SERL_ERR_ARG, "serl_per_tree_doubles: capacity must be 1..SERL_PER_MAX_CAPACITY");
    return 4 * (int64_t)per_leaves(capacity);
}

extern "C" int serl_per_rebuild(double* d_tree, int32_t capacity, void* stream)
{
    if (!d_tree || !capacity_ok(capacity)) return serl_fail(SERL_ERR_ARG, "serl_per_rebuild: null d_tree or bad capacity");
    return rebuild(d_tree, per_leaves(capacity), (cudaStream_t)stream);
}

extern "C" int serl_per_insert(double* d_tree, int32_t capacity, int32_t n_valid, int32_t start, int32_t n, void* stream)
{
    if (!d_tree || !capacity_ok(capacity) || n < 1 || n > capacity || start < 0 || start >= capacity || n_valid < 0 ||
        n_valid > capacity)
        return serl_fail(SERL_ERR_ARG, "serl_per_insert: null d_tree, bad capacity, or n / start / n_valid outside the ring");
    const cudaStream_t s = (cudaStream_t)stream;
    const int leaves = per_leaves(capacity);
    if (const int rc = serl_launch("per_insert_kernel", per_insert_kernel, dim3(1), dim3(NT_MAX), 0, s, d_tree, leaves, (int)capacity,
                                   (int)n_valid, (int)start, (int)n))
        return rc;
    return rebuild(d_tree, leaves, s);
}

extern "C" int serl_per_update(double* d_tree, int32_t capacity, const int32_t* d_rows, const float* d_td, int32_t n, double alpha,
                               void* stream)
{
    if (!d_tree || !d_rows || !d_td || !capacity_ok(capacity) || n < 1 || n > SERL_TD3_MAX_BATCH || !(alpha > 0.0 && alpha <= 1.0))
        return serl_fail(SERL_ERR_ARG, "serl_per_update: null pointer, bad capacity, n outside 1..128 or alpha outside (0, 1]");
    return serl_launch("per_update_kernel", per_update_kernel, dim3(1), dim3(NT), 0, (cudaStream_t)stream, d_tree,
                       per_leaves(capacity), (const int*)d_rows, d_td, (int)n, alpha);
}

extern "C" int serl_per_sample(const double* d_tree, int32_t capacity, int32_t n_valid, int32_t batch, uint64_t seed, int64_t iteration,
                               double beta, int32_t* d_rows, float* d_weights, void* stream)
{
    if (!d_tree || !d_rows || !d_weights || !capacity_ok(capacity) || n_valid < 1 || n_valid > capacity || batch < 1 ||
        !(beta >= 0.0 && beta <= 1.0))
        return serl_fail(SERL_ERR_ARG, "serl_per_sample: null pointer, bad capacity, n_valid outside 1..capacity, batch < 1 or "
                                       "beta outside [0, 1]");
    return serl_launch("per_sample_kernel", per_sample_kernel, dim3((batch + NT - 1) / NT), dim3(NT), 0, (cudaStream_t)stream,
                       d_tree, per_leaves(capacity), (int)n_valid, (int)batch, (unsigned long long)seed, (long long)iteration, beta,
                       (int*)d_rows, d_weights);
}
