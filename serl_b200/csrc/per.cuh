// The priority tree of prioritized replay (include/serl_td3_per.h) on the device: the draw, the importance weight and the
// re-prioritising, shared by K7's PER learner (td3.cu) and the tree's own kernels (per.cu), so that serl_per_sample draws
// exactly the rows K7 draws.  Node n: sum at t[2n], min at t[2n + 1]; leaf i is node leaves + i.
#pragma once
#include <stdint.h>

#include "philox.cuh"

// the Philox stream of PER draws: after K7's index, noise and CAPS streams (0..3)
constexpr uint32_t PER_TAG = 4;

__host__ __device__ inline int per_leaves(int capacity)
{
    int l = 1;
    while (l < capacity) l <<= 1;
    return l;
}

// row `row` of the batch of global iteration `it`: u uniform in [0, 1) with 53 bits, the target u * sum p, and the descent
// from the root — left when the target is below the left sum, else right minus the left sum.  A right child whose sum is 0
// (no stored row under it) is never entered, so a target that rounding leaves at or above the root's sum still ends on a
// stored row.
__device__ __forceinline__ int per_draw(const double* t, int leaves, unsigned long long seed, long long it, int row)
{
    const uint4 r = philox(make_uint4((uint32_t)it, (uint32_t)((unsigned long long)it >> 32), (uint32_t)row, PER_TAG),
                           make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const double u = (double)(((unsigned long long)(r.x >> 5) << 26) | (r.y >> 6)) * 0x1p-53;
    double x = u * t[2];
    int n = 1;
    while (n < leaves) {
        const double l = t[4 * n], rs = t[4 * n + 2];
        if (x < l || rs == 0.0) n = 2 * n;
        else { x -= l; n = 2 * n + 1; }
    }
    return n - leaves;
}

// w = (N P(i))^-beta / (N min P)^-beta of a row with priority p, P = p / sum: the reference buffer's weight, in fp64
__device__ __forceinline__ float per_weight(const double* t, int leaves, int n_valid, int row, double beta)
{
    const double s = t[2], N = (double)n_valid;
    return (float)(pow(N * (t[2 * (leaves + row)] / s), -beta) / pow(N * (t[3] / s), -beta));
}

// One CTA (every thread calls it): rows[j] gets priority (td[j] + 1e-5)^alpha, j in batch order — a leaf is written by
// the last j that holds its row, so the later of two equal rows wins — then the ancestors of the n leaves level by level,
// each node left + right and fmin(left, right).  Two rows that share an ancestor write it twice with the same value.
__device__ __forceinline__ void per_reprioritise(double* t, int leaves, const int* rows, const float* td, int n, double alpha)
{
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const int r = rows[j];
        bool last = true;
        for (int q = j + 1; q < n; ++q) last &= rows[q] != r;
        if (last) {
            const double p = pow((double)td[j] + 1e-5, alpha);
            t[2 * (leaves + r)] = p;
            t[2 * (leaves + r) + 1] = p;
        }
    }
    __syncthreads();
    for (int sh = 1; (leaves >> sh) >= 1; ++sh) {
        for (int j = threadIdx.x; j < n; j += blockDim.x) {
            const int v = (leaves + rows[j]) >> sh;
            t[2 * v] = t[4 * v] + t[4 * v + 2];
            t[2 * v + 1] = fmin(t[4 * v + 1], t[4 * v + 3]);
        }
        __syncthreads();
    }
}
