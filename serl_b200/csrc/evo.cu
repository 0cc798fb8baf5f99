// K2-K5 — neuro-evolution kernels over the flat [pop, P] fp32 genome matrix (sm_90a).
//
//   K2 ssne_select_kernel    rank by fitness + 3-way tournaments        base/core/mod_neuro_evo.py:460-461, :40-47
//   K3 ssne_clone_kernel     genome row copies (elitism)                 :371-376, :489-493
//   K4 ssne_crossover_kernel clone two parents into a pair of slots, then the ordered row / element copies
//                            of crossover_inplace                        :516-523, :61-93
//   K5 ssne_mutate_kernel    ordered point mutations of mutate_inplace   :329-369
//
// Every random draw is made on the host in the reference's order (stdlib `random` / legacy np.random streams,
// serl_b200/evo.py) and shipped as compact op lists; the kernels only apply them, in fp32 with the same
// rounding sequence torch uses for 0-d tensor (x) python-scalar expressions (no FMA contraction).
// HBM-bound integer/float copy work: coalesced row copies, one CTA per genome (pair).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/serl_b200.h"
#include "common.cuh"

// ---- K2 ------------------------------------------------------------------------------------------------
// rank: descending fitness; equal fitness -> larger index first (== np.argsort(kind='stable')[::-1]);
// NaN sorts as +inf like numpy (last ascending, first after the reversal).
__global__ void ssne_select_kernel(const double* __restrict__ fitness, int pop, const int* __restrict__ draws, int n_off,
                                   int* __restrict__ index_rank, int* __restrict__ offs_raw)
{
    extern __shared__ int s_rank[];
    for (int i = threadIdx.x; i < pop; i += blockDim.x) {
        const double fi = fitness[i];
        const bool ni = fi != fi;
        int pos = 0;
        for (int j = 0; j < pop; ++j) {
            const double fj = fitness[j];
            const bool nj = fj != fj;
            bool before;   // j ranks before i
            if (ni || nj) before = (nj && !ni) || (nj && ni && j > i);
            else before = (fj > fi) || (fj == fi && j > i);
            pos += before ? 1 : 0;
        }
        s_rank[pos] = i;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < pop; i += blockDim.x) index_rank[i] = s_rank[i];
    for (int s = threadIdx.x; s < n_off; s += blockDim.x) {
        int w = draws[3 * s];
        w = min(w, draws[3 * s + 1]);
        w = min(w, draws[3 * s + 2]);
        offs_raw[s] = s_rank[w];
    }
}

// ---- K3 ------------------------------------------------------------------------------------------------
__global__ void ssne_clone_kernel(float* __restrict__ W, int P, const int* __restrict__ pairs, int n)
{
    const int op = blockIdx.y;
    if (op >= n) return;
    const int src = pairs[2 * op], dst = pairs[2 * op + 1];
    if (src == dst) return;
    const float* s = W + (size_t)src * P;
    float* d = W + (size_t)dst * P;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) d[i] = s[i];
}

// ---- K4 ------------------------------------------------------------------------------------------------
// desc[pair] = {g1, g2, src1, src2, op_begin, op_count}; ops[k] = {offset, len, dir}; dir 0: g1[..] = g2[..], 1: g2[..] = g1[..].
// A thread always owns the same columns of a row, so ops on the same row stay ordered without barriers.
__global__ void ssne_crossover_kernel(float* __restrict__ W, int P, const int* __restrict__ desc, const int* __restrict__ ops)
{
    const int* d = desc + 6 * blockIdx.x;
    float* g1 = W + (size_t)d[0] * P;
    float* g2 = W + (size_t)d[1] * P;
    const float* s1 = W + (size_t)d[2] * P;
    const float* s2 = W + (size_t)d[3] * P;
    if (d[2] != d[0])
        for (int i = threadIdx.x; i < P; i += blockDim.x) g1[i] = s1[i];
    __syncthreads();                     // g1 == g2 (padded duplicate pair): second clone wins, as in the reference
    if (d[3] != d[1])
        for (int i = threadIdx.x; i < P; i += blockDim.x) g2[i] = s2[i];
    __syncthreads();
    const int* o = ops + 3 * (size_t)d[4];
    for (int k = 0; k < d[5]; ++k) {
        const int off = o[3 * k], len = o[3 * k + 1], dir = o[3 * k + 2];
        float* dst = dir ? g2 : g1;
        const float* src = dir ? g1 : g2;
        for (int c = threadIdx.x; c < len; c += blockDim.x) dst[off + c] = src[off + c];
    }
}

// ---- K5 ------------------------------------------------------------------------------------------------
// seg[s] = {actor, op_begin, op_count}: the ordered point mutations of one 2-D parameter of one actor.
// kind 0: w += z*(mag*w)   1: w += z*(10mag*w)   2: w = z ; then clamp to +-1e6   (mod_neuro_evo.py:360-369, :57-59)
__global__ void ssne_mutate_kernel(float* __restrict__ W, int P, const int* __restrict__ seg, int n_seg,
                                   const int* __restrict__ op_off, const int* __restrict__ op_kind, const float* __restrict__ op_z,
                                   float mag32, float super32)
{
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    float* g = W + (size_t)seg[3 * s] * P;
    const int b = seg[3 * s + 1], n = seg[3 * s + 2];
    for (int k = b; k < b + n; ++k) {
        const int off = op_off[k];
        const int kind = op_kind[k];
        const float z = op_z[k];
        float w = g[off];
        if (kind == 2) w = z;
        else w = __fadd_rn(w, __fmul_rn(z, __fmul_rn(kind == 1 ? super32 : mag32, w)));
        w = fminf(fmaxf(w, -1000000.0f), 1000000.0f);
        g[off] = w;
    }
}

// ---- C-ABI ---------------------------------------------------------------------------------------------
extern "C" int serl_ssne_select(const double* d_fitness, int32_t pop, const int32_t* d_draws, int32_t n_off,
                                int32_t* d_index_rank, int32_t* d_offsprings_raw, void* stream)
{
    if (!d_fitness || !d_index_rank || (n_off > 0 && (!d_draws || !d_offsprings_raw))) return serl_fail(SERL_ERR_ARG, "serl_ssne_select: null pointer");
    if (pop <= 0 || pop > 16384 || n_off < 0) return serl_fail(SERL_ERR_ARG, "serl_ssne_select: 0 < pop <= 16384 required");
    return serl_launch("ssne_select_kernel", ssne_select_kernel, 1, 1024, pop * sizeof(int), (cudaStream_t)stream, d_fitness, pop, d_draws,
                       n_off, d_index_rank, d_offsprings_raw);
}

extern "C" int serl_ssne_clone(float* d_weights, int32_t pop, int32_t P, const int32_t* d_pairs, int32_t n, void* stream)
{
    if (n == 0) return SERL_OK;
    if (!d_weights || !d_pairs || pop <= 0 || P <= 0 || n < 0) return serl_fail(SERL_ERR_ARG, "serl_ssne_clone: bad argument");
    dim3 grid((P + 1023) / 1024 > 8 ? 8 : (P + 1023) / 1024, n);
    return serl_launch("ssne_clone_kernel", ssne_clone_kernel, grid, 256, 0, (cudaStream_t)stream, d_weights, P, d_pairs, n);
}

extern "C" int serl_ssne_crossover(float* d_weights, int32_t pop, int32_t P, const int32_t* d_pair_desc, int32_t n_pairs,
                                   const int32_t* d_ops, void* stream)
{
    if (n_pairs == 0) return SERL_OK;
    if (!d_weights || !d_pair_desc || !d_ops || pop <= 0 || P <= 0 || n_pairs < 0) return serl_fail(SERL_ERR_ARG, "serl_ssne_crossover: bad argument");
    return serl_launch("ssne_crossover_kernel", ssne_crossover_kernel, n_pairs, 256, 0, (cudaStream_t)stream, d_weights, P, d_pair_desc, d_ops);
}

extern "C" int serl_ssne_mutate(float* d_weights, int32_t pop, int32_t P, const int32_t* d_seg, int32_t n_seg,
                                const int32_t* d_op_off, const int32_t* d_op_kind, const float* d_op_z,
                                float mag32, float super32, void* stream)
{
    if (n_seg == 0) return SERL_OK;
    if (!d_weights || !d_seg || !d_op_off || !d_op_kind || !d_op_z || pop <= 0 || P <= 0 || n_seg < 0)
        return serl_fail(SERL_ERR_ARG, "serl_ssne_mutate: bad argument");
    return serl_launch("ssne_mutate_kernel", ssne_mutate_kernel, (n_seg + 63) / 64, 64, 0, (cudaStream_t)stream, d_weights, P, d_seg, n_seg,
                       d_op_off, d_op_kind, d_op_z, mag32, super32);
}
