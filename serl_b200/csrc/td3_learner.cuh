// K7's learner (csrc/td3.cu): one TD3 learner's n_steps on one thread-block cluster (td3_learner), its launch arguments,
// scratch layout, the host-side checks of its descriptors and the packing of a serl_td3_learn call's learners for one
// launch.  td3.cu instantiates it in the solo, group, mixed and PER kernels; td3_group_per.cu in the group launch of
// prioritized and uniform learners.  The kernels of each translation unit are compiled from this one source, so a
// learner's code (and its bits) is the same in every launch that runs it.
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/serl_td3.h"
#include "../../include/serl_td3_per.h"
#include "common.cuh"
#include "per.cuh"

namespace {

constexpr int NT = 256;
constexpr int SD = 7, AD = 3, CI = SD + AD, CH = SERL_TD3_CRITIC_HIDDEN, COLS = 19;
constexpr int CP = CI * CH + 3 * CH + CH * CH + 3 * CH + CH + 1;     // floats per critic head (5185)
constexpr int CHUNK = 64;                                            // gradient-norm partial: 64 consecutive elements
constexpr float LN_EPS = 1e-6f;                                      // core/mod_utils.py LayerNorm: added to the std
enum { ACT_NONE = 3 };

struct Args {
    float* st;
    const float* replay; int cols; int n_valid;
    int B, n_steps, h, L, act, Pa;
    long long it0, tc0, ta0;
    float gamma, tau, noise_sd, noise_clip, lt, ls, eps_sd, max_norm;
    double lr;
    int freq, champion;
    unsigned long long seed;
    const int* idx_in;
    float* losses; int* rec_idx; float* rec_noise; float* rec_caps; int* status;
    float* ws;
};

// what prioritized replay adds (serl_td3_per_desc): the priority tree and its parameters, the optional records
struct Per {
    double* tree; int leaves, n_valid;
    double alpha, beta0, beta_frames;
    float *rec_w, *rec_td;
};

// scratch layout (floats); per block of a net: Z (linear output, LN blocks), A (activation output), dU (gradient at the
// block's LN / activation output), dZ (gradient at the linear output), row mean, row std — for up to 2B rows
struct Lay {
    size_t act_a, act_c, xt, xs, xp, xa, rdy, ga, gc, part, total;
    int stride_a, stride_c;
};
__host__ __device__ inline Lay layout(int B, int h, int L, int Pa)
{
    Lay l;
    size_t o = 0;
    const int R = 2 * B;
    l.stride_a = 4 * R * h + 2 * R;
    l.act_a = o; o += (size_t)(L + 2) * l.stride_a;
    l.stride_c = 4 * R * CH + 2 * R;
    l.act_c = o; o += 3 * (size_t)l.stride_c;
    l.xt = o; o += (size_t)B * CI;            // critic-target input (s', a')
    l.xs = o; o += (size_t)B * CI;            // critic input (s, a)
    l.xp = o; o += (size_t)B * CI;            // actor-loss critic input (s, pi(s))
    l.xa = o; o += (size_t)2 * B * SD;        // actor input: s, then s + U * eps_sd
    l.rdy = o; o += (size_t)4 * B;            // reward, done, target y, Q1(s, pi(s))
    l.ga = o; o += Pa;
    l.gc = o; o += 2 * CP;
    l.part = o; o += ((Pa > 2 * CP ? Pa : 2 * CP) + CHUNK - 1) / CHUNK;
    l.total = o;
    return l;
}

// data written inside the launch by any CTA of the cluster: a plain (L1-cached) load is safe after the cluster barrier's
// acquire, and it keeps the rows a warp re-reads (a layer's inputs, broadcast weight rows) in L1
__device__ __forceinline__ float ld(const float* p) { return *p; }

template <int CS>
__device__ __forceinline__ void csync()
{
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

__device__ __forceinline__ float act_f(int a, float v)
{
    switch (a) {
    case SERL_ACT_TANH: return tanhf(v);
    case SERL_ACT_ELU: return v > 0.f ? v : expm1f(v);
    case SERL_ACT_LEAKY_RELU: return v > 0.f ? v : 0.01f * v;
    default: return v;
    }
}
// derivative from the activation's OUTPUT y (ELU: exp(u) = y + 1 for u <= 0)
__device__ __forceinline__ float act_d(int a, float y)
{
    switch (a) {
    case SERL_ACT_TANH: return 1.f - y * y;
    case SERL_ACT_ELU: return y > 0.f ? 1.f : y + 1.f;
    case SERL_ACT_LEAKY_RELU: return y > 0.f ? 1.f : 0.01f;
    default: return 1.f;
    }
}

__device__ __forceinline__ float warp_sum(float v)
{
#pragma unroll
    for (int m = 16; m; m >>= 1) v += __shfl_xor_sync(0xffffffffu, v, m);
    return v;
}

enum { TAG_INDEX = 0, TAG_NOISE = 1, TAG_CAPS = 2 };      // TAG_CAPS + 1 too; PER_TAG (per.cuh) follows
__device__ __forceinline__ uint4 draw(const Args& a, long long it, int row, int tag)
{
    return philox(make_uint4((uint32_t)it, (uint32_t)((unsigned long long)it >> 32), (uint32_t)row, (uint32_t)tag),
                  make_uint2((uint32_t)a.seed, (uint32_t)(a.seed >> 32)));
}
__device__ __forceinline__ float unit(uint32_t x) { return (float)(x >> 8) * 0x1p-24f; }          // [0, 1)

// one layer block of a net: Linear(in, out) [LayerNorm(out)] activation; parameters at `off`: W [out][in], b, gamma, beta
struct Blk { int in, out, off; bool ln; int act; };

struct Net {
    const float* P; float* G; int hs;        // parameters, gradients, floats between heads
    float* ws; int stride; int cap; int W;   // activations: per block `stride` floats, `cap` rows of <= W values
    bool critic; int h, L, act;
    __device__ Blk blk(int k) const
    {
        if (critic) {
            if (k == 0) return {CI, CH, 0, true, act};
            if (k == 1) return {CH, CH, CI * CH + 3 * CH, true, act};
            return {CH, 1, CI * CH + 3 * CH + CH * CH + 3 * CH, false, ACT_NONE};
        }
        if (k == 0) return {SD, h, 0, false, act};
        const int base = SD * h + h;
        if (k <= L) return {h, h, base + (k - 1) * (h * h + 3 * h), true, act};
        return {h, AD, base + L * (h * h + 3 * h), false, SERL_ACT_TANH};
    }
    __device__ int last() const { return critic ? 2 : L + 1; }
    __device__ float* Z(int k) const { return ws + (size_t)k * stride; }
    __device__ float* A(int k) const { return Z(k) + cap * W; }
    __device__ float* dU(int k) const { return Z(k) + 2 * cap * W; }
    __device__ float* dZ(int k) const { return blk(k).ln ? Z(k) + 3 * cap * W : dU(k); }
    __device__ float* mu(int k) const { return Z(k) + 4 * cap * W; }
    __device__ float* sd(int k) const { return mu(k) + cap; }
};

// the CTA's rank in its cluster: blockIdx.x in a solo launch (the grid is one cluster), %cluster_ctarank in a group
// launch (G: cluster g of the grid runs learner g)
template <bool G> __device__ __forceinline__ int crank()
{
    if (!G) return blockIdx.x;
    unsigned r;
    asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return (int)r;
}
template <int CS, bool G> __device__ __forceinline__ int gt() { return crank<G>() * NT + threadIdx.x; }
template <int CS, bool G> __device__ __forceinline__ int gw() { return (crank<G>() * NT + threadIdx.x) >> 5; }
__host__ __device__ constexpr int GN(int CS) { return CS * NT; }

// Linear part of block k for nh heads x rows rows (row rr = head * rows + r).  Input: X (row stride xs, shared by the
// heads) for block 0, else the previous block's A.  LayerNorm blocks store Z; other blocks store act(.) in A, except the
// last block, whose value goes to epi(head, r, o, value).
template <int CS, bool G, class Epi>
__device__ void fwd_lin(const Net& n, int k, int nh, int rows, const float* X, int xs, Epi epi)
{
    const Blk b = n.blk(k);
    const int per = rows * b.out, total = nh * per;
    for (int e = gt<CS, G>(); e < total; e += GN(CS)) {
        const int hd = e / per, rem = e - hd * per, o = rem / rows, r = rem - o * rows;      // a warp shares a weight row
        const float* w = n.P + hd * n.hs + b.off + o * b.in;
        const float* x = k == 0 ? X + r * xs : n.A(k - 1) + (size_t)(hd * rows + r) * b.in;
        float acc = 0.f;
        for (int i = 0; i < b.in; ++i) acc = fmaf(ld(x + i), ld(w + i), acc);
        acc += ld(n.P + hd * n.hs + b.off + b.out * b.in + o);
        const int rr = hd * rows + r;
        if (b.ln) n.Z(k)[rr * b.out + o] = acc;
        else if (k < n.last()) n.A(k)[rr * b.out + o] = act_f(b.act, acc);
        else epi(hd, r, o, acc);
    }
}
template <int CS, bool G>
__device__ void fwd_lin(const Net& n, int k, int nh, int rows, const float* X, int xs)
{
    fwd_lin<CS, G>(n, k, nh, rows, X, xs, [](int, int, int, float) {});
}

// LayerNorm + activation of block k, one warp per row: y = gamma * (z - mean) / (std + eps) + beta, Bessel-corrected std
template <int CS, bool G>
__device__ void fwd_ln(const Net& n, int k, int nh, int rows)
{
    const Blk b = n.blk(k);
    const int out = b.out, lane = threadIdx.x & 31;
    for (int rr = gw<CS, G>(); rr < nh * rows; rr += GN(CS) / 32) {
        const int hd = rr / rows;
        const float* z = n.Z(k) + rr * out;
        const float* g = n.P + hd * n.hs + b.off + out * b.in + out;
        float s = 0.f;
        for (int o = lane; o < out; o += 32) s += ld(z + o);
        const float mean = warp_sum(s) / (float)out;
        float q = 0.f;
        for (int o = lane; o < out; o += 32) { const float c = ld(z + o) - mean; q = fmaf(c, c, q); }
        const float sd = sqrtf(warp_sum(q) / (float)(out - 1)), rs = sd + LN_EPS;
        for (int o = lane; o < out; o += 32)
            n.A(k)[rr * out + o] = act_f(b.act, ld(g + o) * (ld(z + o) - mean) / rs + ld(g + out + o));
        if (lane == 0) { n.mu(k)[rr] = mean; n.sd(k)[rr] = sd; }
    }
}

// LayerNorm backward of block k, one warp per row: dU (at the LN output) -> dZ (at the linear output); out <= 32 * NJ
template <int CS, bool G, int NJ = 4>
__device__ void bwd_ln(const Net& n, int k, int nh, int rows)
{
    const Blk b = n.blk(k);
    const int out = b.out, lane = threadIdx.x & 31;
    for (int rr = gw<CS, G>(); rr < nh * rows; rr += GN(CS) / 32) {
        const int hd = rr / rows;
        const float* z = n.Z(k) + rr * out;
        const float* du = n.dU(k) + rr * out;
        const float* g = n.P + hd * n.hs + b.off + out * b.in + out;
        const float mean = ld(n.mu(k) + rr), sd = ld(n.sd(k) + rr), rs = sd + LN_EPS;
        float s = 0.f;
        for (int o = lane; o < out; o += 32) s += ld(du + o) * ld(g + o) * (ld(z + o) - mean);
        const float kq = warp_sum(s) / (rs * rs) / ((float)(out - 1) * sd);     // d std / d c_o = c_o / ((n-1) std)
        float gc[NJ];
        float t = 0.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int o = lane + 32 * j;
            gc[j] = 0.f;
            if (o < out) { gc[j] = ld(du + o) * ld(g + o) / rs - kq * (ld(z + o) - mean); t += gc[j]; }
        }
        const float m = warp_sum(t) / (float)out;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int o = lane + 32 * j;
            if (o < out) n.dZ(k)[rr * out + o] = gc[j] - m;
        }
    }
}

// Gradient of block k's bias (v < out), LayerNorm gamma (out <= v < 2 out) or beta (v >= 2 out) for head hd, summed over
// the rows in row order: the sums of bwd_lin's last 3 out elements, for bwd_wide (bwd_lin keeps its own copy inline, which
// keeps the narrow kernel's code as it was)
__device__ __forceinline__ float vec_grad(const Net& n, const Blk& b, int k, int hd, int rows, int v)
{
    const int out = b.out;
    float s = 0.f;
    if (v < out) {
        const float* dzh = n.dZ(k) + (size_t)hd * rows * out;
        for (int r = 0; r < rows; ++r) s += ld(dzh + r * out + v);
    } else {
        const int o = v - out;
        const float* du = n.dU(k) + (size_t)hd * rows * out;
        if (o < out) {             // gamma: sum of dU * (z - mean) / (std + eps)
            const float* z = n.Z(k) + (size_t)hd * rows * out;
            for (int r = 0; r < rows; ++r) {
                const int rr = hd * rows + r;
                s = fmaf(ld(du + r * out + o) / (ld(n.sd(k) + rr) + LN_EPS), ld(z + r * out + o) - ld(n.mu(k) + rr), s);
            }
        } else {                   // beta
            for (int r = 0; r < rows; ++r) s += ld(du + r * out + o - out);
        }
    }
    return s;
}

// Block k backward: its parameter gradients (summed over rows in row order) and, if dx, dU of block k-1 =
// (dZ_k W_k) * act'(A_{k-1}); X / xs is block 0's input.  params = false: only dU of block k-1 (input gradients).
template <int CS, bool G>
__device__ void bwd_lin(const Net& n, int k, int nh, int rows, const float* X, int xs, bool params, bool dx)
{
    const Blk b = n.blk(k);
    const int in = b.in, out = b.out;
    const int np = params ? out * in + out + (b.ln ? 2 * out : 0) : 0;
    const int tp = nh * np, total = tp + (dx ? nh * rows * in : 0);
    const float* dz = n.dZ(k);
    for (int e = gt<CS, G>(); e < total; e += GN(CS)) {
        if (e < tp) {
            const int hd = e / np, j = e - hd * np;
            const float* dzh = dz + (size_t)hd * rows * out;
            float s = 0.f;
            if (j < out * in) {
                const int o = j / in, i = j - o * in;
                if (k == 0) for (int r = 0; r < rows; ++r) s = fmaf(ld(dzh + r * out + o), ld(X + r * xs + i), s);
                else {
                    const float* x = n.A(k - 1) + (size_t)hd * rows * in + i;
                    for (int r = 0; r < rows; ++r) s = fmaf(ld(dzh + r * out + o), ld(x + r * in), s);
                }
            } else if (j < out * in + out) {
                const int o = j - out * in;
                for (int r = 0; r < rows; ++r) s += ld(dzh + r * out + o);
            } else {
                const int o = j - out * in - out;
                const float* du = n.dU(k) + (size_t)hd * rows * out;
                if (o < out) {             // gamma: sum of dU * (z - mean) / (std + eps)
                    const float* z = n.Z(k) + (size_t)hd * rows * out;
                    for (int r = 0; r < rows; ++r) {
                        const int rr = hd * rows + r;
                        s = fmaf(ld(du + r * out + o) / (ld(n.sd(k) + rr) + LN_EPS), ld(z + r * out + o) - ld(n.mu(k) + rr), s);
                    }
                } else {                   // beta
                    for (int r = 0; r < rows; ++r) s += ld(du + r * out + o - out);
                }
            }
            n.G[hd * n.hs + b.off + j] = s;
        } else {
            const int e2 = e - tp, rr = e2 / in, i = e2 - rr * in, hd = rr / rows;
            const float* w = n.P + hd * n.hs + b.off + i;
            const float* d = dz + rr * out;
            float s = 0.f;
            for (int o = 0; o < out; ++o) s = fmaf(ld(d + o), ld(w + o * in), s);
            n.dU(k - 1)[rr * in + i] = s * act_d(n.blk(k - 1).act, ld(n.A(k - 1) + rr * in + i));
        }
    }
}

// ---- the wide actor (128 < h <= SERL_TD3_MAX_HIDDEN): its h x h blocks 1..L as tiled phases ----------------------------
// A tile is TM x TN outputs of C[m][n] = sum_k A(m, k) B(n, k) on one CTA: thread (ty, tx) = (tid / 16, tid % 16) holds
// the outputs m0 + ty + 16 i, n0 + tx + 16 j in registers, and the operands pass through shared memory in K-slabs of KS,
// the next slab loaded into registers while the current one is multiplied.  Every output is still one thread's fmaf
// chain from k = 0 upward, the order of fwd_lin / bwd_lin (slab padding adds fmaf(0, 0, acc) = acc), and the tile shapes
// do not depend on CS: the bits depend on neither the cluster size nor the launch split.  A phase deals its tiles
// round-robin over the cluster's CTAs.  AK (BK): A (B) is contiguous in k in memory, else in m (n) — the loading order
// that keeps a warp's global loads coalesced and its shared-memory stores free of bank conflicts.
constexpr int KS = 32;
constexpr int FWD_TM = 32, FWD_TN = 64;        // forward: rows x output neurons
constexpr int WG_TM = 64, WG_TN = 64;          // weight gradient: output x input neurons, summed over the rows
constexpr int DG_TM = 32, DG_TN = 64;          // input gradient: rows x input neurons, summed over the output neurons
__host__ __device__ constexpr int tile_floats(int tm, int tn) { return KS * (tm + 1) + KS * (tn + 1); }
__host__ __device__ constexpr int cmax(int x, int y) { return x > y ? x : y; }
constexpr size_t WIDE_SMEM = sizeof(float) * cmax(tile_floats(FWD_TM, FWD_TN), cmax(tile_floats(WG_TM, WG_TN), tile_floats(DG_TM, DG_TN)));
// the tiles' shared memory: static, and allocated only in the kernels that reach this function (an extern __shared__
// array would pad the static shared memory of every kernel of the translation unit to 16 bytes)
__device__ __forceinline__ float* tile_smem()
{
    __shared__ float buf[WIDE_SMEM / sizeof(float)];
    return buf;
}

template <int TM, int TN, bool AK, bool BK, class LA, class LB, class Epi>
__device__ __forceinline__ void tile(float* sm, int m0, int n0, int M, int N, int K, LA la, LB lb, Epi epi)
{
    constexpr int MI = TM / 16, NJ = TN / 16, QA = TM * KS / NT, QB = TN * KS / NT;
    static_assert(TM % 16 == 0 && TN % 16 == 0 && QA * NT == TM * KS && QB * NT == TN * KS, "tile shape");
    float* As = sm;                    // [KS][TM + 1]
    float* Bs = sm + KS * (TM + 1);    // [KS][TN + 1]
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
    float acc[MI][NJ], ra[QA], rb[QB];
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[i][j] = 0.f;
    const auto fetch = [&](int k0) {
#pragma unroll
        for (int q = 0; q < QA; ++q) {
            const int e = threadIdx.x + q * NT, m = AK ? e / KS : e % TM, k = AK ? e % KS : e / TM;
            ra[q] = m0 + m < M && k0 + k < K ? la(m0 + m, k0 + k) : 0.f;
        }
#pragma unroll
        for (int q = 0; q < QB; ++q) {
            const int e = threadIdx.x + q * NT, n = BK ? e / KS : e % TN, k = BK ? e % KS : e / TN;
            rb[q] = n0 + n < N && k0 + k < K ? lb(n0 + n, k0 + k) : 0.f;
        }
    };
    fetch(0);
    for (int k0 = 0; k0 < K; k0 += KS) {
        __syncthreads();               // the previous slab (or tile) has been read
#pragma unroll
        for (int q = 0; q < QA; ++q) {
            const int e = threadIdx.x + q * NT, m = AK ? e / KS : e % TM, k = AK ? e % KS : e / TM;
            As[k * (TM + 1) + m] = ra[q];
        }
#pragma unroll
        for (int q = 0; q < QB; ++q) {
            const int e = threadIdx.x + q * NT, n = BK ? e / KS : e % TN, k = BK ? e % KS : e / TN;
            Bs[k * (TN + 1) + n] = rb[q];
        }
        __syncthreads();
        if (k0 + KS < K) fetch(k0 + KS);
#pragma unroll
        for (int k = 0; k < KS; ++k) {
            float av[MI], bv[NJ];
#pragma unroll
            for (int i = 0; i < MI; ++i) av[i] = As[k * (TM + 1) + ty + 16 * i];
#pragma unroll
            for (int j = 0; j < NJ; ++j) bv[j] = Bs[k * (TN + 1) + tx + 16 * j];
#pragma unroll
            for (int i = 0; i < MI; ++i)
#pragma unroll
                for (int j = 0; j < NJ; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
    }
#pragma unroll
    for (int i = 0; i < MI; ++i)
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const int m = m0 + ty + 16 * i, n = n0 + tx + 16 * j;
            if (m < M && n < N) epi(m, n, acc[i][j]);
        }
}

// forward of the wide actor's block k (1..L, h x h, LayerNorm): Z[r][o] = sum_i A_{k-1}[r][i] W[o][i] + b[o]
template <int CS, bool G>
__device__ void fwd_wide(const Net& n, int k, int rows, float* sm)
{
    const Blk b = n.blk(k);
    const int in = b.in, out = b.out;
    const float *x = n.A(k - 1), *w = n.P + b.off, *bias = w + out * in;
    float* z = n.Z(k);
    const int tn = (out + FWD_TN - 1) / FWD_TN, nt = (rows + FWD_TM - 1) / FWD_TM * tn;
    for (int t = crank<G>(); t < nt; t += CS)
        tile<FWD_TM, FWD_TN, true, true>(sm, t / tn * FWD_TM, t % tn * FWD_TN, rows, out, in,
            [&](int r, int i) { return ld(x + r * in + i); },
            [&](int o, int i) { return ld(w + o * in + i); },
            [&](int r, int o, float acc) { z[r * out + o] = acc + ld(bias + o); });
}

// backward of the wide actor's block k (1..L): the weight gradient G[o][i] = sum_r dZ[r][o] A_{k-1}[r][i] and the input
// gradient dU_{k-1}[r][i] = (sum_o dZ[r][o] W[o][i]) * act'(A_{k-1}[r][i]) as tiles, then the bias, gamma and beta
// gradients one per thread (vec_grad, as bwd_lin)
template <int CS, bool G>
__device__ void bwd_wide(const Net& n, int k, int rows, float* sm)
{
    const Blk b = n.blk(k);
    const int in = b.in, out = b.out, pact = n.blk(k - 1).act;
    const float *dz = n.dZ(k), *x = n.A(k - 1), *w = n.P + b.off;
    float *g = n.G + b.off, *du = n.dU(k - 1);
    const int wn = (in + WG_TN - 1) / WG_TN, nw = (out + WG_TM - 1) / WG_TM * wn;
    const int dn = (in + DG_TN - 1) / DG_TN, nd = (rows + DG_TM - 1) / DG_TM * dn;
    for (int t = crank<G>(); t < nw + nd; t += CS) {
        if (t < nw)
            tile<WG_TM, WG_TN, false, false>(sm, t / wn * WG_TM, t % wn * WG_TN, out, in, rows,
                [&](int o, int r) { return ld(dz + r * out + o); },
                [&](int i, int r) { return ld(x + r * in + i); },
                [&](int o, int i, float s) { g[o * in + i] = s; });
        else
            tile<DG_TM, DG_TN, true, false>(sm, (t - nw) / dn * DG_TM, (t - nw) % dn * DG_TN, rows, in, out,
                [&](int r, int o) { return ld(dz + r * out + o); },
                [&](int i, int o) { return ld(w + o * in + i); },
                [&](int r, int i, float s) { du[r * in + i] = s * act_d(pact, ld(x + r * in + i)); });
    }
    for (int v = gt<CS, G>(); v < 3 * out; v += GN(CS)) g[out * in + v] = vec_grad(n, b, k, 0, rows, v);
}

// sum of squares of CHUNK-element slices of the gradient g[0, count)
template <int CS, bool G>
__device__ void norm_partials(const float* g, int count, float* part)
{
    const int nc = (count + CHUNK - 1) / CHUNK;
    for (int c = gt<CS, G>(); c < nc; c += GN(CS)) {
        float s = 0.f;
        const int end = min(count, (c + 1) * CHUNK);
        for (int i = c * CHUNK; i < end; ++i) { const float v = ld(g + i); s = fmaf(v, v, s); }
        part[c] = s;
    }
}

// clip_grad_norm_ (coef = min(1, max / (|g| + 1e-6))) + the torch Adam step (foreach formula, bias corrections)
// + optionally the Polyak update of the target: tgt <- tgt * (1 - tau) + tau * p.  Which product of these two sums of
// two products the compiler fuses into an FFMA depends on where the operands live (tau is a kernel parameter in
// td3_kernel, a register in td3_group_kernel), so the group kernel (G) spells out the fusion td3_kernel's code has, and
// gives td3_kernel's bits; td3_kernel keeps its source and its code.  td3_per_kernel's code fuses the Polyak update the
// other way (tau * p + (tgt * (1 - tau))); PF: a group launch's PER learner spells out that fusion, for its bits.
template <int CS, bool G, bool PF = false>
__device__ void adam(float* p, float* m, float* v, float* tgt, const float* g, int count, const float* part, long long t,
                     const Args& a, bool soft, float* s_coef)
{
    if (threadIdx.x < 32) {           // the partials in a fixed order: lane l sums l, l + 32, ..., then a fixed shuffle tree
        const int nc = (count + CHUNK - 1) / CHUNK;
        float s = 0.f;
        for (int c = threadIdx.x; c < nc; c += 32) s += ld(part + c);
        s = warp_sum(s);
        if (threadIdx.x == 0) *s_coef = fminf(a.max_norm / (sqrtf(s) + 1e-6f), 1.f);
    }
    __syncthreads();
    const float coef = *s_coef;
    const float step = (float)(-a.lr / (1.0 - pow(0.9, (double)t)));
    const float bc2 = (float)sqrt(1.0 - pow(0.999, (double)t));
    const float keep = (float)(1.0 - (double)a.tau);
    for (int i = gt<CS, G>(); i < count; i += GN(CS)) {
        const float gi = ld(g + i) * coef;
        float mi = ld(m + i), vi = ld(v + i);
        mi = mi + 0.1f * (gi - mi);                           // exp_avg.lerp_(grad, 1 - beta1)
        // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
        vi = G ? fmaf(vi, 0.999f, 0.001f * gi * gi) : vi * 0.999f + 0.001f * gi * gi;
        const float pi = ld(p + i) + step * (mi / (sqrtf(vi) / bc2 + 1e-8f));
        m[i] = mi; v[i] = vi; p[i] = pi;
        if (soft) tgt[i] = G ? (PF ? fmaf(pi, a.tau, ld(tgt + i) * keep) : fmaf(ld(tgt + i), keep, a.tau * pi))
                             : ld(tgt + i) * keep + a.tau * pi;
    }
}

// the step's batch (CTA 0): Floyd's sample of B distinct rows of [0, n_valid) — row j draws t_j uniform in
// [0, n - B + j] and keeps it unless an earlier row holds it, else takes n - B + j — then the gathered transitions, the
// clipped target-policy noise and the CAPS perturbation, written to the inputs of the step's networks.  PER: B rows drawn
// with replacement from the priority tree instead, and their importance weights (beta of the learner's critic step) in wt
template <bool PER = false>
__device__ void draw_batch(const Args& a, int k, long long it, int* pick, int* tdraw, float* Xt, float* Xs, float* Xp, float* Xa,
                           float* rw, float* dn, const Per* p = nullptr, float* wt = nullptr)
{
    const int B = a.B, n = a.n_valid, tid = threadIdx.x;
    if (a.idx_in) {
        for (int j = tid; j < B; j += NT) {
            int r = a.idx_in[(size_t)k * B + j];
            if (r < 0 || r >= n) { atomicOr(a.status, SERL_TD3_STATUS_INDEX); r = 0; }
            pick[j] = r;
        }
    } else if constexpr (PER) {
        for (int j = tid; j < B; j += NT) pick[j] = per_draw(p->tree, p->leaves, a.seed, it, j);
    } else {
        for (int j = tid; j < B; j += NT)
            tdraw[j] = (int)__umulhi(draw(a, it, j, TAG_INDEX).x, (uint32_t)(n - B + j + 1));
        __syncthreads();
        if (tid < 32) {
            for (int j = 0; j < B; ++j) {
                const int t = tdraw[j];
                bool hit = false;
                for (int q = tid; q < j; q += 32) hit |= pick[q] == t;
                hit = __any_sync(0xffffffffu, hit);
                if (tid == 0) pick[j] = hit ? n - B + j : t;
                __syncwarp();
            }
        }
    }
    __syncthreads();
    for (int j = tid; j < B; j += NT) {
        const float* row = a.replay + (size_t)pick[j] * a.cols;
        const uint4 zn = draw(a, it, j, TAG_NOISE), u0 = draw(a, it, j, TAG_CAPS), u1 = draw(a, it, j, TAG_CAPS + 1);
        float z[4];
#pragma unroll
        for (int q = 0; q < 2; ++q) {           // Box-Muller
            const uint32_t x = q ? zn.z : zn.x, y = q ? zn.w : zn.y;
            const float rad = sqrtf(-2.f * logf(((float)(x >> 8) + 1.f) * 0x1p-24f));
            float sn, cs;
            sincospif(2.f * unit(y), &sn, &cs);
            z[2 * q] = rad * cs; z[2 * q + 1] = rad * sn;
        }
        const float u[SD] = {unit(u0.x), unit(u0.y), unit(u0.z), unit(u0.w), unit(u1.x), unit(u1.y), unit(u1.z)};
#pragma unroll
        for (int i = 0; i < SD; ++i) {
            const float s = __ldg(row + i);
            Xs[j * CI + i] = s; Xp[j * CI + i] = s; Xa[j * SD + i] = s;
            Xa[(B + j) * SD + i] = s + u[i] * a.eps_sd;
            Xt[j * CI + i] = __ldg(row + SD + AD + i);
        }
#pragma unroll
        for (int i = 0; i < AD; ++i) {
            Xs[j * CI + SD + i] = __ldg(row + SD + i);
            const float nz = fminf(fmaxf(z[i] * a.noise_sd, -a.noise_clip), a.noise_clip);
            Xt[j * CI + SD + i] = nz;            // the target actor's epilogue adds its output
            if (a.rec_noise) a.rec_noise[((size_t)k * B + j) * AD + i] = nz;
        }
        rw[j] = __ldg(row + 2 * SD + AD);
        dn[j] = __ldg(row + 2 * SD + AD + 1);
        if (a.rec_idx) a.rec_idx[(size_t)k * B + j] = pick[j];
        if (a.rec_caps)
#pragma unroll
            for (int i = 0; i < SD; ++i) a.rec_caps[((size_t)k * B + j) * SD + i] = u[i];
        if constexpr (PER) {
            const double f = (double)(a.tc0 + k + 1);          // the learner's f-th sample (the reference's frame)
            const float w = per_weight(p->tree, p->leaves, p->n_valid, pick[j], fmin(1.0, p->beta0 + f * (1.0 - p->beta0) / p->beta_frames));
            wt[j] = w;
            if (p->rec_w) p->rec_w[(size_t)k * B + j] = w;
        }
    }
}

// One learner's n_steps on one cluster.  WIDE: the actor's hidden blocks take the tiled phases (fwd_wide / bwd_wide,
// WIDE_SMEM bytes of shared memory).  G: the cluster is one of a group launch's (crank).  PER: prioritized replay (p) —
// the batch from the priority tree, the critic loss weighted, and CTA 0 re-prioritises the batch's rows in the phase after
// the critic's forward pass; the weights live after the scratch layout (B floats).
template <int CS, bool WIDE, bool G, bool PER = false>
__device__ __forceinline__ void td3_learner(const Args a, const Per* p = nullptr)
{
    __shared__ int pick[SERL_TD3_MAX_BATCH], tdraw[SERL_TD3_MAX_BATCH];
    __shared__ float s_coef;
    float* const wide_sm = WIDE ? tile_smem() : nullptr;
    constexpr int NJ = WIDE ? (SERL_TD3_MAX_HIDDEN + 31) / 32 : 4;     // bwd_ln of the actor: h <= 32 * NJ
    const int B = a.B, Pa = a.Pa;
    const Lay l = layout(B, a.h, a.L, Pa);
    float* ws = a.ws;
    float *Xt = ws + l.xt, *Xs = ws + l.xs, *Xp = ws + l.xp, *Xa = ws + l.xa;
    float *rw = ws + l.rdy, *dn = rw + B, *yt = dn + B, *q1 = yt + B;
    float *part = ws + l.part, *ga = ws + l.ga, *gc = ws + l.gc;
    float *th_a = a.st, *tg_a = th_a + Pa, *m_a = tg_a + Pa, *v_a = m_a + Pa;
    float *th_c = v_a + Pa, *tg_c = th_c + 2 * CP, *m_c = tg_c + 2 * CP, *v_c = m_c + 2 * CP;
    const Net actor{th_a, ga, 0, ws + l.act_a, l.stride_a, 2 * B, a.h, false, a.h, a.L, a.act};
    Net actor_t = actor; actor_t.P = tg_a;
    const Net critic{th_c, gc, CP, ws + l.act_c, l.stride_c, 2 * B, CH, true, a.h, a.L, a.act};
    Net critic_t = critic; critic_t.P = tg_c;
    const int la = a.L + 1;
    const bool caps_s = a.ls != 0.f;
    const int ra = caps_s ? 2 * B : B;                 // actor rows: s, and s + U * eps when the smoothness term is on
    const float inv_b = 1.f / (float)B, mse_a = 2.f / (float)(B * AD);
    long long ta = a.ta0;
    for (int k = 0; k < a.n_steps; ++k) {
        const long long it = a.it0 + k;
        const bool actor_step = it % a.freq == 0;
        float td = 0.f, pg = __int_as_float(0x7fc00000);
        if constexpr (PER) {
            if (crank<G>() == 0) draw_batch<true>(a, k, it, pick, tdraw, Xt, Xs, Xp, Xa, rw, dn, p, ws + l.total);
        } else {
            if (crank<G>() == 0) draw_batch(a, k, it, pick, tdraw, Xt, Xs, Xp, Xa, rw, dn);
        }
        csync<CS>();
        // ---- target: a' = clamp(actor_target(s') + noise, +-1); y = r + gamma * min(q1', q2') * (1 - done)
        for (int kb = 0; kb <= la; ++kb) {
            if (WIDE && kb >= 1 && kb <= a.L) fwd_wide<CS, G>(actor_t, kb, B, wide_sm);
            else fwd_lin<CS, G>(actor_t, kb, 1, B, Xt, CI, [&](int, int r, int o, float v) {
                float* p = Xt + r * CI + SD + o;
                *p = fminf(fmaxf(ld(p) + tanhf(v), -1.f), 1.f);
            });
            csync<CS>();
            if (actor_t.blk(kb).ln) { fwd_ln<CS, G>(actor_t, kb, 1, B); csync<CS>(); }
        }
        for (int kb = 0; kb < 2; ++kb) {
            fwd_lin<CS, G>(critic_t, kb, 2, B, Xt, CI); csync<CS>();
            fwd_ln<CS, G>(critic_t, kb, 2, B); csync<CS>();
        }
        {
            const Blk b = critic_t.blk(2);
            for (int r = gt<CS, G>(); r < B; r += GN(CS)) {
                float q[2];
                for (int hd = 0; hd < 2; ++hd) {
                    const float* w = critic_t.P + hd * CP + b.off;
                    const float* x = critic_t.A(1) + (hd * B + r) * CH;
                    float acc = 0.f;
                    for (int i = 0; i < CH; ++i) acc = fmaf(ld(x + i), ld(w + i), acc);
                    q[hd] = acc + ld(w + CH);
                }
                yt[r] = ld(rw + r) + a.gamma * fminf(q[0], q[1]) * (1.f - ld(dn + r));
            }
        }
        csync<CS>();
        // ---- critic: forward on (s, a), loss mse(q1, y) + mse(q2, y), backward
        for (int kb = 0; kb < 2; ++kb) {
            fwd_lin<CS, G>(critic, kb, 2, B, Xs, CI); csync<CS>();
            fwd_ln<CS, G>(critic, kb, 2, B); csync<CS>();
        }
        fwd_lin<CS, G>(critic, 2, 2, B, Xs, CI, [&](int hd, int r, int, float v) {
            critic.A(2)[hd * B + r] = v;
            if constexpr (PER) critic.dU(2)[hd * B + r] = 2.f * inv_b * ld(ws + l.total + r) * (v - ld(yt + r));
            else critic.dU(2)[hd * B + r] = 2.f * inv_b * (v - ld(yt + r));
        });
        csync<CS>();
        if constexpr (PER) {
            if (crank<G>() == 0) {     // delta of the pre-update critic (in tdraw, which the tree's draw leaves unused)
                float* td_row = reinterpret_cast<float*>(tdraw);
                for (int r = threadIdx.x; r < B; r += NT) {
                    const float y = ld(yt + r);
                    td_row[r] = 0.5f * (fabsf(ld(critic.A(2) + r) - y) + fabsf(ld(critic.A(2) + B + r) - y));
                    if (p->rec_td) p->rec_td[(size_t)k * B + r] = td_row[r];
                }
                __syncthreads();
                per_reprioritise(p->tree, p->leaves, pick, td_row, B, p->alpha);
            }
        }
        bwd_lin<CS, G>(critic, 2, 2, B, Xs, CI, true, true); csync<CS>();
        bwd_ln<CS, G>(critic, 1, 2, B); csync<CS>();
        bwd_lin<CS, G>(critic, 1, 2, B, Xs, CI, true, true); csync<CS>();
        bwd_ln<CS, G>(critic, 0, 2, B); csync<CS>();
        bwd_lin<CS, G>(critic, 0, 2, B, Xs, CI, true, false);
        if (gt<CS, G>() == 0) {
            float s1 = 0.f, s2 = 0.f;
            for (int r = 0; r < B; ++r) {
                const float y = ld(yt + r), d1 = ld(critic.A(2) + r) - y, d2 = ld(critic.A(2) + B + r) - y;
                if constexpr (PER) {
                    const float w = ld(ws + l.total + r);
                    s1 = fmaf(w * d1, d1, s1); s2 = fmaf(w * d2, d2, s2);
                } else {
                    s1 = fmaf(d1, d1, s1); s2 = fmaf(d2, d2, s2);
                }
            }
            td = s1 / (float)B + s2 / (float)B;
        }
        csync<CS>();
        norm_partials<CS, G>(gc, 2 * CP, part); csync<CS>();
        adam<CS, G, G && PER>(th_c, m_c, v_c, tg_c, gc, 2 * CP, part, a.tc0 + k + 1, a, actor_step, &s_coef);
        csync<CS>();
        // ---- actor: -mean(Q1(s, pi(s))) + CAPS terms through the updated critic
        if (actor_step) {
            for (int kb = 0; kb <= la; ++kb) {
                if (WIDE && kb >= 1 && kb <= a.L) fwd_wide<CS, G>(actor, kb, ra, wide_sm);
                else fwd_lin<CS, G>(actor, kb, 1, ra, Xa, SD, [&](int, int r, int o, float v) {
                    const float y = tanhf(v);
                    actor.A(la)[r * AD + o] = y;
                    if (r < B) Xp[r * CI + SD + o] = y;
                });
                csync<CS>();
                if (actor.blk(kb).ln) { fwd_ln<CS, G>(actor, kb, 1, ra); csync<CS>(); }
            }
            for (int kb = 0; kb < 2; ++kb) {
                fwd_lin<CS, G>(critic, kb, 1, B, Xp, CI); csync<CS>();
                fwd_ln<CS, G>(critic, kb, 1, B); csync<CS>();
            }
            {   // Q1 and the gradient of -mean(Q1) at the last hidden layer
                const float* w = critic.P + critic.blk(2).off;
                for (int e = gt<CS, G>(); e < B * CH + B; e += GN(CS)) {
                    if (e < B * CH) {
                        const int i = e % CH;
                        critic.dU(1)[e] = (-inv_b * ld(w + i)) * act_d(a.act, ld(critic.A(1) + e));
                    } else {
                        const int r = e - B * CH;
                        const float* x = critic.A(1) + r * CH;
                        float acc = 0.f;
                        for (int i = 0; i < CH; ++i) acc = fmaf(ld(x + i), ld(w + i), acc);
                        q1[r] = acc + ld(w + CH);
                    }
                }
            }
            csync<CS>();
            bwd_ln<CS, G>(critic, 1, 1, B); csync<CS>();
            bwd_lin<CS, G>(critic, 1, 1, B, Xp, CI, false, true); csync<CS>();
            bwd_ln<CS, G>(critic, 0, 1, B); csync<CS>();
            {   // gradient at the actor's output: dQ1/da (critic input columns 7..9) + the CAPS terms, through tanh
                const float* w = critic.P + critic.blk(0).off;
                for (int e = gt<CS, G>(); e < ra * AD; e += GN(CS)) {
                    const int r = e / AD, j = e - r * AD;
                    const float y = ld(actor.A(la) + e), act = ld(Xs + (r % B) * CI + SD + j);
                    float g;
                    if (r < B) {
                        const float* d = critic.dZ(0) + r * CH;
                        g = 0.f;
                        for (int o = 0; o < CH; ++o) g = fmaf(ld(d + o), ld(w + o * CI + SD + j), g);
                        if (a.lt != 0.f) g += a.lt * mse_a * (y - act);
                    } else {
                        g = a.ls * mse_a * (y - act);
                    }
                    actor.dU(la)[e] = g * (1.f - y * y);
                }
            }
            csync<CS>();
            bwd_lin<CS, G>(actor, la, 1, ra, Xa, SD, true, true); csync<CS>();
            for (int kb = a.L; kb >= 1; --kb) {
                bwd_ln<CS, G, NJ>(actor, kb, 1, ra); csync<CS>();
                if (WIDE) bwd_wide<CS, G>(actor, kb, ra, wide_sm);
                else bwd_lin<CS, G>(actor, kb, 1, ra, Xa, SD, true, true);
                csync<CS>();
            }
            bwd_lin<CS, G>(actor, 0, 1, ra, Xa, SD, true, false);
            if (gt<CS, G>() == 0) {
                float sq = 0.f, st = 0.f, ss = 0.f;
                for (int r = 0; r < B; ++r) sq += ld(q1 + r);
                for (int e = 0; e < B * AD; ++e) {
                    const float act = ld(Xs + (e / AD) * CI + SD + e % AD);
                    const float dt = act - ld(actor.A(la) + e);
                    st = fmaf(dt, dt, st);
                    if (caps_s) { const float ds = act - ld(actor.A(la) + B * AD + e); ss = fmaf(ds, ds, ss); }
                }
                pg = -(sq / (float)B);
                if (a.lt != 0.f) pg += a.lt * (st / (float)(B * AD));
                if (caps_s) pg += a.ls * (ss / (float)(B * AD));
            }
            csync<CS>();
            norm_partials<CS, G>(ga, Pa, part); csync<CS>();
            adam<CS, G, G && PER>(th_a, m_a, v_a, tg_a, ga, Pa, part, ++ta, a, !a.champion, &s_coef);
            csync<CS>();
        }
        if (gt<CS, G>() == 0) {
            a.losses[2 * k] = td;
            a.losses[2 * k + 1] = pg;
            if (a.status && (!isfinite(td) || (actor_step && !isfinite(pg)))) atomicOr(a.status, SERL_STATUS_NONFINITE);
        }
    }
}

int64_t actor_floats(const serl_actor_shape& s)
{
    const int64_t h = s.hidden;
    return (int64_t)s.state_dim * h + h + (int64_t)s.num_layers * (h * h + 3 * h) + h * s.action_dim + s.action_dim;
}

// the narrow widths at any depth, and the wide ones (the tiled instantiation) up to SERL_TD3_MAX_WIDE_LAYERS blocks
bool shape_ok(const serl_actor_shape* s)
{
    const int h = s ? s->hidden : 0;
    const bool narrow = h == 32 || h == 64 || h == 72 || h == 96 || h == 128;
    const bool wide = h > 128 && h <= SERL_TD3_MAX_HIDDEN && s->num_layers <= SERL_TD3_MAX_WIDE_LAYERS;
    return s && s->state_dim == SD && s->action_dim == AD && (narrow || wide) &&
           s->num_layers >= 1 && s->activation >= SERL_ACT_TANH && s->activation <= SERL_ACT_LEAKY_RELU;
}

// why a descriptor cannot be trained (nullptr: it can); checked before any CUDA call
const char* desc_error(const serl_td3_desc* d)
{
    if (!shape_ok(&d->shape))
        return "unsupported actor shape (state 7, action 3, hidden 32/64/72/96/128 with num_layers >= 1 or hidden 129..320 "
               "with num_layers 1..8, activation 0..2)";
    if (d->batch < 1 || d->batch > SERL_TD3_MAX_BATCH) return "batch must be 1..128";
    if (d->n_steps < 0 || d->n_valid < d->batch || d->replay_cols < COLS)
        return "bad n_steps / n_valid (>= batch) / replay_cols (>= 19)";
    if (!d->d_state || !d->d_replay || !d->d_losses) return "null state / replay / losses";
    if (d->policy_update_freq < 1 || d->first_iteration < 0 || d->critic_adam_steps < 0 || d->actor_adam_steps < 0)
        return "bad policy_update_freq / iteration / Adam step count";
    if (d->flags & ~SERL_TD3_CHAMPION_TARGET) return "unknown flag";
    const int cs = d->cluster_size;
    if (cs != 0 && cs != 1 && cs != 2 && cs != 4 && cs != 8) return "cluster_size must be 0, 1, 2, 4 or 8";
    return nullptr;
}

Args make_args(const serl_td3_desc* d)
{
    Args a;
    a.st = d->d_state; a.replay = d->d_replay; a.cols = d->replay_cols; a.n_valid = d->n_valid;
    a.B = d->batch; a.n_steps = d->n_steps; a.h = d->shape.hidden; a.L = d->shape.num_layers; a.act = d->shape.activation;
    a.Pa = (int)actor_floats(d->shape);
    a.it0 = d->first_iteration; a.tc0 = d->critic_adam_steps; a.ta0 = d->actor_adam_steps;
    a.gamma = (float)d->gamma; a.tau = (float)d->tau; a.noise_sd = (float)d->noise_sd; a.noise_clip = (float)d->noise_clip;
    a.lt = (float)d->caps_lambda_t; a.ls = (float)d->caps_lambda_s; a.eps_sd = (float)d->caps_eps_sd; a.max_norm = (float)d->max_grad_norm;
    a.lr = d->lr; a.freq = d->policy_update_freq; a.champion = (d->flags & SERL_TD3_CHAMPION_TARGET) != 0;
    a.seed = d->seed; a.idx_in = d->d_indices;
    a.losses = d->d_losses; a.rec_idx = d->d_rec_indices; a.rec_noise = d->d_rec_noise; a.rec_caps = d->d_rec_caps;
    a.status = d->d_status;
    a.ws = nullptr;
    return a;
}

size_t scratch_floats(const Args& a) { return layout(a.B, a.h, a.L, a.Pa).total; }

const char* per_error(const serl_td3_desc* d, const serl_td3_per_desc* p)
{
    if (!p) return "null per descriptor";
    if (!p->d_tree) return "null d_tree";
    if (p->capacity < 1 || p->capacity > SERL_PER_MAX_CAPACITY) return "capacity must be 1..SERL_PER_MAX_CAPACITY";
    if (p->n_valid != d->n_valid || p->n_valid > p->capacity) return "n_valid must equal the desc's n_valid and be <= capacity";
    if (!(p->alpha > 0.0 && p->alpha <= 1.0)) return "alpha must be in (0, 1]";
    if (!(p->beta0 >= 0.0 && p->beta0 <= 1.0)) return "beta0 must be in [0, 1]";
    if (!(p->beta_frames > 0.0)) return "beta_frames must be > 0";
    return nullptr;
}

// The learners with steps of a checked serl_td3_learn call, in order, packed for one launch: a[m] and p[m] (p[m].tree null
// for a uniform learner), each with its own slice of one scratch buffer.  Slices are aligned to 128 bytes, and a
// prioritized learner's slice holds its batch's B weights after the layout.  Returns the number of learners packed, or a
// negative serl_status when the scratch cannot be had.
int pack(const serl_td3_desc* descs, const serl_td3_per_desc* pers, int n, cudaStream_t s, Args* a, Per* p)
{
    int m = 0;
    size_t total = 0;
    size_t off[SERL_TD3_MAX_GROUP];
    for (int i = 0; i < n; ++i) {
        if (descs[i].n_steps == 0) continue;
        a[m] = make_args(descs + i);
        const serl_td3_per_desc* q = pers && pers[i].d_tree ? pers + i : nullptr;
        p[m] = q ? Per{q->d_tree, per_leaves(q->capacity), q->n_valid, q->alpha, q->beta0, q->beta_frames, q->d_rec_weights, q->d_rec_td}
                 : Per{};
        off[m] = total;
        total += (scratch_floats(a[m]) + (q ? a[m].B : 0) + 31) / 32 * 32;
        ++m;
    }
    if (m == 0) return 0;
    void* ws = nullptr;
    const cudaError_t e = serl_scratch(SERL_SCRATCH_TD3, s, total * sizeof(float), &ws);
    if (e != cudaSuccess) return serl_fail_cuda(e, "td3 scratch");
    for (int g = 0; g < m; ++g) a[g].ws = (float*)ws + off[g];
    return m;
}

}  // namespace

// td3_group_per_kernel<CS> (td3_group_per.cu) on the learners with steps of a checked serl_td3_learn call
template <int CS>
int launch_group_per(const serl_td3_desc* descs, const serl_td3_per_desc* pers, int n, cudaStream_t s);
