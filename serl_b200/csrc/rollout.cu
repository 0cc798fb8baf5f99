// K1 — fused population rollout for sm_90a (+ batched plant step and actor forward; the K6 smoothness metric of the
// recorded actions is smoothness.cu).
//
// One lane = one (actor, env) trajectory; one warp = 32 envs of one actor; one CTA = 1-2 actors x 128 envs with their
// fp32 genomes (and the plant tables) staged once in shared memory.  Per step a warp runs, entirely on chip:
//   Actor.select_action  (base/core/genetic_agent.py:104-109; LayerNorm base/core/mod_utils.py:47-50)        fp32
//   CitationEnv.step     (envs/phlabenv.py:430-482: action scaling :62-73, fault shims envs/{be,jr,sa,se}/citation.py,
//                         reward :362-367, termination + penalty :391-399)                                fp64
//   native plant step    (envs/<variant>/_citation*.so step @0x6030: 6-stage Dormand-Prince ode5, h = 0.01, RHS
//                         generated from the binaries by tools/lift -> csrc/gen/plant_rhs_common.h)          fp64
// and accumulates the episodic return (base/core/agent.py:129).  HBM is touched only at episode start
// (genome, reference-signal parameters) and end (return, step count) unless a trace / action history is requested.
//
// Two actor implementations:
//   rollout_kernel_persist<H, TABS, ...>   persistent grid, one CTA per SM.  The MLP is a register-tiled GEMM inside a warp
//                           (lane = 1/8 of the output neurons x 8 envs, float2 pairs, activations exchanged through a
//                           per-warp shared-memory buffer, weights broadcast from shared memory; h in {32,64,72,96,128}).  The CTA's warps take
//                           their steps in lockstep (one barrier per step: shared instruction fetch), genomes arrive by bulk
//                           TMA copies.
//   rollout_kernel_simple   every thread runs the whole MLP for its env (any h that fits); cross-check / fallback shape.
#include <type_traits>

#define PLANT_SMEM_BUCKETS          // K1 stages the bucketed searches' byte tables with the plant tables (plant_env.cuh)
#include "plant_env.cuh"
#include "rollout_variant.h"

// ---- simple actor: every thread evaluates the whole MLP for its own observation -------------------------
__device__ void actor_forward_simple(const float* __restrict__ w, const serl_actor_shape sh, float* bufA, float* bufB,
                                     int tid, int nthr, const float* obs, float* action)
{
    // same arithmetic specification as actor_forward_warp (dot products: sequential fma from 0; LayerNorm / output-layer
    // sums: four contiguous quarter blocks, combined (q0+q1)+(q2+q3)), so both kernels produce identical bits
    const int S = sh.state_dim, A = sh.action_dim, H = sh.hidden, L = sh.num_layers;
    const int TM = (H + 3) / 4;
    const float* p = w;
    for (int j = 0; j < H; ++j) {
        float acc = 0.f;
        for (int i = 0; i < S; ++i) acc = __fmaf_rn(p[j * S + i], obs[i], acc);
        acc = __fadd_rn(acc, p[H * S + j]);
        bufA[j * nthr + tid] = act_fn(sh.activation, acc);
    }
    p += H * S + H;
    float* in = bufA;
    float* out = bufB;
    for (int l = 0; l < L; ++l) {
        const float* W = p;
        const float* b = p + H * H;
        const float* gamma = b + H;
        const float* beta = gamma + H;
        float q[4];
        for (int g = 0; g < 4; ++g) {
            float sum = 0.f;
            for (int j = g * TM; j < min((g + 1) * TM, H); ++j) {
                float acc = 0.f;
                for (int i = 0; i < H; ++i) acc = __fmaf_rn(W[j * H + i], in[i * nthr + tid], acc);
                acc = __fadd_rn(acc, b[j]);
                out[j * nthr + tid] = acc;
                sum = __fadd_rn(sum, acc);
            }
            q[g] = sum;
        }
        const float mean = __fdiv_rn(__fadd_rn(__fadd_rn(q[0], q[1]), __fadd_rn(q[2], q[3])), (float)H);
        for (int g = 0; g < 4; ++g) {
            float ss = 0.f;
            for (int j = g * TM; j < min((g + 1) * TM, H); ++j) {
                const float d = __fadd_rn(out[j * nthr + tid], -mean);
                out[j * nthr + tid] = d;
                ss = __fmaf_rn(d, d, ss);
            }
            q[g] = ss;
        }
        const float var = __fdiv_rn(__fadd_rn(__fadd_rn(q[0], q[1]), __fadd_rn(q[2], q[3])), (float)(H - 1));
        const float inv = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(var), 1e-6f));
        for (int j = 0; j < H; ++j)
            out[j * nthr + tid] = act_fn(sh.activation, __fmaf_rn(__fmul_rn(gamma[j], out[j * nthr + tid]), inv, beta[j]));
        p += H * H + 3 * H;
        float* t = in; in = out; out = t;
    }
    for (int j = 0; j < A; ++j) {
        float q[4];
        for (int g = 0; g < 4; ++g) {
            float acc = 0.f;
            for (int i = g * TM; i < min((g + 1) * TM, H); ++i) acc = __fmaf_rn(p[j * H + i], in[i * nthr + tid], acc);
            q[g] = acc;
        }
        action[j] = am_tanh1(__fadd_rn(__fadd_rn(__fadd_rn(q[0], q[1]), __fadd_rn(q[2], q[3])), p[A * H + j]));
    }
}

// ---- warp-autonomous actor + env ---------------------------------------------------------------------------
// smem: plant tables [PT_TOTAL] f64 | per actor of the CTA: transposed weights in row-pair blocks (pair_layout_index)
//       Wt0[S][H] b0[H] | L x { Wt[H][H] b[H] gamma[H] beta[H] } | Wo[A][H] bo[A]
// lane = (g = lane>>3, og = lane&7): output neurons og*T8 .. og*T8+T8-1 (T8 = h/8) of the envs 8g .. 8g+7 of this warp.
// The activation of neuron k for env 8g+c lives in lane (g, og = k/T8), register in[k%T8][c/2] (.x / .y).  The next
// layer reads it from the warp's exchange buffer xb in shared memory, one source quarter (lanes og = 2q, 2q+1) at a
// time: before quarter so its lanes store their in[][] as xb[row][8g + c] (two STS.128 per neuron), so that two LDS.128
// per source neuron give a lane the eight envs of its group and the loop over source neurons is a rolled loop with a
// small body (unrolled, the register selection and shuffles of every neuron made the actor too large for the
// instruction cache next to the plant).  A weight load serves 8 envs: per pair of source rows a lane takes its 2·T8
// weights with T8/2 LDS.128 (+ one LDS.64 when T8 is odd) and the 16 inputs with 4 LDS.128, for 16·T8 multiply-adds.
// A quarter's sums (LayerNorm, output layer) run sequentially over its first eighth in lane og = 2q, are handed to
// lane 2q+1 with one shuffle and continue there: the order of the kernel-order oracle's quarter blocks
// (oracle/plant/actor_kernel_order.c).  The quarters are then combined (q0+q1)+(q2+q3) by a butterfly that also
// transposes: each odd lane ends with the totals of two envs, takes their per-env divisions / square root, and every
// lane of the group reads the results back by shuffles, so all eight lanes of a group hold bit-identical means /
// deviations.  Element-wise arithmetic is written on float2 pairs of two envs of one neuron (am_fma2: two independent
// IEEE-rn fmas), and an activation call takes the group's eight envs of one neuron.
__host__ __device__ constexpr int actor_xbuf_floats(int H) { return H / 4 * 32; }    // exchange buffer per warp: a quarter x 32 envs
// ... and for an observation of S entries, which the input layer stages there too (S = 10 exceeds a quarter at h = 32)
__host__ __device__ constexpr int actor_xbuf_floats(int H, int S) { return (H / 4 > S ? H / 4 : S) * 32; }

// Offset of element (source row k, output neuron n) of a transposed [R][H] matrix in the kernel layout: rows in pairs, a
// pair a block of 2H floats in which lane og's 2·T8 weights (row k's T8, then row k+1's) are its N4 float4 (at
// 16-byte chunk i: all eight lanes' chunk i side by side, so that an LDS.128 of the warp touches 128 contiguous bytes)
// and, for odd T8, one float2 after the chunks.  An odd last row (the observation layer: R = 7) is a plain row; the
// incremental-control observation (R = 10) is five pairs, the symmetric-control one (R = 2) one pair.
__host__ __device__ constexpr int pair_layout_index(int k, int n, int R, int H)
{
    const int T8 = H / 8, N4 = T8 / 2 * 4;                 // floats of a lane's pair weights in float4 chunks
    if (k >= (R & ~1)) return (R & ~1) * H + n;
    const int og = n / T8, j = (k & 1) * T8 + n % T8;
    const int base = (k >> 1) * 2 * H;
    return j < N4 ? base + (j / 4) * 32 + og * 4 + j % 4 : base + N4 * 8 + og * 2 + (j - N4);
}

// one pair of source rows: their activations for the group's eight envs and the lane's 2·T8 weights
template <int H>
struct WarpPair {
    static constexpr int T8 = H / 8, N4 = T8 / 2;
    float4 x[4];                                       // row k: envs 0-3, 4-7; row k + 1: envs 0-3, 4-7
    float4 w4[N4];
    float2 w2;                                         // odd T8 only
    // wl = matrix + og * 4, wt = matrix + N4 * 32 + og * 2 (pair_layout_index)
    __device__ __forceinline__ void load(const float* __restrict__ wl, const float* __restrict__ wt, const float* xg, int p)
    {
#pragma unroll
        for (int i = 0; i < 4; ++i) x[i] = *reinterpret_cast<const float4*>(xg + (2 * p + (i >> 1)) * 32 + (i & 1) * 4);
#pragma unroll
        for (int i = 0; i < N4; ++i) w4[i] = *reinterpret_cast<const float4*>(wl + p * 2 * H + i * 32);
        if (T8 & 1) w2 = *reinterpret_cast<const float2*>(wt + p * 2 * H);
    }
    __device__ __forceinline__ float w(int j) const
    {
        if (j >= 4 * N4) return j == 4 * N4 ? w2.x : w2.y;
        const float4 v = w4[j / 4];
        return j % 4 == 0 ? v.x : j % 4 == 1 ? v.y : j % 4 == 2 ? v.z : v.w;
    }
    __device__ __forceinline__ void fma(float2 (&acc)[T8][4]) const
    {
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int m = 0; m < T8; ++m) {
                const float2 wv = am_splat(w(r * T8 + m));
                const float4 a = x[2 * r], b = x[2 * r + 1];
                acc[m][0] = am_fma2(wv, make_float2(a.x, a.y), acc[m][0]);
                acc[m][1] = am_fma2(wv, make_float2(a.z, a.w), acc[m][1]);
                acc[m][2] = am_fma2(wv, make_float2(b.x, b.y), acc[m][2]);
                acc[m][3] = am_fma2(wv, make_float2(b.z, b.w), acc[m][3]);
            }
    }
};

// acc[m][c] += sum over source rows k < nk (in order from 0) of W[k][og*T8 + m] * xg[k*32 + c] for the matrix at `wm`
// (pair_layout_index).  Two row pairs per trip, each pair's loads issued before the multiply-adds of the pair ahead of
// it: the shared-memory latency is hidden without unrolling the loop.
template <int H>
__device__ __forceinline__ void warp_rows(const float* __restrict__ wm, int nk, const float* xg, int og, float2 (&acc)[H / 8][4])
{
    using P = WarpPair<H>;
    const float* wl = wm + og * 4;
    const float* wt = wm + P::N4 * 32 + og * 2;
    const int np = nk >> 1;
    P ra, rb;
    ra.load(wl, wt, xg, 0);
    int p = 0;
#pragma unroll 1
    for (; p + 2 <= np; p += 2) {
        rb.load(wl, wt, xg, p + 1);
        ra.fma(acc);
        ra.load(wl, wt, xg, p + 2 < np ? p + 2 : p + 1);      // (the last trip re-reads pair p + 1: stays in bounds)
        rb.fma(acc);
    }
    if (p < np) ra.fma(acc);
    if (nk & 1) {                                      // a plain last row
        const int k = nk - 1;
        const float4 a = *reinterpret_cast<const float4*>(xg + k * 32), b = *reinterpret_cast<const float4*>(xg + k * 32 + 4);
#pragma unroll
        for (int m = 0; m < P::T8; ++m) {
            const float2 wv = am_splat(wm[k * H + og * P::T8 + m]);
            acc[m][0] = am_fma2(wv, make_float2(a.x, a.y), acc[m][0]);
            acc[m][1] = am_fma2(wv, make_float2(a.z, a.w), acc[m][1]);
            acc[m][2] = am_fma2(wv, make_float2(b.x, b.y), acc[m][2]);
            acc[m][3] = am_fma2(wv, make_float2(b.z, b.w), acc[m][3]);
        }
    }
}

template <int H>
__device__ __forceinline__ void warp_layer(const float* __restrict__ Wt, const float2 (&in)[H / 8][4], float2 (&acc)[H / 8][4],
                                           int og, int g, float* xb)
{
    constexpr int TM = H / 4, T8 = H / 8;
#pragma unroll
    for (int m = 0; m < T8; ++m)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[m][c] = make_float2(0.f, 0.f);
    float* xs = xb + (og & 1) * T8 * 32 + g * 8;       // this lane's rows of its quarter
#pragma unroll 1
    for (int so = 0; so < 4; ++so) {
        __syncwarp();                                  // the previous quarter has been read
        if ((og >> 1) == so) {
#pragma unroll
            for (int m = 0; m < T8; ++m) {
                *reinterpret_cast<float4*>(xs + m * 32) = make_float4(in[m][0].x, in[m][0].y, in[m][1].x, in[m][1].y);
                *reinterpret_cast<float4*>(xs + m * 32 + 4) = make_float4(in[m][2].x, in[m][2].y, in[m][3].x, in[m][3].y);
            }
        }
        __syncwarp();
        warp_rows<H>(Wt + (size_t)(so * TM) * H, TM, xb + g * 8, og, acc);
    }
}

__device__ __forceinline__ float env_of(const float2 (&v)[4], int c) { return c & 1 ? v[c >> 1].y : v[c >> 1].x; }

// Sum over the group's quarter blocks for each of its eight envs.  f(m, c, s) adds the lane's neuron m of env c to s;
// the quarter's first eighth (lane og = 2q) is summed from 0 and continued in lane 2q + 1.  The quarters are combined
// (q0+q1)+(q2+q3) (fadd is commutative, so both lanes of a butterfly pair get the same bits) while each round halves the
// envs a lane keeps: odd lane og ends with the totals of envs 4·og[1] + 2·og[2] + i, i = 0, 1, in tot[i]
// (quarter_src_lane).  The other lanes' tot is meaningless.
template <int T8, typename F>
__device__ __forceinline__ void quarter_totals(F f, int og, float (&tot)[2])
{
    float s[8];
#pragma unroll
    for (int c = 0; c < 8; ++c) s[c] = 0.f;
#pragma unroll 1
    for (int pass = 0; pass < 2; ++pass) {             // rolled: the sums are written once in the code
        if (pass)
#pragma unroll
            for (int c = 0; c < 8; ++c) s[c] = __shfl_xor_sync(0xffffffffu, s[c], 1);
#pragma unroll
        for (int m = 0; m < T8; ++m)
#pragma unroll
            for (int c = 0; c < 8; ++c) s[c] = f(m, c, s[c]);
    }
    const bool hi1 = (og & 2) != 0, hi2 = (og & 4) != 0;
    float r[4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
        r[i] = __fadd_rn(hi1 ? s[4 + i] : s[i], __shfl_xor_sync(0xffffffffu, hi1 ? s[i] : s[4 + i], 2));
#pragma unroll
    for (int i = 0; i < 2; ++i)
        tot[i] = __fadd_rn(hi2 ? r[2 + i] : r[i], __shfl_xor_sync(0xffffffffu, hi2 ? r[i] : r[2 + i], 4));
}

// the lane of group g whose tot[c & 1] holds env c's total
__device__ __forceinline__ int quarter_src_lane(int g, int c) { return g * 8 + 1 + ((c >> 2) & 1) * 2 + ((c >> 1) & 1) * 4; }

// observation in, action out: by value (registers) rather than through pointers, which put them in local memory
template <int S> struct ActorObs { float v[S]; };     // S = 7, 10 with incremental control (+ last_u), 2 with symmetric control
template <int A = 3> struct ActorAct { float v[A]; };  // A = 3, or 1 with symmetric control (the elevator)

// xb: this warp's exchange buffer, actor_xbuf_floats(H) floats in shared memory (actor_xbuf_floats(H, 10) for S = 10),
// 16-byte aligned.  The observation layer sums its S inputs with fma from 0 in index order, then adds the bias (the
// kernel-order specification).  A: outputs, summed and squashed one by one in the same order
template <int H, int ACT, int S = 7, int A = 3>
__device__ __noinline__ ActorAct<A> actor_forward_warp(const float* __restrict__ w, int L, int lane, float* xb, ActorObs<S> obs)
{
    constexpr int TM = H / 4, T8 = H / 8;
    static_assert(S == 10 || TM >= S, "the observation rows fit the exchange buffer");
    const int og = lane & 7, g = lane >> 3, n0 = og * T8;
    const float* Wt0 = w;
    const float* b0 = Wt0 + S * H;
    const float* hid = b0 + H;
    const float* Wo = hid + (size_t)L * (H * H + 3 * H);
    const float* bo = Wo + A * H;
    float2 in[T8][4], acc[T8][4];
    // input layer: the observation of env lane = 8g+c goes to xb[k][8g + c]
#pragma unroll
    for (int m = 0; m < T8; ++m)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[m][c] = make_float2(0.f, 0.f);
    __syncwarp();                                      // the previous call has read the buffer
#pragma unroll
    for (int k = 0; k < S; ++k) xb[k * 32 + lane] = obs.v[k];
    __syncwarp();
    warp_rows<H>(Wt0, S, xb + g * 8, og, acc);
#pragma unroll
    for (int m = 0; m < T8; ++m) {
        const float2 b = am_splat(b0[n0 + m]);
        AmF2x4 v;
#pragma unroll
        for (int c = 0; c < 4; ++c) v.v[c] = am_fma2(acc[m][c], am_splat(1.0f), b);
        v = am_act2x4<ACT>(v);
#pragma unroll
        for (int c = 0; c < 4; ++c) in[m][c] = v.v[c];
    }
    // hidden layers: Linear -> LayerNorm (unbiased std, eps on std; mod_utils.py:47-50) -> activation
#pragma unroll 1
    for (int l = 0; l < L; ++l) {
        const float* Wt = hid + (size_t)l * (H * H + 3 * H);
        const float* bb = Wt + H * H;
        const float* gamma = bb + H;
        const float* beta = gamma + H;
        warp_layer<H>(Wt, in, acc, og, g, xb);
#pragma unroll
        for (int m = 0; m < T8; ++m) {
            const float2 b = am_splat(bb[n0 + m]);
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[m][c] = am_fma2(acc[m][c], am_splat(1.0f), b);
        }
        float t[2], mean[8], den[8];
        quarter_totals<T8>([&](int m, int c, float s) { return __fadd_rn(s, env_of(acc[m], c)); }, og, t);
#pragma unroll
        for (int i = 0; i < 2; ++i) t[i] = __fdiv_rn(t[i], (float)H);
#pragma unroll
        for (int c = 0; c < 8; ++c) mean[c] = __shfl_sync(0xffffffffu, t[c & 1], quarter_src_lane(g, c));
#pragma unroll
        for (int m = 0; m < T8; ++m)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[m][c] = am_fma2(acc[m][c], am_splat(1.0f), make_float2(-mean[2 * c], -mean[2 * c + 1]));
        quarter_totals<T8>([&](int m, int c, float s) { const float d = env_of(acc[m], c); return __fmaf_rn(d, d, s); }, og, t);
        // gamma * (x - mean) / (std + eps) + beta as fma(gamma * d, 1 / (std + eps), beta): one reciprocal per env instead
        // of h divisions (<= 1 ulp from the reference's expression, the order of its summation-order freedom)
#pragma unroll
        for (int i = 0; i < 2; ++i) t[i] = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(__fdiv_rn(t[i], (float)(H - 1))), 1e-6f));
#pragma unroll
        for (int c = 0; c < 8; ++c) den[c] = __shfl_sync(0xffffffffu, t[c & 1], quarter_src_lane(g, c));
#pragma unroll
        for (int m = 0; m < T8; ++m) {
            const float2 gm = am_splat(gamma[n0 + m]), be = am_splat(beta[n0 + m]);
            AmF2x4 v;
#pragma unroll
            for (int c = 0; c < 4; ++c)
                v.v[c] = am_fma2(am_fma2(gm, acc[m][c], am_splat(-0.0f)), make_float2(den[2 * c], den[2 * c + 1]), be);
            v = am_act2x4<ACT>(v);
#pragma unroll
            for (int c = 0; c < 4; ++c) in[m][c] = v.v[c];
        }
    }
    // output layer: quarter-block dot products over the group, combined like the LayerNorm sums; lane og keeps env 8g+og.
    // The three tanh go through two pair calls, a single action through one.
    float y[A];
#pragma unroll
    for (int j = 0; j < A; ++j) {
        float wv[T8], t[2];
#pragma unroll
        for (int m = 0; m < T8; ++m) wv[m] = Wo[j * H + n0 + m];
        quarter_totals<T8>([&](int m, int c, float s) { return __fmaf_rn(wv[m], env_of(in[m], c), s); }, og, t);
        const int src = quarter_src_lane(g, og);
        const float t0 = __shfl_sync(0xffffffffu, t[0], src), t1 = __shfl_sync(0xffffffffu, t[1], src);
        y[j] = __fadd_rn(og & 1 ? t1 : t0, bo[j]);
    }
    static_assert(A == 3 || A == 1, "two tanh pairs, or one");
    ActorAct<A> action;
    if constexpr (A == 1) {
        action.v[0] = am_tanh2(make_float2(y[0], y[0])).x;
    } else {
        const float2 t01 = am_tanh2(make_float2(y[0], y[1])), t2 = am_tanh2(make_float2(y[2], y[2]));
        action.v[0] = t01.x; action.v[1] = t01.y; action.v[2] = t2.x;
    }
    return action;
}

// one instantiation per activation: the choice is compiled into the 4 x h/4 activation calls of every layer
template <int H, int S, int A>
__device__ __forceinline__ void actor_forward(int act, const float* __restrict__ w, int L, int lane, float* xb, const float (&obs)[S],
                                              float (&a)[A])
{
    ActorObs<S> o;
#pragma unroll
    for (int k = 0; k < S; ++k) o.v[k] = obs[k];
    ActorAct<A> r;
    if (act == SERL_ACT_TANH) r = actor_forward_warp<H, SERL_ACT_TANH, S, A>(w, L, lane, xb, o);
    else if (act == SERL_ACT_ELU) r = actor_forward_warp<H, SERL_ACT_ELU, S, A>(w, L, lane, xb, o);
    else r = actor_forward_warp<H, SERL_ACT_LEAKY_RELU, S, A>(w, L, lane, xb, o);
#pragma unroll
    for (int j = 0; j < A; ++j) a[j] = r.v[j];
}


// ---- genome layout in shared memory -------------------------------------------------------------------------
// parameters() order in HBM (row-major [out][in]) -> the kernel's layout (matrices transposed to [in][out], in the
// row-pair blocks of pair_layout_index):
//   Wt0[S][H] b0[H] | L x { Wt[H][H] b[H] gamma[H] beta[H] } | Wo[A][H] bo[A]
__device__ __forceinline__ int genome_layout_index(int i, int S, int H, int L)
{
    int r = i;
    if (r < S * H) { const int j = r / S, k = r % S; return pair_layout_index(k, j, S, H); }
    r -= S * H;
    if (r < H) return S * H + r;
    r -= H;
    const int per = H * H + 3 * H;
    if (r < L * per) {
        const int l = r / per, q = r % per;
        const int base = S * H + H + l * per;
        if (q < H * H) { const int j = q / H, k = q % H; return base + pair_layout_index(k, j, H, H); }
        return base + q;
    }
    return i;      // Wo [A][H] then bo[A]: unchanged
}

// K0: all genomes of a launch into the shared-memory layout, rows padded to 16 bytes, so that the rollout kernel can
// bring a genome into shared memory with ONE bulk TMA copy (cp.async.bulk) instead of a scattered staging loop.
__global__ void genome_layout_kernel(const float* __restrict__ w, float* __restrict__ wt, int pop, int P, int P4, int S, int H, int L)
{
    const long long n = (long long)pop * P;
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += (long long)gridDim.x * blockDim.x) {
        const int a = (int)(g / P), i = (int)(g % P);
        wt[(size_t)a * P4 + genome_layout_index(i, S, H, L)] = w[g];
    }
}

// ---- K1: persistent rollout ------------------------------------------------------------------------------------
// grid = one CTA per SM (or fewer when there is less work); a CTA has `apc` genome slots of `wps` warps each.  A task is
// (actor, chunk of wps*32 envs) x horizon steps.  Tasks are dealt to the slots as EQUAL SHARES OF STEPS: slot s owns
// the range [s W/NS, (s+1) W/NS) of the linearised (task, step) space, W = n_tasks * horizon — i.e. possibly the tail of
// one task, some whole tasks, and the head of another.  A slot flies the head segment FIRST and publishes the
// trajectories' state in HBM (Handoff), then its whole tasks, and LAST the tail segment, whose first part the previous
// slot published long before: no slot ever waits in practice, and all SMs finish together (512 actors x 128 envs on
// 132 SMs x 2 slots = 1.94 tasks per slot: two full rounds without the split).  When there are fewer tasks than
// slots every task is flown whole by one slot.  The genome of a slot is swapped by ONE elected thread with a bulk TMA copy;
// the slot's warps meet at its named barrier for that and for the slot-uniform decisions of the lockstep loop (see there).
// TABS: plant tables staged in shared memory (true) or read from global memory through L1 (false: h = 128, whose
// 207 KB genome leaves no room for them).
// GUST, TRACK, PER_ACTOR, INC, SYM: the launch's variant (rollout_variant.h lists the instantiated ones).
// GUST: the launch contains envs of the gust build (serl_rollout_desc.flags & SERL_ROLLOUT_GUST); an instantiation without
// it carries no trace of the feature (a gust env in it raises SERL_STATUS_GUST_FLAG)
// TRACK: the launch writes the tracking-error sums `tk` (serl_rollout_desc.d_track); the sums travel in the hand-over
// records too
// PER_ACTOR: every actor flies its own env block (SERL_ROLLOUT_PER_ACTOR_REFS): env `env` of actor `actor` binds row
// actor * n_envs + env of env_mode / ref_levels / ref_starts, also when a slot resumes it from a hand-over record
// INC: incremental control (SERL_ROLLOUT_INCREMENTAL): a 10-entry observation and the env's last_u, both carried in the
// hand-over records too (OBS_DIM: plant_env.cuh), next to the tracking sums of a TRACK instantiation.
// SYM: symmetric control (SERL_ROLLOUT_SYMMETRIC): a 2-entry observation, one action
template <int H, bool TABS, bool GUST, bool TRACK = false, bool PER_ACTOR = false, bool INC = false, bool SYM = false>
__global__ void __launch_bounds__(MAX_CTA_THREADS, 1)
rollout_kernel_persist(RolloutArgs ar, TrackArgs tk)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];     // same alignment as plant_smem_tab (plant_env.cuh)
    __shared__ uint64_t gbar[4];                       // one mbarrier per genome slot
    if (TABS) plant_tab_check(smem_raw);
    real* tab_s = reinterpret_cast<real*>(smem_raw);
    // PLANT_TABN2 (plant_env.cuh) spelt out: naming it here reorders a few instructions of the gust instantiations
    constexpr int TABN = PT_TOTAL + SERL_PLANT_COUNT * PLANT_NPV + PLANT_BKT_WORDS;      // tables + parameter rows + bytes
    constexpr int TABN2 = (TABN + 1) & ~1;
    static_assert(TABN2 == PLANT_TABN2, "shared-memory layout of the plant tables");
    float* wbase = reinterpret_cast<float*>(tab_s + (TABS ? TABN2 : 0));
    const real* tab = TABS ? tab_s : plant_tables_blob;
    const real* pv_base = TABS ? tab_s + PT_TOTAL : &plant_pv[0][0];
    const int L = ar.sh.num_layers;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wps = ar.wps;
    const int slot_l = warp / wps, wslot = warp - slot_l * wps;
    const long long slot = (long long)blockIdx.x * ar.apc + slot_l;
    if (TABS) {
        for (int i = tid; i < PT_TOTAL; i += blockDim.x) tab_s[i] = plant_tables_blob[i];
        for (int i = tid; i < SERL_PLANT_COUNT * PLANT_NPV; i += blockDim.x) tab_s[PT_TOTAL + i] = (&plant_pv[0][0])[i];
        plant_stage_buckets(tab_s, tid, blockDim.x);
    }
    if (tid == 0) {
        for (int i = 0; i < ar.apc; ++i) mbar_init(&gbar[i], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    float* w = wbase + (size_t)slot_l * ar.P4;
    float* xb = wbase + (size_t)ar.apc * ar.P4 + warp * (INC ? actor_xbuf_floats(H, OBS_DIM<INC>) : actor_xbuf_floats(H));     // after the genomes
    const int slot_threads = wps * 32;
    const int actfn = ar.sh.activation;
    const int horizon = ar.horizon;
    int cur_actor = -1;
    uint32_t gphase = 0;

    // this slot's share of the (task, step) space
    const long long NT = ar.n_tasks, NS = ar.n_slots;
    long long t_first = 0, t_last = 0;
    int k0 = 0, k1 = 0;
    int stage = 0;                                     // 3 = no (more) segments
    if (NT <= NS) {
        if (slot >= NT) stage = 3;                     // idle slot: still takes part in the CTA barriers below
        t_first = slot; t_last = slot + 1;
    } else {
        const long long W = NT * horizon;
        const long long lo = slot * W / NS, hi = (slot + 1) * W / NS;
        t_first = lo / horizon; t_last = hi / horizon;
        k0 = (int)(lo - t_first * horizon); k1 = (int)(hi - t_last * horizon);
    }
    // segments in the order: head of the last task (published) -> whole tasks -> tail of the first task (continued)
    long long t_cur = t_first + (k0 > 0 ? 1 : 0);
    // LOCKSTEP: all warps of the CTA meet at one CTA barrier per loop trip.  The step body is ~130 KB of code at h = 72
    // (sm_90a SASS: actor 31 KB, right-hand side 41 KB x 6 calls, ode5 step 16 KB, environment and segment bookkeeping up
    // to 40 KB); eight warps drifting through it independently each stream it through the instruction caches on their own,
    // and instruction fetch was the top stall (no_instruction 27 % of the warp samples on B200).  Met at a barrier, a
    // fetched line serves every warp of the SM that runs the same phase.
    // STAGGER (ar.stagger, two slots): a trip is half a step.  Slot 0 runs its actor while slot 1 runs its environment
    // step, then they swap, so that each SM sub-partition (one warp of each slot) has one warp on the fp32 pipe and one on
    // the fp64 pipe instead of both on the same one.  A slot's step boundary (segment close / open, hand-over) comes
    // before its actor half; the action stays in registers until the environment half.  Opt-in: on an H100 it is slower
    // than lockstep (the plant is latency bound and slows down next to a warp in the actor; DESIGN §5).
    Env e;
    e.tab = tab;
    e.done = true; e.k = 0;
    float obs[OBS_DIM<INC, SYM>], a[ACT_DIM<SYM>];
    double last_u[3];                                  // INC only
    double* const ho_u = INC ? reinterpret_cast<double*>(ar.ho.obs + (size_t)OBS_DIM<INC> * ar.ho.n) : nullptr;
    bool in_seg = false, pending = false, to_h = false, valid = false, replay = false;
    int ke = 0, actor = 0;
    size_t traj = 0;
    const bool stagger = ar.stagger != 0;
    bool actor_half = !(stagger && slot_l == 1);       // slot-uniform; slot 1 starts with an empty environment half
    for (;;) {
        // is this slot's segment still flying?  (slot-uniform: OR over the slot's warps at its named barrier)
        bool slot_alive = false;
        if (!actor_half) {
            slot_alive = true;                         // mid-step: the boundary comes with the next actor half
        } else if (in_seg) {
            int any;
            asm volatile("{ .reg .pred p, q; setp.ne.s32 p, %1, 0; barrier.cta.red.or.pred q, %2, %3, p; selp.s32 %0, 1, 0, q; }"
                         : "=r"(any) : "r"((int)(!e.done && e.k < ke)), "r"(1 + slot_l), "r"(slot_threads) : "memory");
            slot_alive = any != 0;
        }
        if (!slot_alive) {
            if (in_seg) {                              // close the finished segment
                if (to_h) {
                    const long long hx = slot * slot_threads + wslot * 32 + lane;
                    if (valid) {
#pragma unroll
                        for (int i = 0; i < NX; ++i) __stcg(ar.ho.X + (size_t)i * ar.ho.n + hx, e.X[i]);
                        __stcg(ar.ho.t + hx, e.t); __stcg(ar.ho.ret + hx, e.ret);
#pragma unroll
                        for (int i = 0; i < OBS_DIM<INC, SYM>; ++i) __stcg(ar.ho.obs + (size_t)i * ar.ho.n + hx, obs[i]);
                        if constexpr (INC)
#pragma unroll
                            for (int i = 0; i < 3; ++i) __stcg(ho_u + (size_t)i * ar.ho.n + hx, last_u[i]);
                        __stcg(ar.ho.k + hx, e.k | ((e.done ? 1 : 0) << 30));
                        if constexpr (TRACK)
#pragma unroll
                            for (int i = 0; i < TRACK_CARRY; ++i) __stcg(tk.ho + (size_t)i * ar.ho.n + hx, e.trk[i]);
                    }
                    __threadfence();
                    __syncwarp();
                    if (lane == 0) atomicExch(ar.ho.flag + slot * wps + wslot, 1);
                } else if (valid) {
                    traj_store(e, ar, traj);
                    if constexpr (TRACK) track_store(e, tk, traj);
                }
                in_seg = false;
            }
            // open the next one, if any.  The tail segment continues trajectories the PREVIOUS slot publishes at the end of
            // its head segment: normally long done, but that slot may sit in this very CTA and advance only with this
            // one's steps (lockstep), so the slot never blocks on the record — it stays `pending` and asks again at the next
            // step.  All decisions are slot-uniform (AND over the slot's warps at its named barrier).
            long long task = 0;
            bool have = false;
            if (!pending) {
                to_h = false;
                while (!have && stage < 3) {
                    if (stage == 0) {
                        stage = 1;
                        if (k1 != 0) { task = t_last; ke = k1; to_h = true; have = true; }
                    } else if (stage == 1) {
                        if (t_cur >= t_last) stage = 2;
                        else { task = t_cur++; ke = horizon; have = true; }
                    } else {
                        stage = 3;
                        if (k0 != 0) { ke = horizon; pending = true; }
                    }
                }
            }
            const bool from_h = pending;
            if (pending) {
                int ok = 0;
                if (lane == 0) ok = *(const volatile int*)(ar.ho.flag + (slot - 1) * wps + wslot) != 0;
                ok = __shfl_sync(0xffffffffu, ok, 0);
                int all;
                asm volatile("{ .reg .pred p, q; setp.ne.s32 p, %1, 0; barrier.cta.red.and.pred q, %2, %3, p; selp.s32 %0, 1, 0, q; }"
                             : "=r"(all) : "r"(ok), "r"(1 + slot_l), "r"(slot_threads) : "memory");
                if (all) { pending = false; task = t_first; have = true; __threadfence(); }
                else __nanosleep(500);
            }
            if (have) {
                actor = (int)(task / ar.n_chunks);
                const int chunk = (int)(task - (long long)actor * ar.n_chunks);
                if (actor != cur_actor) {
                    // swap the genome of this slot: everyone has left the previous segment -> one thread launches the bulk copy
                    asm volatile("bar.sync %0, %1;" ::"r"(1 + slot_l), "r"(slot_threads) : "memory");
                    if (wslot == 0 && lane == 0) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic reads of w before the async write
                        const uint32_t bytes = (uint32_t)ar.P4 * 4u;
                        mbar_expect_tx(&gbar[slot_l], bytes);
                        tma_bulk_g2s(w, ar.wt + (size_t)actor * ar.P4, bytes, &gbar[slot_l]);
                    }
                    mbar_wait(&gbar[slot_l], gphase);
                    gphase ^= 1;
                    cur_actor = actor;
                }
                const int eslot = chunk * slot_threads + wslot * 32 + lane;
                valid = eslot < ar.n_envs;
                const int env = valid ? (ar.env_order ? ar.env_order[eslot] : eslot) : 0;
                traj = (size_t)actor * ar.n_envs + env;
                const int row = PER_ACTOR ? (int)traj : env;
                if (valid) {
                    env_bind<GUST>(e, ar, row, pv_base, traj);
                    if (from_h) {
                        const long long hx = (slot - 1) * slot_threads + wslot * 32 + lane;
#pragma unroll
                        for (int i = 0; i < NX; ++i) e.X[i] = __ldcg(ar.ho.X + (size_t)i * ar.ho.n + hx);
                        e.t = __ldcg(ar.ho.t + hx); e.ret = __ldcg(ar.ho.ret + hx);
#pragma unroll
                        for (int i = 0; i < OBS_DIM<INC, SYM>; ++i) obs[i] = __ldcg(ar.ho.obs + (size_t)i * ar.ho.n + hx);
                        if constexpr (INC)
#pragma unroll
                            for (int i = 0; i < 3; ++i) last_u[i] = __ldcg(ho_u + (size_t)i * ar.ho.n + hx);
                        const int kk = __ldcg(ar.ho.k + hx);
                        e.k = kk & 0x3fffffff; e.done = ((kk >> 30) & 1) != 0;
                        if constexpr (TRACK)
#pragma unroll
                            for (int i = 0; i < TRACK_CARRY; ++i) e.trk[i] = __ldcg(tk.ho + (size_t)i * ar.ho.n + hx);
                    } else {
                        env_reset<TABS, GUST, TRACK, INC, SYM>(e, ar, row, obs, traj, last_u);
                    }
                } else {
                    env_idle<INC, SYM>(e, ar, pv_base, obs, last_u);
                }
                replay = valid && ar.replay != nullptr && env == ar.replay_env;
                in_seg = true;
            }
        }
        // the CTA's warps meet here once per trip; the launch ends when no slot has a segment left (stage < 3: slot 1's
        // first, empty half of a staggered launch)
        if (!__syncthreads_or(in_seg || pending || stage < 3)) break;
        const bool mine = in_seg && !e.done && e.k < ke;
        if (actor_half && __any_sync(0xffffffffu, mine)) actor_forward<H>(actfn, w, L, lane, xb, obs, a);
        if ((!stagger || !actor_half) && mine) env_step<TABS, GUST, TRACK, PER_ACTOR, INC, SYM>(e, ar, traj, actor, replay, a, obs, last_u);
        actor_half ^= stagger;
    }
}

// ---- cross-check kernel: every thread evaluates the whole MLP for its own env (any hidden size that fits) ------
// TRACK, PER_ACTOR, INC, SYM as in rollout_kernel_persist; the gust schedule is always compiled in
template <bool TRACK = false, bool PER_ACTOR = false, bool INC = false, bool SYM = false>
__global__ void __launch_bounds__(128)
rollout_kernel_simple(RolloutArgs ar, TrackArgs tk)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* w = reinterpret_cast<float*>(smem_raw);
    const int P4 = (ar.P + 3) & ~3;
    float* bufA = w + P4;
    float* bufB = bufA + ar.sh.hidden * 128;
    const int actor = blockIdx.y, tid = threadIdx.x;
    const int eslot = blockIdx.x * 128 + tid;
    const float* gw = ar.weights + (size_t)actor * ar.P;
    for (int i = tid; i < ar.P; i += 128) w[i] = gw[i];
    __syncthreads();
    if (eslot >= ar.n_envs) return;
    const int env = ar.env_order ? ar.env_order[eslot] : eslot;
    Env e;
    e.tab = plant_tables_blob;
    float obs[SYM ? 2 : INC ? 10 : 7], a[3];
    double last_u[3];                                  // INC only
    const int row = PER_ACTOR ? actor * ar.n_envs + env : env;
    env_bind<true>(e, ar, row, &plant_pv[0][0], (size_t)actor * ar.n_envs + env);
    env_reset<false, true, TRACK, INC, SYM>(e, ar, row, obs, (size_t)actor * ar.n_envs + env, last_u);
    const size_t traj = (size_t)actor * ar.n_envs + env;
    const bool replay = ar.replay != nullptr && env == ar.replay_env;
    while (!e.done) {
        actor_forward_simple(w, ar.sh, bufA, bufB, tid, 128, obs, a);
        env_step<false, true, TRACK, PER_ACTOR, INC, SYM>(e, ar, traj, actor, replay, a, obs, last_u);   // (the gust schedule costs nothing that matters here)
    }
    traj_store(e, ar, traj);
    if constexpr (TRACK) track_store(e, tk, traj);
}

// ---- Actor.forward for a batch of observations (same device functions as the rollout) --------------------------
// S: observation entries (7, 10 with incremental control, 2 with symmetric control); A: actions (3, or 1 with symmetric control)
template <int H, int S = 7, int A = 3>
__global__ void __launch_bounds__(128)
actor_forward_kernel(const float* __restrict__ genome, int P, serl_actor_shape sh, const float* __restrict__ obs_in, int n,
                     float* __restrict__ act_out)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* w = reinterpret_cast<float*>(smem_raw);
    const int tid = threadIdx.x, lane = tid & 31;
    float* xb = w + ((P + 3) & ~3) + (tid >> 5) * (S == 7 ? actor_xbuf_floats(H) : actor_xbuf_floats(H, S));      // after the genome
    for (int i = tid; i < P; i += 128) w[genome_layout_index(i, sh.state_dim, H, sh.num_layers)] = genome[i];
    __syncthreads();
    const int base = (blockIdx.x * 128 + (tid & ~31));
    if (base >= n) return;
    const int i = base + lane;
    float obs[S], a[A];
#pragma unroll
    for (int k = 0; k < S; ++k) obs[k] = i < n ? obs_in[(size_t)i * S + k] : 0.f;
    actor_forward<H>(sh.activation, w, sh.num_layers, lane, xb, obs, a);
    if constexpr (A == 1) {
        if (i < n) act_out[i] = a[0];
    } else {
        if (i < n) { act_out[(size_t)i * 3] = a[0]; act_out[(size_t)i * 3 + 1] = a[1]; act_out[(size_t)i * 3 + 2] = a[2]; }
    }
}

template <int S = 7, int A = 3>
__global__ void __launch_bounds__(128)
actor_forward_kernel_simple(const float* __restrict__ genome, int P, serl_actor_shape sh, const float* __restrict__ obs_in, int n,
                            float* __restrict__ act_out)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* w = reinterpret_cast<float*>(smem_raw);
    float* bufA = w + ((P + 3) & ~3);
    float* bufB = bufA + sh.hidden * 128;
    const int tid = threadIdx.x;
    for (int i = tid; i < P; i += 128) w[i] = genome[i];
    __syncthreads();
    const int i = blockIdx.x * 128 + tid;
    if (i >= n) return;
    float obs[S], a[A];
    for (int k = 0; k < S; ++k) obs[k] = obs_in[(size_t)i * S + k];
    actor_forward_simple(w, sh, bufA, bufB, tid, 128, obs, a);
    if constexpr (A == 1) act_out[i] = a[0];
    else { act_out[(size_t)i * 3] = a[0]; act_out[(size_t)i * 3 + 1] = a[1]; act_out[(size_t)i * 3 + 2] = a[2]; }
}
// fitness[a] = mean over envs of returns[a, :]  (base/core/agent.py:245, np.mean over the evaluation axis)
__global__ void fitness_mean_kernel(const double* __restrict__ returns, int pop, int n_envs, double* __restrict__ fitness)
{
    const int a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= pop) return;
    double s = 0.0;
    for (int e = 0; e < n_envs; ++e) s += returns[(size_t)a * n_envs + e];
    fitness[a] = s / (double)n_envs;
}

// batched native-plant step: X[n,19] advanced in place by one major step with command cmd[n,3] (inputs 3..9 are 0)
__global__ void plant_step_kernel(double* __restrict__ X, const double* __restrict__ cmd, const int* __restrict__ variant,
                                  const int* __restrict__ call, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    PlantState x;
#pragma unroll
    for (int k = 0; k < NX; ++k) x.v[k] = X[(size_t)i * NX + k];
    const int post = (variant[i] >> 16) & 0xff;
    x = plant_step<false, true>(plant_pv[variant[i] & 0xff], x, cmd[3 * i], cmd[3 * i + 1], cmd[3 * i + 2], plant_tables_blob, false,
                                post ? plant_pv[post] : nullptr,
                                (call ? call[i] : 0) | ((variant[i] & SERL_MODE_GUST) ? PLANT_CALL_GUST : 0) |
                                    ((variant[i] & SERL_MODE_GUST_UP) ? PLANT_CALL_GUST_UP : 0));
#pragma unroll
    for (int k = 0; k < NX; ++k) X[(size_t)i * NX + k] = x.v[k];
}

__global__ void plant_ic_kernel(double* __restrict__ X, const int* __restrict__ variant, int n)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double* ic = plant_ic(variant[i] & 0xff);
    for (int k = 0; k < NX; ++k) X[(size_t)i * NX + k] = ic[k];
}

extern "C" int serl_plant_init(double* d_X, const int32_t* d_variant, int32_t n, void* stream)
{
    if (!d_X || !d_variant || n <= 0) return serl_fail(SERL_ERR_ARG, "serl_plant_init: bad argument");
    return serl_launch("plant_ic_kernel", plant_ic_kernel, (n + 127) / 128, 128, 0, (cudaStream_t)stream, d_X, d_variant, n);
}

// both step APIs: the timed one passes every env's native call index, the plain one none (every step is call 0)
static int plant_step_launch(bool timed, double* d_X, const double* d_cmd, const int32_t* d_variant, const int32_t* d_call, int32_t n,
                             void* stream)
{
    if (!d_X || !d_cmd || !d_variant || (timed && !d_call) || n <= 0)
        return serl_fail(SERL_ERR_ARG, timed ? "serl_plant_step_timed: bad argument" : "serl_plant_step: bad argument");
    return serl_launch("plant_step_kernel", plant_step_kernel, (n + 63) / 64, 64, 0, (cudaStream_t)stream, d_X, d_cmd, d_variant, d_call, n);
}

extern "C" int serl_plant_step(double* d_X, const double* d_cmd, const int32_t* d_variant, int32_t n, void* stream)
{
    return plant_step_launch(false, d_X, d_cmd, d_variant, nullptr, n, stream);
}

extern "C" int serl_plant_step_timed(double* d_X, const double* d_cmd, const int32_t* d_variant, const int32_t* d_call, int32_t n, void* stream)
{
    return plant_step_launch(true, d_X, d_cmd, d_variant, d_call, n, stream);
}

extern "C" int64_t serl_actor_num_params(const serl_actor_shape* s)
{
    if (!s) return -1;
    const int64_t S = s->state_dim, A = s->action_dim, H = s->hidden, L = s->num_layers;
    return S * H + H + L * (H * H + 3 * H) + H * A + A;
}

static int env_int(const char* name)
{
    const char* v = getenv(name);
    return v ? atoi(v) : 0;
}

// SERL_ROLLOUT_IMPL=simple: every launch of the uniform actor takes the one-thread-per-env kernels (cross-check)
static bool force_simple()
{
    static const bool v = [] { const char* s = getenv("SERL_ROLLOUT_IMPL"); return s && strcmp(s, "simple") == 0; }();
    return v;
}

// the uniform actors of the PH-LAB tasks the kernels of this file implement
static bool actor_shape_ok(const serl_actor_shape& sh)
{
    return task_of_shape(sh) && sh.hidden >= 2 && sh.hidden <= 256 && sh.num_layers >= 0 && sh.activation >= 0 && sh.activation <= 2;
}

// CTA shape of the persistent kernel: `apc` genome slots x `wps` warps.  A slot's warps fly wps*32 envs of one actor;
// the estimate below is (rounds of work per slot) x (time of one step with apc*wps resident warps per SM), the latter a
// least-squares fit (ms per 2001-step horizon) of single-round launches at apc x wps = 1x1 .. 2x4 (config 2: pop 50 x 64
// envs, and pop 64 x 128 envs; H100 SXM, 400 W power limit, SERL_ROLLOUT_APC / SERL_ROLLOUT_WPS): flat from 1 to 4 warps,
// a lone warp 1.15x faster than one of eight.
static void choose_shape(int pop, int n_envs, int apc_max, int sms, int* apc_out, int* wps_out)
{
    double best = 1e300;
    *apc_out = 1; *wps_out = 1;
    const int max_wps = (n_envs + 31) / 32;
    for (int wps = 4; wps >= 1; wps >>= 1) {
        if (wps > max_wps && wps > 1) continue;
        const long long chunks = (n_envs + wps * 32 - 1) / (wps * 32);
        const long long nt = (long long)pop * chunks;
        for (int apc = apc_max; apc >= 1; --apc) {
            if (apc * wps * 32 > MAX_CTA_THREADS) continue;
            const long long grid = nt / apc < sms ? (nt + apc - 1) / apc : sms;
            const long long ns = grid * apc;
            const double rounds = nt <= ns ? 1.0 : (double)nt / (double)ns;
            const double lanes = (double)chunks * wps * 32 / n_envs;        // idle-lane overhead of a ragged last chunk
            const double est = rounds * (166.5 + 4.1 * apc * wps) * (lanes > 1.0 ? 1.0 + 0.2 * (lanes - 1.0) : 1.0);
            if (est < best - 1e-9) { best = est; *apc_out = apc; *wps_out = wps; }
        }
    }
}

template <int H, bool TABS>
static int launch_persist(RolloutArgs& ar, TrackArgs tk, int apc_max, bool stagger, const RolloutVariant& v, cudaStream_t s)
{
    const int sms = ar.sm_limit > 0 && ar.sm_limit < serl_device_sms() ? ar.sm_limit : serl_device_sms();
    int apc, wps;
    choose_shape(ar.pop, ar.n_envs, apc_max, sms, &apc, &wps);
    static int f_apc = -1, f_wps = -1;       // experiment knobs
    if (f_apc < 0) { f_apc = env_int("SERL_ROLLOUT_APC"); f_wps = env_int("SERL_ROLLOUT_WPS"); }
    if (f_apc > 0 && f_apc <= apc_max) apc = f_apc;
    if (f_wps == 1 || f_wps == 2 || f_wps == 4) wps = f_wps;
    while (apc * wps * 32 > MAX_CTA_THREADS) --apc;
    ar.apc = apc; ar.wps = wps;
    ar.stagger = apc == 2 && stagger;
    ar.n_chunks = (ar.n_envs + wps * 32 - 1) / (wps * 32);
    ar.n_tasks = (long long)ar.pop * ar.n_chunks;
    const long long grid = ar.n_tasks / apc < sms ? (ar.n_tasks + apc - 1) / apc : sms;
    ar.n_slots = grid * apc;
    // scratch: genomes in the shared-memory layout + hand-over records of the time-split schedule (stream-ordered)
    const size_t wt_bytes = (size_t)ar.pop * ar.P4 * 4;
    const long long hn = ar.n_tasks > ar.n_slots ? ar.n_slots * wps * 32 : 0;
    // a record's observation: the task's observation floats, and last_u (3 f64) with incremental control (Handoff.obs).  A
    // tracking record (tk.ho) follows the flags, after all of these: an incremental-control tracking launch carries both
    const size_t ho_obs = (size_t)v.task.obs * 4 + (v.task.inc ? 3 * 8 : 0);
    const size_t ho_bytes = (size_t)hn * (NX * 8 + 8 + 8 + ho_obs + 4) + (size_t)(hn / 32) * 4 + (tk.out ? (size_t)hn * TRACK_CARRY * 8 + 8 : 0);
    void* scratch = nullptr;
    cudaError_t e = serl_scratch(SERL_SCRATCH_K1, s, wt_bytes + ho_bytes + 512, &scratch);
    if (e != cudaSuccess) return serl_fail_cuda(e, "rollout_kernel launch");
    unsigned char* base = (unsigned char*)scratch;
    float* wt = (float*)base;
    ar.wt = wt;
    ar.ho.n = hn;
    if (hn) {
        unsigned char* p = base + ((wt_bytes + 255) & ~(size_t)255);
        ar.ho.X = (double*)p; p += (size_t)hn * NX * 8;
        ar.ho.t = (double*)p; p += (size_t)hn * 8;
        ar.ho.ret = (double*)p; p += (size_t)hn * 8;
        ar.ho.obs = (float*)p; p += (size_t)hn * ho_obs;
        ar.ho.k = (int*)p; p += (size_t)hn * 4;
        ar.ho.flag = (int*)p; p += (size_t)(hn / 32) * 4;
        if (tk.out) tk.ho = (double*)(((uintptr_t)p + 7) & ~(uintptr_t)7);
        e = cudaMemsetAsync(ar.ho.flag, 0, (size_t)(hn / 32) * 4, s);
        if (e != cudaSuccess) return serl_fail_cuda(e, "rollout_kernel launch");
    }
    const long long n = (long long)ar.pop * ar.P;
    const int lay_grid = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
    const int rc = serl_launch("genome_layout_kernel", genome_layout_kernel, lay_grid, 256, 0, s, ar.weights, wt, ar.pop, ar.P, ar.P4,
                               ar.sh.state_dim, H, ar.sh.num_layers);
    if (rc != SERL_OK) return rc;
    const size_t smem = (TABS ? (size_t)PLANT_TABN2 * sizeof(real) : 0) + (size_t)apc * ar.P4 * 4 +
                        (size_t)apc * wps * actor_xbuf_floats(H, v.task.obs) * 4;
    void (*kernel)(RolloutArgs, TrackArgs) = nullptr;
    visit_rollout_variant(v, [&](auto f) {
        using V = decltype(f);
        kernel = rollout_kernel_persist<H, TABS, V::GUST, V::TRACK, V::PER_ACTOR, V::INC, V::SYM>;
    });
    return serl_launch("rollout_kernel launch", kernel, (unsigned)grid, apc * wps * 32, smem, s, ar, tk);
}

// the hidden sizes the warp actor is instantiated for: when H is one of them, calls f(std::integral_constant<int, H>())
// and returns true
template <typename F>
static bool warp_hidden(int H, F&& f)
{
    switch (H) {
    case 32: f(std::integral_constant<int, 32>()); return true;
    case 64: f(std::integral_constant<int, 64>()); return true;
    case 72: f(std::integral_constant<int, 72>()); return true;
    case 96: f(std::integral_constant<int, 96>()); return true;
    case 128: f(std::integral_constant<int, 128>()); return true;
    }
    return false;
}
static bool warp_hidden(int H) { return warp_hidden(H, [](auto) {}); }

// Shared memory of the warp kernel: the plant tables (unless it reads them from global memory) and `apc` genome slots, a slot
// being the genome and the actor exchange buffers of up to 4 warps, within the opt-in limit less the static shared memory
// (128 B) and the alignment of the dynamic part
constexpr size_t K1_SMEM_BUDGET = SERL_SMEM_OPTIN - 256;
constexpr size_t K1_TAB_BYTES = (size_t)PLANT_TABN2 * sizeof(real);
static size_t k1_slot_bytes(const serl_actor_shape& sh)
{
    const size_t P4 = ((size_t)serl_actor_num_params(&sh) + 3) & ~(size_t)3;
    return P4 * 4 + 4ull * actor_xbuf_floats(sh.hidden, sh.state_dim) * 4;        // h = 128, L = 3: 218 KB
}

// K1's kernel for a valid shape: the warp actor when it can be launched — the hidden size is instantiated and one slot fits
// next to the plant tables, or h = 128, the one size also instantiated with the tables in global memory, and one slot fits
// alone — else the one-thread-per-env kernel, which needs the genome and two activation buffers of 128 envs in shared memory
static bool k1_warp(const serl_actor_shape& sh)
{
    if (force_simple() || !warp_hidden(sh.hidden)) return false;
    const size_t slot = k1_slot_bytes(sh);
    return K1_TAB_BYTES + slot <= K1_SMEM_BUDGET || (sh.hidden == 128 && slot <= K1_SMEM_BUDGET);
}
static bool k1_fits(const serl_actor_shape& sh)
{
    const size_t P4 = ((size_t)serl_actor_num_params(&sh) + 3) & ~(size_t)3;
    return k1_warp(sh) || P4 * 4 + 2ull * sh.hidden * 128 * 4 <= SERL_SMEM_OPTIN;
}

// Which kernel flies a uniform actor: 0 when K1 does (or reports why it cannot: a shape outside the task, L = 0), else
// the L + 1 widths [h] * (L + 1) of the same genome for K1-TC
extern "C" int32_t serl_actor_tc_widths(const serl_actor_shape* shape, int32_t* widths_out, int32_t cap)
{
    if (!shape) return serl_fail(SERL_ERR_ARG, "serl_actor_tc_widths: null shape");
    const serl_actor_shape& sh = *shape;
    const bool task = task_of_shape(sh) && sh.hidden >= 2 && sh.num_layers >= 1 && sh.activation >= 0 && sh.activation <= 2;
    if (!task || (actor_shape_ok(sh) && k1_fits(sh))) return 0;
    const int n = sh.num_layers + 1;
    if (!widths_out || cap < n) return serl_fail(SERL_ERR_ARG, "serl_actor_tc_widths: widths_out holds fewer than num_layers + 1 widths");
    for (int i = 0; i < n; ++i) widths_out[i] = sh.hidden;
    return n;
}

// K1 launch: the checks only this kernel needs, then the genome part of the argument block and the kernel for the hidden size
static int rollout_impl(const serl_rollout_desc& d, RolloutArgs ar, const RolloutVariant& v, cudaStream_t s)
{
    const TrackArgs tk = {d.d_track, nullptr, d.d_cost};
    if (!actor_shape_ok(d.shape))
        return serl_fail(SERL_ERR_ARG, "serl_rollout: unsupported actor shape (state_dim = 7 or 10 with action_dim = 3, or 2 with 1; 2 <= hidden <= 256)");
    if (d.pop > 65535) return serl_fail(SERL_ERR_ARG, "serl_rollout: pop must be <= 65535 per call");       // grid.y of the simple kernel
    if (d.horizon >= (1 << 30)) return serl_fail(SERL_ERR_ARG, "serl_rollout: horizon too long");        // Handoff.k: steps | done << 30
    const int H = d.shape.hidden;
    ar.weights = d.d_weights; ar.P = (int)serl_actor_num_params(&d.shape); ar.sh = d.shape;
    ar.P4 = (ar.P + 3) & ~3;
    if (!k1_warp(d.shape)) {
        if (!k1_fits(d.shape)) return serl_fail(SERL_ERR_UNSUPPORTED, "serl_rollout: genome + activations exceed 227 KB of shared memory");
        const size_t smem = (size_t)ar.P4 * 4 + 2ull * H * 128 * 4;
        void (*kernel)(RolloutArgs, TrackArgs) = nullptr;
        visit_rollout_variant(v, [&](auto f) {
            using V = decltype(f);
            kernel = rollout_kernel_simple<V::TRACK, V::PER_ACTOR, V::INC, V::SYM>;
        });
        return serl_launch("rollout_kernel launch", kernel, dim3((d.n_envs + 127) / 128, d.pop), 128, smem, s, ar, tk);
    }
    // as many genome slots per CTA as shared memory holds next to the plant tables (L = 3: two for h <= 72, one for h = 96);
    // h = 128 from L = 3 on (207 KB genome) reads the tables through L1 instead (k1_warp: every other shape has room for them)
    const size_t slot_bytes = k1_slot_bytes(d.shape);
    const bool tabs = K1_TAB_BYTES + slot_bytes <= K1_SMEM_BUDGET;
    int apc_max = (int)(((tabs ? K1_SMEM_BUDGET - K1_TAB_BYTES : K1_SMEM_BUDGET)) / slot_bytes);
    if (apc_max > 4) apc_max = 4;
    if (apc_max > 2 && H > 32) apc_max = 2;
    const bool stagger = (d.flags & SERL_ROLLOUT_STAGGER) != 0;
    int rc = SERL_OK;
    warp_hidden(H, [&](auto h) {
        constexpr int HH = decltype(h)::value;
        if constexpr (HH == 128)          // the one size instantiated with the tables in global memory too
            rc = tabs ? launch_persist<HH, true>(ar, tk, apc_max, stagger, v, s) : launch_persist<HH, false>(ar, tk, apc_max, stagger, v, s);
        else
            rc = launch_persist<HH, true>(ar, tk, apc_max, stagger, v, s);
    });
    return rc;
}

int rollout_tc_impl(const serl_rollout_desc& d, const RolloutArgs& r, const RolloutVariant& v, cudaStream_t s);     // rollout_tc.cu

// The checks of a launch description that hold for both kernels.  Besides the launch's own consistency they refuse every
// combination no kernel is instantiated for, so that visit_rollout_variant finds the variant of each description that passes.
static int check_desc(const serl_rollout_desc& d)
{
    if (!d.d_weights || !d.d_ref_levels || !d.d_ref_starts || !d.d_env_mode || !d.d_returns || !d.d_steps)
        return serl_fail(SERL_ERR_ARG, "serl_rollout: null pointer argument");
    if (d.pop <= 0 || d.n_envs <= 0 || d.horizon <= 0) return serl_fail(SERL_ERR_ARG, "serl_rollout: pop, n_envs, horizon must be > 0");
    if (d.shape.activation < 0 || d.shape.activation > 2) return serl_fail(SERL_ERR_ARG, "serl_rollout: unsupported activation");
    if (d.d_replay && (d.replay_env < 0 || d.replay_env >= d.n_envs)) return serl_fail(SERL_ERR_ARG, "serl_rollout: replay_env out of range");
    if (d.t_max > 0.0 && !(d.smooth_width > 0.0)) return serl_fail(SERL_ERR_ARG, "serl_rollout: smooth_width must be > 0");
    if (d.n_widths > 0 && !d.widths) return serl_fail(SERL_ERR_ARG, "serl_rollout: n_widths > 0 but widths is null");
    // the tally is counted by the tracking instantiations only
    if (d.d_cost && !d.d_track) return serl_fail(SERL_ERR_ARG, "serl_rollout: d_cost needs d_track");
    if (d.flags & SERL_ROLLOUT_PER_ACTOR_REFS) {
        // inside one actor's block the lanes of a warp already share a mode: no lane permutation
        if (d.d_env_order) return serl_fail(SERL_ERR_ARG, "serl_rollout: SERL_ROLLOUT_PER_ACTOR_REFS does not take d_env_order");
        if (d.d_track) return serl_fail(SERL_ERR_ARG, "serl_rollout: SERL_ROLLOUT_PER_ACTOR_REFS does not take d_track");
        if ((int64_t)d.pop * d.n_envs > INT32_MAX) return serl_fail(SERL_ERR_ARG, "serl_rollout: pop * n_envs must fit int32 with per-actor refs");
    }
    // the evaluation suite / operator study of incremental or symmetric control: a launch of exactly one of the two modes
    const bool suite = (d.flags & SERL_ROLLOUT_SUITE) != 0;
    if (suite && ((d.flags & SERL_ROLLOUT_INCREMENTAL) != 0) == ((d.flags & SERL_ROLLOUT_SYMMETRIC) != 0))
        return serl_fail(SERL_ERR_ARG, "serl_rollout: SERL_ROLLOUT_SUITE needs exactly one of SERL_ROLLOUT_INCREMENTAL / SERL_ROLLOUT_SYMMETRIC");
    // incremental control: a 10-entry observation, on the training instantiations of K1 and K1-TC (and their tracking
    // instantiations in suite launches)
    if (d.flags & SERL_ROLLOUT_INCREMENTAL) {
        if (d.shape.state_dim != TASK_INCREMENTAL.obs) return serl_fail(SERL_ERR_ARG, "serl_rollout: incremental control (SERL_ROLLOUT_INCREMENTAL) needs state_dim = 10");
        if (!suite && (d.d_track || d.d_cost))
            return serl_fail(SERL_ERR_ARG, "serl_rollout: incremental control (SERL_ROLLOUT_INCREMENTAL) does not take d_track / d_cost");
        if (d.flags & SERL_ROLLOUT_GUST) return serl_fail(SERL_ERR_ARG, "serl_rollout: incremental control (SERL_ROLLOUT_INCREMENTAL) does not take SERL_ROLLOUT_GUST");
        if (d.d_sensor_noise) return serl_fail(SERL_ERR_ARG, "serl_rollout: incremental control (SERL_ROLLOUT_INCREMENTAL) does not take d_sensor_noise");
    } else if (d.n_widths == 0 && d.shape.state_dim == TASK_INCREMENTAL.obs) {
        return serl_fail(SERL_ERR_ARG, "serl_rollout: state_dim = 10 is the observation of incremental control: it needs SERL_ROLLOUT_INCREMENTAL");
    }
    // symmetric control: a 2-entry observation and one action, on the training instantiations of K1 and K1-TC (and, in suite
    // launches, their tracking instantiations, which carry the gust schedule, and the sensor-noise shim of every instantiation)
    if (d.flags & SERL_ROLLOUT_SYMMETRIC) {
        if (d.shape.state_dim != TASK_SYMMETRIC.obs || d.shape.action_dim != TASK_SYMMETRIC.act)
            return serl_fail(SERL_ERR_ARG, "serl_rollout: symmetric control (SERL_ROLLOUT_SYMMETRIC) needs state_dim = 2 and action_dim = 1");
        if (d.flags & SERL_ROLLOUT_INCREMENTAL)
            return serl_fail(SERL_ERR_ARG, "serl_rollout: symmetric control (SERL_ROLLOUT_SYMMETRIC) does not take SERL_ROLLOUT_INCREMENTAL");
        if (!suite && (d.d_track || d.d_cost))
            return serl_fail(SERL_ERR_ARG, "serl_rollout: symmetric control (SERL_ROLLOUT_SYMMETRIC) does not take d_track / d_cost");
        if (!suite && (d.flags & SERL_ROLLOUT_GUST))
            return serl_fail(SERL_ERR_ARG, "serl_rollout: symmetric control (SERL_ROLLOUT_SYMMETRIC) does not take SERL_ROLLOUT_GUST");
        if ((d.flags & SERL_ROLLOUT_GUST) && !d.d_track)
            return serl_fail(SERL_ERR_ARG, "serl_rollout: symmetric control (SERL_ROLLOUT_SYMMETRIC | SERL_ROLLOUT_SUITE) takes SERL_ROLLOUT_GUST with d_track only");
        if (!suite && d.d_sensor_noise)
            return serl_fail(SERL_ERR_ARG, "serl_rollout: symmetric control (SERL_ROLLOUT_SYMMETRIC) does not take d_sensor_noise");
    } else if (d.n_widths == 0 && task_of_shape(d.shape) == &TASK_SYMMETRIC) {
        return serl_fail(SERL_ERR_ARG, "serl_rollout: state_dim = 2, action_dim = 1 is the actor of symmetric control: it needs SERL_ROLLOUT_SYMMETRIC");
    }
    return SERL_OK;
}

// the env / output part of the argument block, the same for both kernels; t_max <= 0 selects the training episode
static RolloutArgs rollout_args(const serl_rollout_desc& d)
{
    RolloutArgs ar;
    memset(&ar, 0, sizeof(ar));
    ar.ref_levels = d.d_ref_levels; ar.ref_starts = d.d_ref_starts; ar.env_mode = d.d_env_mode; ar.n_envs = d.n_envs; ar.horizon = d.horizon;
    ar.action_noise = d.d_action_noise; ar.returns = d.d_returns; ar.steps = d.d_steps; ar.trace = d.d_trace; ar.actions = d.d_actions;
    ar.pop = d.pop;
    ar.t_max = d.t_max > 0.0 ? d.t_max : 20.0;
    ar.smooth_w = d.t_max > 0.0 ? d.smooth_width : 3.0;
    ar.env_order = d.d_env_order; ar.replay = d.d_replay; ar.replay_env = d.replay_env; ar.status = d.d_status; ar.sm_limit = d.sm_limit;
    ar.sensor_noise = d.d_sensor_noise;
    return ar;
}

// Every population rollout comes through here: the shared checks, the task and kernel variant they leave, the kernel of the
// actor form (widths: K1-TC, else K1), whose own checks also come before any CUDA call, then the per-actor fitness.
extern "C" int serl_rollout_run(const serl_rollout_desc* desc, void* stream)
{
    if (!desc) return serl_fail(SERL_ERR_ARG, "serl_rollout_run: null descriptor");
    const serl_rollout_desc& d = *desc;
    int rc = check_desc(d);
    if (rc != SERL_OK) return rc;
    cudaStream_t s = (cudaStream_t)stream;
    const RolloutVariant v = rollout_variant(d, task_of_flags(d.flags));
    rc = d.n_widths > 0 ? rollout_tc_impl(d, rollout_args(d), v, s) : rollout_impl(d, rollout_args(d), v, s);
    if (rc != SERL_OK || !d.d_fitness) return rc;
    return serl_launch("fitness_mean_kernel launch", fitness_mean_kernel, (d.pop + 127) / 128, 128, 0, s, d.d_returns, d.pop, d.n_envs,
                       d.d_fitness);
}

extern "C" int serl_actor_forward(const float* d_genome, const serl_actor_shape* shape, const float* d_obs, int32_t n,
                                  float* d_actions, void* stream)
{
    if (!d_genome || !shape || !d_obs || !d_actions || n <= 0) return serl_fail(SERL_ERR_ARG, "serl_actor_forward: bad argument");
    if (!actor_shape_ok(*shape)) return serl_fail(SERL_ERR_ARG, "serl_actor_forward: unsupported actor shape");
    cudaStream_t s = (cudaStream_t)stream;
    const int P = (int)serl_actor_num_params(shape), H = shape->hidden;
    const RolloutTask& task = *task_of_shape(*shape);
    const int grid = (n + 127) / 128;
    const size_t smem = (size_t)((P + 3) & ~3) * 4;
    int rc = SERL_OK;
    const size_t warp_smem = smem + 4ull * actor_xbuf_floats(H, task.obs) * 4;      // genome + 4 warps' buffers
    const auto warp_launch = [&](auto h) {
        visit_task(task, [&](auto S, auto A) {
            rc = serl_launch("actor_forward_kernel", actor_forward_kernel<decltype(h)::value, decltype(S)::value, decltype(A)::value>,
                             grid, 128, warp_smem, s, d_genome, P, *shape, d_obs, n, d_actions);
        });
    };
    // the warp kernel when it holds the genome, else the one-thread-per-env kernel (no static shared memory in either)
    if (!force_simple() && warp_smem <= SERL_SMEM_OPTIN && warp_hidden(H, warp_launch)) return rc;
    const size_t sm2 = smem + 2ull * H * 128 * 4;
    if (sm2 > SERL_SMEM_OPTIN) return serl_fail(SERL_ERR_UNSUPPORTED, "serl_actor_forward: genome + activations exceed shared memory");
    visit_task(task, [&](auto S, auto A) {
        rc = serl_launch("actor_forward_kernel", actor_forward_kernel_simple<decltype(S)::value, decltype(A)::value>,
                         grid, 128, sm2, s, d_genome, P, *shape, d_obs, n, d_actions);
    });
    return rc;
}
