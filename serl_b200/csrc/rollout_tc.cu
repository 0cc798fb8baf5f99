// K1-TC — population rollout for WIDE actors (BASELINE config 5: hidden = [400,300] / [128,128]; the reference's Actor
// beyond hidden 128) on the tensor cores of sm_90a (warpgroup MMA, wgmma).
//
//   actor  Linear(7,w1) -> act -> Linear(w1,w2) -> LayerNorm(w2) -> act -> Linear(w2,3) -> tanh
//          (the two-hidden-layer generalisation of base/core/genetic_agent.py:78-101; LayerNorm base/core/mod_utils.py:47-50)
//   deep   [w0, w1, ..., w_{n-1}], 3 <= n <= 9: every Linear(w_{l-1},w_l) LayerNorm act on the tensor cores in turn
//          (tc_actor_forward_deep; the reference's Actor with num_layers = L is [h] * (L + 1))
//
// The description below is the two-width forward pass (tc_actor_forward); the deep one adds a layer loop around it.
//
// One CTA per SM = 256 threads = two GROUPS of 128 threads (one warpgroup each); a group = 128 envs of one actor
// (thread = env).  The two groups run independent task loops, share the plant tables in shared memory and the A / W1 rings,
// and take turns on the rings (a shared-memory lock): while one group streams its W1 slabs through the tensor cores the
// other integrates its plant step.  Per step of a group, for each half of 64 envs (the M of one wgmma):
//   layer 1   on CUDA cores, 8 neurons at a time (two threads per env, 4 neurons each): the activations, split into
//             TF32 hi + lo parts, are written as one K-slab of the A operand in shared memory (canonical K-major layout,
//             no swizzle);
//   layer 2   D[64 x w2] += A[64 x 8] . W1^T[8 x w2]  by wgmma.mma_async m64n64k8 .tf32 (fp32 accumulator in registers,
//             n2pad / 2 per thread), three products per slab (hi.hi + hi.lo + lo.hi = "3xTF32", fp32-level accuracy); the
//             W1 K-slabs (pre-split and pre-tiled once per launch) are STREAMED from L2 into a 4-stage shared-memory ring by
//             bulk TMA copies (cp.async.bulk + mbarrier complete_tx), two stages ahead — a [400,300] genome is 500 KB and
//             never fits on chip; wgmma.wait_group tells when a ring slot's MMAs have read it;
//   epilogue  from the accumulator fragment (a row lives in the 4 lanes of a quad): bias, LayerNorm (quad shuffles for the
//             row sums), activation, and the 3-row output layer folded into the same pass;
//   plant     CitationEnv.step + the ode5 plant step on CUDA cores (plant_env.cuh), exactly as in K1.
//
// Numerics: tensor-core accumulation order is not reproducible on a CPU, so this path is checked against the torch fp32
// oracle with a tolerance (tests/test_wide_actor_gpu.py), not bit for bit like K1.
#include "plant_env.cuh"
#include "rollout_variant.h"

#define TC_THREADS 128             // a group: one warpgroup
#define TC_M 64                    // rows (envs) of one wgmma
#define TC_STAGES 4
#define TC_KSLAB 8                 // K values per pipeline stage (the wgmma K step for TF32)
#define TC_CH (TC_KSLAB / 4)        // 16-byte K chunks (4 TF32 values) per stage
#define TC_NCH 64                  // accumulator columns per wgmma
#define TC_MAXN 320                // largest padded width of a tensor-core layer
#define TC_MAXL 8                  // tensor-core layers (n_widths - 1) of the deepest list

// tensor-core layer l (1 <= l < n_widths): D[64 x w] = A[64 x win] . W_l^T, then bias, LayerNorm, activation
struct TcLayer {
    int w, npad;                   // output width, padded to TC_NCH (zero neurons)
    int win, n_stages;             // real input width; K-slabs of TC_KSLAB (input padded to a multiple of TC_KSLAB)
    int stage_floats;              // one K-slab: hi[2][npad][4] + lo[2][npad][4]
    int vec;                       // small block: b[npad] gamma[npad] beta[npad] start here
    int tile;                      // per-actor tile block: the layer's K-slabs start here
    int gW;                        // genome: W_l[w][win] b[w] gamma[w] beta[w] start here
};

struct TcArgs {
    RolloutArgs r;                 // env / output part (weights, wt, P4, apc ... unused)
    int w1, w2, n2pad;             // layer widths (w1 already padded to a multiple of TC_KSLAB with zero neurons); w2 padded to TC_NCH
    int w1_real;
    int small_floats;              // per-actor small parameter block (floats, multiple of 4)
    int stage_floats;              // B ring slot: the largest K-slab of any layer (two widths: the W1 slab hi[2][n2pad][4] + lo[2][n2pad][4])
    const float* small;            // [pop][small_floats]
    const float* tiles;            // [pop][tile_floats]
    long long n_tasks; int n_chunks;
    // forward-only mode (serl_actor_forward_wide)
    const float* obs_in; float* act_out; int n_obs;
    // every width list: the layer table (K0-TC); more than two widths also fly it (tc_actor_forward_deep)
    int n_layers;                  // n_widths - 1
    int stages;                    // K-slabs of one forward pass of 64 rows (all layers)
    int tile_floats;               // per-actor tile block
    int abuf_stride;               // row stride of the inter-layer activation buffer (floats)
    int gWo;                       // genome: Wo[3][w_last] bo[3] (symmetric control: Wo[1][w_last] bo[1])
    TcLayer ly[TC_MAXL];
};

__device__ __forceinline__ float rn_tf32(float x)       // round to nearest TF32 (10-bit mantissa), ties away
{
    return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xffffe000u);
}

// Row width of W0p in the small block and of the group's observations in shared memory: 8 floats for the 7-entry
// observation, 12 for the 10 of incremental control (SERL_ROLLOUT_INCREMENTAL: + last_u), 4 for the 2 of symmetric control
// (SERL_ROLLOUT_SYMMETRIC: 2 weights + bias + 0); float4-aligned in every case
__host__ __device__ constexpr int tc_row(int S) { return S == 7 ? 8 : S == 2 ? 4 : 12; }

// small block layout (floats): W0p[w0pad][8] (7 weights + bias; S = 10: [w0pad][12], 10 weights + bias + 0) | per layer l: b[npad] gamma[npad] beta[npad] |
// Wo[3][npad of the last layer] | bo[4].  With two widths [w1, w2] this is W0p[w1][8] | b1 | gamma | beta | Wo | bo.
// A genome with one output (symmetric control) fills Wo's row 0 and bo[0]; rows 1-2 and bo[1..3] are zero neurons, so the
// output block's actions 1-2 are tanh(0) = 0 and nobody reads them.
// Tile block: per layer l, n_stages K-slabs of stage_floats (pre-split TF32 hi / lo, canonical K-major core matrices).

// K0-TC: genome (parameters() order: W0[w0,S] b0[w0], per layer W_l[w_l,w_{l-1}] b gamma beta, Wo[3,w_last] bo[3]) -> small
// block + tile block.  Rows and columns past a layer's real width are zero neurons: zero weights, bias, gamma and beta.
// A: the genome's outputs (3, or 1 with symmetric control); the small block's output rows past A are zero.
template <int S = 7, int A = 3>
__global__ void tc_layout_kernel(const float* __restrict__ w, int pop, int P, const __grid_constant__ TcArgs ar, float* __restrict__ small,
                                 float* __restrict__ tiles)
{
    const int w0 = ar.ly[0].win, w0pad = ar.ly[0].n_stages * TC_KSLAB;
    const TcLayer& last = ar.ly[ar.n_layers - 1];
    const int wo = last.vec + 3 * last.npad;                       // small block: Wo, then bo at wo + 3 npad
    const long long per = (long long)ar.small_floats + ar.tile_floats;
    const long long total = (long long)pop * per;
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
        const int a = (int)(g / per);
        const int i = (int)(g - (long long)a * per);
        const float* ga = w + (size_t)a * P;
        float v = 0.f;
        if (S == 7 && i < w0pad * 8) {
            const int k = i >> 3, c = i & 7;
            v = k >= w0 ? 0.f : (c < 7 ? ga[k * 7 + c] : ga[7 * w0 + k]);
        } else if (S != 7 && i < w0pad * tc_row(S)) {
            const int k = i / tc_row(S), c = i - k * tc_row(S);
            v = k >= w0 || c > S ? 0.f : (c < S ? ga[k * S + c] : ga[S * w0 + k]);
        } else if (i < wo) {
            int l = 0;
            while (i >= ar.ly[l].vec + 3 * ar.ly[l].npad) ++l;
            const TcLayer& L = ar.ly[l];
            const int r = i - L.vec, which = r / L.npad, n = r - which * L.npad;      // which: b, gamma, beta
            v = n < L.w ? ga[L.gW + L.w * L.win + which * L.w + n] : 0.f;
        } else if (i < wo + 3 * last.npad) {
            const int r = i - wo, j = r / last.npad, n = r - j * last.npad;
            v = n < last.w && (A == 3 || j < A) ? ga[ar.gWo + j * last.w + n] : 0.f;
        } else if (i < ar.small_floats) {
            const int r = i - wo - 3 * last.npad;
            v = r < A ? ga[ar.gWo + A * last.w + r] : 0.f;
        } else {
            const int t = i - ar.small_floats;
            int l = 0;
            while (l + 1 < ar.n_layers && t >= ar.ly[l + 1].tile) ++l;
            const TcLayer& L = ar.ly[l];
            const int s = (t - L.tile) / L.stage_floats;
            int r = t - L.tile - s * L.stage_floats;
            const int half = TC_CH * L.npad * 4;
            const int part = r / half;
            r -= part * half;
            const int j = r / (L.npad * 4), n = (r >> 2) % L.npad, kk = r & 3;
            const int k = s * TC_KSLAB + j * 4 + kk;
            const float x = (n < L.w && k < L.win) ? ga[L.gW + n * L.win + k] : 0.f;
            const float hi = rn_tf32(x);
            tiles[(size_t)a * ar.tile_floats + t] = part == 0 ? hi : rn_tf32(x - hi);
            continue;
        }
        small[(size_t)a * ar.small_floats + i] = v;
    }
}

// ---- wgmma primitives -----------------------------------------------------------------------------------------
// shared-memory matrix descriptor, K-major, no swizzle: core matrix = 8 rows x 16 bytes (contiguous 128 B);
// SBO = byte distance between 8-row groups, LBO = byte distance between the two 16-byte K chunks of one MMA K step
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes)
{
    return (uint64_t)((smem_addr & 0x3ffffu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}
// D[64 x 64] (+)= A[64 x 8] . B[64 x 8]^T, TF32 inputs, FP32 accumulator in registers (the m64n64 fragment: lane l of warp w
// of the warpgroup holds rows 16w + l/4 and 16w + l/4 + 8, columns 8i + 2(l%4) + {0,1}, i = 0..7, as d[4i + {0,1,2,3}])
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1;\n\t"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

struct TcCtx {
    const float* small;            // small parameter block of the current actor (smem; global, read through L1, when deep)
    float* abuf;                   // smem, deep lists: the inter-layer activations [64][abuf_stride] of the lock holder
    float* io;                     // smem: the group's observations [128][8] and actions [128][4]
    float* a_ring;                 // smem: TC_STAGES x { hi[2][64][4], lo[2][64][4] }
    float* b_ring;                 // smem: TC_STAGES x stage_floats
    uint64_t* full_b;              // [TC_STAGES] TMA landed
    uint32_t g;                    // stages issued so far (valid while the group holds the lock)
    uint32_t* shared_state;        // smem: {lock, g} shared by the two groups
    int grp, gtid;                 // group of this thread (0/1), thread index inside the group
};

__device__ __forceinline__ void group_sync(int grp) { asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(TC_THREADS) : "memory"); }
__device__ __forceinline__ bool group_any(int grp, bool pred)
{
    uint32_t r;
    asm volatile("{\n\t.reg .pred p, q;\n\tsetp.ne.u32 q, %1, 0;\n\tbar.red.or.pred p, %2, %3, q;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(r) : "r"((uint32_t)pred), "r"(3 + grp), "r"(TC_THREADS) : "memory");
    return r != 0;
}
// the A / W1 rings and their barriers belong to one group at a time
__device__ __forceinline__ void tc_acquire(TcCtx& c)
{
    if (c.gtid == 0) {
        while (atomicCAS(&c.shared_state[0], 0u, 1u) != 0u) __nanosleep(100);
        __threadfence_block();
    }
    group_sync(c.grp);
    c.g = *reinterpret_cast<volatile uint32_t*>(&c.shared_state[1]);
}
__device__ __forceinline__ void tc_release(TcCtx& c)
{
    group_sync(c.grp);                       // every warp of the group has retired its MMAs
    if (c.gtid == 0) {
        c.shared_state[1] = c.g;
        __threadfence_block();
        atomicExch(&c.shared_state[0], 0u);
    }
}

// layer 0 of neuron row `wr` of W0p (CUDA cores): bias, then fma over the S observation entries in index order
template <int S>
__device__ __forceinline__ float tc_layer0(const float* wr, const float (&ob)[S])
{
    const float4 wa = *reinterpret_cast<const float4*>(wr);
    const float4 wb = *reinterpret_cast<const float4*>(wr + 4);
    if constexpr (S == 7) {
        float a = wb.w;                                              // bias
        a = __fmaf_rn(wa.x, ob[0], a); a = __fmaf_rn(wa.y, ob[1], a); a = __fmaf_rn(wa.z, ob[2], a);
        a = __fmaf_rn(wa.w, ob[3], a); a = __fmaf_rn(wb.x, ob[4], a); a = __fmaf_rn(wb.y, ob[5], a);
        a = __fmaf_rn(wb.z, ob[6], a);
        return a;
    } else if constexpr (S == 2) {
        float a = wa.z;                                              // bias (wb is not read)
        a = __fmaf_rn(wa.x, ob[0], a); a = __fmaf_rn(wa.y, ob[1], a);
        return a;
    } else {
        const float4 wc = *reinterpret_cast<const float4*>(wr + 8);
        float a = wc.z;                                              // bias
        a = __fmaf_rn(wa.x, ob[0], a); a = __fmaf_rn(wa.y, ob[1], a); a = __fmaf_rn(wa.z, ob[2], a);
        a = __fmaf_rn(wa.w, ob[3], a); a = __fmaf_rn(wb.x, ob[4], a); a = __fmaf_rn(wb.y, ob[5], a);
        a = __fmaf_rn(wb.z, ob[6], a); a = __fmaf_rn(wb.w, ob[7], a); a = __fmaf_rn(wc.x, ob[8], a);
        a = __fmaf_rn(wc.y, ob[9], a);
        return a;
    }
}

// one actor forward for the 128 envs of the group; every thread passes its own observation and receives its own action.
// The group's rows are done in two halves of TC_M = 64 (the M of one wgmma); each half streams all W1 slabs, so the
// accumulator of a thread is n2pad / 2 registers.
template <int ACT, int S = 7>
__device__ __forceinline__ void tc_actor_forward(TcCtx& c, const TcArgs& ar, const float* tiles_actor, const float* obs, float* action)
{
    const int tid = c.gtid, warp = tid >> 5, lane = tid & 31;
    const int w2 = ar.w2, n2pad = ar.n2pad, nch = n2pad / TC_NCH;
    const int n_stages = ar.w1 / TC_KSLAB, total = 2 * n_stages;
    const uint32_t stage_bytes = (uint32_t)ar.stage_floats * 4u;
    constexpr int A_STAGE_FLOATS = 2 * TC_CH * TC_M * 4;                   // hi + lo, TC_CH chunks x 64 rows x 4 floats
    const float* W0p = c.small;
    float* obs_s = c.io;
    float* act_s = c.io + TC_THREADS * tc_row(S);
#pragma unroll
    for (int k = 0; k < S; ++k) obs_s[tid * tc_row(S) + k] = obs[k];
    tc_acquire(c);                                                         // (its barrier publishes obs_s)
    const uint32_t g0 = c.g;
    // W1 slabs of the first two stages (their slots' MMAs retired before the lock was released)
    if (tid == 0) {
        for (int q = 0; q < 2 && q < total; ++q) {
            const uint32_t sl = (g0 + q) % TC_STAGES;
            mbar_expect_tx(&c.full_b[sl], stage_bytes);
            tma_bulk_g2s(c.b_ring + (size_t)sl * ar.stage_floats, tiles_actor + (size_t)(q % n_stages) * ar.stage_floats, stage_bytes, &c.full_b[sl]);
        }
    }
    const int rr = tid & (TC_M - 1), jj = tid >> 6;                         // layer 1: row rr of the half, K chunk jj of the slab
    const float* b1 = c.small + ar.w1 * tc_row(S);
    const float* gamma = b1 + n2pad;
    const float* beta = gamma + n2pad;
    const float* Wo = beta + n2pad;
    const float* bo = Wo + 3 * n2pad;
    float acc[TC_MAXN / 2];
    for (int h = 0; h < 2; ++h) {
        float ob[S];
#pragma unroll
        for (int k = 0; k < S; ++k) ob[k] = obs_s[(h * TC_M + rr) * tc_row(S) + k];
        for (int s = 0; s < n_stages; ++s) {
            const int q = h * n_stages + s;
            const uint32_t g = g0 + q, slot = g % TC_STAGES;
            // the slot's previous MMAs (stage g - TC_STAGES) retired: every thread waited for stage g - 3 before the
            // barrier of stage g - 1
            float* a_hi = c.a_ring + (size_t)slot * A_STAGE_FLOATS;
            float* a_lo = a_hi + TC_CH * TC_M * 4;
            float hv[4];
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) hv[kk] = tc_layer0<S>(W0p + (size_t)(s * TC_KSLAB + jj * 4 + kk) * tc_row(S), ob);
            const float2 p0 = am_act2<ACT>(make_float2(hv[0], hv[1])), p1 = am_act2<ACT>(make_float2(hv[2], hv[3]));
            const float4 hi = make_float4(rn_tf32(p0.x), rn_tf32(p0.y), rn_tf32(p1.x), rn_tf32(p1.y));
            const float4 lo = make_float4(rn_tf32(p0.x - hi.x), rn_tf32(p0.y - hi.y), rn_tf32(p1.x - hi.z), rn_tf32(p1.y - hi.w));
            *reinterpret_cast<float4*>(a_hi + ((size_t)jj * TC_M + rr) * 4) = hi;
            *reinterpret_cast<float4*>(a_lo + ((size_t)jj * TC_M + rr) * 4) = lo;
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy writes of A -> wgmma (async proxy) reads
            group_sync(c.grp);
            // prefetch stage g + 2 into the slot of stage g - 2, retired by every thread before this barrier
            if (tid == 0 && q + 2 < total) {
                const uint32_t sl = (g + 2) % TC_STAGES;
                mbar_expect_tx(&c.full_b[sl], stage_bytes);
                tma_bulk_g2s(c.b_ring + (size_t)sl * ar.stage_floats, tiles_actor + (size_t)((q + 2) % n_stages) * ar.stage_floats,
                             stage_bytes, &c.full_b[sl]);
            }
            mbar_wait(&c.full_b[slot], (g / TC_STAGES) & 1);               // W1 slab landed
            const uint32_t a_hi_addr = smem_u32(a_hi), a_lo_addr = smem_u32(a_lo);
            const uint32_t b_hi_addr = smem_u32(c.b_ring + (size_t)slot * ar.stage_floats);
            const uint32_t b_lo_addr = b_hi_addr + (uint32_t)TC_CH * (uint32_t)n2pad * 16u;
            const uint32_t lbo_a = TC_M * 16, lbo_b = (uint32_t)n2pad * 16;
            const uint64_t dah = wgmma_desc(a_hi_addr, lbo_a, 128), dal = wgmma_desc(a_lo_addr, lbo_a, 128);
            const uint32_t acc0 = s > 0 ? 1u : 0u;
            wgmma_fence();
#pragma unroll
            for (int cc = 0; cc < TC_MAXN / TC_NCH; ++cc) {
                if (cc < nch) {                                              // hi.hi + hi.lo + lo.hi ("3xTF32")
                    float (&d)[32] = *reinterpret_cast<float (*)[32]>(acc + cc * 32);
                    const uint32_t bo2 = (uint32_t)(cc * TC_NCH) * 16u;
                    wgmma_tf32_n64(d, dah, wgmma_desc(b_hi_addr + bo2, lbo_b, 128), acc0);
                    wgmma_tf32_n64(d, dah, wgmma_desc(b_lo_addr + bo2, lbo_b, 128), 1u);
                    wgmma_tf32_n64(d, dal, wgmma_desc(b_hi_addr + bo2, lbo_b, 128), 1u);
                }
            }
            wgmma_commit();
            wgmma_wait<1>();                                                 // stage g - 1 retired
        }
        wgmma_wait<0>();
        // ---- epilogue of the half: rows r0 and r0 + 8 of the thread's warp, spread over the 4 lanes of a quad ----
        const int r0 = warp * 16 + (lane >> 2), cq = (lane & 3) * 2;
        float s0 = 0.f, s1 = 0.f;
#pragma unroll
        for (int cc = 0; cc < TC_MAXN / TC_NCH; ++cc) {
            if (cc < nch) {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int j = cc * TC_NCH + i * 8 + cq;
                    float* d = acc + cc * 32 + i * 4;
                    d[0] = __fadd_rn(d[0], b1[j]); d[1] = __fadd_rn(d[1], b1[j + 1]);
                    d[2] = __fadd_rn(d[2], b1[j]); d[3] = __fadd_rn(d[3], b1[j + 1]);
                    s0 = __fadd_rn(s0, __fadd_rn(d[0], d[1]));           // padded columns hold 0 (zero weights and bias)
                    s1 = __fadd_rn(s1, __fadd_rn(d[2], d[3]));
                }
            }
        }
        s0 = __fadd_rn(s0, __shfl_xor_sync(0xffffffffu, s0, 1)); s0 = __fadd_rn(s0, __shfl_xor_sync(0xffffffffu, s0, 2));
        s1 = __fadd_rn(s1, __shfl_xor_sync(0xffffffffu, s1, 1)); s1 = __fadd_rn(s1, __shfl_xor_sync(0xffffffffu, s1, 2));
        const float mean0 = __fdiv_rn(s0, (float)w2), mean1 = __fdiv_rn(s1, (float)w2);
        float v0 = 0.f, v1 = 0.f;
#pragma unroll
        for (int cc = 0; cc < TC_MAXN / TC_NCH; ++cc) {
            if (cc < nch) {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int j = cc * TC_NCH + i * 8 + cq;
                    const float* d = acc + cc * 32 + i * 4;
                    const float m0 = j < w2 ? 1.f : 0.f, m1 = j + 1 < w2 ? 1.f : 0.f;
                    const float e00 = __fmul_rn(m0, __fadd_rn(d[0], -mean0)), e01 = __fmul_rn(m1, __fadd_rn(d[1], -mean0));
                    const float e10 = __fmul_rn(m0, __fadd_rn(d[2], -mean1)), e11 = __fmul_rn(m1, __fadd_rn(d[3], -mean1));
                    v0 = __fmaf_rn(e00, e00, v0); v0 = __fmaf_rn(e01, e01, v0);
                    v1 = __fmaf_rn(e10, e10, v1); v1 = __fmaf_rn(e11, e11, v1);
                }
            }
        }
        v0 = __fadd_rn(v0, __shfl_xor_sync(0xffffffffu, v0, 1)); v0 = __fadd_rn(v0, __shfl_xor_sync(0xffffffffu, v0, 2));
        v1 = __fadd_rn(v1, __shfl_xor_sync(0xffffffffu, v1, 1)); v1 = __fadd_rn(v1, __shfl_xor_sync(0xffffffffu, v1, 2));
        const float inv0 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(__fdiv_rn(v0, (float)(w2 - 1))), 1e-6f));
        const float inv1 = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(__fdiv_rn(v1, (float)(w2 - 1))), 1e-6f));
        float o[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
        for (int cc = 0; cc < TC_MAXN / TC_NCH; ++cc) {
            if (cc < nch) {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const int j = cc * TC_NCH + i * 8 + cq;
                    const float* d = acc + cc * 32 + i * 4;
                    // padded columns carry zero weights in Wo, so they add nothing
                    const float2 y0 = am_act2<ACT>(make_float2(__fmaf_rn(__fmul_rn(gamma[j], __fadd_rn(d[0], -mean0)), inv0, beta[j]),
                                                               __fmaf_rn(__fmul_rn(gamma[j + 1], __fadd_rn(d[1], -mean0)), inv0, beta[j + 1])));
                    const float2 y1 = am_act2<ACT>(make_float2(__fmaf_rn(__fmul_rn(gamma[j], __fadd_rn(d[2], -mean1)), inv1, beta[j]),
                                                               __fmaf_rn(__fmul_rn(gamma[j + 1], __fadd_rn(d[3], -mean1)), inv1, beta[j + 1])));
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        o[0][k] = __fmaf_rn(Wo[k * n2pad + j], y0.x, o[0][k]); o[0][k] = __fmaf_rn(Wo[k * n2pad + j + 1], y0.y, o[0][k]);
                        o[1][k] = __fmaf_rn(Wo[k * n2pad + j], y1.x, o[1][k]); o[1][k] = __fmaf_rn(Wo[k * n2pad + j + 1], y1.y, o[1][k]);
                    }
                }
            }
        }
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                o[r][k] = __fadd_rn(o[r][k], __shfl_xor_sync(0xffffffffu, o[r][k], 1));
                o[r][k] = __fadd_rn(o[r][k], __shfl_xor_sync(0xffffffffu, o[r][k], 2));
            }
        if ((lane & 3) == 0) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                act_s[(h * TC_M + r0) * 4 + k] = am_tanh1(__fadd_rn(o[0][k], bo[k]));
                act_s[(h * TC_M + r0 + 8) * 4 + k] = am_tanh1(__fadd_rn(o[1][k], bo[k]));
            }
        }
    }
    c.g = g0 + total;
    tc_release(c);                                                           // (its barrier publishes act_s)
    action[0] = act_s[tid * 4]; action[1] = act_s[tid * 4 + 1]; action[2] = act_s[tid * 4 + 2];
}

// LayerNorm statistics of the accumulator rows r0 and r0 + 8 after the bias (the epilogue of tc_actor_forward): the bias is
// added in place, then mean[] and inv[] = 1 / (unbiased std + eps) over the w real columns (padded columns hold exactly 0)
__device__ __forceinline__ void tc_bias_ln(float* acc, int nch, int w, int cq, const float* b, float (&mean)[2], float (&inv)[2])
{
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int cc = 0; cc < TC_MAXN / TC_NCH; ++cc) {
        if (cc < nch) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int j = cc * TC_NCH + i * 8 + cq;
                float* d = acc + cc * 32 + i * 4;
                d[0] = __fadd_rn(d[0], b[j]); d[1] = __fadd_rn(d[1], b[j + 1]);
                d[2] = __fadd_rn(d[2], b[j]); d[3] = __fadd_rn(d[3], b[j + 1]);
                s0 = __fadd_rn(s0, __fadd_rn(d[0], d[1]));
                s1 = __fadd_rn(s1, __fadd_rn(d[2], d[3]));
            }
        }
    }
    s0 = __fadd_rn(s0, __shfl_xor_sync(0xffffffffu, s0, 1)); s0 = __fadd_rn(s0, __shfl_xor_sync(0xffffffffu, s0, 2));
    s1 = __fadd_rn(s1, __shfl_xor_sync(0xffffffffu, s1, 1)); s1 = __fadd_rn(s1, __shfl_xor_sync(0xffffffffu, s1, 2));
    mean[0] = __fdiv_rn(s0, (float)w); mean[1] = __fdiv_rn(s1, (float)w);
    float v0 = 0.f, v1 = 0.f;
#pragma unroll
    for (int cc = 0; cc < TC_MAXN / TC_NCH; ++cc) {
        if (cc < nch) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int j = cc * TC_NCH + i * 8 + cq;
                const float* d = acc + cc * 32 + i * 4;
                const float m0 = j < w ? 1.f : 0.f, m1 = j + 1 < w ? 1.f : 0.f;
                const float e00 = __fmul_rn(m0, __fadd_rn(d[0], -mean[0])), e01 = __fmul_rn(m1, __fadd_rn(d[1], -mean[0]));
                const float e10 = __fmul_rn(m0, __fadd_rn(d[2], -mean[1])), e11 = __fmul_rn(m1, __fadd_rn(d[3], -mean[1]));
                v0 = __fmaf_rn(e00, e00, v0); v0 = __fmaf_rn(e01, e01, v0);
                v1 = __fmaf_rn(e10, e10, v1); v1 = __fmaf_rn(e11, e11, v1);
            }
        }
    }
    v0 = __fadd_rn(v0, __shfl_xor_sync(0xffffffffu, v0, 1)); v0 = __fadd_rn(v0, __shfl_xor_sync(0xffffffffu, v0, 2));
    v1 = __fadd_rn(v1, __shfl_xor_sync(0xffffffffu, v1, 1)); v1 = __fadd_rn(v1, __shfl_xor_sync(0xffffffffu, v1, 2));
    inv[0] = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(__fdiv_rn(v0, (float)(w - 1))), 1e-6f));
    inv[1] = __fdiv_rn(1.0f, __fadd_rn(__fsqrt_rn(__fdiv_rn(v1, (float)(w - 1))), 1e-6f));
}

// issue the TMA copy of forward stage q (of both halves) into the B ring slot of pipeline stage g
__device__ __forceinline__ void tc_fetch_deep(TcCtx& c, const TcArgs& ar, const float* tiles_actor, uint32_t g, int q)
{
    int r = q % ar.stages, l = 0;
    while (r >= ar.ly[l].n_stages) { r -= ar.ly[l].n_stages; ++l; }
    const uint32_t sl = g % TC_STAGES, bytes = (uint32_t)ar.ly[l].stage_floats * 4u;
    mbar_expect_tx(&c.full_b[sl], bytes);
    tma_bulk_g2s(c.b_ring + (size_t)sl * ar.stage_floats, tiles_actor + ar.ly[l].tile + (size_t)r * ar.ly[l].stage_floats, bytes, &c.full_b[sl]);
}

// The same forward pass for n >= 3 widths [w0, w1, ..., w_{n-1}]: layer 0 on CUDA cores writes the A slabs of layer 1 as in
// tc_actor_forward; every layer l >= 1 streams its K-slabs through the same A / B rings and one pipeline counter, so the
// TMA prefetch runs two stages ahead across layer boundaries.  The epilogue of a layer l < n-1 (bias, LayerNorm,
// activation) writes its rows to the fp32 activation buffer, zero past w_l; layer l+1 then builds each A slab from that
// buffer (TF32 hi / lo split) instead of from layer 0.  The last layer has the epilogue of tc_actor_forward with the output
// layer folded in.  The small block is read from global memory (L1).
template <int ACT, int S = 7>
__device__ __forceinline__ void tc_actor_forward_deep(TcCtx& c, const TcArgs& ar, const float* tiles_actor, const float* obs, float* action)
{
    const int tid = c.gtid, warp = tid >> 5, lane = tid & 31;
    const int total = 2 * ar.stages;
    constexpr int A_STAGE_FLOATS = 2 * TC_CH * TC_M * 4;
    const float* W0p = c.small;
    float* obs_s = c.io;
    float* act_s = c.io + TC_THREADS * tc_row(S);
    float* abuf = c.abuf;
    const int as = ar.abuf_stride;
#pragma unroll
    for (int k = 0; k < S; ++k) obs_s[tid * tc_row(S) + k] = obs[k];
    tc_acquire(c);                                                         // (its barrier publishes obs_s)
    const uint32_t g0 = c.g;
    if (tid == 0)
        for (int q = 0; q < 2 && q < total; ++q) tc_fetch_deep(c, ar, tiles_actor, g0 + q, q);
    const int rr = tid & (TC_M - 1), jj = tid >> 6;                         // A slab: row rr of the half, K chunk jj
    const int r0 = warp * 16 + (lane >> 2), cq = (lane & 3) * 2;            // accumulator: rows r0, r0 + 8, columns cq + {0, 1} + 8i
    float acc[TC_MAXN / 2];
    int q = 0;
    for (int h = 0; h < 2; ++h) {
        float ob[S];
#pragma unroll
        for (int k = 0; k < S; ++k) ob[k] = obs_s[(h * TC_M + rr) * tc_row(S) + k];
        for (int l = 0; l < ar.n_layers; ++l) {
            const int npad = ar.ly[l].npad, nch = npad / TC_NCH, w = ar.ly[l].w, n_stages = ar.ly[l].n_stages;
            for (int s = 0; s < n_stages; ++s, ++q) {
                const uint32_t g = g0 + q, slot = g % TC_STAGES;
                float* a_hi = c.a_ring + (size_t)slot * A_STAGE_FLOATS;
                float* a_lo = a_hi + TC_CH * TC_M * 4;
                float4 x;
                if (l == 0) {
                    float hv[4];
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) hv[kk] = tc_layer0<S>(W0p + (size_t)(s * TC_KSLAB + jj * 4 + kk) * tc_row(S), ob);
                    const float2 p0 = am_act2<ACT>(make_float2(hv[0], hv[1])), p1 = am_act2<ACT>(make_float2(hv[2], hv[3]));
                    x = make_float4(p0.x, p0.y, p1.x, p1.y);
                } else {
                    x = *reinterpret_cast<const float4*>(abuf + (size_t)rr * as + s * TC_KSLAB + jj * 4);
                }
                const float4 hi = make_float4(rn_tf32(x.x), rn_tf32(x.y), rn_tf32(x.z), rn_tf32(x.w));
                const float4 lo = make_float4(rn_tf32(x.x - hi.x), rn_tf32(x.y - hi.y), rn_tf32(x.z - hi.z), rn_tf32(x.w - hi.w));
                *reinterpret_cast<float4*>(a_hi + ((size_t)jj * TC_M + rr) * 4) = hi;
                *reinterpret_cast<float4*>(a_lo + ((size_t)jj * TC_M + rr) * 4) = lo;
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                group_sync(c.grp);
                if (tid == 0 && q + 2 < total) tc_fetch_deep(c, ar, tiles_actor, g + 2, q + 2);
                mbar_wait(&c.full_b[slot], (g / TC_STAGES) & 1);
                const uint32_t b_hi_addr = smem_u32(c.b_ring + (size_t)slot * ar.stage_floats);
                const uint32_t b_lo_addr = b_hi_addr + (uint32_t)TC_CH * (uint32_t)npad * 16u;
                const uint32_t lbo_a = TC_M * 16, lbo_b = (uint32_t)npad * 16;
                const uint64_t dah = wgmma_desc(smem_u32(a_hi), lbo_a, 128), dal = wgmma_desc(smem_u32(a_lo), lbo_a, 128);
                const uint32_t acc0 = s > 0 ? 1u : 0u;
                wgmma_fence();
#pragma unroll
                for (int cc = 0; cc < TC_MAXN / TC_NCH; ++cc) {
                    if (cc < nch) {
                        float (&d)[32] = *reinterpret_cast<float (*)[32]>(acc + cc * 32);
                        const uint32_t bo2 = (uint32_t)(cc * TC_NCH) * 16u;
                        wgmma_tf32_n64(d, dah, wgmma_desc(b_hi_addr + bo2, lbo_b, 128), acc0);
                        wgmma_tf32_n64(d, dah, wgmma_desc(b_lo_addr + bo2, lbo_b, 128), 1u);
                        wgmma_tf32_n64(d, dal, wgmma_desc(b_hi_addr + bo2, lbo_b, 128), 1u);
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();
            }
            wgmma_wait<0>();
            const float* b = c.small + ar.ly[l].vec;
            const float* gamma = b + npad;
            const float* beta = gamma + npad;
            float mean[2], inv[2];
            tc_bias_ln(acc, nch, w, cq, b, mean, inv);
            if (l + 1 < ar.n_layers) {
                // every thread read its last slab of this layer's input before the barrier of that stage: the buffer is free
                const int kout = ar.ly[l + 1].n_stages * TC_KSLAB;        // columns the next layer reads
#pragma unroll
                for (int cc = 0; cc < TC_MAXN / TC_NCH; ++cc) {
                    if (cc < nch) {
#pragma unroll
                        for (int i = 0; i < 8; ++i) {
                            const int j = cc * TC_NCH + i * 8 + cq;
                            if (j < kout) {
                                const float* d = acc + cc * 32 + i * 4;
                                const float2 y0 = am_act2<ACT>(make_float2(__fmaf_rn(__fmul_rn(gamma[j], __fadd_rn(d[0], -mean[0])), inv[0], beta[j]),
                                                                           __fmaf_rn(__fmul_rn(gamma[j + 1], __fadd_rn(d[1], -mean[0])), inv[0], beta[j + 1])));
                                const float2 y1 = am_act2<ACT>(make_float2(__fmaf_rn(__fmul_rn(gamma[j], __fadd_rn(d[2], -mean[1])), inv[1], beta[j]),
                                                                           __fmaf_rn(__fmul_rn(gamma[j + 1], __fadd_rn(d[3], -mean[1])), inv[1], beta[j + 1])));
                                // zero neurons past w feed the next layer exactly 0
                                *reinterpret_cast<float2*>(abuf + (size_t)r0 * as + j) = make_float2(j < w ? y0.x : 0.f, j + 1 < w ? y0.y : 0.f);
                                *reinterpret_cast<float2*>(abuf + (size_t)(r0 + 8) * as + j) = make_float2(j < w ? y1.x : 0.f, j + 1 < w ? y1.y : 0.f);
                            }
                        }
                    }
                }
                group_sync(c.grp);                                           // the next layer's A slabs read other threads' rows
                continue;
            }
            const float* Wo = beta + npad;
            const float* bo = Wo + 3 * npad;
            float o[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
            for (int cc = 0; cc < TC_MAXN / TC_NCH; ++cc) {
                if (cc < nch) {
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int j = cc * TC_NCH + i * 8 + cq;
                        const float* d = acc + cc * 32 + i * 4;
                        const float2 y0 = am_act2<ACT>(make_float2(__fmaf_rn(__fmul_rn(gamma[j], __fadd_rn(d[0], -mean[0])), inv[0], beta[j]),
                                                                   __fmaf_rn(__fmul_rn(gamma[j + 1], __fadd_rn(d[1], -mean[0])), inv[0], beta[j + 1])));
                        const float2 y1 = am_act2<ACT>(make_float2(__fmaf_rn(__fmul_rn(gamma[j], __fadd_rn(d[2], -mean[1])), inv[1], beta[j]),
                                                                   __fmaf_rn(__fmul_rn(gamma[j + 1], __fadd_rn(d[3], -mean[1])), inv[1], beta[j + 1])));
#pragma unroll
                        for (int k = 0; k < 3; ++k) {
                            o[0][k] = __fmaf_rn(Wo[k * npad + j], y0.x, o[0][k]); o[0][k] = __fmaf_rn(Wo[k * npad + j + 1], y0.y, o[0][k]);
                            o[1][k] = __fmaf_rn(Wo[k * npad + j], y1.x, o[1][k]); o[1][k] = __fmaf_rn(Wo[k * npad + j + 1], y1.y, o[1][k]);
                        }
                    }
                }
            }
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    o[r][k] = __fadd_rn(o[r][k], __shfl_xor_sync(0xffffffffu, o[r][k], 1));
                    o[r][k] = __fadd_rn(o[r][k], __shfl_xor_sync(0xffffffffu, o[r][k], 2));
                }
            if ((lane & 3) == 0) {
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    act_s[(h * TC_M + r0) * 4 + k] = am_tanh1(__fadd_rn(o[0][k], bo[k]));
                    act_s[(h * TC_M + r0 + 8) * 4 + k] = am_tanh1(__fadd_rn(o[1][k], bo[k]));
                }
            }
        }
    }
    c.g = g0 + total;
    tc_release(c);                                                           // (its barrier publishes act_s)
    action[0] = act_s[tid * 4]; action[1] = act_s[tid * 4 + 1]; action[2] = act_s[tid * 4 + 2];
}

constexpr int TC_TABN2 = (PLANT_TABN + 15) & ~15;                       // keeps the float regions 128-byte aligned
constexpr int TC_IO_FLOATS = TC_THREADS * 12;                           // per group: observations [128][8], actions [128][4]
// ... for an observation of S entries: observations [128][tc_row(S)], actions [128][4]
__host__ __device__ constexpr int tc_io_floats(int S) { return S == 7 ? TC_IO_FLOATS : TC_THREADS * (tc_row(S) + 4); }

// dynamic shared memory: plant tables | two small blocks (two widths only) | io of both groups | A ring | B ring |
// activation buffer (deep lists only)
template <bool DEEP, int S = 7>
__device__ __forceinline__ void tc_setup(TcCtx& c, const TcArgs& ar, unsigned char* smem_raw, uint64_t* bars, uint32_t* shared_state)
{
    constexpr int A_STAGE_FLOATS = 2 * TC_CH * TC_M * 4;
    real* tab_s = reinterpret_cast<real*>(smem_raw);
    for (int i = threadIdx.x; i < PT_TOTAL; i += blockDim.x) tab_s[i] = plant_tables_blob[i];
    for (int i = threadIdx.x; i < SERL_PLANT_COUNT * PLANT_NPV; i += blockDim.x) tab_s[PT_TOTAL + i] = (&plant_pv[0][0])[i];
    float* f = reinterpret_cast<float*>(tab_s + TC_TABN2);
    const int small_pad = DEEP ? 0 : (ar.small_floats + 31) & ~31;
    c.grp = threadIdx.x >> 7;
    c.gtid = threadIdx.x & (TC_THREADS - 1);
    c.small = f + (size_t)c.grp * small_pad;
    c.io = f + 2 * (size_t)small_pad + (size_t)c.grp * tc_io_floats(S);
    c.a_ring = f + 2 * (size_t)small_pad + 2 * tc_io_floats(S);
    c.b_ring = c.a_ring + TC_STAGES * A_STAGE_FLOATS;
    c.abuf = c.b_ring + (size_t)TC_STAGES * ar.stage_floats;
    c.full_b = bars;
    c.shared_state = shared_state;
    c.g = 0;
    if (threadIdx.x == 0) {
        for (int i = 0; i < TC_STAGES; ++i) mbar_init(&bars[i], 1);
        shared_state[0] = shared_state[1] = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
}

template <bool DEEP>
__device__ __forceinline__ void tc_load_small(TcCtx& c, const TcArgs& ar, int actor)
{
    if constexpr (DEEP) {                       // read in place through L1
        c.small = ar.small + (size_t)actor * ar.small_floats;
        return;
    }
    group_sync(c.grp);                // the group's previous actor's parameters are no longer read
    float* dst = const_cast<float*>(c.small);
    const float4* src = reinterpret_cast<const float4*>(ar.small + (size_t)actor * ar.small_floats);
    for (int i = c.gtid; i < ar.small_floats / 4; i += TC_THREADS) reinterpret_cast<float4*>(dst)[i] = src[i];
    group_sync(c.grp);
}

// GUST, TRACK, PER_ACTOR, INC, SYM: the launch's variant, as in rollout_kernel_persist (rollout_variant.h lists the
// instantiated ones).  GUST: the launch has envs of the gust build, and reset and step share the one plant_step instance of
// the kernel; without it a gust env raises SERL_STATUS_GUST_FLAG.  DEEP: more than two widths (tc_actor_forward_deep); the
// two-width instantiations run tc_actor_forward.  TRACK: the launch writes the tracking-error sums `tk`
// (serl_rollout_desc.d_track).  PER_ACTOR: env `env` of actor `actor` binds row actor * n_envs + env of env_mode /
// ref_levels / ref_starts (SERL_ROLLOUT_PER_ACTOR_REFS).  INC: incremental control (SERL_ROLLOUT_INCREMENTAL): a 10-entry
// observation, layer 0 with 10 inputs, and the env's last_u.  SYM: symmetric control (SERL_ROLLOUT_SYMMETRIC): a 2-entry
// observation, layer 0 with 2 inputs, and action 0 of the output block as the elevator
template <int ACT, bool GUST, bool DEEP, bool TRACK = false, bool PER_ACTOR = false, bool INC = false, bool SYM = false>
__global__ void __launch_bounds__(2 * TC_THREADS, 1)
rollout_kernel_tc(const __grid_constant__ TcArgs ar, TrackArgs tk)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t bars[TC_STAGES];
    __shared__ uint32_t shared_state[2];
    TcCtx c;
    plant_tab_check(smem_raw);
    tc_setup<DEEP, OBS_DIM<INC, SYM>>(c, ar, smem_raw, bars, shared_state);
    const RolloutArgs& r = ar.r;
    const real* tab = reinterpret_cast<const real*>(smem_raw);
    const real* pv_base = tab + PT_TOTAL;
    const int tid = c.gtid;
    // the two groups of a CTA run independent task loops
    for (long long task = (long long)blockIdx.x * 2 + c.grp; task < ar.n_tasks; task += 2LL * gridDim.x) {
        const int actor = (int)(task / ar.n_chunks), chunk = (int)(task - (long long)actor * ar.n_chunks);
        tc_load_small<DEEP>(c, ar, actor);
        const float* tiles_actor = ar.tiles + (size_t)actor * ar.tile_floats;
        const int eslot = chunk * TC_THREADS + tid;
        const bool valid = eslot < r.n_envs;
        const int env = valid ? (r.env_order ? r.env_order[eslot] : eslot) : 0;
        Env e;
        e.tab = tab;
        float obs[OBS_DIM<INC, SYM>], a[3];
        double last_u[3];                              // INC only
        if (valid) {
            const int row = PER_ACTOR ? actor * r.n_envs + env : env;
            env_bind<GUST>(e, r, row, pv_base, (size_t)actor * r.n_envs + env);
            env_reset<true, GUST, TRACK, INC, SYM>(e, r, row, obs, (size_t)actor * r.n_envs + env, last_u);
        } else {
            env_idle<INC, SYM>(e, r, pv_base, obs, last_u);
        }
        const size_t traj = (size_t)actor * r.n_envs + env;
        const bool replay = valid && r.replay != nullptr && env == r.replay_env;
        while (group_any(c.grp, !e.done)) {
            if constexpr (DEEP) tc_actor_forward_deep<ACT, OBS_DIM<INC, SYM>>(c, ar, tiles_actor, obs, a);
            else tc_actor_forward<ACT, OBS_DIM<INC, SYM>>(c, ar, tiles_actor, obs, a);
            if (!e.done) env_step<true, GUST, TRACK, PER_ACTOR, INC, SYM>(e, r, traj, actor, replay, a, obs, last_u);
        }
        if (valid) traj_store(e, r, traj);
        if constexpr (TRACK) if (valid) track_store(e, tk, traj);
    }
}

// Actor.forward for a batch through the same tensor-core device code (parity tests of the GEMM path)
template <int ACT, bool DEEP>
__global__ void __launch_bounds__(2 * TC_THREADS, 1)
actor_forward_tc_kernel(const __grid_constant__ TcArgs ar)
{
    extern __shared__ __align__(128) unsigned char smem_raw[];
    __shared__ uint64_t bars[TC_STAGES];
    __shared__ uint32_t shared_state[2];
    TcCtx c;
    tc_setup<DEEP>(c, ar, smem_raw, bars, shared_state);
    tc_load_small<DEEP>(c, ar, 0);
    const int tid = c.gtid;
    for (int base = (blockIdx.x * 2 + c.grp) * TC_THREADS; base < ar.n_obs; base += 2 * gridDim.x * TC_THREADS) {
        const int i = base + tid;
        float obs[7], a[3];
#pragma unroll
        for (int k = 0; k < 7; ++k) obs[k] = i < ar.n_obs ? ar.obs_in[(size_t)i * 7 + k] : 0.f;
        if constexpr (DEEP) tc_actor_forward_deep<ACT>(c, ar, ar.tiles, obs, a);
        else tc_actor_forward<ACT>(c, ar, ar.tiles, obs, a);
        if (i < ar.n_obs) { ar.act_out[(size_t)i * 3] = a[0]; ar.act_out[(size_t)i * 3 + 1] = a[1]; ar.act_out[(size_t)i * 3 + 2] = a[2]; }
    }
}

// ---- host side ------------------------------------------------------------------------------------------------
extern "C" int64_t serl_actor_num_params_wide(const int32_t* widths, int32_t n_widths)
{
    if (!widths || n_widths < 1) return -1;
    int64_t P = 7 * (int64_t)widths[0] + widths[0];
    for (int i = 1; i < n_widths; ++i) P += (int64_t)widths[i] * widths[i - 1] + 3 * (int64_t)widths[i];
    return P + 3 * (int64_t)widths[n_widths - 1] + 3;
}

// Checks the widths and sizes the layer table, the kernel layout and the shared memory (all before any CUDA call), then
// brings the genomes into the kernel layout (K0-TC) in the stream's scratch buffer.  The task sets the widths of layer 0's
// input and of the output block.
static int tc_prepare(TcArgs& ar, const float* d_weights, int pop, const int32_t* widths, int n_widths, cudaStream_t s, size_t* smem_out,
                      const RolloutTask& task = TASK_ATTITUDE)
{
    const int S = task.obs, A = task.act;
    if (!widths || n_widths < 2 || n_widths > TC_MAXL + 1)
        return serl_fail(SERL_ERR_UNSUPPORTED, "wide actors: the tensor-core path takes 2 to 9 widths [w0, w1, ..., w_{n-1}]");
    if (widths[0] < 8 || widths[0] > 1024) return serl_fail(SERL_ERR_UNSUPPORTED, "wide actors: need 8 <= w0 <= 1024");
    for (int i = 1; i < n_widths; ++i)
        if (widths[i] < 8 || widths[i] > TC_MAXN) return serl_fail(SERL_ERR_UNSUPPORTED, "wide actors: need 8 <= w_i <= 320 for i >= 1");
    const auto pad = [](int x, int m) { return (x + m - 1) / m * m; };
    ar.w1_real = widths[0];
    ar.w1 = pad(widths[0], TC_KSLAB);
    ar.w2 = widths[1]; ar.n2pad = pad(widths[1], TC_NCH);
    ar.n_layers = n_widths - 1;
    int vec = ar.w1 * tc_row(S), tile = 0, gW = (S + 1) * widths[0], kmax = 0;
    ar.stages = 0; ar.stage_floats = 0;
    for (int l = 0; l < ar.n_layers; ++l) {
        TcLayer& L = ar.ly[l];
        L.w = widths[l + 1]; L.npad = pad(L.w, TC_NCH);
        L.win = widths[l]; L.n_stages = pad(L.win, TC_KSLAB) / TC_KSLAB;
        L.stage_floats = 2 * TC_CH * L.npad * 4;
        L.vec = vec; L.tile = tile; L.gW = gW;
        vec += 3 * L.npad;
        tile += L.n_stages * L.stage_floats;
        gW += L.w * L.win + 3 * L.w;
        ar.stages += L.n_stages;
        if (L.stage_floats > ar.stage_floats) ar.stage_floats = L.stage_floats;
        if (l + 1 < ar.n_layers && pad(L.w, TC_KSLAB) > kmax) kmax = pad(L.w, TC_KSLAB);
    }
    ar.gWo = gW;
    ar.small_floats = (vec + 3 * ar.ly[ar.n_layers - 1].npad + 4 + 3) & ~3;
    ar.tile_floats = tile;
    // deep lists: no small blocks in shared memory, one activation buffer for the lock holder; +4 floats per row keeps
    // its float4 reads of 8 consecutive rows on distinct banks
    const bool deep = ar.n_layers > 1;
    ar.abuf_stride = deep ? kmax + 4 : 0;
    constexpr int A_STAGE_FLOATS = 2 * TC_CH * TC_M * 4;
    *smem_out = (size_t)TC_TABN2 * sizeof(real) +
                (size_t)(2 * (deep ? 0 : (ar.small_floats + 31) & ~31) + 2 * tc_io_floats(S) + TC_STAGES * A_STAGE_FLOATS +
                         TC_STAGES * ar.stage_floats + TC_M * ar.abuf_stride) * 4;
    if (*smem_out > SERL_SMEM_OPTIN - 256)
        return serl_fail(SERL_ERR_UNSUPPORTED, deep ? "wide actors: tables + rings + activation buffer exceed the shared memory of an SM"
                                                    : "wide actors: tables + parameters + rings exceed the shared memory of an SM");
    const int P = (int)serl_actor_num_params_wide(widths, n_widths) + (S - 7) * widths[0] + (A - 3) * (widths[n_widths - 1] + 1);
    const size_t small_bytes = (size_t)pop * ar.small_floats * 4;
    const size_t tile_bytes = (size_t)pop * ar.tile_floats * 4;
    void* scratch = nullptr;
    cudaError_t e = serl_scratch(SERL_SCRATCH_TC, s, ((small_bytes + 255) & ~(size_t)255) + tile_bytes + 256, &scratch);
    if (e != cudaSuccess) return serl_fail_cuda(e, "wide actors: scratch allocation");
    float* small = (float*)scratch;
    float* tiles = (float*)((unsigned char*)scratch + ((small_bytes + 255) & ~(size_t)255));
    ar.small = small; ar.tiles = tiles;
    const long long total = (long long)pop * ((long long)ar.small_floats + ar.tile_floats);
    const int grid = (int)((total + 255) / 256 < 8192 ? (total + 255) / 256 : 8192);
    int rc = SERL_OK;
    visit_task(task, [&](auto S, auto A) {
        rc = serl_launch("tc_layout_kernel", tc_layout_kernel<decltype(S)::value, decltype(A)::value>, grid, 256, 0, s, d_weights, pop, P, ar,
                         small, tiles);
    });
    return rc;
}

// calls f(ACT, DEEP) with a K1-TC kernel's activation (SERL_ACT_*) and depth as std::integral_constant
template <typename F>
static void tc_form(int activation, bool deep, F&& f)
{
    const auto with_act = [&](auto act) {
        if (deep) f(act, std::true_type());
        else f(act, std::false_type());
    };
    if (activation == SERL_ACT_TANH) with_act(std::integral_constant<int, SERL_ACT_TANH>());
    else if (activation == SERL_ACT_ELU) with_act(std::integral_constant<int, SERL_ACT_ELU>());
    else with_act(std::integral_constant<int, SERL_ACT_LEAKY_RELU>());
}

// K1-TC launch (serl_rollout_run has checked the descriptor, chosen the variant `v` and built the env / output arguments `r`)
int rollout_tc_impl(const serl_rollout_desc& d, const RolloutArgs& r, const RolloutVariant& v, cudaStream_t s)
{
    TcArgs ar;
    memset(&ar, 0, sizeof(ar));
    ar.r = r;
    size_t smem = 0;
    const int rc = tc_prepare(ar, d.d_weights, d.pop, d.widths, d.n_widths, s, &smem, v.task);
    if (rc != SERL_OK) return rc;
    ar.n_chunks = (d.n_envs + TC_THREADS - 1) / TC_THREADS;
    ar.n_tasks = (long long)d.pop * ar.n_chunks;
    int sms = serl_device_sms();
    if (d.sm_limit > 0 && d.sm_limit < sms) sms = d.sm_limit;
    const long long grid = (ar.n_tasks + 1) / 2 < sms ? (ar.n_tasks + 1) / 2 : sms;
    void (*kernel)(TcArgs, TrackArgs) = nullptr;
    tc_form(d.shape.activation, ar.n_layers > 1, [&](auto act, auto deep) {
        visit_rollout_variant(v, [&](auto f) {
            using V = decltype(f);
            kernel = rollout_kernel_tc<decltype(act)::value, V::GUST, decltype(deep)::value, V::TRACK, V::PER_ACTOR, V::INC, V::SYM>;
        });
    });
    const TrackArgs tk = {d.d_track, nullptr, d.d_cost};
    // one CTA = the two groups of TC_THREADS threads
    return serl_launch("rollout_kernel_tc launch", kernel, (unsigned)grid, 2 * TC_THREADS, smem, s, ar, tk);
}

extern "C" int serl_actor_forward_wide(const float* d_genome, const int32_t* widths, int32_t n_widths, int32_t activation,
                                       const float* d_obs, int32_t n, float* d_actions, void* stream)
{
    if (!d_genome || !widths || !d_obs || !d_actions || n <= 0 || activation < 0 || activation > 2)
        return serl_fail(SERL_ERR_ARG, "serl_actor_forward_wide: bad argument");
    cudaStream_t s = (cudaStream_t)stream;
    TcArgs ar;
    memset(&ar, 0, sizeof(ar));
    size_t smem = 0;
    int rc = tc_prepare(ar, d_genome, 1, widths, n_widths, s, &smem);
    if (rc != SERL_OK) return rc;
    ar.obs_in = d_obs; ar.act_out = d_actions; ar.n_obs = n;
    const int blocks = (n + 2 * TC_THREADS - 1) / (2 * TC_THREADS);
    const int sms = serl_device_sms();
    const int grid = blocks < sms ? blocks : sms;
    tc_form(activation, ar.n_layers > 1, [&](auto act, auto deep) {
        rc = serl_launch("actor_forward_tc_kernel", actor_forward_tc_kernel<decltype(act)::value, decltype(deep)::value>, (unsigned)grid,
                         2 * TC_THREADS, smem, s, ar);
    });
    return rc;
}
