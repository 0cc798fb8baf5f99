// K7 — the TD3 learner (serl_b200/core/td3.py TD3.update_parameters), n_steps gradient steps in one launch, sm_90a.
//
// One persistent thread-block cluster of CS CTAs (256 threads each).  The learner state (actor, critic, both targets, both
// Adam moment sets: 438 KB at h = 72) stays in global memory, where it is L2-resident; the batch's activations and gradients
// live in a small global scratch.  Every phase of a step splits its outputs (a layer's output neurons x batch rows, a
// layer's parameter gradients, ...) over all threads of the cluster, and the phases are separated by cluster barriers
// (barrier.cluster.arrive.release / wait.acquire), whose acquire makes every write of the previous phase visible to the
// plain loads of the next.
//
// Determinism: every output element is computed by one thread (or one warp with a fixed shuffle tree) in a fixed order —
// weight gradients over the batch in row order, the gradient norm as fixed 64-element partials summed in order — and the
// random draws are keyed by (seed, global iteration, row).  The result is therefore the same bits for every cluster size
// and however the steps are split across launches.  Plain fp32 on CUDA cores: at batch <= 128 the work per step is
// 10-30 MFLOP (up to ~0.4 GFLOP for the widest actors), and the step is bound by the ~50 dependent phases, not by
// arithmetic.  Actors wider than 128 run their h x h blocks as tiled phases (td3_kernel<CS, true>, fwd_wide / bwd_wide).
// td3_group_kernel runs several independent learners of one hidden class in one launch, one cluster each
// (serl_td3_train_group); td3_mixed_kernel runs narrow and wide learners together (serl_td3_train_mixed).  The learner
// itself (td3_learner and its phases) is in td3_learner.cuh, which td3_group_per.cu instantiates too.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/serl_td3_mixed.h"
#include "td3_learner.cuh"

namespace {

template <int CS, bool WIDE>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(NT, 1) td3_kernel(const Args a)
{
    td3_learner<CS, WIDE, false>(a);
}

// A group launch: n learners of one actor shape, one cluster each.  Their Args travel as the kernel parameter (no
// host-to-device copy; CUDA 12.1+ allows 32,764 bytes of parameters on sm_90), and cluster g reads entry g from the
// constant bank (__grid_constant__: the table is never copied to local memory).  td3_learner takes its Args by value,
// which keeps td3_kernel's code exactly what it was before the group launch existed.  Clusters never wait for each
// other, so a group larger than the number of resident clusters is correct: later clusters start as earlier ones retire.
struct Group { Args a[SERL_TD3_MAX_GROUP]; };
static_assert(sizeof(Group) <= 32764, "SERL_TD3_MAX_GROUP learners' Args must fit the sm_90 kernel-parameter limit");

template <int CS, bool WIDE>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(NT, 1) td3_group_kernel(const __grid_constant__ Group t)
{
    unsigned g;
    asm("mov.u32 %0, %%clusterid.x;" : "=r"(g));
    td3_learner<CS, WIDE, true>(t.a[g]);
}

// A group of narrow and wide learners in one launch (serl_td3_train_mixed): cluster g branches once, uniformly for the
// whole cluster, on its learner's hidden width into td3_group_kernel's learner of that class, so each learner gets the
// bits its solo launch gives.  Every cluster reserves both branches' static shared memory (the wide tiles' WIDE_SMEM
// included; with one CTA per SM that costs no residency).  The narrow learner is a call: with both learners inlined,
// ptxas spills registers on the narrow path (64-68 bytes), which neither td3_group_kernel does; as a call it spills
// nothing and reads its Args from a 184-byte stack copy.
template <int CS>
__device__ __noinline__ void narrow_learner(const Args& a) { td3_learner<CS, false, true>(a); }

template <int CS>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(NT, 1) td3_mixed_kernel(const __grid_constant__ Group t)
{
    unsigned g;
    asm("mov.u32 %0, %%clusterid.x;" : "=r"(g));
    if (t.a[g].h > 128) td3_learner<CS, true, true>(t.a[g]);
    else narrow_learner<CS>(t.a[g]);
}

// A PER launch (serl_td3_train_per): one learner, its Args and Per as one __grid_constant__ parameter
struct PerLaunch { Args a; Per p; };

template <int CS, bool WIDE>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(NT, 1) td3_per_kernel(const __grid_constant__ PerLaunch t)
{
    td3_learner<CS, WIDE, false, true>(t.a, &t.p);
}

template <int CS>
int launch(const Args& a, cudaStream_t s)
{
    if (a.h > 128) return serl_launch("td3_kernel (wide)", td3_kernel<CS, true>, dim3(CS), dim3(NT), 0, s, a);
    return serl_launch("td3_kernel", td3_kernel<CS, false>, dim3(CS), dim3(NT), 0, s, a);
}

// one launch of the group's n learners with steps: td3_group_kernel of their hidden class, td3_mixed_kernel when they
// hold both narrow and wide actors
template <int CS>
int launch_group(const Group& t, int n, bool narrow, bool wide, cudaStream_t s)
{
    if (narrow && wide) return serl_launch("td3_mixed_kernel", td3_mixed_kernel<CS>, dim3(n * CS), dim3(NT), 0, s, t);
    if (wide) return serl_launch("td3_group_kernel (wide)", td3_group_kernel<CS, true>, dim3(n * CS), dim3(NT), 0, s, t);
    return serl_launch("td3_group_kernel", td3_group_kernel<CS, false>, dim3(n * CS), dim3(NT), 0, s, t);
}

}  // namespace

extern "C" int64_t serl_td3_state_floats(const serl_actor_shape* shape)
{
    if (!shape_ok(shape)) return serl_fail(SERL_ERR_ARG, "serl_td3_state_floats: unsupported actor shape");
    return 4 * actor_floats(*shape) + 8 * (int64_t)CP;
}

extern "C" int serl_td3_train(const serl_td3_desc* d, void* stream)
{
    if (!d) return serl_fail(SERL_ERR_ARG, "serl_td3_train: null descriptor");
    if (const char* why = desc_error(d)) {
        char msg[256];
        snprintf(msg, sizeof(msg), "serl_td3_train: %s", why);
        return serl_fail(SERL_ERR_ARG, msg);
    }
    if (d->n_steps == 0) return SERL_OK;
    Args a = make_args(d);
    const cudaStream_t s = (cudaStream_t)stream;
    void* ws = nullptr;
    const cudaError_t e = serl_scratch(SERL_SCRATCH_TD3, s, scratch_floats(a) * sizeof(float), &ws);
    if (e != cudaSuccess) return serl_fail_cuda(e, "td3 scratch");
    a.ws = (float*)ws;
    switch (d->cluster_size ? d->cluster_size : 8) {
    case 1: return launch<1>(a, s);
    case 2: return launch<2>(a, s);
    case 4: return launch<4>(a, s);
    default: return launch<8>(a, s);
    }
}

namespace {

// serl_td3_train_group (same_shape: every learner has learner 0's actor shape) and serl_td3_train_mixed (any shapes of
// K7's domain); `name` prefixes the error messages
int train_group(const char* name, const serl_td3_desc* descs, int n, void* stream, bool same_shape)
{
    char msg[256];
    if (n < 1 || n > SERL_TD3_MAX_GROUP) {
        snprintf(msg, sizeof(msg), "%s: n must be 1..SERL_TD3_MAX_GROUP (64)", name);
        return serl_fail(SERL_ERR_ARG, msg);
    }
    if (!descs) {
        snprintf(msg, sizeof(msg), "%s: null descriptors", name);
        return serl_fail(SERL_ERR_ARG, msg);
    }
    for (int i = 0; i < n; ++i)
        if (const char* why = desc_error(descs + i)) {
            snprintf(msg, sizeof(msg), "%s: learner %d: %s", name, i, why);
            return serl_fail(SERL_ERR_ARG, msg);
        }
    const serl_actor_shape& sh = descs[0].shape;
    const int cs = descs[0].cluster_size ? descs[0].cluster_size : 8;
    for (int i = 1; i < n; ++i) {
        const serl_actor_shape& si = descs[i].shape;
        if (same_shape && (si.state_dim != sh.state_dim || si.action_dim != sh.action_dim || si.hidden != sh.hidden ||
                           si.num_layers != sh.num_layers || si.activation != sh.activation)) {
            snprintf(msg, sizeof(msg), "%s: learner %d: actor shape differs from learner 0's (one launch trains one shape)", name, i);
            return serl_fail(SERL_ERR_ARG, msg);
        }
        if ((descs[i].cluster_size ? descs[i].cluster_size : 8) != cs) {
            snprintf(msg, sizeof(msg), "%s: learner %d: cluster_size differs from learner 0's", name, i);
            return serl_fail(SERL_ERR_ARG, msg);
        }
    }
    // the learners with steps to take, each with its own slice of one scratch buffer (slices aligned to 128 bytes)
    Group t{};
    int m = 0, wide = 0;             // learners with steps, and how many of them are wide
    size_t total = 0;
    size_t off[SERL_TD3_MAX_GROUP];
    for (int i = 0; i < n; ++i) {
        if (descs[i].n_steps == 0) continue;
        t.a[m] = make_args(descs + i);
        wide += t.a[m].h > 128;
        off[m] = total;
        total += (scratch_floats(t.a[m]) + 31) / 32 * 32;
        ++m;
    }
    if (m == 0) return SERL_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    void* ws = nullptr;
    const cudaError_t e = serl_scratch(SERL_SCRATCH_TD3, s, total * sizeof(float), &ws);
    if (e != cudaSuccess) return serl_fail_cuda(e, "td3 scratch");
    for (int g = 0; g < m; ++g) t.a[g].ws = (float*)ws + off[g];
    switch (cs) {
    case 1: return launch_group<1>(t, m, wide < m, wide > 0, s);
    case 2: return launch_group<2>(t, m, wide < m, wide > 0, s);
    case 4: return launch_group<4>(t, m, wide < m, wide > 0, s);
    default: return launch_group<8>(t, m, wide < m, wide > 0, s);
    }
}

}  // namespace

extern "C" int serl_td3_train_group(const serl_td3_desc* descs, int n, void* stream)
{
    return train_group("serl_td3_train_group", descs, n, stream, true);
}

extern "C" int serl_td3_train_mixed(const serl_td3_desc* descs, int n, void* stream)
{
    return train_group("serl_td3_train_mixed", descs, n, stream, false);
}

namespace {

template <int CS>
int launch_per(const PerLaunch& t, cudaStream_t s)
{
    if (t.a.h > 128) return serl_launch("td3_per_kernel (wide)", td3_per_kernel<CS, true>, dim3(CS), dim3(NT), 0, s, t);
    return serl_launch("td3_per_kernel", td3_per_kernel<CS, false>, dim3(CS), dim3(NT), 0, s, t);
}


}  // namespace

extern "C" int serl_td3_train_per(const serl_td3_desc* d, const serl_td3_per_desc* p, void* stream)
{
    if (!d) return serl_fail(SERL_ERR_ARG, "serl_td3_train_per: null descriptor");
    const char* why = desc_error(d);
    if (!why) why = per_error(d, p);
    if (why) {
        char msg[256];
        snprintf(msg, sizeof(msg), "serl_td3_train_per: %s", why);
        return serl_fail(SERL_ERR_ARG, msg);
    }
    if (d->n_steps == 0) return SERL_OK;
    PerLaunch t;
    t.a = make_args(d);
    t.p = Per{p->d_tree, per_leaves(p->capacity), p->n_valid, p->alpha, p->beta0, p->beta_frames, p->d_rec_weights, p->d_rec_td};
    const cudaStream_t s = (cudaStream_t)stream;
    void* ws = nullptr;
    const cudaError_t e = serl_scratch(SERL_SCRATCH_TD3, s, (scratch_floats(t.a) + t.a.B) * sizeof(float), &ws);    // + the weights
    if (e != cudaSuccess) return serl_fail_cuda(e, "td3 scratch");
    t.a.ws = (float*)ws;
    switch (d->cluster_size ? d->cluster_size : 8) {
    case 1: return launch_per<1>(t, s);
    case 2: return launch_per<2>(t, s);
    case 4: return launch_per<4>(t, s);
    default: return launch_per<8>(t, s);
    }
}
