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
// td3_group_kernel runs several independent learners of one hidden class in one launch, one cluster each;
// td3_mixed_kernel runs narrow and wide learners together.  serl_td3_learn, the one entry point, picks the kernel (see
// launch below).  The learner itself (td3_learner and its phases) is in td3_learner.cuh, which td3_group_per.cu
// instantiates too.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/serl_td3.h"
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

// A group of narrow and wide learners in one launch: cluster g branches once, uniformly for the
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

// A PER launch: one learner, its Args and Per as one __grid_constant__ parameter
struct PerLaunch { Args a; Per p; };

template <int CS, bool WIDE>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(NT, 1) td3_per_kernel(const __grid_constant__ PerLaunch t)
{
    td3_learner<CS, WIDE, false, true>(t.a, &t.p);
}

// The kernel of a serl_td3_learn call, chosen from its learners with steps (live of them, `wide` with hidden > 128, `per`
// prioritized):
//   one, uniform                              td3_kernel<CS, h > 128>
//   one, prioritized                          td3_per_kernel<CS, h > 128>
//   several, all uniform, one width class     td3_group_kernel<CS, WIDE>
//   several, all uniform, narrow and wide     td3_mixed_kernel<CS>
//   several, at least one prioritized         td3_group_per_kernel<CS> (td3_group_per.cu)
template <int CS>
int launch(const serl_td3_desc* descs, const serl_td3_per_desc* pers, int n, int live, int wide, int per, cudaStream_t s)
{
    if (live > 1 && per) return launch_group_per<CS>(descs, pers, n, s);
    Group t{};
    Per p[SERL_TD3_MAX_GROUP];
    const int m = pack(descs, pers, n, s, t.a, p);
    if (m < 0) return m;
    const Args& a = t.a[0];
    if (live == 1 && per) {
        const PerLaunch l{a, p[0]};
        if (wide) return serl_launch("td3_per_kernel (wide)", td3_per_kernel<CS, true>, dim3(CS), dim3(NT), 0, s, l);
        return serl_launch("td3_per_kernel", td3_per_kernel<CS, false>, dim3(CS), dim3(NT), 0, s, l);
    }
    if (live == 1) {
        if (wide) return serl_launch("td3_kernel (wide)", td3_kernel<CS, true>, dim3(CS), dim3(NT), 0, s, a);
        return serl_launch("td3_kernel", td3_kernel<CS, false>, dim3(CS), dim3(NT), 0, s, a);
    }
    if (wide && wide < live) return serl_launch("td3_mixed_kernel", td3_mixed_kernel<CS>, dim3(live * CS), dim3(NT), 0, s, t);
    if (wide) return serl_launch("td3_group_kernel (wide)", td3_group_kernel<CS, true>, dim3(live * CS), dim3(NT), 0, s, t);
    return serl_launch("td3_group_kernel", td3_group_kernel<CS, false>, dim3(live * CS), dim3(NT), 0, s, t);
}

}  // namespace

extern "C" int64_t serl_td3_state_floats(const serl_actor_shape* shape)
{
    if (!shape_ok(shape)) return serl_fail(SERL_ERR_ARG, "serl_td3_state_floats: unsupported actor shape");
    return 4 * actor_floats(*shape) + 8 * (int64_t)CP;
}

extern "C" int serl_td3_learn(const serl_td3_desc* descs, const serl_td3_per_desc* pers, int n, void* stream)
{
    if (!descs) return serl_fail(SERL_ERR_ARG, "serl_td3_learn: null descriptors");
    if (n < 1 || n > SERL_TD3_MAX_GROUP) return serl_fail(SERL_ERR_ARG, "serl_td3_learn: n must be 1..SERL_TD3_MAX_GROUP (64)");
    const int cs = descs[0].cluster_size ? descs[0].cluster_size : 8;
    int live = 0, wide = 0, per = 0;          // the learners with steps, and how many of them are wide or prioritized
    for (int i = 0; i < n; ++i) {
        const serl_td3_desc* d = descs + i;
        const bool tree = pers && pers[i].d_tree;
        const char* why = desc_error(d);
        if (!why && tree) why = per_error(d, pers + i);
        if (!why && (d->cluster_size ? d->cluster_size : 8) != cs) why = "cluster_size differs from learner 0's";
        if (why) {
            char msg[256];
            snprintf(msg, sizeof(msg), "serl_td3_learn: learner %d: %s", i, why);
            return serl_fail(SERL_ERR_ARG, msg);
        }
        if (d->n_steps == 0) continue;
        ++live;
        wide += d->shape.hidden > 128;
        per += tree;
    }
    if (live == 0) return SERL_OK;
    const cudaStream_t s = (cudaStream_t)stream;
    switch (cs) {
    case 1: return launch<1>(descs, pers, n, live, wide, per, s);
    case 2: return launch<2>(descs, pers, n, live, wide, per, s);
    case 4: return launch<4>(descs, pers, n, live, wide, per, s);
    default: return launch<8>(descs, pers, n, live, wide, per, s);
    }
}
