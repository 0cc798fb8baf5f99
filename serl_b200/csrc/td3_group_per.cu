// K7 for a group of learners with prioritized or uniform replay, of any actor shapes, in one launch
// (serl_td3_train_group_per, include/serl_td3_group_per.h).
//
// One cluster per learner, as td3_mixed_kernel (td3.cu).  Cluster g branches once, uniformly for the whole cluster, on its
// learner's hidden width (narrow h <= 128, wide above) and on whether it has a priority tree, into the learner its solo
// launch runs: td3_learner<CS, WIDE, true, true> for a PER learner (td3_per_kernel's code), td3_learner<CS, WIDE, true> for
// a uniform one (td3_kernel's).  Only the CTA rank (crank<G>) differs from the solo launch, which the group and mixed
// launches show leaves the bits unchanged.  The two wide learners are inlined and the two narrow ones are __noinline__
// calls, as in td3_mixed_kernel: so ptxas spills nothing (with all four calls both wide learners spill 120-160 bytes
// inside themselves), and a narrow learner reads its Args from a 184-byte stack copy.  The learners' code is
// td3_learner.cuh's; this translation unit compiles beside td3.cu.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/serl_td3_group_per.h"
#include "../../include/serl_td3_mixed.h"
#include "td3_learner.cuh"

namespace {

// The group's launch arguments as one __grid_constant__ kernel parameter (see td3.cu's Group): learner g's Args and its
// Per, whose tree is null for a uniform learner
struct GroupPer { Args a[SERL_TD3_MAX_GROUP]; Per p[SERL_TD3_MAX_GROUP]; };
static_assert(sizeof(GroupPer) <= 32764, "SERL_TD3_MAX_GROUP learners' Args and Per must fit the sm_90 kernel-parameter limit");

template <int CS>
__device__ __noinline__ void narrow_uniform(const Args& a) { td3_learner<CS, false, true>(a); }

template <int CS>
__device__ __noinline__ void narrow_per(const Args& a, const Per& p) { td3_learner<CS, false, true, true>(a, &p); }

template <int CS>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(NT, 1) td3_group_per_kernel(const __grid_constant__ GroupPer t)
{
    unsigned g;
    asm("mov.u32 %0, %%clusterid.x;" : "=r"(g));
    const bool wide = t.a[g].h > 128, per = t.p[g].tree != nullptr;
    if (wide) {
        if (per) td3_learner<CS, true, true, true>(t.a[g], &t.p[g]);
        else td3_learner<CS, true, true>(t.a[g]);
    } else {
        if (per) narrow_per<CS>(t.a[g], t.p[g]);
        else narrow_uniform<CS>(t.a[g]);
    }
}

template <int CS>
int launch_group_per(const GroupPer& t, int n, cudaStream_t s)
{
    return serl_launch("td3_group_per_kernel", td3_group_per_kernel<CS>, dim3(n * CS), dim3(NT), 0, s, t);
}

}  // namespace

extern "C" int serl_td3_train_group_per(const serl_td3_desc* descs, const serl_td3_per_desc* pers, int n, void* stream)
{
    static const char* name = "serl_td3_train_group_per";
    char msg[256];
    if (!descs || !pers) {
        snprintf(msg, sizeof(msg), "%s: null descriptors", name);
        return serl_fail(SERL_ERR_ARG, msg);
    }
    if (n < 1 || n > SERL_TD3_MAX_GROUP) {
        snprintf(msg, sizeof(msg), "%s: n must be 1..SERL_TD3_MAX_GROUP (64)", name);
        return serl_fail(SERL_ERR_ARG, msg);
    }
    const int cs = descs[0].cluster_size ? descs[0].cluster_size : 8;
    for (int i = 0; i < n; ++i) {
        const char* why = desc_error(descs + i);
        if (!why && pers[i].d_tree) why = per_error(descs + i, pers + i);
        if (!why && (descs[i].cluster_size ? descs[i].cluster_size : 8) != cs) why = "cluster_size differs from learner 0's";
        if (why) {
            snprintf(msg, sizeof(msg), "%s: learner %d: %s", name, i, why);
            return serl_fail(SERL_ERR_ARG, msg);
        }
    }
    // without a prioritized learner with steps, the group is serl_td3_train_mixed's: its kernels inline the narrow uniform
    // learner, which this kernel calls
    bool prioritized = false;
    for (int i = 0; i < n; ++i) prioritized |= descs[i].n_steps > 0 && pers[i].d_tree != nullptr;
    if (!prioritized) return serl_td3_train_mixed(descs, n, stream);
    // the learners with steps to take, each with its own slice of one scratch buffer (slices aligned to 128 bytes); a PER
    // learner's slice holds its batch's weights after the layout, as serl_td3_train_per's scratch does
    GroupPer t{};
    int m = 0;
    size_t total = 0;
    size_t off[SERL_TD3_MAX_GROUP];
    for (int i = 0; i < n; ++i) {
        if (descs[i].n_steps == 0) continue;
        t.a[m] = make_args(descs + i);
        const serl_td3_per_desc* p = pers + i;
        if (p->d_tree)
            t.p[m] = Per{p->d_tree, per_leaves(p->capacity), p->n_valid, p->alpha, p->beta0, p->beta_frames, p->d_rec_weights, p->d_rec_td};
        off[m] = total;
        total += (scratch_floats(t.a[m]) + (p->d_tree ? t.a[m].B : 0) + 31) / 32 * 32;
        ++m;
    }
    const cudaStream_t s = (cudaStream_t)stream;
    void* ws = nullptr;
    const cudaError_t e = serl_scratch(SERL_SCRATCH_TD3, s, total * sizeof(float), &ws);
    if (e != cudaSuccess) return serl_fail_cuda(e, "td3 scratch");
    for (int g = 0; g < m; ++g) t.a[g].ws = (float*)ws + off[g];
    switch (cs) {
    case 1: return launch_group_per<1>(t, m, s);
    case 2: return launch_group_per<2>(t, m, s);
    case 4: return launch_group_per<4>(t, m, s);
    default: return launch_group_per<8>(t, m, s);
    }
}
