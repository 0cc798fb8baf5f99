// K7 for a group of learners with prioritized or uniform replay, of any actor shapes, in one launch: the kernel
// serl_td3_learn (td3.cu) runs for several learners with steps when at least one of them is prioritized.
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

}  // namespace

template <int CS>
int launch_group_per(const serl_td3_desc* descs, const serl_td3_per_desc* pers, int n, cudaStream_t s)
{
    GroupPer t{};
    const int m = pack(descs, pers, n, s, t.a, t.p);
    if (m < 0) return m;
    return serl_launch("td3_group_per_kernel", td3_group_per_kernel<CS>, dim3(m * CS), dim3(NT), 0, s, t);
}
template int launch_group_per<1>(const serl_td3_desc*, const serl_td3_per_desc*, int, cudaStream_t);
template int launch_group_per<2>(const serl_td3_desc*, const serl_td3_per_desc*, int, cudaStream_t);
template int launch_group_per<4>(const serl_td3_desc*, const serl_td3_per_desc*, int, cudaStream_t);
template int launch_group_per<8>(const serl_td3_desc*, const serl_td3_per_desc*, int, cudaStream_t);
