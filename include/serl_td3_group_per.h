/* serl_b200 — K7 for a group of independent TD3 learners, each with prioritized or uniform replay: one launch, one
 * thread-block cluster per learner.  Part of the C-ABI of include/serl_b200.h; same conventions as serl_td3.h and
 * serl_td3_per.h (d_* device pointers owned by the caller, `stream` a cudaStream_t passed as void*, 0 on success or a
 * negative serl_status).
 */
#ifndef SERL_TD3_GROUP_PER_H
#define SERL_TD3_GROUP_PER_H

#include "serl_td3.h"     /* and serl_td3_group.h: SERL_TD3_MAX_GROUP */
#include "serl_td3_per.h"

#ifdef __cplusplus
extern "C" {
#endif

/* descs[0 .. n) and pers[0 .. n) trained in ONE launch of n x cluster_size CTAs, cluster g taking learner g's n_steps.
 * pers[g].d_tree NULL: learner g samples uniformly and takes exactly the steps (and the bits) serl_td3_train(&descs[g])
 * takes; the other fields of pers[g] are ignored.  Otherwise learner g takes exactly the steps, bits, records and tree
 * updates of serl_td3_train_per(&descs[g], &pers[g]).  Either holds whatever else is in the group, in any order and at any
 * cluster size.  Shapes may differ anywhere in K7's domain, as in serl_td3_train_mixed; all learners share `cluster_size`
 * (0 and 8 are the same size).  Learners never wait for each other, a learner with n_steps = 0 is not launched and a
 * group in which no learner has steps makes no launch; a group in which no learner with steps has a tree is launched as
 * serl_td3_train_mixed launches it.  Each learner's state, losses, records, tree and status word are
 * its own (they must not overlap another learner's); its status word receives only its own bits.
 * SERL_ERR_ARG before any CUDA call when descs or pers is null, n is outside 1..SERL_TD3_MAX_GROUP, the cluster sizes
 * differ, a learner fails a check of serl_td3_train, or a learner with a tree fails a check of serl_td3_train_per; a
 * learner's failure reads "serl_td3_train_group_per: learner i: ..." in serl_last_error. */
int serl_td3_train_group_per(const serl_td3_desc* descs, const serl_td3_per_desc* pers, int n, void* stream);

#ifdef __cplusplus
}
#endif
#endif
