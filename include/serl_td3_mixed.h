/* serl_b200 — K7 for a group of independent TD3 learners whose actor shapes differ: one launch, one thread-block cluster
 * per learner.  Part of the C-ABI of include/serl_b200.h (which includes this header); same conventions as serl_td3.h.
 */
#include "serl_td3.h"     /* and serl_td3_group.h */

/* serl_td3.h and serl_td3_group.h include serl_b200.h, and through it this header, before serl_td3_desc and
 * SERL_TD3_MAX_GROUP exist: the declaration waits until they do (through serl_b200.h, or an include of this header after
 * serl_td3.h) */
#if defined(SERL_TD3_MAX_GROUP) && !defined(SERL_TD3_MIXED_H)
#define SERL_TD3_MIXED_H

#ifdef __cplusplus
extern "C" {
#endif

/* serl_td3_train_group's contract, except that every learner may have its own `shape` anywhere in K7's domain (hidden
 * 32/64/72/96/128 at any depth, hidden 129..320 up to SERL_TD3_MAX_WIDE_LAYERS blocks): narrow and wide actors train in
 * the same launch.  Cluster g takes learner g's n_steps, exactly the steps (and the bits) serl_td3_train(&descs[g]) takes,
 * whatever else is in the group, in any order and at any cluster size.  All learners still share `cluster_size` (one
 * launch has one cluster shape; 0 and 8 are the same size).  A group in which no learner has steps makes no launch.
 * Every check serl_td3_train makes is made for every learner before any CUDA call; a failure reads
 * "serl_td3_train_mixed: learner i: ..." in serl_last_error.  SERL_ERR_ARG also when descs is null, n is outside
 * 1..SERL_TD3_MAX_GROUP or the cluster sizes differ. */
int serl_td3_train_mixed(const serl_td3_desc* descs, int n, void* stream);

#ifdef __cplusplus
}
#endif
#endif
