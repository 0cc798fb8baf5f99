/* serl_b200 — K7 for a group of independent TD3 learners: one launch, one thread-block cluster per learner.  Part of the
 * C-ABI of include/serl_b200.h (through include/serl_td3.h, which includes this header); same conventions as serl_td3.h.
 */
#ifndef SERL_TD3_GROUP_H
#define SERL_TD3_GROUP_H

#include "serl_td3.h"

#ifdef __cplusplus
extern "C" {
#endif

/* the largest group: the learners' launch arguments travel as the kernel parameter, which sm_90 caps at 32,764 bytes */
#define SERL_TD3_MAX_GROUP 64

/* descs[0 .. n) trained in ONE launch of n x cluster_size CTAs: cluster g takes learner g's n_steps, exactly the steps
 * (and the bits) serl_td3_train(&descs[g]) takes.  Every field may differ between learners except `shape` and
 * `cluster_size`, which all must share (0 and 8 are the same size).  Learners never wait for each other: one with fewer
 * steps finishes early, one with n_steps = 0 is not launched, and a group larger than the number of clusters the GPU
 * holds at once runs in waves.  Each learner's state, losses, records and status word are its own (they must not overlap
 * another learner's outputs); its status word receives only its own bits.
 * Every check serl_td3_train makes is made for every learner before any CUDA call; a failure names the learner's index
 * in serl_last_error.  SERL_ERR_ARG also when n is outside 1..SERL_TD3_MAX_GROUP or the shapes / cluster sizes differ. */
int serl_td3_train_group(const serl_td3_desc* descs, int n, void* stream);

#ifdef __cplusplus
}
#endif
#endif
