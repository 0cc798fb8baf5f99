/* serl_b200 — prioritized experience replay (PER) for K7: a device priority tree over the replay rows and its sampler;
 * serl_td3_learn trains a learner on it (serl_td3_per_desc, include/serl_td3.h).  Part of the C-ABI of
 * include/serl_b200.h; same conventions as serl_td3.h (d_* device pointers owned by the caller, `stream` a cudaStream_t
 * passed as void*, 0 on success or a negative serl_status).
 */
#ifndef SERL_TD3_PER_H
#define SERL_TD3_PER_H

#include <stdint.h>

#include "serl_td3.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The priority tree of a buffer of `capacity` rows: a binary heap over leaves = the next power of two >= capacity, node n
 * (1 = root, leaf i = node leaves + i) at d_tree[2n] (the sum of its leaves' priorities) and d_tree[2n + 1] (their
 * minimum), all fp64.  A stored row's leaf holds its priority p > 0; every other leaf holds sum 0, min +inf.  Every internal
 * node is left + right and fmin(left, right) of its children, so the tree is a function of its leaves alone.
 * serl_per_tree_doubles: the doubles of d_tree (4 * leaves); SERL_ERR_ARG unless 1 <= capacity <= SERL_PER_MAX_CAPACITY. */
#define SERL_PER_MAX_CAPACITY (1 << 30)
int64_t serl_per_tree_doubles(int32_t capacity);

/* Every internal node recomputed from the leaves (e.g. after the caller wrote the leaves of an empty tree). */
int serl_per_rebuild(double* d_tree, int32_t capacity, void* stream);

/* The add of n rows to a ring of `capacity` rows holding n_valid rows, the first written at row `start`: the leaves of rows
 * start, start + 1, ... (mod capacity) get the largest priority stored before the add (1.0 when n_valid = 0), then the tree
 * is rebuilt.  1 <= n <= capacity, 0 <= start < capacity, 0 <= n_valid <= capacity. */
int serl_per_insert(double* d_tree, int32_t capacity, int32_t n_valid, int32_t start, int32_t n, void* stream);

/* The re-prioritising of n drawn rows: row d_rows[j] gets priority (d_td[j] + 1e-5)^alpha, in batch order (a row drawn twice
 * keeps its later value), then the changed leaves' ancestors are recomputed.  One CTA; 1 <= n <= SERL_TD3_MAX_BATCH. */
int serl_per_update(double* d_tree, int32_t capacity, const int32_t* d_rows, const float* d_td, int32_t n, double alpha,
                    void* stream);

/* K7's draw of one step's batch (global iteration `iteration`, Philox keyed by `seed`), on its own: `batch` rows drawn with
 * replacement with P(i) = p_i / sum p, and their importance weights w_i = (n_valid P(i))^-beta / (n_valid min P)^-beta
 * (fp64, rounded to fp32). */
int serl_per_sample(const double* d_tree, int32_t capacity, int32_t n_valid, int32_t batch, uint64_t seed, int64_t iteration,
                    double beta, int32_t* d_rows, float* d_weights, void* stream);

#ifdef __cplusplus
}
#endif
#endif
