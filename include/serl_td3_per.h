/* serl_b200 — prioritized experience replay (PER) for K7: a device priority tree over the replay rows, its sampler, and
 * the TD3 learner that samples from it and re-prioritises the rows it trained on.  Part of the C-ABI of
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

/* serl_td3_train with prioritized replay: every step draws its `batch` rows from d_tree as serl_per_sample does (rows given
 * in the serl_td3_desc's d_indices replace the draw and are weighted by their leaves), with beta = min(1, beta0 + k (1 -
 * beta0) / beta_frames) at the learner's k-th sample (k = its critic Adam step count after the step).  The critic loss is
 * mean(w (q1 - y)^2) + mean(w (q2 - y)^2) (the td loss reported); the actor loss is unweighted.  After the critic's
 * forward pass, row j of the batch gets priority (delta_j + 1e-5)^alpha with delta_j = (|q1 - y| + |q2 - y|) / 2 of the
 * critic before its update (batch order, the later of two equal rows kept), so the next step samples from the updated tree.
 * The result is bitwise the same for every cluster size and launch split.
 *   n_valid      rows stored in the tree; must equal the serl_td3_desc's n_valid, <= capacity
 *   d_rec_weights / d_rec_td   optional records [n_steps, batch] fp32 of the weights and of delta
 * SERL_ERR_ARG before any CUDA call: every check of serl_td3_train, a null per descriptor or d_tree, capacity outside
 * 1..SERL_PER_MAX_CAPACITY, n_valid other than the desc's or > capacity, alpha not in (0, 1], beta0 not in [0, 1],
 * beta_frames not > 0. */
typedef struct {
    double* d_tree; int32_t capacity; int32_t n_valid;
    double alpha; double beta0; double beta_frames;
    float* d_rec_weights; float* d_rec_td;
} serl_td3_per_desc;
int serl_td3_train_per(const serl_td3_desc* desc, const serl_td3_per_desc* per, void* stream);

#ifdef __cplusplus
}
#endif
#endif
