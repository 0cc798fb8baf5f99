/* serl_b200 — K7: the TD3 learner of the RL half (serl_b200/core/td3.py TD3.update_parameters) as one sm_90a
 * thread-block-cluster kernel that takes n_steps consecutive gradient steps per launch.  Part of the C-ABI of
 * include/serl_b200.h (which includes this header); same conventions: d_* are device pointers owned by the caller,
 * `stream` is a cudaStream_t passed as void*, 0 on success or a negative serl_status.
 */
#ifndef SERL_TD3_H
#define SERL_TD3_H

#include <stdint.h>

#include "serl_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

#define SERL_TD3_CRITIC_HIDDEN 64      /* the 64-64 two-head critic of core/td3.py (Critic) */
#define SERL_TD3_MAX_BATCH 128
#define SERL_TD3_MAX_HIDDEN 320        /* the widest actor; above 128 the hidden blocks run as tiled phases */
#define SERL_TD3_MAX_WIDE_LAYERS 8     /* num_layers limit of the actors wider than 128 */
#define SERL_TD3_CHAMPION_TARGET 1     /* flags: use_champion_target — the actor target is not soft-updated */
#define SERL_TD3_STATUS_INDEX 4        /* d_status bit: a d_indices entry was outside [0, n_valid) (row 0 was used) */

/* Supported actors (serl_actor_shape): state_dim 7, action_dim 3, activation 0..2, and either hidden 32, 64, 72, 96 or 128
 * with any num_layers >= 1, or 129 <= hidden <= SERL_TD3_MAX_HIDDEN with 1 <= num_layers <= SERL_TD3_MAX_WIDE_LAYERS.
 * Any other shape fails with SERL_ERR_ARG before any CUDA call.
 *
 * Learner state: ONE flat fp32 buffer of serl_td3_state_floats(shape) floats,
 *   actor θ | actor target | actor Adam m | actor Adam v | critic θ | critic target | critic Adam m | critic Adam v,
 * each block in nn.Module.parameters() order: the actor's genome layout (serl_actor_num_params floats), and for the critic
 * q1 then q2, each Linear(10,64) LayerNorm(64) Linear(64,64) LayerNorm(64) Linear(64,1) = W, b, gamma, beta, W, b, gamma,
 * beta, W, b (5185 floats per head).  The critic uses the actor's activation. */
int64_t serl_td3_state_floats(const serl_actor_shape* shape);

/* One learner: n_steps consecutive TD3.update_parameters calls on global iterations first_iteration, first_iteration + 1, ...
 *   d_replay     [>= n_valid, replay_cols] fp32 transition rows (obs 7 | action 3 | next_obs 7 | reward | done, the first
 *                19 columns; replay_cols >= 19 is the row stride); every step samples `batch` distinct rows of [0, n_valid)
 *   critic_adam_steps / actor_adam_steps   Adam step counts before the launch (bias corrections continue from there)
 *   the step: target a' = clamp(actor_target(s') + clip(N(0, noise_sd), +-noise_clip), +-1),
 *   y = r + gamma * min(q1', q2') * (1 - done); critic on mse(q1, y) + mse(q2, y), gradient clipped to max_grad_norm
 *   (coef = min(1, max / (|g| + 1e-6))), Adam(lr, 0.9, 0.999, 1e-8); when iteration % policy_update_freq == 0 the actor on
 *   -mean(Q1(s, pi(s))) + caps_lambda_t * mse(a, pi(s)) + caps_lambda_s * mse(a, pi(s + U[0,1) * caps_eps_sd)) through the
 *   updated critic, clipped, Adam, then soft updates (tau) of the actor target (unless SERL_TD3_CHAMPION_TARGET) and critic
 *   target.  caps_lambda_* = 0 drops a term.
 *   Random draws: Philox4x32-10 keyed by `seed`, counter (global iteration, batch row, stream): row indices by Floyd's
 *   algorithm, target noise by Box-Muller.  They depend on neither cluster_size nor how steps are split into launches, and
 *   every reduction is summed in a fixed order: the result is bitwise reproducible.
 *   cluster_size 1, 2, 4 or 8 CTAs (0 = default 8)
 *   d_indices    optional [n_steps, batch] int32: the rows of each step's batch instead of the sampler's draw
 * outputs
 *   d_losses     [n_steps, 2] fp32 (td, pg) per step; pg (the actor loss) is NaN on critic-only steps
 *   d_rec_indices / d_rec_noise / d_rec_caps   optional records of the draws: [n_steps, batch] int32 rows,
 *                [n_steps, batch, 3] clipped target-policy noise, [n_steps, batch, 7] CAPS uniforms U (before * caps_eps_sd)
 *   d_status     optional int32 word: SERL_STATUS_NONFINITE (a loss was NaN / infinite), SERL_TD3_STATUS_INDEX */
typedef struct {
    serl_actor_shape shape;
    float* d_state;
    const float* d_replay; int32_t replay_cols; int32_t n_valid;
    int32_t batch; int32_t n_steps;
    int64_t first_iteration; int64_t critic_adam_steps; int64_t actor_adam_steps;
    double gamma; double tau; double lr; double noise_sd; double noise_clip;
    int32_t policy_update_freq;
    double caps_lambda_t; double caps_lambda_s; double caps_eps_sd;
    double max_grad_norm;
    int32_t flags;                 /* SERL_TD3_* */
    uint64_t seed;
    int32_t cluster_size;
    const int32_t* d_indices;
    float* d_losses;
    int32_t* d_rec_indices; float* d_rec_noise; float* d_rec_caps;
    int32_t* d_status;
} serl_td3_desc;
/* the largest launch: the learners' launch arguments travel as the kernel parameter, which sm_90 caps at 32,764 bytes */
#define SERL_TD3_MAX_GROUP 64

/* What prioritized replay (PER) adds to a learner: every step draws its `batch` rows from the priority tree d_tree
 * (include/serl_td3_per.h) as serl_per_sample does (rows given in the serl_td3_desc's d_indices replace the draw and are
 * weighted by their leaves), with beta = min(1, beta0 + k (1 - beta0) / beta_frames) at the learner's k-th sample (k = its
 * critic Adam step count after the step).  The critic loss is mean(w (q1 - y)^2) + mean(w (q2 - y)^2) (the td loss
 * reported); the actor loss is unweighted.  After the critic's forward pass, row j of the batch gets priority
 * (delta_j + 1e-5)^alpha with delta_j = (|q1 - y| + |q2 - y|) / 2 of the critic before its update (batch order, the later
 * of two equal rows kept), so the next step samples from the updated tree.  The result is bitwise the same for every
 * cluster size and launch split.
 *   n_valid      rows stored in the tree; must equal the serl_td3_desc's n_valid, <= capacity
 *   d_rec_weights / d_rec_td   optional records [n_steps, batch] fp32 of the weights and of delta
 * A learner with a tree is refused when capacity is outside 1..SERL_PER_MAX_CAPACITY, n_valid differs from the desc's or
 * exceeds capacity, alpha is not in (0, 1], beta0 not in [0, 1] or beta_frames not > 0. */
typedef struct {
    double* d_tree; int32_t capacity; int32_t n_valid;
    double alpha; double beta0; double beta_frames;
    float* d_rec_weights; float* d_rec_td;
} serl_td3_per_desc;

/* descs[0 .. n) trained in ONE launch, one cluster of cluster_size CTAs per learner with steps: learner g takes its
 * n_steps, and gets exactly the bits its launch alone (n = 1) gives, whatever else is in the launch, in any order.  Shapes
 * may differ anywhere in K7's domain; all learners share `cluster_size` (0 and 8 are the same size).
 *   pers         NULL: every learner samples uniformly.  Otherwise pers[g].d_tree NULL: learner g samples uniformly and
 *                the other fields of pers[g] are not read; a tree: learner g trains with prioritized replay on it.
 * Learners never wait for each other: one with fewer steps finishes early, one with n_steps = 0 gets no cluster, a call
 * in which no learner has steps makes no launch, and more learners than the GPU holds at once run in waves.  Each
 * learner's state, losses, records, tree and status word are its own (they must not overlap another learner's); its
 * status word receives only its own bits.
 * The kernel follows from the learners with steps: one runs the solo kernel (uniform or PER, narrow or wide), several
 * uniform ones of one width class (hidden <= 128, or above) the group kernel of that class, several uniform ones of both
 * classes the mixed kernel, and several with at least one prioritized the group PER kernel.
 * SERL_ERR_ARG before any CUDA call when descs is NULL, n is outside 1..SERL_TD3_MAX_GROUP, or a learner fails a check
 * above or differs from learner 0 in cluster_size; a learner's failure reads "serl_td3_learn: learner i: ..." in
 * serl_last_error. */
int serl_td3_learn(const serl_td3_desc* descs, const serl_td3_per_desc* pers, int n, void* stream);

#ifdef __cplusplus
}
#endif
#endif
