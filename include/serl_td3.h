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

/* One launch = n_steps consecutive TD3.update_parameters calls on global iterations first_iteration, first_iteration + 1, ...
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
int serl_td3_train(const serl_td3_desc* desc, void* stream);

#ifdef __cplusplus
}
#endif

/* several learners in one launch (serl_td3_train_group) */
#include "serl_td3_group.h"
#endif
