/* serl_b200 — C-ABI of the H100 (sm_90a) population-rollout + neuro-evolution engine.
 *
 * Drop-in boundary for the per-generation fitness hot path of VladGavra98/SERL (paths relative to the
 * reference tree).  All pointers named d_* are DEVICE pointers owned by the caller; `stream` is a
 * cudaStream_t passed as void* (NULL = default stream).  Every entry point returns 0 on success or a
 * negative serl_status; serl_last_error() gives the message of the last failure on the calling thread.
 * There is no CPU fallback: without a CUDA device every compute entry point fails with SERL_ERR_CUDA.
 */
#ifndef SERL_B200_H
#define SERL_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
    SERL_OK = 0,
    SERL_ERR_ARG = -1,      /* bad argument (unsupported hidden size, null pointer, ...) */
    SERL_ERR_CUDA = -2,     /* CUDA runtime error / no device */
    SERL_ERR_UNSUPPORTED = -3
} serl_status;

/* activation ids: base/core/mod_utils.py:14-18 ('relu' is LeakyReLU(0.01) in the reference) */
enum { SERL_ACT_TANH = 0, SERL_ACT_ELU = 1, SERL_ACT_LEAKY_RELU = 2 };

/* plant variants = the reference's distinct native builds envs/<variant>/_citation*.so */
enum { SERL_PLANT_H2000_V90 = 0, SERL_PLANT_ICE = 1, SERL_PLANT_CG = 2, SERL_PLANT_CG_FOR = 3,
       SERL_PLANT_H2000_V150 = 4, SERL_PLANT_H10000_V90 = 5,
       SERL_PLANT_CG_TIMED = 6,        /* envs/cg_timed before its trigger (= the nominal dynamics) */
       SERL_PLANT_CG_TIMED_POST = 7,   /* ... and once the model clock has reached 20 s (envs/phlabenv.py:159-163) */
       SERL_PLANT_COUNT = 8 };
/* command faults = envs/{be,jr,sa,se}/citation.py:71-79; env_mode = variant | (fault << 8) | (post_variant << 16):
 * post_variant != 0 is the parameter row the plant switches to when its clock reaches SERL_TRIGGER_CALLS * 0.01 s (the
 * time-triggered build cg_timed: variant 6, post_variant 7); the switch happens inside the ode5 step whose last stage
 * reaches 20 s, exactly as in the reference binary */
#define SERL_TRIGGER_CALLS 2000
/* env_mode bit 24: the `gust` build (envs/gust, envs/phlabenv.py:165-169: "vertical gust of 15 ft/s at 20 s").  Its binary
 * evaluates the nominal right-hand side with alpha replaced by alpha - atan(w_gust / V) in every aerodynamic term while
 * 20 s <= t <= 23 s (stage times of the ode5 step: the last stage of native call 1999, calls 2000..2299, the first stage of
 * call 2300); checked bit for bit against the binary on the CPU, tests/test_generated_plant.py */
#define SERL_MODE_GUST (1 << 24)
#define SERL_MODE_GUST_UP (1 << 25)    /* with SERL_MODE_GUST: the `test` build (envs/test), the same pulse with the opposite sign:
                                         alpha + atan(w_gust / V); also bit-exact against its binary */
#define SERL_GUST_END_CALLS 2300
#define SERL_GUST_W 0x1.249ba5e353f7dp+2      /* 4.572 m/s = 15 ft/s, the literal of the gust binary */
enum { SERL_FAULT_NONE = 0, SERL_FAULT_BE = 1, SERL_FAULT_JR = 2, SERL_FAULT_SA = 3, SERL_FAULT_SE = 4 };

#define SERL_REF_BLOCKS 6   /* reference-signal blocks per channel (oracle/refsig.py) */

/* Actor shape: base/core/genetic_agent.py:69-101.  Genome layout = order of nn.Module.parameters(). */
typedef struct {
    int32_t state_dim;    /* 7  (envs/phlabenv.py:92-93,220: 3 tracking errors + p,q,r,alpha) */
    int32_t action_dim;   /* 3 */
    int32_t hidden;       /* h */
    int32_t num_layers;   /* L hidden [Linear,LayerNorm,act] blocks */
    int32_t activation;   /* SERL_ACT_* */
} serl_actor_shape;

/* number of fp32 parameters of one actor: S*h+h + L*(h*h+3h) + h*A+A */
int64_t serl_actor_num_params(const serl_actor_shape* shape);

/* Population rollout — replaces the loop `for net in pop: for i in range(num_evals): evaluate(net)` of
 * base/core/agent.py:234-241 with Agent.evaluate (agent.py:63-138), CitationEnv.reset/step
 * (envs/phlabenv.py:401-482), Actor.select_action (genetic_agent.py:107-109) and the native plant
 * step (envs/<variant>/_citation*.so: step @0x6030) fused in one kernel.
 *
 *   d_weights   [pop, P] fp32, row = one actor genome
 *   d_ref_levels[n_envs, 2, SERL_REF_BLOCKS] f64 (deg), d_ref_starts same shape (s)
 *   d_env_mode  [n_envs] int32, variant | fault << 8
 *   horizon     max steps per episode (reference: 2001, phlabenv.py:82,181,392)
 *   d_action_noise optional [pop, n_envs, horizon, 3] fp32: clipped exploration noise added to the policy output
 *               (base/core/agent.py:90-93, is_action_noise=True); NULL for fitness evaluation
 * outputs
 *   d_returns   [pop, n_envs] f64  sum of rewards (agent.py:129)
 *   d_steps     [pop, n_envs] int32 executed steps
 *   d_fitness   [pop] f64 mean over envs (agent.py:245), may be NULL
 *   d_trace     optional [pop, n_envs, horizon, SERL_TRACE_COLS] f64 per-step record (Episode fields, core/utils.py:12-36):
 *               0-11 state before the step (psi, x_e, y_e are integrated only when a trace is requested),
 *               12-14 commanded deflection last_u, 15 reward, 16-18 action fed to the env, 19-21 tracking error
 *   d_actions   optional [pop, n_envs, horizon, 3] fp32: commanded deflection last_u of every executed step (agent.py:98),
 *               the input of the smoothness metric (serl_smoothness, which computes its DFT in fp32)
 */
#define SERL_TRACE_COLS 22
int serl_rollout(const float* d_weights, int32_t pop, const serl_actor_shape* shape,
                 const double* d_ref_levels, const double* d_ref_starts, const int32_t* d_env_mode,
                 int32_t n_envs, int32_t horizon, const float* d_action_noise,
                 double* d_returns, int32_t* d_steps, double* d_fitness, double* d_trace, float* d_actions,
                 void* stream);

/* Same with the episode length and reference-transition width of the reference's evaluation mode
 * (envs/phlabenv.py:295-301 set_eval_mode: t_max = 80 s; init_ref :303-345: smooth_width = t_max // 6, block_width =
 * t_max // 5 are encoded in d_ref_starts by the caller); horizon must cover t_max / 0.01 + 1 steps. */
int serl_rollout_eval(const float* d_weights, int32_t pop, const serl_actor_shape* shape,
                      const double* d_ref_levels, const double* d_ref_starts, const int32_t* d_env_mode,
                      int32_t n_envs, int32_t horizon, const float* d_action_noise,
                      double* d_returns, int32_t* d_steps, double* d_fitness, double* d_trace, float* d_actions,
                      double t_max, double smooth_width, void* stream);

/* The same launch described by a struct, with the optional inputs / outputs the two entry points above do not carry.
 *   d_env_order  optional [n_envs] int32 permutation: lane slot j flies env d_env_order[j] (the host sorts envs so that
 *                the 32 lanes of a warp share fault shims / trim; results are still written at the env's own index)
 *   d_replay     optional [pop, horizon, SERL_REPLAY_COLS] fp32: the transitions of env `replay_env` of every actor, the
 *                tuple Agent.evaluate stores when store_transition is set (base/core/agent.py:101-112):
 *                0-6 obs, 7-9 action fed to the env, 10-16 next_obs, 17 reward, 18 done, 19 cost flag (info['cost'],
 *                envs/phlabenv.py:369-375 -> critical buffer); rows past the episode's length are not written
 *   d_status     optional int32 word the kernel ORs error bits into (SERL_STATUS_*); the caller zeroes it and reads it
 *                after synchronising
 *   widths       HOST pointer to n_widths hidden-layer widths, or NULL.  n_widths == 0: the reference's uniform actor described
 *                by `shape` (K1, warp-GEMV on CUDA cores).  2 <= n_widths <= 9: the width-list generalisation
 *                Linear(7,w0) act {Linear(w_{i-1},w_i) LayerNorm act} for i = 1..n-1, Linear(w_{n-1},3) tanh (BASELINE config 5:
 *                [400,300], [128,128]; the reference's Actor at num_layers = L is [h] * (L + 1), see serl_actor_tc_widths);
 *                8 <= w0 <= 1024, 8 <= w_i <= 320, SERL_ERR_UNSUPPORTED when the list's buffers exceed an SM's shared memory;
 *                genome = parameters() order, serl_actor_num_params_wide floats per actor; only shape.activation is read
 *                from `shape`; layers 1..n-1 run on the tensor cores (wgmma, 3xTF32) with TMA-streamed weight slabs
 *   d_sensor_noise optional [pop, n_envs, horizon + 1, 7] fp32 standard-normal draws: the sensor-noise shim of
 *                envs/noise/citation.py:72-82 (mode 'noise'; also the outputs of envs/gust) applied to every native step
 *                output — row 0 for reset()'s step, row k + 1 for env step k; order p,q,r, alpha, beta, phi, theta
 *   sm_limit     > 0: use at most that many SMs (CTAs of the persistent kernel) — leaves room for small launches that run
 *                concurrently on other streams (the RL / validation episodes of Agent.train); 0 = all SMs
 *   flags        SERL_ROLLOUT_GUST: some env of the launch flies the gust build (SERL_MODE_GUST) — selects the kernel
 *                instantiation with the gust schedule (the training instantiation carries no trace of it; a gust env in a launch
 *                without the flag sets SERL_STATUS_GUST_FLAG)
 *                SERL_ROLLOUT_PER_ACTOR_REFS: every actor flies its own env block.  d_ref_levels / d_ref_starts are then
 *                [pop, n_envs, 2, SERL_REF_BLOCKS] and d_env_mode is [pop, n_envs]; env e of actor a reads row a * n_envs + e
 *                (levels, starts, mode, and the V0 of its replay rows).  The reference's own evaluation draws fresh signals for
 *                every episode of every actor (base/core/agent.py:234-241), and independent runs can share one launch.  Not
 *                with d_env_order (inside an actor's block a warp's lanes already share a mode) or d_track: SERL_ERR_ARG before
 *                any CUDA call; pop * n_envs must fit int32.  Kernel instantiations of their own; a launch without the bit runs
 *                the same code as before the bit existed
 *                SERL_ROLLOUT_STAGGER: K1 launches with two genome slots per CTA run slot 1 half a step behind slot 0
 *                instead of taking both slots' steps together.  Same result bits; slower on an H100 (DESIGN §5), kept to
 *                compare the two schedules in one process
 *   d_track      optional [pop, n_envs, SERL_TRACK_COLS] f64: per trajectory, over its executed steps k, the sums
 *                sum |e_theta|, sum |e_phi|, sum |e_beta|, sum e_beta of the tracking error of base/evaluate.py:71-100,
 *                e_k = ref(t_k) - x[[7, 6, 5]] with x the state env.x holds when step k starts (the native output of reset()'s
 *                step for k = 0, else of step k - 1, sensor noise included), summed in step order in fp64: nMAE
 *                (base/core/utils.py:39-58) without a trace.  Selects kernel instantiations of their own (with the gust
 *                schedule); a launch without it runs the same code as before the field existed
 *   d_cost       optional [pop, n_envs] int32: per trajectory, the number of its executed steps whose cost flag is set — the flag
 *                of the replay rows' column 19 (get_cost, envs/phlabenv.py:369-375, with V0 of the env's own plant variant),
 *                i.e. the safety cost trial_cost = sum info['cost'] of base/core/operator_runner.py:64.  Counted by the
 *                d_track instantiations, so it needs d_track: SERL_ERR_ARG before any CUDA call without it
 *                SERL_ROLLOUT_INCREMENTAL: incremental control (envs/phlabenv.py:174-220, 377-380, 443-466; the env
 *                PHlab_attitude_incremental).  The actor's three outputs are actuator RATES scaled to +-25 deg/s; every step
 *                integrates them in fp64, u = last_u + rate * 0.01 (no clip: the plant's input saturation acts as usual), the
 *                fault shim and the plant take u, and last_u = u.  The observation is the 7 of the absolute mode followed by
 *                (float)last_u: shape.state_dim must be 10 with the flag and 7 without it.  Replay rows then have
 *                SERL_REPLAY_COLS_OF(10) = 26 columns: 0-9 obs, 10-12 action, 13-22 next_obs, 23 reward, 24 done, 25 cost;
 *                the trace's columns 12-14 and d_actions record the integrated u (the reference's env.last_u).  Not with
 *                d_track, d_cost, SERL_ROLLOUT_GUST or d_sensor_noise: SERL_ERR_ARG before any CUDA call.  With widths (K1-TC) the genome
 *                has 10 * w0 layer-0 weights: serl_actor_num_params_wide(widths) + 3 * w0 floats per actor.
 *                The env modes are device data the host does not read: the reference flies incremental control on the
 *                nominal build only (any mode containing 'incremental' selects h2000-v90, no fault, no gust, no noise)
 *                SERL_ROLLOUT_SYMMETRIC: symmetric (pitch-only) control (envs/phlabenv.py:84-90, 226-231, 304-313; the env
 *                PHlab_symmetric_<mode>).  shape.state_dim must be 2 and shape.action_dim 1 with the flag, and a 2 / 1 shape
 *                needs the flag.  The one action is the elevator, scaled to +-10 deg like the attitude mode's; the plant and
 *                the fault shim take [de, 0, 0].  obs = [e_theta, q]; reward = -|clip(6/pi e_theta, -1, 1)|, termination and
 *                penalty as in the attitude mode (they still test phi).  The theta reference's offset is the constant trim
 *                0.22 deg instead of rad2deg(theta0); the phi channel of d_ref_levels is not read; the training episode's
 *                smooth width is t_max // 6.7 = 2 s, which the caller passes (t_max > 0).  d_action_noise is
 *                [pop, n_envs, horizon, 1].  Replay rows have SERL_REPLAY_COLS_SA(2, 1) = 8 columns: 0-1 obs, 2 action,
 *                3-4 next_obs, 5 reward, 6 done, 7 cost.  The trace's u columns and d_actions stay 3 wide and hold the padded
 *                deflection [de, 0, 0].  Not with SERL_ROLLOUT_INCREMENTAL, d_track, d_cost, SERL_ROLLOUT_GUST or
 *                d_sensor_noise: SERL_ERR_ARG before any CUDA call.  With widths (K1-TC) the genome has 2 * w0 layer-0
 *                weights and one output: serl_actor_num_params_wide(widths) - 5 * w0 - 2 * (w_last + 1) floats per actor
 *                SERL_ROLLOUT_SUITE: the launch belongs to the evaluation suite or the operator study of incremental or
 *                symmetric control.  Valid only together with exactly one of SERL_ROLLOUT_INCREMENTAL /
 *                SERL_ROLLOUT_SYMMETRIC (SERL_ERR_ARG otherwise); without it every refusal of both modes above holds.  It
 *                lifts these refusals:
 *                  with SERL_ROLLOUT_INCREMENTAL: d_track and d_cost are allowed (SERL_ROLLOUT_GUST and d_sensor_noise stay
 *                  refused: every incremental mode flies the nominal build);
 *                  with SERL_ROLLOUT_SYMMETRIC: d_track and d_cost are allowed, SERL_ROLLOUT_GUST with d_track only (the
 *                  tracking instantiations carry the gust schedule), d_sensor_noise with or without d_track.
 *                The tracking sums of incremental control are the attitude ones, with the integrated deflection u in the
 *                trace and d_actions.  With symmetric control d_track holds sum |e_theta|, 0, 0, sum e_theta, e_theta =
 *                ref_theta(t_k) (with the 0.22 deg trim) - theta of the state env.x holds when step k starts; the d_cost
 *                tally is the attitude one (it still tests alpha, phi and V)
 * t_max <= 0 selects the training defaults (20 s, smooth width 3 s). */
#define SERL_TRACK_COLS 4
#define SERL_REPLAY_COLS 20                       /* = SERL_REPLAY_COLS_OF(7) */
#define SERL_REPLAY_COLS_OF(S) (2 * (S) + 6)      /* obs S | action 3 | next_obs S | reward | done | cost */
#define SERL_REPLAY_COLS_SA(S, A) (2 * (S) + (A) + 3)     /* obs S | action A | next_obs S | reward | done | cost */
#define SERL_ROLLOUT_GUST 1
#define SERL_ROLLOUT_STAGGER 2
#define SERL_ROLLOUT_PER_ACTOR_REFS 4
#define SERL_ROLLOUT_INCREMENTAL 8
#define SERL_ROLLOUT_SYMMETRIC 16
#define SERL_ROLLOUT_SUITE 32
enum { SERL_STATUS_NONFINITE = 1,     /* a trajectory's state / return became NaN or infinite */
       SERL_STATUS_GUST_FLAG = 2 };   /* an env has SERL_MODE_GUST but the launch was not made with SERL_ROLLOUT_GUST */
typedef struct {
    const float* d_weights; int32_t pop; serl_actor_shape shape;
    const double* d_ref_levels; const double* d_ref_starts; const int32_t* d_env_mode; int32_t n_envs; int32_t horizon;
    const float* d_action_noise;
    double* d_returns; int32_t* d_steps; double* d_fitness; double* d_trace; float* d_actions;
    double t_max; double smooth_width;
    const int32_t* d_env_order;
    float* d_replay; int32_t replay_env;
    int32_t* d_status;
    int32_t sm_limit;
    const int32_t* widths; int32_t n_widths;
    const float* d_sensor_noise;
    int32_t flags;                 /* SERL_ROLLOUT_* */
    double* d_track;
    int32_t* d_cost;
} serl_rollout_desc;
int serl_rollout_run(const serl_rollout_desc* desc, void* stream);

/* Actor.forward / select_action for a batch (base/core/genetic_agent.py:104-109): d_obs [n, state_dim] fp32 ->
 * d_actions [n, action_dim] fp32 with ONE genome d_genome [P]; the arithmetic (summation order, activations) is the
 * rollout kernel's, bit for bit. */
int serl_actor_forward(const float* d_genome, const serl_actor_shape* shape, const float* d_obs, int32_t n,
                       float* d_actions, void* stream);

/* Wide (width-list) actors: parameter count, and Actor.forward for a batch through the tensor-core device code. */
int64_t serl_actor_num_params_wide(const int32_t* widths, int32_t n_widths);
int serl_actor_forward_wide(const float* d_genome, const int32_t* widths, int32_t n_widths, int32_t activation,
                            const float* d_obs, int32_t n, float* d_actions, void* stream);

/* K6: action smoothness of n_traj trajectories (base/core/utils.py:82-120 calc_smoothness; agent.py:128-134):
 * out[t] = -sqrt(sum_i sum_k f_k |FFT(y_i)[k]|^2 dt 2/N) * 100 * 80/(N dt) over the N = d_steps[t] executed steps of
 * d_actions [n_traj, horizon, 3].  horizon <= 2048: a Bluestein FFT; 2049 .. 10240: a direct DFT; longer:
 * SERL_ERR_UNSUPPORTED.  Both remove each channel's mean (bin 0 is not part of the metric) before their fp32 transform. */
int serl_smoothness(const float* d_actions, const int32_t* d_steps, int32_t n_traj, int32_t horizon, double dt,
                    double* d_out, void* stream);

/* Native plant, batched (replaces envs/<variant>/citation.py:65-72 initialize()/step() for n independent models).
 * d_X [n,19] f64 continuous states (rtX order: p q r V alpha beta phi theta psi h x_e y_e | washout | 2 params | N1 N1 N2 N2);
 * d_variant [n] SERL_PLANT_*.  serl_plant_init writes the initial condition of initialize(); serl_plant_step advances
 * every model by one 0.01 s major step (ode5) with the first three inputs d_cmd [n,3] (de, da, dr; inputs 3..9 = 0).
 * psi, x_e, y_e are not integrated (they never feed back; SURVEY.md 2.3) and keep their initial values. */
int serl_plant_init(double* d_X, const int32_t* d_variant, int32_t n, void* stream);
int serl_plant_step(double* d_X, const double* d_cmd, const int32_t* d_variant, int32_t n, void* stream);
/* the same for time-triggered builds: d_variant[i] = variant | post_variant << 16 | SERL_MODE_GUST, d_call[i] = number of native
 * step() calls the model has already made since initialize() (its clock in units of 0.01 s) */
int serl_plant_step_timed(double* d_X, const double* d_cmd, const int32_t* d_variant, const int32_t* d_call, int32_t n, void* stream);

/* ---- neuro-evolution (base/core/mod_neuro_evo.py, classic operators) -------------------------------------
 * All random draws are made on the host in the reference's order; the device applies compact op lists.
 * Launches issued on one stream execute in order; a caller must put ops with a write-after-write or
 * read-after-write hazard on the same genome into separate launches (serl_b200/evo.py does). */

/* K2: index_rank = argsort(fitness)[::-1] (mod_neuro_evo.py:460; ties -> larger index first, NaN first) and the
 * tournament winners offsprings_raw[s] = index_rank[min(draws[s,0..2])] (:44-47). d_draws: [n_off,3] int32. */
int serl_ssne_select(const double* d_fitness, int32_t pop, const int32_t* d_draws, int32_t n_off,
                     int32_t* d_index_rank, int32_t* d_offsprings_raw, void* stream);

/* K3: SSNE.clone (:371-376) for n (src,dst) genome pairs, d_pairs [n,2]. */
int serl_ssne_clone(float* d_weights, int32_t pop, int32_t P, const int32_t* d_pairs, int32_t n, void* stream);

/* K4: per pair {g1,g2,src1,src2,op_begin,op_count} (d_pair_desc [n_pairs,6]): clone src1->g1, src2->g2 (:519-522)
 * then crossover_inplace (:61-93) as ordered copies d_ops [.,3] = {offset,len,dir} (dir 0: g1<-g2, 1: g2<-g1).
 * Ops that touch the same element must have the same offset and len (a whole row of a parameter matrix, or one element
 * of a vector, as crossover_inplace copies them): the ops of a pair are kept in order without barriers. */
int serl_ssne_crossover(float* d_weights, int32_t pop, int32_t P, const int32_t* d_pair_desc, int32_t n_pairs,
                        const int32_t* d_ops, void* stream);

/* K5: mutate_inplace (:329-369): d_seg [n_seg,3] = {actor, op_begin, op_count}; op k: element d_op_off[k],
 * d_op_kind[k] (0 normal, 1 super, 2 reset), standard-normal draw d_op_z[k] already rounded to fp32. */
int serl_ssne_mutate(float* d_weights, int32_t pop, int32_t P, const int32_t* d_seg, int32_t n_seg,
                     const int32_t* d_op_off, const int32_t* d_op_kind, const float* d_op_z,
                     float mag32, float super32, void* stream);

/* Host planner (no CUDA): the crossover / mutation op generation of SSNE.epoch (mod_neuro_evo.py:516-523 + :61-93,
 * :537-539 + :329-369) consuming CPython's `random` and NumPy's legacy RandomState streams draw for draw.
 * py_state: 624 MT19937 words + index (random.getstate()[1]); py_gauss: {has_cached, cached gauss_next};
 * np_state: 624 words + pos (np.random.get_state()); all three are advanced in place.  table: [n_params,3] =
 * (offset, rows, cols).  Returns an opaque handle: query sizes {pairs, crossover ops, mutation segments, mutations, 0},
 * copy the arrays out ([pairs,6], [ops,3], [seg,3], offsets, kinds, fp32 z), destroy. */
void* serl_plan_create(uint32_t* py_state, double* py_gauss, uint32_t* np_state, const int32_t* table, int32_t n_params,
                       const int32_t* unselects, int32_t n_unselects, const int32_t* new_elitists, int32_t n_new_elitists,
                       const int32_t* offsprings, int32_t n_offsprings, const int32_t* mut_order, int32_t n_mut,
                       double mutation_prob);
void serl_plan_sizes(void* plan, int64_t* out5);
void serl_plan_copy(void* plan, int32_t* pairs, int32_t* ops, int32_t* seg, int32_t* m_off, int32_t* m_kind, float* m_z);
void serl_plan_destroy(void* plan);

/* number of kernels serl_* entry points have launched so far in this process (bench bookkeeping) */
int64_t serl_launch_count(void);

const char* serl_last_error(void);

#ifdef __cplusplus
}
#endif

/* K7, the fused TD3 learner (serl_td3_learn, serl_td3_state_floats) */
#include "serl_td3.h"
/* prioritized replay's priority tree (serl_per_*) */
#include "serl_td3_per.h"
/* the kernel of a uniform actor: K1, or K1-TC with the widths [h] * (L + 1) (serl_actor_tc_widths) */
#include "serl_route.h"
#endif
