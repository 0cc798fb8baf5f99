"""Host side of K1: population rollout on one GPU (torch tensors in, torch tensors out).

Mirrors the population-evaluation loop of base/core/agent.py:229-245: every actor of the population is flown
through every environment; fitness[a] = mean over envs of the episodic return.
"""
import functools

import numpy as np
import torch

from . import _native, refsig
from ._native import FAULTS, MODE_GUST, MODE_GUST_UP, PLANT_VARIANTS, REPLAY_COLS, TRACE_COLS, TRACK_COLS

HORIZON = 2001          # envs/phlabenv.py:82,181,392: t_max = 20 s, dt = 0.01, done checked before t += dt
# trace record columns (SERL_TRACE_COLS): state before the step, commanded deflection, reward, action fed to the env, error
TRACE_X, TRACE_U, TRACE_R, TRACE_A, TRACE_ERR = slice(0, 12), slice(12, 15), 15, slice(16, 19), slice(19, 22)
# the observation of incremental control (envs/phlabenv.py:214-220): the 7 of the absolute mode + last_u.  A shape with this
# state_dim flies with SERL_ROLLOUT_INCREMENTAL
INCREMENTAL_STATE_DIM = 10
# the actor of symmetric control (envs/phlabenv.py:86-89): obs = [e_theta, q] -> the elevator.  A shape with these widths flies
# with SERL_ROLLOUT_SYMMETRIC
SYMMETRIC_STATE_DIM, SYMMETRIC_ACTION_DIM = 2, 1


def is_symmetric(shape):
    return shape.state_dim == SYMMETRIC_STATE_DIM and shape.action_dim == SYMMETRIC_ACTION_DIM


# The replay row of an observation of S entries and A actions (SERL_REPLAY_COLS_SA): obs S | action A | next_obs S | reward |
# done | cost.  Every buffer stores the transition, the row without its last column (the cost flag).
def replay_dims(state_dim=7, action_dim=3):
    """widths of the fields of a replay row: obs, action, next_obs, reward, done, cost"""
    return (state_dim, action_dim, state_dim, 1, 1, 1)


def replay_cols(state_dim=7, action_dim=3):
    return sum(replay_dims(state_dim, action_dim))


def transition_cols(state_dim=7, action_dim=3):
    """columns of a stored transition, which is also the column of a replay row's cost flag"""
    return replay_cols(state_dim, action_dim) - 1


TRANSITION_COLS = REPLAY_COST = transition_cols(7)       # SERL_REPLAY_COLS - 1
# time-triggered builds: parameter row the plant switches to when its clock reaches 20 s (envs/phlabenv.py:159-163)
POST_VARIANT = {'cg_timed': 'cg_timed_post'}
# env mode string (envs/phlabenv.py:99-172) -> (plant variant, command fault)
MODES = {
    'nominal': ('h2000_v90', 'none'), 'be': ('h2000_v90', 'be'), 'jr': ('h2000_v90', 'jr'),
    'sa': ('h2000_v90', 'sa'), 'se': ('h2000_v90', 'se'), 'ice': ('ice', 'none'), 'cg': ('cg', 'none'),
    'cg-for': ('cg_for', 'none'), 'h2000-v150': ('h2000_v150', 'none'), 'h10000-v90': ('h10000_v90', 'none'),
    'cg-timed': ('cg_timed', 'none'),
    'gust': ('h2000_v90', 'none'),      # nominal dynamics + MODE_GUST (include/serl_b200.h); the env adds the sensor-noise shim
    'test': ('h2000_v90', 'none'),      # envs/test: the same pulse with the opposite sign (MODE_GUST | MODE_GUST_UP), no shim
}


def mode_code(mode):
    v, f = MODES[mode]
    post = PLANT_VARIANTS.index(POST_VARIANT[v]) if v in POST_VARIANT else 0
    return PLANT_VARIANTS.index(v) | (FAULTS.index(f) << 8) | (post << 16) | (MODE_GUST if mode in ('gust', 'test') else 0) | (MODE_GUST_UP if mode == 'test' else 0)


def mode_variant(code):
    return code & 0xff


def mode_gust(code):
    return bool(code & MODE_GUST)


def timed_plant_code(code):
    """the env_mode without its fault field (serl_plant_step_timed), or None if the plant needs no clock (no post variant, gust)"""
    return code & ~0xff00 if code >> 16 else None


def actor_shape(hidden, num_layers=3, activation='tanh', state_dim=7, action_dim=3):
    return _native.ActorShape(state_dim, action_dim, hidden, num_layers, _native.ACTIVATIONS[activation.lower()])


def num_params(shape):
    return int(_native.lib().serl_actor_num_params(shape))


class RolloutResult:
    __slots__ = ('returns', 'steps', 'fitness', 'trace', 'actions', 'smoothness', 'replay', 'status', 'track', 'cost')

    trace_x = property(lambda s: s.trace[..., TRACE_X])
    trace_u = property(lambda s: s.trace[..., TRACE_U])
    trace_r = property(lambda s: s.trace[..., TRACE_R])
    trace_a = property(lambda s: s.trace[..., TRACE_A])
    trace_err = property(lambda s: s.trace[..., TRACE_ERR])

    def check(self):
        """raise if the kernel flagged a non-finite trajectory (synchronises the device)."""
        st = int(self.status.item()) if self.status is not None else 0
        if st & _native.STATUS_GUST_FLAG:
            raise _native.NativeError("serl_rollout: an env has mode 'gust' but the launch was not made with gust=True")
        if st & _native.STATUS_NONFINITE:
            raise _native.NativeError('serl_rollout: a trajectory produced a non-finite state / return (status flag)')


def variant_sorted_order(env_mode):
    """permutation that groups envs by mode (plant variant, fault shim): the 32 lanes of a warp then share the shim's
    branch and the variant's parameter row.  Results are still written at each env's own index."""
    return torch.argsort(env_mode, stable=True).to(torch.int32)


def population_rollout(weights, shape, ref_levels, ref_starts, env_mode, horizon=HORIZON, trace=False, out=None, action_noise=None,
                       actions=False, t_max=None, smooth_width=None, env_order=None, replay_env=None, status=True, sm_limit=0,
                       fitness=True, widths=None, sensor_noise=None, gust=False, stagger=False, track=False, cost=False,
                       suite=False):
    """weights [pop,P] fp32 cuda; ref_levels/ref_starts [n_envs,2,6] f64 cuda; env_mode [n_envs] int32 cuda.
    Per-actor env blocks: ref_levels/ref_starts [pop,n_envs,2,6] and env_mode [pop,n_envs] give every actor its own n_envs
    envs (SERL_ROLLOUT_PER_ACTOR_REFS; the shapes select the layout; not with env_order or track).
    env_order: optional int32 [n_envs] permutation (see variant_sorted_order); replay_env: record the transitions of that env
    of every actor into result.replay [pop, horizon, REPLAY_COLS]; status: carry the device status word (result.check());
    sm_limit: SMs this launch may occupy (0 = all); fitness=False skips the per-actor mean kernel.
    stagger=True: K1's two genome slots of a CTA run half a step apart instead of taking their steps together (same results,
    slower on an H100; to time the two schedules against each other).
    track=True: result.track [pop, n_envs, TRACK_COLS] f64 holds each trajectory's tracking-error sums
    (sum |e_theta|, sum |e_phi|, sum |e_beta|, sum e_beta; serl_rollout_desc.d_track), the nMAE of a trajectory without a trace.
    cost=True (with track=True): result.cost [pop, n_envs] int32 holds each trajectory's safety cost, the number of its executed
    steps whose cost flag (the replay rows' last column) is set (serl_rollout_desc.d_cost).
    shape.state_dim = INCREMENTAL_STATE_DIM flies incremental control (SERL_ROLLOUT_INCREMENTAL: rate commands integrated into the
    deflection, obs + last_u, replay rows of replay_cols(10) columns; on K1 and K1-TC, without track, cost, gust or sensor_noise).
    A 2 -> 1 shape (is_symmetric) flies symmetric control (SERL_ROLLOUT_SYMMETRIC: the elevator alone, obs = [e_theta, q], the theta
    reference of refsig.make_ref_params(symmetric=True) with its smooth width, action_noise [pop, n_envs, horizon, 1], replay rows
    of replay_cols(2, 1) columns; on K1 and K1-TC, without track, cost, gust or sensor_noise).
    suite=True (SERL_ROLLOUT_SUITE, with incremental or symmetric control only): a launch of the evaluation suite or the operator
    study.  It lifts these refusals: incremental control takes track and cost (still not gust or sensor_noise); symmetric control
    takes track and cost, gust with track, and sensor_noise.  Symmetric control's track holds sum |e_theta|, 0, 0, sum e_theta
    (evaluation.nmae_from_track(symmetric=True)).  Nothing sets it implicitly.
    widths=[w0, w1, ..., w_{n-1}] (2 to 9 widths): width-list actors on the tensor-core kernel K1-TC (csrc/rollout_tc.cu); `shape`
    then only supplies the activation.  widths=None flies the uniform actor `shape` on K1, or on K1-TC with [h] * (L + 1) when its
    genome does not fit K1's kernels (tc_widths)."""
    if not weights.is_cuda:
        raise _native.NativeError('population_rollout needs CUDA tensors (no CPU fallback)')
    if widths is None:
        widths = tc_widths(shape)
    pop, P = weights.shape
    assert weights.dtype == torch.float32 and weights.is_contiguous()
    assert P == (num_params_wide(widths, shape.state_dim, shape.action_dim) if widths else num_params(shape)), (P, widths)
    sym = is_symmetric(shape)
    per_actor = env_mode.dim() == 2
    n_envs = env_mode.shape[-1]
    block = (pop, n_envs) if per_actor else (n_envs,)
    assert env_mode.shape == block and env_mode.dtype == torch.int32 and (env_mode.is_contiguous() or not per_actor)
    assert ref_levels.shape == block + (2, 6) and ref_levels.dtype == torch.float64 and ref_levels.is_contiguous()
    assert ref_starts.shape == block + (2, 6) and ref_starts.dtype == torch.float64 and ref_starts.is_contiguous()
    if action_noise is not None:
        assert action_noise.shape == (pop, n_envs, horizon, shape.action_dim if sym else 3) and action_noise.dtype == torch.float32 and action_noise.is_contiguous()
    if env_order is not None:
        assert env_order.shape == (n_envs,) and env_order.dtype == torch.int32 and env_order.is_cuda
    dev = weights.device
    r = out if out is not None else RolloutResult()
    if out is None:
        r.returns = torch.empty((pop, n_envs), dtype=torch.float64, device=dev)
        r.steps = torch.empty((pop, n_envs), dtype=torch.int32, device=dev)
        r.fitness = torch.empty((pop,), dtype=torch.float64, device=dev) if fitness else None
        r.trace = None
        r.smoothness = None
        r.actions = torch.empty((pop, n_envs, horizon, 3), dtype=torch.float32, device=dev) if actions else None
        r.replay = torch.empty((pop, horizon, replay_cols(shape.state_dim, shape.action_dim)), dtype=torch.float32, device=dev) if replay_env is not None else None
        r.status = torch.zeros((1,), dtype=torch.int32, device=dev) if status else None
        r.track = torch.empty((pop, n_envs, TRACK_COLS), dtype=torch.float64, device=dev) if track else None
        r.cost = torch.empty((pop, n_envs), dtype=torch.int32, device=dev) if cost else None
        if trace:
            r.trace = torch.full((pop, n_envs, horizon, TRACE_COLS), float('nan'), dtype=torch.float64, device=dev)
    elif r.status is not None:
        r.status.zero_()
    p = lambda t: t.data_ptr() if t is not None else None       # device memory owned by the caller or by r
    d = _native.RolloutDesc()
    d.d_weights, d.pop, d.shape = p(weights), pop, shape
    d.d_ref_levels, d.d_ref_starts, d.d_env_mode, d.n_envs, d.horizon = p(ref_levels), p(ref_starts), p(env_mode), n_envs, horizon
    d.d_action_noise = p(action_noise)
    d.d_returns, d.d_steps, d.d_fitness, d.d_trace, d.d_actions = p(r.returns), p(r.steps), p(r.fitness), p(r.trace), p(getattr(r, 'actions', None))
    if t_max is not None:      # evaluation mode (envs/phlabenv.py:295-301): longer episodes, wider reference transitions
        d.t_max = float(t_max)
        d.smooth_width = float(smooth_width if smooth_width is not None else refsig.widths(t_max, sym)[1])
    elif sym:                  # symmetric control's training episode: 20 s with 2 s transitions (t_max // 6.7)
        d.t_max, d.smooth_width = 20.0, float(smooth_width if smooth_width is not None else refsig.widths(20, True)[1])
    d.d_env_order = p(env_order)
    d.d_replay, d.replay_env = p(getattr(r, 'replay', None)), int(replay_env if replay_env is not None else 0)
    d.d_status = p(getattr(r, 'status', None))
    d.d_track = p(getattr(r, 'track', None))
    d.d_cost = p(getattr(r, 'cost', None))
    if sm_limit < 0:         # leave -sm_limit SMs to concurrent small launches
        sm_limit = max(1, torch.cuda.get_device_properties(dev).multi_processor_count + int(sm_limit))
    d.sm_limit = int(sm_limit)
    if sensor_noise is not None:      # envs/noise/citation.py:72-82: standard-normal draws [pop, n_envs, horizon + 1, 7]
        assert sensor_noise.shape == (pop, n_envs, horizon + 1, 7) and sensor_noise.dtype == torch.float32 and sensor_noise.is_contiguous()
        d.d_sensor_noise = p(sensor_noise)
    d.flags = ((_native.ROLLOUT_GUST if gust else 0) | (_native.ROLLOUT_STAGGER if stagger else 0)      # gust: mode_code(...) & MODE_GUST
               | (_native.ROLLOUT_PER_ACTOR_REFS if per_actor else 0)
               | (_native.ROLLOUT_INCREMENTAL if shape.state_dim == INCREMENTAL_STATE_DIM else 0)
               | (_native.ROLLOUT_SYMMETRIC if sym else 0) | (_native.ROLLOUT_SUITE if suite else 0))
    if widths:
        warr = np.asarray(widths, dtype=np.int32)       # host array, alive until the call returns
        d.widths, d.n_widths = warr.ctypes.data, len(widths)
    _native.call('serl_rollout_run', d, device=dev)
    return r


def tc_widths(shape):
    """None when K1 flies the uniform actor `shape` (or reports why it cannot), else the width list [h] * (L + 1) of the same
    genome for K1-TC (serl_actor_tc_widths: K1's fit rule lives in csrc/rollout.cu)"""
    out = np.zeros(max(shape.num_layers + 1, 1), dtype=np.int32)
    n = _native.lib().serl_actor_tc_widths(shape, out.ctypes, out.size)
    _native.check(min(n, 0), 'serl_actor_tc_widths')
    return out[:n].tolist() if n else None


def num_params_wide(widths, state_dim=7, action_dim=3):
    """parameters of a width-list actor; serl_actor_num_params_wide counts a 7-entry observation and 3 actions: incremental
    control's layer 0 has 3 * w0 weights more, symmetric control's 5 * w0 fewer and its output layer 2 * (w_last + 1) fewer"""
    n = int(_native.lib().serl_actor_num_params_wide(np.asarray(widths, dtype=np.int32).ctypes, len(widths)))
    return n + (state_dim - 7) * int(widths[0]) + (action_dim - 3) * (int(widths[-1]) + 1)


def actor_forward_wide(genome, widths, activation, obs):
    """forward pass of a width-list actor [w0, ..., w_{n-1}] (2 to 9 widths) for a batch of observations through the tensor-core
    device code (wgmma 3xTF32)."""
    if not genome.is_cuda:
        raise _native.NativeError('actor_forward_wide needs CUDA tensors (no CPU fallback)')
    assert genome.dtype == torch.float32 and genome.is_contiguous() and genome.numel() == num_params_wide(widths)
    assert obs.dtype == torch.float32 and obs.is_contiguous() and obs.shape[1] == 7
    out = torch.empty((obs.shape[0], 3), dtype=torch.float32, device=genome.device)
    act = _native.ACTIVATIONS[activation.lower()]
    _native.call('serl_actor_forward_wide', genome, np.asarray(widths, dtype=np.int32), len(widths), act, obs, obs.shape[0], out)
    return out


def actor_forward(genome, shape, obs):
    """Actor.forward for a batch (base/core/genetic_agent.py:104-109): genome [P] fp32 cuda, obs [n,7] fp32 cuda -> [n,3].
    Same device code (summation order, activations) as the rollout kernel."""
    if not genome.is_cuda:
        raise _native.NativeError('actor_forward needs CUDA tensors (no CPU fallback)')
    assert genome.dtype == torch.float32 and genome.is_contiguous() and genome.numel() == num_params(shape)
    assert obs.dtype == torch.float32 and obs.is_contiguous() and obs.shape[1] == shape.state_dim
    out = torch.empty((obs.shape[0], shape.action_dim), dtype=torch.float32, device=genome.device)
    _native.call('serl_actor_forward', genome, shape, obs, obs.shape[0], out)
    return out


def smoothness(actions, steps, dt=0.01):
    """K6: per-trajectory action smoothness (core/utils.py calc_smoothness) of `actions` [..., horizon, 3] fp32 (cuda) over the
    first `steps` [...] executed steps. Returns f64 tensor shaped like `steps`."""
    horizon = actions.shape[-2]
    n = steps.numel()
    assert actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous() and actions.numel() == n * horizon * 3
    st = steps.contiguous().to(torch.int32)
    out = torch.empty(st.shape, dtype=torch.float64, device=actions.device)
    _native.call('serl_smoothness', actions, st, n, horizon, dt, out)
    return out


def plant_init(variant):
    """serl_plant_init: the initial conditions [n, 19] f64 of the plant variants `variant` [n] int32 (cuda)."""
    X = torch.empty((variant.shape[0], 19), dtype=torch.float64, device=variant.device)
    _native.call('serl_plant_init', X, variant, X.shape[0])
    return X


def plant_step(X, cmd, variant, call=None):
    """one 0.01 s step of the plants X [n, 19] f64 under cmd [n, 3] f64; variant [n] int32, or timed_plant_code values with call [n]"""
    if call is None:
        _native.call('serl_plant_step', X, cmd, variant, X.shape[0])
    else:
        _native.call('serl_plant_step_timed', X, cmd, variant, call, X.shape[0])


@functools.cache        # only the first call per variant waits for the current stream (DESIGN §6: Agent._collect)
def initial_state(variant):
    """the 12 flight states (read-only host f64) plant variant `variant` starts from"""
    x = plant_init(torch.tensor([variant], dtype=torch.int32, device='cuda'))[0, :12].cpu().numpy()
    x.flags.writeable = False
    return x
