"""Host side of K1: population rollout on one GPU (torch tensors in, torch tensors out).

Mirrors the population-evaluation loop of base/core/agent.py:229-245: every actor of the population is flown
through every environment; fitness[a] = mean over envs of the episodic return.
"""
import ctypes

import torch

from . import _native

HORIZON = 2001          # envs/phlabenv.py:82,181,392: t_max = 20 s, dt = 0.01, done checked before t += dt
PLANT_VARIANTS = ['h2000_v90', 'ice', 'cg', 'cg_for', 'h2000_v150', 'h10000_v90', 'cg_timed', 'cg_timed_post']
# time-triggered builds: parameter row the plant switches to when its clock reaches 20 s (envs/phlabenv.py:159-163)
POST_VARIANT = {'cg_timed': 'cg_timed_post'}
FAULTS = ['none', 'be', 'jr', 'sa', 'se']
# env mode string (envs/phlabenv.py:99-172) -> (plant variant, command fault)
MODES = {
    'nominal': ('h2000_v90', 'none'), 'be': ('h2000_v90', 'be'), 'jr': ('h2000_v90', 'jr'),
    'sa': ('h2000_v90', 'sa'), 'se': ('h2000_v90', 'se'), 'ice': ('ice', 'none'), 'cg': ('cg', 'none'),
    'cg-for': ('cg_for', 'none'), 'h2000-v150': ('h2000_v150', 'none'), 'h10000-v90': ('h10000_v90', 'none'),
    'cg-timed': ('cg_timed', 'none'),
    'gust': ('h2000_v90', 'none'),      # nominal dynamics + MODE_GUST (include/serl_b200.h); the env adds the sensor-noise shim
    'test': ('h2000_v90', 'none'),      # envs/test: the same pulse with the opposite sign (MODE_GUST | MODE_GUST_UP), no shim
}
MODE_GUST = 1 << 24
MODE_GUST_UP = 1 << 25


def mode_code(mode):
    v, f = MODES[mode]
    post = PLANT_VARIANTS.index(POST_VARIANT[v]) if v in POST_VARIANT else 0
    return PLANT_VARIANTS.index(v) | (FAULTS.index(f) << 8) | (post << 16) | (MODE_GUST if mode in ('gust', 'test') else 0) | (MODE_GUST_UP if mode == 'test' else 0)


def actor_shape(hidden, num_layers=3, activation='tanh', state_dim=7, action_dim=3):
    return _native.ActorShape(state_dim, action_dim, hidden, num_layers, _native.ACTIVATIONS[activation.lower()])


def num_params(shape):
    return int(_native.lib().serl_actor_num_params(ctypes.byref(shape)))


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


class RolloutResult:
    __slots__ = ('returns', 'steps', 'fitness', 'trace', 'actions', 'smoothness', 'replay', 'status')

    # views into the trace record (include/serl_b200.h: SERL_TRACE_COLS)
    trace_x = property(lambda s: s.trace[..., 0:12])
    trace_u = property(lambda s: s.trace[..., 12:15])
    trace_r = property(lambda s: s.trace[..., 15])
    trace_a = property(lambda s: s.trace[..., 16:19])
    trace_err = property(lambda s: s.trace[..., 19:22])

    def check(self):
        """raise if the kernel flagged a non-finite trajectory (synchronises the device)."""
        st = int(self.status.item()) if self.status is not None else 0
        if st & _native.STATUS_GUST_FLAG:
            raise _native.NativeError("serl_rollout: an env has mode 'gust' but the launch was not made with gust=True")
        if st & _native.STATUS_NONFINITE:
            raise _native.NativeError('serl_rollout: a trajectory produced a non-finite state / return (status flag)')


TRACE_COLS = 22
REPLAY_COLS = _native.REPLAY_COLS


def variant_sorted_order(env_mode):
    """permutation that groups envs by mode (plant variant, fault shim): the 32 lanes of a warp then share the shim's
    branch and the variant's parameter row.  Results are still written at each env's own index."""
    return torch.argsort(env_mode, stable=True).to(torch.int32)


def population_rollout(weights, shape, ref_levels, ref_starts, env_mode, horizon=HORIZON, trace=False, out=None, action_noise=None,
                       actions=False, t_max=None, smooth_width=None, env_order=None, replay_env=None, status=True, sm_limit=0,
                       fitness=True, widths=None, sensor_noise=None, gust=False):
    """weights [pop,P] fp32 cuda; ref_levels/ref_starts [n_envs,2,6] f64 cuda; env_mode [n_envs] int32 cuda.
    env_order: optional int32 [n_envs] permutation (see variant_sorted_order); replay_env: record the transitions of that env
    of every actor into result.replay [pop, horizon, REPLAY_COLS]; status: carry the device status word (result.check());
    sm_limit: SMs this launch may occupy (0 = all); fitness=False skips the per-actor mean kernel.
    widths=[w1, w2]: wide two-hidden-layer actors on the tensor-core kernel (csrc/rollout_tc.cu); `shape` then only supplies the
    activation."""
    if not weights.is_cuda:
        raise _native.NativeError('population_rollout needs CUDA tensors (no CPU fallback)')
    L = _native.lib()
    pop, P = weights.shape
    assert weights.dtype == torch.float32 and weights.is_contiguous()
    assert P == (num_params_wide(widths) if widths else num_params(shape)), (P, widths)
    n_envs = env_mode.shape[0]
    assert ref_levels.shape == (n_envs, 2, 6) and ref_levels.dtype == torch.float64 and ref_levels.is_contiguous()
    assert ref_starts.shape == (n_envs, 2, 6) and ref_starts.dtype == torch.float64 and ref_starts.is_contiguous()
    assert env_mode.dtype == torch.int32
    if action_noise is not None:
        assert action_noise.shape == (pop, n_envs, horizon, 3) and action_noise.dtype == torch.float32 and action_noise.is_contiguous()
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
        r.replay = torch.empty((pop, horizon, REPLAY_COLS), dtype=torch.float32, device=dev) if replay_env is not None else None
        r.status = torch.zeros((1,), dtype=torch.int32, device=dev) if status else None
        if trace:
            r.trace = torch.full((pop, n_envs, horizon, TRACE_COLS), float('nan'), dtype=torch.float64, device=dev)
    elif r.status is not None:
        r.status.zero_()
    stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    p = lambda t: t.data_ptr() if t is not None else None
    d = _native.RolloutDesc()
    d.d_weights, d.pop, d.shape = p(weights), pop, shape
    d.d_ref_levels, d.d_ref_starts, d.d_env_mode, d.n_envs, d.horizon = p(ref_levels), p(ref_starts), p(env_mode), n_envs, horizon
    d.d_action_noise = p(action_noise)
    d.d_returns, d.d_steps, d.d_fitness, d.d_trace, d.d_actions = p(r.returns), p(r.steps), p(r.fitness), p(r.trace), p(getattr(r, 'actions', None))
    if t_max is not None:      # evaluation mode (envs/phlabenv.py:295-301): longer episodes, wider reference transitions
        d.t_max = float(t_max)
        d.smooth_width = float(smooth_width if smooth_width is not None else float(t_max // 6))
    d.d_env_order = p(env_order)
    d.d_replay, d.replay_env = p(getattr(r, 'replay', None)), int(replay_env if replay_env is not None else 0)
    d.d_status = p(getattr(r, 'status', None))
    if sm_limit < 0:         # leave -sm_limit SMs to concurrent small launches
        sm_limit = max(1, torch.cuda.get_device_properties(dev).multi_processor_count + int(sm_limit))
    d.sm_limit = int(sm_limit)
    if sensor_noise is not None:      # envs/noise/citation.py:72-82: standard-normal draws [pop, n_envs, horizon + 1, 7]
        assert sensor_noise.shape == (pop, n_envs, horizon + 1, 7) and sensor_noise.dtype == torch.float32 and sensor_noise.is_contiguous()
        d.d_sensor_noise = p(sensor_noise)
    d.flags = _native.ROLLOUT_GUST if gust else 0       # some env flies the gust build (mode_code(...) & MODE_GUST)
    if widths:
        warr = (ctypes.c_int32 * len(widths))(*[int(x) for x in widths])
        d.widths, d.n_widths = ctypes.cast(warr, ctypes.c_void_p), len(widths)
    _native.check(L.serl_rollout_run(ctypes.byref(d), stream), 'serl_rollout_run')
    return r


def num_params_wide(widths):
    arr = (ctypes.c_int32 * len(widths))(*[int(x) for x in widths])
    return int(_native.lib().serl_actor_num_params_wide(arr, len(widths)))


def actor_forward_wide(genome, widths, activation, obs):
    """forward pass of a wide [w1, w2] actor for a batch of observations through the tensor-core device code (wgmma 3xTF32)."""
    if not genome.is_cuda:
        raise _native.NativeError('actor_forward_wide needs CUDA tensors (no CPU fallback)')
    assert genome.dtype == torch.float32 and genome.is_contiguous() and genome.numel() == num_params_wide(widths)
    assert obs.dtype == torch.float32 and obs.is_contiguous() and obs.shape[1] == 7
    out = torch.empty((obs.shape[0], 3), dtype=torch.float32, device=genome.device)
    arr = (ctypes.c_int32 * len(widths))(*[int(x) for x in widths])
    stream = ctypes.c_void_p(torch.cuda.current_stream(genome.device).cuda_stream)
    _native.check(_native.lib().serl_actor_forward_wide(_ptr(genome), arr, len(widths), _native.ACTIVATIONS[activation.lower()], _ptr(obs),
                                                        obs.shape[0], _ptr(out), stream), 'serl_actor_forward_wide')
    return out


def actor_forward(genome, shape, obs):
    """Actor.forward for a batch (base/core/genetic_agent.py:104-109): genome [P] fp32 cuda, obs [n,7] fp32 cuda -> [n,3].
    Same device code (summation order, activations) as the rollout kernel."""
    if not genome.is_cuda:
        raise _native.NativeError('actor_forward needs CUDA tensors (no CPU fallback)')
    assert genome.dtype == torch.float32 and genome.is_contiguous() and genome.numel() == num_params(shape)
    assert obs.dtype == torch.float32 and obs.is_contiguous() and obs.shape[1] == shape.state_dim
    out = torch.empty((obs.shape[0], shape.action_dim), dtype=torch.float32, device=genome.device)
    stream = ctypes.c_void_p(torch.cuda.current_stream(genome.device).cuda_stream)
    _native.check(_native.lib().serl_actor_forward(_ptr(genome), ctypes.byref(shape), _ptr(obs), obs.shape[0], _ptr(out), stream),
                  'serl_actor_forward')
    return out


def smoothness(actions, steps, dt=0.01):
    """K6: per-trajectory action smoothness (core/utils.py calc_smoothness) of `actions` [..., horizon, 3] fp32 (cuda) over the
    first `steps` [...] executed steps. Returns f64 tensor shaped like `steps`."""
    L = _native.lib()
    horizon = actions.shape[-2]
    n = steps.numel()
    assert actions.is_cuda and actions.dtype == torch.float32 and actions.is_contiguous() and actions.numel() == n * horizon * 3
    st = steps.contiguous().to(torch.int32)
    out = torch.empty(st.shape, dtype=torch.float64, device=actions.device)
    stream = ctypes.c_void_p(torch.cuda.current_stream(actions.device).cuda_stream)
    _native.check(L.serl_smoothness(_ptr(actions), _ptr(st), n, horizon, dt, _ptr(out), stream), 'serl_smoothness')
    return out
