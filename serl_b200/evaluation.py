"""Evaluation of trained actors on user-defined references — the device version of base/evaluate.py (`evaluate`,
`validate_agent`, `-eval_pop`) and base/evaluation_utils.py (`gen_refs`, `load_pop`, `load_rl_agent`).  Episodes run in
evaluation mode (t_max = 80 s, envs/phlabenv.py:295-301) on any plant variant / fault shim including the sensor-noise shim
(envs/noise/citation.py:72-82).

validate_agent flies the trials of ONE actor on ONE condition in one traced launch and returns what the reference returns:
the time traces of the last trial and Stats(nmae, nmae_sd, sm, sm_sd).  evaluate_population flies every actor of a
population on every condition in one untraced launch per sensor-noise group: the kernel accumulates each trajectory's
tracking-error sums (rollout.population_rollout(track=True)), from which nMAE follows, and K6 takes the smoothness of the
recorded deflections."""
import os
from collections import namedtuple

import numpy as np
import torch

from . import refsig, rollout, signals
from .core.utils import calc_nMAE, calc_smoothness, load_config

Stats = namedtuple('Stats', ('nmae', 'nmae_sd', 'sm', 'sm_sd'))
T_MAX = 80                       # base/evaluate.py: the evaluation episode length [s]
# every flight condition the rollout kernels fly (envs/phlabenv.py:99-172 mode names; `-env all` of examples/evaluate.py)
CONDITIONS = ('nominal', 'low-q', 'high-q', 'be', 'jr', 'sa', 'se', 'cg', 'ice', 'cg-shift', 'noise', 'gust', 'test')
# largest [actors, envs, horizon, 3] fp32 deflection record one launch of evaluate_population keeps for K6 (bytes); more
# actors than fit are flown in chunks
ACTIONS_CAP = 4 << 30


def sensor_noise_draws(n_traj, horizon):
    """standard-normal draws of the sensor-noise shim in ITS order (randn(3), randn(1), randn(1), randn(2) per native call),
    one episode after the other: [n_traj, horizon + 1, 7] float32.  One randn call: legacy np.random keeps its cached second
    gaussian across calls, so the stream is the same as the shim's per-call draws."""
    return np.random.randn(n_traj * (horizon + 1) * 7).reshape(n_traj, horizon + 1, 7).astype(np.float32)


def reset_state(x_ic, z0=None):
    """env.x after reset(): the plant's initial flight states x_ic [12], passed through the sensor-noise shim with the draws
    z0 [7] of reset()'s native call when the env has it (envs/noise/citation.py:72-82, the rollout kernels' arithmetic)"""
    x = np.array(x_ic, dtype=np.float64)
    if z0 is not None:
        z = np.asarray(z0, dtype=np.float32).astype(np.float64)
        x[0:3] += 3.0 * 1e-5 + 6.3 * 1e-4 * z[0:3]
        x[4] += 4.0 * 1e-10 * z[3]
        x[5] += 1.8 * 1e-3 + 2.7 * 1e-4 * z[4]
        x[6] += 4.0 * 1e-3 + 3.2 * 1e-5 * z[5]
        x[7] += 4.0 * 1e-3 + 3.2 * 1e-5 * z[6]
    return x


_MODE_TEXT = {'attitude': 'attitude control with absolute commands', 'incremental': 'incremental control',
              'symmetric': 'symmetric control'}


def control_mode(state_dim=7, action_dim=3):
    """the control mode an actor of these widths flies: 'attitude' (7 -> 3), 'incremental' (10 -> 3) or 'symmetric' (2 -> 1)"""
    if (state_dim, action_dim) == (rollout.SYMMETRIC_STATE_DIM, rollout.SYMMETRIC_ACTION_DIM):
        return 'symmetric'
    return 'incremental' if state_dim == rollout.INCREMENTAL_STATE_DIM else 'attitude'


def env_control_mode(env):
    return 'symmetric' if env.symmetric else 'incremental' if env.incremental else 'attitude'


def full_name(condition):
    """the env name of a condition: a bare name ('nominal', 'be', ..., 'incremental') is the attitude configuration's"""
    return condition if '_' in condition else 'PHlab_attitude_' + condition


def condition_env(condition, t_max=T_MAX, shape=None):
    """the CitationEnv of a condition name ('nominal', 'low-q', ..., or a full env name 'PHlab_<configuration>_<mode>') in
    evaluation mode, for an actor of `shape` (None: the attitude 7 -> 3 actor).  The env's control mode must be the actor's:
    a bare name is an attitude env with absolute commands, 'incremental' (or any mode containing it) one with incremental
    commands, and 'PHlab_symmetric_<mode>' a symmetric one.  A mismatch raises ValueError naming both modes."""
    from .envs import config
    env = config.select_env(full_name(condition))
    mode = 'attitude' if shape is None else control_mode(shape.state_dim, shape.action_dim)
    have = env_control_mode(env)
    if have != mode:
        raise ValueError('evaluation: condition %r is an env of %s, but the actor flies %s' % (condition, _MODE_TEXT[have], _MODE_TEXT[mode]))
    env.set_eval_mode(t_max)
    return env


def _configuration(name):
    """the configuration token of a full env name ('attitude', 'symmetric'), or 'attitude' for a bare condition"""
    return name.split('_')[1].lower() if '_' in name else 'attitude'


def env_conditions(text):
    """the condition list of an -env argument: 'all', a condition, a full name 'PHlab_<configuration>_<mode>' or a comma
    list of them.  Attitude names become their bare mode ('PHlab_attitude_be' -> 'be'); other configurations keep their full name.
    'PHlab_<configuration>_all' is every condition of that configuration.  One list flies one configuration."""
    out, cfgs = [], set()
    for c in (c for c in text.split(',') if c):
        cfg = _configuration(c) if c.lower().startswith('phlab_') else 'attitude'
        cfgs.add(cfg)
        mode = c.split('_')[-1] if c.lower().startswith('phlab_') else c
        if mode == 'all':
            out += list(CONDITIONS) if cfg == 'attitude' else ['PHlab_%s_%s' % (c.split('_')[1], m) for m in CONDITIONS]
        else:
            out.append(mode if cfg == 'attitude' else c)
    if len(cfgs) > 1:
        raise ValueError('evaluation: one condition list flies one configuration, not %s' % ', '.join(sorted(cfgs)))
    return out


def condition_folder(cond):
    """the output folder of a condition under <run>/figures: the mode token, as base/evaluate.py names it"""
    return cond.split('_')[-1]


def env_dims(cond):
    """(state_dim, action_dim) of the env a condition names: env.observation_space / env.action_space, as base/evaluate.py
    sets them"""
    from .envs import config
    env = config.select_env(full_name(cond))
    return env.observation_space.shape[0], env.action_space.shape[0]


def symmetric_refs(num_trails, seed=7, t_max=T_MAX):
    """the theta references of symmetric control's evaluation episodes: the reference's env ignores user_refs and draws one
    RandomizedCosineStepSequence(t_max, ampl_max=30, block_width=t_max // 5, smooth_width=t_max // 6.7, n_levels=40,
    vary_timings=0) per episode (envs/phlabenv.py:303-313); here num_trails + 1 of them from refsig.make_ref_params(seed_base
    = seed, symmetric=True), as (theta, phi) pairs whose phi channel is zero and never read.  The kernels add the 0.22 deg
    trim themselves."""
    levels, starts = refsig.make_ref_params(num_trails + 1, seed_base=seed, t_max=t_max, symmetric=True)
    sw = refsig.widths(t_max, True)[1]
    return [(signals.SmoothedStepSequence(starts[i, 0], levels[i, 0], smooth_width=sw),
             signals.SmoothedStepSequence(starts[i, 1], levels[i, 1], smooth_width=sw)) for i in range(num_trails + 1)]


def gen_refs(t_max, amp_times, ampl_max, num_trails=10):
    """base/evaluation_utils.py:23-55: num_trails SmoothedStepSequence references on the global legacy np.random stream, per
    trial one choice of 6 levels on linspace(-ampl_max, ampl_max, 6) (the first forced to 0), then 5 uniform(-0.05, 0.05)
    jitters of the block times.  The jittered times replace the base times, so the jitter accumulates from trial to trial."""
    grid = np.linspace(-ampl_max, ampl_max, 6)
    times = list(amp_times)
    out = []
    for _ in range(num_trails):
        levels = np.random.choice(grid, size=6, replace=True)
        levels[0] = 0.0
        times = times[:1] + [t + np.random.uniform(-0.05, 0.05) for t in times[1:]]
        out.append(signals.SmoothedStepSequence(times, levels, smooth_width=t_max // 10))
    return out


def eval_refs(num_trails, t_max=T_MAX):
    """the reference list of base/evaluate.py:161-188: num_trails random (theta, phi) pairs from gen_refs (all theta draws
    first), then the fixed base reference as trial num_trails"""
    times = np.linspace(0., t_max, 6)
    theta = gen_refs(t_max, times, 12.0, num_trails=num_trails)
    phi = gen_refs(t_max, times, 10.0, num_trails=num_trails)
    theta.append(signals.SmoothedStepSequence(times, [0, 12, 3, -4, -8, 2], smooth_width=t_max // 10))
    phi.append(signals.SmoothedStepSequence(times, [2, -2, 2, 10, 2, -6], smooth_width=t_max // 10))
    return list(zip(theta, phi))


def nmae_from_track(track, steps, symmetric=False):
    """calc_nMAE (base/core/utils.py:39-58) of trajectories from their tracking-error sums: track [..., 4], steps [...].
    symmetric=True: the sums of symmetric control (sum |e_theta|, 0, 0, sum e_theta), whose (n, 1) error array calc_nMAE
    broadcasts: theta's mean error over [20 deg, 20 deg, max(|mean e_theta|, 3.14159 / 180)], the last range ("beta's") taken
    from theta's own signed mean"""
    track = np.asarray(track, dtype=np.float64)
    n = np.asarray(steps, dtype=np.float64)[..., None]
    mae = np.broadcast_to(track[..., 0:1] / n, track[..., :3].shape) if symmetric else track[..., :3] / n
    beta_range = np.maximum(np.abs(track[..., 3:4] / n), 3.14159 / 180)
    ranges = np.concatenate((np.broadcast_to(np.deg2rad(20), beta_range.shape), np.broadcast_to(np.deg2rad(20), beta_range.shape),
                             beta_range), axis=-1)
    return np.mean(mae / ranges, axis=-1) * 100


def _ref_arrays(refs):
    levels = np.stack([np.stack([th.levels, ph.levels]) for th, ph in refs])
    starts = np.stack([np.stack([th.starts, ph.starts]) for th, ph in refs])
    return levels, starts

class Flight:
    """what validate_agent's launch gives per trial, rebuilt as base/evaluate.py's loop records it: errors [k, c] (c = 3, or 1
    with symmetric control), deflections u_before [k, c], data (the traces of base/evaluate.py), and the launch's own
    tracking-error sums track [T, 4] (None for attitude control with absolute commands, whose launch has no d_track)"""
    __slots__ = ('errors', 'u_before', 'data', 'steps', 'returns', 'track')


def fly_traced(genome, shape, env, user_refs_lst, num_trails=1, device=None, widths=None):
    """validate_agent's one traced launch, with the per-trial records (Flight).  Incremental and symmetric control fly it
    as a tracking launch of the suite (track=True, suite=True): their tracking instantiations are the ones with the gust
    schedule."""
    dev = device or torch.device('cuda', torch.cuda.current_device())
    mode = control_mode(shape.state_dim, shape.action_dim)
    if env_control_mode(env) != mode:
        raise ValueError('validate_agent: the env flies %s, but the actor flies %s' % (_MODE_TEXT[env_control_mode(env)], _MODE_TEXT[mode]))
    sym, suite = mode == 'symmetric', mode != 'attitude'
    refs = user_refs_lst[:num_trails + 1]
    n = len(refs)
    horizon = int(round(env.t_max / env.dt)) + 1
    levels, starts = _ref_arrays(refs)
    smooth_w = float(refs[0][0].smooth_width)
    g = torch.as_tensor(np.asarray(genome, dtype=np.float32) if not torch.is_tensor(genome) else genome, device=dev).reshape(1, -1).contiguous()
    md = torch.full((n,), env.mode_code, dtype=torch.int32, device=dev)
    noise = z = None
    if getattr(env, 'sensor_noise', False):
        z = sensor_noise_draws(n, horizon)
        noise = torch.as_tensor(z.reshape(1, n, horizon + 1, 7), device=dev)
    r = rollout.population_rollout(g, shape, torch.as_tensor(levels, device=dev), torch.as_tensor(starts, device=dev), md,
                                   horizon=horizon, trace=True, t_max=float(env.t_max), smooth_width=smooth_w, sensor_noise=noise,
                                   gust=rollout.mode_gust(env.mode_code), widths=widths, track=suite, suite=suite)
    torch.cuda.synchronize()
    r.check()
    steps = r.steps[0].cpu().numpy()
    trace = r.trace[0].cpu().numpy()
    x_ic = rollout.initial_state(rollout.mode_variant(env.mode_code))
    f = Flight()
    f.errors, f.u_before, f.data = [], [], None
    f.steps, f.returns = steps, r.returns[0].cpu().numpy()
    f.track = r.track[0].cpu().numpy() if suite else None
    for i in range(n):
        errors, u_before, f.data = rebuild_trial(trace[i, :int(steps[i])], reset_state(x_ic, None if z is None else z[i, 0]), sym)
        f.errors.append(errors)
        f.u_before.append(u_before)
    return f


def rebuild_trial(tr, x0, symmetric=False):
    """what base/evaluate.py's loop records for one episode, from its trace rows tr [k, TRACE_COLS] and env.x after reset()
    x0 [12]: errors [k, c] (ref(t) - env.get_controlled_state() when the loop body starts), the deflections env.last_u then
    [k, c], and data = ref c | u c | x 12 | reward (c = 3, or 1 with symmetric control: theta, the elevator)"""
    ctrl = [7] if symmetric else [7, 6, 5]       # env.get_controlled_state(): theta, or theta, phi, beta
    x_after = tr[:, rollout.TRACE_X]                             # env.x after each step() = state before that plant step
    ref_values = tr[:, rollout.TRACE_ERR][:, :len(ctrl)] + x_after[:, ctrl]      # ref(t_k) [rad] = error_k + controlled state
    x_before = np.vstack((np.asarray(x0)[None], x_after[:-1]))   # env.x when the loop body starts (evaluate.py:73)
    u_before = np.vstack((np.zeros((1, len(ctrl))), tr[:-1, rollout.TRACE_U][:, :len(ctrl)]))
    data = np.concatenate((ref_values, u_before, x_before, tr[:, rollout.TRACE_R, None]), axis=1)
    return ref_values - x_before[:, ctrl], u_before, data


def validate_agent(genome, shape, env, user_refs_lst, num_trails=1, device=None, widths=None):
    """genome: [P] fp32 tensor / array of one actor; env: serl_b200.envs CitationEnv (mode, eval t_max) of the actor's control
    mode (condition_env(..., shape=shape)); user_refs_lst: list of (theta_ref, phi_ref) serl_b200.signals.SmoothedStepSequence
    (symmetric control: symmetric_refs); trials 0..num_trails are flown (base/evaluate.py:127).  widths: a width-list actor on
    K1-TC, as in rollout.population_rollout.  Returns the traces of the last trial (ref | u | x 12 | reward: 19 columns, 15
    with symmetric control's ref_theta | de) and Stats."""
    f = fly_traced(genome, shape, env, user_refs_lst, num_trails, device, widths)
    nmaes = [calc_nMAE(e) for e in f.errors]
    sms = [calc_smoothness(u, plot_spectra=False) for u in f.u_before]
    return f.data, Stats(float(np.average(nmaes)), float(np.std(nmaes)), float(np.average(sms)), float(np.std(sms)))


class PopulationEval:
    """what evaluate_population returns: per actor and condition, the trial mean and sd of nMAE and smoothness as
    validate_agent computes them (arrays [N, C]), and the per-trial values [N, C, num_trails + 1]"""

    def __init__(self, conditions, nmae_trials, sm_trials):
        self.conditions = tuple(conditions)
        self.nmae_trials, self.sm_trials = nmae_trials, sm_trials
        self.nmae, self.nmae_sd = np.average(nmae_trials, axis=-1), np.std(nmae_trials, axis=-1)
        self.sm, self.sm_sd = np.average(sm_trials, axis=-1), np.std(sm_trials, axis=-1)

    def _c(self, condition):
        return self.conditions.index(condition)

    def stats(self, actor, condition):
        c = self._c(condition)
        return Stats(float(self.nmae[actor, c]), float(self.nmae_sd[actor, c]), float(self.sm[actor, c]), float(self.sm_sd[actor, c]))

    def champion(self, condition):
        """the actor of lowest nMAE (the first of equals, as base/evaluate.py's strict `<` scan)"""
        return int(np.argmin(self.nmae[:, self._c(condition)]))

    def average(self, condition):
        """the population summary of base/evaluate.py -eval_pop: mean and sd over the actors of their nMAE and smoothness"""
        c = self._c(condition)
        return Stats(float(np.average(self.nmae[:, c])), float(np.std(self.nmae[:, c])), float(np.average(self.sm[:, c])),
                     float(np.std(self.sm[:, c])))

    def split(self, sizes):
        """one PopulationEval per consecutive block of `sizes` actors"""
        edges = np.cumsum([0] + list(sizes))
        return [PopulationEval(self.conditions, self.nmae_trials[a:b], self.sm_trials[a:b]) for a, b in zip(edges[:-1], edges[1:])]


def evaluate_population(genomes, shape, conditions, user_refs_lst, num_trails=1, widths=None, device=None, actions_cap=ACTIONS_CAP,
                        noise_state=None):
    """validate_agent for every actor of `genomes` [N, P] (fp32, parameters() order) on every condition, without traces: one
    rollout launch per sensor-noise group (conditions with and without the shim; the shim's draws are made for the noisy
    conditions only) and one K6 launch.  `shape` / `widths` as in rollout.population_rollout.  The sensor-noise draws are
    taken condition by condition, actor by actor, trial by trial: the order of validate_agent called in that order, on one
    continued np.random stream; with `noise_state` (an np.random.get_state()) every noisy condition's draws start from that
    state instead, as when base/evaluate.py runs once per condition and reseeds (examples/evaluate.py).  When
    the [N, envs, horizon, 3] fp32 deflection record exceeds `actions_cap` bytes, the actors are flown in chunks of equal
    launches (same results).  Incremental (10 -> 3) and symmetric (2 -> 1) actors fly the conditions of their own control
    mode (condition_env(..., shape)) in tracking launches of the suite (suite=True); symmetric control's references come
    from symmetric_refs.  The recorded deflection is [de, 0, 0] with symmetric control: K6 of it is the one-column
    calc_smoothness."""
    envs = [condition_env(c, shape=shape) for c in conditions]      # the conditions of the actor's control mode
    mode = control_mode(shape.state_dim, shape.action_dim)
    sym, suite = mode == 'symmetric', mode != 'attitude'
    dev = device or torch.device('cuda', torch.cuda.current_device())
    refs = user_refs_lst[:num_trails + 1]
    T, C = len(refs), len(conditions)
    smooth_w = float(refs[0][0].smooth_width)
    if any(float(r.smooth_width) != smooth_w for pair in refs for r in pair):
        raise ValueError('evaluate_population: every reference of one launch needs the same smooth_width')
    g = torch.as_tensor(np.asarray(genomes, dtype=np.float32) if not torch.is_tensor(genomes) else genomes, device=dev)
    g = g.reshape(g.shape[0], -1).contiguous()
    N = g.shape[0]
    t_max = float(envs[0].t_max)
    horizon = int(round(t_max / envs[0].dt)) + 1
    lv1, st1 = _ref_arrays(refs)
    groups = [idx for idx in ([i for i, e in enumerate(envs) if not e.sensor_noise], [i for i, e in enumerate(envs) if e.sensor_noise]) if idx]
    noisy = [i for i, e in enumerate(envs) if e.sensor_noise]
    z = None
    if noisy:
        draws = []
        for _ in noisy:
            if noise_state is not None:
                np.random.set_state(noise_state)
            draws.append(sensor_noise_draws(N * T, horizon).reshape(N, T, horizon + 1, 7))
        z = np.stack(draws)
    per_actor = C * T * horizon * 3 * 4
    chunk = max(1, min(N, actions_cap // per_actor))
    nmae = np.empty((N, C, T))
    sm = np.empty((N, C, T))
    for lo in range(0, N, chunk):
        hi = min(N, lo + chunk)
        n = hi - lo
        flat = torch.empty((n * C * T, horizon, 3), dtype=torch.float32, device=dev)
        runs, row = [], 0
        for idx in groups:
            ne = len(idx) * T
            codes = np.repeat([envs[i].mode_code for i in idx], T)
            md = torch.tensor(codes, dtype=torch.int32, device=dev)
            out = rollout.RolloutResult()
            out.returns = torch.empty((n, ne), dtype=torch.float64, device=dev)
            out.steps = torch.empty((n, ne), dtype=torch.int32, device=dev)
            out.track = torch.empty((n, ne, rollout.TRACK_COLS), dtype=torch.float64, device=dev)
            out.actions = flat[row:row + n * ne].view(n, ne, horizon, 3)
            out.status = torch.zeros((1,), dtype=torch.int32, device=dev)
            out.fitness = out.trace = out.replay = out.smoothness = None
            noise = None
            if envs[idx[0]].sensor_noise:
                zz = z[[noisy.index(i) for i in idx], lo:hi].transpose(1, 0, 2, 3, 4).reshape(n, ne, horizon + 1, 7)
                noise = torch.as_tensor(np.ascontiguousarray(zz), device=dev)
            rollout.population_rollout(g[lo:hi], shape, torch.as_tensor(np.tile(lv1, (len(idx), 1, 1)), device=dev),
                                       torch.as_tensor(np.tile(st1, (len(idx), 1, 1)), device=dev), md, horizon=horizon, out=out,
                                       t_max=t_max, smooth_width=smooth_w, env_order=rollout.variant_sorted_order(md), fitness=False,
                                       widths=widths, sensor_noise=noise, gust=any(rollout.mode_gust(int(c)) for c in codes),
                                       suite=suite)
            runs.append((idx, out))
            row += n * ne
        steps = torch.cat([out.steps.reshape(-1) for _, out in runs])
        # validate_agent's u_lst is the deflection BEFORE each step, from zeros: [0, u_0, ..., u_{k-2}], a circular shift of
        # [u_0, ..., u_{k-2}, 0], whose spectrum has the same magnitudes.  So the recorded deflection of the last step is zeroed.
        flat[torch.arange(flat.shape[0], device=dev), steps.long() - 1] = 0.0
        smooth = rollout.smoothness(flat, steps).cpu().numpy()
        row = 0
        for idx, out in runs:
            out.check()
            ne = len(idx) * T
            nm = nmae_from_track(out.track.cpu().numpy(), out.steps.cpu().numpy(), symmetric=sym)
            nmae[lo:hi, idx] = nm.reshape(n, len(idx), T)
            sm[lo:hi, idx] = smooth[row:row + n * ne].reshape(n, len(idx), T)
            row += n * ne
    return PopulationEval(conditions, nmae, sm)


def _genome(state_dict, args):
    from .core.genetic_agent import Actor
    actor = Actor(args)
    actor.load_state_dict(state_dict)
    return actor.flat().detach().cpu().numpy().astype(np.float32)


def load_pop(run_dir, args):
    """base/evaluation_utils.py load_pop: <run_dir>/files/evo_nets.pkl ({'actor_i': state_dict}, as Agent.save_agent writes it)
    -> [N, P] fp32 genomes in parameters() order, actor i in row i.  `args` gives the actor shape (Parameters updated from
    load_config(run_dir))."""
    ck = torch.load(os.path.join(run_dir, 'files', 'evo_nets.pkl'), map_location='cpu')
    return np.stack([_genome(sd, args) for sd in ck.values()])


def load_rl_agent(run_dir, args):
    """base/evaluation_utils.py load_rl_agent: <run_dir>/files/rl_net.pkl (a state_dict) -> [1, P] fp32 genome"""
    return _genome(torch.load(os.path.join(run_dir, 'files', 'rl_net.pkl'), map_location='cpu'), args)[None]


def run_config(run_dir, args):
    """args (Parameters) updated from <run_dir>/files/config.yaml, as base/evaluate.py does before loading actors"""
    args.update_from_dict(load_config(run_dir))
    return args


def write_final_performance(run_dir, condition, sm_lst, nmae_lst):
    """<run_dir>/figures/<condition>/final_performance.csv: one 'sm,nmae' line per actor (base/evaluate.py -save_stats)"""
    path = os.path.join(run_dir, 'figures', condition)
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, 'final_performance.csv'), 'w', encoding='utf-8') as f:
        for s, m in zip(sm_lst, nmae_lst):
            f.write(f'{float(s)!r},{float(m)!r}\n')


def _toml_key(condition):
    return condition if all(ch.isalnum() or ch in '-_' for ch in condition) else '"%s"' % condition


def _toml_table(stats):
    return ''.join(f'{k} = {float(v)!r}\n' for k, v in stats._asdict().items())


def append_rl_stats_toml(run_dir, condition, stats):
    """append one condition's table of base/evaluate.py -eval_rl -save_stats to <run_dir>/stats.toml: two blank lines, then
    [<c>] with nmae, nmae_sd, sm, sm_sd (the layout of a TD3 run's stats.toml)"""
    with open(os.path.join(run_dir, 'stats.toml'), 'a', encoding='utf-8') as f:
        f.write(f'\n\n[{_toml_key(condition)}]\n{_toml_table(stats)}')


def write_trajectory(run_dir, condition, data):
    """<run_dir>/figures/<condition>/nominal_trajectory.csv: the time traces of the last trial (ref 3 | u 3 | x 12 | reward),
    whitespace-separated as base/evaluate.py -save_trajectory writes them"""
    path = os.path.join(run_dir, 'figures', condition)
    os.makedirs(path, exist_ok=True)
    np.savetxt(os.path.join(path, 'nominal_trajectory.csv'), data)


def append_stats_toml(run_dir, condition, champion_idx, champion, average):
    """append one condition's table to <run_dir>/stats.toml in the layout base/evaluate.py's toml.dump writes:
    [<c>] champion_idx, [<c>.champion] and [<c>.average] with nmae, nmae_sd, sm, sm_sd, then two blank lines"""
    key, table = _toml_key(condition), _toml_table
    text = f'[{key}]\nchampion_idx = {int(champion_idx)}\n\n[{key}.champion]\n{table(champion)}\n[{key}.average]\n{table(average)}\n\n'
    with open(os.path.join(run_dir, 'stats.toml'), 'a', encoding='utf-8') as f:
        f.write(text)
