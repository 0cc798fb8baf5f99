"""Evaluation of a trained actor on user-defined references — the device version of base/evaluate.py:59-150
(`evaluate` + `validate_agent`): every trial of a validation run is one trajectory of ONE traced rollout launch, in
evaluation mode (t_max = 80 s, envs/phlabenv.py:295-301), on any plant variant / fault shim including the sensor-noise
shim (envs/noise/citation.py:72-82).  Returns what the reference returns: the time traces of the last trial and
Stats(nmae, nmae_sd, sm, sm_sd)."""
from collections import namedtuple

import numpy as np
import torch

from . import refsig, rollout
from .core.utils import calc_nMAE, calc_smoothness

Stats = namedtuple('Stats', ('nmae', 'nmae_sd', 'sm', 'sm_sd'))


def sensor_noise_draws(n_traj, horizon):
    """standard-normal draws of the sensor-noise shim in ITS order (randn(3), randn(1), randn(1), randn(2) per native call),
    one episode after the other: [n_traj, horizon + 1, 7] float32."""
    z = np.empty((n_traj, horizon + 1, 7), dtype=np.float32)
    for i in range(n_traj):
        for c in range(horizon + 1):
            z[i, c, 0:3] = np.random.randn(3)
            z[i, c, 3] = np.random.randn(1)[0]
            z[i, c, 4] = np.random.randn(1)[0]
            z[i, c, 5:7] = np.random.randn(2)
    return z


def validate_agent(genome, shape, env, user_refs_lst, num_trails=1, device=None):
    """genome: [P] fp32 tensor / array of one actor; env: serl_b200.envs CitationEnv (mode, eval t_max); user_refs_lst: list of
    (theta_ref, phi_ref) serl_b200.signals.SmoothedStepSequence; trials 0..num_trails are flown (base/evaluate.py:127)."""
    dev = device or torch.device('cuda', torch.cuda.current_device())
    refs = user_refs_lst[:num_trails + 1]
    n = len(refs)
    horizon = int(round(env.t_max / env.dt)) + 1
    levels = np.stack([np.stack([th.levels, ph.levels]) for th, ph in refs])
    starts = np.stack([np.stack([th.starts, ph.starts]) for th, ph in refs])
    smooth_w = float(refs[0][0].smooth_width)
    g = torch.as_tensor(np.asarray(genome, dtype=np.float32) if not torch.is_tensor(genome) else genome, device=dev).reshape(1, -1).contiguous()
    md = torch.full((n,), env.mode_code, dtype=torch.int32, device=dev)
    noise = None
    if getattr(env, 'sensor_noise', False):
        noise = torch.as_tensor(sensor_noise_draws(n, horizon).reshape(1, n, horizon + 1, 7), device=dev)
    r = rollout.population_rollout(g, shape, torch.as_tensor(levels, device=dev), torch.as_tensor(starts, device=dev), md,
                                   horizon=horizon, trace=True, t_max=float(env.t_max), smooth_width=smooth_w, sensor_noise=noise,
                                   gust=rollout.mode_gust(env.mode_code))
    torch.cuda.synchronize()
    r.check()
    steps = r.steps[0].cpu().numpy()
    trace = r.trace[0].cpu().numpy()
    x_ic = rollout.initial_state(rollout.mode_variant(env.mode_code))
    nmaes, sms, data = [], [], None
    for i in range(n):
        k = int(steps[i])
        tr = trace[i, :k]
        x_after = tr[:, rollout.TRACE_X]                        # env.x after each step() = state before that plant step
        ref_values = tr[:, rollout.TRACE_ERR] + x_after[:, [7, 6, 5]]      # ref(t_k) [rad] = error_k + controlled state
        x_before = np.vstack((x_ic[None], x_after[:-1]))        # env.x when the loop body starts (evaluate.py:73)
        u_before = np.vstack((np.zeros((1, 3)), tr[:-1, rollout.TRACE_U]))
        errors = ref_values - x_before[:, [7, 6, 5]]
        nmaes.append(calc_nMAE(errors))
        sms.append(calc_smoothness(u_before, plot_spectra=False))
        data = np.concatenate((ref_values, u_before, x_before, tr[:, rollout.TRACE_R, None]), axis=1)
    return data, Stats(float(np.average(nmaes)), float(np.std(nmaes)), float(np.average(sms)), float(np.std(sms)))
