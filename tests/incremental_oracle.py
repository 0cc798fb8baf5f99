"""Oracle of incremental control (checker only): the reference's PHlab_attitude_incremental (envs/phlabenv.py:174-220, 377-380,
425-426, 443-466) restated on top of oracle/phlab.py, with the actor of the device kernel's summation order
(oracle/plant/actor_kernel_order.c, which takes any state width) at 10 inputs.

What incremental control changes against the absolute mode:
  * the nominal plant, no fault shim, no gust, no sensor noise;
  * the scaled action is a rate, bound 25 deg/s instead of 10 deg;
  * u = last_u + rate * dt in float64 (no clip), then the plant step, then last_u = u;
  * obs = [error 3, p q r alpha, last_u 3]; reset() appends last_u = 0.
"""
import ctypes

import numpy as np

from oracle import build as _build, phlab

ACT = {'tanh': 0, 'elu': 1, 'relu': 2}


class IncrementalCitationEnv(phlab.CitationEnv):
    """oracle.phlab.CitationEnv flying incremental control: scale_action returns the integrated deflection, so step() feeds
    the plant u = last_u + rate * dt and stores it as last_u, as the reference's step does."""

    def __init__(self, backend='auto', plant=None, t_max=20):
        super().__init__('nominal', backend, plant, t_max)
        self.bound = np.deg2rad(25)
        self.low = -self.bound * np.ones(3)
        self.high = self.bound * np.ones(3)

    def scale_action(self, a):
        return self.last_u + super().scale_action(a) * self.dt

    def reset(self, levels=None, starts=None):
        self.obs = np.hstack((super().reset(levels, starts), self.last_u))
        return self.obs

    def step(self, action):
        obs, reward, done, info = super().step(action)
        self.obs = np.hstack((obs, self.last_u))
        return self.obs, reward, done, info


class KernelOrderActor:
    """Actor.select_action in the device kernel's summation order (bit-exact with serl_actor_forward / K1) at any state width"""

    def __init__(self, genome, hidden, num_layers=3, activation='tanh', state_dim=10):
        self.lib = ctypes.CDLL(_build.build())
        self.g = np.ascontiguousarray(genome, dtype=np.float32)
        self.args = (state_dim, 3, int(hidden), int(num_layers), ACT[activation])

    def forward(self, obs):
        """obs [n, S] -> actions [n, 3] float32"""
        o = np.ascontiguousarray(obs, dtype=np.float32).reshape(-1, self.args[0])
        out = np.empty((o.shape[0], 3), dtype=np.float32)
        vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        self.lib.ko_actor_forward_batch(vp(self.g), *self.args, vp(o), o.shape[0], vp(out))
        return out

    def select_action(self, obs):
        return self.forward(obs)[0]


def run_episode(env, actor, levels, starts, horizon=2001, noise=None, actions=None):
    """base/core/agent.py:63-138 with incremental control: returns dict(ret, steps, rows [steps, 26] float32 (the transitions
    obs | action | next_obs | reward | done | cost), u [steps, 3] (env.last_u per step)).  noise [horizon, 3]: the clipped
    exploration noise added to the actor's output and clipped to [-1, 1] in float64 (agent.py:90-93); actions [horizon, 3]:
    given float32 actions instead of the actor's (open loop)."""
    obs = env.reset(levels, starts)
    ret, rows, us = 0.0, [], []
    for k in range(horizon):
        a = actions[k] if actions is not None else actor.select_action(obs)
        a_env = np.clip(a.astype(np.float64) + noise[k], -1.0, 1.0) if noise is not None else a
        prev = obs.astype(np.float32)
        obs, reward, done, info = env.step(a_env)
        cost = 1.0 if (np.rad2deg(np.abs(env.x[4])) > 11.0 or np.rad2deg(np.abs(env.x[6])) > 0.75 * env.max_phi
                       or env.x[3] < env.V0 / 3) else 0.0
        ret += reward
        rows.append(np.hstack((prev, np.asarray(a_env, dtype=np.float32), obs.astype(np.float32),
                               np.float32(reward), np.float32(done), np.float32(cost))).astype(np.float32))
        us.append(env.last_u.copy())
        if done:
            break
    return {'ret': ret, 'steps': len(rows), 'rows': np.asarray(rows, dtype=np.float32), 'u': np.asarray(us)}


def evaluate_population(genomes, hidden, levels, starts, num_layers=3, activation='tanh', horizon=2001, noise=None, backend='port'):
    """every genome [pop, P] on every env (levels / starts [n_envs, 2, 6]; noise optional [pop, n_envs, horizon, 3]) ->
    (returns [pop, n_envs], steps [pop, n_envs], episodes [pop][n_envs] of run_episode)"""
    pop, n_envs = len(genomes), len(levels)
    ret, stp = np.zeros((pop, n_envs)), np.zeros((pop, n_envs), dtype=np.int32)
    eps = []
    env = IncrementalCitationEnv(backend)
    for a in range(pop):
        actor = KernelOrderActor(genomes[a], hidden, num_layers, activation)
        eps.append([])
        for e in range(n_envs):
            r = run_episode(env, actor, levels[e], starts[e], horizon, None if noise is None else noise[a, e])
            ret[a, e], stp[a, e] = r['ret'], r['steps']
            eps[-1].append(r)
    return ret, stp, eps
