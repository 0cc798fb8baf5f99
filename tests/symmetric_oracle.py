"""Oracle of symmetric control (checker only): the reference's PHlab_symmetric_<mode> (envs/phlabenv.py:84-90, 226-231,
304-313, 362-367, 373-379) restated on top of oracle/phlab.py, with the actor of the device kernel's summation order
(oracle/plant/actor_kernel_order.c, which takes any state and action width) at 2 inputs and 1 output.

What symmetric control changes against the attitude mode:
  * one action, the elevator, scaled to +-10 deg; the plant and the fault shim take [de, 0, 0] (pad_action);
  * the error is theta's alone, against a reference offset by the constant trim 0.22 deg (never rad2deg(theta0));
  * reward = -|clip(6/pi e_theta, -1, 1)| / 1; termination and penalty unchanged (they still test phi);
  * obs = [e_theta, q]; reset() gives [0, q].
"""
import ctypes

import numpy as np

from oracle import build as _build, phlab, refsig

ACT = {'tanh': 0, 'elu': 1, 'relu': 2}
THETA_TRIM = 0.22


class SymmetricCitationEnv(phlab.CitationEnv):
    """oracle.phlab.CitationEnv flying symmetric control"""

    def __init__(self, mode='nominal', backend='auto', plant=None, t_max=20):
        super().__init__(mode, backend, plant, t_max)
        self.smooth_w = float(t_max // 6.7)          # smooth_width = t_max // 6.7 (:308)
        self.low = -self.bound * np.ones(1)
        self.high = self.bound * np.ones(1)

    def reset(self, levels=None, starts=None):
        super().reset(levels, starts)
        self.theta_trim = THETA_TRIM
        self.last_u = np.zeros(1)
        self.error = np.zeros(1)
        self.obs = np.hstack((self.error, self.x[[1]]))
        return self.obs

    def step(self, action):
        u = self.scale_action(np.asarray(action).reshape(1))
        self.x = self._native_step(np.pad(u, (0, 2)))          # pad_action: [de, 0, 0, ...]
        ref = np.deg2rad(refsig.ref_value_deg(self.levels[0], self.starts[0], self.t, self.theta_trim, self.smooth_w, self.t_max))
        self.error = np.asarray([ref]) - np.asarray([self.x[7]])
        reward_vec = np.abs(np.clip(6 / np.pi * np.array([1.]) * self.error, -np.ones(1), np.ones(1)))
        reward = -reward_vec.sum() / 1
        self.obs = np.hstack((self.error, self.x[[1]]))
        self.last_u = u
        done, penalty = False, 0.
        if self.t >= self.t_max or np.abs(self.x[7]) > self.max_theta or np.abs(self.x[6]) > self.max_phi or self.x[9] < 50:
            penalty = -1 / self.dt * (self.t_max - self.t) * 2
            done = True
        reward += penalty
        self.t += self.dt
        return self.obs, reward, done, {'x': self.x, 't': self.t}


class KernelOrderActor:
    """Actor.select_action in the device kernel's summation order (bit-exact with serl_actor_forward / K1), 2 -> 1"""

    def __init__(self, genome, hidden, num_layers=3, activation='tanh', state_dim=2, action_dim=1):
        self.lib = ctypes.CDLL(_build.build())
        self.g = np.ascontiguousarray(genome, dtype=np.float32)
        self.args = (state_dim, action_dim, int(hidden), int(num_layers), ACT[activation])

    def forward(self, obs):
        """obs [n, S] -> actions [n, A] float32"""
        o = np.ascontiguousarray(obs, dtype=np.float32).reshape(-1, self.args[0])
        out = np.empty((o.shape[0], self.args[1]), dtype=np.float32)
        vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        self.lib.ko_actor_forward_batch(vp(self.g), *self.args, vp(o), o.shape[0], vp(out))
        return out

    def select_action(self, obs):
        return self.forward(obs)[0]


def run_episode(env, actor, levels, starts, horizon=2001, noise=None, actions=None):
    """base/core/agent.py:63-138 with symmetric control: returns dict(ret, steps, rows [steps, 8] float32 (the transitions
    obs | action | next_obs | reward | done | cost), u [steps] (the elevator command)).  noise [horizon, 1]: the clipped
    exploration noise added to the actor's output and clipped to [-1, 1] in float64; actions [horizon, 1]: given float32
    actions instead of the actor's (open loop)."""
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
        rows.append(np.hstack((prev, np.asarray(a_env, dtype=np.float32).reshape(1), obs.astype(np.float32),
                               np.float32(reward), np.float32(done), np.float32(cost))).astype(np.float32))
        us.append(float(env.last_u[0]))
        if done:
            break
    return {'ret': ret, 'steps': len(rows), 'rows': np.asarray(rows, dtype=np.float32), 'u': np.asarray(us)}


def evaluate_population(genomes, hidden, levels, starts, modes, num_layers=3, activation='tanh', horizon=2001, noise=None,
                        backend='port'):
    """every genome [pop, P] on every env (levels / starts [n_envs, 2, 6], modes [n_envs]; noise optional
    [pop, n_envs, horizon, 1]) -> (returns [pop, n_envs], steps [pop, n_envs], episodes [pop][n_envs] of run_episode)"""
    pop, n_envs = len(genomes), len(levels)
    ret, stp = np.zeros((pop, n_envs)), np.zeros((pop, n_envs), dtype=np.int32)
    eps = []
    envs = {m: SymmetricCitationEnv(m, backend) for m in set(modes)}
    for a in range(pop):
        actor = KernelOrderActor(genomes[a], hidden, num_layers, activation)
        eps.append([])
        for e in range(n_envs):
            r = run_episode(envs[modes[e]], actor, levels[e], starts[e], horizon, None if noise is None else noise[a, e])
            ret[a, e], stp[a, e] = r['ret'], r['steps']
            eps[-1].append(r)
    return ret, stp, eps
