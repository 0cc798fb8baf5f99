"""Mirror of envs/phlabenv.py CitationEnv (:76-486), gym-free, with the native plant on the GPU.

The object keeps the reference's per-step API (reset / step / finish, .x .last_u .t .ref .error) so single episodes can be
driven from Python — each step is one batched-plant kernel call (serl_plant_step, n = 1) with the wrapper arithmetic in
float64 numpy exactly as the reference writes it.  The population hot path does NOT go through this class step by step:
Agent.train hands the env's mode and freshly drawn reference-signal parameters to the fused rollout kernel.

Reference signals: `signals.RandomizedCosineStepSequence` (third-party, absent) is replaced by serl_b200/refsig.py's
generator, drawing from the global np.random stream at reset() like the reference's init_ref (:303-345).
"""
import numpy as np
import torch

from .. import _native, refsig, rollout


class Box:
    """the two attributes of gym.spaces.Box the reference reads (shape, low/high)."""

    def __init__(self, low, high):
        self.low, self.high = np.asarray(low, dtype=np.float64), np.asarray(high, dtype=np.float64)
        self.shape = self.low.shape


class _RefSignal:
    def __init__(self, levels, starts, offset, smooth_w=refsig.SMOOTH_W, t_end=None):
        self.levels, self.starts, self.offset, self.smooth_w, self.t_end = levels, starts, offset, smooth_w, t_end

    def __call__(self, t):
        return refsig.ref_value_deg(self.levels, self.starts, t, self.offset, self.smooth_w, self.t_end)


class CitationEnv:
    n_actions_full: int = 10
    n_obs_full: int = 12
    t: float = 0.
    dt = 0.01

    def __init__(self, configuration: str = None, mode: str = 'nominal'):
        configuration = configuration or 'attitude'
        if 'attitude' not in configuration.lower():
            raise ValueError("the B200 rollout engine implements the 'attitude' configuration (3 actions, obs = 3 errors + p,q,r,alpha)")
        self.n_actions = 3
        self.obs_idx = [0, 1, 2, 4]
        m = mode.lower()
        if m == '' or m == 'nominal' or 'h2000-v90' in m:
            m = 'nominal'
        alias = {'high-q': 'h2000-v150', 'low-q': 'h10000-v90', 'cg-aft': 'cg', 'cg-shift': 'cg-timed'}
        m = alias.get(m, m)
        # 'noise' (envs/phlabenv.py:139-142): the nominal plant behind the sensor-noise shim (envs/noise/citation.py:72-82)
        # 'gust' (:165-169): the gust build (nominal dynamics + a vertical gust for 20 s <= t <= 23 s) behind the same shim
        self.sensor_noise = m in ('noise', 'gust')
        if m == 'noise':
            m = 'nominal'
        if 'test' in m:           # phlabenv.py:171-174: any mode containing 'test' selects envs/test (the upward-gust build)
            m = 'test'
        if m not in rollout.MODES:
            raise ValueError('Unknown trim condition or control mode!')
        self.mode = m
        self.mode_code = rollout.mode_code(m)
        self.variant, self.fault = rollout.MODES[m]
        self.eval_mode = False
        self.t_max = 20
        self.x = self.obs = self.last_obs = self.V0 = self.last_u = None
        self.ref = self.ref_values = None
        self.theta_trim = 0.22
        self.bound = np.deg2rad(10)
        self.max_theta = np.deg2rad(60.)
        self.max_phi = np.deg2rad(75.)
        self.n_obs = len(self.obs_idx) + self.n_actions
        self.error = np.zeros((self.n_actions))
        self.error_scaler = (6 / np.pi * np.array([1., 1., 4.]))[:self.n_actions]
        self.max_bound = np.ones(self.error.shape)
        self.levels = self.starts = None
        self._X = None

    # ---- spaces (phlabenv.py:233-249) ----
    @property
    def action_space(self):
        return Box(-self.bound * np.ones(self.n_actions), self.bound * np.ones(self.n_actions))

    @property
    def observation_space(self):
        return Box(-30 * np.ones(self.n_obs), 30 * np.ones(self.n_obs))

    def seed(self, seed=None):
        return [seed]

    @property
    def theta(self):
        return self.x[7]

    @property
    def phi(self):
        return self.x[6]

    @property
    def beta(self):
        return self.x[5]

    @property
    def alpha(self):
        return self.x[4]

    @property
    def V(self):
        return self.x[3]

    @property
    def H(self):
        return self.x[9]

    def scale_action(self, clipped_action):
        low, high = self.action_space.low, self.action_space.high
        return low + 0.5 * (clipped_action + 1.0) * (high - low)

    # ---- reference signals ----
    def set_eval_mode(self, t_max: int = 80) -> None:
        """envs/phlabenv.py:295-301: longer evaluation episodes (reference widths scale with t_max, :321-335)."""
        self.t_max = int(t_max)
        self.eval_mode = True

    def draw_reference(self):
        """consume the global np.random stream like init_ref (:303-345) and return (levels[2,6], starts[2,6])."""
        levels = np.zeros((2, refsig.N_BLOCKS))
        starts = np.zeros((2, refsig.N_BLOCKS))
        for c in range(2):
            grid = np.linspace(-refsig.AMPL[c], refsig.AMPL[c], refsig.N_LEVELS)
            lv = grid[np.random.randint(0, refsig.N_LEVELS, size=refsig.N_BLOCKS)]
            lv[0] = 0.0
            block_w, _, jitter = refsig.widths(self.t_max)
            st = block_w * np.arange(refsig.N_BLOCKS) + np.random.uniform(-jitter, jitter, size=refsig.N_BLOCKS)
            st[0] = 0.0
            levels[c], starts[c] = lv, st
        return levels, starts

    def init_ref(self, **kwargs):
        self.theta_trim = np.rad2deg(self.x[7])
        sw = refsig.widths(self.t_max)[1]
        self.user_smooth_width = None
        if 'user_refs' in kwargs:
            # envs/phlabenv.py:336-341: evaluation references built by the caller (base/evaluate.py:169-180:
            # signals.SmoothedStepSequence(times, amplitudes, smooth_width=t_max//10)); ours carry their block parameters
            th, ph = kwargs['user_refs']['theta_ref'], kwargs['user_refs']['phi_ref']
            self.levels, self.starts = np.stack([th.levels, ph.levels]), np.stack([th.starts, ph.starts])
            sw = self.user_smooth_width = float(th.smooth_width)
        else:
            self.levels, self.starts = self.draw_reference()
        self.ref = [_RefSignal(self.levels[0], self.starts[0], self.theta_trim, sw, self.t_max),
                    _RefSignal(self.levels[1], self.starts[1], 0.0, sw), lambda t: 0.0]

    # ---- native plant on the device ----
    def _native_step(self, u):
        cmd = np.pad(u, (0, self.n_actions_full - self.n_actions), 'constant', constant_values=(0.))
        if self.fault == 'be':
            cmd[0] *= 0.3
        elif self.fault == 'jr':
            cmd[2] = 15 * 3.14159 / 180
        elif self.fault == 'sa':
            b = np.deg2rad(1); cmd[1] = np.clip(cmd[1], -b, b)
        elif self.fault == 'se':
            b = np.deg2rad(2.5); cmd[0] = np.clip(cmd[0], -b, b)
        x = self._X.cpu().numpy()[0, :12].copy()
        if self.sensor_noise:                 # envs/noise/citation.py:72-82, same draw order
            x[:3] += 3.0 * 10**(-5) + 6.3 * 10**(-4) * np.random.randn(3)
            x[4] += 4.0 * 10**(-10) * np.random.randn(1)[0]
            x[5] += 1.8 * 10**(-3) + 2.7 * 10**(-4) * np.random.randn(1)[0]
            x[6:8] += 4.0 * 10**(-3) + 3.2 * 10**(-5) * np.random.randn(2)
        dcmd = torch.as_tensor(cmd[:3].reshape(1, 3), device=self._X.device)
        timed = rollout.timed_plant_code(self.mode_code)
        if timed is not None:          # time-triggered build: the plant needs its clock (native calls made so far)
            call = torch.tensor([self._calls], dtype=torch.int32, device=self._X.device)
            rollout.plant_step(self._X, dcmd, torch.tensor([timed], dtype=torch.int32, device=self._X.device), call)
        else:
            rollout.plant_step(self._X, dcmd, self._variant)
        self._calls += 1
        return x

    def reset(self, **kwargs):
        if not torch.cuda.is_available():
            raise _native.NativeError('CitationEnv needs a CUDA device (no CPU fallback)')
        self.t = 0.
        dev = torch.device('cuda', torch.cuda.current_device())
        self._variant = torch.tensor([rollout.mode_variant(self.mode_code)], dtype=torch.int32, device=dev)
        self._X = rollout.plant_init(self._variant)
        self.last_u = np.zeros(self.n_actions)
        self._calls = 0
        self.x = self._native_step(self.last_u)
        self.V0 = self.V
        self.init_ref(**kwargs)
        self.obs = np.hstack((self.error.flatten(), self.x[self.obs_idx]))     # stale error, as in the reference (:422)
        self.last_obs = self.obs[:]
        return self.obs

    def calc_reference_value(self):
        self.ref_values = np.asarray([np.deg2rad(ref_signal(self.t)) for ref_signal in self.ref])

    def get_reward(self):
        self.calc_reference_value()
        self.error[:self.n_actions] = self.ref_values - np.asarray([self.theta, self.phi, self.beta])
        reward_vec = np.abs(np.clip(self.error_scaler * self.error, -self.max_bound, self.max_bound))
        return -reward_vec.sum() / self.error.shape[0]

    def get_cost(self):
        if np.rad2deg(np.abs(self.alpha)) > 11.0 or np.rad2deg(np.abs(self.phi)) > 0.75 * self.max_phi or self.V < self.V0 / 3:
            return 1
        return 0

    def check_bounds(self):
        if self.t >= self.t_max or np.abs(self.theta) > self.max_theta or np.abs(self.phi) > self.max_phi or self.H < 50:
            return True, -1 / self.dt * (self.t_max - self.t) * 2
        return False, 0.

    def step(self, action):
        self.last_obs = self.obs
        u = self.scale_action(action)
        self.x = self._native_step(u)
        reward = self.get_reward()
        cost = self.get_cost()
        self.obs = np.hstack((self.error.flatten(), self.x[self.obs_idx]))
        self.last_u = u
        is_done, penalty = self.check_bounds()
        reward += penalty
        self.t += self.dt
        return self.obs, reward, is_done, {'ref': self.ref_values, 'x': self.x, 't': self.t, 'cost': cost}

    def finish(self):
        pass
