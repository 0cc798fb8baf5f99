"""The TD3 learner on the device: K7 (csrc/td3.cu) takes a generation's gradient steps in one launch.

`FusedTD3` has TD3's interface (core/td3.py: actor / actor_target / critic / critic_target / buffer / critical_buffer,
update_parameters) and computes the same update up to fp32 summation order.  Every parameter of the four modules is a view
into one flat device buffer, the kernel's learner state (include/serl_td3.h), so state_dict(), rl_to_evo / evo_to_rl copies,
save_agent and the critic handed to SSNE read and write the live weights.  The torch Adam optimisers are not used: the Adam
moments live in the same buffer and the step counts in `critic_steps` / `actor_steps`."""
import ctypes

import numpy as np
import torch

from . import _native
from .core import td3
from .rollout import INCREMENTAL_STATE_DIM, SYMMETRIC_ACTION_DIM, SYMMETRIC_STATE_DIM, TRANSITION_COLS, actor_shape

# steps per launch: keeps every launch well under a second at the largest population
LAUNCH_STEPS = 8192


class TD3Launch:
    """what one or more K7 launches returned: losses [n, 2] (td, pg; pg NaN on critic-only steps), the recorded draws
    (indices [n, B] int32, noise [n, B, 3], caps [n, B, 7]) when asked for, and the status word."""
    __slots__ = ('losses', 'indices', 'noise', 'caps', 'status')

    def check(self):
        st = int(self.status.item())
        if st & _native.STATUS_NONFINITE:
            raise _native.NativeError('serl_td3_train: a loss became NaN or infinite')
        if st & _native.TD3_STATUS_INDEX:
            raise _native.NativeError('serl_td3_train: a given row index was outside the replay rows')


def state_floats(shape):
    n = int(_native.lib().serl_td3_state_floats(ctypes.byref(shape)))
    if n < 0:
        raise _native.NativeError('serl_td3_state_floats: ' + _native.lib().serl_last_error().decode())
    return n


class FusedTD3(td3.TD3):
    def __init__(self, args, cluster_size=0, seed=None):
        if args.state_dim == INCREMENTAL_STATE_DIM:
            raise ValueError('fused_td3: K7 trains the actor of absolute control (state_dim 7); incremental control (state_dim 10) '
                             'trains with the torch TD3 (fused_td3=False)')
        if (args.state_dim, args.action_dim) == (SYMMETRIC_STATE_DIM, SYMMETRIC_ACTION_DIM):
            raise ValueError('fused_td3: K7 trains the actor of attitude control (3 actions); symmetric control (state_dim 2, '
                             'action_dim 1) trains with the torch TD3 (fused_td3=False)')
        super().__init__(args)
        if torch.device(args.device).type != 'cuda':
            raise _native.NativeError('FusedTD3 needs a CUDA device (no CPU fallback)')
        self.actor_optim = self.critic_optim = None            # Adam runs inside the kernel
        self.shape = actor_shape(args.hidden_size, args.num_layers, args.activation_actor, args.state_dim, args.action_dim)
        self.cluster_size = int(cluster_size)
        self.seed = int(getattr(args, 'seed', 7) if seed is None else seed)
        self.critic_steps = self.actor_steps = 0
        dev = next(self.actor.parameters()).device
        self.state = torch.zeros(state_floats(self.shape), dtype=torch.float32, device=dev)
        pa, pc = (sum(q.numel() for q in m.parameters()) for m in (self.actor, self.critic))
        assert 4 * pa + 4 * pc == self.state.numel()
        # actor θ | actor target | actor m | actor v | critic θ | critic target | critic m | critic v
        for mod, off, k in ((self.actor, 0, pa), (self.actor_target, pa, pa), (self.critic, 4 * pa, pc), (self.critic_target, 4 * pa + pc, pc)):
            _bind(mod, self.state[off:off + k])
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)

    def run(self, rows, n_valid, n, first_iteration, champion_target=False, indices=None, record=False, cluster_size=None):
        """n consecutive gradient steps on global iterations first_iteration.. (launches of at most LAUNCH_STEPS) on the replay
        rows [>= n_valid, >= 19] fp32 (device, row-contiguous).  indices [n, B] int32 replaces the sampler's draw."""
        B = int(self.args.batch_size)
        dev = self.state.device
        assert rows.is_cuda and rows.dtype == torch.float32 and rows.dim() == 2 and rows.shape[1] >= TRANSITION_COLS
        assert rows.stride(1) == 1 and rows.shape[0] >= n_valid
        r = self._launch(n, record)
        if indices is not None:
            assert indices.shape == (n, B) and indices.dtype == torch.int32 and indices.is_cuda and indices.is_contiguous()
        k0 = 0
        while k0 < n:
            m = min(LAUNCH_STEPS, n - k0)
            d = self._desc(rows, n_valid, m, int(first_iteration) + k0, champion_target, indices, r, k0, cluster_size)
            _native.call('serl_td3_train', d, device=dev)
            self._advance(int(first_iteration) + k0, m)
            k0 += m
        if n:
            self._bump_versions()
        return r

    def _launch(self, n, record, losses=None):
        """a TD3Launch with losses [n, 2] (new, or the given view) and, when `record`, the draw records; its status word is
        zeroed"""
        B, dev = int(self.args.batch_size), self.state.device
        r = TD3Launch()
        r.losses = torch.empty((n, 2), dtype=torch.float32, device=dev) if losses is None else losses
        r.indices = torch.empty((n, B), dtype=torch.int32, device=dev) if record else None
        r.noise = torch.empty((n, B, 3), dtype=torch.float32, device=dev) if record else None
        r.caps = torch.empty((n, B, 7), dtype=torch.float32, device=dev) if record else None
        r.status = self.status
        self.status.zero_()
        return r

    def _desc(self, rows, n_valid, m, first, champion_target, indices, r, k0, cluster_size=None):
        """the TD3Desc of m steps from global iteration `first`, writing r's rows k0.. (solo and group launches alike)"""
        a = self.args
        caps = self.caps_dict or {'lambda_t': 0.0, 'lambda_s': 0.0, 'eps_sd': 0.0}
        p = lambda t: t[k0:].data_ptr() if t is not None else None
        d = _native.TD3Desc()
        d.shape, d.d_state = self.shape, self.state.data_ptr()
        d.d_replay, d.replay_cols, d.n_valid = rows.data_ptr(), rows.stride(0), int(n_valid)
        d.batch, d.n_steps = int(a.batch_size), m
        d.first_iteration, d.critic_adam_steps, d.actor_adam_steps = int(first), self.critic_steps, self.actor_steps
        d.gamma, d.tau, d.lr, d.noise_sd, d.noise_clip = a.gamma, a.tau, a.lr, a.noise_sd, a.noise_clip
        d.policy_update_freq = int(a.policy_update_freq)
        d.caps_lambda_t, d.caps_lambda_s, d.caps_eps_sd = caps['lambda_t'], caps['lambda_s'], caps['eps_sd']
        d.max_grad_norm = float(td3.MAX_GRAD_NORM)
        d.flags = _native.TD3_CHAMPION_TARGET if champion_target else 0
        d.seed, d.cluster_size = self.seed, int(self.cluster_size if cluster_size is None else cluster_size)
        d.d_indices = p(indices)
        d.d_losses = p(r.losses)
        d.d_rec_indices, d.d_rec_noise, d.d_rec_caps = p(r.indices), p(r.noise), p(r.caps)
        d.d_status = self.status.data_ptr()
        return d

    def _advance(self, first, m):
        """the Adam step counts after m steps from global iteration `first`"""
        its = np.arange(first, first + m)
        self.critic_steps += m
        self.actor_steps += int((its % int(self.args.policy_update_freq) == 0).sum())

    def _bump_versions(self):
        # the kernel wrote the weights behind autograd's back: bump the parameters' version counters, so that anything
        # keyed on them (Agent's prefetched generation front) sees the change
        for mod in (self.actor, self.actor_target, self.critic, self.critic_target):
            for q in mod.parameters():
                torch.autograd.graph.increment_version(q)

    def train_steps(self, replay, n, first_iteration, champion_target=False):
        """n gradient steps sampling from `replay` (DeviceReplayMemory, or a [rows, >= 19] device tensor); returns the device
        losses [n, 2] (td, pg; pg NaN on critic-only steps)."""
        rows, n_valid = _rows(replay)
        return self.run(rows, n_valid, int(n), first_iteration, champion_target).losses

    def update_parameters(self, batch, iteration, champion_policy=False):
        """one step on the given batch (state, action, next_state, reward, done), as TD3.update_parameters"""
        dev = self.state.device
        rows = torch.cat([b.to(dev, torch.float32).reshape(b.shape[0], -1) for b in batch], 1).contiguous()
        B = rows.shape[0]
        assert B == int(self.args.batch_size)
        idx = torch.arange(B, dtype=torch.int32, device=dev).reshape(1, B)
        out = self.run(rows, B, 1, iteration, champion_policy, indices=idx).losses[0].cpu().numpy()
        return (out[1] if iteration % self.args.policy_update_freq == 0 else None), out[0]


def _rows(replay):
    """(rows, n_valid) of a DeviceReplayMemory or of a [rows, >= 19] device tensor"""
    return (replay.data, len(replay)) if hasattr(replay, 'data') else (replay, replay.shape[0])


def train_group(learners, replays, ns, firsts, champion_targets, record=False, mixed_shapes=False):
    """learner g takes ns[g] gradient steps on global iterations firsts[g].. sampling from replays[g] (as
    learners[g].train_steps would), all learners in the same K7 launches (serl_td3_train_group): one cluster per learner,
    lockstep chunks of LAUNCH_STEPS steps, at most TD3_MAX_GROUP learners per launch.  The learners must share cluster
    size, and actor shape unless `mixed_shapes` (serl_td3_train_mixed: narrow and wide actors of any shape K7 trains, in
    the same launches); each gets exactly the bits its solo run gives.  Returns one TD3Launch per learner; their losses
    are views into one device buffer, so `group_losses` reads them back in one copy."""
    G = len(learners)
    assert G == len(replays) == len(ns) == len(firsts) == len(champion_targets)
    assert len(set(id(f) for f in learners)) == G, 'a learner appears twice in the group'
    ns = [int(n) for n in ns]
    firsts = [int(f) for f in firsts]
    if not G:
        return []
    dev = learners[0].state.device
    rows = [_rows(r) for r in replays]
    for (t, nv) in rows:
        assert t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.shape[1] >= TRANSITION_COLS
        assert t.stride(1) == 1 and t.shape[0] >= nv
    flat = torch.empty(2 * sum(ns), dtype=torch.float32, device=dev)
    offs = np.concatenate([[0], np.cumsum(ns)]) * 2
    out = [f._launch(n, record, flat[offs[g]:offs[g + 1]].view(n, 2)) for g, (f, n) in enumerate(zip(learners, ns))]
    k0 = 0
    while k0 < max(ns):
        live = [g for g in range(G) if ns[g] > k0]
        for c in range(0, len(live), _native.TD3_MAX_GROUP):
            part = live[c:c + _native.TD3_MAX_GROUP]
            descs = (_native.TD3Desc * len(part))()
            for j, g in enumerate(part):
                m = min(LAUNCH_STEPS, ns[g] - k0)
                descs[j] = learners[g]._desc(rows[g][0], rows[g][1], m, firsts[g] + k0, champion_targets[g], None, out[g], k0)
            _native.call('serl_td3_train_mixed' if mixed_shapes else 'serl_td3_train_group', descs, len(part), device=dev)
            for g in part:
                learners[g]._advance(firsts[g] + k0, min(LAUNCH_STEPS, ns[g] - k0))
        k0 += LAUNCH_STEPS
    for f, n in zip(learners, ns):
        if n:
            f._bump_versions()
    return out


def group_losses(launches):
    """the host copies (numpy [n, 2]) of train_group's losses, read back in ONE device->host copy"""
    if not launches:
        return []
    base = launches[0].losses._base
    if base is None or any(r.losses._base is not base for r in launches):
        return [r.losses.cpu().numpy() for r in launches]
    host = base.cpu().numpy()
    out, off = [], 0
    for r in launches:
        k = r.losses.numel()
        out.append(host[off:off + k].reshape(-1, 2))
        off += k
    return out


def _bind(module, flat):
    off = 0
    for q in module.parameters():
        k = q.numel()
        flat[off:off + k].copy_(q.data.reshape(-1))
        q.data = flat[off:off + k].view(q.shape)
        off += k
    assert off == flat.numel()
