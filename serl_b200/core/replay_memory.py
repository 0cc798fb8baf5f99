"""Uniform replay ring buffer with the interface the reference's callers use (base/core/replay_memory.py:13-100:
add / add_content_of / get_latest / sample / reset / len), stored as preallocated numpy arrays instead of a list of
namedtuples.  `ReplayMemory` is the host version; `DeviceReplayMemory` / `PopulationBuffers` keep the transitions the
rollout kernel exports (K1 replay rows, csrc/rollout.cu) on the GPU: the shared buffer TD3 samples from and the
per-actor buffers of the population never leave the device (SURVEY.md 8(f) N2)."""
import random
from collections import namedtuple

import numpy as np
import torch

from .. import _native
from ..rollout import replay_dims, transition_cols

Transition = namedtuple('Transition', ('state', 'action', 'next_state', 'reward', 'done'))


class ReplayMemory:
    def __init__(self, capacity, device):
        self.capacity, self.device = int(capacity), device
        self._store = None          # dict of field -> [capacity, dim] float32
        self._count = 0             # transitions ever written
        self.position = 0

    def reset(self):
        self._count, self.position = 0, 0

    def __len__(self):
        return min(self._count, self.capacity)

    def add(self, state, action, next_state, reward, done):
        row = [np.asarray(v, dtype=np.float32).reshape(-1) for v in (state, action, next_state, reward, done)]
        if self._store is None:
            self._store = {f: np.zeros((self.capacity, r.shape[0]), dtype=np.float32) for f, r in zip(Transition._fields, row)}
        for f, r in zip(Transition._fields, row):
            self._store[f][self.position] = r
        self.position = (self.position + 1) % self.capacity
        self._count += 1

    def add_batch(self, states, actions, next_states, rewards, dones):
        """vectorised `add` of n transitions in order (what a traced GPU episode delivers): same ring semantics."""
        cols = [np.asarray(v, dtype=np.float32).reshape(len(rewards), -1) for v in (states, actions, next_states, rewards, dones)]
        n = cols[0].shape[0]
        if n == 0:
            return
        if self._store is None:
            self._store = {f: np.zeros((self.capacity, c.shape[1]), dtype=np.float32) for f, c in zip(Transition._fields, cols)}
        idx = (self.position + np.arange(n)) % self.capacity
        if n > self.capacity:                       # only the last `capacity` rows survive, at the slots they would land in
            idx, cols = idx[-self.capacity:], [c[-self.capacity:] for c in cols]
        for f, c in zip(Transition._fields, cols):
            self._store[f][idx] = c
        self.position = int((self.position + n) % self.capacity)
        self._count += n

    def _chronological(self):
        n = len(self)
        if self._count <= self.capacity:
            return np.arange(n)
        return (np.arange(n) + self.position) % self.capacity

    def get_latest(self, latest):
        order = self._chronological()[-int(latest):]
        return [Transition(*(self._store[f][i:i + 1].copy() for f in Transition._fields)) for i in order]

    def add_content_of(self, other):
        if other._store is None:
            return
        for i in other._chronological()[-self.capacity:]:
            self.add(*(other._store[f][i] for f in Transition._fields))

    def sample(self, batch_size):
        # same stdlib-`random` consumption as the reference's random.sample(self.memory, batch_size) (:66), so that the
        # stream position seen by the next SSNE.epoch does not depend on which buffer implementation is used
        order = self._chronological() if self._count > self.capacity else None
        pick = np.asarray(random.sample(range(len(self)), batch_size))
        return tuple(torch.from_numpy(self._store[f][pick]).to(self.device) for f in Transition._fields)


def _split(rows, state_dim, action_dim=3):
    """the Transition fields (obs, action, next_obs, reward, done) of stored transitions [n, transition_cols(state_dim, action_dim)]"""
    out, off = [], 0
    for d in replay_dims(state_dim, action_dim)[:5]:
        out.append(rows[:, off:off + d])
        off += d
    return tuple(out)


class DeviceReplayMemory:
    """Ring buffer on the GPU with ReplayMemory's interface.  Rows are K1 replay rows (include/serl_b200.h
    SERL_REPLAY_COLS_SA(state_dim, action_dim): obs | action | next_obs | reward | done | cost; rollout.replay_dims) without the cost
    flag; sampling uses a device generator, so the stdlib `random` stream the SSNE planner consumes does not depend on the
    buffer (every rank holds identical buffers and identical generators -> identical batches)."""

    def __init__(self, capacity, device, seed=0, state_dim=7, action_dim=3):
        self.capacity, self.device = int(capacity), torch.device(device)
        self.state_dim, self.action_dim = int(state_dim), int(action_dim)
        self.cols = transition_cols(self.state_dim, self.action_dim)
        self.data = None
        self._count, self.position = 0, 0
        self.gen = None
        self._seed = seed

    def reset(self):
        self._count, self.position = 0, 0

    def __len__(self):
        return min(self._count, self.capacity)

    def _alloc(self):
        if self.data is None:
            self.data = torch.zeros((self.capacity, self.cols), dtype=torch.float32, device=self.device)
            self.gen = torch.Generator(device=self.device)
            self.gen.manual_seed(self._seed)

    def add_rows(self, rows):
        """append n transitions [n, >=cols] (device tensor, chronological order) with ring semantics."""
        n = int(rows.shape[0])
        if n == 0:
            return
        self._alloc()
        rows = rows[:, :self.cols].to(self.device, torch.float32)
        if n > self.capacity:
            skip = n - self.capacity
            rows = rows[skip:]
            self.position = (self.position + skip) % self.capacity
            self._count += skip
            n = self.capacity
        end = self.position + n
        if end <= self.capacity:
            self.data[self.position:end] = rows
        else:
            k = self.capacity - self.position
            self.data[self.position:] = rows[:k]
            self.data[:end - self.capacity] = rows[k:]
        self.position = end % self.capacity
        self._count += n

    def add_batch(self, states, actions, next_states, rewards, dones):
        cols = [np.asarray(v, dtype=np.float32).reshape(len(rewards), -1) for v in (states, actions, next_states, rewards, dones)]
        self.add_rows(torch.from_numpy(np.hstack(cols)))

    def add(self, state, action, next_state, reward, done):
        self.add_batch(np.asarray(state).reshape(1, -1), np.asarray(action).reshape(1, -1), np.asarray(next_state).reshape(1, -1),
                       np.asarray([reward]), np.asarray([done]))

    def _chronological_rows(self):
        n = len(self)
        if n == 0:
            return torch.zeros((0, self.cols), dtype=torch.float32, device=self.device)
        if self._count <= self.capacity:
            return self.data[:n]
        return torch.cat((self.data[self.position:], self.data[:self.position]))

    def get_latest(self, latest):
        rows = self._chronological_rows()[-int(latest):]
        return [Transition(*_split(rows[i:i + 1], self.state_dim, self.action_dim)) for i in range(rows.shape[0])]

    def add_content_of(self, other):
        rows = other._chronological_rows() if hasattr(other, '_chronological_rows') else None
        if rows is None:
            if other._store is None:
                return
            order = other._chronological()
            rows = torch.from_numpy(np.hstack([other._store[f][order] for f in Transition._fields]))
        self.add_rows(rows[-self.capacity:])

    def sample(self, batch_size):
        self._alloc()
        n = len(self)
        pick = torch.randperm(n, device=self.device, generator=self.gen)[:int(batch_size)]
        return _split(self.data[pick], self.state_dim, self.action_dim)


class DevicePrioritizedReplayMemory(DeviceReplayMemory):
    """The reference's PrioritizedReplayMemory (base/core/replay_memory.py:103-176) on the GPU: DeviceReplayMemory's rows plus
    a priority tree over them (include/serl_td3_per.h, csrc/per.cu) in fp64.  A new row gets the largest stored priority
    (1.0 in an empty buffer); `sample` draws B rows with replacement with P(i) = p_i / sum p and returns them with their
    importance weights w = (N P(i))^-beta / (N min P)^-beta and the row indices; `update_priorities` sets p = (|delta| +
    1e-5)^alpha.  beta = min(1, beta_start + frame (1 - beta_start) / beta_frames) at the frame-th sample (frame from 1).
    The draw of the frame-th sample is K7's draw at global iteration `frame` with Philox key `seed`, so FusedTD3 (which
    samples this tree inside K7, td3_fused.FusedTD3.run) and the torch loop of Agent.train_rl draw the same rows."""

    def __init__(self, capacity, device, seed=0, state_dim=7, action_dim=3, alpha=0.6, beta_start=0.4, beta_frames=100000):
        super().__init__(capacity, device, seed, state_dim, action_dim)
        self.prob_alpha, self.beta_start, self.beta_frames = float(alpha), float(beta_start), float(beta_frames)
        self.frame = 1
        self.tree = None

    def beta_by_frame(self, frame_idx):
        return min(1.0, self.beta_start + frame_idx * (1.0 - self.beta_start) / self.beta_frames)

    def _alloc(self):
        super()._alloc()
        if self.tree is None:
            n = int(_native.lib().serl_per_tree_doubles(self.capacity))
            if n < 0:
                raise _native.NativeError('serl_per_tree_doubles: ' + _native.lib().serl_last_error().decode())
            self.tree = torch.empty(n, dtype=torch.float64, device=self.device)
            self._clear_tree()

    def _clear_tree(self):
        t = self.tree.view(-1, 2)
        t[:, 0] = 0.0                      # no stored row: sum 0, min +inf
        t[:, 1] = float('inf')

    def reset(self):
        super().reset()
        if self.tree is not None:
            self._clear_tree()

    def add_rows(self, rows):
        # a bulk add gives every new or overwritten row the max stored before the add: n sequential adds of the reference
        # would give the same, since writing the max never lowers the max
        n = int(rows.shape[0])
        if n == 0:
            return
        self._alloc()
        n_valid, start = len(self), (self.position + max(0, n - self.capacity)) % self.capacity
        super().add_rows(rows)
        _native.call('serl_per_insert', self.tree, self.capacity, n_valid, start, min(n, self.capacity), device=self.device)

    def sample(self, batch_size):
        """(state, action, next_state, reward, done, weights [B, 1] fp32, rows [B] int32)"""
        self._alloc()
        B = int(batch_size)
        rows = torch.empty(B, dtype=torch.int32, device=self.device)
        weights = torch.empty((B, 1), dtype=torch.float32, device=self.device)
        _native.call('serl_per_sample', self.tree, self.capacity, len(self), B, self._seed, self.frame,
                     self.beta_by_frame(self.frame), rows, weights, device=self.device)
        self.frame += 1
        return _split(self.data[rows.long()], self.state_dim, self.action_dim) + (weights, rows)

    def update_priorities(self, batch_indices, batch_priorities):
        """rows batch_indices [B] get (|delta| + 1e-5)^alpha from batch_priorities = delta [B] (batch order: a row drawn twice
        keeps its later delta)"""
        rows = torch.as_tensor(batch_indices, device=self.device).to(torch.int32).reshape(-1).contiguous()
        td = torch.as_tensor(batch_priorities, device=self.device).to(torch.float32).reshape(-1).abs().contiguous()
        _native.call('serl_per_update', self.tree, self.capacity, rows, td, int(rows.numel()), self.prob_alpha, device=self.device)

    def leaves(self):
        """the priorities of the stored rows (fp64 [len])"""
        self._alloc()
        return self.tree.view(-1, 2)[self.tree.numel() // 4:, 0][:len(self)]


class PopulationBuffers:
    """The per-actor replay buffers of the whole population (GeneticAgent.buffer / .critical_buffer,
    base/core/genetic_agent.py:14-16) as ONE device tensor [pop, capacity, cols] with per-actor ring positions, filled
    for all actors of a generation by one vectorised scatter (cols: the transition of an observation of state_dim entries and
    action_dim actions)."""

    def __init__(self, pop, capacity, device, state_dim=7, action_dim=3):
        self.pop, self.capacity, self.device = int(pop), int(capacity), torch.device(device)
        self.state_dim, self.action_dim = int(state_dim), int(action_dim)
        self.cols = transition_cols(self.state_dim, self.action_dim)
        self.data = None
        self.pos = torch.zeros(self.pop, dtype=torch.int64, device=self.device)
        self.count = torch.zeros(self.pop, dtype=torch.int64, device=self.device)
        self.gen = None

    def _alloc(self):
        if self.data is None:
            self.data = torch.zeros((self.pop, self.capacity, self.cols), dtype=torch.float32, device=self.device)
            self.gen = torch.Generator(device=self.device)
            self.gen.manual_seed(1)

    def append(self, actors, rows, select):
        """rows [n, horizon, >=cols]; select [n, horizon] bool (time order): the selected rows of rows[i] go to actor actors[i]."""
        self._alloc()
        n, h = select.shape
        cnt = select.sum(1)
        rank = torch.cumsum(select, 1) - 1
        keep = select & (rank >= (cnt - self.capacity)[:, None])
        a_idx = actors.to(torch.int64)[:, None].expand(n, h)
        slot = (self.pos[actors][:, None] + rank) % self.capacity
        self.data[a_idx[keep], slot[keep]] = rows[..., :self.cols][keep].to(torch.float32)
        self.pos[actors] = (self.pos[actors] + cnt) % self.capacity
        self.count[actors] += cnt

    def copy_actor(self, src, dst):
        if self.data is not None:
            self.data[dst] = self.data[src]
        self.pos[dst] = self.pos[src]
        self.count[dst] = self.count[src]

    def rows_of(self, i):
        n = int(min(int(self.count[i]), self.capacity))
        if n == 0 or self.data is None:
            return torch.zeros((0, self.cols), dtype=torch.float32, device=self.device)
        if int(self.count[i]) <= self.capacity:
            return self.data[i, :n]
        p = int(self.pos[i])
        return torch.cat((self.data[i, p:], self.data[i, :p]))


class ActorBuffer:
    """handle on one actor's ring of a PopulationBuffers with the ReplayMemory interface."""

    def __init__(self, owner, index):
        self.owner, self.index = owner, int(index)

    def __len__(self):
        return int(min(int(self.owner.count[self.index]), self.owner.capacity))

    def reset(self):
        self.owner.pos[self.index] = 0
        self.owner.count[self.index] = 0

    def _chronological_rows(self):
        return self.owner.rows_of(self.index)

    def add_rows(self, rows):
        """append n chronological rows to this actor's ring.  Index arithmetic on the device only: no host<->device copy and
        no synchronisation (this runs while validation episodes fly on other streams, and a pageable copy would wait for them)."""
        n = int(rows.shape[0])
        if n == 0:
            return
        o = self.owner
        o._alloc()
        rows = rows[-o.capacity:, :o.cols].to(o.device, torch.float32)
        m = int(rows.shape[0])
        slot = (o.pos[self.index] + (n - m) + torch.arange(m, device=o.device)) % o.capacity
        o.data[self.index, slot] = rows
        o.pos[self.index] = (o.pos[self.index] + n) % o.capacity
        o.count[self.index] += n

    def add_batch(self, states, actions, next_states, rewards, dones):
        cols = [np.asarray(v, dtype=np.float32).reshape(len(rewards), -1) for v in (states, actions, next_states, rewards, dones)]
        self.add_rows(torch.from_numpy(np.hstack(cols)))

    def add(self, state, action, next_state, reward, done):
        self.add_batch(np.asarray(state).reshape(1, -1), np.asarray(action).reshape(1, -1), np.asarray(next_state).reshape(1, -1),
                       np.asarray([reward]), np.asarray([done]))

    def add_content_of(self, other):
        self.add_rows(other._chronological_rows()[-self.owner.capacity:])

    def get_latest(self, latest):
        rows = self._chronological_rows()[-int(latest):]
        return [Transition(*_split(rows[i:i + 1], self.owner.state_dim, self.owner.action_dim)) for i in range(rows.shape[0])]

    def sample(self, batch_size):
        self.owner._alloc()
        rows = self._chronological_rows()
        pick = torch.randperm(rows.shape[0], device=rows.device, generator=self.owner.gen)[:int(batch_size)]
        return _split(rows[pick], self.owner.state_dim, self.owner.action_dim)
