"""oracle/td3.update_parameters with prioritized replay's importance weights: the reference K7's PER learner
(serl_td3_learn with a priority tree) and the weighted torch path (core/td3.py) are held to.

`update_parameters(agent, rows, iteration, noise, caps_u, champion_policy, norms, weights)` is oracle.td3.update_parameters
with the critic loss mean(w (q1 - y)^2) + mean(w (q2 - y)^2) and returns, after (pg, td), the per-row TD error
delta = (|q1 - y| + |q2 - y|) / 2 of the critic before its update.  With weights = 1 (the default) it gives oracle.td3's
bits (tests/test_td3_per.py); the actor loss and the CAPS terms are unweighted, as there."""
import torch
from torch import nn

from oracle.td3 import split
from serl_b200.core.mod_utils import soft_update
from serl_b200.core.td3 import MAX_GRAD_NORM


def update_parameters(agent, rows, iteration, noise, caps_u=None, champion_policy=False, norms=None, weights=None):
    """rows [B, >= 19]; weights [B] or [B, 1] (default ones).  Returns (pg or None, td, delta [B]) as tensors."""
    norms = [] if norms is None else norms
    state, action, next_state, reward, done = split(rows)
    w = torch.ones_like(reward) if weights is None else weights.reshape(-1, 1).to(reward.dtype)
    with torch.no_grad():
        next_action = torch.clamp(noise + agent.actor_target(next_state), -1, 1)
        q1, q2 = agent.critic_target(next_state, next_action)
        target_q = reward + agent.gamma * torch.min(q1, q2) * (1 - done)
    cq1, cq2 = agent.critic(state, action)
    td = torch.mean(w * (cq1 - target_q) ** 2) + torch.mean(w * (cq2 - target_q) ** 2)
    delta = (((cq1 - target_q).abs() + (cq2 - target_q).abs()) * 0.5).detach().reshape(-1)
    agent.critic_optim.zero_grad()
    td.backward()
    norms.append(float(nn.utils.clip_grad_norm_(agent.critic.parameters(), MAX_GRAD_NORM)))
    agent.critic_optim.step()
    pgl = None
    if iteration % agent.args.policy_update_freq == 0:
        agent.actor_optim.zero_grad()
        loss = -torch.mean(agent.critic(state, agent.actor(state))[0])
        if agent.caps_dict is not None:
            nxt = agent.actor(state)
            bar = agent.actor(state + caps_u * agent.caps_dict['eps_sd'])
            loss = loss + agent.caps_dict['lambda_t'] * nn.functional.mse_loss(action, nxt) + \
                agent.caps_dict['lambda_s'] * nn.functional.mse_loss(action, bar)
        loss.backward()
        norms.append(float(nn.utils.clip_grad_norm_(agent.actor.parameters(), MAX_GRAD_NORM)))
        agent.actor_optim.step()
        if not champion_policy:
            soft_update(agent.actor_target, agent.actor, agent.tau)
        soft_update(agent.critic_target, agent.critic, agent.tau)
        pgl = loss.detach()
    return pgl, td.detach(), delta


def beta_by_frame(frame, beta_start=0.4, beta_frames=100000):
    """the reference buffer's beta (base/core/replay_memory.py beta_by_frame)"""
    return min(1.0, beta_start + frame * (1.0 - beta_start) / beta_frames)


class NumpyTree:
    """include/serl_td3_per.h's priority tree restated in numpy: node n's (sum, min) at t[n]"""

    def __init__(self, capacity):
        import numpy as np
        self.np = np
        self.capacity = int(capacity)
        self.leaves = 1
        while self.leaves < self.capacity:
            self.leaves *= 2
        self.t = np.zeros((2 * self.leaves, 2))
        self.t[:, 1] = np.inf
        self.n_valid = 0
        self.pos = 0

    def _rebuild(self):
        for v in range(self.leaves - 1, 0, -1):
            self.t[v, 0] = self.t[2 * v, 0] + self.t[2 * v + 1, 0]
            self.t[v, 1] = min(self.t[2 * v, 1], self.t[2 * v + 1, 1])

    def add(self, n):
        """n rows at the ring position, each at the max stored before the add (1.0 when empty)"""
        np = self.np
        p = self.t[self.leaves:self.leaves + self.n_valid, 0].max() if self.n_valid else 1.0
        keep = min(n, self.capacity)
        start = (self.pos + n - keep) % self.capacity
        rows = (start + np.arange(keep)) % self.capacity
        self.t[self.leaves + rows] = p
        self.pos = (self.pos + n) % self.capacity
        self.n_valid = min(self.n_valid + n, self.capacity)
        self._rebuild()

    def update(self, rows, td, alpha=0.6):
        for r, d in zip(rows, td):              # batch order: the later of two equal rows wins
            self.t[self.leaves + int(r)] = (float(d) + 1e-5) ** alpha
        self._rebuild()

    def priorities(self):
        return self.t[self.leaves:self.leaves + self.n_valid, 0].copy()
