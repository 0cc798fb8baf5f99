"""TD3 learner used by Agent.train for the RL half (base/core/td3.py:17-198).  Gradient RL is outside the B200 hot path
(SURVEY.md 2.1 "OUT OF SCOPE — keep as-is on host"): this is a plain PyTorch implementation with the reference's
interface (TD3(args): .actor/.actor_target/.critic/.buffer/.critical_buffer, update_parameters(batch, iteration, champion))."""
import torch
import torch.nn as nn
from torch.nn import functional as F
from torch.optim import Adam

from . import replay_memory
from .genetic_agent import Actor
from .mod_utils import LayerNorm, activations, hard_update, soft_update

MAX_GRAD_NORM = 10


class Critic(nn.Module):
    def __init__(self, args):
        super().__init__()
        self.args = args
        l1 = l2 = 64
        self.activation = activations[args.activation_actor.lower()]
        d = args.state_dim + args.action_dim

        def head():
            return nn.ModuleList([nn.Linear(d, l1), LayerNorm(l1), nn.Linear(l1, l2), LayerNorm(l2), nn.Linear(l2, 1)])
        self.q1, self.q2 = head(), head()
        for q in (self.q1, self.q2):
            q[4].weight.data.mul_(0.1)
            q[4].bias.data.mul_(0.1)
        self.to(args.device)

    def _q(self, q, x):
        x = self.activation(q[1](q[0](x)))
        x = self.activation(q[3](q[2](x)))
        return q[4](x)

    def forward(self, state, action):
        x = torch.cat((state, action), 1)
        return self._q(self.q1, x), self._q(self.q2, x)


class TD3:
    def __init__(self, args):
        self.args = args
        if torch.device(args.device).type == 'cuda':
            mem = lambda capacity, device: replay_memory.DeviceReplayMemory(capacity, device, state_dim=args.state_dim,
                                                                               action_dim=args.action_dim)
        else:
            mem = replay_memory.ReplayMemory
        self.buffer = mem(args.individual_bs, args.device)
        self.critical_buffer = mem(args.individual_bs, args.device)
        self.actor = Actor(args, init=True).to(args.device)
        self.actor_target = Actor(args, init=True).to(args.device)
        self.actor_optim = Adam(self.actor.parameters(), lr=args.lr)
        self.critic = Critic(args)
        self.critic_target = Critic(args)
        self.critic_optim = Adam(self.critic.parameters(), lr=args.lr)
        self.gamma, self.tau = args.gamma, args.tau
        hard_update(self.actor_target, self.actor)
        hard_update(self.critic_target, self.critic)
        self.caps_dict = {'lambda_s': 0.5, 'lambda_t': 0.1, 'eps_sd': 0.05} if args.use_caps else None

    def update_parameters(self, batch, iteration, champion_policy=False):
        """batch: (state, action, next_state, reward, done), or a prioritized sample (DevicePrioritizedReplayMemory.sample:
        ..., weights [B, 1], rows): then the critic loss is mean(w (q1 - y)^2) + mean(w (q2 - y)^2), and the per-row TD
        error delta = (|q1 - y| + |q2 - y|) / 2 of the critic before its update is returned third, for update_priorities"""
        state, action, next_state, reward, done = (b.to(self.args.device) for b in batch[:5])
        weights = batch[5].to(self.args.device) if len(batch) > 5 else None
        with torch.no_grad():
            noise = (torch.randn_like(action) * self.args.noise_sd).clamp(-self.args.noise_clip, self.args.noise_clip)
            next_action = torch.clamp(noise + self.actor_target(next_state), -1, 1)
            q1, q2 = self.critic_target(next_state, next_action)
            target_q = reward + self.gamma * torch.min(q1, q2) * (1 - done)
        cq1, cq2 = self.critic(state, action)
        if weights is None:
            td = F.mse_loss(cq1, target_q) + F.mse_loss(cq2, target_q)
        else:
            td = torch.mean(weights * (cq1 - target_q) ** 2) + torch.mean(weights * (cq2 - target_q) ** 2)
            delta = (((cq1 - target_q).abs() + (cq2 - target_q).abs()) * 0.5).detach().reshape(-1)
        self.critic_optim.zero_grad()
        td.backward()
        nn.utils.clip_grad_norm_(self.critic.parameters(), MAX_GRAD_NORM)
        self.critic_optim.step()
        pgl = None
        if iteration % self.args.policy_update_freq == 0:
            self.actor_optim.zero_grad()
            loss = -torch.mean(self.critic(state, self.actor(state))[0])
            if self.caps_dict is not None:
                nxt = self.actor(state)
                bar = self.actor(state + torch.rand_like(state) * self.caps_dict['eps_sd'])
                loss = loss + self.caps_dict['lambda_t'] * F.mse_loss(action, nxt) + self.caps_dict['lambda_s'] * F.mse_loss(action, bar)
            loss.backward()
            nn.utils.clip_grad_norm_(self.actor.parameters(), MAX_GRAD_NORM)
            self.actor_optim.step()
            if not champion_policy:
                soft_update(self.actor_target, self.actor, self.tau)
            soft_update(self.critic_target, self.critic, self.tau)
            pgl = loss.data.cpu().numpy()
        if weights is not None:
            return pgl, td.data.cpu().numpy(), delta
        return pgl, td.data.cpu().numpy()
