"""TD3.update_parameters (serl_b200/core/td3.py) with its random draws made explicit — the fp32 oracle of K7 (csrc/td3.cu).

`update_parameters(agent, rows, iteration, noise, caps_u, champion_policy)` performs the same torch operations in the same
order as TD3.update_parameters on a TD3 instance `agent` (its modules and its torch Adam optimisers), with the clipped
target-policy noise and the CAPS uniforms given instead of drawn: fed the draws TD3 itself would have made, it reproduces
it bit for bit (tests/test_td3_oracle.py); fed the draws K7 recorded, it is the reference the kernel is held to.
`as_float64(agent)` is its float64 copy, the sharper reference of tests/test_td3_reference_gpu.py."""
import copy

import torch
from torch import nn
from torch.nn import functional as F

from serl_b200.core.mod_utils import soft_update
from serl_b200.core.td3 import MAX_GRAD_NORM

REPLAY_DIMS = (7, 3, 7, 1, 1)     # obs | action | next_obs | reward | done


def split(rows):
    out, off = [], 0
    for d in REPLAY_DIMS:
        out.append(rows[:, off:off + d])
        off += d
    return tuple(out)


def as_float64(agent):
    """a deep copy of the TD3 `agent` in float64: the four modules in .double(), both Adam optimisers rebuilt on the double
    parameters and given a copy of the original state (load_state_dict casts exp_avg / exp_avg_sq to the parameter dtype
    and keeps `step`; the copy keeps the two optimisers from sharing their CPU `step` tensors, which Adam increments in
    place).  Fed the same draws (in float64), it is the high-precision reference of the fp32 update."""
    d = copy.deepcopy(agent)
    for m in (d.actor, d.actor_target, d.critic, d.critic_target):
        m.double()
    for name, mod in (('actor_optim', d.actor), ('critic_optim', d.critic)):
        src = getattr(agent, name)
        opt = type(src)(mod.parameters(), **src.defaults)
        opt.load_state_dict(copy.deepcopy(src.state_dict()))
        setattr(d, name, opt)
    return d


def update_parameters(agent, rows, iteration, noise, caps_u=None, champion_policy=False, norms=None):
    """rows [B, >= 19] transitions; noise [B, A] clipped target-policy noise; caps_u [B, S] U[0,1) draws (actor steps with
    CAPS).  Returns (pg or None, td) as 0-d tensors.  A list `norms` receives the pre-clip gradient norms that
    clip_grad_norm_ returned: the critic's, then on actor iterations the actor's."""
    norms = [] if norms is None else norms
    state, action, next_state, reward, done = split(rows)
    with torch.no_grad():
        next_action = torch.clamp(noise + agent.actor_target(next_state), -1, 1)
        q1, q2 = agent.critic_target(next_state, next_action)
        target_q = reward + agent.gamma * torch.min(q1, q2) * (1 - done)
    cq1, cq2 = agent.critic(state, action)
    td = F.mse_loss(cq1, target_q) + F.mse_loss(cq2, target_q)
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
            loss = loss + agent.caps_dict['lambda_t'] * F.mse_loss(action, nxt) + agent.caps_dict['lambda_s'] * F.mse_loss(action, bar)
        loss.backward()
        norms.append(float(nn.utils.clip_grad_norm_(agent.actor.parameters(), MAX_GRAD_NORM)))
        agent.actor_optim.step()
        if not champion_policy:
            soft_update(agent.actor_target, agent.actor, agent.tau)
        soft_update(agent.critic_target, agent.critic, agent.tau)
        pgl = loss.detach()
    return pgl, td.detach()
