"""Distillation crossover (base/core/mod_neuro_evo.py:131-181, :497-513; GeneticAgent.update_parameters
base/core/genetic_agent.py:22-60) batched over all children of a generation (SURVEY.md 8(f) N3).

The reference builds one child at a time: a fresh GeneticAgent initialised with parent 2's weights, a buffer made of the
latest individual_bs/2 transitions of each parent (shuffled), then 12 epochs of len(buffer)//128 Adam(lr=1e-3) steps of
Q-filtered behaviour cloning: per sample the target is the action of the parent whose action the critic values more (by
more than 1e-5), loss = sum of squared errors over the selected samples + mean(child_action^2).  Adam is elementwise, so
the children are independent rows of ONE [C, P] parameter tensor with one optimiser: a step for all children is one
batched forward / backward on the device.  Deviations: batches are drawn with a device generator (the reference uses
stdlib random.sample / shuffle); children of a generation use the common buffer length min_c len(buffer_c)."""
import numpy as np
import torch

from . import evo_prox

EPS_Q = 10 ** -5
EPOCHS = 12
BATCH = 128


def sort_groups_by_fitness(genomes, fitness):
    """mod_neuro_evo.py:388-397: all parent pairs (better one first) sorted by summed fitness, best first."""
    groups = []
    for i, first in enumerate(genomes):
        for second in genomes[i + 1:]:
            if fitness[first] < fitness[second]:
                groups.append((second, first, fitness[first] + fitness[second]))
            else:
                groups.append((first, second, fitness[first] + fitness[second]))
    return sorted(groups, key=lambda group: group[2], reverse=True)


def cloning_loss(child_action, p1_action, p2_action, p1_q, p2_q):
    """genetic_agent.py:41-55 for a stack of children: actions [C, B, A], Q values [C, B] -> (loss summed over children, mse [C])."""
    m1 = (p1_q - p2_q) > EPS_Q
    m2 = (p2_q - p1_q) >= EPS_Q
    sel = (m1 | m2).unsqueeze(-1).to(child_action.dtype)
    target = torch.where(m1.unsqueeze(-1), p1_action, p2_action).detach()
    sq = (child_action - target) ** 2 * sel
    n_sel = sel.sum(dim=(1, 2)).clamp(min=1.0) * child_action.shape[2]
    per_child = sq.sum(dim=(1, 2)) + (child_action ** 2 * sel).sum(dim=(1, 2)) / n_sel
    return per_child.sum(), (sq.sum(dim=(1, 2)) / n_sel).detach()


def distil_children(genomes, first, second, buffers, shape, activation, critic, generator=None, epochs=EPOCHS, batch=BATCH):
    """genomes [pop, P]; first / second: parent indices (first = the fitter, mod_neuro_evo.py:509-510) of the C children;
    buffers: list of C tensors [M_c, >=S] (each child's mixed state buffer); shape = (S, A, h, L).  Returns child genomes [C, P]."""
    dev = genomes.device
    C = len(first)
    S = int(shape[0])
    M = min(int(b.shape[0]) for b in buffers)
    states_all = torch.stack([b[:M, :S] for b in buffers]).to(torch.float32)             # [C, M, S]
    i1 = torch.as_tensor(first, dtype=torch.int64, device=dev)
    i2 = torch.as_tensor(second, dtype=torch.int64, device=dev)
    G1, G2 = genomes[i1].detach(), genomes[i2].detach()
    child = G2.clone().requires_grad_(True)                                              # hard_update(new_agent.actor, gene2.actor)
    opt = torch.optim.Adam([child], lr=1e-3)
    bs = min(batch, M)
    iters = M // bs
    for p in critic.parameters():
        p.requires_grad_(False)
    try:
        for _ in range(epochs * iters):
            pick = torch.rand((C, M), device=dev, generator=generator).argsort(dim=1)[:, :bs]      # without replacement
            st = torch.gather(states_all, 1, pick.unsqueeze(-1).expand(C, bs, S))
            with torch.no_grad():
                a1 = evo_prox.actor_forward_batched(G1, st, shape, activation)
                a2 = evo_prox.actor_forward_batched(G2, st, shape, activation)
                flat = st.reshape(C * bs, S)
                q1a, q1b = critic(flat, a1.reshape(C * bs, -1))
                q2a, q2b = critic(flat, a2.reshape(C * bs, -1))
                p1_q = torch.min(q1a, q1b).reshape(C, bs)
                p2_q = torch.min(q2a, q2b).reshape(C, bs)
            opt.zero_grad()
            loss, _ = cloning_loss(evo_prox.actor_forward_batched(child, st, shape, activation), a1, a2, p1_q, p2_q)
            loss.backward()
            opt.step()
    finally:
        for p in critic.parameters():
            p.requires_grad_(True)
    return child.detach()


def child_buffer(pop, first, second, half, generator=None):
    """new_agent.buffer (:133-135): the latest `half` transitions of each parent, shuffled."""
    rows = torch.cat((pop[first].buffer._chronological_rows()[-half:], pop[second].buffer._chronological_rows()[-half:]))
    if rows.shape[0] == 0:
        raise RuntimeError('distillation crossover: parents %d / %d have empty replay buffers' % (first, second))
    return rows[torch.randperm(rows.shape[0], device=rows.device, generator=generator)]
