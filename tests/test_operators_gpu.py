"""The mutation-operator study on the device: the cost tally of the tracking launches (serl_rollout_desc.d_cost) against the
replay rows' cost column and the oracle plant, the parents' buffers against a restatement of
OperatorRunner.evaluate(save_transitions=True), the children against the reference-order mutation operators, and every
child's scores against that child flown alone."""
import os
import random
import types

import numpy as np
import pytest
import torch

from serl_b200 import evaluation, evo, evo_prox, operators, rollout
from serl_b200.core.genetic_agent import Actor

pytestmark = pytest.mark.gpu
ACT = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'actors.npz'))
DEV = torch.device('cuda:0')
CONDS = ['nominal', 'low-q', 'high-q', 'be', 'jr', 'sa', 'se', 'cg', 'ice', 'cg-shift', 'test', 'noise', 'gust']


class Args:
    state_dim, action_dim = 7, 3

    def __init__(self, hidden, layers, act):
        self.hidden_size, self.num_layers, self.activation_actor = hidden, layers, act


def random_genomes(n, hidden, layers, act, seed=0):
    torch.manual_seed(seed)
    return np.stack([Actor(Args(hidden, layers, act)).flat().detach().numpy() for _ in range(n)]).astype(np.float32)


def wide_genomes(widths, n, seed=1):
    from oracle import actor as A
    torch.manual_seed(seed)
    return np.stack([A.flatten(A.WideActor(widths)) for _ in range(n)]).astype(np.float32)


# K1 warp (h = 72), the one-thread-per-env kernel (h = 141), K1-TC (a width list, and the reference's Actor at h = 256)
CASES = {
    'k1_h72': lambda: (ACT['serl10_pop_h72_tanh'][:3], rollout.actor_shape(72, 3, 'tanh'), None),
    'simple_h141': lambda: (random_genomes(2, 141, 1, 'tanh'), rollout.actor_shape(141, 1, 'tanh'), None),
    'tc_400_300': lambda: (wide_genomes([400, 300], 2), rollout.actor_shape(8, 1, 'tanh'), [400, 300]),
    'tc_256x4': lambda: (random_genomes(2, 256, 3, 'relu'), rollout.actor_shape(256, 3, 'relu'), None),
}


def t(x):
    return torch.as_tensor(np.ascontiguousarray(x), device=DEV)


def shared_launch(g, shape, widths, conds, refs, z, **kw):
    """every actor on every (condition, trial) env: t_max = 20 s, the study's smooth width"""
    codes = np.repeat([evaluation.condition_env(c).mode_code for c in conds], len(refs))
    lv, st = evaluation._ref_arrays(refs)
    md = t(codes.astype(np.int32))
    r = rollout.population_rollout(t(g), shape, t(np.tile(lv, (len(conds), 1, 1))), t(np.tile(st, (len(conds), 1, 1))), md,
                                   t_max=20.0, smooth_width=2.0, env_order=rollout.variant_sorted_order(md), widths=widths,
                                   sensor_noise=None if z is None else t(z), gust=any(rollout.mode_gust(int(c)) for c in codes),
                                   fitness=False, **kw)
    torch.cuda.synchronize()
    r.check()
    return r, codes


def per_trajectory_launch(g, shape, widths, codes, refs, n_conds, z):
    """the same trajectories, each env 0 of its own actor row (per-actor env blocks): every one exports its replay rows"""
    A, E = g.shape[0], len(codes)
    lv, st = evaluation._ref_arrays(refs)
    lv, st = np.tile(lv, (n_conds, 1, 1)), np.tile(st, (n_conds, 1, 1))
    r = rollout.population_rollout(t(np.repeat(g, E, axis=0)), shape, t(np.tile(lv, (A, 1, 1)).reshape(A * E, 1, 2, 6)),
                                   t(np.tile(st, (A, 1, 1)).reshape(A * E, 1, 2, 6)), t(np.tile(codes, A).reshape(A * E, 1).astype(np.int32)),
                                   t_max=20.0, smooth_width=2.0, widths=widths, replay_env=0, fitness=False,
                                   sensor_noise=None if z is None else t(z.reshape(A * E, 1, *z.shape[2:])),
                                   gust=any(rollout.mode_gust(int(c)) for c in codes))
    torch.cuda.synchronize()
    r.check()
    return r


def replay_cost(r):
    k = torch.arange(r.replay.shape[1], device=DEV)
    return ((r.replay[..., rollout.REPLAY_COST] > 0.5) & (k[None] < r.steps[:, :1])).sum(1).to(torch.int32)


@pytest.mark.parametrize('case', sorted(CASES))
def test_cost_tally_equals_the_replay_cost_column_and_leaves_the_launch_unchanged(case):
    g, shape, widths = CASES[case]()
    np.random.seed(5)
    refs = operators.study_refs(1)
    for conds, noisy in ((CONDS[:-2], False), (CONDS[-2:], True)):
        z = np.random.RandomState(9).randn(g.shape[0], len(conds) * len(refs), 2002, 7).astype(np.float32) if noisy else None
        r, codes = shared_launch(g, shape, widths, conds, refs, z, track=True, cost=True)
        assert r.cost.shape == r.steps.shape and r.cost.dtype == torch.int32
        solo = per_trajectory_launch(g, shape, widths, codes, refs, len(conds), z)
        assert torch.equal(solo.returns.reshape(r.returns.shape), r.returns) and torch.equal(solo.steps.reshape(r.steps.shape), r.steps)
        assert torch.equal(replay_cost(solo).reshape(r.cost.shape), r.cost), case
        assert (r.cost > 0).any()
        # the tally changes no other output of the tracking launch, nor what a launch without tracking computes
        tr, _ = shared_launch(g, shape, widths, conds, refs, z, track=True)
        plain, _ = shared_launch(g, shape, widths, conds, refs, z)
        assert torch.equal(tr.track, r.track) and torch.equal(tr.returns, r.returns) and torch.equal(tr.steps, r.steps)
        assert torch.equal(plain.returns, r.returns) and torch.equal(plain.steps, r.steps)


def test_cost_tally_survives_the_time_split_schedule():
    """300 actors x 11 envs at h = 72 on 64 SMs: K1 splits trajectories between slots and hands the tally over"""
    g = ACT['serl10_pop_h72_tanh']
    np.random.seed(5)
    refs = operators.study_refs(0)
    conds = CONDS[:-2]
    small, _ = shared_launch(g, rollout.actor_shape(72), None, conds, refs, None, track=True, cost=True)
    big, _ = shared_launch(np.tile(g, (30, 1)), rollout.actor_shape(72), None, conds, refs, None, track=True, cost=True, sm_limit=64)
    assert (small.cost > 0).any()
    assert torch.equal(big.cost, small.cost.repeat(30, 1)) and torch.equal(big.track, small.track.repeat(30, 1, 1))
    assert torch.equal(big.returns, small.returns.repeat(30, 1))


def test_cost_tally_matches_the_oracle_plant_with_the_kernel_order_actor():
    """a few trajectories flown step by step on oracle/phlab.py: cost = executed steps with get_cost's flag on env.x"""
    from oracle import fast, phlab
    g = ACT['serl10_pop_h72_tanh'][:2]
    np.random.seed(5)
    refs = operators.study_refs(1)
    conds = ['nominal', 'be']
    r, codes = shared_launch(g, rollout.actor_shape(72), None, conds, refs, None, track=True, cost=True)
    lv, st = evaluation._ref_arrays(refs)
    for a in range(2):
        for j, c in enumerate(codes):
            env = phlab.CitationEnv(conds[j // len(refs)], t_max=20)
            env.smooth_w = 2.0
            obs = env.reset(lv[j % len(refs)], st[j % len(refs)])
            done, k, cost = False, 0, 0
            while not done:
                act = fast.actor_forward_kernel_order(g[a], obs[None].astype(np.float32), 72)[0]
                obs, _rew, done, info = env.step(act)
                x = info['x']
                cost += int(np.rad2deg(abs(x[4])) > 11.0 or np.rad2deg(abs(x[6])) > 0.75 * env.max_phi or x[3] < env.V0 / 3)
                k += 1
            assert k == int(r.steps[a, j]) and cost == int(r.cost[a, j]), (a, j, k, cost)


def params(hidden=72, layers=3, act='tanh', bs=10_000, batch=64, mag=0.05, seed=7):
    return types.SimpleNamespace(hidden_size=hidden, num_layers=layers, activation_actor=act, individual_bs=bs,
                                 mutation_batch_size=batch, mutation_mag=mag, seed=seed)


class Ring:
    """base/core/replay_memory.py ReplayMemory.add: the memory list in slot order and the write position"""

    def __init__(self, capacity):
        self.capacity, self.memory, self.position = capacity, [], 0

    def add(self, row):
        if len(self.memory) < self.capacity:
            self.memory.append(None)
        self.memory[self.position] = row
        self.position = (self.position + 1) % self.capacity


def restated_buffers(g, refs, capacity, T, cond='nominal'):
    """operator_runner.evaluate(save_transitions=True) per parent and trial, fed each trial's rows (the trial flown in a
    launch of its own that records it): (obs = next_obs, action, next_obs, reward, done) to the buffer, and to the critical
    buffer when the step's cost flag is set"""
    env = evaluation.condition_env(cond, 20)
    lv, st = evaluation._ref_arrays(refs[:T])
    out = []
    for i in range(g.shape[0]):
        mem, crit = Ring(capacity), Ring(capacity)
        for tr in range(T):
            r = rollout.population_rollout(t(g[i:i + 1]), rollout.actor_shape(72), t(lv), t(st), t(np.full(T, env.mode_code, np.int32)),
                                           t_max=20.0, smooth_width=2.0, replay_env=tr, fitness=False)
            for row in r.replay[0, :int(r.steps[0, tr])].cpu().numpy():
                trans = np.concatenate((row[10:17], row[7:10], row[10:17], row[17:19]))
                mem.add(trans)
                if row[19] > 0.5:
                    crit.add(trans)
        out.append((mem, crit))
    return out


def test_parent_buffers_equal_the_reference_evaluate_with_saved_transitions():
    g = ACT['serl10_pop_h72_tanh'][:3]
    T = 2
    np.random.seed(5)
    refs = operators.study_refs(T - 1)
    cap = 1500                                         # smaller than the 2 x 2001 rows a parent can store: the rings wrap
    runner = operators.OperatorRunner(params(bs=cap), 'nominal', num_trails=T - 1)
    pf = runner.validate_parents(g, refs)
    want = restated_buffers(g, refs, cap, T)
    assert (pf.steps.sum(1) > cap).any()
    for i, rings in enumerate(want):
        for bufs, ring in zip((pf.buffers, pf.critical_buffers), rings):
            n = len(ring.memory)
            assert min(int(bufs.count[i]), cap) == n and int(bufs.pos[i]) == ring.position
            if n:
                np.testing.assert_array_equal(bufs.data[i, :n].cpu().numpy(), np.stack(ring.memory))
        assert int(pf.critical_buffers.count[i]) == pf.costs[i].sum()


def per_actor_reference(genome, states, shape, activation, delta):
    """the reference's proximal_mutate (mod_neuro_evo.py:183-252) on one actor with plain autograd"""
    G = genome.clone().reshape(1, -1).requires_grad_(True)
    out = evo_prox.actor_forward_batched(G, states[None], shape, activation)[0]
    mask = evo_prox.weight_mask(shape, G.device)
    jac = []
    for i in range(3):
        (gr,) = torch.autograd.grad(out[:, i].sum(), G, retain_graph=True)
        jac.append(gr[0, mask])
    scaling = torch.sqrt(sum(j ** 2 for j in jac))
    scaling[scaling == 0] = 1.0
    scaling[scaling < 0.01] = 0.01
    new = genome.clone().detach()
    new[mask] = genome[mask] + delta / scaling
    return new


@pytest.mark.parametrize('cond,mags', [('nominal', None), ('noise', [0.02, 0.1])])
def test_children_follow_the_reference_operators_and_scores_equal_each_child_alone(cond, mags):
    from oracle import ssne
    g = ACT['serl10_pop_h72_tanh'][:3]
    N, T = 3, 2
    args = params()
    M = 1 if mags is None else len(mags)
    mag_list = [args.mutation_mag] if mags is None else mags
    shape_t = (7, 3, 72, 3)
    table, P = evo.param_table(*shape_t)
    random.seed(7); np.random.seed(7); torch.manual_seed(7)
    refs = operators.study_refs(T - 1)
    runner = operators.OperatorRunner(args, cond, num_trails=T - 1)
    state0 = (random.getstate(), np.random.get_state())
    study = runner.test_mutation(g, refs, mags)
    kids = torch.as_tensor(study.child_genomes).reshape(3, M, N, P)
    # the streams restated in test_mutation's order: np.random (sensor noise, ssne_probabilities), stdlib (mutate_inplace,
    # the mutation batches' random.sample)
    random.setstate(state0[0]); np.random.set_state(state0[1])
    h = 2001
    np_before, zc = {}, {}
    for i in range(N):
        if cond == 'noise':
            evaluation.sensor_noise_draws(T, h)
        for m in range(M):
            np_before[i, m] = np.random.get_state()          # where mutate_inplace's ssne_probabilities draw starts
            np.random.uniform(0, 1, len(table))
            for o_i in range(3):
                zc[o_i, m, i] = evaluation.sensor_noise_draws(T, h) if cond == 'noise' else None
    o = ssne.SSNE(N, shape_t)
    W = {m: g.copy() for m in range(M)}
    batches = {}
    for i in range(N):
        for m in range(M):
            np.random.set_state(np_before[i, m])
            o.mutate_inplace(W[m], i, mag_list[m])
            for kind, bufs in ((1, study.buffers), (2, None)):
                if bufs is None:
                    use_crit = min(int(study.critical_buffers.count[i]), args.individual_bs) > 1
                    bufs = study.critical_buffers if use_crit else study.buffers
                n = min(int(bufs.count[i]), bufs.capacity)
                idx = random.sample(range(n), min(args.mutation_batch_size, n))
                batches[kind, m, i] = bufs.data[i, torch.as_tensor(idx, device=DEV), :7]
    for m in range(M):
        assert np.array_equal(kids[0, m].numpy(), W[m]), m            # normal children: bit for bit
    # scores: every child alone in its own launch, on its own sensor-noise draws, gives the study's bits
    for o_i, op in enumerate(operators.OPERATORS):
        for m in range(M):
            for i in range(N):
                z = zc[o_i, m, i]
                ret, cost, nmae = runner.fly_children(t(kids[o_i, m, i].numpy()[None]), refs, None if z is None else z[None])
                assert np.array_equal(ret[0], study.child_returns[op][m, i]) and np.array_equal(cost[0], study.child_costs[op][m, i])
                assert np.array_equal(nmae[0], study.child_nmae[op][m, i])
    # statistics as test_mutation computes them
    for mag, (sr, sc) in study.by_mag.items():
        m = study.mags.index(mag)
        r1, c1 = operators.mutation_stats(study.parent_returns, study.parent_costs,
                                          {op: study.child_returns[op][m] for op in operators.OPERATORS},
                                          {op: study.child_costs[op][m] for op in operators.OPERATORS})
        for op in operators.OPERATORS:
            np.testing.assert_array_equal(sr[op], r1[op])
            np.testing.assert_array_equal(sc[op], c1[op])
    # proximal / safe: the deltas replayed from the study's generator, in its group order
    gen = torch.Generator(device=DEV)
    gen.manual_seed(args.seed + 1)
    nw = int(evo_prox.weight_mask(shape_t, DEV).sum())
    groups = {}
    for (kind, m, i), s in batches.items():
        groups.setdefault((kind, m, s.shape[0]), []).append(i)
    for (kind, m, _b), members in sorted(groups.items()):
        delta = torch.randn((len(members), nw), dtype=torch.float32, device=DEV, generator=gen) * mag_list[m]
        for k, i in enumerate(members):
            # The scaling sums each weight's gradient over the batch, and for some weights those sums cancel: two fp32
            # summation orders (a batch of actors, one actor) then differ in the perturbation's 4th digit.  So both are
            # held to the float64 restatement: the study within 4x the fp32 restatement's own distance from it.
            want32 = per_actor_reference(t(g[i]), batches[kind, m, i], shape_t, 'tanh', delta[k]).cpu().double()
            want64 = per_actor_reference(t(g[i]).cpu().double(), batches[kind, m, i].cpu().double(), shape_t, 'tanh',
                                         delta[k].cpu().double())
            err, own = (kids[kind, m, i].double() - want64).abs().max().item(), (want32 - want64).abs().max().item()
            assert err <= 4 * own + 1e-6, (kind, m, i, err, own)
            assert (want64 - t(g[i]).cpu().double()).abs().max().item() > 0.01          # the child moved
