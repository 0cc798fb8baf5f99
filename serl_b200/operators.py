"""The mutation-operator study of base/evaluate_operators.py and base/core/operator_runner.py on the device, for a whole
population at once.

For every actor of a trained population the reference flies the parent over num_trails + 1 evaluation episodes (t_max =
20 s) and stores those transitions in the parent's own buffers; it then makes one normal, one proximal and one safe child
(clone + mutate_inplace / proximal_mutate / safe_mutate), flies each child on the same references, and reports per
operator the relative change in return (1 - child / parent) and in safety cost (child / parent - 1).  Here:

- the parents fly in ONE rollout launch with per-actor env blocks, one block per (parent, trial), so that every
  trajectory exports its replay rows (K1 records one env per actor); the rows go to the per-actor device rings
  (replay_memory.PopulationBuffers) trial by trial, and the parents' cost is the sum of the rows' cost column;
- the children are mutated in one batch per operator (K5 for the normal children; evo_prox.proximal_mutate_batched for
  the proximal and safe ones);
- all 3 * N * |mags| children fly in ONE tracking launch that also counts every trajectory's cost steps
  (rollout.population_rollout(track=True, cost=True)), and their nMAE comes with it.
"""
import random
from collections import namedtuple

import numpy as np
import torch

from . import evaluation, evo, evo_prox, rollout
from .core.replay_memory import PopulationBuffers

OPERATORS = ('Normal', 'Proximal', 'Safe')
T_MAX = 20                   # base/evaluate_operators.py:46: the study's episode length [s]

ParentFlight = namedtuple('ParentFlight', ('returns', 'costs', 'steps', 'buffers', 'critical_buffers'))


def study_refs(num_trails, t_max=T_MAX):
    """base/evaluate_operators.py:85-104: num_trails random (theta, phi) pairs from gen_refs (smooth width t_max // 10),
    then the fixed base sequences as trial num_trails — evaluation.eval_refs at t_max = 20 s"""
    return evaluation.eval_refs(num_trails, t_max)


def mutation_stats(parent_returns, parent_costs, child_returns, child_costs):
    """the arithmetic of OperatorRunner.test_mutation (operator_runner.py:122-206) on the per-trial values of N models:
    parent_* [N, T], child_*[op] [N, T] for op in OPERATORS.  Each model's trial average is broadcast over its T columns,
    eff = 1 - child / parent and cost = child / parent - 1, flattened model-major.  A parent with zero cost gives what numpy
    gives for x / 0 (inf, or nan for 0 / 0), as in the reference.  Returns (stats_reward, stats_cost)."""
    def avg(v):
        v = np.asarray(v, dtype=np.float64)
        return np.broadcast_to(np.average(v, axis=1)[:, None], v.shape)
    pr, pc = avg(parent_returns), avg(parent_costs)
    with np.errstate(divide='ignore', invalid='ignore'):
        stats_reward = {op: (1 - avg(child_returns[op]) / pr).flatten() for op in OPERATORS}
        stats_cost = {op: (avg(child_costs[op]) / pc - 1).flatten() for op in OPERATORS}
    return stats_reward, stats_cost


def _toml_float(v):
    # toml.TomlNumpyEncoder's _dump_float: "{}".format(v) with the exponent's leading zero dropped
    return '{}'.format(np.float64(v)).replace('e+0', 'e+').replace('e-0', 'e-')


def mutation_stats_toml(stats_reward, stats_cost):
    """the text base/evaluate_operators.py:145-156 writes to mutation_stats.toml: toml.dump of {'stats_cost': ...}, a blank
    line, toml.dump of {'stats_reward': ...}; arrays as the toml package writes them ('[ a, b,]')"""
    def section(name, d):
        return f'[{name}]\n' + ''.join(f'{k} = [' + ''.join(f' {_toml_float(x)},' for x in np.asarray(v).ravel()) + ']\n'
                                       for k, v in d.items())
    return section('stats_cost', stats_cost) + '\n' + section('stats_reward', stats_reward)


class MutationStudy:
    """what OperatorRunner.test_mutation returns.  Unpacks as (stats_reward, stats_cost), the reference's return value.

    stats_reward / stats_cost: {op: [M * N * T]} over the magnitudes in order (M = 1: exactly the reference's arrays);
    by_mag: {mag: (stats_reward, stats_cost)} per magnitude; parent_returns / parent_costs [N, T] per trial;
    child_returns / child_costs / child_nmae: {op: [M, N, T]} per trial; child_genomes [3, M, N, P] (operator-major)."""

    def __init__(self, mags, parent, child_returns, child_costs, child_nmae, child_genomes):
        self.mags = list(mags)
        self.parent_returns, self.parent_costs = parent.returns, parent.costs
        self.buffers, self.critical_buffers = parent.buffers, parent.critical_buffers
        self.child_returns, self.child_costs, self.child_nmae = child_returns, child_costs, child_nmae
        self.child_genomes = child_genomes
        self.by_mag = {}
        for m, mag in enumerate(self.mags):
            self.by_mag[mag] = mutation_stats(parent.returns, parent.costs, {op: child_returns[op][m] for op in OPERATORS},
                                              {op: child_costs[op][m] for op in OPERATORS})
        per = list(self.by_mag.values())
        self.stats_reward = {op: np.concatenate([sr[op] for sr, _ in per]) for op in OPERATORS}
        self.stats_cost = {op: np.concatenate([sc[op] for _, sc in per]) for op in OPERATORS}

    def __iter__(self):
        return iter((self.stats_reward, self.stats_cost))


class OperatorRunner:
    """base/core/operator_runner.py OperatorRunner over a [N, P] genome matrix (fp32, parameters() order) of the uniform
    actor `args` describes (hidden_size, num_layers, activation_actor), on one flight condition ('nominal', 'be', ...).

    Draws.  The legacy np.random stream and the stdlib random stream are consumed as test_mutation consumes them for
    mags = [args.mutation_mag], model by model: the sensor-noise draws of the episodes (noisy conditions; the full
    horizon + 1 steps of every episode, as evaluation.evaluate_population draws them), the normal mutation's
    ssne_probabilities and point mutations (mutate_inplace, replayed through evo.plan_mutate_inplace for K5, with its
    exclusive index bound, evo.py), and the mutation batches' random.sample over the parent's buffer, whose row order is
    the reference's ReplayMemory order.  The proximal / safe perturbations delta ~ N(0, mag) come from a torch generator on
    the device seeded with args.seed + 1 (the reference draws them from torch's global CPU generator), so proximal and safe
    children match the reference given the same deltas only.  With several magnitudes every model takes the three operators
    for each magnitude in turn."""

    def __init__(self, args, condition='nominal', num_trails=0, device=None):
        if getattr(args, 'state_dim', None) == rollout.INCREMENTAL_STATE_DIM:
            raise ValueError('OperatorRunner: the operator study flies absolute control only, not incremental control')
        if (getattr(args, 'state_dim', None), getattr(args, 'action_dim', None)) == (rollout.SYMMETRIC_STATE_DIM, rollout.SYMMETRIC_ACTION_DIM):
            raise ValueError('OperatorRunner: the operator study flies attitude control only, not symmetric control')
        self.args = args
        self.num_trails = int(num_trails)
        self.device = device or torch.device('cuda', torch.cuda.current_device())
        self.env = evaluation.condition_env(condition, T_MAX)
        self.shape = rollout.actor_shape(args.hidden_size, args.num_layers, args.activation_actor)
        self.shape_tuple = (7, 3, int(args.hidden_size), int(args.num_layers))
        self.horizon = int(round(self.env.t_max / self.env.dt)) + 1
        self.gen = None

    def _noise(self, n_traj):
        return evaluation.sensor_noise_draws(n_traj, self.horizon) if self.env.sensor_noise else None

    def validate_parents(self, genomes, user_refs_lst, noise=None):
        """validate_agent(..., save_transitions=True) of every parent in one launch of per-actor env blocks, one block per
        (parent, trial).  The stored transition is (obs, action, next_obs, reward, done) with obs already overwritten by
        the step's result (operator_runner.py:52-58): its state column is the next observation.  Rows with the cost flag
        also go to the critical buffer.  Returns ParentFlight: returns, costs, steps [N, T] and the filled rings
        (PopulationBuffers of capacity args.individual_bs).  noise: optional [N, T, horizon + 1, 7] sensor-noise draws."""
        g = torch.as_tensor(genomes, device=self.device).reshape(len(genomes), -1).contiguous()
        N, T = g.shape[0], self.num_trails + 1
        refs = user_refs_lst[:T]
        lv, st = evaluation._ref_arrays(refs)
        dev, h = self.device, self.horizon
        weights = g.repeat_interleave(T, dim=0).contiguous()                  # row i * T + t: parent i, trial t
        levels = torch.as_tensor(np.tile(lv, (N, 1, 1)).reshape(N * T, 1, 2, 6), device=dev)
        starts = torch.as_tensor(np.tile(st, (N, 1, 1)).reshape(N * T, 1, 2, 6), device=dev)
        md = torch.full((N * T, 1), self.env.mode_code, dtype=torch.int32, device=dev)
        sn = None if noise is None else torch.as_tensor(np.ascontiguousarray(noise.reshape(N * T, 1, h + 1, 7)), device=dev)
        r = rollout.population_rollout(weights, self.shape, levels, starts, md, horizon=h, t_max=float(self.env.t_max),
                                       smooth_width=float(refs[0][0].smooth_width), replay_env=0, fitness=False, sensor_noise=sn,
                                       gust=rollout.mode_gust(self.env.mode_code))
        r.check()
        steps = r.steps.reshape(N, T)
        rows = r.replay.reshape(N, T, h, rollout.REPLAY_COLS).clone()
        rows[..., 0:7] = rows[..., 10:17]                                     # state = next_obs (operator_runner.py:52-57)
        live = torch.arange(h, device=dev)[None, None, :] < steps[..., None]
        crit = live & (rows[..., rollout.REPLAY_COST] > 0.5)
        costs = crit.sum(-1)
        buffers = PopulationBuffers(N, self.args.individual_bs, dev)
        critical = PopulationBuffers(N, self.args.individual_bs, dev)
        actors = torch.arange(N, device=dev)
        for t in range(T):                                                    # trial by trial, as validate_agent fills them
            buffers.append(actors, rows[:, t], live[:, t])
            critical.append(actors, rows[:, t], crit[:, t])
        return ParentFlight(r.returns.reshape(N, T).cpu().numpy(), costs.cpu().numpy(), steps.cpu().numpy(), buffers, critical)

    def _batch_states(self, bufs, actor):
        """buffer.sample(min(mutation_batch_size, len(buffer)))'s states: random.sample over the ring in slot order (the
        reference's ReplayMemory.memory order)"""
        n = int(min(int(bufs.count[actor]), bufs.capacity))
        idx = random.sample(range(n), min(int(self.args.mutation_batch_size), n))
        return bufs.data[actor, torch.as_tensor(idx, dtype=torch.int64, device=self.device), :7]

    def test_mutation(self, genomes, user_eval_refs, mags=None):
        """OperatorRunner.test_mutation for every model of `genomes` [N, P] and every magnitude of `mags` (None:
        [args.mutation_mag], the reference's study).  Returns a MutationStudy; `stats_reward, stats_cost = ...` unpacks it."""
        mags = [float(self.args.mutation_mag)] if mags is None else [float(m) for m in mags]
        g = torch.as_tensor(np.asarray(genomes, dtype=np.float32) if not torch.is_tensor(genomes) else genomes, device=self.device)
        g = g.reshape(g.shape[0], -1).contiguous()
        N, M, T, h = g.shape[0], len(mags), self.num_trails + 1, self.horizon
        table, P = evo.param_table(*self.shape_tuple)
        assert P == g.shape[1], (P, g.shape)
        # the legacy np.random stream in test_mutation's order: parent episodes, then per magnitude the normal mutation's
        # ssne_probabilities and the three children's episodes
        zp, probs = [], {}
        zc = np.zeros((3, M, N, T, h + 1, 7), np.float32) if self.env.sensor_noise else None
        for i in range(N):
            zp.append(self._noise(T))
            for m in range(M):
                probs[i, m] = np.random.uniform(0, 1, len(table)) * 2
                for o in range(3):
                    z = self._noise(T)
                    if z is not None:
                        zc[o, m, i] = z
        parent = self.validate_parents(g, user_eval_refs, None if zc is None else np.stack(zp))
        # children: clones of their parent, in [operator, magnitude, model] order
        children = g.repeat(3 * M, 1).reshape(3, M, N, P).contiguous()
        flat = children.view(3 * M * N, P)
        plans = [([], [], [], []) for _ in range(M)]
        prox = {}                                              # (operator, magnitude, batch size) -> [(row, states)]
        for i in range(N):                                     # the stdlib random stream in test_mutation's order
            for m in range(M):
                evo.plan_mutate_inplace(table, (0 * M + m) * N + i, probs[i, m], *plans[m])
                s = self._batch_states(parent.buffers, i)
                prox.setdefault((1, m, s.shape[0]), []).append(((1 * M + m) * N + i, s))
                use_crit = int(min(int(parent.critical_buffers.count[i]), parent.critical_buffers.capacity)) > 1
                s = self._batch_states(parent.critical_buffers if use_crit else parent.buffers, i)
                prox.setdefault((2, m, s.shape[0]), []).append(((2 * M + m) * N + i, s))
        for m, mag in enumerate(mags):
            plan = evo.EvoPlan()
            plan.clone_waves, plan.cross_waves = [], []
            plan.mut_seg, plan.mut_off, plan.mut_kind, plan.mut_z = evo.mutation_arrays(*plans[m])
            evo.apply_plan(flat, plan, mag, phase='mut')
        if self.gen is None:
            self.gen = torch.Generator(device=self.device)
            self.gen.manual_seed(int(getattr(self.args, 'seed', 7)) + 1)
        for (o, m, _b), items in sorted(prox.items()):
            rows = [r for r, _ in items]
            states = torch.stack([s for _, s in items])
            evo_prox.proximal_mutate_batched(flat, rows, states, self.shape_tuple, self.args.activation_actor, mags[m],
                                             generator=self.gen)
        ret, cost, nmae = self.fly_children(flat, user_eval_refs, None if zc is None else zc.reshape(3 * M * N, T, h + 1, 7))
        shape = (3, M, N, T)
        ret, cost, nmae = ret.reshape(shape), cost.reshape(shape), nmae.reshape(shape)
        return MutationStudy(mags, parent, {op: ret[o] for o, op in enumerate(OPERATORS)},
                             {op: cost[o] for o, op in enumerate(OPERATORS)}, {op: nmae[o] for o, op in enumerate(OPERATORS)},
                             children.cpu().numpy())

    def fly_children(self, genomes, user_refs_lst, noise=None):
        """validate_agent of every genome [n, P] on the shared references in one tracking launch that also counts the cost
        steps: per trial returns [n, T] (f64), costs [n, T] (int) and nMAE [n, T].  noise: optional [n, T, horizon + 1, 7]."""
        T = self.num_trails + 1
        refs = user_refs_lst[:T]
        lv, st = evaluation._ref_arrays(refs)
        dev, h = self.device, self.horizon
        md = torch.full((T,), self.env.mode_code, dtype=torch.int32, device=dev)
        sn = None if noise is None else torch.as_tensor(np.ascontiguousarray(noise), device=dev)
        r = rollout.population_rollout(genomes.contiguous(), self.shape, torch.as_tensor(lv, device=dev), torch.as_tensor(st, device=dev),
                                       md, horizon=h, t_max=float(self.env.t_max), smooth_width=float(refs[0][0].smooth_width),
                                       fitness=False, sensor_noise=sn, gust=rollout.mode_gust(self.env.mode_code), track=True, cost=True)
        r.check()
        steps = r.steps.cpu().numpy()
        return r.returns.cpu().numpy(), r.cost.cpu().numpy(), evaluation.nmae_from_track(r.track.cpu().numpy(), steps)
