"""Several independent SERL / TD3 trainings in one process on one GPU, each giving the bits it gives when trained alone.

With `fused_td3`, a generation's RL half is K7 (csrc/td3.cu), one thread-block cluster on a few of the GPU's SMs, and it is
most of a run's wall-clock time.  `Sweep` moves S runs forward one generation at a time: the head of every run's
generation (population rollout, SSNE epoch, exploration episode: Agent.train_head), then ONE grouped K7 launch that takes
every run's gradient steps on its own cluster (td3_fused.train_group), then every run's tail (validation, actor injection,
next front: Agent.train_tail).  The runs may differ in seed and in any `Parameters` attribute that keeps the actor's shape;
with `mixed_shapes` they may differ in actor shape too (hidden_size, num_layers, activation_actor, anywhere K7 trains):
the K7 launch then trains narrow and wide actors together.  With `per` the runs may set `per`
(prioritized experience replay): the K7 launch then trains every run with a priority tree on it and every other run
uniformly, of any shapes, together.

A SERL10 population (10 actors x 3 envs) fills a few warps for the serial latency of one 2001-step trajectory, so the
populations fly together too: every run draws its front's references at their usual place (its np.random stream advances
as it would alone) and leaves the launch to the Sweep, which then makes ONE rollout launch with per-actor env blocks
(SERL_ROLLOUT_PER_ACTOR_REFS) for each group of runs whose agent.population_key agrees (`launch_groups`), both for the
fronts the heads take and for the next generation's fronts the tails queue.  Runs of different actor shapes fall into
different launch groups; the first group's launch is queued on the current stream and every further group's on a stream
of its own, so that they run side by side.  Each run reads its slice of the result, bit for bit what its own launch
gives.  A merged launch has ONE status word: a non-finite trajectory in any run of it raises
in every run that shares it.  A run whose queued front is invalidated at its next head (its population, RL actor or
environment changed) flies its population alone.

Each run keeps its own state of the global generators the Agent draws from — stdlib `random` (the SSNE planner), legacy
`np.random` (reference signals, exploration noise, tournaments) and torch's CPU generator (actor initialisation) — and
every phase of a run runs with that state swapped in (`RNGState`).  Nothing on the fused path draws from torch's default
CUDA generator (the replay buffers, SSNE and K7 have generators of their own, seeded from the run's `seed`), but
`torch.manual_seed` also seeds it, so its state is swapped too: the caller's generators come back exactly as they were.
"""
import contextlib
import copy
import os
import random

import numpy as np
import torch

from . import evaluation, td3_fused
from .core import agent as agent_mod
from ._native import NativeError
from .rollout import INCREMENTAL_STATE_DIM, SYMMETRIC_ACTION_DIM, SYMMETRIC_STATE_DIM, actor_shape


class RNGState:
    """the states of stdlib `random`, legacy `np.random`, torch's CPU generator and, with CUDA, torch's default generator
    of the current device"""
    __slots__ = ('py', 'np', 'torch', 'cuda')

    @classmethod
    def capture(cls):
        s = cls()
        s.py, s.np, s.torch = random.getstate(), np.random.get_state(), torch.get_rng_state()
        s.cuda = torch.cuda.get_rng_state() if torch.cuda.is_available() else None
        return s

    def restore(self):
        random.setstate(self.py)
        np.random.set_state(self.np)
        torch.set_rng_state(self.torch)
        if self.cuda is not None:
            torch.cuda.set_rng_state(self.cuda)


@contextlib.contextmanager
def rng_scope(state):
    """run the block with the global generators in `state`, store their advanced state back in it, and give the caller's
    generators back exactly as they were"""
    outer = RNGState.capture()
    state.restore()
    try:
        yield
    finally:
        now = RNGState.capture()
        state.py, state.np, state.torch, state.cuda = now.py, now.np, now.torch, now.cuda
        outer.restore()


class Run:
    """one training of a sweep: its Parameters, environment, Agent, generator states and last statistics"""
    __slots__ = ('params', 'env', 'agent', 'rng', 'stats')

    @property
    def finished(self):
        return self.agent.num_frames > self.params.num_frames          # base/train.py's `while num_frames <= frames`


def launch_groups(keys):
    """the runs that share one population launch: lists of run indices with equal agent.population_key, in order of first
appearance; runs without a population (key None) are in none"""
    groups = {}
    for i, k in enumerate(keys):
        if k is not None:
            groups.setdefault(k, []).append(i)
    return list(groups.values())


def _shape(p):
    return tuple(getattr(actor_shape(p.hidden_size, p.num_layers, p.activation_actor, p.state_dim, p.action_dim), f)
                 for f in ('state_dim', 'action_dim', 'hidden', 'num_layers', 'activation'))


class Sweep:
    def __init__(self, runs, mixed_shapes=False, per=False):
        """runs: a list of (Parameters, env), each seeded and built as base/train.py:88-94 builds one run.  mixed_shapes: the
        runs' actor shapes may differ (each inside K7's domain); without it they must agree.  per: runs may set `per`
        (prioritized replay) and train beside uniform ones; without it a `per` run is refused."""
        runs = list(runs)
        if not runs:
            raise ValueError('Sweep: no runs')
        if torch.distributed.is_available() and torch.distributed.is_initialized() and torch.distributed.get_world_size() > 1:
            raise NotImplementedError('Sweep: runs on one GPU; a torch.distributed world larger than 1 is not supported')
        for i, (p, _) in enumerate(runs):
            if p.state_dim == INCREMENTAL_STATE_DIM:
                raise ValueError('Sweep: run %d flies incremental control (state_dim 10), which fused_td3 (K7) does not train' % i)
            if (p.state_dim, p.action_dim) == (SYMMETRIC_STATE_DIM, SYMMETRIC_ACTION_DIM):
                raise ValueError('Sweep: run %d flies symmetric control (state_dim 2, action_dim 1), which fused_td3 (K7) does not train' % i)
            if getattr(p, 'per', False) and not per:
                raise ValueError('Sweep: run %d sets per (prioritized experience replay), which the grouped K7 launch does not '
                                 'train; build the Sweep with per=True, or train it alone with Agent' % i)
            if not getattr(p, 'fused_td3', False):
                raise ValueError('Sweep: run %d does not set fused_td3 (the sweep trains every RL half in one K7 launch)' % i)
            if mixed_shapes:
                try:
                    td3_fused.state_floats(actor_shape(p.hidden_size, p.num_layers, p.activation_actor, p.state_dim, p.action_dim))
                except NativeError as e:
                    raise ValueError('Sweep: run %d has actor shape %s, which K7 does not train (%s)' % (i, _shape(p), e)) from None
            elif _shape(p) != _shape(runs[0][0]):
                raise ValueError('Sweep: run %d has actor shape %s, run 0 has %s (one K7 launch trains one shape)'
                                 % (i, _shape(p), _shape(runs[0][0])))
        self.mixed_shapes = bool(mixed_shapes)
        self.per = bool(per)
        self._streams = []             # the population launch groups' streams after the first, created once and kept
        self.runs = []
        outer = RNGState.capture()
        try:
            for p, env in runs:
                r = Run()
                r.params, r.env, r.stats = p, env, None
                env.seed(p.seed)
                torch.manual_seed(p.seed)
                np.random.seed(p.seed)
                random.seed(p.seed)
                r.agent = agent_mod.Agent(p, env)
                r.agent.defer_population = True
                r.rng = RNGState.capture()
                self.runs.append(r)
        finally:
            outer.restore()

    @property
    def finished(self):
        return all(r.finished for r in self.runs)

    def train(self):
        """one generation of every run that has not reached its `frames`: returns one statistics dict per run (Agent.train's),
        None for a finished run"""
        live = [r for r in self.runs if not r.finished]
        for r in live:
            with rng_scope(r.rng):
                r.agent.take_front()
        self._launch_populations([(r, r.agent._front) for r in live])
        for r in live:
            with rng_scope(r.rng):
                r.agent.train_head()
        plans = []
        for r in live:
            with rng_scope(r.rng):
                plans.append(r.agent.plan_rl_fused(r.agent.gen_frames))
        group = [(r, n) for r, n in zip(live, plans) if n]
        # the heads appended their rows (and, with per, inserted them into the runs' trees) on the current stream, after
        # joining the population streams: the K7 launch, queued on it too, sees every run's rows and tree
        launches = td3_fused.train_group([r.agent.rl_agent for r, _ in group], [r.agent.replay_buffer for r, _ in group],
                                         [n for _, n in group], [r.agent.rl_iteration + 1 for r, _ in group],
                                         [r.agent.args.use_champion_target for r, _ in group], mixed_shapes=self.mixed_shapes,
                                         prioritized=self.per)
        losses = dict(zip((id(r) for r, _ in group), td3_fused.group_losses(launches)))
        for r, n in zip(live, plans):
            with rng_scope(r.rng):
                r.stats = r.agent.train_tail(r.agent.finish_rl_fused(n, losses.get(id(r))))
        self._launch_populations([(r, r.agent._prefetched) for r in live])
        live_ids = set(id(r) for r in live)
        return [r.stats if id(r) in live_ids else None for r in self.runs]

    def _launch_populations(self, fronts):
        """one rollout launch per launch group for the fronts [(run, front)] whose population launch is still deferred: the
        first group's on the current stream, each further group's on a stream of its own, so that launches of different
        shapes do not queue behind each other"""
        pending = [(r, f) for r, f in fronts if f is not None and f.pop_draws is not None]
        keys = [agent_mod.population_key(r.params, r.env) for r, _ in pending]
        groups = launch_groups(keys)
        if not groups:
            return
        dev = pending[0][0].agent.device
        cur = torch.cuda.current_stream(dev)
        while len(self._streams) < len(groups) - 1:
            self._streams.append(torch.cuda.Stream(dev))
        side = self._streams[:len(groups) - 1]
        for s in side:                 # fork before anything is queued: the genomes are written on the current stream
            s.wait_stream(cur)
        for g, s in zip(groups, [None] + side):
            with torch.cuda.stream(s) if s is not None else contextlib.nullcontext():
                agent_mod.launch_population_group([(pending[i][0].agent, pending[i][1]) for i in g])
        # join before anything reads a front: SSNE rewrites the genomes in place on the current stream, and the caching
        # allocator hands the side streams' blocks out again once their tensors are freed
        for s in side:
            cur.wait_stream(s)

    def evaluate(self, conditions, refs, num_trails=1):
        """evaluation.evaluate_population of every run's population on `conditions` with the references `refs`: the
        populations of one actor shape stack into one call, one call per shape in order of first appearance (runs in run
        order within it), so the sensor-noise draws continue on the np.random stream in that order.  Returns one
        PopulationEval per run (None for a run without a population)."""
        out = [None] * len(self.runs)
        shapes = [_shape(r.params) if len(r.agent.pop) else None for r in self.runs]
        for g in launch_groups(shapes):
            res = evaluation.evaluate_population(torch.cat([self.runs[i].agent.pop.genomes for i in g]), self.runs[g[0]].agent.shape,
                                                 conditions, refs, num_trails)
            for i, part in zip(g, res.split([self.runs[i].agent.pop.genomes.shape[0] for i in g])):
                out[i] = part
        return out

    def save_checkpoint(self, folder):
        """checkpoint every run between two train() calls: run i's Agent, generator states and last statistics go to
        folder/run<i>.pt (serl_b200/checkpoint.py), and folder/manifest.json names the run count and each run's identifying
        Parameters.  A finished run is saved as it stands and stays finished."""
        from . import checkpoint
        os.makedirs(folder, exist_ok=True)
        for i, r in enumerate(self.runs):
            checkpoint.save(r.agent, os.path.join(folder, 'run%d.pt' % i), rng=r.rng, extra={'stats': r.stats})
        manifest = {'format': checkpoint.FORMAT, 'version': checkpoint.VERSION, 'runs': len(self.runs),
                    'params': [checkpoint.identity(r.params) for r in self.runs]}
        checkpoint.write(manifest, os.path.join(folder, 'manifest.json'), json_doc=True)

    def load_checkpoint(self, folder):
        """continue the sweep saved in `folder` in this Sweep, built from the same runs (Parameters and envs, in the same
        order; `frames` may differ).  Every run is checked before any is written.  The runs' queued fronts are re-launched
        and their populations launched in their launch groups, as the saved sweep's last train() left them."""
        from . import checkpoint
        manifest = checkpoint.read_json(os.path.join(folder, 'manifest.json'))
        if manifest.get('runs') != len(self.runs):
            raise ValueError('Sweep.load_checkpoint: %s holds %s runs, this sweep has %d' % (folder, manifest.get('runs'), len(self.runs)))
        cks = []
        for i, r in enumerate(self.runs):
            ck = checkpoint.read(os.path.join(folder, 'run%d.pt' % i))
            try:
                checkpoint.check(ck, r.params)
            except ValueError as e:
                raise ValueError('Sweep.load_checkpoint: run %d: %s' % (i, e)) from None
            cks.append(ck)
        for r, ck in zip(self.runs, cks):
            r.stats = checkpoint.apply(r.agent, ck, rng=r.rng)['stats']
        self._launch_populations([(r, r.agent._prefetched) for r in self.runs])

    def save_agent(self, folder=None):
        """Agent.save_agent of every run into its own folder <folder or the run's save_foldername>/run<i>"""
        for i, r in enumerate(self.runs):
            p = copy.copy(r.params)
            p.save_foldername = os.path.join(folder or r.params.save_foldername, 'run%d' % i) + '/'
            os.makedirs(p.save_foldername, exist_ok=True)
            elite = r.stats['elite_index'] if r.stats is not None else None
            r.agent.save_agent(p, elite)
