"""Mirror of base/core/agent.py (Agent :13-352): same constructor, evaluate(), train(), validate_agent(), save_agent() and
stats keys, with the per-generation fitness hot path on the GPU:

  * the population loop `for net in pop: for i in range(num_evals): evaluate(net)` (:234-241) is ONE fused rollout launch
    over pop x num_envs trajectories (serl_b200/rollout.py, csrc/rollout.cu), sharded over ranks when torch.distributed
    is initialised (serl_b200/engine.py);
  * validate_agent (:188-209) flies its 5 episodes as ONE launch; the champion's validation (:255-258) runs on a side
    stream while SSNE.epoch works on the main stream (a single 2001-step trajectory is ~0.15 s of serial latency however
    few of them there are — the one part of a generation that cannot be hidden, since the champion is only known once the
    population has been ranked);
  * the transitions of the stored evaluation (:101-112, `store_transition=(i == num_evals-1)`) are written by the kernel
    (K1 replay rows) and appended on the device to the shared replay buffer and the per-actor buffers — no traced
    re-flight, no per-actor host loop;
  * the RL exploration episode (:267-268) — and, when no gradient step can change the RL actor this generation
    (`frac_frames_train == 0`, i.e. -test_ea), the RL validation episodes (:273-275) — are launched on a side stream BEFORE
    the population kernel, which leaves them two SMs (`sm_limit`), so they cost no wall-clock time;
  * `self.evolver.epoch` runs on the device-resident genomes (core/mod_neuro_evo.py -> serl_b200/evo.py).

Documented deviations from the reference (DESIGN.md): the conditions at agent.py:45,228 are read as intended
(`if self.pop`), save_agent's `isEmpty()` works; by default all actors of a generation see the SAME num_envs reference
signals (fair ranking) — `independent_references` gives every episode of every actor its own draw, as the reference does;
every trajectory starts from a fresh env (zero stale error); TD3 samples its batches with a device generator instead of
stdlib `random` (so the SSNE planner's stream does not depend on buffer sizes).
"""
import os
import time
from typing import Dict

import numpy as np
import torch

from . import mod_utils, replay_memory, td3
from . import mod_neuro_evo as utils_ne
from .utils import Episode, calc_smoothness
from .. import engine, refsig, rollout
from ..population import PopulationList


class _Flight:
    """an asynchronous launch of n episodes of ONE actor (result tensors stay on the device until collected)."""
    __slots__ = ('r', 'levels', 'starts', 'n', 'noise_state', 'stream', 'event', 'keep')


class _Generation:
    """what train_head hands train_tail: the population's statistics and the validation flights in the air"""
    __slots__ = ('best_train_fitness', 'worst_train_fitness', 'population_avg', 'sm', 'sm_sd', 'elite_index', 'ep_len_avg',
                 'ep_len_sd', 'pop_fitness', 'f_rlval', 'f_champ')


class _Front:
    """the launches a generation starts with: RL exploration / validation flights, speculative champion validations, the
    population rollout — and the signature of what they read.  `pop_draws` holds the population's reference draws while
    its launch is deferred (launch_population_group), `pop` the launched rollout, `draws` the draws either way."""
    __slots__ = ('signature', 'f_explore', 'f_rlval', 'spec', 'val_draws', 'pop', 'pop_draws', 'draws', 'sm_limit')


class _PopDraws:
    """the population's reference draws of one generation (host f64): levels / starts [n_envs, 2, 6] shared by every actor,
    or [pop, n_envs, 2, 6] with independent_references"""
    __slots__ = ('levels', 'starts')


def population_draws(env, pop, n_envs, independent):
    """the reference signals of a generation's population evaluation, drawn from the global np.random stream.
    independent=False: n_envs draws that every actor flies (fair ranking).  independent=True: the reference's
    `for net in pop: for i in range(num_evals): evaluate(net)` (base/core/agent.py:234-241), whose every reset() draws
    anew — pop x n_envs draws, actor by actor, evaluation by evaluation.  Returns the list of (levels, starts) in draw order."""
    return [env.draw_reference() for _ in range(pop * n_envs if independent else n_envs)]


class Agent:
    def __init__(self, args, environment):
        self.args = args
        self.env = environment
        if bool(getattr(environment, 'incremental', False)) != (args.state_dim == rollout.INCREMENTAL_STATE_DIM):
            raise ValueError('Agent: args.state_dim = %s does not match the env: the observation of incremental control has 10 entries, '
                             'that of absolute control 7' % args.state_dim)
        n_actions = int(getattr(environment, 'n_actions', 3))
        if args.action_dim != n_actions:
            raise ValueError('Agent: args.action_dim = %s does not match the env, which takes %d actions (symmetric control: the elevator '
                             'alone, attitude control: 3)' % (args.action_dim, n_actions))
        if bool(getattr(environment, 'symmetric', False)) and args.state_dim != rollout.SYMMETRIC_STATE_DIM:
            raise ValueError('Agent: args.state_dim = %s does not match the env: the observation of symmetric control has 2 entries'
                             % args.state_dim)
        if not torch.cuda.is_available():
            from .._native import NativeError
            raise NativeError('serl_b200.Agent needs a CUDA device: the rollout / evolution engine has no CPU fallback')
        self.device = torch.device('cuda', torch.cuda.current_device())
        self.pop = PopulationList(args, self.device) if args.pop_size else []
        if getattr(args, 'fused_td3', False):
            from ..td3_fused import FusedTD3
            self.rl_agent = FusedTD3(args)
        else:
            self.rl_agent = td3.TD3(args)
        if getattr(args, 'per', False):
            # the reference's agent.py:30-32 (alpha 0.6 and beta_start 0.4 are the buffer's defaults there too)
            self.replay_buffer = replay_memory.DevicePrioritizedReplayMemory(
                args.buffer_size, self.device, seed=int(getattr(args, 'seed', 7)), state_dim=args.state_dim,
                action_dim=args.action_dim, beta_frames=args.num_frames)
        else:
            self.replay_buffer = replay_memory.DeviceReplayMemory(args.buffer_size, self.device, seed=int(getattr(args, 'seed', 7)),
                                                                  state_dim=args.state_dim, action_dim=args.action_dim)
        self.noise_process = mod_utils.GaussianNoise(args.action_dim, sd=args.noise_sd)
        if len(self.pop):
            self.evolver = utils_ne.SSNE(self.args, self.rl_agent.critic, self.evaluate)
        self.shape = rollout.actor_shape(args.hidden_size, args.num_layers, args.activation_actor, args.state_dim, args.action_dim)
        self.validation_tests = 5
        self.num_episodes = 0
        self.num_frames = 0
        self.iterations = 0
        self.gen_frames = None
        self.rl_history = None
        self.rl_iteration = 0
        self.champion = None
        self.champion_actor = None
        self.champion_history = None
        self.store_population_transitions = stores_population_transitions(args)
        # single-actor flights run next to the population rollout, each on its own high-priority stream and spare SM
        self._side, self._side2, self._champ = (torch.cuda.Stream(self.device, priority=-1) for _ in range(3))
        # launch the next generation's rollouts at the end of train() (see there); False = strictly one generation per call
        self.prefetch_generation = bool(getattr(args, 'prefetch_generation', True))
        self._prefetched = None
        # the fronts this Agent launches leave their population rollout to the caller (Sweep: launch_population_group)
        self.defer_population = False
        self._front = None
        self._front_prefetched = False
        # speculative validation of last generation's elites hides the champion's validation latency INSIDE a generation;
        # with the next generation's front launched ahead it is hidden anyway, and the spare SMs go to the population
        self.speculative_validations = int(getattr(args, 'speculative_validations', 0 if self.prefetch_generation else 3))
        self._spec_streams = [torch.cuda.Stream(self.device, priority=-1) for _ in range(self.speculative_validations)]
        self.spec_hits = self.spec_tries = 0
        self.timing = {}
        self._t_prev = 0.0
        self._gen = None

    # ------------------------------------------------------------------------------------------------ episodes
    def _genome_of(self, agent):
        idx = getattr(agent, 'index', None)
        if idx is not None and len(self.pop) and self.pop[idx] is agent:
            return self.pop.genomes[idx:idx + 1]
        return agent.actor.flat().to(self.device).reshape(1, -1).contiguous()

    def _final_time(self, n):
        t = 0.
        for _ in range(n):
            t += self.env.dt
        return t

    def _horizon(self):
        return int(round(self.env.t_max / self.env.dt)) + 1

    def _eval_kw(self):
        env = self.env
        sym = rollout.is_symmetric(self.shape)
        kw = {} if env.t_max == 20 else {'t_max': float(env.t_max), 'smooth_width': refsig.widths(env.t_max, sym)[1]}
        return dict(kw, gust=rollout.mode_gust(env.mode_code))

    def _fly(self, agent, n, is_action_noise=False, store_transition=False, trace=False, stream=None, copy_genome=False, draws=None,
             noise_state=None) -> _Flight:
        """launch n episodes of one actor (fresh reference signals each, or the given `draws`) without waiting for them.  The
        action noise is drawn from the global np.random stream, or from the given legacy state `noise_state` (a flight
        re-launched from a checkpoint), which leaves the global stream untouched."""
        env = self.env
        draws = draws if draws is not None else [env.draw_reference() for _ in range(n)]
        f = _Flight()
        f.levels, f.starts, f.n = [d[0] for d in draws], [d[1] for d in draws], n
        f.noise_state = None
        horizon = self._horizon()
        noise_host = None
        if is_action_noise:
            # one np.random.randn(action_dim) per executed step (agent.py:90-93): draw a full horizon, rewind the global stream to
            # "exactly the steps that ran" once the episode length is known (collect)
            assert n == 1
            A = self.shape.action_dim
            if noise_state is None:
                f.noise_state = np.random.get_state()
                z = np.random.randn(horizon, A)
            else:
                f.noise_state = noise_state
                rs = np.random.RandomState()
                rs.set_state(noise_state)
                z = rs.randn(horizon, A)
            noise_host = np.clip(self.args.noise_sd * z, -self.args.noise_clip, self.args.noise_clip).astype(np.float32).reshape(1, 1, -1, A)
        f.stream = stream
        ctx = torch.cuda.stream(stream) if stream is not None else _null()
        pre = self._genome_of(agent).clone() if copy_genome else None        # copied on the main stream, before later edits
        if stream is not None:
            stream.wait_stream(torch.cuda.current_stream(self.device))        # genomes / weights written on the main stream
        with ctx:
            genome = pre if pre is not None else self._genome_of(agent)
            if stream is not None:
                genome.record_stream(stream)
            # pinned staging + non_blocking: a pageable host->device copy would wait for the kernels queued on this stream
            lv = _to_device(np.stack(f.levels), self.device)
            st = _to_device(np.stack(f.starts), self.device)
            md = torch.full((n,), env.mode_code, dtype=torch.int32, device=self.device)
            noise = _to_device(noise_host, self.device) if noise_host is not None else None
            f.r = rollout.population_rollout(genome, self.shape, lv, st, md, trace=trace, action_noise=noise, horizon=horizon,
                                             actions=True, replay_env=0 if store_transition else None, **self._eval_kw())
            f.r.smoothness = rollout.smoothness(f.r.actions, f.r.steps)
            f.event = torch.cuda.Event()
            f.event.record()
            f.keep = (genome, lv, st, md, noise)      # inputs stay alive until the flight is collected
        return f

    def _store_rows(self, agent, rows, n):
        """append the n transitions of one stored episode (device rows) to the shared and the agent's own buffers."""
        rows = rows[:n]
        self.replay_buffer.add_rows(rows)
        agent.buffer.add_rows(rows)
        crit = rows[rows[:, rollout.transition_cols(self.shape.state_dim, self.shape.action_dim)] > 0.5]
        if crit.shape[0]:
            agent.critical_buffer.add_rows(crit)
        self.num_frames += n
        self.gen_frames += n
        self.num_episodes += 1

    def _collect(self, agent, f: _Flight, store_transition=False, want_history=False):
        """wait for a flight and rebuild the reference's per-episode records: list of Episode."""
        f.event.synchronize()
        # read the results back on the flight's own stream: the current stream may already be running the next
        # generation's population rollout, and a copy queued there would wait for it
        with (torch.cuda.stream(f.stream) if f.stream is not None else _null()):
            f.r.check()
            steps = f.r.steps[0].cpu().numpy()
            returns = f.r.returns[0].cpu().numpy()
            sm = f.r.smoothness[0].cpu().numpy()
            hist = {}
            if f.r.trace is not None and (want_history or f.n == 1):
                hist = {e: f.r.trace[0, e, :int(steps[e])].cpu().numpy() for e in range(f.n)}
            elif want_history:
                hist = {e: f.r.actions[0, e, :int(steps[e])].cpu().numpy().astype(np.float64) for e in range(f.n)}
        if f.noise_state is not None:
            np.random.set_state(f.noise_state)
            np.random.randn(int(steps[0]), self.shape.action_dim)
        if store_transition:
            if f.stream is not None:
                f.r.replay.record_stream(torch.cuda.current_stream(self.device))     # read below by kernels of this stream
            self._store_rows(agent, f.r.replay[0], int(steps[0]))
        env = self.env
        sym = rollout.is_symmetric(self.shape)
        # symmetric control keeps the env's constant trim (envs/phlabenv.py:194, 313)
        theta_trim = env.theta_trim if sym else np.rad2deg(rollout.initial_state(rollout.mode_variant(env.mode_code))[7])
        from ..envs.phlabenv import _RefSignal
        sw = refsig.widths(env.t_max, sym)[1]
        A = self.shape.action_dim        # the deflection record is [de, 0, 0] in symmetric control; env.last_u has 1 entry
        eps = []
        for e in range(f.n):
            n = int(steps[e])
            refs = [_RefSignal(f.levels[e][0], f.starts[e][0], theta_trim, sw, env.t_max), _RefSignal(f.levels[e][1], f.starts[e][1], 0.0, sw), lambda t: 0.0]
            if sym:      # the theta reference alone, as the env's ref (envs/phlabenv.py:313)
                refs = refs[:1]
            fitness = float(returns[e]) + (float(sm[e]) if self.args.smooth_fitness else 0.0)
            state_lst, actions, rewards = [], None, None
            if f.r.trace is not None and (want_history or f.n == 1):
                tr = hist[e]
                rewards = [float(x) for x in tr[:, rollout.TRACE_R]]
                actions = tr[:, rollout.TRACE_U][:, :A].copy()
                state_lst = [] if store_transition else [tr[k, rollout.TRACE_X].copy() for k in range(n)]
            else:
                actions = hist[e][:, :A] if want_history else np.zeros((0, A))
                rewards = _ReturnOnly(float(returns[e]))
            eps.append(Episode(fitness=fitness, smoothness=float(sm[e]), length=self._final_time(n), state_history=state_lst,
                               ref_signals=refs, actions=actions, reward_lst=rewards))
        return eps

    def evaluate(self, agent, is_action_noise: bool, store_transition: bool) -> Episode:
        """Play one episode (agent.py:63-138) on the GPU."""
        f = self._fly(agent, 1, is_action_noise=is_action_noise, store_transition=store_transition, trace=True)
        return self._collect(agent, f, store_transition=store_transition, want_history=True)[0]

    def rl_to_evo(self, rl_agent, evo_net):
        for target_param, param in zip(evo_net.actor.parameters(), rl_agent.actor.parameters()):
            target_param.data.copy_(param.data)
        evo_net.buffer.reset()
        evo_net.buffer.add_content_of(rl_agent.buffer)
        evo_net.critical_buffer.reset()
        evo_net.critical_buffer.add_content_of(rl_agent.critical_buffer)

    def evo_to_rl(self, rl_net, evo_net):
        for target_param, param in zip(rl_net.parameters(), evo_net.parameters()):
            target_param.data.copy_(param.data)

    def _rl_prologue(self) -> bool:
        """train_rl's preamble: False while the buffer holds at most learn_start transitions; else the actor is put in
        training mode and, with use_champion_target, the champion's weights become the actor target"""
        if len(self.replay_buffer) <= self.args.learn_start:
            return False
        self.rl_agent.actor.train()
        if self.args.use_champion_target and self.champion_actor is not None:
            self.evo_to_rl(self.rl_agent.actor_target, self.champion_actor)
        return True

    def train_rl(self, rl_transitions: int) -> Dict[str, float]:
        pgs_obj, TD_loss = [], []
        if self._rl_prologue():
            if getattr(self.args, 'fused_td3', False):
                return self._train_rl_fused(int(rl_transitions * self.args.frac_frames_train))
            for _ in range(int(rl_transitions * self.args.frac_frames_train)):
                self.rl_iteration += 1
                batch = self.replay_buffer.sample(self.args.batch_size)
                pgl, TD, *delta = self.rl_agent.update_parameters(batch, self.rl_iteration, self.args.use_champion_target)
                if delta:                       # a prioritized batch: its rows get the step's TD errors
                    self.replay_buffer.update_priorities(batch[6], delta[0])
                if pgl is not None:
                    pgs_obj.append(-pgl)
                if TD is not None:
                    TD_loss.append(TD)
        return {'PG_obj': np.mean(pgs_obj) if pgs_obj else float('nan'), 'TD_loss': np.median(TD_loss) if TD_loss else float('nan')}

    def plan_rl_fused(self, rl_transitions: int):
        """the fused train_rl up to its K7 launch: None when the buffer is below learn_start, else the number of gradient
        steps n (0 or more) on global iterations rl_iteration + 1.. (the champion target is already in place)"""
        return int(rl_transitions * self.args.frac_frames_train) if self._rl_prologue() else None

    def finish_rl_fused(self, n, losses) -> Dict[str, float]:
        """the fused train_rl after its K7 launch: the statistics of the host losses [n, 2] and the iteration count"""
        if n is None or n <= 0:
            return {'PG_obj': float('nan'), 'TD_loss': float('nan')}
        first = self.rl_iteration + 1
        self.rl_iteration += n
        pg = losses[(np.arange(first, first + n) % self.args.policy_update_freq) == 0, 1]
        return {'PG_obj': np.mean(-pg) if pg.size else float('nan'), 'TD_loss': np.median(losses[:, 0])}

    def _train_rl_fused(self, n):
        """train_rl's loop as K7 launches; the statistics come from ONE device->host copy of the losses"""
        if n <= 0:
            return self.finish_rl_fused(n, None)
        losses = self.rl_agent.train_steps(self.replay_buffer, n, self.rl_iteration + 1, self.args.use_champion_target).cpu().numpy()
        return self.finish_rl_fused(n, losses)

    @staticmethod
    def _validation_stats(eps):
        scores = [np.sum(e.reward_lst) if not isinstance(e.reward_lst, _ReturnOnly) else e.reward_lst.total for e in eps]
        lengths = [e.length for e in eps]
        sms = [e.smoothness for e in eps]
        return (np.mean(scores), np.std(scores), np.mean(lengths), np.std(lengths), eps[-1], np.median(sms), np.std(sms))

    def validate_agent(self, agent):
        """agent.py:188-209: `validation_tests` episodes, none stored — flown as ONE launch of 5 trajectories."""
        f = self._fly(agent, self.validation_tests, trace=bool(self.args.should_log))
        return self._validation_stats(self._collect(agent, f, want_history=bool(self.args.should_log)))

    # ------------------------------------------------------------------------------------------------ generation
    def evaluate_population(self, sm_limit=0):
        """agent.py:229-245 as one fused launch: every actor x num_envs references.  Returns (pop_fitness f64[pop] numpy,
        device fitness, per-actor record matrix numpy [fitness, sum len, sum len^2, stored frames, sum sm, sum sm^2, has sm])
        — identical on every rank."""
        return self._finish_population(self._launch_population(sm_limit))

    def _n_envs(self):
        return int(getattr(self.args, 'num_envs', self.args.num_evals))

    def _want_population_smoothness(self):
        return bool(getattr(self.args, 'population_smoothness', False)) or bool(self.args.smooth_fitness)

    def _draw_population(self) -> _PopDraws:
        """the population's reference draws (population_draws; the host side of _launch_population)"""
        n_envs = self._n_envs()
        independent = bool(getattr(self.args, 'independent_references', False))
        draws = population_draws(self.env, len(self.pop), n_envs, independent)
        d = _PopDraws()
        d.levels, d.starts = np.stack([x[0] for x in draws]), np.stack([x[1] for x in draws])
        if independent:
            d.levels, d.starts = d.levels.reshape(len(self.pop), n_envs, 2, -1), d.starts.reshape(len(self.pop), n_envs, 2, -1)
        return d

    def _launch_population(self, sm_limit=0, draws=None):
        """the asynchronous half: reference draws (unless given), K0 + K1 (+ K6) and the per-actor record of this rank's shard,
        all queued on the current stream; nothing here waits for the device and nothing is stored yet.  Independent draws fly
        as per-actor env blocks, of which this rank passes its shard's rows."""
        draws = draws if draws is not None else self._draw_population()
        n_envs = self._n_envs()
        store = self.store_population_transitions
        world, rank = engine.world_info()
        pop = len(self.pop)
        lo, hi = engine.shard_bounds(pop, world, rank)
        if draws.levels.ndim == 4:
            lv, st = _to_device(draws.levels[lo:hi], self.device), _to_device(draws.starts[lo:hi], self.device)
            md = torch.full((hi - lo, n_envs), self.env.mode_code, dtype=torch.int32, device=self.device)
        else:
            lv, st = _to_device(draws.levels, self.device), _to_device(draws.starts, self.device)
            md = torch.full((n_envs,), self.env.mode_code, dtype=torch.int32, device=self.device)
        want_sm = self._want_population_smoothness()
        rec = torch.zeros((hi - lo, 7), dtype=torch.float64, device=self.device)
        r = None
        if hi > lo:
            r = rollout.population_rollout(self.pop.genomes[lo:hi], self.shape, lv, st, md, horizon=self._horizon(), actions=want_sm,
                                           replay_env=(n_envs - 1) if store else None, sm_limit=sm_limit, fitness=False,
                                           **self._eval_kw())
            sm_all = None
            if want_sm:
                sm_all = rollout.smoothness(r.actions, r.steps)
                r.actions = None
            rec = self._population_record(r, sm_all)
        return (r, rec, (lv, st, md))

    def _population_record(self, r, sm_all):
        """the per-actor record [fitness, sum len, sum len^2, stored frames, sum sm, sum sm^2, has sm] of the rollout result r
        (K6 smoothness sm_all, or None), queued on the current stream"""
        n_envs = r.returns.shape[1]
        rec = torch.zeros((r.returns.shape[0], 7), dtype=torch.float64, device=self.device)
        ret_p = r.returns + sm_all if self.args.smooth_fitness else r.returns
        stp = r.steps.to(torch.float64)
        rec[:, 0] = ret_p.mean(dim=1)                                     # fitness (agent.py:245)
        rec[:, 1] = stp.sum(1)                                            # episode-length statistics
        rec[:, 2] = (stp ** 2).sum(1)
        rec[:, 3] = stp[:, n_envs - 1]                                    # frames of the stored evaluation
        if sm_all is not None:
            rec[:, 4] = sm_all.sum(1)
            rec[:, 5] = (sm_all ** 2).sum(1)
            rec[:, 6] = 1.0
        return rec

    def _finish_population(self, launched):
        """the collecting half: all-gather of the record (and of the stored transitions), buffers, counters."""
        r, rec, _inputs = launched
        store = self.store_population_transitions
        world, rank = engine.world_info()
        pop = len(self.pop)
        horizon = self._horizon()
        rec_all = engine.gather_rows(rec, pop, world, rank)
        self._last_result = r
        if store:
            # the stored transitions of EVERY actor reach EVERY rank (identical shared / per-actor buffers on all ranks)
            cols = rollout.replay_cols(self.shape.state_dim, self.shape.action_dim)
            rows = r.replay if r is not None else torch.zeros((0, horizon, cols), dtype=torch.float32, device=self.device)
            rows_all = engine.gather_rows(rows.reshape(rows.shape[0], -1), pop, world, rank).reshape(pop, horizon, cols)
            steps_all = rec_all[:, 3].to(torch.int64)
            sel = torch.arange(horizon, device=self.device)[None, :] < steps_all[:, None]
            self.replay_buffer.add_rows(rows_all[sel])
            actors = torch.arange(pop, device=self.device)
            self.pop.buffers.append(actors, rows_all, sel)
            self.pop.critical_buffers.append(actors, rows_all, sel & (rows_all[..., rollout.transition_cols(self.shape.state_dim, self.shape.action_dim)] > 0.5))
        rec_host = rec_all.cpu().numpy()
        if r is not None:
            r.check()
        frames = int(rec_host[:, 3].sum())
        self.num_frames += frames
        self.gen_frames += frames
        self.num_episodes += pop
        return rec_host[:, 0].copy(), rec_all[:, 0].contiguous(), rec_host

    # A generation's FRONT: everything that can be queued before any of its results is needed.
    def _signature(self):
        """what the front of a generation read: a front launched ahead of time is only used if none of it changed."""
        env = self.env
        return (self.pop.genomes._version if len(self.pop) else 0,
                tuple(p._version for p in self.rl_agent.actor.parameters()),
                id(env), env.mode_code, float(env.t_max), int(getattr(self.args, 'num_envs', self.args.num_evals)), len(self.pop))

    def _launch_front(self, inputs=None):
        """queue a generation's front.  With defer_population the population's references are drawn at their place in the
        front (the np.random stream advances as without it) and its launch is left to launch_population_group.  `inputs`
        (checkpoint.front_inputs of a front launched earlier) re-launches that front from its host-side draws: the same
        launches on the same inputs, and no draw from the global streams."""
        args = self.args
        fr = _Front()
        fr.signature = self._signature()
        fr.pop_draws, fr.draws, fr.sm_limit = None, None, 0
        log = bool(args.should_log)
        given = inputs if inputs is not None else {}
        # RL exploration episode (agent.py:267-268): independent of the population -> side stream, launched first.  The RL
        # validation (:273-275) reads the RL actor AFTER train_rl; when no gradient step can happen it joins the side stream.
        fr.f_explore = self._fly(self.rl_agent, 1, is_action_noise=True, store_transition=True, trace=log, stream=self._side,
                                 draws=given.get('explore'), noise_state=given.get('noise_state'))
        fr.f_rlval = (self._fly(self.rl_agent, self.validation_tests, trace=log, stream=self._side2, draws=given.get('rlval'))
                      if args.frac_frames_train == 0 else None)
        fr.spec, fr.val_draws, fr.pop = {}, None, None
        if len(self.pop):
            # Speculative champion validation: the champion is only known after the ranking, and its 5 validation episodes
            # are ~0.15 s of serial latency.  The ranked elites of the previous generation survive unchanged (and so do
            # their protected clones), and one of the best of them usually wins again: their validation episodes are
            # launched NOW, next to the population rollout; a miss falls back to the serial launch.
            fr.val_draws = given['val_draws'] if inputs is not None else [self.env.draw_reference() for _ in range(self.validation_tests)]
            plan = getattr(self.evolver, 'last_plan', None)
            if plan is not None and self.speculative_validations > 0:
                for j, (o, c) in enumerate(list(zip(plan.elitist_index, plan.new_elitists))[:self.speculative_validations]):
                    fr.spec[o] = fr.spec[c] = self._fly(self.pop[o], self.validation_tests, trace=log,
                                                        stream=self._spec_streams[j], draws=fr.val_draws)
            # leave one SM per flight that can be in the air next to the rollout: exploration, RL validation, the previous
            # generation's champion validation, speculative validations
            fr.sm_limit = -(3 + len(fr.spec) // 2)
            fr.draws = given['pop_draws'] if inputs is not None else self._draw_population()
            if self.defer_population:
                fr.pop_draws = fr.draws
            else:
                fr.pop = self._launch_population(sm_limit=fr.sm_limit, draws=fr.draws)
        return fr

    def take_front(self):
        """the front this generation starts with: the one the previous train_tail queued if nothing it read has changed, else
        a new one.  train_head takes it itself unless the caller has (Sweep takes every run's front, then launches the
        deferred populations together)."""
        if self._front is None:
            fr, self._prefetched = self._prefetched, None
            if fr is not None and fr.signature != self._signature():
                fr = None              # the population / RL actor / environment changed since it was launched: fly again
            self._front_prefetched = fr is not None
            self._front = fr if fr is not None else self._launch_front()
        return self._front

    def train(self):
        """one generation (agent.py:211-315): its head (population, epoch, exploration episode), the RL half, its tail"""
        self.train_head()
        return self.train_tail(self.train_rl(self.gen_frames))

    def _lap(self, name):
        now = time.perf_counter()
        self.timing[name] = self.timing.get(name, 0.0) + 1e3 * (now - self._t_prev)
        self._t_prev = now

    def train_head(self):
        """a generation up to its RL half: the front's rollouts, the population's statistics and SSNE epoch, the champion's
        validation launch and the collected exploration episode.  The RL half (train_rl(self.gen_frames)) and train_tail
        follow; train() runs the three in order."""
        self.iterations += 1
        self.gen_frames = 0
        g = self._gen = _Generation()
        g.best_train_fitness = g.worst_train_fitness = g.population_avg = 1.
        g.sm = 1.
        g.sm_sd = g.elite_index = -1.
        g.ep_len_avg = g.ep_len_sd = 0.
        g.pop_fitness = None
        args = self.args
        self.timing = {}
        self._t_prev = time.perf_counter()
        lap, tm = self._lap, self.timing
        fr = self.take_front()
        self._front = None
        tm['front_prefetched'] = float(self._front_prefetched)
        if fr.pop_draws is not None:     # deferred, and no group launch took it: it flies alone
            fr.pop, fr.pop_draws = self._launch_population(fr.sm_limit, fr.pop_draws), None
        f_explore, g.f_rlval, spec, val_draws = fr.f_explore, fr.f_rlval, fr.spec, fr.val_draws
        lap('launch_front')
        g.f_champ = None
        if len(self.pop):
            pop_fitness, dev_fitness, rec = self._finish_population(fr.pop)
            g.pop_fitness = pop_fitness
            lap('evaluate_population')
            n_envs = int(getattr(args, 'num_envs', args.num_evals))
            n_ep = len(self.pop) * n_envs
            dt = self.env.dt
            mean_steps = rec[:, 1].sum() / n_ep
            g.ep_len_avg = mean_steps * dt
            g.ep_len_sd = float(np.sqrt(max(rec[:, 2].sum() / n_ep - mean_steps ** 2, 0.0))) * dt
            if rec[:, 6].any():                  # K6: per-episode action smoothness on the device (agent.py:242-243)
                g.sm = rec[:, 4].sum() / n_ep
                g.sm_sd = float(np.sqrt(max(rec[:, 5].sum() / n_ep - g.sm ** 2, 0.0)))
            else:
                g.sm, g.sm_sd = float('nan'), float('nan')
            g.best_train_fitness = np.max(pop_fitness)
            g.worst_train_fitness = np.min(pop_fitness)
            g.population_avg = np.average(pop_fitness)
            self.champion = self.pop[int(np.argmax(pop_fitness))]
            self.champion_actor = self.champion.actor
            # validate_agent(champion) (:255-258) on the side stream, from a COPY of its genome: the epoch below may mutate
            # the champion's own row (elites are protected as clones, mod_neuro_evo.py:494-505)
            ci = int(np.argmax(pop_fitness))
            if spec:
                self.spec_tries += 1
                self.spec_hits += ci in spec
            g.f_champ = spec.get(ci)
            if g.f_champ is None:
                g.f_champ = self._fly(self.champion, self.validation_tests, trace=bool(args.should_log), stream=self._champ,
                                      copy_genome=True, draws=val_draws)
            lap('stats')
            g.elite_index = self.evolver.epoch(self.pop, dev_fitness)
            lap('epoch')
        # RL half (agent.py:267-281)
        self._collect(self.rl_agent, f_explore, store_transition=True)
        lap('collect_exploration')

    def train_tail(self, rl_train_scores):
        """the rest of a generation after its RL half (train_rl's statistics): the RL validation, the actor injection, the
        next generation's front, the validation scores; returns train()'s statistics"""
        g, self._gen = self._gen, None
        args = self.args
        lap = self._lap
        lap('train_rl')
        test_score, test_sd, pop_novelty = 1., -1., -1.
        f_rlval, f_champ, pop_fitness, elite_index = g.f_rlval, g.f_champ, g.pop_fitness, g.elite_index
        ep_len_avg, ep_len_sd = g.ep_len_avg, g.ep_len_sd
        if f_rlval is None:
            f_rlval = self._fly(self.rl_agent, self.validation_tests, trace=bool(args.should_log), stream=self._side2)
        # actor injection (agent.py:283-294)
        if args.pop_size and self.iterations % args.rl_to_ea_synch_period == 0:
            replace_index = int(np.argmin(pop_fitness))
            if replace_index == elite_index:
                replace_index = (replace_index + 1) % len(self.pop)
            self.rl_to_evo(self.rl_agent, self.pop[replace_index])
            self.evolver.rl_policy = replace_index
        # Everything the NEXT generation can start without this generation's validation scores is queued now, so that the
        # validation episodes (serial latency, side streams) run next to the next population rollout instead of next to an
        # idle GPU.  The next train() picks the front up if population, RL actor and environment are unchanged.
        if self.prefetch_generation:
            self._prefetched = self._launch_front()
            lap('launch_next_front')
        rl_reward, rl_std, rl_ep_len, rl_ep_std, rl_episode, rl_sm, rl_sm_sd = self._validation_stats(
            self._collect(self.rl_agent, f_rlval, want_history=bool(args.should_log)))
        lap('rl_validation')
        if args.pop_size == 0:
            ep_len_avg, ep_len_sd = rl_ep_len, rl_ep_std
        if args.should_log:
            self.rl_history = rl_episode.get_history()
        if f_champ is not None:
            test_score, test_sd, _, _, last_episode, _, _ = self._validation_stats(
                self._collect(self.champion, f_champ, want_history=bool(args.should_log)))
            if args.should_log:
                self.champion_history = last_episode.get_history()
        lap('champion_validation')
        return {
            'best_train_fitness': g.best_train_fitness, 'test_score': test_score, 'test_sd': test_sd,
            'pop_avg': g.population_avg, 'pop_min': g.worst_train_fitness, 'elite_index': elite_index,
            'avg_smoothness': g.sm, 'smoothness_sd': g.sm_sd, 'rl_reward': rl_reward, 'rl_smoothness': rl_sm,
            'rl_smoothness_std': rl_sm_sd, 'rl_std': rl_std, 'avg_ep_len': ep_len_avg, 'ep_len_sd': ep_len_sd,
            'PG_obj': rl_train_scores['PG_obj'], 'TD_loss': rl_train_scores['TD_loss'], 'pop_novelty': pop_novelty,
        }

    def validate_agent_on(self, agent, draw) -> Episode:
        """one traced episode on a GIVEN reference (the champion's last validation episode, for its logged history)."""
        env = self.env
        lv = torch.as_tensor(draw[0][None], device=self.device)
        st = torch.as_tensor(draw[1][None], device=self.device)
        md = torch.tensor([env.mode_code], dtype=torch.int32, device=self.device)
        f = _Flight()
        f.levels, f.starts, f.n, f.noise_state, f.stream, f.keep = [draw[0]], [draw[1]], 1, None, None, None
        f.r = rollout.population_rollout(self._genome_of(agent), self.shape, lv, st, md, trace=True, horizon=self._horizon(),
                                         actions=True, **self._eval_kw())
        f.r.smoothness = rollout.smoothness(f.r.actions, f.r.steps)
        f.event = torch.cuda.Event()
        f.event.record()
        return self._collect(agent, f, want_history=True)[0]

    def save_checkpoint(self, path, extra=None) -> None:
        """write everything the next train() reads to `path` (serl_b200/checkpoint.py); `extra`: plain values kept with it"""
        from .. import checkpoint
        checkpoint.save(self, path, extra=extra)

    def load_checkpoint(self, path):
        """continue the run saved at `path` (this Agent must be built from the same Parameters and env); returns its `extra`"""
        from .. import checkpoint
        return checkpoint.load(self, path)

    def save_agent(self, parameters, elite_index: int = None) -> None:
        """agent.py:317-352: evo_nets.pkl ({'actor_i': state_dict}), elite_net.pkl, rl_net.pkl, state histories."""
        if len(self.pop):
            pop_dict = {f'actor_{i}': {k: v.detach().cpu().clone() for k, v in ind.actor.state_dict().items()}
                        for i, ind in enumerate(self.pop)}
            torch.save(pop_dict, os.path.join(parameters.save_foldername, 'evo_nets.pkl'))
            torch.save(pop_dict[f'actor_{int(elite_index)}'], os.path.join(parameters.save_foldername, 'elite_net.pkl'))
            if self.champion_history is not None:
                np.savetxt(os.path.join(parameters.save_foldername, 'statehistory_episode%d.txt' % self.num_episodes),
                           self.champion_history, header=str(self.num_episodes))
        torch.save({k: v.detach().cpu() for k, v in self.rl_agent.actor.state_dict().items()},
                   os.path.join(parameters.save_foldername, 'rl_net.pkl'))
        if self.rl_history is not None:
            np.savetxt(os.path.join(parameters.save_foldername, 'rl_statehistory_episode%d.txt' % self.num_episodes),
                       self.rl_history, header=str(self.num_episodes))


def stores_population_transitions(args):
    """the population's stored evaluations feed a buffer: the RL half trains, or proximal / safe mutation or the
    distillation crossover read the per-actor buffers"""
    return (args.frac_frames_train > 0 or getattr(args, 'mut_type', 'normal') in ('proximal', 'safe')
            or bool(getattr(args, 'distil_crossover', False)))


def population_key(args, env):
    """what runs must agree on to fly their populations in one launch (Sweep), None for a run without a population: actor
    shape, envs per actor, horizon and episode length, the gust flag, whether actions are recorded for the smoothness and
    whether transitions are stored.  Everything else (genomes, references, env mode) travels per actor."""
    if not args.pop_size:
        return None
    shape = (args.state_dim, args.action_dim, args.hidden_size, args.num_layers, args.activation_actor.lower())
    want_sm = bool(getattr(args, 'population_smoothness', False)) or bool(args.smooth_fitness)
    return (shape, int(getattr(args, 'num_envs', args.num_evals)), int(round(env.t_max / env.dt)) + 1, float(env.t_max),
            rollout.mode_gust(env.mode_code), want_sm, stores_population_transitions(args))


def launch_population_group(members):
    """ONE rollout launch for the deferred populations of several Agents on one device whose population_key agrees:
    members = [(agent, front)], each front holding its run's reference draws.  Every actor flies its own env block
    (SERL_ROLLOUT_PER_ACTOR_REFS): a run's shared draws repeat for each of its actors, independent ones are its actors'
    own.  Each front gets its slice of the result (returns, steps, replay rows, K6 smoothness) and its per-actor record,
    bit for bit what its own launch gives.  The launch has ONE status word: a non-finite trajectory in any run of it
    raises in every run that shares it.  A group of one flies alone, as Agent.train does."""
    a0, f0 = members[0]
    if len(members) == 1:
        f0.pop, f0.pop_draws = a0._launch_population(f0.sm_limit, f0.pop_draws), None
        return
    n_envs = a0._n_envs()
    blocks = lambda a, x: np.broadcast_to(x, (len(a.pop), n_envs) + x.shape[-2:])
    lv = _to_device(np.concatenate([blocks(a, f.pop_draws.levels) for a, f in members]), a0.device)
    st = _to_device(np.concatenate([blocks(a, f.pop_draws.starts) for a, f in members]), a0.device)
    md = _to_device(np.concatenate([np.full((len(a.pop), n_envs), a.env.mode_code, dtype=np.int32) for a, _ in members]), a0.device)
    genomes = torch.cat([a.pop.genomes for a, _ in members])
    want_sm = a0._want_population_smoothness()
    r = rollout.population_rollout(genomes, a0.shape, lv, st, md, horizon=a0._horizon(), actions=want_sm,
                                   replay_env=(n_envs - 1) if a0.store_population_transitions else None,
                                   sm_limit=min(f.sm_limit for _, f in members), fitness=False, **a0._eval_kw())
    sm_all = None
    if want_sm:
        sm_all = rollout.smoothness(r.actions, r.steps)        # one block per trajectory: the same bits in any batch
        r.actions = None
    lo = 0
    for a, f in members:
        hi = lo + len(a.pop)
        part = rollout.RolloutResult()
        part.returns, part.steps, part.status = r.returns[lo:hi], r.steps[lo:hi], r.status
        part.replay = r.replay[lo:hi] if r.replay is not None else None
        part.fitness = part.trace = part.actions = part.smoothness = part.track = None
        f.pop = (part, a._population_record(part, sm_all[lo:hi] if sm_all is not None else None), (lv, st, md, genomes))
        f.pop_draws = None
        lo = hi


def _to_device(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().to(device, non_blocking=True)


class _ReturnOnly:
    """reward list of an episode whose per-step record was not requested: only the sum is known."""

    def __init__(self, total):
        self.total = total

    def __len__(self):
        return 0


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False
