"""The population evaluation suite on the device: the tracking-error accumulators of K1 / K1-TC (serl_rollout_desc.d_track)
against the errors validate_agent rebuilds from a trace, evaluate_population against validate_agent called per actor and
condition, Sweep.evaluate, and examples/evaluate.py on a run directory."""
import os
import sys
import tomllib

import numpy as np
import pytest
import torch

from serl_b200 import _native, evaluation, rollout
from serl_b200.core.genetic_agent import Actor
from serl_b200.core.utils import calc_nMAE

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ACT = np.load(os.path.join(HERE, 'golden', 'actors.npz'))
DEV = torch.device('cuda:0')


class Args:
    state_dim, action_dim = 7, 3

    def __init__(self, hidden, layers, act):
        self.hidden_size, self.num_layers, self.activation_actor = hidden, layers, act


def random_genomes(n, hidden, layers, act, seed=0):
    torch.manual_seed(seed)
    return np.stack([Actor(Args(hidden, layers, act)).flat().detach().numpy() for _ in range(n)]).astype(np.float32)


# (genomes, shape, widths): K1 at h = 32, 72, 96 and K1-TC at [256] * 4 (the reference's Actor) and [400, 300]
CASES = {
    'k1_h32_relu': lambda: (ACT['serl50_pop8_h32_tanh'][:2], rollout.actor_shape(32, 3, 'relu'), None),
    'k1_h72_tanh': lambda: (ACT['serl10_pop_h72_tanh'][:2], rollout.actor_shape(72, 3, 'tanh'), None),
    'k1_h96_relu': lambda: (ACT['td3_h96_relu'][None], rollout.actor_shape(96, 3, 'relu'), None),
    'tc_256x4_relu': lambda: (random_genomes(2, 256, 3, 'relu'), rollout.actor_shape(256, 3, 'relu'), None),
    'tc_400_300_tanh': lambda: (wide_genomes([400, 300], 2), rollout.actor_shape(8, 1, 'tanh'), [400, 300]),
}
NOISELESS = ['nominal', 'low-q', 'high-q', 'be', 'jr', 'sa', 'se', 'cg', 'ice', 'cg-shift', 'test']


def wide_genomes(widths, n, seed=1):
    """width-list actors [w0, ..., w_{n-1}] in parameters() order (`shape` then supplies only the activation)"""
    from oracle import actor as A
    torch.manual_seed(seed)
    return np.stack([A.flatten(A.WideActor(widths)) for _ in range(n)]).astype(np.float32)


def launch(genomes, shape, widths, conds, refs, noise=None, **kw):
    envs = [evaluation.condition_env(c) for c in conds]
    codes = np.repeat([e.mode_code for e in envs], len(refs))
    lv, st = evaluation._ref_arrays(refs)
    md = torch.tensor(codes, dtype=torch.int32, device=DEV)
    r = rollout.population_rollout(torch.as_tensor(genomes, device=DEV).contiguous(), shape,
                                   torch.as_tensor(np.tile(lv, (len(conds), 1, 1)), device=DEV),
                                   torch.as_tensor(np.tile(st, (len(conds), 1, 1)), device=DEV), md, horizon=8001, t_max=80.0,
                                   smooth_width=8.0, env_order=rollout.variant_sorted_order(md), widths=widths,
                                   sensor_noise=None if noise is None else torch.as_tensor(noise, device=DEV),
                                   gust=any(rollout.mode_gust(int(c)) for c in codes), fitness=False, **kw)
    torch.cuda.synchronize()
    r.check()
    return r, envs


def host_sums(r, envs, n_refs, z=None):
    """validate_agent's errors (ref(t_k) rebuilt from the trace, minus env.x before the step) summed on the host"""
    steps, trace = r.steps.cpu().numpy(), r.trace.cpu().numpy()
    out = np.zeros(steps.shape + (4,))
    for a in range(steps.shape[0]):
        for j in range(steps.shape[1]):
            k = int(steps[a, j])
            tr = trace[a, j, :k]
            x_after = tr[:, rollout.TRACE_X]
            ref = tr[:, rollout.TRACE_ERR] + x_after[:, [7, 6, 5]]
            x_ic = rollout.initial_state(rollout.mode_variant(envs[j // n_refs].mode_code))
            x0 = evaluation.reset_state(x_ic, None if z is None else z[a, j, 0])
            if z is not None:
                assert np.abs(x0 - x_ic).max() > 1e-3        # reset()'s output carries the noise of call 0
            x_before = np.vstack((x0[None], x_after[:-1]))
            e = ref - x_before[:, [7, 6, 5]]
            out[a, j] = [np.abs(e[:, 0]).sum(), np.abs(e[:, 1]).sum(), np.abs(e[:, 2]).sum(), e[:, 2].sum()]
            assert evaluation.nmae_from_track(r.track[a, j].cpu().numpy()[None], [k])[0] == pytest.approx(calc_nMAE(e), rel=1e-12)
    return out


@pytest.mark.parametrize('case', sorted(CASES))
def test_track_equals_the_host_sums_of_validate_agent_errors(case):
    g, shape, widths = CASES[case]()
    np.random.seed(5)
    refs = evaluation.eval_refs(1)
    for conds, noisy in ((NOISELESS, False), (['noise', 'gust'], True)):
        z = np.random.RandomState(9).randn(g.shape[0], len(conds) * len(refs), 8002, 7).astype(np.float32) if noisy else None
        r, envs = launch(g, shape, widths, conds, refs, noise=z, trace=True, track=True)
        want = host_sums(r, envs, len(refs), z)
        got = r.track.cpu().numpy()
        assert np.all(np.abs(got - want) <= 1e-12 * np.abs(want) + 1e-300), (case, conds, np.abs(got - want).max())
        # tracking does not perturb the trajectories
        plain, _ = launch(g, shape, widths, conds, refs, noise=z)
        assert torch.equal(plain.returns, r.returns) and torch.equal(plain.steps, r.steps)


def test_track_survives_the_time_split_schedule():
    """300 actors x 13 envs are 300 tasks (13 envs: one warp per task).  At h = 72 a CTA holds at most two genome slots
    (rollout.cu: apc_max), so 64 SMs give at most 128 slots: K1 must split trajectories between slots and hand the sums
    over in the hand-over records, on any card.  Each actor must give the bits it gives in a 10-actor launch."""
    g = ACT['serl10_pop_h72_tanh']
    sms = 64
    assert 30 * g.shape[0] > 2 * sms
    np.random.seed(5)
    refs = evaluation.eval_refs(0)
    conds = NOISELESS + ['ice', 'nominal']
    small, _ = launch(g, rollout.actor_shape(72), None, conds, refs, track=True)
    big, _ = launch(np.tile(g, (30, 1)), rollout.actor_shape(72), None, conds, refs, track=True, sm_limit=sms)
    assert torch.equal(big.track, small.track.repeat(30, 1, 1))
    assert torch.equal(big.steps, small.steps.repeat(30, 1)) and torch.equal(big.returns, small.returns.repeat(30, 1))


def per_call(genomes, shape, conds, refs, num_trails):
    out = {}
    for c in conds:
        env = evaluation.condition_env(c)
        for a in range(genomes.shape[0]):
            out[a, c] = evaluation.validate_agent(genomes[a], shape, env, refs, num_trails)[1]
    return out


def test_evaluate_population_equals_validate_agent_per_actor_and_condition():
    g = ACT['serl10_pop_h72_tanh']
    shape = rollout.actor_shape(72)
    conds = list(evaluation.CONDITIONS)
    np.random.seed(7)
    refs = evaluation.eval_refs(2)
    state = np.random.get_state()
    want = per_call(g, shape, conds, refs, 2)
    lib = _native.lib()
    # launches of one rollout (K0 layout + K1) and of one K6 call
    md = torch.zeros(1, dtype=torch.int32, device=DEV)
    lv, st = evaluation._ref_arrays(refs[:1])
    c0 = lib.serl_launch_count()
    rollout.population_rollout(torch.as_tensor(g[:1], device=DEV), shape, torch.as_tensor(lv, device=DEV), torch.as_tensor(st, device=DEV),
                               md, horizon=10, fitness=False, track=True)
    c1 = lib.serl_launch_count()
    rollout.smoothness(torch.zeros((1, 8001, 3), device=DEV), torch.full((1,), 8001, dtype=torch.int32, device=DEV))   # 80 s: one DFT kernel
    c2 = lib.serl_launch_count()
    np.random.set_state(state)
    res = evaluation.evaluate_population(g, shape, conds, refs, 2)
    c3 = lib.serl_launch_count()
    assert c3 - c2 == 2 * (c1 - c0) + (c2 - c1)          # one rollout per sensor-noise group, one K6
    for (a, c), s in want.items():
        got = res.stats(a, c)
        assert got.nmae == pytest.approx(s.nmae, rel=1e-12) and got.nmae_sd == pytest.approx(s.nmae_sd, rel=1e-9, abs=1e-12), (a, c)
        assert abs(got.sm - s.sm) <= 2e-5 * abs(s.sm) + 1e-9, (a, c, got.sm, s.sm)
    for c in conds:
        nm = [want[a, c].nmae for a in range(10)]
        assert res.champion(c) == int(np.argmin(nm))
        assert res.average(c).nmae == pytest.approx(np.average(nm), rel=1e-12)
    # an actor-chunked run gives the same numbers
    np.random.set_state(state)
    per_actor = len(conds) * 3 * 8001 * 3 * 4
    chunked = evaluation.evaluate_population(g, shape, conds, refs, 2, actions_cap=3 * per_actor)
    assert np.array_equal(chunked.nmae_trials, res.nmae_trials) and np.array_equal(chunked.sm_trials, res.sm_trials)


def test_sweep_evaluate_splits_the_stacked_populations_back_per_run(tmp_path):
    """a Sweep of real Agents (two SERL runs of 4 and 6 actors, h = 72, and a TD3 run without a population), their
    populations overwritten with SERL10's actors: each run gets what evaluate_population gives its population alone"""
    import types
    from serl_b200.envs import config
    from serl_b200.parameters import Parameters
    from serl_b200.sweep import Sweep
    g = torch.as_tensor(ACT['serl10_pop_h72_tanh'], device=DEV)
    shape = rollout.actor_shape(72)

    def params(seed, pop_size):
        cwd = os.getcwd()
        os.chdir(tmp_path)
        try:
            p = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=seed, pop_size=pop_size, mut_type='normal',
                                                 test_ea=False, fused_td3=True))
        finally:
            os.chdir(cwd)
        p.save_foldername = str(tmp_path) + '/'
        p.state_dim, p.action_dim = 7, 3
        p.num_envs = p.num_evals = 2          # num_evals / smooth_fitness: Parameters sets them only with a population
        p.smooth_fitness = getattr(p, 'smooth_fitness', False)
        return p
    sw = Sweep([(params(s, n), config.select_env('PHlab_attitude_nominal')) for s, n in ((7, 4), (8, 6), (9, 0))])
    sw.runs[0].agent.pop.genomes.copy_(g[:4])
    sw.runs[1].agent.pop.genomes.copy_(g[4:])
    conds = ['nominal', 'be', 'noise']
    np.random.seed(3)
    refs = evaluation.eval_refs(1)
    state = np.random.get_state()
    got = sw.evaluate(conds, refs, 1)
    assert got[2] is None
    np.random.set_state(state)
    alone0 = evaluation.evaluate_population(g[:4], shape, conds, refs, 1)
    np.random.set_state(state)
    evaluation.sensor_noise_draws(4 * 2, 8001)          # the stacked call draws run 0's noise first
    alone1 = evaluation.evaluate_population(g[4:], shape, conds, refs, 1)
    for part, alone in zip(got[:2], (alone0, alone1)):
        assert np.array_equal(part.nmae_trials, alone.nmae_trials)
        assert np.allclose(part.sm_trials, alone.sm_trials, rtol=1e-12, atol=0)


def test_cli_eval_pop_all_conditions_saves_stats(tmp_path, monkeypatch):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'examples'))
    try:
        from test_eval_suite_population import write_run
        import evaluate as cli
    finally:
        del sys.path[:2]
    g = ACT['serl10_pop_h72_tanh']
    run = str(tmp_path / 'run')
    write_run(run, g, Args(72, 3, 'tanh'))
    monkeypatch.chdir(tmp_path)
    res = cli.main(['-agent_name', run, '-env', 'all', '-eval_pop', '-num_trails', '1', '-save_stats'])
    with open(os.path.join(run, 'stats.toml'), 'rb') as f:
        t = tomllib.load(f)
    assert sorted(t) == sorted(evaluation.CONDITIONS)
    for c in evaluation.CONDITIONS:
        rows = np.loadtxt(os.path.join(run, 'figures', c, 'final_performance.csv'), delimiter=',')
        ci = res.conditions.index(c)
        assert rows.shape == (10, 2) and np.array_equal(rows[:, 1], res.nmae[:, ci]) and np.array_equal(rows[:, 0], res.sm[:, ci])
        assert t[c]['champion_idx'] == res.champion(c) and t[c]['average']['nmae'] == res.average(c).nmae
    # every condition as base/evaluate.py run on it alone (seed 7, refs, then that condition's noise draws)
    for c in ('gust', 'noise', 'be'):
        np.random.seed(7)
        alone = evaluation.evaluate_population(g, rollout.actor_shape(72), [c], evaluation.eval_refs(1), 1)
        assert np.array_equal(alone.nmae_trials[:, 0], res.nmae_trials[:, res.conditions.index(c)]), c
    # -eval_rl -save_stats appends one table per condition; -save_trajectory writes the last trial's traces
    write_run(str(tmp_path / 'rl'), g[:1], Args(72, 3, 'tanh'), rl=g[3])
    rl = cli.main(['-agent_name', str(tmp_path / 'rl'), '-env', 'nominal,gust', '-eval_rl', '-save_stats', '-save_trajectory'])
    with open(os.path.join(tmp_path, 'rl', 'stats.toml'), 'rb') as f:
        t = tomllib.load(f)
    assert t == {c: rl[c]._asdict() for c in ('nominal', 'gust')}
    # actor 3 of the population run (without sensor noise: its draws there follow those of actors 0-2)
    assert abs(rl['nominal'].nmae - res.stats(3, 'nominal').nmae) <= 1e-12 * res.stats(3, 'nominal').nmae
    for c in ('nominal', 'gust'):
        tr = np.loadtxt(os.path.join(tmp_path, 'rl', 'figures', c, 'nominal_trajectory.csv'))
        assert tr.shape[1] == 19
