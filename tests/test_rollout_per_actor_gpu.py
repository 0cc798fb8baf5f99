"""Per-actor env blocks (SERL_ROLLOUT_PER_ACTOR_REFS) on the device, bit for bit: every actor of a per-actor launch gives what a
shared launch of that actor alone on its own block gives (K1 warp kernel, the one-thread-per-env kernel, K1-TC; mixed modes,
the gust build, sensor noise, the time-split schedule), the Agent's independent reference draws, and a Sweep whose
populations share one launch per group and generation."""
import os
import random
import types

import numpy as np
import pytest
import torch

from serl_b200 import _native, rollout
from serl_b200.core.genetic_agent import Actor

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ACT = np.load(os.path.join(HERE, 'golden', 'actors.npz'))
DEV = torch.device('cuda:0')
MODES = ['nominal', 'be', 'jr', 'sa', 'se', 'ice', 'cg', 'cg-timed']


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


# (genomes, shape, widths): K1 warp at h = 32, 72, 96, 128 (tables in shared memory at L = 2, in global memory at L = 3),
# the one-thread-per-env kernel (h = 141), K1-TC [400, 300] and [256] * 4
CASES = {
    'k1_h32': lambda: (ACT['serl50_pop8_h32_tanh'][:3], rollout.actor_shape(32, 3, 'tanh'), None),
    'k1_h72': lambda: (ACT['serl10_pop_h72_tanh'][:3], rollout.actor_shape(72, 3, 'tanh'), None),
    'k1_h96': lambda: (np.stack([ACT['td3_h96_relu']] * 2 + [random_genomes(1, 96, 3, 'relu')[0]]), rollout.actor_shape(96, 3, 'relu'), None),
    'k1_h128_tabs_shared': lambda: (random_genomes(3, 128, 2, 'elu'), rollout.actor_shape(128, 2, 'elu'), None),
    'k1_h128_tabs_global': lambda: (random_genomes(3, 128, 3, 'tanh'), rollout.actor_shape(128, 3, 'tanh'), None),
    'simple_h141': lambda: (random_genomes(3, 141, 1, 'tanh'), rollout.actor_shape(141, 1, 'tanh'), None),
    'tc_400_300': lambda: (wide_genomes([400, 300], 3), rollout.actor_shape(8, 1, 'tanh'), [400, 300]),
    'tc_256x4': lambda: (random_genomes(3, 256, 3, 'relu'), rollout.actor_shape(256, 3, 'relu'), None),
}


def blocks(pop, n_envs, seed, modes=MODES, t_max=20):
    """per-actor env blocks: levels / starts [pop, n_envs, 2, 6] f64 and mode codes [pop, n_envs] drawn from `modes`"""
    from oracle import refsig
    lv, st = refsig.make_ref_params(pop * n_envs, seed_base=seed, t_max=t_max)
    rs = np.random.RandomState(seed)
    md = np.array([rollout.mode_code(m) for m in rs.choice(modes, pop * n_envs)], dtype=np.int32)
    return lv.reshape(pop, n_envs, 2, 6), st.reshape(pop, n_envs, 2, 6), md.reshape(pop, n_envs)


def fly(g, shape, widths, lv, st, md, **kw):
    t = lambda x: torch.as_tensor(np.ascontiguousarray(x), device=DEV)
    r = rollout.population_rollout(t(g), shape, t(lv), t(st), t(md), widths=widths, fitness=False, **kw)
    torch.cuda.synchronize()
    r.check()
    return r


def written(r, f):
    """field f of result r with the rows the kernel does not write (steps past an episode's end) zeroed: actions and trace
    per trajectory, replay per actor (its stored env's steps)"""
    x = getattr(r, f).clone()
    k = torch.arange(x.shape[-2], device=x.device)
    n = r.steps[:, -1] if f == 'replay' else r.steps
    x[k >= n[..., None]] = 0
    return x


def outputs(r, fields):
    return {f: written(r, f) if f in ('actions', 'trace', 'replay') else getattr(r, f) for f in fields}


def assert_actor_equal(big, a, small, fields):
    x, y = outputs(big, fields), outputs(small, fields)
    for f in fields:
        assert torch.equal(x[f][a], y[f][0]), (f, a)


def per_actor_equals_solo(g, shape, widths, lv, st, md, noise=None, **kw):
    n_envs = md.shape[1]
    fields = ['returns', 'steps', 'actions', 'replay', 'trace']
    kw = dict(kw, actions=True, trace=True, replay_env=n_envs - 1)
    big = fly(g, shape, widths, lv, st, md, sensor_noise=None if noise is None else torch.as_tensor(noise, device=DEV), **kw)
    assert (big.steps > 0).all()
    for a in range(g.shape[0]):
        small = fly(g[a:a + 1], shape, widths, lv[a], st[a], md[a],
                    sensor_noise=None if noise is None else torch.as_tensor(noise[a:a + 1], device=DEV), **kw)
        assert_actor_equal(big, a, small, fields)
    return big


@pytest.mark.parametrize('case', sorted(CASES))
def test_per_actor_launch_equals_each_actor_alone_on_its_block(case):
    g, shape, widths = CASES[case]()
    lv, st, md = blocks(g.shape[0], 6, 1000 + len(case))
    big = per_actor_equals_solo(g, shape, widths, lv, st, md)
    # the blocks differ: actors that share a genome but not a block fly different trajectories
    assert not torch.equal(big.returns[0], fly(g[:1], shape, widths, lv[1], st[1], md[1]).returns[0])


@pytest.mark.parametrize('case', ['k1_h72', 'simple_h141', 'tc_400_300'])
def test_per_actor_gust_build_and_sensor_noise(case):
    """the gust instantiations (80 s episodes reach the 20-23 s pulse; 'gust' and 'test' envs among nominal and faulty
    ones) and per-trajectory sensor-noise draws"""
    g, shape, widths = CASES[case]()
    g = g[:2]
    lv, st, md = blocks(2, 4, 77, modes=['gust', 'test', 'nominal', 'be', 'cg-timed'], t_max=80)
    horizon = 8001
    noise = np.random.RandomState(3).randn(2, 4, horizon + 1, 7).astype(np.float32)
    per_actor_equals_solo(g, shape, widths, lv, st, md, noise=noise, horizon=horizon, t_max=80.0, smooth_width=13.0, gust=True)


def test_blocks_that_repeat_the_shared_rows_give_the_shared_launch():
    g, shape, _ = CASES['k1_h72']()
    lv, st, md = blocks(1, 8, 5)
    shared = fly(g, shape, None, lv[0], st[0], md[0], actions=True, replay_env=7)
    rep = lambda x: np.repeat(x, g.shape[0], axis=0)
    per = fly(g, shape, None, rep(lv), rep(st), rep(md), actions=True, replay_env=7)
    fields = ('returns', 'steps', 'actions', 'replay')
    x, y = outputs(per, fields), outputs(shared, fields)
    for f in fields:
        assert torch.equal(x[f], y[f]), f


def test_per_actor_blocks_survive_the_time_split_schedule():
    """300 actors x 13 envs on 64 SMs at h = 72 (at most 128 genome slots for 300 tasks): K1 splits trajectories between
    slots, and the slot that resumes one binds the actor's own row.  Actor a flies genome a % 10 on block a % 10, so every
    actor must give the bits of that actor in a 10-actor launch."""
    g = ACT['serl10_pop_h72_tanh']
    lv, st, md = blocks(10, 13, 31)
    kw = dict(actions=True, replay_env=12)
    small = fly(g, rollout.actor_shape(72), None, lv, st, md, **kw)
    tile = lambda x: np.tile(x, (30,) + (1,) * (x.ndim - 1))
    big = fly(tile(g), rollout.actor_shape(72), None, tile(lv), tile(st), tile(md), sm_limit=64, **kw)
    fields = ('returns', 'steps', 'actions', 'replay')
    x, y = outputs(big, fields), outputs(small, fields)
    for f in fields:
        assert torch.equal(x[f], y[f].repeat((30,) + (1,) * (y[f].dim() - 1))), f


# ------------------------------------------------------------------------------------------------------------- Agent
def _params(tmp_path, seed, **kw):
    from serl_b200.parameters import Parameters
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        p = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=seed, pop_size=kw.pop('pop_size', 4),
                                             mut_type='normal', test_ea=False, fused_td3=True))
    finally:
        os.chdir(cwd)
    p.save_foldername = str(tmp_path) + '/'
    p.state_dim, p.action_dim, p.hidden_size = 7, 3, 32
    p.num_envs = p.num_evals = 3
    p.learn_start, p.frac_frames_train = 300, 0.2
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _seeded_agent(p, env_name='PHlab_attitude_nominal'):
    from serl_b200.core import agent as agent_mod
    from serl_b200.envs import config
    env = config.select_env(env_name)
    env.seed(p.seed)
    torch.manual_seed(p.seed)
    np.random.seed(p.seed)
    random.seed(p.seed)
    return agent_mod.Agent(p, env)


def test_agent_independent_references_equal_a_hand_made_per_actor_launch(tmp_path):
    from serl_b200.core import agent as agent_mod
    p = _params(tmp_path, 3, independent_references=True)
    ag = _seeded_agent(p)
    pop, n_envs = len(ag.pop), 3
    genomes = ag.pop.genomes.clone()
    ag.gen_frames = 0
    state = np.random.get_state()
    fitness, _, rec = ag.evaluate_population()
    after = np.random.get_state()
    np.random.set_state(state)
    draws = agent_mod.population_draws(ag.env, pop, n_envs, True)
    assert np.array_equal(np.random.get_state()[1], after[1])
    lv = np.stack([d[0] for d in draws]).reshape(pop, n_envs, 2, 6)
    st = np.stack([d[1] for d in draws]).reshape(pop, n_envs, 2, 6)
    md = np.full((pop, n_envs), ag.env.mode_code, dtype=np.int32)
    hand = fly(genomes.cpu().numpy(), ag.shape, None, lv, st, md, replay_env=n_envs - 1)
    assert np.array_equal(fitness, hand.returns.mean(dim=1).cpu().numpy())
    assert np.array_equal(rec[:, 3], hand.steps[:, -1].cpu().numpy())
    rows, k = [], 0
    for a in range(pop):
        n = int(hand.steps[a, -1])
        mine = hand.replay[a, :n, :rollout.TRANSITION_COLS]
        assert torch.equal(ag.pop.buffers.rows_of(a), mine), a
        rows.append(mine)
        # actor a's stored rows are those of its OWN last draw
        last = fly(genomes[a:a + 1].cpu().numpy(), ag.shape, None, lv[a, -1:], st[a, -1:], md[a, -1:], replay_env=0)
        assert torch.equal(last.replay[0, :n], hand.replay[a, :n])
    assert torch.equal(ag.replay_buffer.data[:len(ag.replay_buffer)], torch.cat(rows))
    # the draws differ from actor to actor
    assert not np.array_equal(lv[0], lv[1])


# ------------------------------------------------------------------------------------------------------------- Sweep
def _snapshot(ag, stats):
    return dict(stats=stats, num_frames=ag.num_frames, rl_iteration=ag.rl_iteration, state=ag.rl_agent.state.clone(),
                genomes=ag.pop.genomes.clone() if len(ag.pop) else None,
                replay=ag.replay_buffer.data[:len(ag.replay_buffer)].clone())


def test_sweep_shares_one_population_launch_per_group_and_equals_solo_runs(tmp_path, monkeypatch):
    """3 runs of one launch group (different seeds; one with lr / CAPS changed; one on the `be` fault env, one with
    independent references) over 3 generations equal the same runs trained alone, and every generation makes one
    population rollout launch for the group"""
    from serl_b200.sweep import Sweep
    specs = [(7, dict(), 'PHlab_attitude_nominal'), (8, dict(lr=4e-4, use_caps=False), 'PHlab_attitude_nominal'),
             (9, dict(independent_references=True), 'PHlab_attitude_be')]
    gens = 3
    calls = []
    real = rollout.population_rollout

    def counting(weights, *a, **kw):
        if kw.get('replay_env') is not None and weights.shape[0] > 1:       # population launches (single-actor flights: pop 1)
            calls.append(weights.shape[0])
        return real(weights, *a, **kw)
    from serl_b200.core import agent as agent_mod
    monkeypatch.setattr(agent_mod.rollout, 'population_rollout', counting)
    from serl_b200.envs import config
    sw = Sweep([(_params(tmp_path, s, **dict(kw)), config.select_env(e)) for s, kw, e in specs])
    lib = _native.lib()
    swept = [[] for _ in specs]
    for g in range(gens):
        calls.clear()
        c0 = lib.serl_launch_count()
        for i, stats in enumerate(sw.train()):
            swept[i].append(_snapshot(sw.runs[i].agent, stats))
        torch.cuda.synchronize()
        # the heads' fronts (generation 1) or none (later: prefetched), and the tails' next fronts: one launch each
        assert calls == ([12, 12] if g == 0 else [12]), (g, calls)
        assert lib.serl_launch_count() > c0
    monkeypatch.setattr(agent_mod.rollout, 'population_rollout', real)
    for i, (seed, kw, e) in enumerate(specs):
        ag = _seeded_agent(_params(tmp_path, seed, **dict(kw)), e)
        for g in range(gens):
            a, b = swept[i][g], _snapshot(ag, ag.train())
            assert sorted(a['stats']) == sorted(b['stats'])
            for k in a['stats']:
                assert np.array_equal(np.asarray(a['stats'][k], dtype=np.float64), np.asarray(b['stats'][k], dtype=np.float64),
                                      equal_nan=True), (i, g, k)
            assert a['num_frames'] == b['num_frames'] and a['rl_iteration'] == b['rl_iteration'], (i, g)
            assert torch.equal(a['state'], b['state']), (i, g)
            assert torch.equal(a['replay'], b['replay']), (i, g)
            assert torch.equal(a['genomes'], b['genomes']), (i, g)
