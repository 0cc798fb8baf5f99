"""K7 for learners of different actor shapes in one launch (serl_td3_learn, td3_fused.train_group(mixed_shapes=True))
and the mixed-shape sweep driver on the GPU.  Every comparison is bitwise against the same learners trained alone
(FusedTD3.run, Agent.train) from copies of the same initial state, as in test_td3_group_gpu.py."""
import random
import types

import numpy as np
import pytest
import torch

from test_td3_group_gpu import SPECS, _run_params, _same_stats, _snapshot, assert_same, replay

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')

# (hidden, num_layers, activation): both hidden classes, the class edges 128 / 129 and the widest actor
SHAPES = [(32, 1, 'tanh'), (72, 3, 'elu'), (128, 2, 'relu'), (129, 1, 'tanh'), (256, 3, 'elu'), (320, 2, 'tanh')]
# learners that differ in batch, n_steps (one of them 0), champion flag and CAPS besides their shapes (SPECS' fields);
# the wide ones take fewer steps to keep the test short
MIXED = [dict(SPECS[0], n=60), dict(SPECS[1], n=45), dict(SPECS[3]), dict(SPECS[2], n=7), dict(SPECS[4], n=30),
         dict(SPECS[5], n=17)]


def learner(spec, shape, cluster_size=0):
    """a FusedTD3 of `spec` with actor `shape`, its weights drawn from torch's CPU generator seeded with spec['seed']"""
    from serl_b200.td3_fused import FusedTD3
    h, L, act = shape
    args = types.SimpleNamespace(device=DEV, individual_bs=100, hidden_size=h, num_layers=L, activation_actor=act,
                                 state_dim=7, action_dim=3, lr=spec['lr'], gamma=spec['gamma'], tau=spec['tau'],
                                 noise_sd=spec['noise_sd'], noise_clip=0.5, policy_update_freq=spec['freq'], use_caps=spec['caps'],
                                 batch_size=spec['batch'], seed=spec['seed'])
    torch.manual_seed(spec['seed'])
    f = FusedTD3(args, cluster_size=cluster_size)
    f.critic_steps = spec['first'] - 1
    f.actor_steps = (spec['first'] - 1) // spec['freq']
    return f


def solo(specs, shapes, **kw):
    out = []
    for s, sh in zip(specs, shapes):
        f = learner(s, sh, **kw)
        r = f.run(replay(s), s['n_valid'], s['n'], s['first'], s['champ'], record=True)
        out.append((f, r))
    torch.cuda.synchronize()
    return out


def mixed(specs, shapes, record=True, **kw):
    from serl_b200 import td3_fused
    fs = [learner(s, sh, **kw) for s, sh in zip(specs, shapes)]
    rs = td3_fused.train_group(fs, [replay(s) for s in specs], [s['n'] for s in specs], [s['first'] for s in specs],
                               [s['champ'] for s in specs], record=record, mixed_shapes=True)
    torch.cuda.synchronize()
    return list(zip(fs, rs))


def test_mixed_group_equals_solo_runs_bit_for_bit():
    from serl_b200 import _native
    ref = solo(MIXED, SHAPES)
    assert all(torch.isfinite(r.losses[:, 0]).all() for _, r in ref)
    before = _native.lib().serl_launch_count()
    got = mixed(MIXED, SHAPES)
    assert _native.lib().serl_launch_count() - before == 1          # one launch for both hidden classes
    for a, b in zip(ref, got):
        assert_same(a, b)
    assert torch.equal(got[2][0].state, learner(MIXED[2], SHAPES[2]).state)     # no steps: untouched


def test_mixed_group_order_and_cluster_size_do_not_change_the_bits():
    ref = solo(MIXED, SHAPES)
    rev = mixed(MIXED[::-1], SHAPES[::-1])
    for a, b in zip(ref, rev[::-1]):
        assert_same(a, b)
    for cs in (2, 8):
        ref_cs = solo(MIXED, SHAPES, cluster_size=cs)
        for a, b, c in zip(ref, ref_cs, mixed(MIXED, SHAPES, cluster_size=cs)):
            assert_same(a, b)
            assert_same(a, c)


def test_one_class_groups_take_the_uniform_kernels():
    """a mixed group of narrow shapes only (and of wide shapes only) equals its solo runs too"""
    for idx in ([0, 1, 2], [3, 4, 5]):
        specs, shapes = [MIXED[i] for i in idx], [SHAPES[i] for i in idx]
        for a, b in zip(solo(specs, shapes), mixed(specs, shapes)):
            assert_same(a, b)


def test_full_mixed_group_runs_in_waves_and_matches():
    from serl_b200 import _native
    G = _native.TD3_MAX_GROUP
    specs = [dict(SPECS[k % len(SPECS)], seed=100 + k, n=1 + k % 3) for k in range(G)]
    shapes = [SHAPES[k % len(SHAPES)] for k in range(G)]
    got = mixed(specs, shapes, record=False, cluster_size=8)
    sample = [0, 3, 10, 29, 40, G - 1]
    ref = solo([specs[k] for k in sample], [shapes[k] for k in sample], cluster_size=8)
    for k, a in zip(sample, ref):
        assert_same(a, got[k], record=False)


def test_bad_index_in_one_learn_call_sets_only_its_learners_status():
    from serl_b200 import _native
    specs = [dict(MIXED[k], n=5) for k in (0, 4, 1)]
    shapes = [SHAPES[k] for k in (0, 4, 1)]
    fs = [learner(s, sh) for s, sh in zip(specs, shapes)]
    rs, descs = [], (_native.TD3Desc * 3)()
    rows = [replay(s) for s in specs]
    bad = torch.zeros((5, specs[1]['batch']), dtype=torch.int32, device=DEV)
    bad[2, 7] = specs[1]['n_valid']                       # one past the valid rows
    for j, (f, s) in enumerate(zip(fs, specs)):
        r = f._launch(5, False)
        rs.append(r)
        descs[j] = f._desc(rows[j], s['n_valid'], 5, s['first'], s['champ'], bad if j == 1 else None, r, 0)
    _native.call('serl_td3_learn', descs, None, 3, device=DEV)
    torch.cuda.synchronize()
    assert [int(r.status.item()) for r in rs] == [0, _native.TD3_STATUS_INDEX, 0]


def test_mixed_group_split_into_chunks_equals_one_launch(monkeypatch):
    from serl_b200 import _native, td3_fused
    one = mixed(MIXED, SHAPES)
    before = _native.lib().serl_launch_count()
    monkeypatch.setattr(td3_fused, 'LAUNCH_STEPS', 20)
    split = mixed(MIXED, SHAPES)
    # chunks of 20 steps up to 60: learners with steps left per chunk 5, 3, 2 -> one launch each
    assert _native.lib().serl_launch_count() - before == 3
    for a, b in zip(one, split):
        assert_same(a, b)


# ---------------------------------------------------------------------------------------------------------------- Sweep
def test_mixed_sweep_runs_equal_the_same_runs_trained_alone(tmp_path, monkeypatch):
    from serl_b200.core import agent as agent_mod
    from serl_b200.envs import config
    from serl_b200.sweep import Sweep
    # two (32, 3, tanh) runs sharing one population launch, (64, 1, elu), (144, 1, tanh) flown on K1-TC, and a wide TD3 run
    kws = [dict(), dict(lr=4e-4, use_caps=False), dict(hidden_size=64, num_layers=1, activation_actor='elu'),
           dict(hidden_size=144, num_layers=1), dict(hidden_size=160, num_layers=2, activation_actor='relu', pop_size=0,
                                                     smooth_fitness=False)]
    seeds = [7, 8, 9, 10, 11]
    gens = 3
    calls = []                     # per Sweep._launch_populations call: (hidden, runs, stream) of each group's launch
    real = agent_mod.launch_population_group

    def spy(members):
        calls[-1].append((members[0][0].args.hidden_size, len(members), torch.cuda.current_stream(DEV).cuda_stream))
        return real(members)
    monkeypatch.setattr(agent_mod, 'launch_population_group', spy)
    random.seed(123); np.random.seed(123); torch.manual_seed(123)
    outer = (random.getstate(), np.random.get_state()[1].copy(), torch.get_rng_state())
    cuda_rng = torch.cuda.get_rng_state()
    sw = Sweep([(_run_params(tmp_path, s, **dict(kw)), config.select_env('PHlab_attitude_nominal')) for s, kw in zip(seeds, kws)],
               mixed_shapes=True)
    launch_all = sw._launch_populations

    def batch(fronts):
        calls.append([])
        return launch_all(fronts)
    sw._launch_populations = batch
    swept = [[] for _ in seeds]
    for _ in range(gens):
        for i, st in enumerate(sw.train()):
            swept[i].append(_snapshot(sw.runs[i].agent, st))
    torch.cuda.synchronize()
    assert random.getstate() == outer[0] and np.array_equal(np.random.get_state()[1], outer[1])
    assert torch.equal(torch.get_rng_state(), outer[2])
    assert torch.equal(torch.cuda.get_rng_state(), cuda_rng)
    # one population launch per shape, the two 32-wide runs together; the first group's on the current stream, each
    # further group's on a stream of its own
    main = torch.cuda.current_stream(DEV).cuda_stream
    assert [(h, n) for h, n, _ in calls[0]] == [(32, 2), (64, 1), (144, 1)]
    for c in calls:
        assert len({s for _, _, s in c}) == len(c)
        assert not c or c[0][2] == main
    sw._launch_populations = launch_all
    assert all(s[-1]['rl_iteration'] > 0 for s in swept)
    monkeypatch.setattr(agent_mod, 'launch_population_group', real)
    for i, (seed, kw) in enumerate(zip(seeds, kws)):
        p = _run_params(tmp_path, seed, **dict(kw))
        env = config.select_env('PHlab_attitude_nominal')
        env.seed(p.seed)
        torch.manual_seed(p.seed)
        np.random.seed(p.seed)
        random.seed(p.seed)
        ag = agent_mod.Agent(p, env)
        for g in range(gens):
            a, b = swept[i][g], _snapshot(ag, ag.train())
            _same_stats(a['stats'], b['stats'])
            assert a['num_frames'] == b['num_frames'] and a['rl_iteration'] == b['rl_iteration'], (i, g)
            assert torch.equal(a['state'], b['state']), (i, g)
            assert torch.equal(a['replay'], b['replay']), (i, g)
            assert (a['genomes'] is None) == (b['genomes'] is None)
            if a['genomes'] is not None:
                assert torch.equal(a['genomes'], b['genomes']), (i, g)


def test_mixed_sweep_evaluate_runs_one_call_per_shape(tmp_path):
    """Sweep.evaluate over two shapes with a sensor-noise condition: each shape group's populations, stacked in run order,
    in one evaluate_population call, the calls in order of first appearance on one continued np.random stream"""
    from serl_b200 import evaluation
    from serl_b200.envs import config
    from serl_b200.sweep import Sweep
    kws = [dict(hidden_size=72), dict(hidden_size=32, activation_actor='elu'), dict(hidden_size=72, pop_size=3),
           dict(hidden_size=32, pop_size=0, smooth_fitness=False)]
    sw = Sweep([(_run_params(tmp_path, 7 + i, **dict(kw)), config.select_env('PHlab_attitude_nominal')) for i, kw in enumerate(kws)],
               mixed_shapes=True)
    conds = ['nominal', 'noise']
    np.random.seed(3)
    refs = evaluation.eval_refs(1)
    state = np.random.get_state()
    got = sw.evaluate(conds, refs, 1)
    after = np.random.get_state()[1].copy()
    assert got[3] is None
    np.random.set_state(state)
    pops = [r.agent.pop.genomes for r in sw.runs[:3]]
    a72 = evaluation.evaluate_population(torch.cat([pops[0], pops[2]]), sw.runs[0].agent.shape, conds, refs, 1)
    a32 = evaluation.evaluate_population(pops[1], sw.runs[1].agent.shape, conds, refs, 1)
    assert np.array_equal(np.random.get_state()[1], after)
    want = a72.split([4, 3]) + a32.split([4])
    for part, alone in zip([got[0], got[2], got[1]], [want[0], want[1], want[2]]):
        assert np.array_equal(part.nmae_trials, alone.nmae_trials)
        assert np.array_equal(part.sm_trials, alone.sm_trials)
