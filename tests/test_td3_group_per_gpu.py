"""K7's group launch of prioritized and uniform learners (serl_td3_learn, td3_fused.train_group(prioritized=True))
and Sweep(per=True) on the GPU.  Every comparison is bitwise against the same learners or runs trained alone
(FusedTD3.run with and without its priority tree, Agent.train) from copies of the same initial state: the learner state,
the losses, the recorded draws (rows, target noise, CAPS uniforms, and for prioritized learners the weights and TD errors),
every double of every tree, the status words and the Adam step counts."""
import random

import numpy as np
import pytest
import torch

from test_td3_group_gpu import SPECS, _run_params, _same_stats, _snapshot, replay, synthetic_rows
from test_td3_mixed_gpu import learner
from test_td3_per_gpu import check_internal_nodes, per_buffer

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')

# prioritized learners that differ in everything: SPECS' fields (seed, lr, batch 32 / 86 / 128, n_steps 0 / 1 / hundreds,
# n_valid, champion target, CAPS, first iteration) plus the tree's capacity (powers of two and not), the replay row
# stride (19 / 20) and alpha / beta0 / beta_frames
PER = [dict(SPECS[0], per=True, cap=3001, stride=20, alpha=0.6, beta0=0.4, bf=1000.0),
       dict(SPECS[1], per=True, cap=1500, stride=19, alpha=1.0, beta0=0.0, bf=50.0),
       dict(SPECS[2], per=True, cap=128, stride=20, alpha=0.3, beta0=1.0, bf=1e6),
       dict(SPECS[3], per=True, cap=777, stride=20, alpha=0.6, beta0=0.4, bf=1e5),
       dict(SPECS[4], per=True, cap=4096, stride=19, alpha=0.8, beta0=0.2, bf=200.0),
       dict(SPECS[5], per=True, cap=700, stride=20, alpha=0.5, beta0=0.7, bf=3000.0)]
H72 = (72, 3, 'tanh')


def per_buf(spec):
    """spec's prioritized buffer: its n_valid rows in a tree of spec['cap'] leaves, priorities made uneven, rows of stride
    spec['stride']"""
    buf = per_buffer(synthetic_rows(spec['n_valid'], spec['seed']), seed=spec['seed'], capacity=spec['cap'])
    buf.prob_alpha, buf.beta_start, buf.beta_frames = spec['alpha'], spec['beta0'], spec['bf']
    if spec['stride'] == 20:          # the buffer's own rows are 19 wide: a 20-wide copy, read by its first 19 columns
        buf.data = torch.cat([buf.data, torch.zeros((buf.capacity, 1), device=DEV)], 1)
    assert buf.data.stride(0) == spec['stride']
    return buf


def source(spec):
    return per_buf(spec) if spec.get('per') else replay(spec)


def solo(specs, shapes, **kw):
    """each learner alone: FusedTD3.run, on its tree or uniformly"""
    out = []
    for s, sh in zip(specs, shapes):
        f, src = learner(s, sh, **kw), source(s)
        if s.get('per'):
            r = f.run(src.data, len(src), s['n'], s['first'], s['champ'], record=True, per=src)
        else:
            r = f.run(src, s['n_valid'], s['n'], s['first'], s['champ'], record=True)
        out.append((f, r, src if s.get('per') else None))
    torch.cuda.synchronize()
    return out


def grouped(specs, shapes, record=True, **kw):
    """the learners in train_group(prioritized=True); grouped.launches: the launches that call made (building the trees
    makes launches of its own)"""
    from serl_b200 import _native, td3_fused
    fs, srcs = [learner(s, sh, **kw) for s, sh in zip(specs, shapes)], [source(s) for s in specs]
    before = _native.lib().serl_launch_count()
    rs = td3_fused.train_group(fs, srcs, [s['n'] for s in specs], [s['first'] for s in specs], [s['champ'] for s in specs],
                               record=record, mixed_shapes=True, prioritized=True)
    grouped.launches = _native.lib().serl_launch_count() - before
    torch.cuda.synchronize()
    return [(f, r, src if s.get('per') else None) for f, r, src, s in zip(fs, rs, srcs, specs)]


def assert_same(a, b, record=True):
    (fa, ra, ba), (fb, rb, bb) = a, b
    assert torch.equal(fa.state, fb.state)
    assert torch.equal(ra.losses.nan_to_num(7.0), rb.losses.nan_to_num(7.0))
    if record:
        assert torch.equal(ra.indices, rb.indices) and torch.equal(ra.noise, rb.noise) and torch.equal(ra.caps, rb.caps)
    assert (ba is None) == (bb is None)
    if ba is not None:
        assert torch.equal(ba.tree, bb.tree)
        if record:
            assert torch.equal(ra.weights, rb.weights) and torch.equal(ra.td, rb.td)
    elif record:
        assert ra.weights is None and rb.weights is None and ra.td is None and rb.td is None
    assert int(ra.status.item()) == int(rb.status.item()) == 0
    assert (fa.critic_steps, fa.actor_steps) == (fb.critic_steps, fb.actor_steps)


def test_per_learners_that_differ_in_everything_equal_their_solo_runs():
    shapes = [H72] * len(PER)
    ref = solo(PER, shapes)
    assert all(torch.isfinite(r.losses[:, 0]).all() for _, r, _ in ref)
    got = grouped(PER, shapes)
    assert grouped.launches == 1
    for a, b in zip(ref, got):
        assert_same(a, b)
    # the learner with no steps and its tree are untouched; the others' trees were re-prioritised, and stay consistent
    assert torch.equal(got[3][0].state, learner(PER[3], H72).state) and torch.equal(got[3][2].tree, per_buf(PER[3]).tree)
    for f, r, b in got:
        check_internal_nodes(b.tree.view(-1, 2).cpu().numpy())
    assert not torch.equal(got[0][2].tree, per_buf(PER[0]).tree)


# prioritized and uniform learners, narrow and wide, at depths 3 and two more (1, 5); the wide ones take fewer steps
MIX_SHAPES = [H72, H72, (256, 3, 'elu'), (256, 3, 'relu'), (72, 1, 'relu'), (256, 5, 'tanh')]
MIX = [dict(PER[0], n=60), dict(SPECS[1], n=45), dict(PER[4], n=30), dict(SPECS[2]), dict(PER[5], n=40),
       dict(SPECS[4], n=17)]


def test_per_and_uniform_narrow_and_wide_in_one_launch():
    ref = solo(MIX, MIX_SHAPES)
    got = grouped(MIX, MIX_SHAPES)
    assert grouped.launches == 1
    for a, b in zip(ref, got):
        assert_same(a, b)


def test_uniform_only_group_equals_solo_runs():
    """no learner with a tree: the group takes the uniform learners' kernels, in one launch"""
    idx = [1, 3, 5]
    specs, shapes = [MIX[i] for i in idx], [MIX_SHAPES[i] for i in idx]
    ref = solo(specs, shapes)
    got = grouped(specs, shapes)
    assert grouped.launches == 1
    for a, b in zip(ref, got):
        assert_same(a, b)


def test_order_and_cluster_size_do_not_change_the_bits():
    ref = solo(MIX, MIX_SHAPES)
    perm = [3, 0, 5, 2, 4, 1]
    got = grouped([MIX[i] for i in perm], [MIX_SHAPES[i] for i in perm])
    for i, b in zip(perm, got):
        assert_same(ref[i], b)
    for cs in (1, 2, 4, 8):
        for a, b in zip(ref, grouped(MIX, MIX_SHAPES, cluster_size=cs)):
            assert_same(a, b)


def _many(k0, count):
    """count learners: prioritized and uniform alternately, narrow and wide, 1-3 steps each"""
    specs = [dict(PER[k % len(PER)] if k % 2 else SPECS[k % len(SPECS)], seed=100 + k, n=1 + k % 3) for k in range(k0, k0 + count)]
    shapes = [[H72, (256, 2, 'tanh'), (32, 1, 'elu')][k % 3] for k in range(k0, k0 + count)]
    return specs, shapes


def test_full_group_runs_in_waves_and_a_larger_one_is_chunked():
    from serl_b200 import _native
    G = _native.TD3_MAX_GROUP
    for count, launches in ((G, 1), (G + 6, 2)):
        specs, shapes = _many(0, count)
        got = grouped(specs, shapes, record=False, cluster_size=8)
        assert grouped.launches == launches
        sample = [0, 1, 3, 10, 29, 40, G - 1] + ([G, count - 1] if count > G else [])
        ref = solo([specs[k] for k in sample], [shapes[k] for k in sample], cluster_size=8)
        for k, a in zip(sample, ref):
            assert_same(a, got[k], record=False)


def test_launch_split_equals_one_launch(monkeypatch):
    from serl_b200 import td3_fused
    one = grouped(MIX, MIX_SHAPES)
    monkeypatch.setattr(td3_fused, 'LAUNCH_STEPS', 20)
    split = grouped(MIX, MIX_SHAPES)
    # chunks of 20 steps up to 60: learners with steps left per chunk 6, 4, 2 -> one launch each
    assert grouped.launches == 3
    for a, b in zip(one, split):
        assert_same(a, b)


def test_bad_index_in_one_learn_call_sets_only_its_learners_status():
    from serl_b200 import _native
    from serl_b200.td3_fused import FusedTD3
    specs = [dict(MIX[k], n=5) for k in (1, 0, 2)]           # uniform, prioritized (the bad one), prioritized wide
    shapes = [MIX_SHAPES[k] for k in (1, 0, 2)]
    fs, srcs = [learner(s, sh) for s, sh in zip(specs, shapes)], [source(s) for s in specs]
    descs, pers, rs = (_native.TD3Desc * 3)(), (_native.TD3PerDesc * 3)(), []
    bad = torch.zeros((5, specs[1]['batch']), dtype=torch.int32, device=DEV)
    bad[2, 7] = specs[1]['n_valid']                          # one past the valid rows
    for j, (f, s, src) in enumerate(zip(fs, specs, srcs)):
        rows = src.data if s.get('per') else src
        r = f._launch(5, False, per=s.get('per', False))
        rs.append(r)
        descs[j] = f._desc(rows, s['n_valid'], 5, s['first'], s['champ'], bad if j == 1 else None, r, 0)
        if s.get('per'):
            pers[j] = FusedTD3._per_desc(src, s['n_valid'], r, 0)
    _native.call('serl_td3_learn', descs, pers, 3, device=DEV)
    torch.cuda.synchronize()
    assert [int(r.status.item()) for r in rs] == [0, _native.TD3_STATUS_INDEX, 0]
    with pytest.raises(_native.NativeError):
        rs[1].check()


# ---------------------------------------------------------------------------------------------------------------- Sweep
# a prioritized and a uniform run at h = 72 (sharing one population launch) and a prioritized wide run
SWEEP_KWS = [dict(hidden_size=72, per=True), dict(hidden_size=72, lr=4e-4), dict(hidden_size=256, per=True, pop_size=0,
                                                                                   smooth_fitness=False)]
SWEEP_SEEDS = [7, 8, 9]


def _sweep(tmp_path):
    from serl_b200.envs import config
    from serl_b200.sweep import Sweep
    return Sweep([(_run_params(tmp_path, s, **dict(kw)), config.select_env('PHlab_attitude_nominal'))
                  for s, kw in zip(SWEEP_SEEDS, SWEEP_KWS)], mixed_shapes=True, per=True)


def _snap(ag, stats):
    s = _snapshot(ag, stats)
    s['tree'] = ag.replay_buffer.tree.clone() if getattr(ag.replay_buffer, 'tree', None) is not None else None
    s['steps'] = (ag.rl_agent.critic_steps, ag.rl_agent.actor_steps)
    return s


def _assert_same_snap(a, b, where):
    _same_stats(a['stats'], b['stats'])
    assert a['num_frames'] == b['num_frames'] and a['rl_iteration'] == b['rl_iteration'] and a['steps'] == b['steps'], where
    assert torch.equal(a['state'], b['state']), where
    assert torch.equal(a['replay'], b['replay']), where
    assert (a['genomes'] is None) == (b['genomes'] is None) and (a['tree'] is None) == (b['tree'] is None), where
    if a['genomes'] is not None:
        assert torch.equal(a['genomes'], b['genomes']), where
    if a['tree'] is not None:
        assert torch.equal(a['tree'], b['tree']), where


def test_per_sweep_runs_equal_the_same_runs_trained_alone(tmp_path):
    from serl_b200.core import agent as agent_mod
    from serl_b200.core.replay_memory import DevicePrioritizedReplayMemory
    from serl_b200.envs import config
    gens = 3
    random.seed(123); np.random.seed(123); torch.manual_seed(123)
    outer = (random.getstate(), np.random.get_state()[1].copy(), torch.get_rng_state())
    sw = _sweep(tmp_path)
    assert [isinstance(r.agent.replay_buffer, DevicePrioritizedReplayMemory) for r in sw.runs] == [True, False, True]
    swept = [[] for _ in SWEEP_SEEDS]
    for _ in range(gens):
        for i, st in enumerate(sw.train()):
            swept[i].append(_snap(sw.runs[i].agent, st))
    torch.cuda.synchronize()
    assert random.getstate() == outer[0] and np.array_equal(np.random.get_state()[1], outer[1])
    assert torch.equal(torch.get_rng_state(), outer[2])
    assert all(s[-1]['rl_iteration'] > 0 for s in swept)
    for i, (seed, kw) in enumerate(zip(SWEEP_SEEDS, SWEEP_KWS)):
        p = _run_params(tmp_path, seed, **dict(kw))
        env = config.select_env('PHlab_attitude_nominal')
        env.seed(p.seed)
        torch.manual_seed(p.seed)
        np.random.seed(p.seed)
        random.seed(p.seed)
        ag = agent_mod.Agent(p, env)
        for g in range(gens):
            _assert_same_snap(swept[i][g], _snap(ag, ag.train()), (i, g))


def test_per_sweep_resumes_from_a_checkpoint_bit_for_bit(tmp_path):
    sw = _sweep(tmp_path)
    for _ in range(2):
        sw.train()
    folder = str(tmp_path / 'ck')
    sw.save_checkpoint(folder)
    want = [_snap(r.agent, st) for r, st in zip(sw.runs, sw.train())]
    torch.cuda.synchronize()
    del sw
    fresh = _sweep(tmp_path)
    fresh.load_checkpoint(folder)
    got = [_snap(r.agent, st) for r, st in zip(fresh.runs, fresh.train())]
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(want, got)):
        _assert_same_snap(a, b, i)
